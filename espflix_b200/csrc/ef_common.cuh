// espflix_b200/csrc/ef_common.cuh — shared device/host definitions of libespflix_b200.so.
//
// HBM layout (one context = one GPU):
//   es            [es_capacity + 64]            elementary streams of the current submit, back to back
//   es_off        [n_streams + 1]  u64          byte offset of each stream in `es`
//   frames        [n_streams][2][101,376]       the reference's two Frame stores per decoder
//                                               (video.h:36-44), MACROBLOCK-TILED on the device: tile
//                                               (mx,my) = 384 contiguous bytes at (my*22+mx)*384 =
//                                               Y[16][16], block-4 chroma [8][8], block-5 chroma [8][8].
//                                               One macroblock = 12 whole 32-byte sectors, so K1 never
//                                               writes a partial sector and a motion-compensated read
//                                               touches at most 4 tiles. ef_read_frame/ef_write_frame
//                                               convert to/from the reference's strip layout
//                                               (12 strips x 16 rows x 528 B, player.cpp:33-46).
//   seq           [n_streams][max_seq+1]        sequence-header state (quantiser matrices, mb_width/height);
//                                               entry 0 = state carried in from the previous submit
//   pics          [n_streams][max_pictures]     per picture: type, full_pel, r_size, seq index, first slice
//   slices        [n_streams][max_slices]       per slice: byte offset after its start code, slice code
//   work          [total slices]                flat per-picture slice work lists (K1a's unit of work)
//   mb_info/mb_rec[rec_pics][n_streams][264]    macroblock records K1a -> K1b, slot = macroblock address
//   coef          [3 x es bytes] u32            coefficient lists K1a -> K1b; the list of a slice starts at
//                                               entry 3 x (its byte offset in `es`); entry = (block << 24 |
//                                               raster position << 18) + dequantised, AAN-prescaled value
//   fields        [n_streams][field samples]    composite output of K2 (u16)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define EF_W 352
#define EF_H 192
#define EF_STRIDE 528
#define EF_FRAME 101376
#define EF_MBW_MAX 22
#define EF_MBH_MAX 12
#define EF_TILE 384          // bytes per macroblock tile: 256 Y + 64 + 64 chroma
#ifndef EF_K1A_THREADS
#define EF_K1A_THREADS 224   // K1a (parse): threads per CTA, CTAs per SM (28 warps per SM with 72 registers measured faster than 32 with 64)
#endif
#ifndef EF_K1A_CTAS
#define EF_K1A_CTAS 4
#endif
#ifndef EF_K1A_HDR_BATCH
#define EF_K1A_HDR_BATCH 24      // K1a: waiting lanes that end a symbol loop early (32: the loop runs until no lane is busy); 24 measured fastest of 8-32
#endif
#ifndef EF_K1A_UNROLL
#define EF_K1A_UNROLL 3          // K1a: symbol steps per pass of the loop (one vote + branch per pass)
#endif
#ifndef EF_K1B_WARPS
#define EF_K1B_WARPS 2       // K1b (reconstruct): warps per CTA, CTAs per SM. 30 warps per SM at 64 registers in small CTAs: of 7 x 4, 8 x 4, 16 x 2,
                             // 6 x 5, 5 x 6, 10 x 3, 4 x 7, 4 x 8, 3 x 10 and 2 x 15, measured fastest on the H100 (DESIGN.md 4)
#endif
#ifndef EF_K1B_CTAS
#define EF_K1B_CTAS 15
#endif

// ---- decode tables (built on the host by ef_tables.cpp from ISO 11172-2 Annex B) -------------
// All VLC tables are indexed by (leading zeros, next 5 bits) so that one CLZ + one shared-memory
// load decodes a symbol. Entry formats:
//   dct:  bits 0-4 code length INCLUDING the sign bit (0 = invalid), 5-9 run, 10-15 level. level 0 marks
//         the specials: length 2 = end of block ('10'), run 1 = escape. Rows 0-12 = dct_coeff_next context
//         ('10' / '11s' in row 0, row 12 all invalid for >= 12 leading zeros); rows 13-25 = the same for
//         the first coefficient of a non-intra block, where row 13 is '1s' = (0,1).           [26][32] u16
//   mba:  bits 0-3 length, 4-9 value (1..33, 34 stuffing, 35 escape)             [8][32]  u16
//   mv:   bits 0-3 length (sign included), 4-9 value+16                          [7][32]  u16
//   cbp:  bits 0-3 length, 4-9 pattern, indexed by the next 9 bits               [512]    u16
//   ptype:bits 0-2 length, 3-7 macroblock_type flags, indexed by next 6 bits     [64]     u8
//   qz:   per scan position n: quantiser byte | AAN prescale << 8 | raster index zig_zag[n] << 18; [0..63] intra,
//         [64..127] non-intra (the layout of a coefficient-list entry above bit 18)     [128]    u32
struct EfTables {
    uint16_t dct[26 * 32];
    uint16_t mba[8 * 32];
    uint16_t mv[7 * 32];
    uint16_t cbp[512];
    uint8_t ptype[64];
    uint8_t qdef[128];      // default quantiser matrices in SCAN order: [0..63] intra, [64..127] non-intra (all 16)
    uint16_t zp[64];        // scan position n -> zig_zag[n] | scale_dct_q[zig_zag[n]] << 8 (player.cpp:150-170)
    uint32_t qz[128];       // default matrices in the parser's combined form (see above)
    uint8_t izz[64];        // raster index -> zig-zag scan position
    uint8_t prescale[64];   // AAN prescale, raster (reference scale_dct_q, player.cpp:161)
    uint8_t zigzag[64];     // scan position -> raster index
};

// sequence state as the decode kernel reads it: quantiser matrices in SCAN order (the parser
// dequantises symbol by symbol), with quirk Q4 already applied: entry n = the byte the reference
// finds at raster index zigzag[n] of its stream-order copy (player.cpp:646-651, 1113), in the
// combined form of EfTables::qz (quantiser | prescale << 8 | raster index << 18).
struct __align__(16) EfSeq {
    uint32_t qz[128];        // [0..63] intra, [64..127] non-intra
    uint16_t mb_width, mb_height;
    uint16_t valid, custom;  // custom = a matrix was loaded from the stream (else K1 uses the shared-memory defaults)
    uint32_t fp_rs;          // full_pel_forward | forward_r_size << 1 of the last P picture header (decoder members in the reference: a B/D picture at the start of the next submit is parsed with them)
    uint32_t pad1;
};

struct __align__(16) EfPic {
    uint32_t first_slice;   // index into the stream's slice list
    uint32_t n_slices;
    uint16_t seq;           // index into the stream's EfSeq table (0 = state carried over from the previous submit)
    uint8_t type;           // picture_coding_type 1..4 (0 = none)
    uint8_t fp_rsize;       // bit0 full_pel_forward, bits1-3 forward_r_size, as slice() will see them
    uint32_t code_off;      // stream-relative offset of the picture start code's code byte (0x00), for the PTS latch
};

struct __align__(16) EfWork {   // one slice of one stream for one picture index
    uint32_t stream;
    uint32_t es_off;        // byte offset (relative to the stream start) of the first byte after the start code
    uint32_t info;          // bits0-7 slice code, 8-10 picture type, 11 full_pel, 12-14 r_size, 16-31 seq index
    uint32_t pic;           // picture index inside the submit
};

struct __align__(16) EfMbRec {  // one parsed macroblock (K1a -> K1b); its info word lives in EfDev::mb_info
    uint32_t cnt;           // coefficient entries | skipped macroblocks before this one << 16
    uint32_t mv;            // (int16 h) | (int16 v) << 16, half-pel units
    uint32_t list_lo, list_hi;   // index of the first entry in EfDev::coef
    int32_t dc[6];          // intra DC, pixel scale
    uint32_t pad[2];
};

struct EfGeometry {          // video.cpp:572-630, values probe-verified in tests/golden/composite_pins.json
    int ntsc, line_width, line_count, hsync, hsync_long, hsync_short, burst_start, burst_width, active_start;
    int active_top, vsync_start, blit_start;      // blit_start = active_start + 16 (+80 PAL)
};

struct EfPresent {           // presentation state of video_isr beyond the plain frame (video.cpp:839-887, 1146-1154)
    int hscroll;             // _hscroll: multiple of 8 in -344..344; negative scrolls in from the other side
    int blend;               // _video_composite_blend: 0 off, -1 or >= 32 full, 1..31 fading
    int progress;            // _video_composite_progress
    const uint8_t* bitmap;   // _video_composite[16][80]
};

struct EfDev {               // device-visible context (lives in device memory)
    int n_streams, max_pictures, max_slices, max_seq;
    const uint8_t* es;
    const uint64_t* es_off;
    uint8_t* frames;
    EfSeq* seq;              // [n_streams][max_seq + 1]
    EfPic* pics;             // [n_streams][max_pictures]
    uint32_t* slice_off;     // [n_streams][max_slices]
    uint8_t* slice_code;     // [n_streams][max_slices]
    uint32_t* n_pics;        // [n_streams] pictures in the current submit
    uint32_t* base_pics;     // [n_streams] pictures decoded before the current submit (ping-pong phase)
    uint32_t* n_seq;         // [n_streams] sequence headers seen in the current submit
    uint32_t* pic_pref;      // [max_pictures][n_streams] exclusive prefix of n_slices over streams
    uint32_t* pic_total;     // [max_pictures] slices of that picture index over all streams
    uint32_t* pic_base;      // [max_pictures] start of that picture's range in `work`
    uint32_t* cursor;        // [max_pictures] (kept for the index kernels)
    uint32_t* parse_cursor;  // work-stealing cursor of K1a, zeroed before every launch
    uint32_t* recon_cursor;  // [rec_pics] work cursors of the K1b launches, zeroed with it
    EfWork* work;            // flat, grouped by picture index
    uint32_t* info;          // [8]: 0 max pictures, 1 total pictures, 2 total slices, 3 error flags
    const EfTables* tables;
    uint32_t* mb_info;       // [rec_pics][n_streams][264] info word per macroblock slot (0 = nothing to rebuild), zeroed before every K1a launch
    EfMbRec* mb_rec;         // [rec_pics][n_streams][264]
    uint32_t* coef;          // [3 * (es_capacity + 1024)] coefficient entries
    int rec_pics;            // picture indices one K1a launch can cover
    uint16_t* fields;        // [n_streams][field_stride]
    const uint32_t* color_tab;   // [768]
    const int16_t* pal_burst;    // [2][64]
    size_t field_stride;     // samples
    size_t work_capacity;
    EfGeometry geo;
};

// TS submits cut at any packet boundary (ef_carry_enable): what K0 and the PTS resolve pass keep per stream between submits.
// A stream's region of a submit is its held bytes followed by the submit's new video ES.
#define EF_NO_PICTURE 0xFFFFFFFFu
struct EfCarryArgs {
    uint32_t* held;          // [n_streams] bytes held after the submit (the unfinished access unit; written by K0)
    uint32_t* held_code;     // [n_streams] offset of the held picture's code byte in the region, EF_NO_PICTURE when none
    uint8_t* flags;          // [n_streams] bit 0: held bytes exceeded max_carry (sticky until op 1, end of stream or ef_reset)
    const uint8_t* end;      // [n_streams] ef_end_streams flags of the submit
    const uint32_t* held_in; // [n_streams] bytes at the head of the region that the previous submit held
    int64_t* pts_hold;       // [n_streams] pts of the held picture, resolved over the bytes received so far
    int64_t* pts_pre;        // [n_streams] last valid PTS before the held bytes
    uint32_t max_carry;
};

// Per-stream audio state that one ef_decode_audio call hands to the next (ef_audio.cu). All zero = a fresh stream.
#define EF_SBC_MAX_BITPOOL 128   // 8 subbands x 16 bits: the bit allocation's slice loop cannot reach a larger pool (outside the domain)
#define EF_AUDIO_CARRY (8 + 2 * EF_SBC_MAX_BITPOOL)   // most bytes one SBC frame's bit loader reads (264): header + scale factors 8 + 16 blocks x 128 bits
struct __align__(16) EfAudioState {
    int32_t frame_size;      // 0 not learned yet, > 0 learned by the probe, -1 / -2 first frame rejected / outside the domain
    int32_t carry_len;       // bytes held back: [0, EF_AUDIO_CARRY)
    int32_t i0, i1, i2;      // delta-sigma modulator of pdm_second_order()
    int32_t synced;          // a frame was decoded: a probe that fails the sync byte re-synthesises sb (sbc_decoder.cpp:343-372)
    int32_t pad[2];
    int32_t sb[16][8];       // subband samples of the last accepted frame (a rejected frame re-synthesises them)
    int32_t vhist[9][16];    // V rows of the last 9 blocks (the window reaches 9 blocks back)
    uint8_t carry[EF_AUDIO_CARRY];
};

// Paced presentation (ef_present_*, ef_composite.cu): one stream's display under the instant-decoder model. Between calls
// nothing is pending (every push runs to its flip), so push_video's _next_frame / _next_frame_time and _animate need no
// slot; _hscroll is a function of _animate_index after every animate() call.
struct __align__(16) EfPaceState {
    uint32_t fc, line;           // position: _frame_counter of the field being drawn, next line to draw
    uint32_t pts_origin, fc_origin;   // _pts_origin, _video_frame_counter_origin (0 = latch at the next push)
    int32_t cur;                 // current frame store, -1 before the first flip
    int32_t ai;                  // _animate_index
    uint32_t flags;              // bit 0: a picture was not pushed (pts -1, mode 0): outside the domain
    uint32_t pad;
};
struct __align__(16) EfPaceRun {     // what one call emits for a stream: fields fc0, fc0 + 1, ... n of them
    uint32_t fc0;
    int32_t cur;                 // current frame store while they are drawn (-1: blank fields)
    int32_t ai;                  // _animate_index on the first one's active lines
    uint32_t n;
};
struct EfPaceOut {               // layout of ef_present_info (include/espflix_b200.h)
    uint64_t first;
    uint32_t n_fields, frame_counter, flip_field;
    int32_t flip_line, flags;
};
struct __align__(16) EfFieldDesc {   // one paced K2 field; its output slot is its index
    uint32_t stream;
    int32_t fb;                  // frame store, -2 = no frame presented yet
    uint32_t frame_counter;
    int32_t hscroll;
};
// The overlay of paced presentation (ef_present_overlay): composite()'s bitmap, blend and progress per stream (video.cpp:839-887).
// Staged changes wait in `pending` (the bitmap in slot ^ 1) and latch at line 0 of the first field that starts at or after the
// position where the next present call begins. A latched blend b > 0 counts down once per field end (video.cpp:1193-1194): field
// G shows max(0, b - (G - blend_fc)).
#define EF_OVERLAY_BYTES 1280    // _video_composite[16][80]
struct __align__(16) EfOverlayState {
    int32_t blend;               // latched _video_composite_blend
    uint32_t blend_fc;           // the field it was latched at
    int32_t progress;            // latched _video_composite_progress
    uint32_t slot;               // the stream's bitmap slot (0 / 1) the latched bitmap is in
    uint32_t pending;            // staged and not latched yet: bit 0 bitmap (in slot ^ 1), bit 1 p_blend, bit 2 p_progress
    int32_t p_blend, p_progress;
    uint32_t latch_fc;           // scratch copy of a call only: the field its staged changes latch at
};
struct __align__(16) EfOverlayCmd {  // one stream's change of one ef_present_overlay call
    int32_t blend, progress;
    uint32_t set;                // bit 0 bitmap, bit 1 blend, bit 2 progress
    uint32_t pad;
};
struct __align__(16) EfFieldOverlay {    // the overlay one paced K2 field is drawn with, beside its EfFieldDesc
    int32_t blend, progress;
    uint32_t slot, pad;
};
// The clock of paced presentation (ef_present_clock): ESPFlix::update_progress() (espflix.cpp:862-874) per stream, run at the start
// of every present call. It maps the stream's pts to the title's main timeline with the title's video.idx header (idx_hdr::pts2pts,
// espflix.cpp:589-604), redraws show_time()'s text into the overlay bitmap when the whole second changed and sets the progress; both
// are staged as ef_present_overlay stages them. seconds / draw are scratch of the call being made, committed (last_seconds and the
// bitmap slot) only once the call takes effect.
#define EF_FONT_W 1024           // _font8 atlas: 16 rows of 1024 columns
struct __align__(16) EfClockState {
    int64_t v_first, v_last;     // idx_hdr: video.first_pts, video.last_pts
    int64_t f_first, f_last;     // fwd.first_pts, fwd.last_pts
    int64_t r_first, r_last;     // rwd.first_pts, rwd.last_pts
    int32_t speed;               // _speed: 0 the title, 1 the fast-forward stream, -1 the rewind stream
    uint32_t flags;              // bit 0 on (_nav != -1), bit 1 paused (_state == PAUSED: the pause icon)
    int32_t last_seconds;        // _last_seconds
    int32_t seconds;             // scratch: the seconds the call shows
    uint32_t draw;               // scratch: the call rendered a new bitmap
    uint32_t pad[3];
};

// idx_hdr::pts2pts (espflix.cpp:589-604): a pts of the stream played at `speed` (0 the title, 1 the fast-forward stream, -1 the
// rewind stream) on the title's main timeline, from the video.idx records (first, last) of the main stream (v), fwd (f) and rwd (r).
// int64 throughout, truncating division; a trick record whose last_pts equals its first_pts divides by zero (callers refuse it).
static inline __host__ __device__ int64_t ef_pts2pts(int64_t pts, int speed, int64_t v_first, int64_t v_last, int64_t f_first, int64_t f_last,
                                                     int64_t r_first, int64_t r_last)
{
    if (speed == 1) return v_first + (pts - f_first) * (v_last - v_first) / (f_last - f_first);
    if (speed == -1) return v_last - (pts - r_first) * (v_last - v_first) / (r_last - r_first);
    return pts;
}

// The title library (ef_library_*, ef_library.cu): titles held in device memory and every stream's place in one of them.
// A title is its video.idx image and its transport streams: the three in the reference's _vid_names order (espflix.cpp:641),
// 0 video_rwd.ts, 1 video.ts, 2 video_fwd.ts, then 3 poster.ts (load_poster, espflix.cpp:1060-1069); a missing file has ts NULL
// and bytes 0. Stream states and commands: EF_LIB_* of include/espflix_b200.h.
#define EF_LIB_POSTER_FILE 3
struct __align__(16) EfLibTitle {
    const uint8_t* idx;          // the video.idx image: idx_hdr (104 bytes), then the main, fwd and rwd sample arrays (uint32)
    const uint8_t* ts[4];
    uint32_t bytes[4];           // file sizes, multiples of 188 below 4 GiB
    uint32_t idx_bytes;
    int64_t v_first, v_last, f_first, f_last, r_first, r_last;   // the header's records
    uint32_t v_bin, f_bin, r_bin, f_trick, r_trick, v_n, f_n, r_n;
};
struct __align__(16) EfLibStream {   // layout of ef_library_status (include/espflix_b200.h)
    int32_t title;               // -1 before the first PLAY_AT
    int32_t speed;               // _speed: -1, 0, 1
    int32_t state;               // EF_LIB_IDLE ... EF_LIB_POSTER
    int32_t file;                // speed + 1, or EF_LIB_POSTER_FILE: the file the cursor is in
    uint64_t cursor;             // byte offset of the next packet in that file
    int64_t pos;                 // _info[_nav].pos: the main pts the next PLAY, SKIP, FAST_FORWARD or REWIND starts from
};

// coded pictures (csrc/ef_encode.cu): an I picture's 28 header bytes (sequence, GOP and picture headers), a P picture's 9, and the
// slice region of one coded slice, the larger of two worst cases in whole words: an intra slice (start code + 6 bits + 22 macroblocks
// of 2 bits + 6 blocks of a 16-bit DC code, 63 28-bit escapes and the end of block) and a P slice (22 macroblocks of an 11-bit
// address increment, a 5-bit type, two 11-bit vector codes, a 9-bit pattern and 6 non-intra blocks of 64 28-bit escapes and the end
// of block; an intra macroblock's blocks are shorter). One output picture of the mux: its ES bytes, its first packet among all output
// packets, its pts and its file's continuity counter.
constexpr int kTrickHeaderBytes = 28;
constexpr int kTrickSliceBytes = 29736;
static_assert(kTrickSliceBytes >= ((32 + 6 + 22 * (2 + 6 * (16 + 63 * 28 + 2)) + 31) / 32) * 4, "worst-case I slice");
static_assert(kTrickSliceBytes >= ((32 + 6 + 22 * (11 + 5 + 2 * 11 + 9 + 6 * (64 * 28 + 2)) + 31) / 32) * 4, "worst-case P slice");
constexpr int kEncPHeaderBytes = 9;
// rate-controlled titles (ef_encode_build_rate): a picture's quantiser byte is q, or qmax | kQFallback for its fallback coding (P: every
// macroblock not coded; I: the DC levels alone); the census holds every slice's bytes at up to 31 candidates and the fallback in slot
// kCensusFallback
constexpr int kQFallback = 0x80;
constexpr int kCensusFallback = 31;
constexpr int64_t kRateUnit = 90000;       // bucket fullness is counted in 1/90000 bit, so that a refill R * pts_step is exact
// The I picture's share of a GOP's budget against one P picture's (tests/rate_cases.I_WEIGHT, where the measurement behind it is)
constexpr int kIWeight = 3;
struct EfRateBucket {
    int64_t full;                          // B * kRateUnit
    int64_t r;                             // min(R * pts_step, full): a refill beyond a full buffer changes no choice
    int64_t fb_p;                          // the P fallback's bits * kRateUnit
};
struct EfTrickPic {
    uint64_t es_off, pkt_first;
    int64_t pts;
    uint32_t es_len, cc0;
};

static inline __host__ __device__ int64_t ef_lib_pts2pts(const EfLibTitle& t, int64_t pts, int speed)
{
    return ef_pts2pts(pts, speed, t.v_first, t.v_last, t.f_first, t.f_last, t.r_first, t.r_last);
}

static inline __host__ __device__ int ef_overlay_blend(int32_t b, uint32_t blend_fc, uint32_t fc)
{
    const uint32_t d = fc - blend_fc;    // fields since the latch, modulo 2^32
    return b <= 0 ? b : d >= (uint32_t)b ? 0 : b - (int)d;
}

static inline __host__ __device__ size_t ef_frame_offset(int stream, int fb) { return ((size_t)stream * 2 + (size_t)fb) * EF_FRAME; }
static inline __host__ __device__ int ef_tile_offset(int mx, int my) { return (my * EF_MBW_MAX + mx) * EF_TILE; }
// byte offset inside a tiled frame of luma pixel (x,y) / of chroma plane p (0 = block 4, 1 = block 5) pixel (x,y)
static inline __host__ __device__ int ef_luma_offset(int x, int y) { return ef_tile_offset(x >> 4, y >> 4) + (y & 15) * 16 + (x & 15); }
static inline __host__ __device__ int ef_chroma_offset(int p, int x, int y) { return ef_tile_offset(x >> 3, y >> 3) + 256 + p * 64 + (y & 7) * 8 + (x & 7); }
// byte index in the I420 dump (Y rows, block-4 rows, block-5 rows) -> offset in the tiled frame
static inline __host__ __device__ int ef_i420_to_tiled(int b)
{
    if (b < EF_W * EF_H) return ef_luma_offset(b % EF_W, b / EF_W);
    const int c = b - EF_W * EF_H, plane = c / (176 * 96), r = c % (176 * 96);
    return ef_chroma_offset(plane, r % 176, r / 176);
}
// byte index in the reference's strip layout (12 contiguous strips of 16 x 528) -> offset in the tiled frame
static inline __host__ __device__ int ef_strips_to_tiled(int b)
{
    const int row = b / EF_STRIDE, x = b % EF_STRIDE;
    if (x < EF_W) return ef_luma_offset(x, row);
    const int r = row & 15;
    return ef_chroma_offset(r >> 3, x - EF_W, (row >> 4) * 8 + (r & 7));
}

// ---- 188-byte transport-stream packets and their PES headers (ISO 13818-1) ---------------------------------------------------------
// The 33-bit PTS of the 5 PTS bytes of a PES header (marker bits and prefix nibble ignored)
static inline __host__ __device__ int64_t ef_pts_decode(const uint8_t* q)
{
    return (int64_t)(q[0] & 0x0E) << 29 | (int64_t)q[1] << 22 | (int64_t)(q[2] >> 1) << 15 | (int64_t)q[3] << 7 | (q[4] >> 1);
}

// What one packet holds, read as more() / demux() read it (player.cpp:381-493), with no read outside its 188 bytes. It decides nothing:
// each caller applies its own rule to the fields (DESIGN.md §4, K0 index kernels).
struct EfTsPacket {
    bool sync, pusi, payload;      // sync byte 0x47, payload_unit_start, adaptation_field_control 1 or 3
    int pid;
    int pes;                       // the byte after the adaptation field (past the packet when the field runs past it)
    int start;                     // the first ES byte, 188 = none: pes, or on pusi the byte after the 9 + header_data_length PES bytes
    bool pts_prefix;               // pusi, PTS flag set, first PTS byte inside the packet and parse_pts()'s prefix nibble (player.cpp:299)
    int64_t pts;                   // the PTS when pts_prefix holds and all 5 of its bytes are inside the packet, else -1
};

static inline __host__ __device__ EfTsPacket ef_ts_read(const uint8_t* d)
{
    EfTsPacket r;
    r.sync = d[0] == 0x47;
    r.pusi = (d[1] & 0x40) != 0;
    r.payload = (d[3] & 0x10) != 0;
    r.pid = ((d[1] << 8) | d[2]) & 0x1FFF;
    r.pes = (d[3] & 0x20) ? 5 + d[4] : 4;
    r.start = r.pes < 188 ? r.pes : 188;
    r.pts_prefix = false;
    r.pts = -1;
    if (r.pusi) {                                              // the PES header: 9 bytes and header_data_length more
        const int o = r.pes, e = o + 9;
        r.start = 188;
        if (e <= 188) {
            const int flags = d[o + 7];                        // PTS_DTS_flags in bits 6-7
            if (e + d[o + 8] < 188) r.start = e + d[o + 8];
            r.pts_prefix = (flags & 0x80) && e < 188 && (d[e] & 0xF0) == ((flags >> 2) & 0x30);   // '0010' PTS only, '0011' with DTS
            if (r.pts_prefix && e + 5 <= 188) r.pts = ef_pts_decode(d + e);
        }
    }
    return r;
}

// Writes bytes first, first + step, ... of packet j of one PES in the muxes' layout (efs_wrap_ts's): the packet header with the
// continuity counter cc, the last packet's stuffing adaptation field, then the PES: a 14-byte header (stream_id, PES_packet_length
// `length`, flags 80 80 05 and the PTS with prefix '0010') and the n payload bytes, 184 PES bytes to a full packet. A warp writes a
// packet with first = lane and step = 32, the host with 0 and 1. The payload bytes take a loop of their own, which on the host is a
// plain copy: a test per byte made ef_mux_audio slower.
static inline __host__ __device__ void ef_pes_packet(uint8_t* pkt, uint32_t first, uint32_t step, uint32_t j, int pid, int stream_id,
                                                     uint32_t length, int64_t pts, uint32_t cc, const uint8_t* payload, uint32_t n)
{
    const uint32_t left = 14 + n - j * 184, af = left >= 184 ? 0 : 184 - left;    // adaptation field bytes, its length byte included
    const uint32_t p0 = (j ? 4 : 18) + af;                                          // the packet's first payload byte
    const uint64_t v = (uint64_t)pts;
    auto head = [&](uint32_t t) -> uint8_t {
        if (t == 0) return 0x47;
        if (t == 1) return (uint8_t)((j ? 0 : 0x40) | pid >> 8);
        if (t == 2) return (uint8_t)pid;
        if (t == 3) return (uint8_t)((af ? 0x30 : 0x10) | (cc & 15));
        if (t < 4 + af) return t == 4 ? (uint8_t)(af - 1) : t == 5 ? 0 : 0xFF;
        switch (t - 4 - af) {                                                       // the PES header, in packet 0
        case 2: return 1;
        case 3: return (uint8_t)stream_id;
        case 4: return (uint8_t)(length >> 8);
        case 5: return (uint8_t)length;
        case 6: case 7: return 0x80;
        case 8: return 5;
        case 9: return (uint8_t)(0x21 | ((v >> 29) & 0x0E));
        case 10: return (uint8_t)(v >> 22);
        case 11: return (uint8_t)(0x01 | ((v >> 14) & 0xFE));
        case 12: return (uint8_t)(v >> 7);
        case 13: return (uint8_t)(0x01 | ((v << 1) & 0xFE));
        default: return 0;
        }
    };
    uint32_t t = first;
    for (; t < p0; t += step) pkt[t] = head(t);
    for (; t < 188; t += step) pkt[t] = payload[j * 184 + t - 18 - af];
}

#ifdef __CUDACC__    // device code only: ef_tables.cpp reads this header through the host compiler
// Integer prefix sums over one CTA of a 1-D launch (lane = threadIdx.x & 31).
// Lane i of a full warp gets x_0 + ... + x_i; all 32 lanes must call it.
template <typename T>
__device__ __forceinline__ T ef_warp_inclusive_scan(T x)
{
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const T y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= d) x += y; }
    return x;
}

// The exclusive scan of a sequence longer than a CTA of kThreads threads, one tile of kThreads values at a time: thread t holds
// value base + t, and base steps by kThreads. Declare it __shared__. init() zeroes the carry (the sum of the tiles before);
// exclusive(v) returns the carry plus the v of the threads below the caller in this tile, then adds the tile's sum to the carry.
// Both end on a barrier, so `carry` may be read after either. Every thread of the CTA must call both, the same number of times:
// a thread past the end of the sequence passes 0. Four barriers per tile: warp totals written, warp totals scanned, the carry
// and the offsets read, the carry advanced.
template <typename T, int kThreads>
struct EfBlockScan {
    static_assert(kThreads % 32 == 0 && kThreads <= 1024, "whole warps, one CTA");
    T warp_sum[kThreads / 32];
    T carry;

    __device__ __forceinline__ void init()
    {
        if (threadIdx.x == 0) carry = 0;
        __syncthreads();
    }

    __device__ __forceinline__ T exclusive(T v)
    {
        constexpr int kWarps = kThreads / 32;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const T x = ef_warp_inclusive_scan(v);
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        // warp 0: the exclusive offsets of the warps. The vote makes the branch warp-uniform to the compiler; on `warp == 0` it
        // keeps a divergent fallback path for the shuffles, which costs registers (and spills in ef_audio_size_kernel).
        if (__all_sync(0xFFFFFFFFu, warp == 0)) {
            const T t = lane < kWarps ? warp_sum[lane] : T(0);
            const T z = ef_warp_inclusive_scan(t);
            if (lane < kWarps) warp_sum[lane] = z - t;
        }
        __syncthreads();
        const T excl = carry + warp_sum[warp] + x - v;
        __syncthreads();
        if (threadIdx.x == kThreads - 1) carry = excl + v;
        __syncthreads();
        return excl;
    }
};
#endif
