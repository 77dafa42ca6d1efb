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
#ifndef EF_K1A_PF_L2
#define EF_K1A_PF_L2 1           // K1a: prefetch.global.L2 128 bytes ahead of a slice's read position (besides the cp.async ring)
#endif
#ifndef EF_K1A_HDR_BATCH
#define EF_K1A_HDR_BATCH 24      // K1a: waiting lanes that end a symbol loop early (32: the loop runs until no lane is busy); 24 measured fastest of 8-32
#endif
#ifndef EF_K1A_V3
#define EF_K1A_V3 1              // K1a: one symbol per step through the clz-indexed table, a following end of block folded in (0: the two-symbol table step)
#endif
#ifndef EF_K1B_DEQUANT
#define EF_K1B_DEQUANT 0         // 1: K1a v3 stores raw tokens and K1b dequantises while it expands the list (measured: K1a -4 %, K1b +12 %: lost)
#endif
#ifndef EF_K1A_ES16
#define EF_K1A_ES16 1            // K1a: the bitstream comes in through 16-byte cp.async.cg chunks (4 per lane in flight) instead of 4-byte words: a quarter of the
#endif                           //      scattered-address global-memory instructions, and no reliance on L1 hits
#ifndef EF_K1A_UNROLL
#define EF_K1A_UNROLL 3          // K1a v3: symbol steps per pass of the loop (one vote + branch per pass)
#endif
#ifndef EF_PROBE_NOSTORE
#define EF_PROBE_NOSTORE 0       // measurement probe only: K1a drops its coefficient stores (output wrong)
#endif
#ifndef EF_K1A_RING_AHEAD
#define EF_K1A_RING_AHEAD 1      // K1a: the word after `lo` is already in a register when a refill needs it (its ring load was issued one refill earlier)
#endif
#ifndef EF_K1A_LUT_BITS
#if EF_K1A_V3
#define EF_K1A_LUT_BITS 0
#else
#define EF_K1A_LUT_BITS 10
#endif
#endif
// EF_K1A_LUT_BITS (EF_K1A_V3 = 0 only): the two-symbol coefficient table is indexed by the next 2^K bits of the stream
#ifndef EF_K1B_PIN16
#define EF_K1B_PIN16 1           // K1b: clamp two pixels per DPX instruction (VIADDMNMX.S16x2) instead of one
#endif
#ifndef EF_K1B_WARPS
#define EF_K1B_WARPS 7       // K1b (reconstruct): warps per CTA, CTAs per SM
#endif
#ifndef EF_K1B_CTAS
#define EF_K1B_CTAS 4
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
//   lut2: the fast path of the coefficient parser, indexed by the next EF_K1A_LUT_BITS bits: up to two
//         (run, level) symbols and a trailing end-of-block that lie wholly inside those bits.
//         .x = bits consumed | run1 << 8 | (int8) level1 << 16 | span << 24, span = scan positions advanced before
//              the last coefficient (run1, or run1 + 1 + run2); 127 = not decodable from these bits (long code,
//              escape, invalid): the parser then decodes one symbol through `dct`
//         .y = flags (1 first coefficient, 2 second coefficient, 4 end of block) | run2 << 8 | (int8) level2 << 16
//         [0] = dct_coeff_next context, [1] = first coefficient of a non-intra block   [2][2^K]  u32 x 2
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
    uint2 lut2[(2 << EF_K1A_LUT_BITS) > 16 ? (2 << EF_K1A_LUT_BITS) : 16];
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

// Per-stream audio state that one ef_decode_audio call hands to the next (ef_audio.cu). All zero = a fresh stream.
#define EF_AUDIO_CARRY 264       // most bytes one SBC frame's bit loader reads: header + scale factors 8 + 16 blocks x 128 bits
struct __align__(16) EfAudioState {
    int32_t frame_size;      // 0 not learned yet, > 0 learned by the probe, -1 / -2 first frame rejected / outside the domain
    int32_t carry_len;       // bytes held back: [0, EF_AUDIO_CARRY)
    int32_t i0, i1, i2;      // delta-sigma modulator of pdm_second_order()
    int32_t pad[3];
    int32_t sb[16][8];       // subband samples of the last accepted frame (a rejected frame re-synthesises them)
    int32_t vhist[9][16];    // V rows of the last 9 blocks (the window reaches 9 blocks back)
    uint8_t carry[EF_AUDIO_CARRY];
};

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
