/* include/espflix_b200.h — C-ABI of libespflix_b200.so: the H100 drop-in for the espflix hot path
 * (MPEG-1 decode of a batch of independent 352x192 streams + NTSC/PAL composite synthesis).
 *
 * Plain C, plain pointers and sizes, no exceptions, no torch types. Every function returns
 * EF_OK (0) or a negative EF_E* code; ef_last_error() gives a text for the last failure on
 * the calling thread. A context owns all device memory for one GPU; calls on one context are
 * single-threaded (like the reference's one decoder thread, espflix.cpp:657). There is NO CPU
 * fallback: every entry point fails with EF_ECUDA if the CUDA device is missing.
 *
 * What each entry point replaces in the reference (paths relative to the reference's src/):
 *
 *   ef_create / ef_destroy        MpegDecoder::MpegDecoder(Frame*,Frame*) player.cpp:354 and the
 *                                 two Frame::init() calls (player.cpp:25) of espflix.cpp:651 -
 *                                 here for n_streams independent decoders at once
 *   ef_reset                      MpegDecoder::reset() player.cpp:439 (+ video_reset video.cpp:1076)
 *   ef_submit_es / ef_submit_ts   MpegDecoder::push_full(Buffer*) player.cpp:371 — the producer side
 *                                 of the Buffer queue (streamer.h:139); _ts takes the reference's wire
 *                                 format (188-byte TS, PID 0x100; demux of player.cpp:381-493), _es
 *                                 takes the video elementary stream the demux yields
 *   ef_index                      the start-code search of MpegDecoder::run() player.cpp:1360-1363 and
 *                                 the marker dispatch player.cpp:1318 for sequence/gop/picture headers
 *                                 (player.cpp:658-724), done once per submit for the whole batch
 *   ef_decode_picture             MpegDecoder::slice() player.cpp:1251 and everything under it
 *                                 (block/idct/mocomp/predict/copy_block..., player.cpp:733-1236) for
 *                                 picture #pic of every stream: one parse launch (slice/block: bitstream ->
 *                                 macroblock records) + one reconstruction launch (idct/mocomp/copy_block)
 *   ef_decode_all                 the for(;;) of MpegDecoder::run() player.cpp:1355 over one submit: every
 *                                 slice of every picture is parsed in ONE launch, then one reconstruction
 *                                 launch per picture index
 *   ef_decode_all_to_host         the same loop with the push_video() hand-over of every picture (video.h:49)
 *   ef_read_frame / _i420         what push_video(Frame*,front,pts,mode) video.h:49 hands to the
 *                                 display side: the striped Frame (video.h:36-44) of one stream
 *   ef_video_init                 video_init(int ntsc) video.cpp:572
 *   ef_composite_field            one field's worth of video_isr() calls video.cpp:1122 (sync, burst,
 *                                 blit video.cpp:690, blanking, vsync) for every stream: ONE launch
 *   ef_read_field / ef_video_isr  the uint16 line buffer video_isr(volatile void*) fills
 *   ef_blit                       blit(Frame*,uint16_t*,line,x,width) video.cpp:690
 *   ef_video_set_scroll / _overlay  _hscroll video.cpp:1146-1154, composite() video.cpp:839-887
 *   ef_tsidx_scan                 make_index(const string&, vector<idx>&) indexer/indexer.cpp:90
 *   ef_tsidx_samples              pts2seq(idx&,int,int) + pts2pos indexer/indexer.cpp:193-228
 *   ef_trick_build                the ffmpeg re-encodes of make_video() indexer/indexer.cpp:308-309: video_fwd.ts, video_rwd.ts
 *   ef_audio_demux_ts             MpegDecoder::demux() for the audio PIDs -> push_audio() player.cpp:381-432, video.cpp:1007
 *   ef_audio_decode               decode_audio() video.cpp:964, sbc_decoder() sbc_decoder.cpp:343, pdm_second_order()
 *                                 espflix.ino:73
 *   ef_audio_enable / ef_decode_audio  the same audio path fed by the context's TS submits, one submit at a time
 *   ef_decode_audio_async / ef_audio_wait  the same into device memory, returning before the decode is done: the
 *                                 reference's audio thread decoding on its own core beside video_isr (espflix.cpp:658)
 *   ef_pts_enable / ef_picture_pts     the pts push_video(frame, front, _last_pts, mode) hands over with every picture
 *                                 (flush_picture() player.cpp:692-702, latched from demux() player.cpp:399-419) and
 *                                 get_pts() player.cpp:653-656, for every stream of a TS submit
 *   ef_present_enable / _picture / _idle  push_video(frame, front, pts, mode) video.cpp:1023-1057 against the frame flip
 *                                 of video_isr video.cpp:1122-1198: every stream's paced composite fields, in HBM
 *   ef_present_*_async / ef_present_wait  the same, enqueued without waiting for the device
 *   ef_present_format             the paced fields as the DMA line buffer (uint16) or as the bytes the video DAC plays
 *   ef_present_overlay            composite() video.cpp:839-887 of every paced field: the overlay bitmap, blend and progress
 *   ef_present_font / _clock      ESPFlix::update_progress() espflix.cpp:862-874 with show_time() espflix.cpp:163-174: every
 *                                 stream's time text and progress drawn into its paced overlay on the device
 *   ef_restart_streams           MpegDecoder::reset() + video_reset() (player.cpp:439, video.cpp:1070) or video_pause(0)
 *                                 (video.cpp:1060) for chosen streams of the batch
 *   ef_carry_enable / ef_end_streams / ef_carry_info  the decoder pulling bytes on demand across the producer's Buffers
 *                                 (FILL_BITS -> more(), player.cpp:348-352, 459-493; espflix.cpp:723-737): TS submits cut at any
 *                                 packet boundary, and the len <= 0 Buffer that ends a stream (player.cpp:456, 469-473)
 *   ef_library_add / _command / _submit / _info / _add_trick  Streamer::get() + read() of a title (espflix.cpp:723-747) and ESPFlix's play, skip,
 *                                 fast_forward, rewind, play_pause, get_index and save_pos (espflix.cpp:787-859): titles in HBM, every
 *                                 stream's seek resolved from video.idx and its bytes gathered on the device
 *   ef_library_add_poster / _nv_read / _nv_write, EF_LIB_NAV / _NAV_STEP / _MENU  ESPFlix::nav(), menu() and load_poster()
 *                                 (espflix.cpp:704-720, 778-785, 1060-1069) and the NVS resume (espflix.cpp:851-859; espflix.ino:160-178):
 *                                 the poster menu, its scroll mode pushed on the device, and one saved position per title and stream
 * Calls run on the context's device and restore the caller's current device.
 */
#ifndef ESPFLIX_B200_H
#define ESPFLIX_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EF_OK        0
#define EF_EINVAL   (-1)   /* bad argument */
#define EF_ECUDA    (-2)   /* CUDA runtime error / no device (no CPU fallback exists) */
#define EF_ENOMEM   (-3)   /* a capacity given to ef_create was exceeded */
#define EF_ESTATE   (-4)   /* call out of order (e.g. decode before index) */

#define EF_FB_WIDTH    352           /* video.h:30 */
#define EF_FB_HEIGHT   192
#define EF_FB_STRIDE   528           /* video.h:32: 352 luma + 176 chroma per strip row */
#define EF_FB_STRIPS   12
#define EF_STRIP_BYTES 8448          /* 16 rows x 528 */
#define EF_FRAME_BYTES 101376        /* 12 strips back to back (host layout); the device keeps frames macroblock-tiled */
#define EF_I420_BYTES  101376
#define EF_NTSC_FIELD_SAMPLES (262 * 912)
#define EF_PAL_FIELD_SAMPLES  (312 * 1136)

typedef struct ef_ctx ef_ctx;

typedef struct {
    int device;                 /* CUDA device ordinal */
    int n_streams;              /* independent decoders in this context (1..65535) */
    int max_pictures;           /* per stream per submit */
    int max_slices_per_picture; /* per stream (reference accepts slice codes 1..12) */
    size_t es_capacity;         /* bytes of elementary stream per submit, whole batch */
    int fields;                 /* 1: allocate composite field buffers (n_streams x PAL field) */
} ef_config;

const char* ef_last_error(void);
const char* ef_version(void);

int ef_create(ef_ctx** out, const ef_config* cfg);
void ef_destroy(ef_ctx* ctx);
int ef_reset(ef_ctx* ctx);      /* zero frame stores, picture counters and sequence state */

/* Submit one batch. es/ts = all streams back to back; off[n_streams+1] = byte offsets of each
 * stream in it. The *_host forms copy from (pinned or pageable) host memory; *_device forms take
 * device pointers (inputs already resident in HBM). `stream` is a cudaStream_t (0 = default).
 * Each submit must hold whole pictures (cut at picture/sequence start codes), unless ef_carry_enable lets TS submits be cut at
 * any packet boundary. A submit is queued on an
 * internal upload stream into the back one of two device buffers and returns at once when the input is
 * pinned (or device) memory, so batch k+1 can be submitted while batch k is still being decoded; the
 * next ef_index() orders the compute stream after the upload. */
int ef_submit_es_host(ef_ctx* ctx, const uint8_t* es, const uint64_t* off, void* stream);
int ef_submit_es_device(ef_ctx* ctx, const uint8_t* es, const uint64_t* off, void* stream);
int ef_submit_ts_host(ef_ctx* ctx, const uint8_t* ts, const uint64_t* off, void* stream);
int ef_submit_ts_device(ef_ctx* ctx, const uint8_t* ts, const uint64_t* off, void* stream);

/* K0: start-code scan, header parse, per-picture slice work lists (device side, asynchronous). */
int ef_index(ef_ctx* ctx, void* stream);
/* Synchronising query of the last ef_index: max pictures in any stream, total pictures, total slices. */
int ef_index_info(ef_ctx* ctx, int* max_pictures, uint64_t* total_pictures, uint64_t* total_slices, uint64_t* es_bytes);
/* Per-stream picture count of the last submit and pictures decoded before it (host arrays, may be NULL). */
int ef_stream_info(ef_ctx* ctx, int stream_index, int* n_pictures, int* base_pictures);

/* K1: decode picture #pic (0-based within the submit) of every stream: one parse launch (K1a, bitstream ->
 * macroblock records) + one reconstruction launch (K1b). */
int ef_decode_picture(ef_ctx* ctx, int pic, void* stream);
/* All pictures 0..n_pictures-1 of the submit on `stream`: K1a parses every slice of all of them in ONE launch
 * (parsing needs no pixels), then K1b runs once per picture index. Prefer this over a loop of ef_decode_picture. */
int ef_decode_all(ef_ctx* ctx, int n_pictures, void* stream);
/* The same, handing EVERY picture to the host the way the reference's decoder hands every picture to push_video()
 * (video.h:49; player.cpp:692-702): after the K1b launch of picture index p the batch is exported as I420 and copied
 * to dst[p][stream] (n_pictures x n_streams x EF_FRAME_BYTES, should be pinned) on the context's read-back stream
 * while picture index p + 1 is rebuilt. layout 0 = I420, 1 = the reference's strips (video.h:36-44). Complete after
 * ef_sync. Streams with fewer pictures repeat stale data. */
int ef_decode_all_to_host(ef_ctx* ctx, int n_pictures, uint8_t* dst, int layout, void* stream);

/* Frame stores. fb = 0/1 is the reference's _fb[] index; -1 = the frame holding the most recently
 * decoded picture of that stream (what the next push_video would present). Synchronous. */
int ef_read_frame(ef_ctx* ctx, int stream_index, int fb, uint8_t* dst_strips /* EF_FRAME_BYTES */);
int ef_read_frame_i420(ef_ctx* ctx, int stream_index, int fb, uint8_t* dst /* EF_I420_BYTES */);
int ef_write_frame_i420(ef_ctx* ctx, int stream_index, int fb, const uint8_t* src);   /* tests / GUI-drawn frames */
int ef_write_frame(ef_ctx* ctx, int stream_index, int fb, const uint8_t* src_strips /* EF_FRAME_BYTES */);
/* Device address of a stream's frame store (for zero-copy consumers; macroblock-tiled: tile (mx,my) at
 * (my*22+mx)*384 = Y[16][16], block-4 chroma [8][8], block-5 chroma [8][8]); fb as above but not -1. */
int ef_frame_device_ptr(ef_ctx* ctx, int stream_index, int fb, void** ptr);
/* Batched read-back of the most recent picture of streams [first, first+count) as I420. The _async form
 * returns once the copy is queued (dst should be pinned; it is complete after ef_sync) so that it overlaps
 * the next submit/decode; the plain form waits for it. Which picture is "most recent" is frozen when the call is made;
 * the library orders the read against everything that writes a frame store afterwards (the next decode, ef_write_frame,
 * ef_reset). */
int ef_read_latest_i420(ef_ctx* ctx, int first, int count, uint8_t* dst, void* stream);
int ef_read_latest_i420_async(ef_ctx* ctx, int first, int count, uint8_t* dst, void* stream);
/* Wait for `stream` and for the context's internal upload / read-back streams. */
int ef_sync(ef_ctx* ctx, void* stream);

/* K2: composite synthesis. */
int ef_video_init(ef_ctx* ctx, int ntsc);                          /* 1 NTSC, 0 PAL */
int ef_video_geometry(ef_ctx* ctx, int* line_width, int* line_count);
/* One field for every stream from frame `fb` (-1 = most recent picture, -2 = no frame presented yet:
 * active lines come out as blank lines, the reference's _current_frame == -1 case, video.cpp:1140),
 * `frame_counter` = the reference's _frame_counter (dither phase), one launch. */
int ef_composite_field(ef_ctx* ctx, int fb, int frame_counter, void* stream);
/* Presentation extras of video_isr, applied by the next ef_composite_field calls (SURVEY.md 8f-2):
 * ef_video_set_scroll   the reference's _hscroll two-frame scroll (video.cpp:1146-1154): the other frame
 *                       store of each stream scrolls in; hscroll = multiple of 8 in (-352, 352), 0 = off.
 * ef_video_set_overlay  _video_composite / _video_composite_blend / _video_composite_progress
 *                       (video.cpp:839-887): 80x16 bitmap (may be NULL to keep the last one), blend 0 = off,
 *                       -1 or >= 32 = full, 1..31 = fading; progress 0..240. */
int ef_video_set_scroll(ef_ctx* ctx, int hscroll);
int ef_video_set_overlay(ef_ctx* ctx, const uint8_t* bitmap80x16, int blend, int progress);
int ef_read_field(ef_ctx* ctx, int stream_index, uint16_t* dst /* line_count*line_width */);
/* video_isr-style single line fetch from the last synthesised field of stream_index. */
int ef_video_isr(ef_ctx* ctx, int stream_index, int line, uint16_t* buf /* line_width */);
/* blit(): luma pixels x & ~3 .. of line (0..191) -> samples at dst (host). Like the reference loop (video.cpp:709) it
 * works in groups of 8 pixels: 2 * round_up(width, 8) samples are written, starting at dst + 80 under PAL (blit() itself
 * offsets its output there, video.cpp:698); (x & ~3) + round_up(width, 8) must not exceed 352. Synchronous. */
int ef_blit(ef_ctx* ctx, int stream_index, int fb, uint16_t* dst, int line, int x, int width, int frame_counter);

/* Pinned host memory for the asynchronous entry points (ef_submit_es_host, ef_read_latest_i420_async,
 * ef_decode_all_to_host) for callers that do not link the CUDA runtime themselves; the counterpart of the Buffers and
 * Frames the reference's decoder allocates for its caller (player.cpp:367-368; Frame::init player.cpp:25). */
int ef_host_alloc(void** ptr, size_t bytes);
void ef_host_free(void* ptr);
/* Launch counter: kernels this library has launched since ef_create (bench.py "gpu_launches"). */
uint64_t ef_launch_count(ef_ctx* ctx);
/* Stage timing, the counterpart of the reference's MEASURE() tick counters (player.cpp:1001, streamer.h): with
 * profiling on, ef_index and ef_decode_* bracket K0, K1a and the K1b launches with CUDA events on the caller's
 * stream; ef_stage_ms waits for and returns the durations of the LAST ef_index / last ef_decode_* range. */
int ef_set_profiling(ef_ctx* ctx, int on);
int ef_stage_ms(ef_ctx* ctx, float* index_ms, float* parse_ms, float* recon_ms);

/* ---- trick-mode index (SURVEY.md 8f-4): the reference's offline tool, indexer/indexer.cpp -------------------
 * Stateless (no context); host buffers; the scans run on `device`.
 * ef_tsidx_scan     make_index() (indexer.cpp:90-187) for n_files transport streams packed back to back
 *                   (off[n_files + 1], multiples of 188): the table of (PES pts, TS packet number) of the
 *                   video packets whose PES payload starts with a sequence header, first_pts (pts of the first,
 *                   -1 if none) and last_pts (pts of the last video PES start, -1 if none). The table of file f
 *                   is written at seq_pts/seq_pos[off[f] / 188 ...] (capacity = packets of the file).
 *                   info[f].n_samples = what pts2seq() will produce for bin_size.
 * ef_tsidx_samples  pts2seq() + pts2pos() (indexer.cpp:193-228): one uint32 packet number per bin_size ticks
 *                   from first_pts to last_pts, nearest table entry in pts (the reference's tie-breaking and its
 *                   int-cast distance). n_seq == 0 yields no samples (the reference indexes an empty vector). */
typedef struct { int64_t first_pts, last_pts; uint32_t n_seq, n_samples; } ef_tsidx_info;
int ef_tsidx_scan(int device, const uint8_t* ts, const uint64_t* off, int n_files, uint32_t bin_size,
                  ef_tsidx_info* info, int64_t* seq_pts, uint32_t* seq_pos);
int ef_tsidx_samples(int device, const int64_t* seq_pts, const uint32_t* seq_pos, int n_seq, int64_t first_pts, int64_t last_pts,
                     uint32_t bin_size, uint32_t* samples, uint32_t cap, uint32_t* n_samples);

/* ---- trick streams: the fwd / rwd half of the reference's indexer (indexer/indexer.cpp:308-309), without ffmpeg ---------------
 * Stateless (no context); host buffers; the decode, the encoder and the mux run on `device`. The rule, byte for byte, is
 * tests/trick_cases.py.
 * ef_trick_build  video_fwd.ts and video_rwd.ts of n_files mains packed back to back (off[n_files + 1], multiples of 188). Every
 *                 main is decoded as the reference decodes it, cut at its sequence headers into segments decoded as one batch. A
 *                 sequence header starts a segment only when its PES has a valid PTS, its first picture is intra and codes every
 *                 macroblock, and the next picture codes or skips every one (a host walk of their macroblocks); otherwise it joins
 *                 the segment before it, so each segment, decoded from cleared frame stores, gives a continuous decode's frames. fwd
 *                 picture k is main picture 15 k (the trick_speed merge_index writes), with pts p_0 + (p_15k - p_0) / 15 (a C
 *                 division; p_j = ef_picture_pts of main picture j); rwd holds the same pictures in reverse order with pts
 *                 f_0 + (f_{n-1} - f_{n-1-j}) (setpts=PTS/15 and -vf reverse). Every picture is one random-access point: a sequence
 *                 header (352 x 192, the aspect and picture-rate codes of the main's first one, default matrices), a closed GOP, an
 *                 I picture of 12 slices of intra macroblocks at quantiser scale qscale (1..31; 8 is the project's default). The
 *                 mux is efs_wrap_ts's: PID 0x100, one PES (stream id 0xE0, a PTS) per picture, the last packet of every PES
 *                 padded with adaptation-field stuffing, one continuity counter per file. No audio (the reference uses -an).
 *                 fwd_off / rwd_off[n_files + 1] receive the byte offsets of every file's output. A capacity below the total (or a
 *                 NULL buffer) returns EF_ENOMEM with both offset arrays filled and nothing written: a sizing call.
 *                 EF_EINVAL: qscale outside 1..31, offsets that are not non-decreasing multiples of 188, an empty main or one
 *                 without a sequence header at the start of a video PES (make_index()'s table), and a main with more than 4,096
 *                 pictures between two sequence headers that start a segment (or pictures of more than 16 slices).
 *                 Device memory: the mains' TS, their encoded pictures and output packets are held for the call, plus one decode
 *                 batch of at most 256 segments and 64 MB of TS and at most max(256, one batch's selected pictures) frames being
 *                 encoded: pass a catalogue in calls of a size the card holds. A too-small capacity is found only after the whole
 *                 build, so size the buffers generously (the mains' total is usually enough, but not at every qscale).
 * ef_trick_stage_ms  device milliseconds of the last ef_trick_build on the calling thread: the decode (upload, K0, K1a, K1b), the
 *                 gather of the selected frames, the encode (FDCT, quantiser, VLC and the picture assembly) and the mux. */
int ef_trick_build(int device, const uint8_t* ts, const uint64_t* off, int n_files, int qscale, uint8_t* fwd, uint64_t fwd_cap, uint64_t* fwd_off,
                   uint8_t* rwd, uint64_t rwd_cap, uint64_t* rwd_off);
int ef_trick_stage_ms(float* decode_ms, float* gather_ms, float* encode_ms, float* mux_ms);

/* ---- encoded titles: make_video()'s video step (indexer/indexer.cpp:306) without ffmpeg -----------------------------------------
 * Stateless (no context); host buffers; the encoder, its reconstruction and the mux run on `device`. The rule, byte for byte, is
 * tests/encode_cases.py.
 * ef_encode_build  video.ts of n_titles titles from raw pictures: i420 holds 352 x 192 I420 pictures (101,376 bytes each) back to
 *                  back in display order, title t being pictures pic_off[t] .. pic_off[t + 1] - 1. Every title is cut into GOPs of
 *                  p->gop pictures (the last may be shorter): a sequence header (352 x 192, p->aspect, p->rate, default matrices), a
 *                  closed GOP header and an I picture coded as ef_trick_build codes its pictures at p->qscale_i, then P pictures at
 *                  p->qscale_p predicted from the decoder's own reconstruction of the picture before them, with a full-pel search of
 *                  radius p->search (vectors stay inside forward_f_code 1's range, -8..7.5 pixels) and a half-pel refinement. Picture
 *                  k of a title has pts p->pts0 + k p->pts_step. The mux is ef_trick_build's: PID 0x100, one PES per picture, one
 *                  continuity counter per file; no audio. ts_off[n_titles + 1] receives the byte offsets of every title's output.
 *                  A capacity below the total (or a NULL ts) returns EF_ENOMEM with ts_off filled and nothing written: a sizing call.
 *                  EF_EINVAL: NULL arguments, gop outside 1..1024 (the temporal reference has 10 bits), a quantiser outside 1..31,
 *                  search outside 0..15, aspect outside 1..14, rate outside 1..8, an empty title, a pts outside 0..2^33 - 1.
 *                  Device memory: the encoded pictures and output packets of the whole call, plus one batch of at most 512 GOPs
 *                  and 6,144 source pictures (two frame stores and the slice regions of one picture per GOP, about 1.5 MB per GOP
 *                  of 12).
 * ef_encode_stage_ms  device milliseconds of the last ef_encode_build on the calling thread: the upload of the pictures, the tiling
 *                  and motion search, the coding (FDCT, quantiser, VLC, assembly), the reconstruction (submit, K0, K1a, K1b) and the mux. */
typedef struct {
    int gop;                     /* pictures per GOP, 1..1024 (12: ffmpeg's mpeg1video default) */
    int qscale_i, qscale_p;      /* 1..31: the slice quantiser of I and of P pictures */
    int search;                  /* full-pel search radius 0..15 */
    int aspect, rate;            /* sequence-header codes: aspect 1..14, picture_rate 1..8 */
    int64_t pts0;                /* pts of picture k of a title = pts0 + k * pts_step */
    uint32_t pts_step;
} ef_encode_params;
int ef_encode_build(int device, const uint8_t* i420, const uint64_t* pic_off, int n_titles, const ef_encode_params* p,
                    uint8_t* ts, uint64_t ts_cap, uint64_t* ts_off);
int ef_encode_stage_ms(float* upload_ms, float* search_ms, float* code_ms, float* recon_ms, float* mux_ms);

/* ---- encoded titles to a bit rate: make_video()'s "-b:v 1500k -maxrate 1500k -bufsize 0.25M -qmin 3" (indexer/indexer.cpp:307) --------
 * Stateless; host buffers. The rule, byte for byte, is tests/rate_cases.py.
 * ef_encode_build_rate  ef_encode_build with each picture's quantiser chosen on the device so that every GOP fits a leaky bucket of
 *                  rc->vbv_bits filled at rc->bit_rate: each GOP starts with a full buffer, no picture takes more bits than the buffer
 *                  holds, and every GOP but a title's last hands on a full buffer, so a player may start at any GOP after buffering
 *                  vbv_bits. The quantiser of picture j is the smallest of qmin..qmax whose exact coded size (a census of every
 *                  candidate, on the device) fits the picture's share of what the GOP may still spend and keeps the rest of the GOP
 *                  feasible; else the smallest that keeps it feasible; else a fallback (P: every macroblock not coded, a copy of the
 *                  reference picture; I: the DC levels alone) that always fits. p supplies gop, search, aspect, rate and the pts; its
 *                  qscale_i and qscale_p are not read. Every sequence header carries bit_rate = ceil(bit_rate / 400) and
 *                  vbv_buffer_size = ceil(vbv_bits / 16384), vbv_delay stays 0xFFFF (variable rate, bit_rate the peak); the audio is
 *                  not counted, as ffmpeg's -b:v does not count it. pic_q[i] (may be NULL) receives input picture i's quantiser, 0 for
 *                  a fallback, and pic_bytes[i] (may be NULL) its ES bytes; both are filled by a sizing call too.
 *                  ts, ts_cap, ts_off, the sizing call, the batch limits and the EF_EINVAL cases are ef_encode_build's, and further
 *                  EF_EINVAL: bit_rate outside 400 .. 400 * 0x3FFFE, vbv_bits outside 1 .. 1023 * 16384, not 1 <= qmin <= qmax <= 31,
 *                  or a bucket too small for any guarantee: the I fallback's worst case (3,592 bytes) does not fit a full GOP that must
 *                  end full. The census and the choice count in ef_encode_stage_ms's coding stage. */
typedef struct {
    uint32_t bit_rate;           /* bits per second, 400 .. 400 * 0x3FFFE (1,500,000: -b:v / -maxrate 1500k) */
    uint32_t vbv_bits;           /* the buffer, 1 .. 1023 * 16384 bits (250,000: -bufsize 0.25M) */
    int qmin, qmax;              /* the candidate quantisers, 1 <= qmin <= qmax <= 31 (3 .. 31: -qmin 3) */
} ef_rate_params;
int ef_encode_build_rate(int device, const uint8_t* i420, const uint64_t* pic_off, int n_titles, const ef_encode_params* p,
                         const ef_rate_params* rc, uint8_t* ts, uint64_t ts_cap, uint64_t* ts_off, uint8_t* pic_q, uint32_t* pic_bytes);

/* ---- encoded titles, audio: SBC from PCM and its interleave into video.ts ----------------------------------------------------------
 * The audio of the reference's make_video() (indexer/indexer.cpp:306-309: ffmpeg's "-codec:a sbc -ar 48000 -b:a 192k -ac 1
 * -streamid 1:258 -pes_payload_size 512"). Stateless; host buffers. The rule, byte for byte, is tests/sbc_encode_cases.py.
 * ef_sbc_encode   mono / 16-block / 8-subband SBC (the frames decode_audio() plays, video.cpp:964-986) of n_streams mono int16 PCM
 *                 streams at the header's rate, stream s being pcm[pcm_off[s] .. pcm_off[s + 1]): ceil(n / 128) frames of
 *                 8 + 2 p->bitpool bytes each (the bit allocation spends exactly the bit pool in every block), samples outside
 *                 the stream read as zero. The A2DP analysis filterbank in integers, gain 1 through the decoder's synthesis
 *                 (sbc_decoder.cpp:70-139), scale factors, the decoder's bit allocation (sbc_decoder.cpp:141-231), a quantiser that
 *                 never reaches IQUANT's 32-bit wrap (sbc_decoder.cpp:257), and the CRC-8 ffmpeg checks. Runs on `device`.
 *                 sbc_off[n_streams + 1] receives the byte offsets; a capacity below the total (or a NULL sbc) returns EF_ENOMEM
 *                 with sbc_off filled and nothing written. EF_EINVAL: NULL arguments, decreasing offsets, frequency outside 0..3,
 *                 allocation outside 0..1, bit pool outside 2..128.
 * ef_mux_audio    each title's video transport stream (ts_off[n_titles + 1], multiples of 188) with its SBC (sbc_off, whole frames
 *                 of p->bitpool) interleaved: PES of p->frames_per_pes frames (0: floor(512 / frame bytes), ffmpeg's
 *                 -pes_payload_size 512) on PID 0x102, stream_id 0xBD, a PTS on every one (player.cpp:423-432 plays audio only
 *                 after one), PES k at pts p->pts0 + floor(k frames_per_pes 128 90000 / fs); PES k goes right before the first
 *                 video PES start whose pts is >= its own, or at the end. Input packets keep their bytes and order. out_off
 *                 receives the offsets; EF_ENOMEM as above. EF_EINVAL: NULL arguments, offsets not multiples of 188, an input
 *                 packet on PID 0x101 / 0x102, a video PES start without a PTS, SBC that is not whole frames, frames_per_pes
 *                 outside 0..(65535 - 8) / frame bytes, an audio pts outside 0..2^33 - 1. The mux runs on the host: it moves every
 *                 byte once, between host buffers, and a device mux would add two host-link crossings of the whole file to that.
 * ef_audio_encode_stage_ms  milliseconds of the last ef_sbc_encode / ef_mux_audio on the calling thread: the upload of the PCM, the
 *                 encode kernel (filterbank, allocation, quantiser, packing), the download of the SBC (device events), and the
 *                 mux (host clock). */
typedef struct {
    int frequency;               /* header code 0..3: 16, 32, 44.1, 48 kHz (the PCM is taken at that rate; no resampling) */
    int allocation;              /* 0 loudness (ffmpeg's), 1 SNR */
    int bitpool;                 /* 2..128 */
    int frames_per_pes;          /* 0 = floor(512 / (8 + 2 bitpool)) */
    int64_t pts0;                /* pts of the first audio PES */
} ef_audio_params;
int ef_sbc_encode(int device, const int16_t* pcm, const uint64_t* pcm_off, int n_streams, const ef_audio_params* p,
                  uint8_t* sbc, uint64_t cap, uint64_t* sbc_off);
int ef_mux_audio(int device, const uint8_t* ts, const uint64_t* ts_off, const uint8_t* sbc, const uint64_t* sbc_off, int n_titles,
                 const ef_audio_params* p, uint8_t* out, uint64_t cap, uint64_t* out_off);
int ef_audio_encode_stage_ms(float* upload_ms, float* encode_ms, float* download_ms, float* mux_ms);

/* ---- audio (SURVEY.md 8f-3): the SBC decoder and the PDM modulator of the reference, batched ---------------------
 * Stateless (no context); host buffers; the kernels run on `device`.
 * ef_audio_demux_ts  MpegDecoder::demux() for PID 0x101 / 0x102 (src/player.cpp:381-432): the payload bytes that reach
 *                    push_audio() (video.cpp:1007) for n_files transport streams packed back to back (off[n_files + 1],
 *                    multiples of 188). A PES that starts without a (well-formed) PTS mutes its stream until the next
 *                    PES that has one. es_off[n_files + 1] receives the byte offsets of every file's audio in `es`.
 * ef_audio_decode    decode_audio() (video.cpp:964-986) + sbc_decoder() (sbc_decoder.cpp:343) + pdm_second_order()
 *                    (espflix.ino:73) for n_streams SBC byte streams (off[n_streams + 1]): the frame size is learned
 *                    from the first frame (which the reference decodes twice), whole frames are decoded in order to 128
 *                    int16 samples each at pcm + info[s].pcm_offset, and - when pdm is not NULL - every sample becomes
 *                    2 x 16 one-bit samples at pdm + 2 * pcm_offset (modulator state zero at the start of a stream).
 *                    pcm == NULL: sizing call, only info[] is filled. info[s].frame_size: > 0 bytes, 0 empty stream,
 *                    -1 first frame rejected by the reference (bad sync byte or 4 subbands; nothing decoded), -2 first
 *                    frame outside its domain (nothing decoded). The domain: mono, 8 subbands, 16 blocks, bit pool
 *                    <= 128; joint stereo (mode 3) is outside it. A later frame that the reference rejects or that is
 *                    outside the domain re-synthesises the previous accepted frame's samples. A 4-subband frame is the
 *                    one rejected frame whose output the reference leaves undefined (it emits uninitialised samples and
 *                    does not advance its filter; every later frame agrees with the re-synthesis). */
typedef struct { int32_t frame_size; uint32_t n_frames; uint64_t pcm_offset; } ef_audio_info;
int ef_audio_demux_ts(int device, const uint8_t* ts, const uint64_t* off, int n_files, uint8_t* es, uint64_t es_cap, uint64_t* es_off);
int ef_audio_decode(int device, const uint8_t* sbc, const uint64_t* off, int n_streams, ef_audio_info* info,
                    int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm);

/* ---- audio through a context: the same decode, continued submit after submit ------------------------------------
 * ef_audio_enable  from now on every ef_submit_ts_* of this context also demuxes PID 0x101 / 0x102 of every stream
 *                  (MpegDecoder::demux() -> push_audio(), player.cpp:381-432); the demux gate of a stream carries from
 *                  one submit to the next. Audio state lives in the context until ef_reset, which clears it and keeps
 *                  audio enabled. ES submits carry no audio.
 * ef_decode_audio  decode_audio() (video.cpp:964-986) + sbc_decoder() + pdm_second_order() for every stream, continuing
 *                  where the previous call stopped: consumes the audio of the TS submit the last ef_index made current,
 *                  appended to the bytes each stream still holds, and emits every frame that has become decodable (all
 *                  the bytes its bit loader reads are present). Output and info[] as ef_audio_decode: info[s].n_frames /
 *                  pcm_offset = this call's frames, frame_size = the stream's learned size or 0 / -1 / -2.
 *                  end_of_stream[n_streams] (may be NULL): the stream ends after this call; its held-back frames are
 *                  decoded as the whole-stream call decodes them, then its audio state and demux gate start over (also
 *                  for a TS submit already queued behind the current one). pcm == NULL: sizing call, fills info[] and
 *                  changes no state. pdm == NULL: no PDM, and the modulator state stays where it is. Synchronous.
 *                  Concatenated over the calls, PCM and PDM equal ef_audio_decode on the stream's whole audio.
 *                  Errors: EF_ESTATE before ef_audio_enable; EF_ENOMEM when pcm_cap is too small (state untouched).
 *                  On an audio-enabled context, ef_index of a new submit returns EF_ESTATE while the current TS submit's
 *                  audio has not been consumed; indexing the same submit again adds no audio. */
int ef_audio_enable(ef_ctx* ctx);
int ef_decode_audio(ef_ctx* ctx, const uint8_t* end_of_stream, ef_audio_info* info,
                    int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm, void* stream);

/* ef_decode_audio_async  the same decode as ef_decode_audio, with its output in device memory: info[n_streams], pcm[pcm_cap]
 *                  and pdm[2 * pcm_cap] (may be NULL) are device pointers. Every size is computed on the device and the call
 *                  returns once its work is enqueued on `stream`, without waiting for the device, so the decode runs beside
 *                  whatever the caller runs on other streams (paced presentation). info[] is written on the device, in stream
 *                  order, before the samples. Sync and async calls may be mixed in any order; concatenated, their output
 *                  equals ef_audio_decode on the whole stream.
 *                  Capacity is checked on the device: when the call's samples exceed pcm_cap, nothing is written but
 *                  info[] (the counts, so the call doubles as an asynchronous sizing call), no stream state changes,
 *                  end_of_stream has no effect, the submit's audio stays unconsumed, and ef_audio_wait returns EF_ENOMEM;
 *                  a call with a larger buffer may follow before the next ef_index. The kernels' grids follow pcm_cap, so
 *                  size it to the call (an asynchronous sizing call, or the previous submit's need plus a margin).
 *                  Errors: EF_EINVAL for a NULL pcm or a host pointer; EF_ESTATE before ef_audio_enable.
 * ef_audio_wait    waits for the last ef_decode_audio_async of the context: EF_OK, or EF_ENOMEM when it did not fit.
 *                  ef_index of a new submit, ef_decode_audio, ef_restart_streams, ef_reset and ef_audio_enable wait for
 *                  an outstanding call themselves (only the host knows whether it consumed the submit's audio); an async
 *                  call waits for the one before it only when that one consumed the submit's audio. Everything else is
 *                  ordered on the device: a later submit's upload and demux wait for the call with an event. */
int ef_decode_audio_async(ef_ctx* ctx, const uint8_t* end_of_stream, ef_audio_info* info,
                          int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm, void* stream);
int ef_audio_wait(ef_ctx* ctx);

/* ---- presentation timestamps of the pictures of TS submits -----------------------------------------------------
 * The reference's decoder latches _pts when a video PES start carries a PTS with a valid prefix (demux(), parse_pts(),
 * player.cpp:299-306, 399-419; a missing or malformed PTS keeps the previous value, reset() does not clear it) and pushes
 * every picture with the value latched at its header (flush_picture(), player.cpp:692-702). Its bit reader keeps 24 bits
 * buffered (player.cpp:348-352) and demuxes a packet when it fetches the packet's first payload byte (more(), player.cpp:
 * 459-493), so at picture() (player.cpp:1360-1363) it has demuxed up to the code byte + 2. The rule, over the stream's
 * whole video ES across submits:
 *     pts(picture) = PTS of the last video PES start with a valid PTS whose first payload byte lies at ES offset
 *                    <= (offset of the picture start code's 0x00 code byte) + 2; -1 if there is none.
 * B/D picture headers latch like I/P headers. The reference pushes nothing while the first picture's pts is -1 (the
 * frame buffers do not swap); the rule's value is reported there all the same.
 * ef_pts_enable   from now on every ef_submit_ts_* also lists the video PES starts of every stream (one device pass on
 *                 the upload stream) and every ef_index resolves the pts of every picture (one pass). A context that
 *                 never calls it launches no extra kernel. ES submits, and TS submits made before enabling, carry no PES:
 *                 their pictures get the carried value. ef_reset sets every stream back to -1 and keeps PTS enabled.
 *                 Indexing the same submit again carries the state on as if the same input followed itself.
 * ef_picture_pts  synchronous; about the submit made current by the last ef_index, streams [first, first + count):
 *                 pic_pts[k * n_pictures + p] = pts of picture p of stream first + k (-1 for p >= its picture count),
 *                 last_pts[k] = what get_pts() returns after that submit: the pts of the stream's most recent picture over
 *                 all submits (-1 if none). Either pointer may be NULL. EF_ESTATE before ef_pts_enable or before an
 *                 ef_index that followed it; EF_EINVAL for a bad stream range or n_pictures outside 0..max_pictures. */
int ef_pts_enable(ef_ctx* ctx);
int ef_picture_pts(ef_ctx* ctx, int first, int count, int n_pictures, int64_t* pic_pts, int64_t* last_pts);

/* Paced presentation: the composite fields each stream's TV shows. Every stream has its own display under the instant-decoder
 * model (time passes only while push_video waits): position (frame counter F, last line drawn), _pts_origin and
 * _video_frame_counter_origin, the current frame store and the poster scroll (_animate_index / _hscroll). Pushing picture k
 * runs push_video's arithmetic at the current F (video.cpp:1023-1057: pts / 1500 NTSC or / 1800 PAL, the origin latch, mode != 0
 * due now, more than two fields late re-latches), then draws lines until the flip (video_isr, video.cpp:1122-1198): the first
 * line below vsync_start that is not an active line of a presented frame, once F >= _next_frame_time. animate() runs at the
 * flip and at every field end (video.cpp:1076-1088). A push emits the fields whose line active_bottom - 1 it draws, each as
 * K2 draws it from the current store (picture k - 1), the other store (picture k), the hscroll of its active lines, its F and
 * the stream's overlay (ef_present_overlay; none until it is called). Fields are line_count x line_width uint16 samples
 * (ef_present_format EF_FIELD_DAC8: bytes).
 * ef_present_enable   needs ef_pts_enable and ef_video_init first (else EF_ESTATE) and fixes the standard: a later
 *                     ef_video_init that changes it returns EF_ESTATE. Each display starts at line 0 of field
 *                     frame_counter0[s] (NULL: 0) with no frame presented. Presentation starts with the next ef_index. From
 *                     then on ef_decode_picture / ef_decode_all / ef_decode_all_to_host return EF_ESTATE (frames decoded
 *                     outside the schedule would desynchronise it), and ef_index returns EF_ESTATE while picture indices
 *                     of the current submit are unpresented. ef_reset does video_reset() (video.cpp:1070-1074) on every
 *                     display: the next push latches a new origin; position, current store and scroll stay.
 * ef_present_picture  pic = 0, 1, ... of the current submit, in order (else EF_ESTATE). Decodes picture index `pic` of every
 *                     stream (K1a once per rec_pics indices and K1b, as ef_decode_all) and pushes it, with its pts
 *                     (ef_picture_pts) and modes[s] (NULL: 0; 1 = flush_picture(1) at the end of a stream, 2 / 3 =
 *                     load_poster's scroll; > 3: EF_EINVAL), on every stream that has it. A picture with pts -1 and mode 0
 *                     is not pushed (player.cpp:692-702): flags |= 1 (outside the domain), later fields unspecified.
 * ef_present_idle     every display runs on with nothing pending until it has emitted n_fields[s] more fields (the tail
 *                     after a stream's last flip; fields before any flip are blank).
 * Both write every stream's emitted fields, packed in stream order, to dst (device, 16-byte aligned): stream s's
 * info[s].n_fields fields start at dst + info[s].first x line_count x line_width and carry frame counters
 * info[s].frame_counter, + 1, ... flip_field / flip_line: where the pushed picture flipped (-1: no picture pushed). flags:
 * bit 0 = outside the domain. dst == NULL is a sizing call: info only, nothing changes. dst_fields below the total:
 * EF_ENOMEM, nothing decoded and nothing changed. Synchronous on `stream`. */
typedef struct {
    uint64_t first;
    uint32_t n_fields, frame_counter, flip_field;
    int32_t flip_line, flags;
} ef_present_info;
int ef_present_enable(ef_ctx* ctx, const uint32_t* frame_counter0);
int ef_present_picture(ef_ctx* ctx, int pic, const uint8_t* modes, uint16_t* dst, uint64_t dst_fields, ef_present_info* info, void* stream);
int ef_present_idle(ef_ctx* ctx, const uint32_t* n_fields, uint16_t* dst, uint64_t dst_fields, ef_present_info* info, void* stream);

/* ef_present_picture_async / ef_present_idle_async  the same work as ef_present_picture / ef_present_idle with the same arguments
 *                     (schedule, decode, push and render; modes 0..3, the overlay latch, K1a once per rec_pics indices), returning
 *                     once it is enqueued on `stream`: nothing is read back, so a player can enqueue a whole submit and prepare
 *                     the next upload, or hand earlier fields to a device consumer, while the GPU renders. dst and info are device
 *                     memory (NULL, a host pointer or an unaligned dst: EF_EINVAL); info[] gets the ef_present_info rows, written
 *                     on the device in stream order before the fields, so every stream's fields can be located without a host
 *                     read. modes / n_fields are host memory, read before the call returns. Order and EF_ESTATE as the
 *                     synchronous calls; the next picture index advances when a call is enqueued. The host waits only for the
 *                     picture count of a submit (once per submit, as the synchronous calls), when dst_fields grows past every
 *                     earlier call's (the descriptor arrays grow), and when 16 calls are still queued ahead of this one.
 *                     The async calls since the last ef_present_wait form a chain; the capacity is checked on the device. When a
 *                     call's fields exceed dst_fields, its info[] carries the counts and offsets it would have needed (an
 *                     asynchronous sizing call) and flags bit 1; nothing is decoded, no display or overlay state changes and dst
 *                     is not written. Every later call of the chain then does nothing either: its info[] rows have n_fields 0
 *                     and flags bit 1. Sync and async calls may be mixed in any order; concatenated, their fields and info[]
 *                     equal an all-synchronous run.
 *                     K2's grid follows dst_fields (its CTAs past the call's fields exit at once), so size dst_fields to the call:
 *                     from an asynchronous sizing call, or the previous submit's need plus a margin.
 *                     Launches per call: the schedule and the size kernel; K1a when `pic` starts a rec_pics range (and at the
 *                     index a failed chain is retried from); K1b; the descriptors; ceil(dst_fields / 65,535) K2. An idle call
 *                     launches the same without K1a and K1b.
 * ef_present_wait     waits for the chain: EF_OK, or EF_ENOMEM when a call did not fit. *n_presented (may be NULL) = the calls of
 *                     the chain that took effect. After EF_ENOMEM the next picture index rolls back to the failing call's, and
 *                     a retry with a larger dst continues bit for bit as if the failed call had never been made. ef_index,
 *                     ef_present_picture, ef_present_idle, ef_present_overlay, ef_restart_streams, ef_reset and ef_video_init
 *                     wait for an outstanding chain themselves (only the host knows how far it got); its result stays
 *                     available to ef_present_wait until the next async call. */
int ef_present_picture_async(ef_ctx* ctx, int pic, const uint8_t* modes, uint16_t* dst, uint64_t dst_fields, ef_present_info* info,
                             void* stream);
int ef_present_idle_async(ef_ctx* ctx, const uint32_t* n_fields, uint16_t* dst, uint64_t dst_fields, ef_present_info* info,
                          void* stream);
int ef_present_wait(ef_ctx* ctx, int* n_presented);

/* ef_present_format   what the four present calls write to dst, chosen before ef_present_enable (after it: EF_ESTATE; an unknown
 *                     format: EF_EINVAL; ef_reset keeps it). EF_FIELD_U16, the default, is the reference's DMA line buffer: uint16
 *                     samples whose high byte drives the 8-bit DAC (levels IRE(x) << 8, video.cpp:520) and whose low byte is
 *                     blit()'s junk. The I2S unit plays the two 16-bit halves of each word in swapped order, which the reference's
 *                     buffers are written for (burst_pal(), video.cpp:640-644; blit(), video.cpp:727-733), so buffer sample t ^ 1
 *                     plays at time t. EF_FIELD_DAC8 is what the DAC plays: byte t of line l is u16[l][t ^ 1] >> 8, where u16 is the
 *                     same field in EF_FIELD_U16; a field is line_count x line_width bytes (NTSC 238,944, PAL 354,432), half the
 *                     bytes to write and to move. dst stays a uint16_t* in the prototypes: on a DAC8 context pass a byte buffer
 *                     cast to it. dst_fields, info[] and the 16-byte alignment of dst, the capacity checks, sizing calls, EF_ENOMEM,
 *                     the async gate and retries, the schedule, overlay and clock are the same in both formats. ef_composite_field,
 *                     ef_read_field, ef_video_isr and ef_blit stay uint16: they stand for the line buffer itself. */
#define EF_FIELD_U16   0   /* default: the reference's uint16 DMA buffer, as today */
#define EF_FIELD_DAC8  1   /* what the video DAC plays: one byte per sample, in playback order */
int ef_present_format(ef_ctx* ctx, int format);

/* ef_present_overlay  composite() of every paced field (video.cpp:839-887, 1181-1194): the 80 x 16 bitmap and the progress bar
 *                     on the 16 lines from active_bottom + 2, faded by the blend. Stages changes for streams [first, first +
 *                     count): bitmaps = count x 1280 bytes (_video_composite[16][80] of each stream), blend and progress (int32
 *                     each) and set[i] (bit 0 bitmap, bit 1 blend, bit 2 progress; set NULL = all three; a NULL array = that
 *                     attribute is not set). Staged changes merge, the last write winning per attribute, and latch at line 0
 *                     of the first field that starts at or after the position where the next ef_present_picture /
 *                     ef_present_idle call begins: field F at (F, line 0), F + 1 otherwise. A call that does not draw that
 *                     line (it emits no field past it) leaves them pending, as do a sizing call and EF_ENOMEM. Every field is
 *                     drawn with the state latched at its line 0; a latched blend b > 0 counts down at every field end, so
 *                     field G shows max(0, b - (G - G_latch)) (frame counters modulo 2^32); -1 and >= 32 are full strength,
 *                     0 draws nothing. The bar fills step i = 0, 2, ..., 238 where i < progress. Every stream starts with
 *                     blend 0; ef_reset keeps latched and staged overlays (video_reset() leaves them alone). Synchronous,
 *                     host memory. EF_ESTATE before ef_present_enable; EF_EINVAL for a bad stream range or a blend below -1
 *                     (the reference's fade arithmetic wraps there). */
int ef_present_overlay(ef_ctx* ctx, int first, int count, const uint8_t* bitmaps, const int32_t* blend, const int32_t* progress,
                       const uint8_t* set);

/* ef_present_font     the glyph atlas of the overlay's time text, in the layout of the reference's _font8 / _font8_rights
 *                     (font.h): atlas = 16 rows x 1024 columns of 8-bit coverage, glyph i (character i + 0x18) = columns
 *                     [rights[i - 1], rights[i]) (from 0 for i = 0). Copied to the device; the library embeds no font.
 *                     EF_EINVAL unless the rights increase from above 0 up to at most 1024 and n_rights covers 0x18..':' (35).
 * ef_present_clock    ESPFlix::update_progress() (espflix.cpp:862-874) for streams [first, first + count): idx_hdrs = count x the
 *                     104-byte video.idx header of the stream's title (idx_hdr, host/ef_indexer.h: what merge_index writes and nav()
 *                     reads), speed[i] = _speed (0 the title, 1 the fast-forward stream, -1 the rewind stream), flags[i] bit 0 = the
 *                     clock is on (off is _nav == -1, the default), bit 1 = paused (the pause icon at speed 0), bit 2 = _last_seconds
 *                     = 0 (what play_pause() and the pause do, espflix.cpp:819, 935). From then on every ef_present_picture /
 *                     ef_present_idle (and _async) call that is not a sizing call runs, at its start and on every stream whose clock
 *                     is on: main = pts2pts(get_pts(), speed) (espflix.cpp:597-604; get_pts() = the pts of the picture the call
 *                     pushes, else the stream's last_pts of ef_picture_pts), seconds = (int)(main / 90000); when seconds !=
 *                     _last_seconds, show_time(seconds, icon) redraws the bitmap (espflix.cpp:163-174; icon PAUSE / PLAY at speed 0,
 *                     FFWD, RWND) and _last_seconds = seconds; always progress = (int)(main * 240 / video.last_pts). Bitmap and
 *                     progress are staged as ef_present_overlay stages them, after what it staged before the call (the last write
 *                     wins per attribute) and latch by the same rule; the blend stays the caller's. A sizing call, EF_ENOMEM and an
 *                     async call that does not take effect change no clock state and no bitmap slot. Outside the domain, not
 *                     checked: products that overflow int64, |main / 90000| >= 2^31 and text over 15 characters. Synchronous, host
 *                     memory. EF_ESTATE before ef_present_enable or ef_present_font; EF_EINVAL for a bad stream range, a speed
 *                     outside -1..1, or a stream turned on with video.last_pts 0 or speed +-1 on a trick record whose last_pts
 *                     equals its first_pts (the reference divides by zero there). ef_reset and ef_restart_streams keep the clocks.
 *                     A context adds two launches per present call once a clock has been set (one for a sizing call). */
int ef_present_font(ef_ctx* ctx, const uint8_t* atlas, const int16_t* rights, int n_rights);
int ef_present_clock(ef_ctx* ctx, int first, int count, const uint8_t* idx_hdrs, const int8_t* speed, const uint8_t* flags);

/* ---- per-stream restart: what the reference's player does on play / skip / fast_forward / rewind / load_poster / play_pause --
 * ef_restart_streams  ops[i] for stream first + i: 0 = nothing; 1 = MpegDecoder::reset() with its video_reset() (player.cpp:439-453,
 *                     video.cpp:1070-1074); 2 = video_pause(0) (video.cpp:1060-1068). The restart falls between the current submit
 *                     and the next one, whether that one is already queued or not. Op 1: get_pts() reads -1 until the next picture
 *                     (the carried _pts stays, so a program whose first video PES has no PTS takes the old one); the audio demux
 *                     gate shuts (the next submit's audio bytes before its first PES start are dropped, also for a TS submit
 *                     already queued); the SBC bytes held back and the learned frame size are dropped (the next frame is probed
 *                     and decoded twice) while the filter memory, the last subband samples and the delta-sigma modulator
 *                     carry on; the display latches a new origin at the next push. Ops 1 and 2 both clear the display origin;
 *                     frame stores, sequence state, display position, current store, scroll and overlay stay. Streams with op 0
 *                     and all other streams do not change; subsystems never enabled are not touched. Synchronous, host memory.
 *                     EF_EINVAL for a bad stream range or an op above 2; EF_ESTATE (as ef_index) on a presenting context while
 *                     picture indices of the current submit are unpresented, or on an audio context while the current TS
 *                     submit's audio has not been through ef_decode_audio. */
int ef_restart_streams(ef_ctx* ctx, int first, int count, const uint8_t* ops);

/* ---- TS submits cut at any packet boundary: each stream holds its unfinished picture on the device --------------------------
 * Access unit: an optional sequence header, an optional GOP header, a picture header and its slices. A unit is complete once all
 * four bytes of a later sequence (B3), GOP (B8), picture (00) or sequence-end (B7) start code are present in the bytes received
 * so far (the marker dispatch, player.cpp:1318).
 * ef_carry_enable  from the next submit on, TS submits may be cut at any 188-byte packet boundary, per stream. Each stream's part
 *                  of a submit is the bytes it held after the previous one followed by the submit's new video ES; its pictures
 *                  are the complete units in that part, and everything from the first byte of the first incomplete unit to the
 *                  end is held for the next submit (a sequence header cut inside its matrices, a start code split across the
 *                  cut, a picture whose last slice has arrived but no start code after it). With no unit open, the last 3
 *                  bytes are held (they may begin a start code); after a sequence-end code nothing is. Held pictures count in
 *                  no n_pictures, max_pictures, ef_index_info, ef_stream_info or base_pictures until the submit that completes
 *                  them. Concatenated over the submits, decoded pictures, ef_picture_pts values (the rule above is over the
 *                  whole ES already; a held picture's latch may fall in the next submit), paced fields with their info rows
 *                  and audio equal what the uncut program gives.
 *                  Capacity: both ES buffers and the coefficient lists sized from es_capacity (12 bytes per ES byte) grow by
 *                  n_streams x max_carry, so the es_capacity check of a submit still suffices. A stream whose held bytes would
 *                  exceed max_carry (which must exceed its largest picture) drops them: its flag (ef_carry_info) stays set and
 *                  ef_index_info returns EF_ENOMEM with info bit 2 until op 1, the end of the stream or ef_reset; its output is
 *                  unspecified meanwhile, every other stream's is exact.
 *                  Interactions: ef_restart_streams op 1 drops the held bytes and the PES starts in them (also from a submit
 *                  already queued); op 2 keeps them. ef_reset drops every stream's and keeps carry enabled. ef_index without a
 *                  fresh submit, and ES submits, return EF_ESTATE. get_pts() (last_pts) refers to the complete pictures.
 *                  Launches per TS submit: ef_ts_len_kernel (with packets), ef_ts_scan_kernel, ef_carry_lead_kernel,
 *                  ef_ts_offsets_kernel, ef_carry_copy_kernel, ef_ts_copy_kernel (with packets). The held bytes are copied on
 *                  the device after the previous ef_index; the host does not wait.
 *                  Errors: EF_ESTATE with a submit pending or on a second call; EF_EINVAL for max_carry < 4.
 * ef_end_streams   the input of streams [first, first + count) with ends[i] != 0 ends with the most recent (pending) submit, as
 *                  the reference's len <= 0 Buffer ends it (player.cpp:456, 469-473): at its ef_index the stream's last unit
 *                  counts as complete, as if SEQUENCE_END followed; held bytes that hold no picture are dropped, and afterwards
 *                  the stream holds nothing (the next submit may start a new program). Calls for one submit accumulate.
 *                  EF_ESTATE if no submit is pending or carry is off; EF_EINVAL for a bad stream range.
 * ef_carry_info    synchronous: held_bytes[i] = bytes stream first + i holds after the current submit, flags[i] bit 0 = its held
 *                  bytes exceeded max_carry. Either pointer may be NULL. EF_ESTATE before ef_carry_enable; EF_EINVAL for a bad
 *                  stream range. */
int ef_carry_enable(ef_ctx* ctx, uint32_t max_carry);
int ef_end_streams(ef_ctx* ctx, int first, int count, const uint8_t* ends);
int ef_carry_info(ef_ctx* ctx, int first, int count, uint32_t* held_bytes, uint8_t* flags);

/* ---- titles held in device memory: the reference's Streamer and ESPFlix's play / skip / fast_forward / rewind / pause ------------
 * The reference reads a title through Streamer::get(url, offset) and 8-packet Buffers (espflix.cpp:723-747, 787-798) and seeks with
 * the uint32 packet number that video.idx holds at idx_hdr::pts2offset(pts, speed) (get_index, espflix.cpp:607-629, 823-829). Here
 * the titles live in HBM: a viewer's action is a few bytes from the host, and no TS byte crosses the host link again.
 * ef_library_add      copies one title to device memory: its video.idx image (idx_hdr, host/ef_indexer.h, then the main, fwd and rwd
 *                     sample arrays) and its three transport streams in _vid_names order (espflix.cpp:641): ts[0] video_rwd.ts,
 *                     ts[1] video.ts, ts[2] video_fwd.ts; the trick files may be NULL / 0. *title = its number (0, 1, ...). Titles stay
 *                     until ef_destroy. The first call allocates every stream's state and a staging buffer of es_capacity bytes.
 *                     EF_EINVAL: a bad sig or len != 3; samples past the end of the image; a video record with bin_size or
 *                     sample_count 0; a present trick file whose record has trick_speed, bin_size or sample_count 0 or last_pts ==
 *                     first_pts (the reference divides by zero there); no main file; a file size that is not a multiple of 188 or is
 *                     >= 4 GiB, or an image >= 4 GiB (the offset arithmetic is uint32).
 * ef_library_command  cmd for every stream of [first, first + count): the ESPFlix methods (espflix.cpp:800-859), with the restart op
 *                     each one implies run as ef_restart_streams runs it (same EF_ESTATE cases):
 *                       EF_LIB_PLAY_AT (title, arg = main pts)  nav(title) with pos = arg, then play_pause() from NAV        op 1
 *                       EF_LIB_PLAY                             play(nav, 0, get_index(0, pos) * 188)                          op 1
 *                       EF_LIB_SKIP (arg = seconds, an int)     skip(s): pos += s * 90000 (an int product), kept unclamped      op 1
 *                       EF_LIB_FAST_FORWARD / EF_LIB_REWIND     fast_forward() / rewind(): play at speed +-1 from pos          op 1
 *                       EF_LIB_PAUSE                            pause: a PLAYING stream becomes PAUSED and gets no more bytes  op 0
 *                       EF_LIB_RESUME                           video_pause(0): a PAUSED stream plays on from its cursor        op 2
 *                       EF_LIB_STOP                             menu: the stream gets no more bytes (STOPPED)                   op 0
 *                     Every command but PLAY_AT and RESUME first saves, on a PLAYING stream, pos = pts2pts(get_pts(), speed)
 *                     (save_pos, espflix.cpp:843-852), get_pts() being ef_picture_pts's last_pts after the current submit; PAUSED,
 *                     STOPPED and ENDED streams keep the pos they have. The offset arithmetic and the sample read run on the device,
 *                     one thread per stream; the host never reads a pts. A sample that names a packet at or past the end of its file
 *                     puts the cursor there (the reference's uint32 product would wrap only for such samples). Synchronous, host
 *                     memory. EF_ESTATE before the first ef_library_add or without ef_pts_enable and ef_carry_enable. EF_EINVAL: a bad
 *                     stream range or command; PLAY_AT of an unknown title; any other command on a stream that never played;
 *                     FAST_FORWARD / REWIND on a title without that file; RESUME on a stream that is not PAUSED; SKIP outside int.
 * ef_library_submit   a TS submit made on the device (as ef_submit_ts_device): every PLAYING stream gets min(per_stream[s], or
 *                     packets when per_stream is NULL, the packets left in its file) packets from its cursor, every other stream
 *                     none. A stream whose cursor reaches the end of its file ends with this submit (as ef_end_streams ends it) and
 *                     becomes ENDED with pos = pts2pts(0, speed), what save_pos(0) leaves at DONE (espflix.cpp:906-911): 0 at speed 0.
 *                     ef_index follows as usual. per_stream is host memory. EF_ESTATE before the first ef_library_add, without
 *                     ef_pts_enable and ef_carry_enable, or with a submit pending; EF_ENOMEM, nothing changed, when the budgets'
 *                     packets x 188 exceed es_capacity (a bound the host checks, so nothing is read back but the upload's offsets).
 *                     ef_end_streams on a library submit returns EF_ESTATE. Launches: a count kernel, a gather kernel (its grid
 *                     follows the bound) and the TS upload sequence of ef_carry_enable. ef_reset keeps titles, states and cursors
 *                     (video_reset() leaves the Streamer alone); a library submit it drops is not given again.
 * ef_library_info     synchronous: status[i] = stream first + i's title (-1 before PLAY_AT), speed, state, file (speed + 1), byte
 *                     cursor in that file and pos (what save_pos(..., true) writes to NVS). EF_ESTATE before the first
 *                     ef_library_add; EF_EINVAL for a bad stream range. */
#define EF_LIB_PLAY_AT      0
#define EF_LIB_PLAY         1
#define EF_LIB_SKIP         2
#define EF_LIB_FAST_FORWARD 3
#define EF_LIB_REWIND       4
#define EF_LIB_PAUSE        5
#define EF_LIB_RESUME       6
#define EF_LIB_STOP         7
#define EF_LIB_NAV          8    /* the poster menu: ef_library_add_poster below */
#define EF_LIB_NAV_STEP     9
#define EF_LIB_MENU         10
#define EF_LIB_IDLE    0         /* stream states: never played */
#define EF_LIB_PLAYING 1
#define EF_LIB_PAUSED  2
#define EF_LIB_STOPPED 3
#define EF_LIB_ENDED   4         /* its cursor reached the end of its file */
#define EF_LIB_POSTER  5         /* the reference's NAV: the title's poster.ts is streamed (file 3) or shown */
typedef struct { int32_t title, speed, state, file; uint64_t cursor; int64_t pos; } ef_library_status;
int ef_library_add(ef_ctx* ctx, const uint8_t* idx, uint64_t idx_bytes, const uint8_t* const* ts, const uint64_t* bytes, int* title);
int ef_library_command(ef_ctx* ctx, int first, int count, int cmd, int title, int64_t arg);
int ef_library_submit(ef_ctx* ctx, uint32_t packets, const uint32_t* per_stream, void* stream);
int ef_library_info(ef_ctx* ctx, int first, int count, ef_library_status* status);
/* ef_library_add_trick  gives a title added with its main only (ts[0] and ts[2] NULL) its fast-forward and rewind files: ef_trick_build
 *                     on the main already in device memory (read back once: the segment plan reads its packets on the host), then the
 *                     fwd and rwd records and samples of the title's video.idx as merge_index() computes them for the built files
 *                     (bin_size 7,500, trick_speed 15, pts2seq()'s samples); the header's video record, its padding bytes and the main's
 *                     samples stay byte for byte as added. The image equals what ef_tsidx_scan + ef_tsidx_samples (capi.build_video_idx)
 *                     give for (main, fwd, rwd) when the title's own records were built that way. From then on FAST_FORWARD and REWIND
 *                     play the built files. Synchronous. EF_ESTATE before the first ef_library_add, or when the title already has either
 *                     trick file (a second call); EF_EINVAL for an unknown title, qscale outside 1..31, the cases of ef_trick_build, or a
 *                     main of fewer than 16 pictures (a one-picture trick file, whose record the reference divides by zero with). Nothing
 *                     changes on an error. */
int ef_library_add_trick(ef_ctx* ctx, int title, int qscale);
/* ef_library_read     copies part `what` of a title to host memory: -1 its video.idx image, 0 / 1 / 2 its rwd / main / fwd file (after
 *                     ef_library_add_trick: the built files and the rewritten image, for a service to store beside video.ts), 3 its
 *                     poster.ts. *bytes = the part's size (0: no such file, nothing copied). EF_ENOMEM when dst is NULL or cap is below
 *                     it (a sizing call). EF_ESTATE before the first ef_library_add; EF_EINVAL for an unknown title or part. Synchronous. */
int ef_library_read(ef_ctx* ctx, int title, int what, uint8_t* dst, uint64_t cap, uint64_t* bytes);

/* ---- the poster menu: ESPFlix::nav(), menu(), load_poster() and the NVS resume (espflix.cpp:704-720, 763-785, 851-859, 906-939,
 * 1060-1069; espflix.ino:160-178) ---------------------------------------------------------------------------------------------------
 * ef_library_add_poster  attaches a title's poster.ts (what the reference's make_video() writes with ffmpeg -bf 0 -q 2, indexer.cpp:306;
 *                     capi.encode_poster makes it) as the title's file 3. Synchronous. EF_EINVAL for an unknown title, a NULL poster or a
 *                     size that is 0, not whole packets or >= 4 GiB; EF_ESTATE before the first ef_library_add or when the title has a
 *                     poster already. Nothing changes on an error.
 * The saved positions (the reference's NVS, one int64 per title and stream): nv[title x n_streams + s], title-major, every entry 0 at
 * first (nv_read's default for a missing key); it grows with the title table. ef_library_nv_read / _nv_write copy entries
 * [first, first + count) of one title to / from host memory, synchronously, so that a service can keep its viewers' places across
 * sessions as NVS survives a reboot. EF_ESTATE before the first ef_library_add; EF_EINVAL for an unknown title or a bad stream range.
 * Commands of ef_library_command, where nav(s, i) is the reference's nav(i) for stream s: dir = (title == -1) ? 0 : title - i from the
 * old title, mode = dir == 0 ? 1 : dir < 0 ? 2 : 3; title = i, pos = nv[i][s], state EF_LIB_POSTER, file 3 from byte 0, restart op 1
 * (load_poster's _decoder.reset()), and on a presenting context a blend of 0 staged as ef_present_overlay stages it (hide_progress()).
 * speed is kept (nav() leaves _speed alone).
 *   EF_LIB_NAV (title i)                 from IDLE or POSTER: nav(s, i). The first nav(0) after init_service(), or any jump.
 *   EF_LIB_NAV_STEP (arg = step, an int) from POSTER: nav(s, title + step); a stream whose target is outside [0, titles) is left as it
 *                                        is, with no restart and no blend (nav()'s early return). The left / right keys.
 *   EF_LIB_MENU                          menu() and then loop()'s pending-NAV branch. PLAYING at speed 0: pos = pts2pts(get_pts(), 0),
 *                                        nv[title][s] = pos, nav(s, title) (mode 1). PLAYING at speed +-1: pos = pts2pts(get_pts(),
 *                                        speed), nv[title][s] = pos, then play at speed 0 from pos (op 1, no poster; espflix.cpp:911-913).
 *                                        PAUSED, STOPPED, ENDED: nav(s, title) with no NVS write, so pos becomes the last saved value.
 *                                        POSTER: nothing (set_state()'s early return).
 * EF_EINVAL, nothing changed: NAV or NAV_STEP from any other state, MENU on IDLE, NAV to an unknown title, a nav to a title without a
 * poster, a step outside int. The other commands treat a POSTER stream by their existing rules: PLAY plays the title at speed 0 from pos
 * (play_pause() from NAV, so it resumes from the saved position), SKIP / FAST_FORWARD / REWIND start from pos, PAUSE does nothing,
 * RESUME is EF_EINVAL, STOP stops the poster's bytes. The host reads back the commanded streams' states only, as for every command.
 * ef_library_submit gives a POSTER stream packets of file 3 as it gives a PLAYING stream packets of its file; the submit that reaches
 * the poster's end ends the stream (as ef_end_streams) and carries the stream's mode, but the stream stays POSTER with its pos and takes
 * no more packets. On a presenting context the push of that stream's last picture of that submit (index n_pics - 1) uses the mode, in
 * ef_present_picture and ef_present_picture_async alike, where the call's modes[s] is 0 or modes is NULL (a caller's mode wins);
 * the poster's earlier pictures are pushed at mode 0. A later nav before the poster ended replaces the mode. */
int ef_library_add_poster(ef_ctx* ctx, int title, const uint8_t* ts, uint64_t bytes);
int ef_library_nv_read(ef_ctx* ctx, int title, int first, int count, int64_t* pos);
int ef_library_nv_write(ef_ctx* ctx, int title, int first, int count, const int64_t* pos);

/* ---- the remote: one iteration of ESPFlix::loop() (espflix.cpp:886-1010) for every stream ----------------------------------------
 * ef_library_keys     keys[s] = stream s's key for this iteration (the HID codes key_event() produces, espflix.cpp:1020-1040; 0 = none,
 *                     any other code is ignored as loop()'s default: ignores it): n_streams bytes in host memory (read before the call
 *                     returns) or device memory (a producer on the device, ordered by `stream`). Every stream runs, in the reference's
 *                     order:
 *                     1. the pause branch of a title that ended (_pending == DONE): an ENDED stream navs to its title's poster as
 *                        EF_LIB_MENU does on ENDED, also with key 0. A title without a poster stays ENDED and ignores the key.
 *                     2. the key, on the state step 1 left; the pending branch resolves at once (the library pauses at the submit
 *                        boundary), get_pts() being ef_picture_pts's last_pts, so each key runs as one command of ef_library_command:
 *                          key             POSTER            PLAYING speed 0        PLAYING speed +-1   PAUSED              STOPPED
 *                          MENU            nothing           EF_LIB_MENU            EF_LIB_MENU         EF_LIB_MENU         EF_LIB_MENU
 *                          PLAY / SELECT   EF_LIB_PLAY       EF_LIB_PAUSE           EF_LIB_PLAY         EF_LIB_RESUME       nothing
 *                          RIGHT / LEFT    NAV_STEP +1 / -1  FAST_FORWARD / REWIND  EF_LIB_PLAY         FAST_FORWARD / REW  nothing
 *                          UP / DOWN       nothing           EF_LIB_SKIP +30 / -30  EF_LIB_PLAY         nothing             nothing
 *                        IDLE streams ignore every key. A command ef_library_command would refuse with EF_EINVAL (a missing trick
 *                        file, no poster at the target) does nothing; a step outside the row does nothing (nav()'s early return).
 *                     done (device memory, n_streams bytes, or NULL): the low nibble = the EF_LIB_* command the key ran as, or
 *                     EF_KEY_DONE_NOTHING; bit 4 (EF_KEY_DONE_ENDED) = step 1 ran. The restart op of the commands runs as
 *                     ef_library_command runs it (op 1 when either step restarts). On a presenting context each stream also gets the
 *                     blend loop() leaves, staged as ef_present_overlay stages it: 0 after a nav (hide_progress()), 180 after a play at
 *                     speed 0, a pause or a resume (show_progress()), -1 after a play at speed +-1. On a stream whose clock is on
 *                     (ef_present_clock flag bit 0) the clock's speed and paused bit follow the stream, _last_seconds becomes 0 where
 *                     play_pause() or the pause zero it (espflix.cpp:819, 935: PLAY / SELECT on a stream that takes keys, and every
 *                     key that acts at speed +-1), and a nav to another title writes that title's video.idx records.
 *                     Asynchronous: enqueued on `stream`, no wait for the device and no read-back. The keys act between the current
 *                     submit and the next one, where ef_library_command acts; the next ef_library_submit, submit, ef_index, present and
 *                     audio call are ordered after it on the device through an event (the synchronous calls wait for the device).
 *                     Launches per call: the keys kernel, ef_restart_kernel, ef_carry_restart_kernel and, on an audio context, the
 *                     audio end kernel; a context that never calls it launches what it launched before. EF_ESTATE: the cases of
 *                     ef_library_command (no title, no PTS or carry) and of ef_restart_streams (unpresented pictures, unconsumed
 *                     audio; an outstanding async present chain or audio call is waited for first). EF_EINVAL: keys NULL, or done in
 *                     host memory. */
#define EF_KEY_MENU   16
#define EF_KEY_PLAY   19
#define EF_KEY_SELECT 40
#define EF_KEY_RIGHT  79
#define EF_KEY_LEFT   80
#define EF_KEY_DOWN   81
#define EF_KEY_UP     82
#define EF_KEY_DONE_NOTHING 0x0F  /* done[s]: the key ran no command */
#define EF_KEY_DONE_ENDED   0x10  /* done[s]: the title had ended and the DONE branch ran first */
int ef_library_keys(ef_ctx* ctx, const uint8_t* keys, uint8_t* done, void* stream);

/* ---- experiment, NOT on the decode path (north_star: "the 8x8 IDCT ... batched onto tensor cores") ------------
 * The linearised IDCT of MpegDecoder::idct() (player.cpp:922-996) as a [n_blocks x 64] x [64 x 64] TF32 GEMM on
 * Hopper wgmma with register accumulators and TMA-fed operand tiles (csrc/ef_idct_tc.cu). coefs: n_blocks x 64 prescaled
 * int32 coefficients as idct() receives them; L: the 64 x 64 linear map (row = output sample, column = input
 * coefficient; tests/idct_linear.py derives it from the butterfly); out: n_blocks x 64 rounded residuals. The reference
 * transform rounds inside every butterfly, so this differs from it by up to +-1 (tests/test_idct_tc_gpu.py measures how
 * often) and cannot replace the integer kernel where YUV must be bit-exact. prep_ms / mma_ms: best-of-`repeats` device
 * times of the operand pre-pass and of the MMA kernel. */
int ef_idct_tc_run(int device, const int32_t* coefs, int n_blocks, const double* L, int32_t* out, float* prep_ms, float* mma_ms, int repeats);

#ifdef __cplusplus
}
#endif
#endif
