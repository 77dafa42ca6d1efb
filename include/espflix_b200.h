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
 *   ef_audio_demux_ts             MpegDecoder::demux() for the audio PIDs -> push_audio() player.cpp:381-432, video.cpp:1007
 *   ef_audio_decode               decode_audio() video.cpp:964, sbc_decoder() sbc_decoder.cpp:343, pdm_second_order()
 *                                 espflix.ino:73
 *   ef_audio_enable / ef_decode_audio  the same audio path fed by the context's TS submits, one submit at a time
 *   ef_pts_enable / ef_picture_pts     the pts push_video(frame, front, _last_pts, mode) hands over with every picture
 *                                 (flush_picture() player.cpp:692-702, latched from demux() player.cpp:399-419) and
 *                                 get_pts() player.cpp:653-656, for every stream of a TS submit
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
 * Each submit must hold whole pictures (cut at picture/sequence start codes). A submit is queued on an
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
 *                    -1 first frame rejected by the reference (nothing decoded), -2 outside its domain (the reference
 *                    handles mono, 8 subbands, 16 blocks only). */
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
