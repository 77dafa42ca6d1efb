/* oracle/ef_oracle.h — CPU restatement of the espflix hot path. TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this library;
 * the product (espflix_b200/) never links, imports or calls it.
 *
 * Parity status: PINNED. The restatement reproduces, bit for bit, the I420 dumps and composite
 * fields that the UNMODIFIED reference (oracle/_ref, built from the reference's src/) produces for
 * the reference's embedded media fixtures (tests/golden, decode_pins.json and composite_pins.json) and for the synthetic coverage
 * streams (tests/test_oracle_vs_ref.py, pinned in tests/golden/ref_pins.json).
 */
#ifndef EF_ORACLE_H
#define EF_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EFO_FB_WIDTH   352
#define EFO_FB_HEIGHT  192
#define EFO_FB_STRIDE  528          /* video.h:32 FB_STRIDE */
#define EFO_FRAME_BYTES (EFO_FB_STRIDE * EFO_FB_HEIGHT)   /* 12 strips x 8448 B, strips contiguous */
#define EFO_I420_BYTES (352 * 192 * 3 / 2)

/* MPEG-TS (188-byte packets, video PID 0x100) -> elementary stream, following
 * MpegDecoder::more/demux (player.cpp:381-493). pes_off/pes_pts (optional, cap entries each)
 * receive, per PES header seen on the video PID, the ES offset it starts at and its PTS (-1 if
 * none). Returns ES byte count; *n_pes gets the PES count. */
size_t efo_demux_ts(const uint8_t* ts, size_t len, uint8_t* es, size_t es_cap,
                    uint64_t* pes_off, int64_t* pes_pts, size_t pes_cap, size_t* n_pes);

/* Decode an elementary stream the way MpegDecoder::run does (player.cpp:1355), pushing frames
 * as push_video would see them (player.cpp:692-702) and finishing with flush_picture(1).
 * has_pts: 1 = every picture carries a PTS (normal TS input); 0 = none does (quirk Q10: no
 * push, no buffer swap). Frames are written as I420 (SURVEY.md 8c layout) into out (cap frames).
 * strips_out (optional): the two striped frame stores (2 x EFO_FRAME_BYTES) after the last picture.
 * Returns the number of frames pushed. */
long efo_decode_es(const uint8_t* es, size_t len, int has_pts,
                   uint8_t* out_i420, size_t cap_frames, uint8_t* strips_out);

/* The marker walk of efo_decode_es (run(), player.cpp:1355-1366) over an elementary stream: every marker it dispatches,
 * in order, as the bit position of its 24-bit prefix (pos[], may lie in the end-of-stream padding the reader appends) and
 * its code byte (code[]), the first cap of them. counts[3] (optional) = the picture, slice (codes 0x01-0xAF) and
 * sequence-header markers dispatched. Returns the number of markers dispatched. */
long efo_walk(const uint8_t* es, size_t len, uint64_t* pos, uint8_t* code, size_t cap, long counts[3]);

/* Macroblocks the first 8 pictures of the last efo_decode_es call wrote, 264 bytes per picture (row * 22 + column): 2 decoded
 * from the picture's own codes, 1 copied by a skip (the last write counts), 0 not written. Returns the pictures decoded. */
int efo_coverage(uint8_t* out, int max_pictures);

/* Coverage counters accumulated by efo_decode_es since the last reset (process-global; tests only). */
typedef struct {
    uint64_t pictures[8];      /* by picture_coding_type */
    uint64_t f_code[8];        /* forward_f_code histogram over P pictures */
    uint64_t slices, skipped, blocks, blocks_dc_only, escapes, escapes16, saturated, q2_zero, full_pel_mbs;
    uint64_t mb_type[32];      /* by macroblock_type flags (0x10 quant | 0x08 fwd | 0x02 pattern | 0x01 intra) */
    uint64_t mocomp_xy[4];     /* luma mocomp cases (yhalf<<1 | xhalf), non-zero vectors only */
    uint64_t pin_out_of_domain; /* clamp inputs outside [-256,511]: the reference reads out of bounds there (UB) */
} efo_stats;
void efo_stats_reset(void);
void efo_stats_get(efo_stats* s);

/* TS convenience wrapper = efo_demux_ts + efo_decode_es (has_pts from the PES headers). */
long efo_decode_ts(const uint8_t* ts, size_t len, uint8_t* out_i420, size_t cap_frames);

/* The reference IDCT (player.cpp:922-996) on 64 prescaled int32 coefficients, in place. */
void efo_idct(int32_t* b);

/* I420 <-> striped frame store (video.h:36-44; player.cpp:33-46) */
void efo_i420_to_strips(const uint8_t* i420, uint8_t* strips);
void efo_strips_to_i420(const uint8_t* strips, uint8_t* i420);

/* Composite synthesis (video.cpp:554-630, 690-934, 1122-1198). ntsc: 1 NTSC, 0 PAL. */
typedef struct {
    int ntsc, line_width, line_count, hsync, hsync_long, hsync_short, burst_start, burst_width, active_start;
    uint32_t color_tab[768];
    int16_t burst0[64], burst1[64];
} efo_video;
void efo_video_init(efo_video* v, int ntsc);
/* one blit() call (video.cpp:690): frame in strips layout */
void efo_blit(const efo_video* v, const uint8_t* strips, uint16_t* dst, int line, int x, int width, int frame_counter);
/* whole field as video_isr would emit it line by line (two ping-pong line buffers, hscroll=0,
 * no overlay); out = line_count x line_width uint16 */
void efo_field(const efo_video* v, const uint8_t* strips, int frame_counter, uint16_t* out);

/* the same with video_isr's presentation extras: hscroll (video.cpp:1146-1154; strips_b = the other
 * frame store) and the 80x16 overlay bitmap + progress bar of composite() (video.cpp:845-887);
 * blend 0 = off, -1 or >= 32 = full, 1..31 = fading; bitmap may be NULL when blend == 0 */
void efo_field_ex(const efo_video* v, const uint8_t* strips_a, const uint8_t* strips_b, int frame_counter, int hscroll,
                  const uint8_t* bitmap, int blend, int progress, uint16_t* out);

/* ---- PTS -> field pacing (SURVEY.md 8f-2; push_video video.cpp:1023-1057 + the flip in video_isr :1165-1177) --------
 * "Instant decoder" model: frame k is queued the moment frame k-1 became the current frame, and the line
 * interrupt only advances while a frame is queued. flip_field[k] / flip_line[k] = _frame_counter and line at
 * which frame k becomes _current_frame. Returns the number of whole fields emitted up to and including the one
 * in which the last frame flipped (stops at max_fields). modes (may be NULL = all 0): 1 = show at once, as
 * MpegDecoder::flush_picture(1) pushes the last picture; 2 / 3 also start the poster scroll animation (_animate, animate(),
 * _easd: video.cpp:1041, 1076-1088, 1168-1174): the _ex form reports the _hscroll each field's active lines are drawn with
 * (field_hscroll[field], may be NULL) and keeps the line interrupt running for tail_fields more fields after the last flip. */
long efo_paced_schedule(const int64_t* pts, const int* modes, int n_frames, int ntsc, uint32_t frame_counter0, long max_fields,
                        uint32_t* flip_field, int* flip_line);
long efo_paced_schedule_ex(const int64_t* pts, const int* modes, int n_frames, int ntsc, uint32_t frame_counter0, long max_fields, long tail_fields,
                           uint32_t* flip_field, int* flip_line, int16_t* field_hscroll);

/* ---- trick-mode index (SURVEY.md 8f-4; indexer/indexer.cpp:90-253) --------------------------------------
 * make_index(): table of (PES pts, TS packet number) of every video packet that starts a PES whose payload
 * begins with a sequence header; first_pts = pts of the first one (-1: none), last_pts = pts of the last video
 * PES start (-1: none). len must be a multiple of 188. Returns the number of table entries (stores <= cap). */
int efo_make_index(const uint8_t* ts, size_t len, int64_t* pts, uint32_t* pos188, int cap, int64_t* first_pts, int64_t* last_pts);
/* pts2seq() + pts2pos(): one sample per bin_size ticks from 0 to last-first: the packet number of the table
 * entry nearest in pts (first minimum; distance cast to int, entries at >= 0x7FFFFFF ticks never win, which
 * leaves entry 0). n == 0 gives no samples (the reference indexes an empty vector there). Returns the count. */
int efo_pts2seq(const int64_t* pts, const uint32_t* pos188, int n, int64_t first_pts, int64_t last_pts, uint32_t bin_size,
                uint32_t* samples, int cap);
/* merge_index(): the video.idx image for (main, fast-forward, rewind) streams; struct padding bytes (which the
 * reference leaves indeterminate) are zero here. Returns the image size, 0 if cap is too small. */
size_t efo_build_idx(const uint8_t* const ts[3], const size_t len[3], uint8_t* out, size_t cap);

/* ---- audio (SURVEY.md 8f-3; oracle/ef_oracle_audio.c) ---------------------------------------------------------
 * efo_demux_audio_ts  payload of PID 0x101 / 0x102 as push_audio() receives it (player.cpp:381-432); returns the byte count
 * efo_sbc_frame       one SBC frame -> sb_sample[16][8] (get_samples, sbc_decoder.cpp:274-341); bytes consumed, -1 rejected
 *                     (bad sync, 4 subbands), -2 outside the reference's domain (not mono / not 16 blocks, joint stereo,
 *                     bit pool > 128)
 * efo_sbc_bits        the same frame's header, scale factors and bit allocation (sbc_decoder.cpp:142-233): the sum of the
 *                     8 sample widths, -1 or -2 as efo_sbc_frame; bits[8] = the widths (zero unless the sum is >= 0)
 * efo_sbc_decode      decode_audio() + sbc_decoder() over the pushed bytes (video.cpp:964-986): PCM samples produced
 *                     (stores <= cap_samples), -1 frame 0 rejected, -2 frame 0 outside the domain; a later out-of-domain
 *                     frame re-synthesises the previous samples, like a rejected frame
 * efo_pdm             pdm_second_order (espflix.ino:73-107) from reset state: 2 n words of 16 one-bit samples */
size_t efo_demux_audio_ts(const uint8_t* ts, size_t len, uint8_t* es, size_t cap);
int efo_sbc_frame(const uint8_t* data, size_t len, int32_t sb_sample[16][8]);
int efo_sbc_bits(const uint8_t* data, size_t len, int bits[8]);
long efo_sbc_decode(const uint8_t* es, size_t len, int16_t* pcm, size_t cap_samples);
void efo_pdm(const int16_t* pcm, size_t n, uint16_t* out);

#ifdef __cplusplus
}
#endif
#endif
