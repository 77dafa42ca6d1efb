// espflix_b200/csrc/ef_capi.cu — the C-ABI of libespflix_b200.so (include/espflix_b200.h).
// Context management, submits, launches and read-back. No CPU fallback: every path goes through
// the CUDA kernels in ef_index.cu / ef_decode.cu / ef_composite.cu or fails with EF_ECUDA.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <thread>
#include <vector>

#include "../../include/espflix_b200.h"
#include "../host/ef_indexer.h"
#include "ef_common.cuh"
#include "ef_iso11172_tables.h"
#include <stdlib.h>

// from the other translation units
int ef_build_tables(EfTables* t);
void ef_build_color_tab(uint32_t* tab768, int ntsc);
void ef_build_pal_burst(int16_t* b0, int16_t* b1, int width);
cudaError_t ef_index_upload_constants();
cudaError_t ef_launch_scan(EfDev* Dp, const EfCarryArgs* carry, int n_streams, cudaStream_t st);
cudaError_t ef_launch_pts_resolve(const EfDev* Dp, const uint2* span, const uint32_t* list_off, const int64_t* list_pts, int64_t* carry,
                                  int64_t* last, int64_t* pic_pts, const EfCarryArgs* C, int n_streams, cudaStream_t st);
__global__ void ef_carry_lead_kernel(const uint32_t* held, int n_streams, uint64_t* stream_total, uint32_t* held_in);
__global__ void ef_carry_copy_kernel(const uint8_t* src_es, const uint64_t* src_off, const uint32_t* held, const uint64_t* es_off, uint8_t* es,
                                     uint64_t* pay_off, int n_streams);
__global__ void ef_carry_restart_kernel(const uint8_t* ops, int first, int count, EfCarryArgs C, int64_t* pts_carry, uint8_t* q_es,
                                        const uint64_t* q_off, const uint32_t* q_held_in);
__global__ void ef_prefix_kernel(EfDev* Dp);
__global__ void ef_fill_kernel(EfDev* Dp);
__global__ void ef_ts_len_kernel(const uint8_t* ts, uint64_t n_packets, uint32_t* out_len);
__global__ void ef_ts_copy_kernel(const uint8_t* ts, uint64_t n_packets, const uint32_t* local_off, const uint16_t* pkt_stream, const uint64_t* es_off, uint8_t* es);
__global__ void ef_ts_scan_kernel(const uint32_t* len, const uint64_t* ts_off, uint32_t* local_off, uint16_t* pkt_stream, uint64_t* stream_total);
__global__ void ef_ts_offsets_kernel(const uint64_t* stream_total, int n_streams, uint64_t* es_off, uint8_t* es);
__global__ void ef_pts_packet_kernel(const uint8_t* ts, const uint64_t* ts_off, const uint32_t* local_off, uint32_t* list_off, int64_t* list_pts, uint2* span);
size_t ef_recon_smem_bytes();
cudaError_t ef_decode_configure();
int ef_decode_resident_ctas(int which);
cudaError_t ef_trick_upload_tables();
cudaError_t ef_trick_launch_gather(const uint8_t* frames, const uint32_t* streams, const uint32_t* slots, int count, int fb, uint8_t* dst, cudaStream_t st);
cudaError_t ef_trick_launch_encode(const uint8_t* in, int n_pics, int qscale, uint32_t* slots, uint32_t* slice_len, cudaStream_t st);
cudaError_t ef_trick_launch_assemble(const uint32_t* slots, const uint32_t* slice_len, const uint64_t* pic_dst, const uint8_t* headers, int n_pics,
                                     uint8_t* es, cudaStream_t st);
cudaError_t ef_trick_launch_mux(const uint8_t* es, const EfTrickPic* pics, int n_pics, uint64_t n_packets, uint8_t* out, cudaStream_t st);
__global__ void ef_tsidx_packet_kernel(const uint8_t* ts, const uint64_t* pkt_off, int n_files, uint64_t n_packets, int64_t* pkt_pts, uint8_t* pkt_kind);
__global__ void ef_tsidx_compact_kernel(const uint64_t* pkt_off, const int64_t* pkt_pts, const uint8_t* pkt_kind, int64_t* seq_pts, uint32_t* seq_pos, int64_t* info);
__global__ void ef_tsidx_sample_kernel(const int64_t* seq_pts, const uint32_t* seq_pos, int n, int64_t first_pts, uint32_t bin_size, uint32_t n_samples, uint32_t* samples);
__global__ void ef_audio_len_kernel(const EfAudioState* st, const uint64_t* new_off, const uint32_t* lead, const uint8_t* skip, int n_streams, uint64_t* len);
__global__ void ef_audio_assemble_kernel(const EfAudioState* st, const uint8_t* src, const uint64_t* new_off, const uint32_t* lead, const uint8_t* skip, const uint64_t* blob_off, uint8_t* blob);
__global__ void ef_sbc_probe_kernel(const uint8_t* es, const uint64_t* off, const EfAudioState* st, const uint8_t* ended, int n_streams, int4* plan);
__global__ void ef_sbc_count_kernel(const uint8_t* es, const uint64_t* off, const uint8_t* ended, int n_streams, int4* plan);
__global__ void ef_sbc_matrix_kernel(const uint8_t* es, const uint64_t* off, const int4* plan, const EfAudioState* st, const uint64_t* slot_base, int n_streams, int32_t* vrows, int32_t* sb_last);
__global__ void ef_sbc_window_kernel(const int32_t* vrows, const uint64_t* slot_base, const uint64_t* pcm_off, int n_streams, int16_t* pcm);
__global__ void ef_pdm_kernel(const int16_t* pcm, const uint64_t* pcm_off, int n_streams, EfAudioState* st, uint16_t* pdm);
__global__ void ef_audio_size_kernel(const int4* plan, int n_streams, uint64_t pcm_cap, uint64_t* slot_base, uint64_t* pcm_off, ef_audio_info* info, int* verdict);
cudaError_t ef_launch_audio_commit(EfAudioState* st, const uint8_t* blob, const uint64_t* blob_off, const int4* plan, const uint64_t* slot_base,
                                   const int32_t* vrows, const int32_t* sb_last, const uint8_t* ended, int n_streams, const int* verdict, cudaStream_t cs);
cudaError_t ef_launch_audio_end(const uint8_t* ended, int n_streams, uint8_t* gate_cur, uint8_t* gate_next, uint8_t* skip_next, int next_is_ts,
                                const int* verdict, cudaStream_t cs);
__global__ void ef_audio_ts_packet_kernel(const uint8_t* ts, uint64_t n_packets, uint8_t* start, uint8_t* kind);
__global__ void ef_audio_ts_scan_kernel(const uint64_t* ts_off, int n_files, const uint8_t* start, const uint8_t* kind, const uint8_t* gate_in, uint8_t* gate_out,
                                        uint32_t* lead, uint8_t* skip, uint32_t* out_pos, uint64_t* es_len);
__global__ void ef_audio_ts_copy_kernel(const uint8_t* ts, const uint64_t* ts_off, int n_files, uint64_t n_packets, const uint8_t* start, const uint32_t* out_pos, const uint64_t* es_off, uint8_t* es);
cudaError_t ef_audio_upload_constants();
cudaError_t ef_launch_parse(const EfDev& dev, int pic0, int n_pics, int sm_count, size_t max_slices, cudaStream_t stream);
cudaError_t ef_launch_recon(const EfDev& dev, int pic_rel, int sm_count, size_t n_slots, cudaStream_t stream);
cudaError_t ef_launch_composite(const EfDev* dev, int n_streams, const EfGeometry& g, int fb, int frame_counter, const EfPresent& pr, cudaStream_t stream);
cudaError_t ef_launch_blit(const EfDev* dev, int stream_index, int fb, int line, int x, int width, int frame_counter, uint16_t* dst, cudaStream_t stream);
cudaError_t ef_launch_composite_paced(const EfDev* dev, const EfGeometry& g, const EfFieldDesc* desc, uint64_t n_fields, uint8_t* dst, bool dac8,
                                      cudaStream_t stream, uint64_t* launches, const EfFieldOverlay* fovl, const uint8_t* bitmaps, const uint64_t* total);
__global__ void ef_pace_kernel(const EfPaceState* st, EfPaceState* next, EfPaceRun* run, EfPaceOut* out, const int64_t* pic_pts, const uint32_t* n_pics,
                               const uint32_t* base_pics, const uint8_t* modes, const uint32_t* idle_n, int pic, int max_pictures, int n_streams, int ntsc,
                               const EfOverlayState* ovl, EfOverlayState* ovl_next);
cudaError_t ef_launch_pace_fill(EfPaceState* st, const EfPaceState* next, const EfPaceRun* run, const uint64_t* first, EfFieldDesc* desc, EfOverlayState* ovl,
                                const EfOverlayState* ovl_next, EfFieldOverlay* fovl, int n_streams, const int* chain, cudaStream_t stream);
__global__ void ef_pace_size_kernel(const EfPaceOut* out, int n_streams, uint64_t cap, uint64_t* first, EfPaceOut* info, uint64_t* total, int* chain,
                                    uint32_t* rec);
__global__ void ef_overlay_stage_kernel(EfOverlayState* ovl, uint8_t* slots, const EfOverlayCmd* cmd, const uint8_t* bitmaps, int first);
__global__ void ef_clock_kernel(EfClockState* clk, const EfOverlayState* ovl, EfOverlayState* ovl_clk, uint8_t* bm, const int64_t* pic_pts,
                                const uint32_t* n_pics, const int64_t* pts_last, int pic, int max_pictures, const uint8_t* font, const int16_t* rights);
cudaError_t ef_launch_clock_commit(EfClockState* clk, const EfOverlayState* ovl_clk, const uint8_t* bm, uint8_t* slots, int n_streams, const int* chain,
                                   cudaStream_t stream);
cudaError_t ef_launch_library_resolve(EfLibStream* ls, const EfLibTitle* titles, const int64_t* pts_last, int first, int count, int cmd, int title,
                                      int64_t arg);
cudaError_t ef_launch_library_gather(EfLibStream* ls, const EfLibTitle* titles, const uint32_t* budget, uint32_t packets, int n_streams,
                                     const uint8_t** src, uint64_t* off, uint8_t* end, uint8_t* dst, uint64_t max_bytes, cudaStream_t st,
                                     uint64_t* launches);
static_assert(sizeof(idx_hdr) == 104, "video.idx header: the reference's idx_hdr");
static_assert(sizeof(EfLibStream) == sizeof(ef_library_status), "EfLibStream mirrors ef_library_status");
static_assert(sizeof(EfPaceOut) == sizeof(ef_present_info), "EfPaceOut mirrors ef_present_info");

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return fail(EF_ECUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// the counterpart of CK for calls that return an EF_* code (and have set the message already)
#define TRY(call)                                                                                  \
    do {                                                                                           \
        const int rc_ = (call);                                                                    \
        if (rc_ != EF_OK) return rc_;                                                              \
    } while (0)

int usable_device(int device)
{
    int ndev = 0;
    const cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || device < 0 || ndev <= device)
        return fail(EF_ECUDA, "no usable CUDA device %d (%s); this library has no CPU path", device, cudaGetErrorString(e));
    return EF_OK;
}

// Every entry point runs on its context's device whatever the caller's current device is, and leaves the
// caller's current device as it found it (several contexts on several GPUs may share a host thread).
struct DeviceScope {
    int prev = -1;
    explicit DeviceScope(int dev)
    {
        if (dev < 0 || cudaGetDevice(&prev) != cudaSuccess) { prev = -1; return; }
        if (prev == dev) prev = -1; else cudaSetDevice(dev);
    }
    ~DeviceScope() { if (prev >= 0) cudaSetDevice(prev); }
};

// device frame stores are macroblock-tiled (ef_common.cuh); these kernels convert to/from the two
// host-visible layouts: the I420 dump and the reference's strips (video.h:36-44; player.cpp:33-46).
// mode 0 = I420, 1 = strips. One thread per 8 bytes (8 aligned consecutive bytes never straddle a tile row:
// luma tile rows are 16 bytes, chroma tile rows 8, and 352, 176 and 528 are multiples of 8).
// fb_sel: 0 / 1 = that frame store; -1 = the most recent picture of each stream; -2 - p = picture p of the current
// submit (the store flush_picture() gave it, player.cpp:692)
// fb_snap (optional, fb_sel == -1): the frame store of every stream's most recent picture, frozen by ef_latest_fb_kernel
// when the read-back was requested (the export itself may run while the next submit is already being indexed)
__global__ void ef_latest_fb_kernel(const uint32_t* __restrict__ base_pics, const uint32_t* __restrict__ n_pics, int first, int count, uint8_t* __restrict__ fb_snap)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < count) fb_snap[k] = (uint8_t)((base_pics[first + k] + n_pics[first + k]) & 1u);
}

__global__ void ef_export_frames_kernel(const uint8_t* __restrict__ frames, const uint32_t* __restrict__ base_pics,
                                        const uint32_t* __restrict__ n_pics, int first, int count, int fb_sel, int mode, uint8_t* __restrict__ dst,
                                        const uint8_t* __restrict__ fb_snap = nullptr)
{
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t per = EF_FRAME / 8;
    const uint32_t k = (uint32_t)(t / per), w = (uint32_t)(t % per);
    if (k >= (uint32_t)count) return;
    const int s = first + (int)k;
    const int fb = fb_sel >= 0 ? fb_sel : fb_sel == -1 ? (fb_snap ? (int)fb_snap[k] : (int)((base_pics[s] + n_pics[s]) & 1u)) : (int)((base_pics[s] + (uint32_t)(-2 - fb_sel) + 1u) & 1u);
    const uint8_t* f = frames + ef_frame_offset(s, fb);
    const int b = (int)w * 8;
    const int src = mode == 0 ? ef_i420_to_tiled(b) : ef_strips_to_tiled(b);
    *(uint2*)(dst + (size_t)k * EF_FRAME + b) = *(const uint2*)(f + src);
}

__global__ void ef_import_frame_kernel(uint8_t* __restrict__ frame, const uint8_t* __restrict__ src, int mode)
{
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= EF_FRAME / 4) return;
    const int b = (int)w * 4;
    const int dst = mode == 0 ? ef_i420_to_tiled(b) : ef_strips_to_tiled(b);
    *(uint32_t*)(frame + dst) = *(const uint32_t*)(src + b);
}

__global__ void ef_reset_seq_kernel(EfDev* Dp)
{
    EfDev& D = *Dp;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= D.n_streams) return;
    EfSeq* q = D.seq + (size_t)s * (D.max_seq + 1);
    for (int n = 0; n < 128; n++) q->qz[n] = D.tables->qz[n];
    q->mb_width = 22; q->mb_height = 12; q->valid = 1; q->custom = 0; q->fp_rs = 0;
    D.n_pics[s] = 0; D.base_pics[s] = 0; D.n_seq[s] = 0;
}

// ef_restart_streams: one thread per stream of [first, first + count). op 1 = MpegDecoder::reset() + video_reset()
// (player.cpp:439-453, video.cpp:1070-1074): get_pts() back to -1 (the carried _pts stays), the SBC ring and the learned
// frame size cleared (the filter memory, the last subband samples and the modulator stay), the display latches a new
// origin; ended[s] marks the stream for ef_audio_end_kernel, which shuts its demux gate. op 2 = video_pause(0)
// (video.cpp:1060-1068): the new origin only. Null arrays belong to subsystems that were never enabled.
__global__ void ef_restart_kernel(const uint8_t* __restrict__ ops, int first, int count, EfPaceState* __restrict__ pace, int64_t* __restrict__ pts_last,
                                  EfAudioState* __restrict__ aud, uint8_t* __restrict__ ended)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const int s = first + k, op = ops[k];
    if (ended) ended[s] = op == 1;
    if (!op) return;
    if (pace) pace[s].fc_origin = 0;
    if (op != 1) return;
    if (pts_last) pts_last[s] = -1;
    if (aud) { aud[s].frame_size = 0; aud[s].carry_len = 0; }
}

}  // namespace

// Device buffers of the audio decode whose size follows the frames of one call, grown on demand. The stateless calls
// use a scratch of their own, a context keeps one.
struct AudioScratch {
    enum { PLAN, SB_LAST, SLOT, POFF, VROWS, PCM, PDM, INFO, VERDICT, N };
    void* p[N] = {};
    size_t cap[N] = {};
    ~AudioScratch() { for (void* q : p) if (q) cudaFree(q); }
    cudaError_t get(int k, size_t bytes, void** out)
    {
        if (cap[k] < bytes) {
            if (p[k]) cudaFree(p[k]);
            p[k] = nullptr; cap[k] = 0;
            const cudaError_t e = cudaMalloc(&p[k], bytes);
            if (e != cudaSuccess) return e;
            cap[k] = bytes;
        }
        *out = p[k];
        return cudaSuccess;
    }
    bool fits(int k, size_t bytes) const { return cap[k] >= bytes; }
};

struct ef_ctx {
    ef_config cfg;
    int sm_count = 0;
    EfDev h;                   // host copy of the device context
    EfDev* d = nullptr;           // = dd[active]
    // everything the context owns, released by ef_destroy: device memory (dev_alloc), pinned host memory (host_alloc), events (event)
    std::vector<void*> allocs, pinned;
    std::vector<cudaEvent_t> events;
    // Two elementary-stream buffers: a submit uploads into the back one on an internal stream while
    // the kernels of the previous submit still read the front one; ef_index flips them.
    uint8_t* d_es2[2] = { nullptr, nullptr };
    uint64_t* d_es_off2[2] = { nullptr, nullptr };
    EfDev* dd[2] = { nullptr, nullptr };          // device copies of `h`, one per ES buffer
    uint64_t* h_off[2] = { nullptr, nullptr };    // pinned copies of the offsets of the submit in flight
    int active = 0, pending = -1;
    cudaStream_t up_stream = nullptr, down_stream = nullptr;
    cudaEvent_t ev_user = nullptr, ev_up_done[2] = { nullptr, nullptr }, ev_buf_free[2] = { nullptr, nullptr };
    cudaEvent_t ev_export = nullptr, ev_down_done[2] = { nullptr, nullptr };
    uint8_t* d_fb_snap[2] = { nullptr, nullptr };  // per staging buffer: frame store of every stream's latest picture at request time
    cudaEvent_t ev_frames_read = nullptr;         // the asynchronous read-back has finished reading the frame stores (its export kernel runs on the read-back stream)
    bool frames_read_pending = false;
    uint8_t* d_stage2[2] = { nullptr, nullptr };  // read-back staging of ef_read_latest_i420(_async), alternating
    size_t stage2_bytes[2] = { 0, 0 };
    int stage_idx = 0;
    uint8_t* d_ts = nullptr;  // TS staging (same capacity) + packet tables, allocated on first TS submit
    uint32_t* d_pkt_len = nullptr;
    uint32_t* d_pkt_off = nullptr;   // payload offset of a packet inside its stream's ES
    uint16_t* d_pkt_stream = nullptr;
    uint64_t* d_stream_total = nullptr;
    uint64_t* d_ts_off = nullptr;
    uint8_t* d_stage = nullptr;      // read-back staging (I420 / strips), one frame
    uint32_t* d_color_tab = nullptr;
    int16_t* d_pal_burst = nullptr;
    uint8_t* d_overlay = nullptr;     // _video_composite bitmap, 16 x 80
    EfPresent present = { 0, 0, 0, nullptr };
    bool indexed = false, submitted = false, video = false;
    uint64_t launches = 0;
    uint64_t es_bytes = 0;
    bool profiling = false;                       // ef_set_profiling: CUDA events around K0 / K1a / K1b
    cudaEvent_t ev_prof[5] = { nullptr, nullptr, nullptr, nullptr, nullptr };
    bool prof_index = false, prof_decode = false;
    // audio (ef_audio_enable): every TS submit also demuxes PID 0x101 / 0x102 into the audio staging of its ES buffer;
    // ef_decode_audio continues every stream's SBC decode from d_aud_state
    bool audio = false;
    bool aud_ts[2] = { false, false };            // ES buffer b holds the demuxed audio of a TS submit
    bool aud_unconsumed = false;                  // the current submit's audio has not been through ef_decode_audio yet
    EfAudioState* d_aud_state = nullptr;          // [n_streams]
    uint8_t* d_aud2[2] = { nullptr, nullptr };    // per ES buffer: audio bytes of its submit, back to back
    uint64_t* d_aud_off2[2] = { nullptr, nullptr };
    uint8_t* d_gate2[2] = { nullptr, nullptr };   // per ES buffer: demux gate of every stream after its submit
    uint32_t* d_lead2[2] = { nullptr, nullptr };  // per ES buffer: audio bytes before the first PES start
    uint8_t* d_skip2[2] = { nullptr, nullptr };   // per ES buffer: drop those (the stream ended after the scan)
    uint8_t* d_aud_start = nullptr;               // per TS packet: payload start, kind, output position
    uint8_t* d_aud_kind = nullptr;
    uint32_t* d_aud_pos = nullptr;
    uint64_t* d_aud_len = nullptr;                // [n_streams + 1]
    uint8_t* d_blob = nullptr;                    // one call's input: held-back bytes + new bytes of every stream
    uint64_t* d_blob_len = nullptr;
    uint64_t* d_blob_off = nullptr;
    uint8_t* d_ended = nullptr;
    uint8_t* h_ended = nullptr;                   // pinned
    AudioScratch aud_scratch;
    // ef_decode_audio_async: whether a call is outstanding, whether it took the current submit's audio, and its verdict
    // (pinned, written by the call's stream). ev_aud_done follows every audio call; ev_ended_free the upload of h_ended.
    bool aud_async = false, aud_async_new = false;
    int aud_async_rc = EF_OK;
    int* h_aud_verdict = nullptr;                 // pinned
    cudaEvent_t ev_aud_done = nullptr, ev_ended_free = nullptr;
    // presentation timestamps (ef_pts_enable): every TS submit also lists the video PES starts with a valid PTS of every
    // stream in its ES buffer's list; ef_index resolves the PTS of every picture from it
    bool pts = false;
    bool pts_resolved = false;                    // the last ef_index ran the resolve pass (ef_picture_pts has something to report)
    uint32_t* d_pts_off2[2] = { nullptr, nullptr };   // per ES buffer, one entry per packet: stream-local ES offset of the PES payload
    int64_t* d_pts_val2[2] = { nullptr, nullptr };    // ... and its PTS
    uint2* d_pts_span2[2] = { nullptr, nullptr };     // per ES buffer: (first entry, entries) of every stream
    int64_t* d_pts_carry = nullptr;               // [n_streams] the last valid PTS of all submits so far (the reference's _pts)
    int64_t* d_pts_last = nullptr;                // [n_streams] PTS of the most recent picture (get_pts())
    int64_t* d_pic_pts = nullptr;                 // [n_streams][max_pictures] PTS of every picture of the current submit
    // paced presentation (ef_present_enable): every stream's display, advanced by ef_present_picture / ef_present_idle
    bool paced = false;
    bool pace_indexed = false;                    // an ef_index followed ef_present_enable: its pictures are to be presented
    int pace_ntsc = 1;                            // the standard, fixed at ef_present_enable
    int pace_format = EF_FIELD_U16;               // what the present calls write (ef_present_format), fixed at ef_present_enable
    int pace_next = 0;                            // the picture index ef_present_picture takes next
    int pace_npics = -1;                          // picture indices of the current submit (-1: not read yet)
    int pace_p0 = 0;                              // first picture index of the current K1a range
    int pace_parse_at = 0;                        // the picture index whose present call runs the next K1a
    EfPaceState* d_pace = nullptr;                // [n_streams]
    EfPaceState* d_pace_next = nullptr;           // [n_streams] the state after the call being made
    EfPaceRun* d_pace_run = nullptr;              // [n_streams]
    EfPaceOut* d_pace_out = nullptr;              // [n_streams]
    EfPaceOut* h_pace_out = nullptr;              // pinned
    uint32_t* h_pace_npics = nullptr;             // pinned: the picture indices of the submit, copied by ef_index
    cudaEvent_t ev_indexed = nullptr;             // ef_index has finished (its stream)
    uint64_t* d_pace_first = nullptr;             // [n_streams] output offset of every stream's fields
    uint64_t* h_pace_first = nullptr;             // pinned
    uint32_t* d_pace_arg = nullptr;               // [n_streams] modes (bytes) or idle field counts
    uint32_t* h_pace_arg = nullptr;               // pinned
    EfFieldDesc* d_desc = nullptr;                // one per emitted field, grown on demand
    uint64_t desc_cap = 0;
    // overlay of paced presentation (ef_present_overlay): allocated by its first call; until then the present calls run the
    // kernels they ran before
    EfOverlayState* d_ovl = nullptr;              // [n_streams]
    EfOverlayState* d_ovl_next = nullptr;         // [n_streams] the state after the call being made
    uint8_t* d_ovl_slots = nullptr;               // [n_streams][2][1280] latched and staged bitmap
    uint8_t* d_ovl_in = nullptr;                  // [n_streams][1280] the bitmaps of one ef_present_overlay call
    EfOverlayCmd* d_ovl_cmd = nullptr;            // [n_streams]
    EfFieldOverlay* d_fovl = nullptr;             // one per emitted field, beside d_desc
    uint64_t fovl_cap = 0;
    // clock of paced presentation: the glyph atlas (ef_present_font) and, from the first ef_present_clock, every stream's clock; until
    // then the present calls run the kernels they ran before
    uint8_t* d_font = nullptr;                    // [16][1024] _font8
    int16_t* d_font_rights = nullptr;             // _font8_rights
    EfClockState* d_clk = nullptr;                // [n_streams]
    EfOverlayState* d_ovl_clk = nullptr;          // [n_streams] the overlay state with the clock's changes staged: ef_pace_kernel's input
    uint8_t* d_clk_bm = nullptr;                  // [n_streams][1280] the bitmap a call rendered, until its commit
    uint8_t* d_restart_ops = nullptr;             // [n_streams] the ops of one ef_restart_streams call, allocated by its first call
    // ef_present_*_async, allocated by the first call: the chain of calls since the last ef_present_wait (or the last call that
    // resolved it) and its verdict. d_pace_chain = { a call did not fit, calls that took effect }, copied to h_pace_chain at the end
    // of every call, which then records ev_pace_done. chain_next / chain_pic: pace_next before each call of the chain, and its pic.
    bool pace_async = false;                      // a chain is outstanding
    int pace_async_rc = EF_OK, pace_async_n = 0;  // the result of the last resolved chain
    int* d_pace_chain = nullptr;
    int* h_pace_chain = nullptr;                  // pinned
    uint64_t* d_pace_total = nullptr;             // the fields of the call being made (0 when it does not take effect)
    std::vector<int> chain_next, chain_pic;
    cudaEvent_t ev_pace_done = nullptr;
    // modes / idle field counts of async calls: a pinned ring, slot k free again once ev_pace_ring[k] has passed
    enum { kPaceRing = 16 };
    uint32_t* h_pace_ring = nullptr;              // pinned [kPaceRing][n_streams]
    cudaEvent_t ev_pace_ring[kPaceRing] = {};
    int pace_ring_i = 0;
    // TS submits cut anywhere (ef_carry_enable): K0 leaves every stream's unfinished access unit in the front ES buffer and its
    // length in d_held; the next upload copies it to the head of the stream's region once that ef_index has finished (ev_scanned)
    bool carry = false;
    uint32_t max_carry = 0;
    uint32_t* d_held = nullptr;                   // [n_streams] EfCarryArgs::held
    uint32_t* d_held_code = nullptr;              // [n_streams] EfCarryArgs::held_code
    uint8_t* d_carry_flags = nullptr;             // [n_streams] EfCarryArgs::flags
    uint32_t* d_held_in2[2] = { nullptr, nullptr };   // per ES buffer: held bytes at the head of each stream's region
    uint8_t* d_end2[2] = { nullptr, nullptr };    // per ES buffer: ef_end_streams flags of its submit
    std::vector<uint8_t> h_end2[2];               // their host copies (merged over the calls for one submit)
    uint64_t* d_pay_off = nullptr;                // [n_streams + 1] where each stream's new payload starts in the back buffer
    int64_t* d_pts_hold = nullptr;                // [n_streams] EfCarryArgs::pts_hold
    int64_t* d_pts_pre = nullptr;                 // [n_streams] EfCarryArgs::pts_pre
    cudaEvent_t ev_scanned = nullptr;             // the last ef_index has written d_held (and resolved the held picture's pts)
    // the title library (ef_library_*): allocated by the first ef_library_add; until then nothing of it exists
    std::vector<EfLibTitle> lib_titles;           // host copies of the titles' records
    EfLibTitle* d_lib_titles = nullptr;           // [lib_cap]
    size_t lib_cap = 0;
    EfLibStream* d_lib = nullptr;                 // [n_streams] every stream's title, speed, state, file, cursor and pos
    uint8_t* d_lib_stage = nullptr;               // [es_capacity + 64] the gathered TS of a library submit
    const uint8_t** d_lib_src = nullptr;          // [n_streams] where each stream's run starts
    uint64_t* d_lib_off = nullptr;                // [n_streams + 1] each stream's run in the staging buffer
    uint8_t* d_lib_end = nullptr;                 // [n_streams] the streams the submit ends
    uint32_t* d_lib_budget = nullptr;             // [n_streams] per-stream packet budgets of a submit
    cudaEvent_t ev_lib_staged = nullptr;          // the upload has copied the staging buffer
    bool lib_submit = false;                      // the pending submit is a library submit (its ends are the library's)
};

namespace {

template <typename T>
int dev_alloc(ef_ctx* c, T** p, size_t n)
{
    void* v = nullptr;
    cudaError_t e = cudaMalloc(&v, n * sizeof(T) + 256);
    if (e != cudaSuccess) return fail(EF_ECUDA, "cudaMalloc(%zu bytes): %s", n * sizeof(T), cudaGetErrorString(e));
    c->allocs.push_back(v);
    *p = (T*)v;
    return EF_OK;
}

template <typename T>
int host_alloc(ef_ctx* c, T** p, size_t n)             // pinned
{
    CK(cudaHostAlloc((void**)p, n * sizeof(T), cudaHostAllocDefault));
    c->pinned.push_back(*p);
    return EF_OK;
}

int event(ef_ctx* c, cudaEvent_t* e, bool timing = false)
{
    CK(timing ? cudaEventCreate(e) : cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    c->events.push_back(*e);
    return EF_OK;
}

// streams [first, first + count) of the context; args_ok: the per-stream arguments are there (when count > 0)
int stream_range(const ef_ctx* c, int first, int count, bool args_ok = true)
{
    const int n = c->cfg.n_streams;
    if (first < 0 || count < 0 || first > n || count > n - first || (count && !args_ok))
        return fail(EF_EINVAL, "streams [%d, %d + %d) out of range", first, first, count);
    return EF_OK;
}

// write the host copy of the device context to both device copies (they differ in the ES buffer only)
int push_dev(ef_ctx* c)
{
    for (int b = 0; b < 2; b++) {
        EfDev t = c->h;
        t.es = c->d_es2[b]; t.es_off = c->d_es_off2[b];
        CK(cudaMemcpy(c->dd[b], &t, sizeof(EfDev), cudaMemcpyHostToDevice));
    }
    return EF_OK;
}

// the carry state of a carrying context, as K0 and the PTS resolve pass of ES buffer b see it
EfCarryArgs carry_args(ef_ctx* c, int b)
{
    EfCarryArgs a;
    a.held = c->d_held; a.held_code = c->d_held_code; a.flags = c->d_carry_flags; a.end = c->d_end2[b]; a.held_in = c->d_held_in2[b];
    a.pts_hold = c->d_pts_hold; a.pts_pre = c->d_pts_pre; a.max_carry = c->max_carry;
    return a;
}

// every stream holds nothing (ef_carry_enable, ef_reset)
int carry_clear(ef_ctx* c)
{
    const size_t n = (size_t)c->cfg.n_streams;
    CK(cudaMemset(c->d_held, 0, n * 4));
    CK(cudaMemset(c->d_held_code, 0xFF, n * 4));
    CK(cudaMemset(c->d_carry_flags, 0, n));
    CK(cudaMemset(c->d_pts_hold, 0xFF, n * 8));
    CK(cudaMemset(c->d_pts_pre, 0xFF, n * 8));
    for (int b = 0; b < 2; b++) {
        CK(cudaMemset(c->d_held_in2[b], 0, n * 4));
        CK(cudaMemset(c->d_end2[b], 0, n));
        c->h_end2[b].assign(n, 0);
    }
    return EF_OK;
}

// Replace the device allocation *p of old_n elements (or none) by one of new_n, zero-filled after the old contents when keep.
// The old one is freed (cudaFree waits for the whole device); whatever else may still use it, the caller has waited for.
template <typename T>
int dev_grow(ef_ctx* c, T** p, size_t old_n, size_t new_n, bool keep)
{
    T* q = nullptr;
    TRY(dev_alloc(c, &q, new_n));
    if (keep) {
        CK(cudaMemset(q, 0, new_n * sizeof(T)));
        CK(cudaMemcpy(q, *p, old_n * sizeof(T), cudaMemcpyDeviceToDevice));
    }
    for (size_t i = 0; *p && i < c->allocs.size(); i++)
        if (c->allocs[i] == (void*)*p) { cudaFree(*p); c->allocs.erase(c->allocs.begin() + (long)i); break; }
    *p = q;
    return EF_OK;
}

int ensure_stage(ef_ctx* c)
{
    if (!c->d_stage) TRY(dev_alloc(c, &c->d_stage, EF_FRAME));
    return EF_OK;
}

int resolve_fb(ef_ctx* c, int stream_index, int fb, int* out)
{
    if (stream_index < 0 || stream_index >= c->cfg.n_streams) return fail(EF_EINVAL, "stream index %d out of range", stream_index);
    if (fb == 0 || fb == 1) { *out = fb; return EF_OK; }
    if (fb != -1) return fail(EF_EINVAL, "fb must be 0, 1 or -1");
    uint32_t a = 0, b = 0;
    CK(cudaMemcpy(&a, c->h.base_pics + stream_index, 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&b, c->h.n_pics + stream_index, 4, cudaMemcpyDeviceToHost));
    *out = (int)((a + b) & 1u);
    return EF_OK;
}

// picture indices of the submit the last ef_index made current (waits for that ef_index the first time per submit; work
// on other streams, such as an audio decode, runs on)
int pace_pictures(ef_ctx* c)
{
    if (c->pace_npics >= 0) return EF_OK;
    CK(cudaEventSynchronize(c->ev_indexed));
    c->pace_npics = (int)*c->h_pace_npics;
    return EF_OK;
}

}  // namespace

extern "C" {

const char* ef_last_error(void) { return g_err; }
const char* ef_version(void) { return "espflix_b200 0.1 (sm_90a)"; }

int ef_create(ef_ctx** out, const ef_config* cfg)
{
    if (!out || !cfg) return fail(EF_EINVAL, "null argument");
    if (cfg->n_streams < 1 || cfg->n_streams > 65535 || cfg->max_pictures < 1 || cfg->max_pictures > 4096 ||
        cfg->max_slices_per_picture < 1 || cfg->max_slices_per_picture > 176 || cfg->es_capacity < 16)
        return fail(EF_EINVAL, "bad config (n_streams=%d max_pictures=%d max_slices_per_picture=%d es_capacity=%zu)",
                    cfg->n_streams, cfg->max_pictures, cfg->max_slices_per_picture, cfg->es_capacity);
    TRY(usable_device(cfg->device));
    DeviceScope scope_(cfg->device);
    ef_ctx* c = new ef_ctx();
    c->cfg = *cfg;
    struct Guard {                                // every failure path below releases what has been created so far
        ef_ctx* c;
        ~Guard() { if (c) ef_destroy(c); }
    } guard{ c };
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, cfg->device));
    c->sm_count = prop.multiProcessorCount;
    if ((size_t)prop.sharedMemPerBlockOptin < ef_recon_smem_bytes()) {
        return fail(EF_ECUDA, "device offers %zu B shared memory per CTA, kernel needs %zu", (size_t)prop.sharedMemPerBlockOptin, ef_recon_smem_bytes());
    }
    CK(ef_decode_configure());
    if (getenv("EF_VERBOSE")) fprintf(stderr, "espflix_b200: %d SMs, resident CTAs per SM: parse %d, reconstruct %d\n", c->sm_count, ef_decode_resident_ctas(0), ef_decode_resident_ctas(1));
    CK(ef_index_upload_constants());

    const int n = cfg->n_streams;
    EfDev& h = c->h;
    memset(&h, 0, sizeof(h));
    h.n_streams = n; h.max_pictures = cfg->max_pictures;
    h.max_slices = cfg->max_pictures * cfg->max_slices_per_picture;
    h.max_seq = cfg->max_pictures;
    for (int b = 0; b < 2; b++) {
        TRY(dev_alloc(c, &c->d_es2[b], cfg->es_capacity + 1024));
        TRY(dev_alloc(c, &c->d_es_off2[b], (size_t)n + 1));
        TRY(dev_alloc(c, &c->dd[b], 1));
        TRY(host_alloc(c, &c->h_off[b], (size_t)n + 1));
        TRY(event(c, &c->ev_up_done[b])); TRY(event(c, &c->ev_buf_free[b])); TRY(event(c, &c->ev_down_done[b]));
    }
    TRY(event(c, &c->ev_user)); TRY(event(c, &c->ev_export)); TRY(event(c, &c->ev_frames_read));
    TRY(event(c, &c->ev_indexed)); TRY(event(c, &c->ev_aud_done)); TRY(event(c, &c->ev_ended_free));
    CK(cudaStreamCreateWithFlags(&c->up_stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->down_stream, cudaStreamNonBlocking));
    TRY(dev_alloc(c, &h.frames, (size_t)n * 2 * EF_FRAME + 1024));
    TRY(dev_alloc(c, &h.seq, (size_t)n * (h.max_seq + 1)));
    TRY(dev_alloc(c, &h.pics, (size_t)n * h.max_pictures));
    TRY(dev_alloc(c, &h.slice_off, (size_t)n * h.max_slices));
    TRY(dev_alloc(c, &h.slice_code, (size_t)n * h.max_slices));
    TRY(dev_alloc(c, &h.n_pics, n)); TRY(dev_alloc(c, &h.base_pics, n)); TRY(dev_alloc(c, &h.n_seq, n));
    TRY(dev_alloc(c, &h.pic_pref, (size_t)n * h.max_pictures));
    TRY(dev_alloc(c, &h.pic_total, h.max_pictures)); TRY(dev_alloc(c, &h.pic_base, h.max_pictures)); TRY(dev_alloc(c, &h.cursor, h.max_pictures));
    h.work_capacity = (size_t)n * h.max_slices;
    TRY(dev_alloc(c, &h.work, h.work_capacity));
    TRY(dev_alloc(c, &h.info, 8));
    EfTables* dt;
    TRY(dev_alloc(c, &dt, 1));
    {   // macroblock records: as many picture indices per K1a launch as fit in 2 GiB
        const size_t per_pic = (size_t)n * EF_MBW_MAX * EF_MBH_MAX * (sizeof(EfMbRec) + 4);
        size_t k = ((size_t)2 << 30) / per_pic;
        if (const char* e = getenv("EF_REC_PICS")) { const long v = atol(e); if (v >= 1) k = (size_t)v; }   // tuning / test knob
        h.rec_pics = (int)(k < 1 ? 1 : k > (size_t)h.max_pictures ? (size_t)h.max_pictures : k);
        const size_t slots = (size_t)h.rec_pics * n * EF_MBW_MAX * EF_MBH_MAX;
        TRY(dev_alloc(c, &h.mb_info, slots)); TRY(dev_alloc(c, &h.mb_rec, slots));
        TRY(dev_alloc(c, &h.parse_cursor, (size_t)h.rec_pics + 4));      // [0] K1a, [1..] one per K1b launch
        h.recon_cursor = h.parse_cursor + 1;
        TRY(dev_alloc(c, &h.coef, 3 * (cfg->es_capacity + 1024) + 1024));
    }
    TRY(dev_alloc(c, &c->d_color_tab, 768)); TRY(dev_alloc(c, &c->d_pal_burst, 128)); TRY(dev_alloc(c, &c->d_overlay, 1280));
    c->present.bitmap = c->d_overlay;
    if (cfg->fields) { h.field_stride = EF_PAL_FIELD_SAMPLES; TRY(dev_alloc(c, &h.fields, (size_t)n * h.field_stride)); }
    h.es = c->d_es2[0]; h.es_off = c->d_es_off2[0]; h.tables = dt;
    c->d = c->dd[0];
    h.color_tab = c->d_color_tab; h.pal_burst = c->d_pal_burst;

    EfTables t;
    const int bad = ef_build_tables(&t);
    if (bad) return fail(EF_EINVAL, "internal: VLC table %d does not fit its lookup shape", bad);
    CK(cudaMemcpy(dt, &t, sizeof(t), cudaMemcpyHostToDevice));
    for (int b = 0; b < 2; b++) {
        CK(cudaMemset(c->d_es2[b], 0, cfg->es_capacity + 1024));
        CK(cudaMemset(c->d_es_off2[b], 0, ((size_t)n + 1) * 8));
    }
    CK(cudaMemset(c->d_overlay, 0, 1280));
    TRY(push_dev(c));
    TRY(ef_reset(c));
    TRY(ef_video_init(c, 1));
    guard.c = nullptr;
    *out = c;
    return EF_OK;
}

void ef_destroy(ef_ctx* c)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return;
    cudaDeviceSynchronize();
    for (void* p : c->allocs) cudaFree(p);
    for (void* p : c->pinned) cudaFreeHost(p);
    for (cudaEvent_t e : c->events) cudaEventDestroy(e);
    if (c->up_stream) cudaStreamDestroy(c->up_stream);
    if (c->down_stream) cudaStreamDestroy(c->down_stream);
    delete c;
}

// an asynchronous read-back may still be reading the frame stores on the read-back stream: host-driven writers wait for it
static int wait_frames_read(ef_ctx* c)
{
    if (c->frames_read_pending) { CK(cudaEventSynchronize(c->ev_frames_read)); c->frames_read_pending = false; }
    return EF_OK;
}

// An outstanding ef_decode_audio_async: wait for it and settle the bookkeeping only the host keeps (whether the current
// submit's audio has been consumed). Every call whose outcome depends on that resolves first.
static int audio_resolve(ef_ctx* c)
{
    if (!c->aud_async) return EF_OK;
    CK(cudaEventSynchronize(c->ev_aud_done));
    c->aud_async = false;
    c->aud_async_rc = *c->h_aud_verdict ? EF_ENOMEM : EF_OK;
    if (c->aud_async_rc == EF_OK && c->aud_async_new) c->aud_unconsumed = false;
    return EF_OK;
}

// An outstanding chain of ef_present_*_async calls: wait for it and settle what only the host keeps. After a call that did not
// fit, the next picture index rolls back to that call's, and when a picture call of the chain did not take effect its records
// are gone (the size kernel zeroed them): the next picture call parses again from there.
static int pace_resolve(ef_ctx* c)
{
    if (!c->pace_async) return EF_OK;
    CK(cudaEventSynchronize(c->ev_pace_done));
    c->pace_async = false;
    const int failed = c->h_pace_chain[0], done = c->h_pace_chain[1];
    c->pace_async_n = done;
    c->pace_async_rc = failed ? EF_ENOMEM : EF_OK;
    if (failed) {
        c->pace_next = c->chain_next[(size_t)done];
        for (size_t i = (size_t)done; i < c->chain_pic.size(); i++)
            if (c->chain_pic[i] >= 0) { c->pace_parse_at = c->pace_next; break; }
    }
    return EF_OK;
}

int ef_reset(ef_ctx* c)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(wait_frames_read(c));
    TRY(audio_resolve(c));
    TRY(pace_resolve(c));
    CK(cudaMemset(c->h.frames, 0, (size_t)c->cfg.n_streams * 2 * EF_FRAME + 1024));     // Frame::init zero-fills (player.cpp:25)
    ef_reset_seq_kernel<<<(c->cfg.n_streams + 127) / 128, 128>>>(c->d);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaMemset(c->h.info, 0, 32));
    if (c->audio) {                                       // every stream's audio starts over; audio stays enabled
        CK(cudaStreamSynchronize(c->up_stream));          // a queued submit's demux may still read a gate
        CK(cudaMemset(c->d_aud_state, 0, (size_t)c->cfg.n_streams * sizeof(EfAudioState)));
        for (int b = 0; b < 2; b++) { CK(cudaMemset(c->d_gate2[b], 0, (size_t)c->cfg.n_streams)); c->aud_ts[b] = false; }
        c->aud_unconsumed = false;
    }
    if (c->pts) {                                         // every stream's PTS starts over at -1; PTS stays enabled
        CK(cudaDeviceSynchronize());                      // a resolve pass on a caller's stream may still write them
        CK(cudaMemset(c->d_pts_carry, 0xFF, (size_t)c->cfg.n_streams * 8));
        CK(cudaMemset(c->d_pts_last, 0xFF, (size_t)c->cfg.n_streams * 8));
        c->pts_resolved = false;
    }
    if (c->paced)                                         // video_reset() (video.cpp:1070-1074): every display latches a new origin
        CK(cudaMemset2D((uint8_t*)c->d_pace + offsetof(EfPaceState, fc_origin), sizeof(EfPaceState), 0, 4, (size_t)c->cfg.n_streams));
    if (c->carry) {                                       // every stream's held bytes are dropped; carry stays enabled
        CK(cudaDeviceSynchronize());
        TRY(carry_clear(c));
    }
    CK(cudaDeviceSynchronize());
    c->indexed = false; c->submitted = false; c->pending = -1;
    c->pace_indexed = false;
    return EF_OK;
}

// When a restart may fall between the current submit and the next one: every picture index of the current submit presented, and
// its audio consumed (EF_ESTATE otherwise). `what` names the caller in the message.
static int restart_ready(ef_ctx* c, const char* what)
{
    TRY(pace_resolve(c));
    if (c->paced && c->pace_indexed) {                    // the schedule of the current submit must be complete
        TRY(pace_pictures(c));
        if (c->pace_next < c->pace_npics) return fail(EF_ESTATE, "%s while pictures %d..%d of the current submit are not presented", what, c->pace_next, c->pace_npics - 1);
    }
    TRY(audio_resolve(c));
    if (c->audio && c->aud_unconsumed) return fail(EF_ESTATE, "%s before ef_decode_audio consumed the current submit's audio", what);
    return EF_OK;
}

// The restart itself (ops checked, restart_ready passed): ef_restart_streams and ef_library_command
static int restart_apply(ef_ctx* c, int first, int count, const uint8_t* ops)
{
    const int n = c->cfg.n_streams;
    bool any_reset = false;
    for (int i = 0; i < count; i++) any_reset |= ops[i] == 1;
    if (!count) return EF_OK;
    CK(cudaDeviceSynchronize());
    const bool audio = c->audio && any_reset;
    if (!c->d_restart_ops) TRY(dev_alloc(c, &c->d_restart_ops, (size_t)n));
    CK(cudaMemcpy(c->d_restart_ops, ops, (size_t)count, cudaMemcpyHostToDevice));
    if (audio) CK(cudaMemset(c->d_ended, 0, (size_t)n));
    ef_restart_kernel<<<(count + 127) / 128, 128>>>(c->d_restart_ops, first, count, c->paced ? c->d_pace : nullptr, c->pts ? c->d_pts_last : nullptr,
                                                     audio ? c->d_aud_state : nullptr, audio ? c->d_ended : nullptr);
    CK(cudaGetLastError());
    c->launches++;
    if (audio) {                                          // the demux gates: the current one, and that of a submit queued behind it
        const int p = c->pending;
        CK(ef_launch_audio_end(c->d_ended, n, c->d_gate2[c->active], p >= 0 ? c->d_gate2[p] : nullptr, p >= 0 ? c->d_skip2[p] : nullptr,
                               p >= 0 && c->aud_ts[p], nullptr, 0));
        c->launches++;
    }
    if (c->carry && any_reset) {                          // MpegDecoder::reset() clears the bit reader (player.cpp:446-447)
        const int p = c->pending;
        ef_carry_restart_kernel<<<(count * 32 + 127) / 128, 128>>>(c->d_restart_ops, first, count, carry_args(c, c->active), c->pts ? c->d_pts_carry : nullptr,
                                                                   p >= 0 ? c->d_es2[p] : nullptr, p >= 0 ? c->d_es_off2[p] : nullptr,
                                                                   p >= 0 ? c->d_held_in2[p] : nullptr);
        CK(cudaGetLastError());
        c->launches++;
    }
    CK(cudaDeviceSynchronize());
    return EF_OK;
}

// Per-stream restart between the current submit and the next one (queued or not). Synchronous: everything already
// queued on the device (a resolve pass, a queued submit's demux) has finished before the state changes.
int ef_restart_streams(ef_ctx* c, int first, int count, const uint8_t* ops)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(stream_range(c, first, count, ops));
    for (int i = 0; i < count; i++)
        if (ops[i] > 2) return fail(EF_EINVAL, "op %d of stream %d is not 0..2", ops[i], first + i);
    TRY(restart_ready(c, "ef_restart_streams"));
    return restart_apply(c, first, count, ops);
}

// Uploads go to the BACK elementary-stream buffer on the context's own upload stream, so that a
// caller that has pinned its input can submit batch k+1 while the kernels of batch k still run
// (the producer side of the reference's Buffer queue is asynchronous in the same way). ef_index()
// makes the compute stream wait for the upload and flips the buffers.
static int submit_common(ef_ctx* c, const uint8_t* src, const uint64_t* off, bool host, bool ts, cudaStream_t st)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !src || !off) return fail(EF_EINVAL, "null argument");
    if (c->carry && !ts) return fail(EF_ESTATE, "ES submits on a carrying context: submit transport streams");
    const int n = c->cfg.n_streams;
    const int b = c->pending >= 0 ? c->pending : (c->active ^ 1);
    CK(cudaEventSynchronize(c->ev_up_done[b]));          // the pinned offsets of the previous upload into this buffer are free again
    uint64_t* hoff = c->h_off[b];
    if (host) memcpy(hoff, off, ((size_t)n + 1) * 8);
    else { CK(cudaMemcpyAsync(hoff, off, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st)); }
    const uint64_t total = hoff[n];
    if (total > c->cfg.es_capacity) return fail(EF_ENOMEM, "submit of %llu bytes exceeds es_capacity %zu", (unsigned long long)total, c->cfg.es_capacity);
    for (int i = 0; i < n; i++) if (hoff[i] > hoff[i + 1]) return fail(EF_EINVAL, "stream offsets must be non-decreasing");
    if (ts) for (int i = 0; i <= n; i++) if (hoff[i] % 188) return fail(EF_EINVAL, "TS stream offsets must be multiples of 188");
    const cudaMemcpyKind kind = host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
    cudaStream_t up = c->up_stream;
    if (!host) {                                          // device-resident input may still be in production on the caller's stream
        CK(cudaEventRecord(c->ev_user, st));
        CK(cudaStreamWaitEvent(up, c->ev_user, 0));
    }
    CK(cudaStreamWaitEvent(up, c->ev_buf_free[b], 0));    // kernels of the submit that last used this buffer are done
    if (c->audio) CK(cudaStreamWaitEvent(up, c->ev_aud_done, 0));   // and the last audio call: it reads this buffer's audio, or
                                                                     // shuts demux gates the demux below reads
    uint8_t* d_es = c->d_es2[b];
    uint64_t* d_es_off = c->d_es_off2[b];
    if (!ts) {
        CK(cudaMemcpyAsync(d_es, src, total, kind, up));
        CK(cudaMemsetAsync(d_es + total, 0, 256, up));
        CK(cudaMemcpyAsync(d_es_off, hoff, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, up));
    } else {
        const uint64_t n_packets = total / 188;
        if (!c->d_ts) {
            TRY(dev_alloc(c, &c->d_ts, c->cfg.es_capacity + 64));
            TRY(dev_alloc(c, &c->d_pkt_len, c->cfg.es_capacity / 188 + 1));
            TRY(dev_alloc(c, &c->d_pkt_off, c->cfg.es_capacity / 188 + 1));
            TRY(dev_alloc(c, &c->d_pkt_stream, c->cfg.es_capacity / 188 + 1));
            TRY(dev_alloc(c, &c->d_stream_total, (size_t)n + 1));
            TRY(dev_alloc(c, &c->d_ts_off, (size_t)n + 1));
        }
        CK(cudaMemcpyAsync(c->d_ts, src, total, kind, up));
        CK(cudaMemcpyAsync(c->d_ts_off, hoff, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, up));
        // packet lengths, every stream's payload bytes and packet positions, the ES offsets, the payload copy; on a carrying
        // context every stream's region starts with its held bytes (known once the last ef_index has run), then the new payload
        const bool carry = c->carry;
        const int a = c->active;
        if (carry || n_packets) {
            if (n_packets) {
                ef_ts_len_kernel<<<(unsigned)((n_packets + 255) / 256), 256, 0, up>>>(c->d_ts, n_packets, c->d_pkt_len);
                CK(cudaGetLastError());
                c->launches++;
            }
            ef_ts_scan_kernel<<<n, 256, 0, up>>>(c->d_pkt_len, c->d_ts_off, c->d_pkt_off, c->d_pkt_stream, c->d_stream_total);
            CK(cudaGetLastError());
            c->launches++;
            if (carry) {
                CK(cudaStreamWaitEvent(up, c->ev_scanned, 0));
                ef_carry_lead_kernel<<<(n + 255) / 256, 256, 0, up>>>(c->d_held, n, c->d_stream_total, c->d_held_in2[b]);
                CK(cudaGetLastError());
                c->launches++;
            }
            ef_ts_offsets_kernel<<<1, 1024, 0, up>>>(c->d_stream_total, n, d_es_off, d_es);
            CK(cudaGetLastError());
            c->launches++;
            if (carry) {
                ef_carry_copy_kernel<<<(n * 32 + 127) / 128, 128, 0, up>>>(c->d_es2[a], c->d_es_off2[a], c->d_held, d_es_off, d_es, c->d_pay_off, n);
                CK(cudaGetLastError());
                c->launches++;
            }
            if (n_packets) {
                ef_ts_copy_kernel<<<(unsigned)((n_packets * 32 + 255) / 256), 256, 0, up>>>(c->d_ts, n_packets, c->d_pkt_off, c->d_pkt_stream,
                                                                                            carry ? c->d_pay_off : d_es_off, d_es);
                CK(cudaGetLastError());
                c->launches++;
            }
        } else CK(cudaMemsetAsync(d_es_off, 0, ((size_t)n + 1) * 8, up));
        if (carry) {
            CK(cudaMemsetAsync(c->d_end2[b], 0, (size_t)n, up));
            c->h_end2[b].assign((size_t)n, 0);
        }
    }
    if (c->pts) {                                         // the video PES starts of this submit, into its ES buffer's list
        if (ts) {
            ef_pts_packet_kernel<<<n, 256, 0, up>>>(c->d_ts, c->d_ts_off, c->d_pkt_off, c->d_pts_off2[b], c->d_pts_val2[b], c->d_pts_span2[b]);
            CK(cudaGetLastError());
            c->launches++;
        } else CK(cudaMemsetAsync(c->d_pts_span2[b], 0, (size_t)n * sizeof(uint2), up));   // ES submits carry no PES
    }
    if (c->audio) {
        // The demux gate of every stream continues from the submit that is current now (the front buffer): submits are
        // demuxed in submit order on this stream, and a submit that replaces a queued one starts from the same gate.
        const uint8_t* gate_in = c->d_gate2[c->active];
        if (ts) {
            const uint64_t n_packets = total / 188;
            if (n_packets) {
                ef_audio_ts_packet_kernel<<<(unsigned)((n_packets + 255) / 256), 256, 0, up>>>(c->d_ts, n_packets, c->d_aud_start, c->d_aud_kind);
                CK(cudaGetLastError());
                c->launches++;
            }
            ef_audio_ts_scan_kernel<<<(n + 63) / 64, 64, 0, up>>>(c->d_ts_off, n, c->d_aud_start, c->d_aud_kind, gate_in, c->d_gate2[b], c->d_lead2[b], c->d_skip2[b],
                                                                  c->d_aud_pos, c->d_aud_len);
            CK(cudaGetLastError());
            ef_ts_offsets_kernel<<<1, 1024, 0, up>>>(c->d_aud_len, n, c->d_aud_off2[b], c->d_aud2[b]);
            CK(cudaGetLastError());
            c->launches += 2;
            if (n_packets) {
                ef_audio_ts_copy_kernel<<<(unsigned)((n_packets * 32 + 255) / 256), 256, 0, up>>>(c->d_ts, c->d_ts_off, n, n_packets, c->d_aud_start, c->d_aud_pos,
                                                                                                  c->d_aud_off2[b], c->d_aud2[b]);
                CK(cudaGetLastError());
                c->launches++;
            }
        } else CK(cudaMemcpyAsync(c->d_gate2[b], gate_in, (size_t)n, cudaMemcpyDeviceToDevice, up));   // ES submits carry no audio
        c->aud_ts[b] = ts;
    }
    CK(cudaEventRecord(c->ev_up_done[b], up));
    c->es_bytes = total;                        // for TS input an upper bound; the exact ES size is on the device
    c->pending = b;
    c->submitted = true; c->indexed = false;
    c->lib_submit = false;
    return EF_OK;
}

int ef_submit_es_host(ef_ctx* c, const uint8_t* es, const uint64_t* off, void* stream) { return submit_common(c, es, off, true, false, (cudaStream_t)stream); }
int ef_submit_es_device(ef_ctx* c, const uint8_t* es, const uint64_t* off, void* stream) { return submit_common(c, es, off, false, false, (cudaStream_t)stream); }
int ef_submit_ts_host(ef_ctx* c, const uint8_t* ts, const uint64_t* off, void* stream) { return submit_common(c, ts, off, true, true, (cudaStream_t)stream); }
int ef_submit_ts_device(ef_ctx* c, const uint8_t* ts, const uint64_t* off, void* stream) { return submit_common(c, ts, off, false, true, (cudaStream_t)stream); }

int ef_index(ef_ctx* c, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->submitted) return fail(EF_ESTATE, "ef_index before any submit");
    if (c->carry && c->pending < 0) return fail(EF_ESTATE, "ef_index without a fresh submit on a carrying context (its held bytes have moved on)");
    cudaStream_t st = (cudaStream_t)stream;
    const int n = c->cfg.n_streams;
    TRY(pace_resolve(c));
    if (c->paced && c->pace_indexed) {                    // the schedule needs every picture of the current submit
        TRY(pace_pictures(c));
        if (c->pace_next < c->pace_npics) return fail(EF_ESTATE, "ef_index while pictures %d..%d of the current submit are not presented", c->pace_next, c->pace_npics - 1);
    }
    if (c->pending >= 0) {                       // a fresh submit: wait for its upload, make it the front buffer
        TRY(audio_resolve(c));
        if (c->audio && c->aud_unconsumed)       // the audio of a TS submit is delivered exactly once
            return fail(EF_ESTATE, "ef_index of a new submit before ef_decode_audio consumed the current submit's audio");
        CK(cudaStreamWaitEvent(st, c->ev_up_done[c->pending], 0));
        c->active = c->pending; c->pending = -1;
        c->d = c->dd[c->active];
        c->aud_unconsumed = c->audio && c->aud_ts[c->active];
    }                                            // else: index the front buffer again (same input, next GOP period)
    if (c->profiling) { CK(cudaEventRecord(c->ev_prof[0], st)); c->prof_index = true; }
    CK(cudaMemsetAsync(c->h.info, 0, 32, st));
    const EfCarryArgs carry = c->carry ? carry_args(c, c->active) : EfCarryArgs{};
    CK(ef_launch_scan(c->d, c->carry ? &carry : nullptr, n, st));
    ef_prefix_kernel<<<c->h.max_pictures, 1024, 0, st>>>(c->d);
    CK(cudaGetLastError());
    const size_t threads = (size_t)n * c->h.max_pictures;
    ef_fill_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(c->d);
    CK(cudaGetLastError());
    c->launches += 3;
    if (c->profiling) CK(cudaEventRecord(c->ev_prof[1], st));
    if (c->pts) {
        const int a = c->active;
        CK(ef_launch_pts_resolve(c->d, c->d_pts_span2[a], c->d_pts_off2[a], c->d_pts_val2[a], c->d_pts_carry, c->d_pts_last, c->d_pic_pts,
                                 c->carry ? &carry : nullptr, n, st));
        c->launches++;
        c->pts_resolved = true;
    }
    if (c->carry) CK(cudaEventRecord(c->ev_scanned, st));   // the next upload copies the held bytes after this
    CK(cudaEventRecord(c->ev_buf_free[c->active], st));
    if (c->paced) {                              // the picture indices the present calls need, without a device-wide wait
        CK(cudaMemcpyAsync(c->h_pace_npics, c->h.info, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(c->ev_indexed, st));
    }
    c->indexed = true;
    if (c->paced) { c->pace_indexed = true; c->pace_next = 0; c->pace_npics = -1; c->pace_parse_at = 0; }
    return EF_OK;
}

int ef_index_info(ef_ctx* c, int* max_pictures, uint64_t* total_pictures, uint64_t* total_slices, uint64_t* es_bytes)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->indexed) return fail(EF_ESTATE, "ef_index_info before ef_index");
    uint32_t info[8];
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(info, c->h.info, 32, cudaMemcpyDeviceToHost));
    if (max_pictures) *max_pictures = (int)info[0];
    if (total_pictures) *total_pictures = info[1];
    if (total_slices) *total_slices = info[2];
    if (es_bytes) {
        uint64_t last = 0;
        CK(cudaMemcpy(&last, c->d_es_off2[c->active] + c->cfg.n_streams, 8, cudaMemcpyDeviceToHost));
        *es_bytes = last;
    }
    if ((info[3] & 4u) && (info[3] & 3u))
        return fail(EF_ENOMEM, "index overflow (flags %u): raise max_pictures / max_slices_per_picture; and a stream's held bytes exceeded "
                               "max_carry: see ef_carry_info", info[3]);
    if (info[3] & 4u) return fail(EF_ENOMEM, "a stream's held bytes exceeded max_carry (flags %u): see ef_carry_info", info[3]);
    if (info[3]) return fail(EF_ENOMEM, "index overflow (flags %u): raise max_pictures / max_slices_per_picture", info[3]);
    return EF_OK;
}

// ---- TS submits cut at any packet boundary: the reference's decoder pulls bytes on demand (FILL_BITS -> more(),
// player.cpp:348-352, 459-493), so a picture may span any number of the producer's Buffers (espflix.cpp:723-737) ----------
int ef_carry_enable(ef_ctx* c, uint32_t max_carry)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (c->carry) return fail(EF_ESTATE, "carry is already enabled");
    if (c->pending >= 0) return fail(EF_ESTATE, "ef_carry_enable with a submit pending: enable it before the next submit");
    if (max_carry < 4) return fail(EF_EINVAL, "max_carry %u must be at least 4 bytes", max_carry);
    TRY(pace_resolve(c));
    TRY(audio_resolve(c));
    const size_t n = (size_t)c->cfg.n_streams, extra = n * max_carry;
    const size_t es_old = c->cfg.es_capacity + 1024, es_new = es_old + extra;
    CK(cudaDeviceSynchronize());
    // both ES buffers and everything sized from them (the coefficient lists of K1a, 3 entries per ES byte) grow by n x max_carry;
    // the front buffer keeps the current submit, which may still be decoded
    for (int b = 0; b < 2; b++) TRY(dev_grow(c, &c->d_es2[b], es_old, es_new, true));
    TRY(dev_grow(c, &c->h.coef, 3 * es_old + 1024, 3 * es_new + 1024, true));
    TRY(dev_alloc(c, &c->d_held, n)); TRY(dev_alloc(c, &c->d_held_code, n)); TRY(dev_alloc(c, &c->d_carry_flags, n));
    TRY(dev_alloc(c, &c->d_pay_off, n + 1)); TRY(dev_alloc(c, &c->d_pts_hold, n)); TRY(dev_alloc(c, &c->d_pts_pre, n));
    for (int b = 0; b < 2; b++) { TRY(dev_alloc(c, &c->d_held_in2[b], n)); TRY(dev_alloc(c, &c->d_end2[b], n)); }
    c->max_carry = max_carry;
    TRY(carry_clear(c));
    TRY(push_dev(c));
    if (!c->ev_scanned) TRY(event(c, &c->ev_scanned));
    CK(cudaEventRecord(c->ev_scanned, 0));
    CK(cudaDeviceSynchronize());
    c->carry = true;
    return EF_OK;
}

int ef_end_streams(ef_ctx* c, int first, int count, const uint8_t* ends)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(stream_range(c, first, count, ends));
    if (!c->carry) return fail(EF_ESTATE, "ef_end_streams before ef_carry_enable");
    if (c->pending < 0) return fail(EF_ESTATE, "ef_end_streams with no submit pending");
    if (c->lib_submit) return fail(EF_ESTATE, "ef_end_streams on an ef_library_submit: the library ends its streams itself");
    if (!count) return EF_OK;
    const int p = c->pending;
    std::vector<uint8_t>& h = c->h_end2[p];
    for (int i = 0; i < count; i++) h[(size_t)first + i] |= ends[i] ? 1 : 0;
    // pageable source: the copy takes the flags before it returns; the upload stream orders it after the submit's own clear
    CK(cudaMemcpyAsync(c->d_end2[p] + first, h.data() + first, (size_t)count, cudaMemcpyHostToDevice, c->up_stream));
    CK(cudaEventRecord(c->ev_up_done[p], c->up_stream));
    return EF_OK;
}

int ef_carry_info(ef_ctx* c, int first, int count, uint32_t* held_bytes, uint8_t* flags)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(stream_range(c, first, count));
    if (!c->carry) return fail(EF_ESTATE, "ef_carry_info before ef_carry_enable");
    CK(cudaDeviceSynchronize());
    if (held_bytes && count) CK(cudaMemcpy(held_bytes, c->d_held + first, (size_t)count * 4, cudaMemcpyDeviceToHost));
    if (flags && count) CK(cudaMemcpy(flags, c->d_carry_flags + first, (size_t)count, cudaMemcpyDeviceToHost));
    return EF_OK;
}

int ef_stream_info(ef_ctx* c, int stream_index, int* n_pictures, int* base_pictures)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || stream_index < 0 || stream_index >= c->cfg.n_streams) return fail(EF_EINVAL, "bad stream index");
    uint32_t a = 0, b = 0;
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(&a, c->h.n_pics + stream_index, 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&b, c->h.base_pics + stream_index, 4, cudaMemcpyDeviceToHost));
    if (n_pictures) *n_pictures = (int)a;
    if (base_pictures) *base_pictures = (int)b;
    return EF_OK;
}

// staging buffer k (of two) for batched read-back, grown on demand
static int ensure_stage2(ef_ctx* c, int k, size_t bytes)
{
    if (c->stage2_bytes[k] >= bytes) return EF_OK;
    CK(cudaEventSynchronize(c->ev_down_done[k]));
    TRY(dev_grow(c, &c->d_stage2[k], c->stage2_bytes[k], bytes, false));
    c->stage2_bytes[k] = bytes;
    return EF_OK;
}

static EfDev decode_dev(ef_ctx* c)                      // K1 takes the context by value (kernel parameter space)
{
    EfDev dev = c->h;
    dev.es = c->d_es2[c->active]; dev.es_off = c->d_es_off2[c->active];
    return dev;
}

// K1a over picture indices [p0, p0 + k): their macroblock records for decode_recon
static int decode_parse(ef_ctx* c, int p0, int k, cudaStream_t st)
{
    const size_t slots = (size_t)k * c->cfg.n_streams * EF_MBW_MAX * EF_MBH_MAX;
    CK(cudaMemsetAsync(c->h.mb_info, 0, slots * 4, st));
    CK(cudaMemsetAsync(c->h.parse_cursor, 0, ((size_t)k + 1) * 4, st));
    if (c->profiling) { CK(cudaEventRecord(c->ev_prof[2], st)); c->prof_decode = true; }
    CK(ef_launch_parse(decode_dev(c), p0, k, c->sm_count, (size_t)k * c->cfg.n_streams * c->cfg.max_slices_per_picture, st));
    if (c->profiling) CK(cudaEventRecord(c->ev_prof[3], st));
    if (c->frames_read_pending) { CK(cudaStreamWaitEvent(st, c->ev_frames_read, 0)); c->frames_read_pending = false; }   // an asynchronous read-back still reads the frame stores
    c->launches++;
    return EF_OK;
}

// K1b of record picture i of the last decode_parse into the frame stores
static int decode_recon(ef_ctx* c, int i, cudaStream_t st)
{
    CK(ef_launch_recon(decode_dev(c), i, c->sm_count, (size_t)c->cfg.n_streams * EF_MBW_MAX * EF_MBH_MAX, st));
    c->launches++;
    return EF_OK;
}

// K1a over picture indices [p0, p0 + k), then K1b once per picture index. host_dst != nullptr: every picture index
// is exported (I420) straight after its K1b launch and copied to host_dst[p][stream] on the read-back stream while
// the next picture index is being rebuilt - what push_video() sees, picture by picture (video.h:49).
// after (optional) runs after the K1b launch of every picture index (ef_trick_build gathers the frames it encodes).
static int decode_range(ef_ctx* c, int p0, int k, cudaStream_t st, uint8_t* host_dst = nullptr, int layout = 0,
                        int (*after)(void*, int, cudaStream_t) = nullptr, void* after_arg = nullptr)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    TRY(decode_parse(c, p0, k, st));
    const size_t batch_bytes = (size_t)c->cfg.n_streams * EF_FRAME;
    for (int i = 0; i < k; i++) {
        TRY(decode_recon(c, i, st));
        if (after) TRY(after(after_arg, p0 + i, st));
        if (host_dst) {
            const int b = c->stage_idx ^= 1;
            TRY(ensure_stage2(c, b, batch_bytes));
            CK(cudaStreamWaitEvent(st, c->ev_down_done[b], 0));            // the previous copy out of this staging buffer has finished
            const uint64_t threads = (uint64_t)c->cfg.n_streams * (EF_FRAME / 8);
            ef_export_frames_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(c->h.frames, c->h.base_pics, c->h.n_pics, 0, c->cfg.n_streams, -2 - (p0 + i), layout, c->d_stage2[b]);
            CK(cudaGetLastError());
            c->launches++;
            CK(cudaEventRecord(c->ev_export, st));
            CK(cudaStreamWaitEvent(c->down_stream, c->ev_export, 0));
            CK(cudaMemcpyAsync(host_dst + (size_t)(p0 + i) * batch_bytes, c->d_stage2[b], batch_bytes, cudaMemcpyDeviceToHost, c->down_stream));
            CK(cudaEventRecord(c->ev_down_done[b], c->down_stream));
        }
    }
    if (c->profiling) CK(cudaEventRecord(c->ev_prof[4], st));
    CK(cudaEventRecord(c->ev_buf_free[c->active], st));     // the front ES buffer is in use until here
    return EF_OK;
}

int ef_decode_picture(ef_ctx* c, int pic, void* stream)
{
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->indexed) return fail(EF_ESTATE, "ef_decode_picture before ef_index");
    if (c->paced) return fail(EF_ESTATE, "ef_decode_picture on a presenting context: ef_present_picture decodes");
    if (pic < 0 || pic >= c->cfg.max_pictures) return fail(EF_EINVAL, "picture index %d out of range", pic);
    return decode_range(c, pic, 1, (cudaStream_t)stream);
}

// ef_decode_all(_to_host): picture indices [0, n_pictures), rec_pics of them per K1a launch
static int decode_all(ef_ctx* c, const char* what, int n_pictures, void* stream, uint8_t* host_dst = nullptr, int layout = 0)
{
    if (!c->indexed) return fail(EF_ESTATE, "%s before ef_index", what);
    if (c->paced) return fail(EF_ESTATE, "%s on a presenting context: ef_present_picture decodes", what);
    if (n_pictures < 0 || n_pictures > c->cfg.max_pictures) return fail(EF_EINVAL, "n_pictures %d out of range", n_pictures);
    for (int p = 0; p < n_pictures; p += c->h.rec_pics) {
        const int k = n_pictures - p < c->h.rec_pics ? n_pictures - p : c->h.rec_pics;
        TRY(decode_range(c, p, k, (cudaStream_t)stream, host_dst, layout));
    }
    return EF_OK;
}

int ef_decode_all(ef_ctx* c, int n_pictures, void* stream)
{
    if (!c) return fail(EF_EINVAL, "null context");
    return decode_all(c, "ef_decode_all", n_pictures, stream);
}

int ef_decode_all_to_host(ef_ctx* c, int n_pictures, uint8_t* dst, int layout, void* stream)
{
    if (!c || !dst) return fail(EF_EINVAL, "null argument");
    if (layout != 0 && layout != 1) return fail(EF_EINVAL, "layout must be 0 (I420) or 1 (strips)");
    return decode_all(c, "ef_decode_all_to_host", n_pictures, stream, dst, layout);
}

// one frame store to the host (ef_read_frame(_i420)) or from it (ef_write_frame(_i420)) in `layout`: 0 = I420, 1 = strips
static int read_frame(ef_ctx* c, int stream_index, int fb, uint8_t* dst, int layout)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !dst) return fail(EF_EINVAL, "null argument");
    CK(cudaDeviceSynchronize());
    int f;
    TRY(resolve_fb(c, stream_index, fb, &f));
    TRY(ensure_stage(c));
    ef_export_frames_kernel<<<(EF_FRAME / 8 + 255) / 256, 256>>>(c->h.frames, c->h.base_pics, c->h.n_pics, stream_index, 1, f, layout, c->d_stage);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaMemcpy(dst, c->d_stage, EF_FRAME, cudaMemcpyDeviceToHost));
    return EF_OK;
}

static int write_frame(ef_ctx* c, int stream_index, int fb, const uint8_t* src, int layout)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !src) return fail(EF_EINVAL, "null argument");
    int f;
    TRY(resolve_fb(c, stream_index, fb, &f));
    TRY(ensure_stage(c));
    TRY(wait_frames_read(c));
    CK(cudaMemcpy(c->d_stage, src, EF_FRAME, cudaMemcpyHostToDevice));
    ef_import_frame_kernel<<<(EF_FRAME / 4 + 255) / 256, 256>>>(c->h.frames + ef_frame_offset(stream_index, f), c->d_stage, layout);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaDeviceSynchronize());
    return EF_OK;
}

int ef_read_frame(ef_ctx* c, int stream_index, int fb, uint8_t* dst) { return read_frame(c, stream_index, fb, dst, 1); }
int ef_read_frame_i420(ef_ctx* c, int stream_index, int fb, uint8_t* dst) { return read_frame(c, stream_index, fb, dst, 0); }
int ef_write_frame(ef_ctx* c, int stream_index, int fb, const uint8_t* src) { return write_frame(c, stream_index, fb, src, 1); }
int ef_write_frame_i420(ef_ctx* c, int stream_index, int fb, const uint8_t* src) { return write_frame(c, stream_index, fb, src, 0); }

int ef_read_latest_i420_async(ef_ctx* c, int first, int count, uint8_t* dst, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !dst) return fail(EF_EINVAL, "null argument");
    if (first < 0 || count < 1 || first + count > c->cfg.n_streams) return fail(EF_EINVAL, "stream range out of bounds");
    const int k = c->stage_idx ^= 1;
    const size_t bytes = (size_t)count * EF_FRAME;
    TRY(ensure_stage2(c, k, bytes));
    cudaStream_t st = (cudaStream_t)stream;
    // The tiled -> I420 export runs on the read-back stream, behind everything queued on the caller's stream so far and
    // behind the previous copy out of this staging buffer: it overlaps the index / parse kernels of the next submit. The
    // next reconstruction launch (the first thing that writes a frame store again) waits for ev_frames_read.
    if (!c->d_fb_snap[k]) TRY(dev_alloc(c, &c->d_fb_snap[k], (size_t)c->cfg.n_streams));
    CK(cudaStreamWaitEvent(st, c->ev_down_done[k], 0));        // the previous read-back through this staging buffer (and its snapshot) has finished
    ef_latest_fb_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(c->h.base_pics, c->h.n_pics, first, count, c->d_fb_snap[k]);
    CK(cudaGetLastError());
    CK(cudaEventRecord(c->ev_export, st));
    CK(cudaStreamWaitEvent(c->down_stream, c->ev_export, 0));
    const uint64_t threads = (uint64_t)count * (EF_FRAME / 8);
    ef_export_frames_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, c->down_stream>>>(c->h.frames, c->h.base_pics, c->h.n_pics, first, count, -1, 0, c->d_stage2[k], c->d_fb_snap[k]);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaEventRecord(c->ev_frames_read, c->down_stream));
    c->frames_read_pending = true;
    CK(cudaMemcpyAsync(dst, c->d_stage2[k], bytes, cudaMemcpyDeviceToHost, c->down_stream));   // overlaps the next decode when dst is pinned
    CK(cudaEventRecord(c->ev_down_done[k], c->down_stream));
    return EF_OK;
}

int ef_sync(ef_ctx* c, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    CK(cudaStreamSynchronize((cudaStream_t)stream));
    CK(cudaStreamSynchronize(c->up_stream));
    CK(cudaStreamSynchronize(c->down_stream));
    return EF_OK;
}

int ef_read_latest_i420(ef_ctx* c, int first, int count, uint8_t* dst, void* stream)
{
    TRY(ef_read_latest_i420_async(c, first, count, dst, stream));
    CK(cudaStreamSynchronize(c->down_stream));
    return EF_OK;
}

int ef_frame_device_ptr(ef_ctx* c, int stream_index, int fb, void** ptr)
{
    if (!c || !ptr || stream_index < 0 || stream_index >= c->cfg.n_streams || (fb != 0 && fb != 1)) return fail(EF_EINVAL, "bad argument");
    *ptr = c->h.frames + ef_frame_offset(stream_index, fb);
    return EF_OK;
}

int ef_video_init(ef_ctx* c, int ntsc)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (c->paced && (ntsc ? 1 : 0) != c->pace_ntsc) return fail(EF_ESTATE, "the standard of a presenting context is fixed by ef_present_enable");
    TRY(pace_resolve(c));
    EfGeometry g;
    memset(&g, 0, sizeof(g));
    g.ntsc = ntsc ? 1 : 0;
    if (g.ntsc) {      // video_init(), video.cpp:572-600 (values probe-verified: tests/golden/composite_pins.json)
        g.line_width = 912; g.line_count = 262; g.hsync = 64; g.hsync_long = 840; g.active_start = 144;
        g.active_top = 32; g.vsync_start = 259; g.blit_start = g.active_start + 16;
    } else {           // pal_init(), video.cpp:607-630
        g.line_width = 1136; g.line_count = 312; g.hsync = 80; g.hsync_short = 32; g.hsync_long = 536;
        g.burst_start = 96; g.burst_width = 44; g.active_start = 184;
        g.active_top = 64; g.vsync_start = 304; g.blit_start = g.active_start + 16 + 80;
    }
    uint32_t tab[768];
    int16_t burst[128];
    memset(burst, 0, sizeof(burst));
    ef_build_color_tab(tab, g.ntsc);
    ef_build_pal_burst(burst, burst + 64, 44);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(c->d_color_tab, tab, sizeof(tab), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_pal_burst, burst, sizeof(burst), cudaMemcpyHostToDevice));
    c->h.geo = g;
    TRY(push_dev(c));
    c->video = true;
    return EF_OK;
}

int ef_video_geometry(ef_ctx* c, int* line_width, int* line_count)
{
    if (!c) return fail(EF_EINVAL, "null context");
    if (line_width) *line_width = c->h.geo.line_width;
    if (line_count) *line_count = c->h.geo.line_count;
    return EF_OK;
}

int ef_composite_field(ef_ctx* c, int fb, int frame_counter, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->h.fields) return fail(EF_ESTATE, "context was created without field buffers (ef_config.fields = 0)");
    if (fb < -2 || fb > 1) return fail(EF_EINVAL, "fb must be 0, 1, -1 or -2");
    CK(ef_launch_composite(c->d, c->cfg.n_streams, c->h.geo, fb, frame_counter, c->present, (cudaStream_t)stream));
    c->launches++;
    return EF_OK;
}

int ef_video_set_scroll(ef_ctx* c, int hscroll)
{
    if (!c) return fail(EF_EINVAL, "null context");
    if (hscroll <= -EF_W || hscroll >= EF_W || (hscroll & 7)) return fail(EF_EINVAL, "hscroll must be a multiple of 8 in (-352, 352)");
    c->present.hscroll = hscroll;
    return EF_OK;
}

int ef_video_set_overlay(ef_ctx* c, const uint8_t* bitmap, int blend, int progress)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (blend != 0 && !bitmap && c->present.blend == 0) return fail(EF_EINVAL, "overlay bitmap required when blend != 0");
    if (bitmap) { CK(cudaDeviceSynchronize()); CK(cudaMemcpy(c->d_overlay, bitmap, 1280, cudaMemcpyHostToDevice)); }
    c->present.blend = blend; c->present.progress = progress;
    return EF_OK;
}

int ef_read_field(ef_ctx* c, int stream_index, uint16_t* dst)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !dst || stream_index < 0 || stream_index >= c->cfg.n_streams) return fail(EF_EINVAL, "bad argument");
    if (!c->h.fields) return fail(EF_ESTATE, "no field buffers");
    CK(cudaDeviceSynchronize());
    const size_t n = (size_t)c->h.geo.line_width * c->h.geo.line_count;
    CK(cudaMemcpy(dst, c->h.fields + (size_t)stream_index * c->h.field_stride, n * 2, cudaMemcpyDeviceToHost));
    return EF_OK;
}

int ef_video_isr(ef_ctx* c, int stream_index, int line, uint16_t* buf)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !buf || stream_index < 0 || stream_index >= c->cfg.n_streams) return fail(EF_EINVAL, "bad argument");
    if (!c->h.fields) return fail(EF_ESTATE, "no field buffers");
    if (line < 0 || line >= c->h.geo.line_count) return fail(EF_EINVAL, "line %d out of range", line);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(buf, c->h.fields + (size_t)stream_index * c->h.field_stride + (size_t)line * c->h.geo.line_width,
                  (size_t)c->h.geo.line_width * 2, cudaMemcpyDeviceToHost));
    return EF_OK;
}

int ef_blit(ef_ctx* c, int stream_index, int fb, uint16_t* dst, int line, int x, int width, int frame_counter)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !dst) return fail(EF_EINVAL, "null argument");
    const int w8 = (width + 7) & ~7;          // the reference loop advances 8 pixels per iteration (video.cpp:709): the whole last group is written
    if (line < 0 || line >= EF_H || x < 0 || width < 0 || (x & ~3) + w8 > EF_W) return fail(EF_EINVAL, "blit span out of range (the width is rounded up to a multiple of 8 pixels)");
    int f;
    TRY(resolve_fb(c, stream_index, fb, &f));
    if (!w8) return EF_OK;
    CK(cudaDeviceSynchronize());              // like ef_read_frame: a decode may still be running on a non-blocking user stream
    TRY(ensure_stage(c));
    CK(ef_launch_blit(c->d, stream_index, f, line, x, w8, frame_counter, (uint16_t*)c->d_stage, 0));
    c->launches++;
    // blit() itself offsets PAL output by 80 samples (video.cpp:698)
    CK(cudaMemcpy(dst + (c->h.geo.ntsc ? 0 : 80), c->d_stage, (size_t)w8 * 4, cudaMemcpyDeviceToHost));
    return EF_OK;
}

uint64_t ef_launch_count(ef_ctx* c) { return c ? c->launches : 0; }

int ef_host_alloc(void** p, size_t bytes)
{
    if (!p || !bytes) return fail(EF_EINVAL, "null argument");
    CK(cudaHostAlloc(p, bytes, cudaHostAllocDefault));
    return EF_OK;
}

void ef_host_free(void* p) { if (p) cudaFreeHost(p); }

int ef_set_profiling(ef_ctx* c, int on)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (on && !c->ev_prof[0]) for (int i = 0; i < 5; i++) TRY(event(c, &c->ev_prof[i], true));
    c->profiling = on != 0;
    c->prof_index = c->prof_decode = false;
    return EF_OK;
}

int ef_stage_ms(ef_ctx* c, float* index_ms, float* parse_ms, float* recon_ms)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->profiling) return fail(EF_ESTATE, "ef_stage_ms without ef_set_profiling(ctx, 1)");
    float a = 0, b = 0, r = 0;
    if (c->prof_index) { CK(cudaEventSynchronize(c->ev_prof[1])); CK(cudaEventElapsedTime(&a, c->ev_prof[0], c->ev_prof[1])); }
    if (c->prof_decode) {
        CK(cudaEventSynchronize(c->ev_prof[4]));
        CK(cudaEventElapsedTime(&b, c->ev_prof[2], c->ev_prof[3]));
        CK(cudaEventElapsedTime(&r, c->ev_prof[3], c->ev_prof[4]));
    }
    if (index_ms) *index_ms = a;
    if (parse_ms) *parse_ms = b;
    if (recon_ms) *recon_ms = r;
    return EF_OK;
}

// ---- trick-mode index (indexer/indexer.cpp), stateless --------------------------------------------------
namespace {
struct DevBuf {                      // scoped device allocation
    void* p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, n ? n : 1); }
};
uint32_t tsidx_sample_count(uint32_t n_seq, int64_t first, int64_t last, uint32_t bin)
{
    if (!n_seq || !bin || last < first) return 0;
    return (uint32_t)((last - first) / bin + 1);
}
}  // namespace

int ef_tsidx_scan(int device, const uint8_t* ts, const uint64_t* off, int n_files, uint32_t bin_size,
                  ef_tsidx_info* info, int64_t* seq_pts, uint32_t* seq_pos)
{
    if (!ts || !off || !info || !seq_pts || !seq_pos || n_files < 1) return fail(EF_EINVAL, "null argument");
    TRY(usable_device(device));
    DeviceScope scope_(device);
    for (int f = 0; f <= n_files; f++) if (off[f] % 188 || (f && off[f] < off[f - 1])) return fail(EF_EINVAL, "offsets must be non-decreasing multiples of 188");
    const uint64_t total = off[n_files] - off[0], n_packets = total / 188;
    std::vector<uint64_t> poff((size_t)n_files + 1);
    for (int f = 0; f <= n_files; f++) poff[f] = (off[f] - off[0]) / 188;
    DevBuf d_ts, d_pts, d_kind, d_off, d_spts, d_spos, d_info;
    CK(d_ts.alloc(total)); CK(d_pts.alloc(n_packets * 8)); CK(d_kind.alloc(n_packets)); CK(d_off.alloc(poff.size() * 8));
    CK(d_spts.alloc(n_packets * 8)); CK(d_spos.alloc(n_packets * 4)); CK(d_info.alloc((size_t)n_files * 24));
    CK(cudaMemcpy(d_ts.p, ts + off[0], total, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_off.p, poff.data(), poff.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemset(d_spts.p, 0, n_packets * 8 + (n_packets ? 0 : 1)));
    CK(cudaMemset(d_spos.p, 0, n_packets * 4 + (n_packets ? 0 : 1)));
    if (n_packets) {
        ef_tsidx_packet_kernel<<<(unsigned)((n_packets + 255) / 256), 256>>>((const uint8_t*)d_ts.p, (const uint64_t*)d_off.p, n_files, n_packets, (int64_t*)d_pts.p, (uint8_t*)d_kind.p);
        CK(cudaGetLastError());
    }
    ef_tsidx_compact_kernel<<<n_files, 256>>>((const uint64_t*)d_off.p, (const int64_t*)d_pts.p, (const uint8_t*)d_kind.p,
                                              (int64_t*)d_spts.p, (uint32_t*)d_spos.p, (int64_t*)d_info.p);
    CK(cudaGetLastError());
    std::vector<int64_t> hinfo((size_t)n_files * 3);
    CK(cudaMemcpy(hinfo.data(), d_info.p, hinfo.size() * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(seq_pts, d_spts.p, n_packets * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(seq_pos, d_spos.p, n_packets * 4, cudaMemcpyDeviceToHost));
    for (int f = 0; f < n_files; f++) {
        info[f].first_pts = hinfo[f * 3]; info[f].last_pts = hinfo[f * 3 + 1]; info[f].n_seq = (uint32_t)hinfo[f * 3 + 2];
        info[f].n_samples = tsidx_sample_count(info[f].n_seq, info[f].first_pts, info[f].last_pts, bin_size);
    }
    return EF_OK;
}

int ef_tsidx_samples(int device, const int64_t* seq_pts, const uint32_t* seq_pos, int n_seq, int64_t first_pts, int64_t last_pts,
                     uint32_t bin_size, uint32_t* samples, uint32_t cap, uint32_t* n_samples)
{
    if (!n_samples || n_seq < 0 || (n_seq && (!seq_pts || !seq_pos))) return fail(EF_EINVAL, "null argument");
    const uint32_t n = tsidx_sample_count((uint32_t)n_seq, first_pts, last_pts, bin_size);
    *n_samples = n;
    if (!n) return EF_OK;
    if (!samples || cap < n) return fail(EF_ENOMEM, "%u samples needed, capacity %u", n, cap);
    TRY(usable_device(device));
    DeviceScope scope_(device);
    DevBuf d_pts, d_pos, d_out;
    CK(d_pts.alloc((size_t)n_seq * 8)); CK(d_pos.alloc((size_t)n_seq * 4)); CK(d_out.alloc((size_t)n * 4));
    CK(cudaMemcpy(d_pts.p, seq_pts, (size_t)n_seq * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_pos.p, seq_pos, (size_t)n_seq * 4, cudaMemcpyHostToDevice));
    ef_tsidx_sample_kernel<<<(n + 127) / 128, 128>>>((const int64_t*)d_pts.p, (const uint32_t*)d_pos.p, n_seq, first_pts, bin_size, n, (uint32_t*)d_out.p);
    CK(cudaGetLastError());
    CK(cudaMemcpy(samples, d_out.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return EF_OK;
}

// ---- audio (SURVEY.md 8f-3): SBC decode + PDM ---------------------------------------------------------------------
static int audio_constants(int device)
{
    static bool constants = false;                       // per process; every device gets its copy on first use
    static int constants_dev = -1;
    if (!constants || constants_dev != device) { CK(ef_audio_upload_constants()); constants = true; constants_dev = device; }
    return EF_OK;
}

// One decode call once its input is in HBM (blob + blob_off[n + 1]: every stream's held-back bytes followed by its new
// bytes), in two halves on `cs`, neither of which waits for the device:
//   audio_plan  probe, count, and ef_audio_size_kernel: slot and PCM offsets, info[] (device) and the verdict against pcm_cap
//   audio_run   SBC -> PCM (-> PDM) into pcm / pdm (device) and the update of the per-stream state
// The grids of audio_run come from a bound on the call's samples (bound_pcm), not from its totals, which only the device
// knows: a stream has at most 2 + frames slots (history, probe, frames), so slots <= 2 n + bound_pcm / 128. Blocks past
// the totals return at once (the kernels read their totals from HBM); when the caller sizes pcm_cap to its call, as a
// sizing call lets it, the bound is the need and few blocks are idle. The V-row scratch follows the same bound.
static size_t audio_vrow_bytes(int n, uint64_t bound_pcm) { return (2 * (size_t)n + bound_pcm / 128) * 16 * 16 * 4; }

static int audio_scratch(AudioScratch& w, int n, uint64_t bound_pcm)
{
    void* q;
    CK(w.get(AudioScratch::PLAN, (size_t)n * sizeof(int4), &q));
    CK(w.get(AudioScratch::SLOT, ((size_t)n + 1) * 8, &q));
    CK(w.get(AudioScratch::POFF, ((size_t)n + 1) * 8, &q));
    CK(w.get(AudioScratch::SB_LAST, (size_t)n * 128 * 4, &q));
    CK(w.get(AudioScratch::INFO, (size_t)n * sizeof(ef_audio_info), &q));
    CK(w.get(AudioScratch::VERDICT, sizeof(int), &q));
    CK(w.get(AudioScratch::VROWS, audio_vrow_bytes(n, bound_pcm), &q));
    return EF_OK;
}

static int audio_plan(const uint8_t* blob, const uint64_t* blob_off, const EfAudioState* st, const uint8_t* ended, int n, AudioScratch& w,
                      uint64_t pcm_cap, ef_audio_info* d_info, cudaStream_t cs, uint64_t* launches)
{
    int4* plan = (int4*)w.p[AudioScratch::PLAN];
    ef_sbc_probe_kernel<<<(n + 127) / 128, 128, 0, cs>>>(blob, blob_off, st, ended, n, plan);
    CK(cudaGetLastError());
    ef_sbc_count_kernel<<<(unsigned)(((size_t)n * 32 + 255) / 256), 256, 0, cs>>>(blob, blob_off, ended, n, plan);
    CK(cudaGetLastError());
    ef_audio_size_kernel<<<1, 1024, 0, cs>>>(plan, n, pcm_cap, (uint64_t*)w.p[AudioScratch::SLOT], (uint64_t*)w.p[AudioScratch::POFF], d_info,
                                             (int*)w.p[AudioScratch::VERDICT]);
    CK(cudaGetLastError());
    *launches += 3;
    return EF_OK;
}

// gated: the commit is skipped on the device when the call exceeded its capacity (the caller has not checked it)
static int audio_run(const uint8_t* blob, const uint64_t* blob_off, EfAudioState* st, const uint8_t* ended, int n, AudioScratch& w, uint64_t bound_pcm,
                     int16_t* pcm, uint16_t* pdm, bool gated, cudaStream_t cs, uint64_t* launches)
{
    const int4* plan = (const int4*)w.p[AudioScratch::PLAN];
    const uint64_t* d_slot = (const uint64_t*)w.p[AudioScratch::SLOT];
    const uint64_t* d_poff = (const uint64_t*)w.p[AudioScratch::POFF];
    int32_t* sb_last = (int32_t*)w.p[AudioScratch::SB_LAST];
    int32_t* vrows = (int32_t*)w.p[AudioScratch::VROWS];
    const uint64_t slots = 2 * (uint64_t)n + bound_pcm / 128;
    ef_sbc_matrix_kernel<<<(unsigned)((slots + 3) / 4), 128, 0, cs>>>(blob, blob_off, plan, st, d_slot, n, vrows, sb_last);
    CK(cudaGetLastError());
    *launches += 1;
    if (bound_pcm) {
        ef_sbc_window_kernel<<<(unsigned)((bound_pcm + 255) / 256), 256, 0, cs>>>(vrows, d_slot, d_poff, n, pcm);
        CK(cudaGetLastError());
        *launches += 1;
        if (pdm) {
            ef_pdm_kernel<<<(n + 31) / 32, 32, 0, cs>>>(pcm, d_poff, n, st, pdm);
            CK(cudaGetLastError());
            *launches += 1;
        }
    }
    CK(ef_launch_audio_commit(st, blob, blob_off, plan, d_slot, vrows, sb_last, ended, n, gated ? (const int*)w.p[AudioScratch::VERDICT] : nullptr, cs));
    *launches += 1;
    return EF_OK;
}

// The synchronous call: the plan, one read of info[], then - unless pcm is NULL (sizing: info[] only, no state changes) or
// the call does not fit - the decode with the bound at the call's own samples, the copies to the host and a wait.
// after(): launches that belong to the call once it decoded (the context's demux-gate kernel).
extern "C++" {
template <typename After>
static int audio_decode_blob(const uint8_t* blob, const uint64_t* blob_off, EfAudioState* st, const uint8_t* ended, int n, AudioScratch& w,
                             ef_audio_info* info, int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm, cudaStream_t cs, uint64_t* launches, After after)
{
    TRY(audio_scratch(w, n, 0));
    ef_audio_info* d_info = (ef_audio_info*)w.p[AudioScratch::INFO];
    TRY(audio_plan(blob, blob_off, st, ended, n, w, pcm ? pcm_cap : ~0ull, d_info, cs, launches));
    CK(cudaMemcpyAsync(info, d_info, (size_t)n * sizeof(ef_audio_info), cudaMemcpyDeviceToHost, cs));
    CK(cudaStreamSynchronize(cs));
    const uint64_t n_pcm = info[n - 1].pcm_offset + (uint64_t)info[n - 1].n_frames * 128;
    if (!pcm) return EF_OK;                                  // sizing call
    if (n_pcm > pcm_cap) return fail(EF_ENOMEM, "%llu PCM samples, capacity %llu", (unsigned long long)n_pcm, (unsigned long long)pcm_cap);
    int16_t* d_pcm = nullptr;
    uint16_t* d_pdm = nullptr;
    TRY(audio_scratch(w, n, n_pcm));
    CK(w.get(AudioScratch::PCM, n_pcm * 2, (void**)&d_pcm));
    if (pdm) CK(w.get(AudioScratch::PDM, n_pcm * 4, (void**)&d_pdm));
    TRY(audio_run(blob, blob_off, st, ended, n, w, n_pcm, d_pcm, pdm ? d_pdm : nullptr, false, cs, launches));
    TRY(after());
    if (n_pcm) {
        CK(cudaMemcpyAsync(pcm, d_pcm, n_pcm * 2, cudaMemcpyDeviceToHost, cs));
        if (pdm) CK(cudaMemcpyAsync(pdm, d_pdm, n_pcm * 4, cudaMemcpyDeviceToHost, cs));
    }
    CK(cudaStreamSynchronize(cs));
    return EF_OK;
}
}  // extern "C++"

int ef_audio_demux_ts(int device, const uint8_t* ts, const uint64_t* off, int n_files, uint8_t* es, uint64_t es_cap, uint64_t* es_off)
{
    if (!ts || !off || !es_off || n_files < 1) return fail(EF_EINVAL, "null argument");
    TRY(usable_device(device));
    DeviceScope scope_(device);
    for (int f = 0; f <= n_files; f++) if (off[f] % 188 || (f && off[f] < off[f - 1])) return fail(EF_EINVAL, "offsets must be non-decreasing multiples of 188");
    const uint64_t total = off[n_files] - off[0], n_packets = total / 188;
    std::vector<uint64_t> roff((size_t)n_files + 1);
    for (int f = 0; f <= n_files; f++) roff[f] = off[f] - off[0];
    DevBuf d_ts, d_start, d_kind, d_off, d_pos, d_len, d_esoff, d_es, d_gate, d_lead, d_skip;
    CK(d_ts.alloc(total)); CK(d_start.alloc(n_packets)); CK(d_kind.alloc(n_packets)); CK(d_off.alloc(roff.size() * 8));
    CK(d_pos.alloc(n_packets * 4)); CK(d_len.alloc((size_t)n_files * 8)); CK(d_esoff.alloc(roff.size() * 8));
    CK(d_gate.alloc((size_t)n_files * 2)); CK(d_lead.alloc((size_t)n_files * 4)); CK(d_skip.alloc((size_t)n_files));
    CK(cudaMemcpy(d_ts.p, ts + off[0], total, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_off.p, roff.data(), roff.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemset(d_gate.p, 0, (size_t)n_files));                       // every file starts with the gate shut (MpegDecoder::reset())
    if (n_packets) {
        ef_audio_ts_packet_kernel<<<(unsigned)((n_packets + 255) / 256), 256>>>((const uint8_t*)d_ts.p, n_packets, (uint8_t*)d_start.p, (uint8_t*)d_kind.p);
        CK(cudaGetLastError());
    }
    uint8_t* gate = (uint8_t*)d_gate.p;
    ef_audio_ts_scan_kernel<<<(n_files + 63) / 64, 64>>>((const uint64_t*)d_off.p, n_files, (const uint8_t*)d_start.p, (const uint8_t*)d_kind.p, gate, gate + n_files,
                                                         (uint32_t*)d_lead.p, (uint8_t*)d_skip.p, (uint32_t*)d_pos.p, (uint64_t*)d_len.p);
    CK(cudaGetLastError());
    std::vector<uint64_t> len((size_t)n_files);
    CK(cudaMemcpy(len.data(), d_len.p, len.size() * 8, cudaMemcpyDeviceToHost));
    es_off[0] = 0;
    for (int f = 0; f < n_files; f++) es_off[f + 1] = es_off[f] + len[f];
    if (es_off[n_files] > es_cap || (!es && es_off[n_files])) return fail(EF_ENOMEM, "%llu audio bytes, capacity %llu", (unsigned long long)es_off[n_files], (unsigned long long)es_cap);
    if (es_off[n_files]) {
        CK(d_es.alloc(es_off[n_files]));
        CK(cudaMemcpy(d_esoff.p, es_off, roff.size() * 8, cudaMemcpyHostToDevice));
        ef_audio_ts_copy_kernel<<<(unsigned)((n_packets * 32 + 255) / 256), 256>>>((const uint8_t*)d_ts.p, (const uint64_t*)d_off.p, n_files, n_packets,
                                                                                   (const uint8_t*)d_start.p, (const uint32_t*)d_pos.p, (const uint64_t*)d_esoff.p, (uint8_t*)d_es.p);
        CK(cudaGetLastError());
        CK(cudaMemcpy(es, d_es.p, es_off[n_files], cudaMemcpyDeviceToHost));
    }
    return EF_OK;
}

// the whole-stream call: the context's kernels with a fresh state for every stream, every stream ending in this call
int ef_audio_decode(int device, const uint8_t* sbc, const uint64_t* off, int n_streams, ef_audio_info* info, int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm)
{
    if (!sbc || !off || !info || n_streams < 1) return fail(EF_EINVAL, "null argument");
    TRY(usable_device(device));
    DeviceScope scope_(device);
    for (int s = 0; s < n_streams; s++) if (off[s] > off[s + 1]) return fail(EF_EINVAL, "stream offsets must be non-decreasing");
    TRY(audio_constants(device));
    const uint64_t total = off[n_streams] - off[0];
    std::vector<uint64_t> roff((size_t)n_streams + 1);
    for (int s = 0; s <= n_streams; s++) roff[s] = off[s] - off[0];
    DevBuf d_es, d_off, d_st, d_end;
    CK(d_es.alloc(total + 16)); CK(d_off.alloc(roff.size() * 8));
    CK(d_st.alloc((size_t)n_streams * sizeof(EfAudioState))); CK(d_end.alloc((size_t)n_streams));
    CK(cudaMemcpy(d_es.p, sbc + off[0], total, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_off.p, roff.data(), roff.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemset(d_st.p, 0, (size_t)n_streams * sizeof(EfAudioState)));
    CK(cudaMemset(d_end.p, 1, (size_t)n_streams));
    AudioScratch w;
    uint64_t launches = 0;
    return audio_decode_blob((const uint8_t*)d_es.p, (const uint64_t*)d_off.p, (EfAudioState*)d_st.p, (const uint8_t*)d_end.p, n_streams, w,
                             info, pcm, pcm_cap, pdm, 0, &launches, [] { return EF_OK; });
}

int ef_audio_enable(ef_ctx* c)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(audio_resolve(c));
    if (c->audio) return EF_OK;
    TRY(audio_constants(c->cfg.device));
    const int n = c->cfg.n_streams;
    const size_t cap = c->cfg.es_capacity, packets = cap / 188 + 1;
    TRY(dev_alloc(c, &c->d_aud_state, (size_t)n));
    for (int b = 0; b < 2; b++) {
        TRY(dev_alloc(c, &c->d_aud2[b], cap + 1024));     // a submit's audio is never longer than its transport stream
        TRY(dev_alloc(c, &c->d_aud_off2[b], (size_t)n + 1));
        TRY(dev_alloc(c, &c->d_gate2[b], (size_t)n)); TRY(dev_alloc(c, &c->d_lead2[b], (size_t)n)); TRY(dev_alloc(c, &c->d_skip2[b], (size_t)n));
    }
    TRY(dev_alloc(c, &c->d_aud_start, packets)); TRY(dev_alloc(c, &c->d_aud_kind, packets)); TRY(dev_alloc(c, &c->d_aud_pos, packets));
    TRY(dev_alloc(c, &c->d_aud_len, (size_t)n + 1));
    TRY(dev_alloc(c, &c->d_blob, cap + (size_t)n * EF_AUDIO_CARRY + 1024));
    TRY(dev_alloc(c, &c->d_blob_len, (size_t)n + 1)); TRY(dev_alloc(c, &c->d_blob_off, (size_t)n + 1));
    TRY(dev_alloc(c, &c->d_ended, (size_t)n));
    if (!c->h_ended) TRY(host_alloc(c, &c->h_ended, (size_t)n));
    CK(cudaMemset(c->d_aud_state, 0, (size_t)n * sizeof(EfAudioState)));
    for (int b = 0; b < 2; b++) {
        CK(cudaMemset(c->d_gate2[b], 0, (size_t)n)); CK(cudaMemset(c->d_skip2[b], 0, (size_t)n)); CK(cudaMemset(c->d_lead2[b], 0, (size_t)n * 4));
        CK(cudaMemset(c->d_aud_off2[b], 0, ((size_t)n + 1) * 8));
        c->aud_ts[b] = false;
    }
    CK(cudaDeviceSynchronize());
    c->aud_unconsumed = false;
    c->audio = true;
    return EF_OK;
}

// The front half of a context's audio call on `cs`: after the demux of the current submit (and of one queued behind it, whose
// gate ef_audio_end_kernel may shut) and after the previous audio call (it shares the blob, the scratch and h_ended), the
// end flags go up and every stream's held-back bytes and new bytes are assembled into the blob. Returns whether any ends.
static int audio_assemble(ef_ctx* c, const uint8_t* end_of_stream, cudaStream_t cs, bool* any_end)
{
    const int n = c->cfg.n_streams, a = c->active, p = c->pending;
    CK(cudaEventSynchronize(c->ev_ended_free));              // the previous call's upload of h_ended has left it
    *any_end = false;
    for (int s = 0; s < n; s++) { c->h_ended[s] = end_of_stream && end_of_stream[s] ? 1 : 0; *any_end |= c->h_ended[s] != 0; }
    CK(cudaStreamWaitEvent(cs, c->ev_up_done[a], 0));        // the demux of the current submit has finished
    if (p >= 0) CK(cudaStreamWaitEvent(cs, c->ev_up_done[p], 0));   // and that of a submit queued behind it (ef_audio_end_kernel)
    CK(cudaStreamWaitEvent(cs, c->ev_aud_done, 0));
    CK(cudaMemcpyAsync(c->d_ended, c->h_ended, (size_t)n, cudaMemcpyHostToDevice, cs));
    CK(cudaEventRecord(c->ev_ended_free, cs));
    const uint64_t* new_off = c->aud_unconsumed ? c->d_aud_off2[a] : nullptr;
    ef_audio_len_kernel<<<(n + 255) / 256, 256, 0, cs>>>(c->d_aud_state, new_off, c->d_lead2[a], c->d_skip2[a], n, c->d_blob_len);
    CK(cudaGetLastError());
    ef_ts_offsets_kernel<<<1, 1024, 0, cs>>>(c->d_blob_len, n, c->d_blob_off, c->d_blob);
    CK(cudaGetLastError());
    ef_audio_assemble_kernel<<<n, 256, 0, cs>>>(c->d_aud_state, c->d_aud2[a], new_off, c->d_lead2[a], c->d_skip2[a], c->d_blob_off, c->d_blob);
    CK(cudaGetLastError());
    c->launches += 3;
    return EF_OK;
}

// ef_audio_end_kernel for the streams this call ends: the current demux gate, and that of a submit queued behind it
static int audio_end(ef_ctx* c, const int* verdict, cudaStream_t cs)
{
    const int n = c->cfg.n_streams, a = c->active, p = c->pending;
    CK(ef_launch_audio_end(c->d_ended, n, c->d_gate2[a], p >= 0 ? c->d_gate2[p] : nullptr, p >= 0 ? c->d_skip2[p] : nullptr, p >= 0 && c->aud_ts[p], verdict, cs));
    c->launches++;
    return EF_OK;
}

int ef_decode_audio(ef_ctx* c, const uint8_t* end_of_stream, ef_audio_info* info, int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !info) return fail(EF_EINVAL, "null argument");
    if (!c->audio) return fail(EF_ESTATE, "ef_decode_audio before ef_audio_enable");
    TRY(audio_constants(c->cfg.device));
    TRY(audio_resolve(c));
    const int n = c->cfg.n_streams;
    cudaStream_t cs = (cudaStream_t)stream;
    bool any_end = false;
    TRY(audio_assemble(c, end_of_stream, cs, &any_end));
    const int rc = audio_decode_blob(c->d_blob, c->d_blob_off, c->d_aud_state, c->d_ended, n, c->aud_scratch, info, pcm, pcm_cap, pdm, cs, &c->launches,
                                     [&] { return any_end ? audio_end(c, nullptr, cs) : EF_OK; });
    CK(cudaEventRecord(c->ev_aud_done, cs));
    if (rc != EF_OK || !pcm) return rc;
    c->aud_unconsumed = false;
    return EF_OK;
}

static bool is_device_ptr(const void* p)
{
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

int ef_decode_audio_async(ef_ctx* c, const uint8_t* end_of_stream, ef_audio_info* info, int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !info || !pcm) return fail(EF_EINVAL, "null argument");
    if (!c->audio) return fail(EF_ESTATE, "ef_decode_audio_async before ef_audio_enable");
    if (!is_device_ptr(info) || !is_device_ptr(pcm) || (pdm && !is_device_ptr(pdm)))
        return fail(EF_EINVAL, "ef_decode_audio_async takes device memory for info, pcm and pdm");
    TRY(audio_constants(c->cfg.device));
    // whether this call takes the current submit's audio depends on the outstanding call only when that one took it
    if (c->aud_async && c->aud_async_new) TRY(audio_resolve(c));
    const int n = c->cfg.n_streams;
    AudioScratch& w = c->aud_scratch;
    if (!w.fits(AudioScratch::VROWS, audio_vrow_bytes(n, pcm_cap)) || !w.fits(AudioScratch::VERDICT, sizeof(int))) {
        CK(cudaEventSynchronize(c->ev_aud_done));            // the scratch grows: no earlier call may still use it
        TRY(audio_scratch(w, n, pcm_cap));
    }
    if (!c->h_aud_verdict) TRY(host_alloc(c, &c->h_aud_verdict, 1));
    cudaStream_t cs = (cudaStream_t)stream;
    bool any_end = false;
    TRY(audio_assemble(c, end_of_stream, cs, &any_end));
    TRY(audio_plan(c->d_blob, c->d_blob_off, c->d_aud_state, c->d_ended, n, w, pcm_cap, info, cs, &c->launches));
    TRY(audio_run(c->d_blob, c->d_blob_off, c->d_aud_state, c->d_ended, n, w, pcm_cap, pcm, pdm, true, cs, &c->launches));
    if (any_end) TRY(audio_end(c, (const int*)w.p[AudioScratch::VERDICT], cs));
    CK(cudaMemcpyAsync(c->h_aud_verdict, w.p[AudioScratch::VERDICT], sizeof(int), cudaMemcpyDeviceToHost, cs));
    CK(cudaEventRecord(c->ev_aud_done, cs));
    c->aud_async = true;
    c->aud_async_new = c->aud_unconsumed;
    return EF_OK;
}

int ef_audio_wait(ef_ctx* c)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(audio_resolve(c));
    if (c->aud_async_rc == EF_ENOMEM) return fail(EF_ENOMEM, "the last ef_decode_audio_async exceeded its pcm_cap: nothing was decoded, no state changed");
    return c->aud_async_rc;
}

// ---- presentation timestamps: push_video(frame, front, _last_pts, mode) player.cpp:692-702, get_pts() player.cpp:653-656 ----
int ef_pts_enable(ef_ctx* c)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (c->pts) return EF_OK;
    const int n = c->cfg.n_streams;
    const size_t packets = c->cfg.es_capacity / 188 + 1;
    for (int b = 0; b < 2; b++) {
        TRY(dev_alloc(c, &c->d_pts_off2[b], packets)); TRY(dev_alloc(c, &c->d_pts_val2[b], packets)); TRY(dev_alloc(c, &c->d_pts_span2[b], (size_t)n));
    }
    TRY(dev_alloc(c, &c->d_pts_carry, (size_t)n)); TRY(dev_alloc(c, &c->d_pts_last, (size_t)n));
    TRY(dev_alloc(c, &c->d_pic_pts, (size_t)n * c->cfg.max_pictures));
    CK(cudaDeviceSynchronize());                          // a queued TS submit was demuxed without PES lists: it carries none
    for (int b = 0; b < 2; b++) CK(cudaMemset(c->d_pts_span2[b], 0, (size_t)n * sizeof(uint2)));
    CK(cudaMemset(c->d_pts_carry, 0xFF, (size_t)n * 8));
    CK(cudaMemset(c->d_pts_last, 0xFF, (size_t)n * 8));
    CK(cudaMemset(c->d_pic_pts, 0xFF, (size_t)n * c->cfg.max_pictures * 8));
    CK(cudaDeviceSynchronize());
    c->pts = true;
    c->pts_resolved = false;
    return EF_OK;
}

int ef_picture_pts(ef_ctx* c, int first, int count, int n_pictures, int64_t* pic_pts, int64_t* last_pts)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->pts) return fail(EF_ESTATE, "ef_picture_pts before ef_pts_enable");
    if (!c->pts_resolved) return fail(EF_ESTATE, "ef_picture_pts before ef_index");
    if (first < 0 || count < 1 || first > c->cfg.n_streams - count) return fail(EF_EINVAL, "stream range out of bounds");
    if (n_pictures < 0 || n_pictures > c->cfg.max_pictures) return fail(EF_EINVAL, "n_pictures %d out of range", n_pictures);
    CK(cudaDeviceSynchronize());
    const size_t mp = (size_t)c->cfg.max_pictures;
    if (pic_pts && n_pictures)
        CK(cudaMemcpy2D(pic_pts, (size_t)n_pictures * 8, c->d_pic_pts + (size_t)first * mp, mp * 8, (size_t)n_pictures * 8, (size_t)count, cudaMemcpyDeviceToHost));
    if (last_pts) CK(cudaMemcpy(last_pts, c->d_pts_last + first, (size_t)count * 8, cudaMemcpyDeviceToHost));
    return EF_OK;
}

// ---- paced presentation: push_video(frame, front, pts, mode) video.cpp:1023-1057 + video_isr video.cpp:1122-1198 per stream ----
int ef_present_enable(ef_ctx* c, const uint32_t* frame_counter0)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (c->paced) return fail(EF_ESTATE, "ef_present_enable: already enabled");
    if (!c->pts || !c->video) return fail(EF_ESTATE, "ef_present_enable needs ef_pts_enable and ef_video_init first");
    const int n = c->cfg.n_streams;
    if (!c->d_pace) {
        TRY(dev_alloc(c, &c->d_pace, (size_t)n)); TRY(dev_alloc(c, &c->d_pace_next, (size_t)n)); TRY(dev_alloc(c, &c->d_pace_run, (size_t)n));
        TRY(dev_alloc(c, &c->d_pace_out, (size_t)n)); TRY(dev_alloc(c, &c->d_pace_first, (size_t)n)); TRY(dev_alloc(c, &c->d_pace_arg, (size_t)n));
        TRY(host_alloc(c, &c->h_pace_out, (size_t)n)); TRY(host_alloc(c, &c->h_pace_first, (size_t)n)); TRY(host_alloc(c, &c->h_pace_arg, (size_t)n));
        TRY(host_alloc(c, &c->h_pace_npics, 1));
    }
    std::vector<EfPaceState> st((size_t)n);
    for (int s = 0; s < n; s++) {                         // line 0 of field frame_counter0[s], no frame presented, no origin
        memset(&st[s], 0, sizeof(EfPaceState));
        st[s].fc = frame_counter0 ? frame_counter0[s] : 0u;
        st[s].cur = -1;
    }
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(c->d_pace, st.data(), st.size() * sizeof(EfPaceState), cudaMemcpyHostToDevice));
    c->paced = true;
    c->pace_ntsc = c->h.geo.ntsc;
    c->pace_indexed = false;
    return EF_OK;
}

int ef_present_format(ef_ctx* c, int format)
{
    if (!c) return fail(EF_EINVAL, "null context");
    if (format != EF_FIELD_U16 && format != EF_FIELD_DAC8) return fail(EF_EINVAL, "unknown field format %d", format);
    if (c->paced) return fail(EF_ESTATE, "ef_present_format after ef_present_enable");
    c->pace_format = format;
    return EF_OK;
}

// The halves of a presentation call that the synchronous and the asynchronous calls share, all on `st`:
//   present_schedule  the call's modes / idle field counts (through the pinned buffer `pinned`) and the schedule, one thread per
//                     stream, into scratch
//   present_parse     K1a when `pic` starts a range: once per rec_pics picture indices, as ef_decode_all, and again from the index
//                     an asynchronous chain failed at
//   present_recon     K1b of picture index `pic`
//   present_room      the descriptor and per-field overlay arrays grown to `fields` (waits for what may still read them)
//   present_render    descriptors and state commit, then the paced K2 over `slots` output slots; gated: both decided on the device
static int present_schedule(ef_ctx* c, int pic, const uint8_t* modes, const uint32_t* idle_n, void* pinned, cudaStream_t st)
{
    const int n = c->cfg.n_streams;
    if (pic >= 0 && modes) memcpy(pinned, modes, (size_t)n);
    if (pic < 0) memcpy(pinned, idle_n, (size_t)n * 4);
    const bool arg = pic < 0 || modes;
    if (arg) CK(cudaMemcpyAsync(c->d_pace_arg, pinned, pic < 0 ? (size_t)n * 4 : (size_t)n, cudaMemcpyHostToDevice, st));
    if (c->d_clk) {                                        // update_progress() at the call's start, staged after the caller's changes
        ef_clock_kernel<<<n, 128, 0, st>>>(c->d_clk, c->d_ovl, c->d_ovl_clk, c->d_clk_bm, c->d_pic_pts, c->h.n_pics, c->d_pts_last, pic, c->cfg.max_pictures,
                                           c->d_font, c->d_font_rights);
        CK(cudaGetLastError());
        c->launches++;
    }
    ef_pace_kernel<<<(n + 127) / 128, 128, 0, st>>>(c->d_pace, c->d_pace_next, c->d_pace_run, c->d_pace_out, c->d_pic_pts, c->h.n_pics, c->h.base_pics,
                                                   pic >= 0 && modes ? (const uint8_t*)c->d_pace_arg : nullptr, (const uint32_t*)c->d_pace_arg, pic,
                                                   c->cfg.max_pictures, n, c->pace_ntsc, c->d_clk ? c->d_ovl_clk : c->d_ovl, c->d_ovl_next);
    CK(cudaGetLastError());
    c->launches++;
    return EF_OK;
}

static int present_parse(ef_ctx* c, int pic, cudaStream_t st)
{
    if (pic != c->pace_parse_at) return EF_OK;
    const int k = c->pace_npics - pic < c->h.rec_pics ? c->pace_npics - pic : c->h.rec_pics;
    c->pace_p0 = pic;
    c->pace_parse_at = pic + k;
    return decode_parse(c, pic, k, st);
}

static int present_recon(ef_ctx* c, int pic, cudaStream_t st)
{
    TRY(decode_recon(c, pic - c->pace_p0, st));
    CK(cudaEventRecord(c->ev_buf_free[c->active], st));   // the front ES buffer is in use until here
    c->pace_next = pic + 1;
    return EF_OK;
}

static int present_room(ef_ctx* c, uint64_t fields, cudaStream_t st)
{
    const bool desc = fields > c->desc_cap, fovl = c->d_ovl && fields > c->fovl_cap;
    if (!desc && !fovl) return EF_OK;
    CK(cudaStreamSynchronize(st));
    if (c->pace_async) CK(cudaEventSynchronize(c->ev_pace_done));   // the calls of the outstanding chain, on whatever stream
    if (desc) { TRY(dev_grow(c, &c->d_desc, c->desc_cap, fields, false)); c->desc_cap = fields; }
    if (fovl) { TRY(dev_grow(c, &c->d_fovl, c->fovl_cap, fields, false)); c->fovl_cap = fields; }
    return EF_OK;
}

static int present_render(ef_ctx* c, uint8_t* dst, uint64_t slots, bool gated, cudaStream_t st)
{
    EfFieldOverlay* fovl = c->d_ovl ? c->d_fovl : nullptr;
    CK(ef_launch_pace_fill(c->d_pace, c->d_pace_next, c->d_pace_run, c->d_pace_first, c->d_desc, c->d_ovl, c->d_ovl_next, fovl, c->cfg.n_streams,
                           gated ? c->d_pace_chain : nullptr, st));
    c->launches++;
    if (c->d_clk) {
        CK(ef_launch_clock_commit(c->d_clk, c->d_ovl_clk, c->d_clk_bm, c->d_ovl_slots, c->cfg.n_streams, gated ? c->d_pace_chain : nullptr, st));
        c->launches++;
    }
    CK(ef_launch_composite_paced(c->d, c->h.geo, c->d_desc, slots, dst, c->pace_format == EF_FIELD_DAC8, st, &c->launches, fovl, c->d_ovl_slots,
                                 gated ? c->d_pace_total : nullptr));
    return EF_OK;
}

static int present_check_modes(ef_ctx* c, int pic, const uint8_t* modes)
{
    if (pic >= 0) for (int s = 0; modes && s < c->cfg.n_streams; s++) if (modes[s] > 3) return fail(EF_EINVAL, "mode %d of stream %d is not 0..3", modes[s], s);
    return EF_OK;
}

// The synchronous call: the schedule, one read of the counts, then - unless this is a sizing call or dst is too small - the decode
// of picture index `pic`, the descriptors and state commit, and the paced K2.
static int present_common(ef_ctx* c, int pic, const uint8_t* modes, const uint32_t* idle_n, uint16_t* dst, uint64_t dst_fields, ef_present_info* info,
                          cudaStream_t st)
{
    const int n = c->cfg.n_streams;
    if ((uintptr_t)dst & 15) return fail(EF_EINVAL, "dst must be 16-byte aligned");
    TRY(present_check_modes(c, pic, modes));
    TRY(present_schedule(c, pic, modes, idle_n, c->h_pace_arg, st));
    CK(cudaMemcpyAsync(c->h_pace_out, c->d_pace_out, (size_t)n * sizeof(EfPaceOut), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    uint64_t total = 0;
    for (int s = 0; s < n; s++) {
        c->h_pace_out[s].first = c->h_pace_first[s] = total;
        total += c->h_pace_out[s].n_fields;
    }
    memcpy(info, c->h_pace_out, (size_t)n * sizeof(EfPaceOut));
    if (!dst) return EF_OK;                                // sizing call: nothing decoded, no state changed
    if (total > dst_fields) return fail(EF_ENOMEM, "%llu fields, capacity %llu", (unsigned long long)total, (unsigned long long)dst_fields);
    if (pic >= 0) {
        TRY(present_parse(c, pic, st));
        TRY(present_recon(c, pic, st));
    }
    TRY(present_room(c, total, st));
    CK(cudaMemcpyAsync(c->d_pace_first, c->h_pace_first, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    TRY(present_render(c, (uint8_t*)dst, total, false, st));
    CK(cudaStreamSynchronize(st));                         // the pinned offsets and the scratch are free for the next call
    return EF_OK;
}

// The asynchronous call: the same work, sized on the device (ef_pace_size_kernel) between the parse and the reconstruction, with
// the fill and K2 gated on the chain's verdict. Waits for the host only when the descriptor arrays grow (dst_fields grew) and
// when the ring slot of its arguments is still in use by the call kPaceRing calls back.
static int present_async(ef_ctx* c, int pic, const uint8_t* modes, const uint32_t* idle_n, uint16_t* dst, uint64_t dst_fields, ef_present_info* info,
                         cudaStream_t st)
{
    const int n = c->cfg.n_streams;
    if (!dst || !info || !is_device_ptr(dst) || !is_device_ptr(info)) return fail(EF_EINVAL, "the async present calls take device memory for dst and info");
    if ((uintptr_t)dst & 15) return fail(EF_EINVAL, "dst must be 16-byte aligned");
    TRY(present_check_modes(c, pic, modes));
    if (!c->d_pace_chain) {
        TRY(dev_alloc(c, &c->d_pace_chain, 2)); TRY(dev_alloc(c, &c->d_pace_total, 1));
        TRY(host_alloc(c, &c->h_pace_chain, 2)); TRY(host_alloc(c, &c->h_pace_ring, (size_t)ef_ctx::kPaceRing * n));
        TRY(event(c, &c->ev_pace_done));
        for (cudaEvent_t& e : c->ev_pace_ring) TRY(event(c, &e));
    }
    TRY(present_room(c, dst_fields, st));
    if (!c->pace_async) {                                  // a new chain
        CK(cudaMemsetAsync(c->d_pace_chain, 0, 2 * sizeof(int), st));
        c->chain_next.clear(); c->chain_pic.clear();
        c->pace_async = true;
        c->pace_async_rc = EF_OK; c->pace_async_n = 0;
    } else CK(cudaStreamWaitEvent(st, c->ev_pace_done, 0)); // after the chain's previous call, on whatever stream it ran
    const int k = c->pace_ring_i;
    c->pace_ring_i = (k + 1) % ef_ctx::kPaceRing;
    CK(cudaEventSynchronize(c->ev_pace_ring[k]));
    TRY(present_schedule(c, pic, modes, idle_n, c->h_pace_ring + (size_t)k * n, st));
    CK(cudaEventRecord(c->ev_pace_ring[k], st));
    c->chain_next.push_back(c->pace_next);
    c->chain_pic.push_back(pic);
    if (pic >= 0) TRY(present_parse(c, pic, st));       // before the size kernel, which may zero its records
    uint32_t* rec = pic >= 0 ? c->h.mb_info + (size_t)(pic - c->pace_p0) * n * EF_MBW_MAX * EF_MBH_MAX : nullptr;
    ef_pace_size_kernel<<<1, 1024, 0, st>>>(c->d_pace_out, n, dst_fields, c->d_pace_first, (EfPaceOut*)info, c->d_pace_total, c->d_pace_chain, rec);
    CK(cudaGetLastError());
    c->launches++;
    if (pic >= 0) TRY(present_recon(c, pic, st));
    TRY(present_render(c, (uint8_t*)dst, dst_fields, true, st));
    CK(cudaMemcpyAsync(c->h_pace_chain, c->d_pace_chain, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(c->ev_pace_done, st));
    return EF_OK;
}

// the checks of a picture call: order and state
static int present_picture_check(ef_ctx* c, int pic, const char* what)
{
    if (!c->paced) return fail(EF_ESTATE, "%s before ef_present_enable", what);
    if (!c->pace_indexed) return fail(EF_ESTATE, "%s before an ef_index that followed ef_present_enable", what);
    TRY(pace_pictures(c));
    if (pic != c->pace_next || pic >= c->pace_npics)
        return fail(EF_ESTATE, "%s(%d): the next picture index is %d of %d", what, pic, c->pace_next, c->pace_npics);
    return EF_OK;
}

int ef_present_picture(ef_ctx* c, int pic, const uint8_t* modes, uint16_t* dst, uint64_t dst_fields, ef_present_info* info, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !info) return fail(EF_EINVAL, "null argument");
    TRY(pace_resolve(c));
    TRY(present_picture_check(c, pic, "ef_present_picture"));
    return present_common(c, pic, modes, nullptr, dst, dst_fields, info, (cudaStream_t)stream);
}

int ef_present_idle(ef_ctx* c, const uint32_t* n_fields, uint16_t* dst, uint64_t dst_fields, ef_present_info* info, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !info || !n_fields) return fail(EF_EINVAL, "null argument");
    if (!c->paced) return fail(EF_ESTATE, "ef_present_idle before ef_present_enable");
    TRY(pace_resolve(c));
    return present_common(c, -1, nullptr, n_fields, dst, dst_fields, info, (cudaStream_t)stream);
}

int ef_present_picture_async(ef_ctx* c, int pic, const uint8_t* modes, uint16_t* dst, uint64_t dst_fields, ef_present_info* info, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(present_picture_check(c, pic, "ef_present_picture_async"));
    return present_async(c, pic, modes, nullptr, dst, dst_fields, info, (cudaStream_t)stream);
}

int ef_present_idle_async(ef_ctx* c, const uint32_t* n_fields, uint16_t* dst, uint64_t dst_fields, ef_present_info* info, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !n_fields) return fail(EF_EINVAL, "null argument");
    if (!c->paced) return fail(EF_ESTATE, "ef_present_idle_async before ef_present_enable");
    return present_async(c, -1, nullptr, n_fields, dst, dst_fields, info, (cudaStream_t)stream);
}

int ef_present_wait(ef_ctx* c, int* n_presented)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(pace_resolve(c));
    if (n_presented) *n_presented = c->pace_async_n;
    if (c->pace_async_rc == EF_ENOMEM)
        return fail(EF_ENOMEM, "call %d of the last ef_present_*_async chain exceeded its dst_fields: it and the calls after it changed nothing", c->pace_async_n);
    return c->pace_async_rc;
}

// ---- overlay of paced presentation: _video_composite, _video_composite_blend, _video_composite_progress per stream (video.cpp:839-887) ----
// the overlay state, allocated by the first ef_present_overlay or ef_present_clock
static int overlay_alloc(ef_ctx* c)
{
    if (c->d_ovl) return EF_OK;
    const int n = c->cfg.n_streams;
    TRY(dev_alloc(c, &c->d_ovl, (size_t)n)); TRY(dev_alloc(c, &c->d_ovl_next, (size_t)n)); TRY(dev_alloc(c, &c->d_ovl_cmd, (size_t)n));
    TRY(dev_alloc(c, &c->d_ovl_slots, (size_t)n * 2 * EF_OVERLAY_BYTES)); TRY(dev_alloc(c, &c->d_ovl_in, (size_t)n * EF_OVERLAY_BYTES));
    CK(cudaMemset(c->d_ovl, 0, (size_t)n * sizeof(EfOverlayState)));   // blend 0: nothing drawn
    CK(cudaMemset(c->d_ovl_slots, 0, (size_t)n * 2 * EF_OVERLAY_BYTES));
    return EF_OK;
}

int ef_present_overlay(ef_ctx* c, int first, int count, const uint8_t* bitmaps, const int32_t* blend, const int32_t* progress, const uint8_t* set)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->paced) return fail(EF_ESTATE, "ef_present_overlay before ef_present_enable");
    TRY(pace_resolve(c));
    TRY(stream_range(c, first, count));
    std::vector<EfOverlayCmd> cmd((size_t)count);
    for (int i = 0; i < count; i++) {
        uint32_t m = set ? set[i] & 7u : 7u;
        if (!bitmaps) m &= ~1u;
        if (!blend) m &= ~2u;
        if (!progress) m &= ~4u;
        if ((m & 2u) && blend[i] < -1) return fail(EF_EINVAL, "blend %d of stream %d is below -1", blend[i], first + i);
        cmd[i] = { (m & 2u) ? blend[i] : 0, (m & 4u) ? progress[i] : 0, m, 0u };
    }
    TRY(overlay_alloc(c));
    if (!count) return EF_OK;
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(c->d_ovl_cmd, cmd.data(), cmd.size() * sizeof(EfOverlayCmd), cudaMemcpyHostToDevice));
    if (bitmaps) CK(cudaMemcpy(c->d_ovl_in, bitmaps, (size_t)count * EF_OVERLAY_BYTES, cudaMemcpyHostToDevice));
    ef_overlay_stage_kernel<<<count, 96>>>(c->d_ovl, c->d_ovl_slots, c->d_ovl_cmd, c->d_ovl_in, first);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaDeviceSynchronize());
    return EF_OK;
}

// ---- clock of paced presentation: ESPFlix::update_progress() (espflix.cpp:862-874) per stream ----
int ef_present_font(ef_ctx* c, const uint8_t* atlas, const int16_t* rights, int n_rights)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !atlas || !rights) return fail(EF_EINVAL, "null argument");
    if (n_rights < ':' - 0x18 + 1 || n_rights > EF_FONT_W) return fail(EF_EINVAL, "n_rights %d does not cover glyphs 0x18..':' (%d)", n_rights, ':' - 0x18 + 1);
    for (int i = 0; i < n_rights; i++)
        if (rights[i] > EF_FONT_W || rights[i] <= (i ? rights[i - 1] : 0))
            return fail(EF_EINVAL, "rights[%d] = %d: the glyph edges must increase from above 0 up to %d", i, rights[i], EF_FONT_W);
    TRY(pace_resolve(c));
    if (!c->d_font) { TRY(dev_alloc(c, &c->d_font, (size_t)16 * EF_FONT_W)); TRY(dev_alloc(c, &c->d_font_rights, (size_t)EF_FONT_W)); }
    CK(cudaDeviceSynchronize());                          // a present call may still draw with the old atlas
    CK(cudaMemcpy(c->d_font, atlas, (size_t)16 * EF_FONT_W, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_font_rights, rights, (size_t)n_rights * 2, cudaMemcpyHostToDevice));
    return EF_OK;
}

int ef_present_clock(ef_ctx* c, int first, int count, const uint8_t* idx_hdrs, const int8_t* speed, const uint8_t* flags)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->paced) return fail(EF_ESTATE, "ef_present_clock before ef_present_enable");
    if (!c->d_font) return fail(EF_ESTATE, "ef_present_clock before ef_present_font");
    const int n = c->cfg.n_streams;
    TRY(stream_range(c, first, count));
    if (count && (!idx_hdrs || !speed || !flags)) return fail(EF_EINVAL, "null argument");
    std::vector<idx_hdr> hdr((size_t)count);
    if (count) memcpy(hdr.data(), idx_hdrs, (size_t)count * sizeof(idx_hdr));
    for (int i = 0; i < count; i++) {
        if (speed[i] < -1 || speed[i] > 1) return fail(EF_EINVAL, "speed %d of stream %d is not -1..1", speed[i], first + i);
        if (!(flags[i] & 1u)) continue;
        const idx_hdr& h = hdr[(size_t)i];
        if (h.video.last_pts == 0) return fail(EF_EINVAL, "stream %d: video.last_pts is 0 (the progress divides by it)", first + i);
        if (speed[i] == 1 && h.fwd.last_pts == h.fwd.first_pts) return fail(EF_EINVAL, "stream %d: the fwd record spans no pts", first + i);
        if (speed[i] == -1 && h.rev.last_pts == h.rev.first_pts) return fail(EF_EINVAL, "stream %d: the rwd record spans no pts", first + i);
    }
    TRY(pace_resolve(c));
    TRY(overlay_alloc(c));
    if (!c->d_clk) {
        TRY(dev_alloc(c, &c->d_clk, (size_t)n)); TRY(dev_alloc(c, &c->d_ovl_clk, (size_t)n)); TRY(dev_alloc(c, &c->d_clk_bm, (size_t)n * EF_OVERLAY_BYTES));
        CK(cudaMemset(c->d_clk, 0, (size_t)n * sizeof(EfClockState)));    // every clock off, _last_seconds 0
    }
    if (!count) return EF_OK;
    CK(cudaDeviceSynchronize());
    std::vector<EfClockState> st((size_t)count);
    CK(cudaMemcpy(st.data(), c->d_clk + first, (size_t)count * sizeof(EfClockState), cudaMemcpyDeviceToHost));
    for (int i = 0; i < count; i++) {
        EfClockState& k = st[(size_t)i];
        const idx_hdr& h = hdr[(size_t)i];
        k.v_first = h.video.first_pts; k.v_last = h.video.last_pts;
        k.f_first = h.fwd.first_pts; k.f_last = h.fwd.last_pts;
        k.r_first = h.rev.first_pts; k.r_last = h.rev.last_pts;
        k.speed = speed[i];
        k.flags = flags[i] & 3u;
        if (flags[i] & 4u) k.last_seconds = 0;
    }
    CK(cudaMemcpy(c->d_clk + first, st.data(), (size_t)count * sizeof(EfClockState), cudaMemcpyHostToDevice));
    return EF_OK;
}

// ---- titles held in device memory: the reference's Streamer (espflix.cpp:723-747) and ESPFlix's navigation (espflix.cpp:787-859) --
int ef_library_add(ef_ctx* c, const uint8_t* idx, uint64_t idx_bytes, const uint8_t* const* ts, const uint64_t* bytes, int* title)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !idx || !ts || !bytes || !title) return fail(EF_EINVAL, "null argument");
    if (idx_bytes < sizeof(idx_hdr) || idx_bytes >> 32) return fail(EF_EINVAL, "video.idx of %llu bytes: a header of 104 bytes and below 4 GiB", (unsigned long long)idx_bytes);
    idx_hdr h;
    memcpy(&h, idx, sizeof(h));
    if (h.sig != 0x00584449u || h.len != 3) return fail(EF_EINVAL, "video.idx: signature %08x and %u records, not 'IDX' and 3", h.sig, h.len);
    if (!ts[1] || !bytes[1]) return fail(EF_EINVAL, "the title needs its main file (video.ts)");
    for (int f = 0; f < 3; f++) {
        if (!ts[f] != !bytes[f]) return fail(EF_EINVAL, "file %d: a pointer and a size, or neither", f);
        if (bytes[f] % 188 || bytes[f] >> 32) return fail(EF_EINVAL, "file %d of %llu bytes: whole 188-byte packets below 4 GiB", f, (unsigned long long)bytes[f]);
    }
    const uint64_t samples = (uint64_t)h.video.sample_count + h.fwd.sample_count + h.rev.sample_count;
    if (sizeof(idx_hdr) + 4 * samples > idx_bytes) return fail(EF_EINVAL, "video.idx: %llu samples run past its %llu bytes", (unsigned long long)samples, (unsigned long long)idx_bytes);
    if (!h.video.bin_size || !h.video.sample_count) return fail(EF_EINVAL, "video.idx: the video record has bin_size %u and %u samples", h.video.bin_size, h.video.sample_count);
    const idx_rec* trick[2] = { &h.rev, &h.fwd };
    for (int k = 0; k < 2; k++) {
        const idx_rec& r = *trick[k];
        if (ts[2 * k] && (!r.trick_speed || !r.bin_size || !r.sample_count || r.last_pts == r.first_pts))
            return fail(EF_EINVAL, "video.idx: the %s record (trick_speed %u, bin_size %u, %u samples, pts %lld..%lld) cannot be played", k ? "fwd" : "rwd",
                        r.trick_speed, r.bin_size, r.sample_count, (long long)r.first_pts, (long long)r.last_pts);
    }
    const int n = c->cfg.n_streams;
    if (!c->d_lib) {                                      // the first title: every stream's state, the staging buffer of the submits
        TRY(dev_alloc(c, &c->d_lib, (size_t)n));
        TRY(dev_alloc(c, &c->d_lib_stage, c->cfg.es_capacity + 64));
        TRY(dev_alloc(c, &c->d_lib_src, (size_t)n)); TRY(dev_alloc(c, &c->d_lib_off, (size_t)n + 1));
        TRY(dev_alloc(c, &c->d_lib_end, (size_t)n)); TRY(dev_alloc(c, &c->d_lib_budget, (size_t)n));
        TRY(event(c, &c->ev_lib_staged));
        CK(cudaEventRecord(c->ev_lib_staged, 0));
        std::vector<EfLibStream> idle((size_t)n, EfLibStream{ -1, 0, EF_LIB_IDLE, 1, 0, 0 });
        CK(cudaMemcpy(c->d_lib, idle.data(), (size_t)n * sizeof(EfLibStream), cudaMemcpyHostToDevice));
    }
    if (c->lib_titles.size() == c->lib_cap) {
        const size_t cap = c->lib_cap ? 2 * c->lib_cap : 16;
        CK(cudaDeviceSynchronize());                      // a command or a submit may still read the title table
        TRY(dev_grow(c, &c->d_lib_titles, c->lib_cap, cap, c->lib_cap > 0));
        c->lib_cap = cap;
    }
    EfLibTitle t;
    memset(&t, 0, sizeof(t));
    uint8_t* p = nullptr;
    TRY(dev_alloc(c, &p, idx_bytes));
    CK(cudaMemcpy(p, idx, idx_bytes, cudaMemcpyHostToDevice));
    t.idx = p; t.idx_bytes = (uint32_t)idx_bytes;
    for (int f = 0; f < 3; f++) {
        if (!bytes[f]) continue;
        TRY(dev_alloc(c, &p, bytes[f]));
        CK(cudaMemcpy(p, ts[f], bytes[f], cudaMemcpyHostToDevice));
        t.ts[f] = p; t.bytes[f] = (uint32_t)bytes[f];
    }
    t.v_first = h.video.first_pts; t.v_last = h.video.last_pts; t.f_first = h.fwd.first_pts; t.f_last = h.fwd.last_pts;
    t.r_first = h.rev.first_pts; t.r_last = h.rev.last_pts;
    t.v_bin = h.video.bin_size; t.f_bin = h.fwd.bin_size; t.r_bin = h.rev.bin_size;
    t.f_trick = h.fwd.trick_speed; t.r_trick = h.rev.trick_speed;
    t.v_n = h.video.sample_count; t.f_n = h.fwd.sample_count; t.r_n = h.rev.sample_count;
    CK(cudaMemcpy(c->d_lib_titles + c->lib_titles.size(), &t, sizeof(t), cudaMemcpyHostToDevice));
    *title = (int)c->lib_titles.size();
    c->lib_titles.push_back(t);
    return EF_OK;
}

// The state that commands and submits need: a title loaded, PTS (get_pts()) and carry (submits cut at any packet) enabled
static int library_ready(ef_ctx* c, const char* what)
{
    if (!c->d_lib) return fail(EF_ESTATE, "%s before the first ef_library_add", what);
    if (!c->pts || !c->carry) return fail(EF_ESTATE, "%s needs ef_pts_enable and ef_carry_enable", what);
    return EF_OK;
}

int ef_library_command(ef_ctx* c, int first, int count, int cmd, int title, int64_t arg)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(library_ready(c, "ef_library_command"));
    TRY(stream_range(c, first, count));
    if (cmd < EF_LIB_PLAY_AT || cmd > EF_LIB_STOP) return fail(EF_EINVAL, "unknown command %d", cmd);
    if (cmd == EF_LIB_PLAY_AT && (title < 0 || (size_t)title >= c->lib_titles.size())) return fail(EF_EINVAL, "unknown title %d", title);
    if (cmd == EF_LIB_SKIP && (arg < INT32_MIN || arg > INT32_MAX)) return fail(EF_EINVAL, "skip of %lld seconds is not an int", (long long)arg);
    TRY(restart_ready(c, "ef_library_command"));
    if (!count) return EF_OK;
    CK(cudaDeviceSynchronize());                          // a library submit may still move the cursors
    std::vector<EfLibStream> st((size_t)count);
    CK(cudaMemcpy(st.data(), c->d_lib + first, (size_t)count * sizeof(EfLibStream), cudaMemcpyDeviceToHost));
    for (int i = 0; i < count; i++) {
        const EfLibStream& v = st[(size_t)i];
        if (cmd == EF_LIB_PLAY_AT) continue;
        if (v.state == EF_LIB_IDLE) return fail(EF_EINVAL, "stream %d has never played: start it with EF_LIB_PLAY_AT", first + i);
        if (cmd == EF_LIB_RESUME && v.state != EF_LIB_PAUSED) return fail(EF_EINVAL, "EF_LIB_RESUME on stream %d, which is not paused", first + i);
        const EfLibTitle& t = c->lib_titles[(size_t)v.title];
        if ((cmd == EF_LIB_FAST_FORWARD && !t.ts[2]) || (cmd == EF_LIB_REWIND && !t.ts[0]))
            return fail(EF_EINVAL, "stream %d: title %d has no %s file", first + i, v.title, cmd == EF_LIB_REWIND ? "rewind" : "fast-forward");
    }
    CK(ef_launch_library_resolve(c->d_lib, c->d_lib_titles, c->d_pts_last, first, count, cmd, title, arg));
    c->launches++;
    const uint8_t op = cmd <= EF_LIB_REWIND ? 1 : cmd == EF_LIB_RESUME ? 2 : 0;   // play(): reset + video_reset; video_pause(0)
    if (op) {
        const std::vector<uint8_t> ops((size_t)count, op);
        return restart_apply(c, first, count, ops.data());
    }
    CK(cudaDeviceSynchronize());
    return EF_OK;
}

int ef_library_submit(ef_ctx* c, uint32_t packets, const uint32_t* per_stream, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    TRY(library_ready(c, "ef_library_submit"));
    if (c->pending >= 0) return fail(EF_ESTATE, "ef_library_submit with a submit pending: ef_index it first");
    const int n = c->cfg.n_streams;
    uint64_t bound = 0;                                   // packets the submit can hold at most, known without reading the device
    if (per_stream) for (int i = 0; i < n; i++) bound += per_stream[i];
    else bound = (uint64_t)n * packets;
    if (bound * 188 > c->cfg.es_capacity)
        return fail(EF_ENOMEM, "a library submit of up to %llu packets exceeds es_capacity %zu", (unsigned long long)bound, c->cfg.es_capacity);
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaStreamWaitEvent(st, c->ev_lib_staged, 0));   // the upload of the previous library submit has copied the staging buffer
    if (per_stream) CK(cudaMemcpyAsync(c->d_lib_budget, per_stream, (size_t)n * 4, cudaMemcpyHostToDevice, st));
    CK(ef_launch_library_gather(c->d_lib, c->d_lib_titles, per_stream ? c->d_lib_budget : nullptr, packets, n, c->d_lib_src, c->d_lib_off,
                                c->d_lib_end, c->d_lib_stage, bound * 188, st, &c->launches));
    TRY(submit_common(c, c->d_lib_stage, c->d_lib_off, false, true, st));
    const int b = c->pending;                             // the streams whose file ends with this submit, as ef_end_streams marks them
    CK(cudaMemcpyAsync(c->d_end2[b], c->d_lib_end, (size_t)n, cudaMemcpyDeviceToDevice, c->up_stream));
    CK(cudaEventRecord(c->ev_up_done[b], c->up_stream));
    CK(cudaEventRecord(c->ev_lib_staged, c->up_stream));
    c->lib_submit = true;
    return EF_OK;
}

int ef_library_info(ef_ctx* c, int first, int count, ef_library_status* status)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->d_lib) return fail(EF_ESTATE, "ef_library_info before the first ef_library_add");
    TRY(stream_range(c, first, count, status));
    if (!count) return EF_OK;
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(status, c->d_lib + first, (size_t)count * sizeof(EfLibStream), cudaMemcpyDeviceToHost));
    return EF_OK;
}

}  // extern "C"

// ---- trick streams: video_fwd.ts and video_rwd.ts of many mains (csrc/ef_trick.cu; the rule is tests/trick_cases.py) --------------
namespace {

constexpr int kTrickSpeed = 15;                  // merge_index's trick_speed
constexpr int kTrickChunkStreams = 256;          // segments decoded in one batch (about 2.2 MB of device memory each)
constexpr uint64_t kTrickChunkBytes = 64u << 20; // TS bytes of one batch (a longer segment is a batch of its own)
constexpr int kTrickEncodeBatch = 256;           // pictures per encode launch (26 MB of frames, 90 MB of slice regions)

struct GrowBuf {                                 // device buffer that keeps its contents when it grows
    uint8_t* p = nullptr;
    size_t cap = 0;
    ~GrowBuf() { if (p) cudaFree(p); }
    cudaError_t reserve(size_t n, size_t keep = 0)
    {
        if (n <= cap) return cudaSuccess;
        uint8_t* q = nullptr;
        cudaError_t e = cudaMalloc(&q, n);
        if (e != cudaSuccess) return e;
        if (keep) { e = cudaMemcpy(q, p, keep, cudaMemcpyDeviceToDevice); if (e != cudaSuccess) { cudaFree(q); return e; } }
        if (p) cudaFree(p);
        p = q; cap = n;
        return cudaSuccess;
    }
};

// Appends to es the video ES of packets pkt.. (PID 0x100 payloads, as demux() reads them, player.cpp:381-432) until es holds `cap`
// bytes or packet `end`; returns the packet after the last one read. *pts_ok (unless null) = packet `pkt` starts a video PES whose
// PTS parse_pts() accepts (player.cpp:299-306).
uint64_t trick_video_es(const uint8_t* ts, uint64_t pkt, uint64_t end, size_t cap, std::vector<uint8_t>& es, bool* pts_ok)
{
    if (pts_ok) *pts_ok = false;
    uint64_t k = pkt;
    for (; k < end && es.size() < cap; k++) {
        const uint8_t* d = ts + k * 188;
        if (d[0] != 0x47 || (((d[1] << 8) | d[2]) & 0x1FFF) != 0x100 || !(d[3] & 0x10)) continue;
        int o = (d[3] & 0x20) ? 5 + d[4] : 4;
        if ((d[1] & 0x40) && o + 14 <= 188) {
            const int flags = (d[o + 6] << 8) | d[o + 7];
            if (k == pkt && pts_ok) *pts_ok = (flags & 0x80) && (d[o + 9] & 0xF0) == ((flags >> 2) & 0x30);
            o += 9 + d[o + 8];
        }
        if (o < 188) es.insert(es.end(), d + o, d + 188);
    }
    return k;
}

// VLC lookup of one ISO 11172-2 table, two levels so that it stays in cache: e[next `first` bits] = (code length << 16) |
// (uint16_t)value, (1 << 31) | offset of a table of the next `bits` - `first` bits for longer codes, or 0 where no code starts
struct TrickVlc {
    std::vector<uint32_t> e;
    int bits = 0, first = 0;
    TrickVlc(const ef_vlc_code* c, int n, const char* extra = nullptr, int extra_value = 0)
    {
        for (int i = 0; i < n; i++) bits = std::max(bits, (int)strlen(c[i].code));
        first = std::min(bits, 10);
        const int sub = bits - first;
        e.assign((size_t)1 << first, 0);
        for (int i = 0; i <= n; i++) {
            const char* code = i < n ? c[i].code : extra;
            if (!code) break;
            const int len = (int)strlen(code);
            const uint32_t val = ((uint32_t)len << 16) | (uint16_t)(i < n ? c[i].value : extra_value);
            uint32_t v = 0;
            for (int k = 0; k < len; k++) v = (v << 1) | (uint32_t)(code[k] == '1');
            if (len <= first) {
                for (uint32_t t = 0; t < (1u << (first - len)); t++) e[(v << (first - len)) | t] = val;
                continue;
            }
            const uint32_t pre = v >> (len - first);
            if (!(e[pre] >> 31)) { e[pre] = (1u << 31) | (uint32_t)e.size(); e.resize(e.size() + ((size_t)1 << sub), 0); }
            const uint32_t off = e[pre] & 0x7FFFFFFFu, rest = v & ((1u << (len - first)) - 1);
            for (uint32_t t = 0; t < (1u << (bits - len)); t++) e[off + ((rest << (bits - len)) | t)] = val;
        }
    }
};

struct TrickBits {                               // MSB-first reader; bytes past the end read as 0
    const uint8_t* p; size_t n, pos;
    uint32_t peek(int k) const                   // k <= 25
    {
        const size_t b = pos >> 3;
        uint64_t w = 0;
        if (b + 8 <= n) { memcpy(&w, p + b, 8); w = __builtin_bswap64(w); }
        else for (size_t i = 0; i < 8; i++) w = (w << 8) | (b + i < n ? p[b + i] : 0);
        return (uint32_t)((w << (pos & 7)) >> (64 - k));
    }
    uint32_t get(int k) { const uint32_t v = k ? peek(k) : 0; pos += k; return v; }
    bool vlc(const TrickVlc& t, int* v)
    {
        uint32_t e = t.e[peek(t.first)];
        if (e >> 31) e = t.e[(e & 0x7FFFFFFFu) + (peek(t.bits) & ((1u << (t.bits - t.first)) - 1))];
        if (!e) return false;
        pos += e >> 16; *v = (int16_t)(e & 0xFFFF);
        return true;
    }
};

// one block's codes (block(), player.cpp:999-1148); false on a code the tables do not hold or a run past the block
bool trick_skip_block(TrickBits& r, int blk, bool intra)
{
    static const TrickVlc dct(ef_vlc_dct, EF_VLC_DCT_COUNT, "000001", 0), dcl(ef_vlc_dc_luma, EF_VLC_DC_LUMA_COUNT),
        dcc(ef_vlc_dc_chroma, EF_VLC_DC_CHROMA_COUNT);
    int n = 0, v;
    if (intra) {
        if (!r.vlc(blk < 4 ? dcl : dcc, &v)) return false;
        r.get(v);
        n = 1;
    }
    for (;;) {
        const uint32_t p = r.peek(2);
        if (n && p == 2) { r.pos += 2; return true; }
        int run = 0;
        if (p >> 1) r.pos += n ? 3 : 2;                          // run 0 level 1 and its sign
        else {
            if (!r.vlc(dct, &v)) return false;
            if (v == 0) { run = (int)r.get(6); const uint32_t l = r.get(8); if (l == 0 || l == 128) r.get(8); }
            else { run = v >> 8; r.pos += 1; }
        }
        n += run;
        if (n >= 64) return false;
        n++;
    }
}

// Whether a segment may start at es, which begins with a sequence header: a decode from the cleared frame stores then gives
// the frames of a continuous decode. The two stores alternate, so the first picture must write every macroblock of the
// picture from its own codes, and the second every one, coded or skipped (a skip copies from the first). The slices are
// walked as the decoder walks them (slice(), player.cpp:1238-1316): a slice starts at column 0 of its row whatever its first
// increment, runs across rows, and an increment above 1 skips macroblocks, which an I picture copies from the other store.
// The first picture must be intra and the second intra or predicted. 1 yes, 0 no, -1 es ends before the answer (`whole`: es
// holds the rest of the main).
int trick_pictures_whole(const std::vector<uint8_t>& es, bool whole)
{
    static const TrickVlc mba(ef_vlc_mba, EF_VLC_MBA_COUNT), type_i(ef_vlc_mbtype_i, EF_VLC_MBTYPE_I_COUNT),
        type_p(ef_vlc_mbtype_p, EF_VLC_MBTYPE_P_COUNT), cbp(ef_vlc_cbp, EF_VLC_CBP_COUNT), mv(ef_vlc_mv, EF_VLC_MV_COUNT);
    if (es.size() < 8 || es[0] || es[1] || es[2] != 1 || es[3] != 0xB3) return whole ? 0 : -1;
    const int mbw = (((es[4] << 4) | (es[5] >> 4)) + 15) >> 4, mbh = ((((es[5] & 15) << 8) | es[6]) + 15) >> 4;
    if (mbw < 1 || mbh < 1) return 0;
    const int tw = std::min(mbw, EF_MBW_MAX), th = std::min(mbh, EF_MBH_MAX);
    uint8_t mb[2][EF_MBW_MAX * EF_MBH_MAX] = {};    // per picture: 0 not written, 1 skipped, 2 coded (the last write counts)
    int pics = 0, type = 0, r_size = 0;
    bool done = false;
    const uint8_t* d = es.data();
    for (size_t j = 2; j + 1 < es.size(); j++) {                        // j: the 0x01 of a start code, found with memchr
        const uint8_t* hit = (const uint8_t*)memchr(d + j, 1, es.size() - 1 - j);
        if (!hit) break;
        j = (size_t)(hit - d);
        if (d[j - 1] || d[j - 2]) continue;
        const size_t i = j - 2;
        const uint8_t c = es[i + 3];
        if (c == 0x00) {
            if (pics == 2) { done = true; break; }
            if (i + 9 > es.size()) return whole ? 0 : -1;
            TrickBits h = { d + i + 4, 5, 0 };
            h.get(10);
            type = (int)h.get(3);
            if (type != 1 && (pics == 0 || type != 2)) return 0;
            h.get(16);
            if (type == 2) { h.get(1); r_size = (int)h.get(3) - 1; if (r_size < 0) return 0; }
            pics++;
        } else if (c == 0xB7) { done = true; break; }
        else if (pics && c >= 0x01 && c <= 0xAF) {
            const uint8_t* nx = nullptr;                                 // the next start code ends the slice's bytes
            for (size_t k = i + 4; k + 2 < es.size() && !nx; k++) {
                const uint8_t* q = (const uint8_t*)memchr(d + k, 1, es.size() - k);
                if (!q) break;
                k = (size_t)(q - d);
                if (k >= i + 6 && !q[-1] && !q[-2]) nx = q - 2;
            }
            if (!nx && !whole) return -1;
            TrickBits r = { d + i + 4, (size_t)((nx ? nx : d + es.size()) - (d + i + 4)), 0 };
            int x = mbw - 1, y = c - 2;
            if (y >= mbh) continue;
            r.get(5);
            while (r.get(1)) r.get(8);
            uint8_t* m = mb[pics - 1];
            auto step = [&]() { if (++x >= mbw) { x -= mbw; y++; } };
            for (int k = 0; r.peek(23) != 0; k++) {
                int inc = 0, v;
                if (!r.vlc(mba, &v)) return 0;
                while (v == 34) if (!r.vlc(mba, &v)) return 0;
                while (v == 35) { inc += 33; if (!r.vlc(mba, &v)) return 0; }
                inc += v;
                if (k) for (; inc > 1 && y < EF_MBH_MAX; inc--) { step(); if (y < EF_MBH_MAX && x < EF_MBW_MAX) m[y * EF_MBW_MAX + x] = 1; }
                step();
                if (y >= EF_MBH_MAX) break;
                if (x < EF_MBW_MAX) m[y * EF_MBW_MAX + x] = 2;
                int t;
                if (!r.vlc(type == 1 ? type_i : type_p, &t)) return 0;
                const bool intra = t & 0x01;
                if (t & 0x10) r.get(5);
                if (!intra && (t & 0x08))
                    for (int a = 0; a < 2; a++) { if (!r.vlc(mv, &v)) return 0; if (v && r_size) r.get(r_size); }
                int pat = intra ? 63 : 0;
                if ((t & 0x02) && !r.vlc(cbp, &pat)) return 0;
                for (int b = 0; b < 6; b++)
                    if ((pat & (0x20 >> b)) && !trick_skip_block(r, b, intra)) return 0;
            }
        }
    }
    if (!done && !whole) return -1;
    if (!pics) return 0;
    for (int yy = 0; yy < th; yy++)
        for (int xx = 0; xx < tw; xx++)
            if (mb[0][yy * EF_MBW_MAX + xx] != 2 || (pics == 2 && !mb[1][yy * EF_MBW_MAX + xx])) return 0;
    return 1;
}

// trick_pictures_whole for the sequence header at packet `pkt`, whose PES must have a PTS parse_pts() accepts: the main (to
// packet `end`) is read on to its third picture start code first, so the pictures are walked once
int trick_cut_ok(const uint8_t* ts, uint64_t pkt, uint64_t end)
{
    std::vector<uint8_t> es;
    bool ok;
    uint64_t next = trick_video_es(ts, pkt, end, 4096, es, &ok);
    if (!ok) return 0;
    for (;;) {
        int pics = 0;
        for (size_t j = 2; j + 1 < es.size() && pics < 3; j++) {
            const uint8_t* hit = (const uint8_t*)memchr(es.data() + j, 1, es.size() - 1 - j);
            if (!hit) break;
            j = (size_t)(hit - es.data());
            if (!es[j - 1] && !es[j - 2] && es[j + 1] == 0x00) pics++;
        }
        if (pics >= 3 || next == end) break;
        next = trick_video_es(ts, next, end, es.size() * 2, es, nullptr);
    }
    return trick_pictures_whole(es, next == end) == 1;
}

void trick_bits(std::vector<uint8_t>& out, uint32_t& acc, int& n, uint32_t v, int bits)
{
    for (int i = bits - 1; i >= 0; i--) {
        acc = (acc << 1) | ((v >> i) & 1);
        if (++n == 8) { out.push_back((uint8_t)acc); acc = 0; n = 0; }
    }
}

// sequence header (352 x 192, the main's aspect and picture-rate codes, bit_rate 0x3FFFF, vbv 20, default matrices), closed GOP
// header, I picture header: tests/trick_cases.header_bytes()
std::vector<uint8_t> trick_header(int aspect, int rate)
{
    std::vector<uint8_t> h = { 0, 0, 1, 0xB3 };
    uint32_t acc = 0; int n = 0;
    trick_bits(h, acc, n, 352, 12); trick_bits(h, acc, n, 192, 12); trick_bits(h, acc, n, aspect, 4); trick_bits(h, acc, n, rate, 4);
    trick_bits(h, acc, n, 0x3FFFF, 18); trick_bits(h, acc, n, 1, 1); trick_bits(h, acc, n, 20, 10); trick_bits(h, acc, n, 0, 3);
    h.insert(h.end(), { 0, 0, 1, 0xB8 });
    trick_bits(h, acc, n, 1u << 12, 25); trick_bits(h, acc, n, 1, 1); trick_bits(h, acc, n, 0, 6);
    h.insert(h.end(), { 0, 0, 1, 0x00 });
    trick_bits(h, acc, n, 0, 10); trick_bits(h, acc, n, 1, 3); trick_bits(h, acc, n, 0xFFFF, 16); trick_bits(h, acc, n, 0, 3);
    return h;
}

struct TrickSeg { int file; uint64_t pkt0, pkt1; };

struct TrickTimer {                              // CUDA event pairs per phase, read once the build has finished
    std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> spans;
    cudaEvent_t open_ev = nullptr;
    ~TrickTimer() { for (auto& s : spans) { cudaEventDestroy(s.second.first); cudaEventDestroy(s.second.second); } if (open_ev) cudaEventDestroy(open_ev); }
    cudaError_t begin(cudaStream_t st)
    {
        cudaError_t e = cudaEventCreate(&open_ev);
        return e != cudaSuccess ? e : cudaEventRecord(open_ev, st);
    }
    cudaError_t end(int phase, cudaStream_t st)
    {
        cudaEvent_t b;
        cudaError_t e = cudaEventCreate(&b);
        if (e != cudaSuccess) return e;
        spans.push_back({ phase, { open_ev, b } });
        open_ev = nullptr;
        return cudaEventRecord(b, st);
    }
};
thread_local float g_trick_ms[4] = { 0, 0, 0, 0 };

// the state of one decode batch, for the K1b hook: after picture index p, gather the frames of the selected pictures with that index
struct TrickGather {
    ef_ctx* c;
    const std::vector<uint32_t>* first;          // [p]: first entry of picture index p in the lists
    const uint32_t* d_streams;
    const uint32_t* d_slots;
    uint8_t* d_in;
    TrickTimer* timer;
};

int trick_gather(void* arg, int p, cudaStream_t st)
{
    TrickGather& g = *(TrickGather*)arg;
    const std::vector<uint32_t>& f = *g.first;
    const int count = (int)(f[p + 1] - f[p]);
    if (!count) return EF_OK;
    CK(g.timer->end(0, st));
    CK(g.timer->begin(st));
    CK(ef_trick_launch_gather(g.c->h.frames, g.d_streams + f[p], g.d_slots + f[p], count, (p + 1) & 1, g.d_in, st));
    g.c->launches++;
    CK(g.timer->end(1, st));
    CK(g.timer->begin(st));
    return EF_OK;
}

}  // namespace

extern "C" {

int ef_trick_build(int device, const uint8_t* ts, const uint64_t* off, int n_files, int qscale, uint8_t* fwd, uint64_t fwd_cap, uint64_t* fwd_off,
                   uint8_t* rwd, uint64_t rwd_cap, uint64_t* rwd_off)
{
    if (!off || n_files < 1 || !fwd_off || !rwd_off) return fail(EF_EINVAL, "null argument");
    if (qscale < 1 || qscale > 31) return fail(EF_EINVAL, "qscale %d outside 1..31", qscale);
    for (int f = 0; f <= n_files; f++)
        if (off[f] % 188 || (f && off[f] < off[f - 1])) return fail(EF_EINVAL, "offsets must be non-decreasing multiples of 188");
    if (off[n_files] > off[0] && !ts) return fail(EF_EINVAL, "null argument");
    TRY(usable_device(device));
    DeviceScope scope_(device);
    const uint8_t* base = ts + off[0];
    std::vector<uint64_t> poff((size_t)n_files + 1);
    for (int f = 0; f <= n_files; f++) poff[f] = (off[f] - off[0]) / 188;
    const uint64_t n_packets = poff[n_files];

    // sequence headers: make_index()'s table (ef_tsidx_scan); cut before each one that starts a PES with a PTS and whose first two
    // pictures are whole (trick_pictures_whole), so that the segment decoded from reset frame stores gives a continuous decode's frames
    std::vector<ef_tsidx_info> info((size_t)n_files);
    std::vector<int64_t> spts(n_packets + 1);
    std::vector<uint32_t> spos(n_packets + 1);
    std::vector<uint64_t> soff(poff.begin(), poff.end());
    for (auto& o : soff) o *= 188;
    for (int f = 0; f < n_files; f++) if (poff[f + 1] == poff[f]) return fail(EF_EINVAL, "main %d is empty: it has no sequence header", f);
    TRY(ef_tsidx_scan(device, base, soff.data(), n_files, 7500, info.data(), spts.data(), spos.data()));
    std::vector<TrickSeg> segs;
    std::vector<std::vector<uint8_t>> headers((size_t)n_files);
    std::vector<uint8_t> es;
    for (int f = 0; f < n_files; f++) {
        if (!info[f].n_seq) return fail(EF_EINVAL, "main %d has no sequence header", f);
        bool ok;
        es.clear();
        trick_video_es(base, poff[f] + spos[poff[f]], poff[f + 1], 16, es, &ok);
        int i = 0;
        while (i + 8 <= (int)es.size() && !(es[i] == 0 && es[i + 1] == 0 && es[i + 2] == 1 && es[i + 3] == 0xB3)) i++;
        if (i + 8 > (int)es.size()) return fail(EF_EINVAL, "main %d: its first sequence header is cut short", f);
        headers[f] = trick_header(es[i + 7] >> 4, es[i + 7] & 15);
    }
    std::vector<std::pair<uint64_t, uint64_t>> cand;                    // (packet, end of its main) of every later sequence header
    for (int f = 0; f < n_files; f++)
        for (uint32_t k = 1; k < info[f].n_seq; k++) cand.push_back({ poff[f] + spos[poff[f] + k], poff[f + 1] });
    std::vector<uint8_t> cut(cand.size(), 0);
    {   // each check walks two pictures' macroblocks: spread them over the host's cores
        std::atomic<size_t> next_cand{ 0 };
        auto work = [&]() { for (size_t c; (c = next_cand++) < cand.size();) cut[c] = trick_cut_ok(base, cand[c].first, cand[c].second) == 1; };
        std::vector<std::thread> pool;
        const unsigned nt = std::min<size_t>(std::max(1u, std::thread::hardware_concurrency()), std::min<size_t>(cand.size() / 64 + 1, 32));
        for (unsigned t = 1; t < nt; t++) pool.emplace_back(work);
        work();
        for (std::thread& t : pool) t.join();
    }
    for (int f = 0, c = 0; f < n_files; f++) {
        segs.push_back({ f, poff[f], poff[f + 1] });
        for (uint32_t k = 1; k < info[f].n_seq; k++, c++) {
            const uint64_t p = cand[c].first;
            if (p <= segs.back().pkt0 || !cut[c]) continue;                // joins the segment before it
            segs.back().pkt1 = p;
            segs.push_back({ f, p, poff[f + 1] });
        }
    }

    // batches of segments
    std::vector<size_t> chunk = { 0 };
    for (size_t s = 0; s < segs.size(); s++) {
        const size_t c0 = chunk.back();
        if (s > c0 && (s - c0 >= (size_t)kTrickChunkStreams || (segs[s].pkt1 - segs[c0].pkt0) * 188 > kTrickChunkBytes)) chunk.push_back(s);
    }
    chunk.push_back(segs.size());
    int max_streams = 1;
    uint64_t max_bytes = 188, max_pusi = 1;
    for (size_t c = 0; c + 1 < chunk.size(); c++) {
        max_streams = std::max(max_streams, (int)(chunk[c + 1] - chunk[c]));
        max_bytes = std::max(max_bytes, (segs[chunk[c + 1] - 1].pkt1 - segs[chunk[c]].pkt0) * 188);
    }
    for (const TrickSeg& s : segs) {                 // a first guess of the pictures per segment: its video PES starts
        uint64_t n = 1;
        for (uint64_t k = s.pkt0; k < s.pkt1; k++) {
            const uint8_t* d = base + k * 188;
            n += (d[1] & 0x40) && (((d[1] << 8) | d[2]) & 0x1FFF) == 0x100;
        }
        max_pusi = std::max(max_pusi, n);
    }

    CK(ef_trick_upload_tables());
    cudaStream_t st = 0;
    TrickTimer timer;
    GrowBuf d_ts, d_off, d_list, d_in, d_slots, d_len, d_es, d_dst, d_hdr;
    CK(d_ts.reserve(n_packets * 188 + 16));
    CK(cudaMemcpy(d_ts.p, base, n_packets * 188, cudaMemcpyHostToDevice));
    CK(d_off.reserve(((size_t)max_streams + 1) * 8));
    int max_pictures = (int)std::min<uint64_t>(max_pusi, 4096);
    ef_ctx* ctx = nullptr;
    struct CtxGuard { ef_ctx** c; ~CtxGuard() { if (*c) ef_destroy(*c); } } ctx_guard{ &ctx };

    // every encoded picture: its file, its main pts, where its bytes are in d_es
    struct Enc { int file; int64_t main_pts; uint64_t es_off; uint32_t es_len; };
    std::vector<Enc> enc;
    std::vector<std::vector<uint32_t>> fwd_of((size_t)n_files);   // encoded picture ids of every file's fwd pictures, in order
    std::vector<uint64_t> seen((size_t)n_files, 0);                 // main pictures of every file so far
    std::vector<int64_t> p0((size_t)n_files, -1);
    uint64_t es_total = 0;
    size_t pending = 0;                                             // gathered, not yet encoded: enc[enc.size() - pending ..)
    size_t in_cap = 0;

    auto encode_pending = [&]() -> int {
        if (!pending) return EF_OK;
        const int n = (int)pending;
        const size_t e0 = enc.size() - pending;
        CK(d_slots.reserve((size_t)n * EF_MBH_MAX * kTrickSliceBytes));
        CK(d_len.reserve((size_t)n * EF_MBH_MAX * 4));
        CK(timer.begin(st));
        CK(ef_trick_launch_encode(d_in.p, n, qscale, (uint32_t*)d_slots.p, (uint32_t*)d_len.p, st));
        std::vector<uint32_t> len((size_t)n * EF_MBH_MAX);
        CK(cudaMemcpyAsync(len.data(), d_len.p, len.size() * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        std::vector<uint64_t> dst((size_t)n);
        std::vector<uint8_t> hdr((size_t)n * kTrickHeaderBytes);
        const uint64_t es0 = es_total;
        for (int p = 0; p < n; p++) {
            uint32_t bytes = kTrickHeaderBytes;
            for (int s = 0; s < EF_MBH_MAX; s++) bytes += len[(size_t)p * EF_MBH_MAX + s];
            Enc& e = enc[e0 + p];
            e.es_off = dst[p] = es_total; e.es_len = bytes;
            es_total += bytes;
            memcpy(&hdr[(size_t)p * kTrickHeaderBytes], headers[e.file].data(), kTrickHeaderBytes);
        }
        if (es_total + 16 > d_es.cap) CK(d_es.reserve(std::max<size_t>(es_total + 16, d_es.cap * 2), es0));   // grows geometrically
        CK(d_dst.reserve(dst.size() * 8)); CK(d_hdr.reserve(hdr.size()));
        CK(cudaMemcpyAsync(d_dst.p, dst.data(), dst.size() * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_hdr.p, hdr.data(), hdr.size(), cudaMemcpyHostToDevice, st));
        CK(ef_trick_launch_assemble((const uint32_t*)d_slots.p, (const uint32_t*)d_len.p, (const uint64_t*)d_dst.p, d_hdr.p, n, d_es.p, st));
        CK(timer.end(2, st));
        CK(cudaStreamSynchronize(st));                    // the host buffers above go out of scope
        pending = 0;
        return EF_OK;
    };

    for (size_t c = 0; c + 1 < chunk.size(); c++) {
        const size_t s0 = chunk[c], ns = chunk[c + 1] - s0;
        std::vector<uint32_t> npics(ns);
        std::vector<int64_t> pts;
        for (;;) {                                        // (re)create the decode context until a batch's pictures fit it
            if (!ctx) {
                ef_config cfg = { device, max_streams, max_pictures, 16, (size_t)max_bytes, 0 };
                TRY(ef_create(&ctx, &cfg));
                TRY(ef_pts_enable(ctx));
            } else TRY(ef_reset(ctx));
            std::vector<uint64_t> so((size_t)max_streams + 1);
            for (int s = 0; s <= max_streams; s++) so[s] = ((s < (int)ns ? segs[s0 + s].pkt0 : segs[s0 + ns - 1].pkt1) - segs[s0].pkt0) * 188;
            CK(cudaMemcpy(d_off.p, so.data(), so.size() * 8, cudaMemcpyHostToDevice));
            CK(timer.begin(st));
            TRY(ef_submit_ts_device(ctx, d_ts.p + segs[s0].pkt0 * 188, (const uint64_t*)d_off.p, st));
            TRY(ef_index(ctx, st));
            const int rc = ef_index_info(ctx, nullptr, nullptr, nullptr, nullptr);
            CK(timer.end(0, st));
            if (rc == EF_ENOMEM && max_pictures < 4096) {
                max_pictures = std::min(4096, max_pictures * 2);
                ef_destroy(ctx); ctx = nullptr;
                continue;
            }
            if (rc == EF_ENOMEM)                          // EF_ENOMEM stays the output-capacity answer
                return fail(EF_EINVAL, "a main holds more than 4,096 pictures between two sequence headers that start a segment, or "
                                       "pictures of more than 16 slices: outside what ef_trick_build decodes");
            TRY(rc);
            break;
        }
        CK(cudaMemcpy(npics.data(), ctx->h.n_pics, ns * 4, cudaMemcpyDeviceToHost));
        pts.resize((size_t)max_streams * max_pictures);
        CK(cudaMemcpy(pts.data(), ctx->d_pic_pts, pts.size() * 8, cudaMemcpyDeviceToHost));
        // the selected pictures of the batch, listed by picture index
        int maxp = 0;
        for (size_t s = 0; s < ns; s++) maxp = std::max(maxp, (int)npics[s]);
        std::vector<std::vector<std::pair<uint32_t, uint32_t>>> by_p((size_t)maxp);    // (stream, index in the batch's selection)
        std::vector<Enc> sel;
        for (size_t s = 0; s < ns; s++) {
            const int f = segs[s0 + s].file;
            for (uint32_t p = 0; p < npics[s]; p++, seen[f]++) {
                const int64_t v = pts[s * max_pictures + p];
                if (seen[f] == 0) p0[f] = v;
                if (seen[f] % kTrickSpeed) continue;
                by_p[p].push_back({ (uint32_t)s, (uint32_t)sel.size() });
                sel.push_back({ f, v, 0, 0 });
            }
        }
        if (pending + sel.size() > in_cap) {             // room for the batch's frames: encode what is waiting, grow if still short
            TRY(encode_pending());
            if (sel.size() > in_cap) { in_cap = std::max(sel.size(), (size_t)kTrickEncodeBatch); CK(d_in.reserve(in_cap * EF_FRAME)); }
        }
        for (auto& v : by_p) for (auto& e : v) e.second += (uint32_t)pending;
        for (const Enc& e : sel) { fwd_of[e.file].push_back((uint32_t)enc.size()); enc.push_back(e); }
        std::vector<uint32_t> first((size_t)maxp + 1, 0), lst_s, lst_slot;
        for (int p = 0; p < maxp; p++) {
            first[p + 1] = first[p] + (uint32_t)by_p[p].size();
            for (auto& e : by_p[p]) { lst_s.push_back(e.first); lst_slot.push_back(e.second); }
        }
        CK(d_list.reserve(std::max<size_t>(lst_s.size(), 1) * 8));
        if (!lst_s.empty()) {
            CK(cudaMemcpy(d_list.p, lst_s.data(), lst_s.size() * 4, cudaMemcpyHostToDevice));
            CK(cudaMemcpy(d_list.p + lst_s.size() * 4, lst_slot.data(), lst_slot.size() * 4, cudaMemcpyHostToDevice));
        }
        TrickGather g = { ctx, &first, (const uint32_t*)d_list.p, (const uint32_t*)(d_list.p + lst_s.size() * 4), d_in.p, &timer };
        CK(timer.begin(st));
        for (int p = 0; p < maxp && !sel.empty(); p += ctx->h.rec_pics)
            TRY(decode_range(ctx, p, std::min(ctx->h.rec_pics, maxp - p), st, nullptr, 0, trick_gather, &g));
        CK(timer.end(0, st));
        pending += sel.size();
        if (pending >= (size_t)kTrickEncodeBatch) TRY(encode_pending());
        else CK(cudaStreamSynchronize(st));
    }
    TRY(encode_pending());

    // the plan of both outputs: every file's fwd pictures, then every file's rwd pictures
    std::vector<EfTrickPic> plan;
    uint64_t pk = 0;
    for (int dir = 0; dir < 2; dir++) {
        uint64_t* o = dir ? rwd_off : fwd_off;
        o[0] = 0;
        for (int f = 0; f < n_files; f++) {
            const std::vector<uint32_t>& ids = fwd_of[f];
            const size_t n = ids.size();
            std::vector<int64_t> fp(n);
            for (size_t k = 0; k < n; k++) fp[k] = p0[f] + (enc[ids[k]].main_pts - p0[f]) / kTrickSpeed;
            uint32_t cc = 0;
            for (size_t k = 0; k < n; k++) {
                const size_t src = dir ? n - 1 - k : k;
                const Enc& e = enc[ids[src]];
                const int64_t t = dir ? fp[0] + (fp[n - 1] - fp[n - 1 - k]) : fp[k];
                plan.push_back({ e.es_off, pk, t, e.es_len, cc });
                const uint32_t pkts = (14 + e.es_len + 183) / 184;
                pk += pkts; cc += pkts;
            }
            o[f + 1] = o[f] + (uint64_t)cc * 188;
        }
    }
    const uint64_t fwd_need = fwd_off[n_files], rwd_need = rwd_off[n_files];
    if (fwd_cap < fwd_need || rwd_cap < rwd_need || (fwd_need && !fwd) || (rwd_need && !rwd))
        return fail(EF_ENOMEM, "the trick files need %llu (fwd) and %llu (rwd) bytes", (unsigned long long)fwd_need, (unsigned long long)rwd_need);
    GrowBuf d_plan, d_out;
    CK(d_plan.reserve(std::max<size_t>(plan.size(), 1) * sizeof(EfTrickPic)));
    CK(d_out.reserve(pk * 188 + 16));
    CK(cudaMemcpy(d_plan.p, plan.data(), plan.size() * sizeof(EfTrickPic), cudaMemcpyHostToDevice));
    CK(timer.begin(st));
    CK(ef_trick_launch_mux(d_es.p, (const EfTrickPic*)d_plan.p, (int)plan.size(), pk, d_out.p, st));
    CK(timer.end(3, st));
    if (fwd_need) CK(cudaMemcpy(fwd, d_out.p, fwd_need, cudaMemcpyDeviceToHost));
    if (rwd_need) CK(cudaMemcpy(rwd, d_out.p + fwd_need, rwd_need, cudaMemcpyDeviceToHost));
    CK(cudaDeviceSynchronize());
    for (float& m : g_trick_ms) m = 0;
    for (auto& s : timer.spans) {
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, s.second.first, s.second.second));
        g_trick_ms[s.first] += ms;
    }
    return EF_OK;
}

// ef_library_add_trick: ef_trick_build on a title's main, then merge_index()'s fwd and rwd records and samples for the built files
int ef_library_add_trick(ef_ctx* c, int title, int qscale)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->d_lib) return fail(EF_ESTATE, "ef_library_add_trick before the first ef_library_add");
    if (title < 0 || title >= (int)c->lib_titles.size()) return fail(EF_EINVAL, "no title %d", title);
    if (qscale < 1 || qscale > 31) return fail(EF_EINVAL, "qscale %d outside 1..31", qscale);
    EfLibTitle t = c->lib_titles[title];
    if (t.ts[0] || t.ts[2]) return fail(EF_ESTATE, "title %d already has a trick file", title);
    CK(cudaDeviceSynchronize());
    // the plan reads the main's packets on the host (make_index()'s table, the segment cuts): one copy of the main back
    std::vector<uint8_t> main(t.bytes[1]), img(t.idx_bytes);
    CK(cudaMemcpy(main.data(), t.ts[1], main.size(), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(img.data(), t.idx, img.size(), cudaMemcpyDeviceToHost));
    const uint64_t moff[2] = { 0, main.size() };
    uint64_t fo[2], ro[2], cap = main.size() + 188 * 1024;
    std::vector<uint8_t> fwd, rwd;
    for (int attempt = 0;; attempt++) {
        fwd.resize(cap); rwd.resize(cap);
        const int rc = ef_trick_build(c->cfg.device, main.data(), moff, 1, qscale, fwd.data(), cap, fo, rwd.data(), cap, ro);
        if (rc == EF_ENOMEM && attempt == 0 && std::max(fo[1], ro[1]) > cap) { cap = std::max(fo[1], ro[1]); continue; }
        TRY(rc);
        break;
    }
    fwd.resize(fo[1]); rwd.resize(ro[1]);
    // merge_index() (indexer.cpp:230) for the two built files: records of bin IDX_BIN and trick speed 15, pts2seq()'s samples
    const uint32_t bin = 90000 / 12;
    std::vector<uint8_t> both(fwd);
    both.insert(both.end(), rwd.begin(), rwd.end());
    const uint64_t off2[3] = { 0, fwd.size(), both.size() };
    const size_t np = both.size() / 188 + 1;
    std::vector<int64_t> spts(np);
    std::vector<uint32_t> spos(np);
    ef_tsidx_info info[2];
    TRY(ef_tsidx_scan(c->cfg.device, both.data(), off2, 2, bin, info, spts.data(), spos.data()));
    idx_hdr h;
    memcpy(&h, img.data(), sizeof(h));
    std::vector<uint32_t> smp[2];
    idx_rec* rec[2] = { &h.fwd, &h.rev };
    for (int k = 0; k < 2; k++) {
        const size_t p0 = off2[k] / 188;
        smp[k].resize(std::max<uint32_t>(info[k].n_samples, 1));
        uint32_t n = 0;
        TRY(ef_tsidx_samples(c->cfg.device, spts.data() + p0, spos.data() + p0, (int)info[k].n_seq, info[k].first_pts, info[k].last_pts, bin,
                             smp[k].data(), (uint32_t)smp[k].size(), &n));
        smp[k].resize(n);
        *rec[k] = idx_rec{ info[k].first_pts, info[k].last_pts, bin, 15, n };
        if (!n || info[k].last_pts == info[k].first_pts)
            return fail(EF_EINVAL, "title %d: its %s file has one picture (pts %lld): the reference divides by zero playing it", title,
                        k ? "rwd" : "fwd", (long long)info[k].first_pts);
    }
    std::vector<uint8_t> out(sizeof(idx_hdr) + 4 * ((size_t)h.video.sample_count + smp[0].size() + smp[1].size()));
    memcpy(out.data(), img.data(), sizeof(idx_hdr));                          // the padding bytes stay as added
    for (int k = 0; k < 2; k++) memcpy(out.data() + 8 + 32 * (k + 1), rec[k], 28);
    memcpy(out.data() + sizeof(idx_hdr), img.data() + sizeof(idx_hdr), 4 * (size_t)h.video.sample_count);   // the main's samples as added
    memcpy(out.data() + sizeof(idx_hdr) + 4 * (size_t)h.video.sample_count, smp[0].data(), 4 * smp[0].size());
    memcpy(out.data() + sizeof(idx_hdr) + 4 * ((size_t)h.video.sample_count + smp[0].size()), smp[1].data(), 4 * smp[1].size());
    if (out.size() >> 32 || fwd.size() >> 32) return fail(EF_EINVAL, "title %d: its trick files or video.idx reach 4 GiB", title);
    uint8_t* p = nullptr;
    TRY(dev_alloc(c, &p, out.size()));
    CK(cudaMemcpy(p, out.data(), out.size(), cudaMemcpyHostToDevice));
    t.idx = p; t.idx_bytes = (uint32_t)out.size();
    const std::vector<uint8_t>* files[3] = { &rwd, nullptr, &fwd };
    for (int f = 0; f < 3; f += 2) {
        TRY(dev_alloc(c, &p, files[f]->size()));
        CK(cudaMemcpy(p, files[f]->data(), files[f]->size(), cudaMemcpyHostToDevice));
        t.ts[f] = p; t.bytes[f] = (uint32_t)files[f]->size();
    }
    t.f_first = h.fwd.first_pts; t.f_last = h.fwd.last_pts; t.r_first = h.rev.first_pts; t.r_last = h.rev.last_pts;
    t.f_bin = t.r_bin = bin; t.f_trick = t.r_trick = 15; t.f_n = h.fwd.sample_count; t.r_n = h.rev.sample_count;
    CK(cudaMemcpy(c->d_lib_titles + title, &t, sizeof(t), cudaMemcpyHostToDevice));
    c->lib_titles[title] = t;
    return EF_OK;
}

int ef_library_read(ef_ctx* c, int title, int what, uint8_t* dst, uint64_t cap, uint64_t* bytes)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !bytes) return fail(EF_EINVAL, "null argument");
    if (!c->d_lib) return fail(EF_ESTATE, "ef_library_read before the first ef_library_add");
    if (title < 0 || title >= (int)c->lib_titles.size() || what < -1 || what > 2) return fail(EF_EINVAL, "no title %d or part %d", title, what);
    const EfLibTitle& t = c->lib_titles[title];
    const uint8_t* src = what < 0 ? t.idx : t.ts[what];
    *bytes = what < 0 ? t.idx_bytes : t.bytes[what];
    if (!*bytes) return EF_OK;
    if (!dst || cap < *bytes) return fail(EF_ENOMEM, "part %d of title %d has %llu bytes", what, title, (unsigned long long)*bytes);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(dst, src, *bytes, cudaMemcpyDeviceToHost));
    return EF_OK;
}

int ef_trick_stage_ms(float* decode_ms, float* gather_ms, float* encode_ms, float* mux_ms)
{
    if (decode_ms) *decode_ms = g_trick_ms[0];
    if (gather_ms) *gather_ms = g_trick_ms[1];
    if (encode_ms) *encode_ms = g_trick_ms[2];
    if (mux_ms) *mux_ms = g_trick_ms[3];
    return EF_OK;
}

}  // extern "C"
