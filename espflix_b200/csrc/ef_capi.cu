// espflix_b200/csrc/ef_capi.cu — the C-ABI of libespflix_b200.so (include/espflix_b200.h).
// Context management, submits, launches and read-back. No CPU fallback: every path goes through
// the CUDA kernels in ef_index.cu / ef_decode.cu / ef_composite.cu or fails with EF_ECUDA.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../../include/espflix_b200.h"
#include "ef_common.cuh"
#include <stdlib.h>

// from the other translation units
int ef_build_tables(EfTables* t);
void ef_build_color_tab(uint32_t* tab768, int ntsc);
void ef_build_pal_burst(int16_t* b0, int16_t* b1, int width);
cudaError_t ef_index_upload_constants();
const unsigned char* ef_default_intra_ptr();
__global__ void ef_scan_kernel(EfDev* Dp);
__global__ void ef_prefix_kernel(EfDev* Dp);
__global__ void ef_fill_kernel(EfDev* Dp);
__global__ void ef_ts_len_kernel(const uint8_t* ts, uint64_t n_packets, uint32_t* out_len);
__global__ void ef_ts_copy_kernel(const uint8_t* ts, uint64_t n_packets, const uint32_t* local_off, const uint16_t* pkt_stream, const uint64_t* es_off, uint8_t* es);
__global__ void ef_ts_scan_kernel(const uint32_t* len, const uint64_t* ts_off, uint32_t* local_off, uint16_t* pkt_stream, uint64_t* stream_total);
__global__ void ef_ts_offsets_kernel(const uint64_t* stream_total, int n_streams, uint64_t* es_off, uint8_t* es);
__global__ void ef_pts_packet_kernel(const uint8_t* ts, const uint64_t* ts_off, const uint32_t* local_off, uint32_t* list_off, int64_t* list_pts, uint2* span);
__global__ void ef_pts_resolve_kernel(const EfDev* Dp, const uint2* span, const uint32_t* list_off, const int64_t* list_pts, int64_t* carry, int64_t* last,
                                      int64_t* pic_pts);
size_t ef_recon_smem_bytes();
cudaError_t ef_decode_configure();
int ef_decode_resident_ctas(int which);
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
__global__ void ef_audio_commit_kernel(EfAudioState* st, const uint8_t* blob, const uint64_t* blob_off, const int4* plan, const uint64_t* slot_base, const int32_t* vrows,
                                       const int32_t* sb_last, const uint8_t* ended, int n_streams);
__global__ void ef_audio_ts_packet_kernel(const uint8_t* ts, uint64_t n_packets, uint8_t* start, uint8_t* kind);
__global__ void ef_audio_ts_scan_kernel(const uint64_t* ts_off, int n_files, const uint8_t* start, const uint8_t* kind, const uint8_t* gate_in, uint8_t* gate_out,
                                        uint32_t* lead, uint8_t* skip, uint32_t* out_pos, uint64_t* es_len);
__global__ void ef_audio_ts_copy_kernel(const uint8_t* ts, const uint64_t* ts_off, int n_files, uint64_t n_packets, const uint8_t* start, const uint32_t* out_pos, const uint64_t* es_off, uint8_t* es);
__global__ void ef_audio_end_kernel(const uint8_t* ended, int n_streams, uint8_t* gate_cur, uint8_t* gate_next, uint8_t* skip_next, int next_is_ts);
cudaError_t ef_audio_upload_constants();
cudaError_t ef_launch_parse(const EfDev& dev, int pic0, int n_pics, int sm_count, size_t max_slices, cudaStream_t stream);
cudaError_t ef_launch_recon(const EfDev& dev, int pic_rel, int sm_count, size_t n_slots, cudaStream_t stream);
cudaError_t ef_launch_composite(const EfDev* dev, int n_streams, const EfGeometry& g, int fb, int frame_counter, const EfPresent& pr, cudaStream_t stream);
cudaError_t ef_launch_blit(const EfDev* dev, int stream_index, int fb, int line, int x, int width, int frame_counter, uint16_t* dst, cudaStream_t stream);

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

__global__ void ef_reset_seq_kernel(EfDev* Dp, const uint8_t* default_intra)
{
    EfDev& D = *Dp;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= D.n_streams) return;
    EfSeq* q = D.seq + (size_t)s * (D.max_seq + 1);
    for (int n = 0; n < 128; n++) q->qz[n] = D.tables->qz[n];
    (void)default_intra;
    q->mb_width = 22; q->mb_height = 12; q->valid = 1; q->custom = 0; q->fp_rs = 0;
    D.n_pics[s] = 0; D.base_pics[s] = 0; D.n_seq[s] = 0;
}

}  // namespace

struct ef_ctx {
    ef_config cfg;
    int sm_count = 0;
    EfDev h;                   // host copy of the device context
    EfDev* d = nullptr;           // = dd[active]
    std::vector<void*> allocs;
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
    uint8_t* d_stage = nullptr;      // read-back staging (I420 / strips)
    size_t stage_bytes = 0;
    uint8_t* d_default_intra = nullptr;
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
    struct AudioScratch* aud_scratch = nullptr;
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
};

// Device buffers of the audio decode whose size follows the frames of one call, grown on demand. The stateless calls
// use a scratch of their own, a context keeps one.
struct AudioScratch {
    enum { PLAN, SB_LAST, SLOT, POFF, VROWS, PCM, PDM, N };
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

int ensure_stage(ef_ctx* c, size_t bytes)
{
    if (c->stage_bytes >= bytes) return EF_OK;
    void* v = nullptr;
    CK(cudaMalloc(&v, bytes));
    c->allocs.push_back(v);
    c->d_stage = (uint8_t*)v; c->stage_bytes = bytes;
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
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || cfg->device < 0 || ndev <= cfg->device)
        return fail(EF_ECUDA, "no usable CUDA device %d (%s); this library has no CPU path", cfg->device, cudaGetErrorString(e));
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
    int rc;
#define A(ptr, count) if ((rc = dev_alloc(c, &(ptr), (count))) != EF_OK) return rc;
    for (int b = 0; b < 2; b++) {
        A(c->d_es2[b], cfg->es_capacity + 1024);
        A(c->d_es_off2[b], (size_t)n + 1);
        A(c->dd[b], 1);
        CK(cudaHostAlloc((void**)&c->h_off[b], ((size_t)n + 1) * 8, cudaHostAllocDefault));
        CK(cudaEventCreateWithFlags(&c->ev_up_done[b], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->ev_buf_free[b], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->ev_down_done[b], cudaEventDisableTiming));
    }
    CK(cudaEventCreateWithFlags(&c->ev_user, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&c->ev_export, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&c->ev_frames_read, cudaEventDisableTiming));
    CK(cudaStreamCreateWithFlags(&c->up_stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->down_stream, cudaStreamNonBlocking));
    A(h.frames, (size_t)n * 2 * EF_FRAME + 1024);
    A(h.seq, (size_t)n * (h.max_seq + 1));
    A(h.pics, (size_t)n * h.max_pictures);
    A(h.slice_off, (size_t)n * h.max_slices);
    A(h.slice_code, (size_t)n * h.max_slices);
    A(h.n_pics, n); A(h.base_pics, n); A(h.n_seq, n);
    A(h.pic_pref, (size_t)n * h.max_pictures);
    A(h.pic_total, h.max_pictures); A(h.pic_base, h.max_pictures); A(h.cursor, h.max_pictures);
    h.work_capacity = (size_t)n * h.max_slices;
    A(h.work, h.work_capacity);
    A(h.info, 8);
    EfTables* dt; A(dt, 1);
    {   // macroblock records: as many picture indices per K1a launch as fit in 2 GiB
        const size_t per_pic = (size_t)n * EF_MBW_MAX * EF_MBH_MAX * (sizeof(EfMbRec) + 4);
        size_t k = ((size_t)2 << 30) / per_pic;
        if (const char* e = getenv("EF_REC_PICS")) { const long v = atol(e); if (v >= 1) k = (size_t)v; }   // tuning / test knob
        h.rec_pics = (int)(k < 1 ? 1 : k > (size_t)h.max_pictures ? (size_t)h.max_pictures : k);
        const size_t slots = (size_t)h.rec_pics * n * EF_MBW_MAX * EF_MBH_MAX;
        A(h.mb_info, slots); A(h.mb_rec, slots);
        A(h.parse_cursor, (size_t)h.rec_pics + 4);      // [0] K1a, [1..] one per K1b launch
        h.recon_cursor = h.parse_cursor + 1;
        A(h.coef, 3 * (cfg->es_capacity + 1024) + 1024);
    }
    A(c->d_color_tab, 768); A(c->d_pal_burst, 128); A(c->d_default_intra, 64); A(c->d_overlay, 1280);
    c->present.bitmap = c->d_overlay;
    if (cfg->fields) { h.field_stride = EF_PAL_FIELD_SAMPLES; A(h.fields, (size_t)n * h.field_stride); }
#undef A
    h.es = c->d_es2[0]; h.es_off = c->d_es_off2[0]; h.tables = dt;
    c->d = c->dd[0];
    h.color_tab = c->d_color_tab; h.pal_burst = c->d_pal_burst;

    EfTables t;
    const int bad = ef_build_tables(&t);
    if (bad) return fail(EF_EINVAL, "internal: VLC table %d does not fit its lookup shape", bad);
    CK(cudaMemcpy(dt, &t, sizeof(t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_default_intra, ef_default_intra_ptr(), 64, cudaMemcpyHostToDevice));
    for (int b = 0; b < 2; b++) {
        CK(cudaMemset(c->d_es2[b], 0, cfg->es_capacity + 1024));
        CK(cudaMemset(c->d_es_off2[b], 0, ((size_t)n + 1) * 8));
    }
    CK(cudaMemset(c->d_overlay, 0, 1280));
    { int rcp = push_dev(c); if (rcp != EF_OK) return rcp; }
    rc = ef_reset(c);
    if (rc != EF_OK) return rc;
    rc = ef_video_init(c, 1);
    if (rc != EF_OK) return rc;
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
    delete c->aud_scratch;
    if (c->h_ended) cudaFreeHost(c->h_ended);
    for (int b = 0; b < 2; b++) {
        if (c->h_off[b]) cudaFreeHost(c->h_off[b]);
        if (c->ev_up_done[b]) cudaEventDestroy(c->ev_up_done[b]);
        if (c->ev_buf_free[b]) cudaEventDestroy(c->ev_buf_free[b]);
        if (c->ev_down_done[b]) cudaEventDestroy(c->ev_down_done[b]);
    }
    for (int i = 0; i < 5; i++) if (c->ev_prof[i]) cudaEventDestroy(c->ev_prof[i]);
    if (c->ev_user) cudaEventDestroy(c->ev_user);
    if (c->ev_export) cudaEventDestroy(c->ev_export);
    if (c->ev_frames_read) cudaEventDestroy(c->ev_frames_read);
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

int ef_reset(ef_ctx* c)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    { int rcw = wait_frames_read(c); if (rcw != EF_OK) return rcw; }
    CK(cudaMemset(c->h.frames, 0, (size_t)c->cfg.n_streams * 2 * EF_FRAME + 1024));     // Frame::init zero-fills (player.cpp:25)
    ef_reset_seq_kernel<<<(c->cfg.n_streams + 127) / 128, 128>>>(c->d, c->d_default_intra);
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
    CK(cudaDeviceSynchronize());
    c->indexed = false; c->submitted = false; c->pending = -1;
    return EF_OK;
}

// Uploads go to the BACK elementary-stream buffer on the context's own upload stream, so that a
// caller that has pinned its input can submit batch k+1 while the kernels of batch k still run
// (the producer side of the reference's Buffer queue is asynchronous in the same way). ef_index()
// makes the compute stream wait for the upload and flips the buffers.
static int submit_common(ef_ctx* c, const uint8_t* src, const uint64_t* off, bool host, bool ts, cudaStream_t st)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !src || !off) return fail(EF_EINVAL, "null argument");
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
    uint8_t* d_es = c->d_es2[b];
    uint64_t* d_es_off = c->d_es_off2[b];
    if (!ts) {
        CK(cudaMemcpyAsync(d_es, src, total, kind, up));
        CK(cudaMemsetAsync(d_es + total, 0, 256, up));
        CK(cudaMemcpyAsync(d_es_off, hoff, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, up));
    } else {
        const uint64_t n_packets = total / 188;
        if (!c->d_ts) {
            int rc;
            if ((rc = dev_alloc(c, &c->d_ts, c->cfg.es_capacity + 64)) != EF_OK) return rc;
            if ((rc = dev_alloc(c, &c->d_pkt_len, c->cfg.es_capacity / 188 + 1)) != EF_OK) return rc;
            if ((rc = dev_alloc(c, &c->d_pkt_off, c->cfg.es_capacity / 188 + 1)) != EF_OK) return rc;
            if ((rc = dev_alloc(c, &c->d_pkt_stream, c->cfg.es_capacity / 188 + 1)) != EF_OK) return rc;
            if ((rc = dev_alloc(c, &c->d_stream_total, (size_t)n + 1)) != EF_OK) return rc;
            if ((rc = dev_alloc(c, &c->d_ts_off, (size_t)n + 1)) != EF_OK) return rc;
        }
        CK(cudaMemcpyAsync(c->d_ts, src, total, kind, up));
        CK(cudaMemcpyAsync(c->d_ts_off, hoff, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, up));
        if (n_packets) {
            ef_ts_len_kernel<<<(unsigned)((n_packets + 255) / 256), 256, 0, up>>>(c->d_ts, n_packets, c->d_pkt_len);
            CK(cudaGetLastError());
            ef_ts_scan_kernel<<<n, 256, 0, up>>>(c->d_pkt_len, c->d_ts_off, c->d_pkt_off, c->d_pkt_stream, c->d_stream_total);
            CK(cudaGetLastError());
            ef_ts_offsets_kernel<<<1, 1024, 0, up>>>(c->d_stream_total, n, d_es_off, d_es);
            CK(cudaGetLastError());
            ef_ts_copy_kernel<<<(unsigned)((n_packets * 32 + 255) / 256), 256, 0, up>>>(c->d_ts, n_packets, c->d_pkt_off, c->d_pkt_stream, d_es_off, d_es);
            CK(cudaGetLastError());
            c->launches += 4;
        } else CK(cudaMemsetAsync(d_es_off, 0, ((size_t)n + 1) * 8, up));
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
    cudaStream_t st = (cudaStream_t)stream;
    const int n = c->cfg.n_streams;
    if (c->pending >= 0) {                       // a fresh submit: wait for its upload, make it the front buffer
        if (c->audio && c->aud_unconsumed)       // the audio of a TS submit is delivered exactly once
            return fail(EF_ESTATE, "ef_index of a new submit before ef_decode_audio consumed the current submit's audio");
        CK(cudaStreamWaitEvent(st, c->ev_up_done[c->pending], 0));
        c->active = c->pending; c->pending = -1;
        c->d = c->dd[c->active];
        c->aud_unconsumed = c->audio && c->aud_ts[c->active];
    }                                            // else: index the front buffer again (same input, next GOP period)
    if (c->profiling) { CK(cudaEventRecord(c->ev_prof[0], st)); c->prof_index = true; }
    CK(cudaMemsetAsync(c->h.info, 0, 32, st));
    ef_scan_kernel<<<(n * 32 + 127) / 128, 128, 0, st>>>(c->d);
    CK(cudaGetLastError());
    ef_prefix_kernel<<<c->h.max_pictures, 1024, 0, st>>>(c->d);
    CK(cudaGetLastError());
    const size_t threads = (size_t)n * c->h.max_pictures;
    ef_fill_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(c->d);
    CK(cudaGetLastError());
    c->launches += 3;
    if (c->profiling) CK(cudaEventRecord(c->ev_prof[1], st));
    if (c->pts) {
        const int a = c->active;
        ef_pts_resolve_kernel<<<(n * 32 + 127) / 128, 128, 0, st>>>(c->d, c->d_pts_span2[a], c->d_pts_off2[a], c->d_pts_val2[a], c->d_pts_carry, c->d_pts_last,
                                                                    c->d_pic_pts);
        CK(cudaGetLastError());
        c->launches++;
        c->pts_resolved = true;
    }
    CK(cudaEventRecord(c->ev_buf_free[c->active], st));
    c->indexed = true;
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
    if (info[3]) return fail(EF_ENOMEM, "index overflow (flags %u): raise max_pictures / max_slices_per_picture", info[3]);
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
    void* v = nullptr;
    CK(cudaMalloc(&v, bytes));
    c->allocs.push_back(v);
    c->d_stage2[k] = (uint8_t*)v; c->stage2_bytes[k] = bytes;
    return EF_OK;
}

// K1a over picture indices [p0, p0 + k), then K1b once per picture index. host_dst != nullptr: every picture index
// is exported (I420) straight after its K1b launch and copied to host_dst[p][stream] on the read-back stream while
// the next picture index is being rebuilt - what push_video() sees, picture by picture (video.h:49).
static int decode_range(ef_ctx* c, int p0, int k, cudaStream_t st, uint8_t* host_dst = nullptr, int layout = 0)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    const size_t slots = (size_t)k * c->cfg.n_streams * EF_MBW_MAX * EF_MBH_MAX;
    CK(cudaMemsetAsync(c->h.mb_info, 0, slots * 4, st));
    CK(cudaMemsetAsync(c->h.parse_cursor, 0, ((size_t)k + 1) * 4, st));
    if (c->profiling) { CK(cudaEventRecord(c->ev_prof[2], st)); c->prof_decode = true; }
    EfDev dev = c->h;                                       // K1 takes the context by value (kernel parameter space)
    dev.es = c->d_es2[c->active]; dev.es_off = c->d_es_off2[c->active];
    CK(ef_launch_parse(dev, p0, k, c->sm_count, (size_t)k * c->cfg.n_streams * c->cfg.max_slices_per_picture, st));
    if (c->profiling) CK(cudaEventRecord(c->ev_prof[3], st));
    const size_t batch_bytes = (size_t)c->cfg.n_streams * EF_FRAME;
    if (c->frames_read_pending) { CK(cudaStreamWaitEvent(st, c->ev_frames_read, 0)); c->frames_read_pending = false; }   // an asynchronous read-back still reads the frame stores
    for (int i = 0; i < k; i++) {
        CK(ef_launch_recon(dev, i, c->sm_count, (size_t)c->cfg.n_streams * EF_MBW_MAX * EF_MBH_MAX, st));
        if (host_dst) {
            const int b = c->stage_idx ^= 1;
            int rc = ensure_stage2(c, b, batch_bytes);
            if (rc != EF_OK) return rc;
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
    c->launches += 1 + (uint64_t)k;
    return EF_OK;
}

int ef_decode_picture(ef_ctx* c, int pic, void* stream)
{
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->indexed) return fail(EF_ESTATE, "ef_decode_picture before ef_index");
    if (pic < 0 || pic >= c->cfg.max_pictures) return fail(EF_EINVAL, "picture index %d out of range", pic);
    return decode_range(c, pic, 1, (cudaStream_t)stream);
}

int ef_decode_all(ef_ctx* c, int n_pictures, void* stream)
{
    if (!c) return fail(EF_EINVAL, "null context");
    if (!c->indexed) return fail(EF_ESTATE, "ef_decode_all before ef_index");
    if (n_pictures < 0 || n_pictures > c->cfg.max_pictures) return fail(EF_EINVAL, "n_pictures %d out of range", n_pictures);
    for (int p = 0; p < n_pictures; p += c->h.rec_pics) {
        const int k = n_pictures - p < c->h.rec_pics ? n_pictures - p : c->h.rec_pics;
        int rc = decode_range(c, p, k, (cudaStream_t)stream);
        if (rc != EF_OK) return rc;
    }
    return EF_OK;
}

int ef_decode_all_to_host(ef_ctx* c, int n_pictures, uint8_t* dst, int layout, void* stream)
{
    if (!c || !dst) return fail(EF_EINVAL, "null argument");
    if (layout != 0 && layout != 1) return fail(EF_EINVAL, "layout must be 0 (I420) or 1 (strips)");
    if (!c->indexed) return fail(EF_ESTATE, "ef_decode_all_to_host before ef_index");
    if (n_pictures < 0 || n_pictures > c->cfg.max_pictures) return fail(EF_EINVAL, "n_pictures %d out of range", n_pictures);
    for (int p = 0; p < n_pictures; p += c->h.rec_pics) {
        const int k = n_pictures - p < c->h.rec_pics ? n_pictures - p : c->h.rec_pics;
        int rc = decode_range(c, p, k, (cudaStream_t)stream, dst, layout);
        if (rc != EF_OK) return rc;
    }
    return EF_OK;
}

int ef_read_frame(ef_ctx* c, int stream_index, int fb, uint8_t* dst)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !dst) return fail(EF_EINVAL, "null argument");
    CK(cudaDeviceSynchronize());
    int f; int rc = resolve_fb(c, stream_index, fb, &f);
    if (rc != EF_OK) return rc;
    rc = ensure_stage(c, EF_FRAME);
    if (rc != EF_OK) return rc;
    ef_export_frames_kernel<<<(EF_FRAME / 8 + 255) / 256, 256>>>(c->h.frames, c->h.base_pics, c->h.n_pics, stream_index, 1, f, 1, c->d_stage);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaMemcpy(dst, c->d_stage, EF_FRAME, cudaMemcpyDeviceToHost));
    return EF_OK;
}

int ef_read_latest_i420_async(ef_ctx* c, int first, int count, uint8_t* dst, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !dst) return fail(EF_EINVAL, "null argument");
    if (first < 0 || count < 1 || first + count > c->cfg.n_streams) return fail(EF_EINVAL, "stream range out of bounds");
    const int k = c->stage_idx ^= 1;
    const size_t bytes = (size_t)count * EF_FRAME;
    { int rc = ensure_stage2(c, k, bytes); if (rc != EF_OK) return rc; }
    cudaStream_t st = (cudaStream_t)stream;
    // The tiled -> I420 export runs on the read-back stream, behind everything queued on the caller's stream so far and
    // behind the previous copy out of this staging buffer: it overlaps the index / parse kernels of the next submit. The
    // next reconstruction launch (the first thing that writes a frame store again) waits for ev_frames_read.
    if (!c->d_fb_snap[k]) { int rc = dev_alloc(c, &c->d_fb_snap[k], (size_t)c->cfg.n_streams); if (rc != EF_OK) return rc; }
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
    int rc = ef_read_latest_i420_async(c, first, count, dst, stream);
    if (rc != EF_OK) return rc;
    CK(cudaStreamSynchronize(c->down_stream));
    return EF_OK;
}

int ef_read_frame_i420(ef_ctx* c, int stream_index, int fb, uint8_t* dst)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !dst) return fail(EF_EINVAL, "null argument");
    CK(cudaDeviceSynchronize());
    int f; int rc = resolve_fb(c, stream_index, fb, &f);
    if (rc != EF_OK) return rc;
    rc = ensure_stage(c, EF_FRAME);
    if (rc != EF_OK) return rc;
    ef_export_frames_kernel<<<(EF_FRAME / 8 + 255) / 256, 256>>>(c->h.frames, c->h.base_pics, c->h.n_pics, stream_index, 1, f, 0, c->d_stage);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaMemcpy(dst, c->d_stage, EF_FRAME, cudaMemcpyDeviceToHost));
    return EF_OK;
}

int ef_write_frame_i420(ef_ctx* c, int stream_index, int fb, const uint8_t* src)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !src) return fail(EF_EINVAL, "null argument");
    int f; int rc = resolve_fb(c, stream_index, fb, &f);
    if (rc != EF_OK) return rc;
    rc = ensure_stage(c, EF_FRAME);
    if (rc != EF_OK) return rc;
    if ((rc = wait_frames_read(c)) != EF_OK) return rc;
    CK(cudaMemcpy(c->d_stage, src, EF_FRAME, cudaMemcpyHostToDevice));
    ef_import_frame_kernel<<<(EF_FRAME / 4 + 255) / 256, 256>>>(c->h.frames + ef_frame_offset(stream_index, f), c->d_stage, 0);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaDeviceSynchronize());
    return EF_OK;
}

int ef_write_frame(ef_ctx* c, int stream_index, int fb, const uint8_t* src)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !src) return fail(EF_EINVAL, "null argument");
    int f; int rc = resolve_fb(c, stream_index, fb, &f);
    if (rc != EF_OK) return rc;
    rc = ensure_stage(c, EF_FRAME);
    if (rc != EF_OK) return rc;
    if ((rc = wait_frames_read(c)) != EF_OK) return rc;
    CK(cudaMemcpy(c->d_stage, src, EF_FRAME, cudaMemcpyHostToDevice));
    ef_import_frame_kernel<<<(EF_FRAME / 4 + 255) / 256, 256>>>(c->h.frames + ef_frame_offset(stream_index, f), c->d_stage, 1);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaDeviceSynchronize());
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
    { int rcp = push_dev(c); if (rcp != EF_OK) return rcp; }
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
    int f; int rc = resolve_fb(c, stream_index, fb, &f);
    if (rc != EF_OK) return rc;
    if (!w8) return EF_OK;
    CK(cudaDeviceSynchronize());              // like ef_read_frame: a decode may still be running on a non-blocking user stream
    rc = ensure_stage(c, EF_FRAME);
    if (rc != EF_OK) return rc;
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
    if (on && !c->ev_prof[0]) for (int i = 0; i < 5; i++) CK(cudaEventCreate(&c->ev_prof[i]));
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
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= device) return fail(EF_ECUDA, "no usable CUDA device %d (%s); this library has no CPU path", device, cudaGetErrorString(e));
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
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= device) return fail(EF_ECUDA, "no usable CUDA device %d (%s); this library has no CPU path", device, cudaGetErrorString(e));
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
static int audio_device(int device)
{
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || device < 0 || ndev <= device) return fail(EF_ECUDA, "no usable CUDA device %d (%s); this library has no CPU path", device, cudaGetErrorString(e));
    return EF_OK;
}

static int audio_constants(int device)
{
    static bool constants = false;                       // per process; every device gets its copy on first use
    static int constants_dev = -1;
    if (!constants || constants_dev != device) { CK(ef_audio_upload_constants()); constants = true; constants_dev = device; }
    return EF_OK;
}

// One decode call once its input is in HBM (blob + blob_off[n + 1]: every stream's held-back bytes followed by its new
// bytes): probe and count, then - unless pcm is NULL (sizing: info[] only, no state changes) - SBC -> PCM (-> PDM) and
// the update of the per-stream state. Synchronous on `cs`.
static int audio_decode_blob(const uint8_t* blob, const uint64_t* blob_off, EfAudioState* st, const uint8_t* ended, int n, AudioScratch& w,
                             ef_audio_info* info, int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm, cudaStream_t cs, uint64_t* launches)
{
    int4* plan = nullptr;
    CK(w.get(AudioScratch::PLAN, (size_t)n * sizeof(int4), (void**)&plan));
    ef_sbc_probe_kernel<<<(n + 127) / 128, 128, 0, cs>>>(blob, blob_off, st, ended, n, plan);
    CK(cudaGetLastError());
    ef_sbc_count_kernel<<<(unsigned)(((size_t)n * 32 + 255) / 256), 256, 0, cs>>>(blob, blob_off, ended, n, plan);
    CK(cudaGetLastError());
    *launches += 2;
    std::vector<int4> hp((size_t)n);
    CK(cudaMemcpyAsync(hp.data(), plan, (size_t)n * sizeof(int4), cudaMemcpyDeviceToHost, cs));
    CK(cudaStreamSynchronize(cs));
    std::vector<uint64_t> slot((size_t)n + 1, 0), poff((size_t)n + 1, 0);
    for (int s = 0; s < n; s++) {
        const uint32_t frames = (uint32_t)hp[s].z;
        info[s].frame_size = hp[s].x; info[s].n_frames = frames; info[s].pcm_offset = poff[s];
        slot[s + 1] = slot[s] + (frames ? 1 + (uint64_t)hp[s].y + frames : 0);   // history rows (+ the probe decode of frame 0) + frames
        poff[s + 1] = poff[s] + (uint64_t)frames * 128;
    }
    const uint64_t n_pcm = poff[n];
    if (!pcm) return EF_OK;                                  // sizing call
    if (n_pcm > pcm_cap) return fail(EF_ENOMEM, "%llu PCM samples, capacity %llu", (unsigned long long)n_pcm, (unsigned long long)pcm_cap);
    uint64_t *d_slot = nullptr, *d_poff = nullptr;
    int32_t *sb_last = nullptr, *vrows = nullptr;
    int16_t* d_pcm = nullptr;
    uint16_t* d_pdm = nullptr;
    CK(w.get(AudioScratch::SLOT, slot.size() * 8, (void**)&d_slot));
    CK(w.get(AudioScratch::POFF, poff.size() * 8, (void**)&d_poff));
    CK(w.get(AudioScratch::SB_LAST, (size_t)n * 128 * 4, (void**)&sb_last));
    CK(cudaMemcpyAsync(d_slot, slot.data(), slot.size() * 8, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(d_poff, poff.data(), poff.size() * 8, cudaMemcpyHostToDevice, cs));
    if (n_pcm) {
        CK(w.get(AudioScratch::VROWS, slot[n] * 16 * 16 * 4, (void**)&vrows));
        CK(w.get(AudioScratch::PCM, n_pcm * 2, (void**)&d_pcm));
        ef_sbc_matrix_kernel<<<(unsigned)((slot[n] + 3) / 4), 128, 0, cs>>>(blob, blob_off, plan, st, d_slot, n, vrows, sb_last);
        CK(cudaGetLastError());
        ef_sbc_window_kernel<<<(unsigned)((n_pcm + 255) / 256), 256, 0, cs>>>(vrows, d_slot, d_poff, n, d_pcm);
        CK(cudaGetLastError());
        *launches += 2;
        if (pdm) {
            CK(w.get(AudioScratch::PDM, n_pcm * 4, (void**)&d_pdm));
            ef_pdm_kernel<<<(n + 31) / 32, 32, 0, cs>>>(d_pcm, d_poff, n, st, d_pdm);
            CK(cudaGetLastError());
            *launches += 1;
        }
    }
    ef_audio_commit_kernel<<<(unsigned)(((size_t)n * 32 + 255) / 256), 256, 0, cs>>>(st, blob, blob_off, plan, d_slot, vrows, sb_last, ended, n);
    CK(cudaGetLastError());
    *launches += 1;
    if (n_pcm) {
        CK(cudaMemcpyAsync(pcm, d_pcm, n_pcm * 2, cudaMemcpyDeviceToHost, cs));
        if (pdm) CK(cudaMemcpyAsync(pdm, d_pdm, n_pcm * 4, cudaMemcpyDeviceToHost, cs));
    }
    CK(cudaStreamSynchronize(cs));
    return EF_OK;
}

int ef_audio_demux_ts(int device, const uint8_t* ts, const uint64_t* off, int n_files, uint8_t* es, uint64_t es_cap, uint64_t* es_off)
{
    if (!ts || !off || !es_off || n_files < 1) return fail(EF_EINVAL, "null argument");
    int rc = audio_device(device);
    if (rc != EF_OK) return rc;
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
    int rc = audio_device(device);
    if (rc != EF_OK) return rc;
    DeviceScope scope_(device);
    for (int s = 0; s < n_streams; s++) if (off[s] > off[s + 1]) return fail(EF_EINVAL, "stream offsets must be non-decreasing");
    if ((rc = audio_constants(device)) != EF_OK) return rc;
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
                             info, pcm, pcm_cap, pdm, 0, &launches);
}

int ef_audio_enable(ef_ctx* c)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (c->audio) return EF_OK;
    int rc = audio_constants(c->cfg.device);
    if (rc != EF_OK) return rc;
    const int n = c->cfg.n_streams;
    const size_t cap = c->cfg.es_capacity, packets = cap / 188 + 1;
#define A(ptr, count) if ((rc = dev_alloc(c, &(ptr), (count))) != EF_OK) return rc;
    A(c->d_aud_state, (size_t)n);
    for (int b = 0; b < 2; b++) {
        A(c->d_aud2[b], cap + 1024);                      // a submit's audio is never longer than its transport stream
        A(c->d_aud_off2[b], (size_t)n + 1);
        A(c->d_gate2[b], (size_t)n); A(c->d_lead2[b], (size_t)n); A(c->d_skip2[b], (size_t)n);
    }
    A(c->d_aud_start, packets); A(c->d_aud_kind, packets); A(c->d_aud_pos, packets); A(c->d_aud_len, (size_t)n + 1);
    A(c->d_blob, cap + (size_t)n * EF_AUDIO_CARRY + 1024); A(c->d_blob_len, (size_t)n + 1); A(c->d_blob_off, (size_t)n + 1);
    A(c->d_ended, (size_t)n);
#undef A
    if (!c->h_ended) CK(cudaHostAlloc((void**)&c->h_ended, (size_t)n, cudaHostAllocDefault));
    if (!c->aud_scratch) c->aud_scratch = new AudioScratch();
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

int ef_decode_audio(ef_ctx* c, const uint8_t* end_of_stream, ef_audio_info* info, int16_t* pcm, uint64_t pcm_cap, uint16_t* pdm, void* stream)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c || !info) return fail(EF_EINVAL, "null argument");
    if (!c->audio) return fail(EF_ESTATE, "ef_decode_audio before ef_audio_enable");
    int rc = audio_constants(c->cfg.device);
    if (rc != EF_OK) return rc;
    const int n = c->cfg.n_streams, a = c->active, p = c->pending;
    cudaStream_t cs = (cudaStream_t)stream;
    bool any_end = false;
    for (int s = 0; s < n; s++) { c->h_ended[s] = end_of_stream && end_of_stream[s] ? 1 : 0; any_end |= c->h_ended[s] != 0; }
    CK(cudaStreamWaitEvent(cs, c->ev_up_done[a], 0));        // the demux of the current submit has finished
    if (p >= 0) CK(cudaStreamWaitEvent(cs, c->ev_up_done[p], 0));   // and that of a submit queued behind it (ef_audio_end_kernel)
    CK(cudaMemcpyAsync(c->d_ended, c->h_ended, (size_t)n, cudaMemcpyHostToDevice, cs));
    const uint64_t* new_off = c->aud_unconsumed ? c->d_aud_off2[a] : nullptr;
    ef_audio_len_kernel<<<(n + 255) / 256, 256, 0, cs>>>(c->d_aud_state, new_off, c->d_lead2[a], c->d_skip2[a], n, c->d_blob_len);
    CK(cudaGetLastError());
    ef_ts_offsets_kernel<<<1, 1024, 0, cs>>>(c->d_blob_len, n, c->d_blob_off, c->d_blob);
    CK(cudaGetLastError());
    ef_audio_assemble_kernel<<<n, 256, 0, cs>>>(c->d_aud_state, c->d_aud2[a], new_off, c->d_lead2[a], c->d_skip2[a], c->d_blob_off, c->d_blob);
    CK(cudaGetLastError());
    c->launches += 3;
    rc = audio_decode_blob(c->d_blob, c->d_blob_off, c->d_aud_state, c->d_ended, n, *c->aud_scratch, info, pcm, pcm_cap, pdm, cs, &c->launches);
    if (rc != EF_OK || !pcm) return rc;
    c->aud_unconsumed = false;
    if (any_end) {
        ef_audio_end_kernel<<<(n + 255) / 256, 256, 0, cs>>>(c->d_ended, n, c->d_gate2[a], p >= 0 ? c->d_gate2[p] : nullptr, p >= 0 ? c->d_skip2[p] : nullptr,
                                                             p >= 0 && c->aud_ts[p]);
        CK(cudaGetLastError());
        c->launches++;
        CK(cudaStreamSynchronize(cs));
    }
    return EF_OK;
}

// ---- presentation timestamps: push_video(frame, front, _last_pts, mode) player.cpp:692-702, get_pts() player.cpp:653-656 ----
int ef_pts_enable(ef_ctx* c)
{
    DeviceScope scope_(c ? c->cfg.device : -1);
    if (!c) return fail(EF_EINVAL, "null context");
    if (c->pts) return EF_OK;
    const int n = c->cfg.n_streams;
    const size_t packets = c->cfg.es_capacity / 188 + 1;
    int rc;
#define A(ptr, count) if ((rc = dev_alloc(c, &(ptr), (count))) != EF_OK) return rc;
    for (int b = 0; b < 2; b++) { A(c->d_pts_off2[b], packets); A(c->d_pts_val2[b], packets); A(c->d_pts_span2[b], (size_t)n); }
    A(c->d_pts_carry, (size_t)n); A(c->d_pts_last, (size_t)n); A(c->d_pic_pts, (size_t)n * c->cfg.max_pictures);
#undef A
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

}  // extern "C"
