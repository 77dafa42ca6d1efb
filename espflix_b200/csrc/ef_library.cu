// espflix_b200/csrc/ef_library.cu — titles held in device memory (ef_library_*): every stream's place in its title resolved on the
// device from the title's video.idx, and every stream's run of packets gathered from the title into one TS submit.
//
// The reference's player reads a title through Streamer::get(url, offset) and 8-packet Buffers (espflix.cpp:723-747, 787-798) and
// seeks with the video.idx sample at idx_hdr::pts2offset (espflix.cpp:607-629, 823-829). Here the titles live in HBM: a command is
// a few bytes from the host, the offset arithmetic and the sample read run on the device, and a submit is a device-to-device gather.
#include "../../include/espflix_b200.h"
#include "ef_common.cuh"

namespace {

// idx_hdr::pts2offset (espflix.cpp:607-629): the byte offset in video.idx of the sample for main pts `pts` at `speed`. The casts and
// unsigned divisions are the reference's: at speed 1 (uint32) applies to the difference before the two divisions, at -1 first_pts
// is subtracted a second time (and wraps), and every min() is unsigned.
__device__ __forceinline__ uint32_t lib_pts2offset(const EfLibTitle& t, int64_t pts, int speed)
{
    uint32_t offset;
    pts = max(min(pts, t.v_last), t.v_first);
    if (speed == 1) {
        offset = (uint32_t)(pts - t.v_first) / t.f_trick / t.f_bin;
        offset = min(t.f_n - 1u, offset);
        offset += t.v_n;
    } else if (speed == -1) {
        offset = (uint32_t)((t.v_last - pts) - t.v_first) / t.r_trick / t.r_bin;
        offset = min(t.r_n - 1u, offset);
        offset += t.v_n + t.f_n;
    } else {
        offset = (uint32_t)((pts - t.v_first) / (int64_t)t.v_bin);
        offset = min(t.v_n - 1u, offset);
    }
    return offset * 4u + 104u;                                             // sizeof(idx_hdr)
}

// play(i, speed, get_index(speed, pos) * 188) (espflix.cpp:800-811, 823-829): the stream reads its title's file speed + 1 from the
// packet the sample names. A sample that points at or past the end of its file leaves the cursor there (the stream ends at its next
// submit); the reference's uint32 product would wrap only for such samples.
__device__ __forceinline__ void lib_play(EfLibStream& v, const EfLibTitle& t, int speed)
{
    const uint32_t at = lib_pts2offset(t, v.pos, speed);
    const uint32_t sample = *(const uint32_t*)(t.idx + at);                 // 4-byte aligned: 104 + 4k into a cudaMalloc'd image
    v.speed = speed;
    v.file = speed + 1;
    v.cursor = (uint64_t)sample * 188u;
    v.state = EF_LIB_PLAYING;
}

}  // namespace

// One thread per commanded stream of [first, first + count): the ESPFlix method the command names (espflix.cpp:800-859). Every command
// but PLAY_AT and RESUME first saves pos = pts2pts(get_pts(), _speed) on a PLAYING stream (save_pos, espflix.cpp:843-852); get_pts()
// is the stream's last_pts after the current submit. The host has checked the arguments against every stream's state.
__global__ void ef_library_resolve_kernel(EfLibStream* __restrict__ ls, const EfLibTitle* __restrict__ titles, const int64_t* __restrict__ pts_last,
                                          int first, int count, int cmd, int title, int64_t arg)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const int s = first + k;
    EfLibStream v = ls[s];
    if (cmd == EF_LIB_PLAY_AT) {                                        // nav(i) with pos, then play_pause() from NAV
        v.title = title;
        v.pos = arg;
        lib_play(v, titles[title], 0);
    } else {
        const EfLibTitle& t = titles[v.title];
        if (cmd != EF_LIB_RESUME && v.state == EF_LIB_PLAYING) v.pos = ef_lib_pts2pts(t, pts_last[s], v.speed);
        switch (cmd) {
        case EF_LIB_PLAY: lib_play(v, t, 0); break;
        case EF_LIB_SKIP:                                               // n.pos += s * 90000: an int product
            v.pos += (int32_t)((uint32_t)(int32_t)arg * 90000u);
            lib_play(v, t, 0);
            break;
        case EF_LIB_FAST_FORWARD: lib_play(v, t, 1); break;
        case EF_LIB_REWIND: lib_play(v, t, -1); break;
        case EF_LIB_PAUSE: if (v.state == EF_LIB_PLAYING) v.state = EF_LIB_PAUSED; break;
        case EF_LIB_RESUME: v.state = EF_LIB_PLAYING; break;
        default: v.state = EF_LIB_STOPPED; break;                           // STOP
        }
    }
    ls[s] = v;
}

// One CTA: every PLAYING stream takes min(its budget, packets left in its file) packets from its cursor; the exclusive prefix of the
// run lengths gives each stream's place in the submit (off[n_streams + 1], EfBlockScan). A stream whose cursor
// reaches the end of its file ends with this submit: end[s] = 1, state ENDED, pos = pts2pts(0, _speed) (save_pos(0) at DONE,
// espflix.cpp:906-911). src[s] = where the stream's run starts.
__global__ void __launch_bounds__(1024)
ef_library_count_kernel(EfLibStream* __restrict__ ls, const EfLibTitle* __restrict__ titles, const uint32_t* __restrict__ budget, uint32_t packets,
                        int n_streams, const uint8_t** __restrict__ src, uint64_t* __restrict__ off, uint8_t* __restrict__ end)
{
    __shared__ EfBlockScan<uint64_t, 1024> scan;
    scan.init();
    for (int base = 0; base < n_streams; base += 1024) {
        const int k = base + threadIdx.x;
        uint64_t v = 0;
        if (k < n_streams) {
            EfLibStream q = ls[k];
            uint8_t e = 0;
            if (q.state == EF_LIB_PLAYING) {
                const EfLibTitle& t = titles[q.title];
                const uint64_t size = t.bytes[q.file];
                const uint64_t left = q.cursor < size ? (size - q.cursor) / 188u : 0;
                const uint64_t b = budget ? budget[k] : packets;
                const uint64_t take = b < left ? b : left;
                v = take * 188u;
                src[k] = t.ts[q.file] + (q.cursor < size ? q.cursor : 0);
                q.cursor += v;
                if (take == left) {
                    e = 1;
                    q.state = EF_LIB_ENDED;
                    q.pos = ef_lib_pts2pts(t, 0, q.speed);
                }
                ls[k] = q;
            }
            end[k] = e;
        }
        const uint64_t excl = scan.exclusive(v);
        if (k < n_streams) off[k] = excl;
    }
    if (threadIdx.x == 0) off[n_streams] = scan.carry;
}

// The gather: the submit is one flat range of 16-byte units, EF_LIB_UNITS of them per thread, a CTA's units contiguous. Every stream's
// run is one contiguous range of its file copied to one contiguous range of the submit; both ends are multiples of 188 (4-byte
// aligned, not 16). Each unit is stored with one aligned 16-byte store, its four words loaded from whichever runs they belong to
// (a unit may straddle runs). Thread 0 finds the CTA's first run by binary search over off[]; each thread then walks forward.
// Words past the end of the submit are stored as 0 (the staging buffer has room for the last unit).
#define EF_LIB_GATHER_THREADS 256
#define EF_LIB_UNITS 4
__global__ void __launch_bounds__(EF_LIB_GATHER_THREADS)
ef_library_gather_kernel(const uint8_t* const* __restrict__ src, const uint64_t* __restrict__ off, int n_streams, uint8_t* __restrict__ dst)
{
    __shared__ int s0;
    const uint64_t total = off[n_streams];
    const uint64_t unit0 = (uint64_t)blockIdx.x * (EF_LIB_GATHER_THREADS * EF_LIB_UNITS);
    if (unit0 * 16 >= total) return;
    if (threadIdx.x == 0) {                                                 // the last run with off[s] <= the CTA's first byte
        int lo = 0, hi = n_streams - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (off[mid] <= unit0 * 16) lo = mid; else hi = mid - 1;
        }
        s0 = lo;
    }
    __syncthreads();
    int s = s0;
    uint64_t s_lo = off[s], s_hi = off[s + 1];
    uint4 out[EF_LIB_UNITS];
#pragma unroll
    for (int j = 0; j < EF_LIB_UNITS; j++) {
        const uint64_t b0 = (unit0 + (uint64_t)j * EF_LIB_GATHER_THREADS + threadIdx.x) * 16;
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint64_t b = b0 + 4 * i;
            w[i] = 0;
            if (b < total) {
                while (b >= s_hi) { s++; s_lo = s_hi; s_hi = off[s + 1]; }
                w[i] = __ldg((const uint32_t*)(src[s] + (b - s_lo)));
            }
        }
        out[j] = make_uint4(w[0], w[1], w[2], w[3]);
    }
#pragma unroll
    for (int j = 0; j < EF_LIB_UNITS; j++) {
        const uint64_t b0 = (unit0 + (uint64_t)j * EF_LIB_GATHER_THREADS + threadIdx.x) * 16;
        if (b0 < total) *(uint4*)(dst + b0) = out[j];
    }
}

cudaError_t ef_launch_library_resolve(EfLibStream* ls, const EfLibTitle* titles, const int64_t* pts_last, int first, int count, int cmd, int title,
                                      int64_t arg)
{
    ef_library_resolve_kernel<<<(count + 127) / 128, 128>>>(ls, titles, pts_last, first, count, cmd, title, arg);
    return cudaGetLastError();
}

// count, then gather over at most max_bytes of submit (the host's bound: its grid follows it, CTAs past the submit's end exit)
cudaError_t ef_launch_library_gather(EfLibStream* ls, const EfLibTitle* titles, const uint32_t* budget, uint32_t packets, int n_streams,
                                     const uint8_t** src, uint64_t* off, uint8_t* end, uint8_t* dst, uint64_t max_bytes, cudaStream_t st,
                                     uint64_t* launches)
{
    ef_library_count_kernel<<<1, 1024, 0, st>>>(ls, titles, budget, packets, n_streams, src, off, end);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ++*launches;
    const uint64_t per_cta = (uint64_t)EF_LIB_GATHER_THREADS * EF_LIB_UNITS * 16;
    const uint64_t ctas = (max_bytes + per_cta - 1) / per_cta;
    if (!ctas) return cudaSuccess;
    ef_library_gather_kernel<<<(unsigned)ctas, EF_LIB_GATHER_THREADS, 0, st>>>(src, off, n_streams, dst);
    ++*launches;
    return cudaGetLastError();
}
