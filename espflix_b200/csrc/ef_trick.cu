// csrc/ef_trick.cu — the trick streams of a title (video_fwd.ts, video_rwd.ts) made on the device: the reference's indexer makes them
// with two ffmpeg re-encodes (indexer/indexer.cpp:308-309); here the decoded frames of every 15th main picture are intra-coded and
// muxed. The rule, byte for byte, is tests/trick_cases.py. The host side (segmenting, the decode, the plan) is ef_trick_build in
// ef_capi.cu. Kernels:
//   ef_trick_gather_kernel    after K1b of a picture index: copies the frames of the selected pictures out of the frame stores
//   ef_trick_encode_kernel    one warp per slice (macroblock row): FDCT, quantiser, code lengths, a warp prefix sum for the bit
//                             offsets, codes OR-ed into a shared window and flushed to a per-slice region of kTrickSliceBytes
//   ef_trick_assemble_kernel  one CTA per picture: header + its 12 slices, back to back, at the picture's offset in the ES
//   ef_trick_mux_kernel       one warp per output TS packet, fwd and rwd of every file in one launch
#include <stdint.h>

#include "ef_vlc_put.cuh"

namespace {
constexpr int kWarps = 4;
}  // namespace

__global__ void ef_trick_gather_kernel(const uint8_t* __restrict__ frames, const uint32_t* __restrict__ streams, const uint32_t* __restrict__ slots,
                                       int count, int fb, uint8_t* __restrict__ dst)
{
    constexpr uint32_t per = EF_FRAME / 16;
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t k = (uint32_t)(t / per), w = (uint32_t)(t % per);
    if (k >= (uint32_t)count) return;
    const uint4* src = (const uint4*)(frames + ef_frame_offset((int)streams[k], fb));
    ((uint4*)(dst + (size_t)slots[k] * EF_FRAME))[w] = src[w];
}

__global__ void __launch_bounds__(kWarps * 32) ef_trick_encode_kernel(const uint8_t* __restrict__ in, int n_pics, int qscale_all,
                                                                     const uint8_t* __restrict__ qpic, uint32_t* __restrict__ slots,
                                                                     uint32_t* __restrict__ slice_len)
{
    __shared__ uint32_t s_ac[32 * 41];
    __shared__ int s_t[kWarps][64], s_f[kWarps][64];
    __shared__ uint32_t s_win[kWarps][kWin + 2];
    for (int i = threadIdx.x; i < 32 * 41; i += blockDim.x) s_ac[i] = c_trick.ac[i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * kWarps + warp;
    if (gw >= n_pics * EF_MBH_MAX) return;
    const int pic = gw / EF_MBH_MAX, row = gw % EF_MBH_MAX;
    const int qv = qpic ? (int)qpic[pic] : qscale_all, qscale = qv & 31;
    const bool fallback = qv & kQFallback;   // every AC level zero: the DC levels alone
    uint32_t* out = slots + (size_t)gw * (kTrickSliceBytes / 4);
    const uint8_t* frame = in + (size_t)pic * EF_FRAME;
    uint32_t* win = s_win[warp];
    int* T = s_t[warp];
    int* F = s_f[warp];
    for (int i = lane; i < kWin + 2; i += 32) win[i] = 0;
    __syncwarp();
    if (lane == 0) { win[0] = 0x00000100u | (uint32_t)(row + 1); win[1] = (uint32_t)qscale << 27; }   // slice start code, quantiser, extra bit
    uint32_t P = 38, wbase = 0;              // bit position in the slice, slice word held in win[0]
    int pred[3] = { 128, 128, 128 };
    const int r = lane >> 2, k0 = (lane & 3) * 2;
    for (int mb = 0; mb < EF_MBW_MAX; mb++) {
        const uint8_t* tile = frame + ef_tile_offset(mb, row);
        __syncwarp();
        if (lane == 0) put_bits(win, P - wbase * 32, 3u, 2);    // address increment 1, intra macroblock type
        P += 2;
        for (int b = 0; b < 6; b++) {
            // row pass: lane = (row r, outputs k0, k0 + 1)
            const int po = b < 4 ? ((b >> 1) * 8 + r) * 16 + (b & 1) * 8 : 256 + (b - 4) * 64 + r * 8;
            const uint2 px = *(const uint2*)(tile + po);
            int x[8];
            #pragma unroll
            for (int n = 0; n < 4; n++) { x[n] = (px.x >> (8 * n)) & 0xFF; x[n + 4] = (px.y >> (8 * n)) & 0xFF; }
            fdct_block(x, T, F, r, k0);
            // quantise zig-zag indices 2 lane and 2 lane + 1 (so the lanes' codes follow each other in bitstream order); the DC
            // counts as coded
            int lv0 = quant(2 * lane, F, qscale), lv1 = quant(2 * lane + 1, F, qscale);
            if (fallback) { lv1 = 0; if (lane) lv0 = 0; }
            const uint32_t ev = __ballot_sync(0xFFFFFFFFu, lane == 0 || lv0 != 0), od = __ballot_sync(0xFFFFFFFFu, lv1 != 0);
            const uint64_t mask = spread_bits(ev) | (spread_bits(od) << 1);
            uint32_t c0, n0, c1, n1;
            code_of(2 * lane, lv0, mask, s_ac, &c0, &n0);
            code_of(2 * lane + 1, lv1, mask, s_ac, &c1, &n1);
            const int dc = __shfl_sync(0xFFFFFFFFu, lv0, 0);
            const int comp = b < 4 ? 0 : b - 3;
            if (lane == 0) {                 // DC difference: size code, then the difference bits
                const int diff = dc - pred[comp], a = diff < 0 ? -diff : diff;
                const uint32_t size = 32 - __clz(a);
                const uint32_t e = c_trick.dc[comp ? 1 : 0][size];
                c0 = ((e >> 8) << size) | (uint32_t)(diff > 0 ? diff : diff + (1 << size) - 1);
                n0 = (e & 0xFF) + size;
            }
            pred[comp] = dc;
            const uint32_t sum = n0 + n1;
            uint32_t incl = sum;
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, d);
                if (lane >= d) incl += v;
            }
            const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
            const uint32_t q = P - wbase * 32 + incl - sum;
            put_bits(win, q, c0, n0);
            put_bits(win, q + n0, c1, n1);
            if (lane == 0) put_bits(win, P - wbase * 32 + total, 2u, 2);     // end of block "10"
            P += total + 2;
            __syncwarp();
            // flush the complete words, keep the partial one
            const uint32_t full = (P >> 5) - wbase;
            for (uint32_t i = lane; i < full; i += 32) out[wbase + i] = __byte_perm(win[i], 0, 0x0123);
            __syncwarp();
            const uint32_t carry = win[full];
            __syncwarp();
            for (int i = lane; i < kWin + 2; i += 32) win[i] = 0;
            __syncwarp();
            if (lane == 0) win[0] = carry;
            wbase += full;
        }
    }
    __syncwarp();
    const uint32_t words = ((P + 31) >> 5) - wbase;          // the slice ends on a byte boundary, zero-padded
    for (uint32_t i = lane; i < words; i += 32) out[wbase + i] = __byte_perm(win[i], 0, 0x0123);
    if (lane == 0) slice_len[gw] = (P + 7) >> 3;
}

// one CTA per picture: the 28 header bytes of its file, then its slices, at pic_dst[p] in es
__global__ void ef_trick_assemble_kernel(const uint32_t* __restrict__ slots, const uint32_t* __restrict__ slice_len, const uint64_t* __restrict__ pic_dst,
                                         const uint8_t* __restrict__ headers, uint8_t* __restrict__ es)
{
    const int p = blockIdx.x;
    __shared__ uint32_t off[EF_MBH_MAX + 1];
    if (threadIdx.x == 0) {
        off[0] = kTrickHeaderBytes;
        for (int s = 0; s < EF_MBH_MAX; s++) off[s + 1] = off[s] + slice_len[p * EF_MBH_MAX + s];
    }
    __syncthreads();
    uint8_t* dst = es + pic_dst[p];
    for (int i = threadIdx.x; i < kTrickHeaderBytes; i += blockDim.x) dst[i] = headers[(size_t)p * kTrickHeaderBytes + i];
    for (int s = 0; s < EF_MBH_MAX; s++) {
        const uint8_t* src = (const uint8_t*)(slots + (size_t)(p * EF_MBH_MAX + s) * (kTrickSliceBytes / 4));
        const uint32_t n = off[s + 1] - off[s];
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[off[s] + i] = src[i];
    }
}

// one warp per output packet: out[k] is packet k of all the trick files back to back; pics[] (ascending pkt_first) says which picture
// and which part of its PES the packet carries (efs_wrap_ts's layout: a 14-byte PES header, full packets, the last one stuffed)
__global__ void ef_trick_mux_kernel(const uint8_t* __restrict__ es, const EfTrickPic* __restrict__ pics, int n_pics, uint64_t n_packets, uint8_t* __restrict__ out)
{
    const uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (k >= n_packets) return;
    int lo = 0, hi = n_pics - 1;
    while (lo < hi) { const int m = (lo + hi + 1) >> 1; if (pics[m].pkt_first <= k) lo = m; else hi = m - 1; }
    const EfTrickPic d = pics[lo];
    const uint32_t j = (uint32_t)(k - d.pkt_first);
    const uint32_t pes_len = 14 + d.es_len, pos = j * 184, left = pes_len - pos;
    const uint32_t af = left >= 184 ? 0 : 184 - left;                   // adaptation field bytes, its length byte included
    const uint64_t pts = (uint64_t)d.pts & ((1ull << 33) - 1);
    uint8_t* pkt = out + k * 188;
    for (int t = lane; t < 188; t += 32) {
        uint8_t v;
        if (t == 0) v = 0x47;
        else if (t == 1) v = (uint8_t)((j == 0 ? 0x40 : 0) | 0x01);
        else if (t == 2) v = 0x00;
        else if (t == 3) v = (uint8_t)((af ? 0x30 : 0x10) | ((d.cc0 + j) & 15));
        else if ((uint32_t)t < 4 + af) v = t == 4 ? (uint8_t)(af - 1) : t == 5 ? 0 : 0xFF;
        else {
            const uint32_t b = pos + (uint32_t)t - 4 - af;             // byte of the PES
            if (b >= 14) v = es[d.es_off + b - 14];
            else {
                switch (b) {
                case 2: v = 1; break;
                case 3: v = 0xE0; break;
                case 6: case 7: v = 0x80; break;
                case 8: v = 5; break;
                case 9: v = (uint8_t)(0x21 | ((pts >> 29) & 0x0E)); break;
                case 10: v = (uint8_t)(pts >> 22); break;
                case 11: v = (uint8_t)(0x01 | ((pts >> 14) & 0xFE)); break;
                case 12: v = (uint8_t)(pts >> 7); break;
                case 13: v = (uint8_t)(0x01 | ((pts << 1) & 0xFE)); break;
                default: v = 0;
                }
            }
        }
        pkt[t] = v;
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------------------------
cudaError_t ef_trick_upload_tables() { return upload_trick_tables(); }

cudaError_t ef_trick_launch_gather(const uint8_t* frames, const uint32_t* streams, const uint32_t* slots, int count, int fb, uint8_t* dst, cudaStream_t st)
{
    if (!count) return cudaSuccess;
    const uint64_t threads = (uint64_t)count * (EF_FRAME / 16);
    ef_trick_gather_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(frames, streams, slots, count, fb, dst);
    return cudaGetLastError();
}

cudaError_t ef_trick_launch_encode(const uint8_t* in, int n_pics, int qscale, uint32_t* slots, uint32_t* slice_len, cudaStream_t st,
                                  const uint8_t* qpic)
{
    const int warps = n_pics * EF_MBH_MAX;
    ef_trick_encode_kernel<<<(warps + kWarps - 1) / kWarps, kWarps * 32, 0, st>>>(in, n_pics, qscale, qpic, slots, slice_len);
    return cudaGetLastError();
}

cudaError_t ef_trick_launch_assemble(const uint32_t* slots, const uint32_t* slice_len, const uint64_t* pic_dst, const uint8_t* headers, int n_pics,
                                     uint8_t* es, cudaStream_t st)
{
    ef_trick_assemble_kernel<<<n_pics, 256, 0, st>>>(slots, slice_len, pic_dst, headers, es);
    return cudaGetLastError();
}

cudaError_t ef_trick_launch_mux(const uint8_t* es, const EfTrickPic* pics, int n_pics, uint64_t n_packets, uint8_t* out, cudaStream_t st)
{
    if (!n_packets) return cudaSuccess;
    ef_trick_mux_kernel<<<(unsigned)((n_packets * 32 + 255) / 256), 256, 0, st>>>(es, pics, n_pics, n_packets, out);
    return cudaGetLastError();
}
