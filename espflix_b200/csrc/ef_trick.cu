// csrc/ef_trick.cu — the trick streams of a title (video_fwd.ts, video_rwd.ts) made on the device: the reference's indexer makes them
// with two ffmpeg re-encodes (indexer/indexer.cpp:308-309); here the decoded frames of every 15th main picture are intra-coded (the
// I pictures of ef_encode.cu's slice coder) and muxed. The rule, byte for byte, is tests/trick_cases.py. The host side (segmenting,
// the decode, the plan) is ef_trick_build in ef_capi.cu. Kernels:
//   ef_trick_gather_kernel    after K1b of a picture index: copies the frames of the selected pictures out of the frame stores
//   ef_trick_mux_kernel       one warp per output TS packet, every output file of a build in one launch (the trick files' fwd and
//                             rwd, or ef_encode_build's titles)
#include <stdint.h>

#include "ef_common.cuh"

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

// one warp per output packet: out[k] is packet k of all the output files back to back; pics[] (ascending pkt_first) says which picture
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
cudaError_t ef_trick_launch_gather(const uint8_t* frames, const uint32_t* streams, const uint32_t* slots, int count, int fb, uint8_t* dst, cudaStream_t st)
{
    if (!count) return cudaSuccess;
    const uint64_t threads = (uint64_t)count * (EF_FRAME / 16);
    ef_trick_gather_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(frames, streams, slots, count, fb, dst);
    return cudaGetLastError();
}

cudaError_t ef_trick_launch_mux(const uint8_t* es, const EfTrickPic* pics, int n_pics, uint64_t n_packets, uint8_t* out, cudaStream_t st)
{
    if (!n_packets) return cudaSuccess;
    ef_trick_mux_kernel<<<(unsigned)((n_packets * 32 + 255) / 256), 256, 0, st>>>(es, pics, n_pics, n_packets, out);
    return cudaGetLastError();
}
