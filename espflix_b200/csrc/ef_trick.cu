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
    ef_pes_packet(out + k * 188, lane, 32, j, 0x100, 0xE0, 0, d.pts, d.cc0 + j, es + d.es_off, d.es_len);
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
