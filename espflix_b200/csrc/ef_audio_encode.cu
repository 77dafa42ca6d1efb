// ef_audio_encode.cu — SBC encoder: mono 16-bit PCM to mono / 16-block / 8-subband SBC frames, the audio of a title's video.ts (the
// reference's make_video() has ffmpeg make it: indexer/indexer.cpp:306-309). The rule, byte for byte, is tests/sbc_encode_cases.py;
// the host side (argument checks, chunks of frames, copies) is ef_sbc_encode in ef_capi.cu.
//   ef_sbc_encode_kernel  one warp per frame: the 200 samples frame f reads (128 f - 72 .. 128 f + 127) into shared memory, the
//                         A2DP analysis filterbank in int64 (window: 8 values per lane, matrixing: 4), scale factors by a warp
//                         max, the bit allocation once per frame on lane 0, the quantiser, the bits packed MSB first with
//                         shared-memory ORs, then header, CRC-8 and payload stored by the whole warp.
// A frame needs no state from the frame before it, so frames of every stream of a call are spread over one grid.
#include <stdint.h>

#include "../../include/espflix_b200.h"
#include "ef_common.cuh"
#include "ef_sbc_analysis_tables.h"
#include "ef_sbc_tables.h"

namespace {

constexpr int kWarps = 8;
constexpr int kSpan = 200;                    // samples one frame reads: 72 of history and its own 128

__constant__ int c_awin[80];
__constant__ int c_amat[8][16];
__constant__ signed char c_aoffset8[4][8];

// the bit allocation of mono / 8-subband frames (A2DP 12.6.3; sbc_decoder.cpp:141-231, which ef_audio.cu's sbc_frame_bits
// restates from a frame's bytes): scale factors in, widths out
__device__ void sbc_alloc(int frequency, int allocation, int bitpool, const int* sf, int* bits)
{
    int bitneed[8], max_bitneed = 0;
    for (int sb = 0; sb < 8; sb++) {
        int need;
        if (allocation) need = sf[sb];
        else if (sf[sb] == 0) need = -5;
        else { need = sf[sb] - c_aoffset8[frequency][sb]; if (need > 0) need /= 2; }
        bitneed[sb] = need;
        max_bitneed = max(max_bitneed, need);
    }
    int bitcount = 0, slicecount = 0, bitslice = max_bitneed + 1;
    do {
        bitslice--;
        bitcount += slicecount;
        slicecount = 0;
        for (int sb = 0; sb < 8; sb++) {
            if (bitneed[sb] > bitslice + 1 && bitneed[sb] < bitslice + 16) slicecount++;
            else if (bitneed[sb] == bitslice + 1) slicecount += 2;
        }
    } while (bitcount + slicecount < bitpool);
    if (bitcount + slicecount == bitpool) { bitcount += slicecount; bitslice--; }
    for (int sb = 0; sb < 8; sb++) bits[sb] = bitneed[sb] < bitslice + 2 ? 0 : min(bitneed[sb] - bitslice, 16);
    for (int sb = 0; sb < 8 && bitcount < bitpool; sb++) {
        if (bits[sb] >= 2 && bits[sb] < 16) { bits[sb]++; bitcount++; }
        else if (bitneed[sb] == bitslice + 1 && bitpool > bitcount + 1) { bits[sb] = 2; bitcount += 2; }
    }
    for (int sb = 0; sb < 8 && bitcount < bitpool; sb++)
        if (bits[sb] < 16) { bits[sb]++; bitcount++; }
}

__device__ uint32_t crc8_byte(uint32_t c, uint32_t b)
{
    for (int i = 7; i >= 0; i--) {
        const uint32_t bit = ((b >> i) & 1) ^ (c >> 7);
        c = (c << 1) & 0xFF;
        if (bit) c ^= 0x1D;
    }
    return c;
}

struct WarpSmem {
    int32_t x[kSpan];
    long long y[16][16];
    uint32_t words[65];                        // the payload, MSB first, as big-endian words (one spare for a straddling value)
};

// frames [frame0, frame0 + n_frames) of the call; frame_first[s] is stream s's first frame, pcm_off[s] its first sample;
// pcm holds samples pcm_base .. of the call's PCM
__global__ void __launch_bounds__(kWarps * 32) ef_sbc_encode_kernel(const int16_t* __restrict__ pcm, uint64_t pcm_base, uint64_t pcm_len,
    const uint64_t* __restrict__ pcm_off, const uint64_t* __restrict__ frame_first, int n_streams, uint64_t frame0, uint64_t n_frames,
    int frequency, int allocation, int bitpool, uint8_t* __restrict__ out)
{
    __shared__ WarpSmem sm_all[kWarps];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t fr = frame0 + (uint64_t)blockIdx.x * kWarps + w;
    if (fr >= frame0 + n_frames) return;
    WarpSmem& sm = sm_all[w];
    int lo = 0, hi = n_streams - 1;                                    // the stream: the last one whose first frame is <= fr
    while (lo < hi) { const int m = (lo + hi + 1) >> 1; if (frame_first[m] <= fr) lo = m; else hi = m - 1; }
    const uint64_t s_begin = pcm_off[lo], s_end = pcm_off[lo + 1];
    const int64_t first = (int64_t)(s_begin + (fr - frame_first[lo]) * 128) - 72;      // sample of x[0]
    for (int t = lane; t < kSpan; t += 32) {
        const int64_t g = first + t;
        sm.x[t] = g >= (int64_t)s_begin && g < (int64_t)s_end && (uint64_t)g - pcm_base < pcm_len ? pcm[(uint64_t)g - pcm_base] : 0;
    }
    for (int t = lane; t < 65; t += 32) sm.words[t] = 0;
    __syncwarp();
    // windowing: Y[b][i] = sum_m C[i + 16 m] X[i + 16 m], X[j] = x[72 + 8 b + 7 - j]
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int idx = lane + 32 * r, b = idx >> 4, i = idx & 15;
        long long acc = 0;
#pragma unroll
        for (int m = 0; m < 5; m++) acc += (long long)(c_awin[i + 16 * m] * sm.x[79 + 8 * b - i - 16 * m]);
        sm.y[b][i] = acc;
    }
    __syncwarp();
    // matrixing: lane holds subband k = lane & 7 of blocks (lane >> 3) + 4 r
    const int k = lane & 7;
    int32_t v[4];
    uint32_t mx = 0;
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int b = (lane >> 3) + 4 * r;
        long long acc = 0;
#pragma unroll
        for (int i = 0; i < 16; i++) acc += (long long)c_amat[k][i] * sm.y[b][i];
        long long q = (acc + (1ll << 17)) >> 18;
        q = q < -(1ll << 31) ? -(1ll << 31) : q > (1ll << 31) - 1 ? (1ll << 31) - 1 : q;
        v[r] = (int32_t)q;
        mx = max(mx, (uint32_t)(q < 0 ? -q : q));
    }
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, 8));
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, 16));
    int s = 0;
    for (int t = 0; t < 15; t++) s += mx >= (1u << (t + 16));
    // bit allocation once per frame, on lane 0
    int sf[8], bits[8];
#pragma unroll
    for (int sb = 0; sb < 8; sb++) sf[sb] = __shfl_sync(0xffffffffu, s, sb);
    int lo_w = 0, hi_w = 0;                                             // the widths, a byte each
    if (lane == 0) {
        sbc_alloc(frequency, allocation, bitpool, sf, bits);
#pragma unroll
        for (int sb = 0; sb < 4; sb++) { lo_w |= bits[sb] << (8 * sb); hi_w |= bits[sb + 4] << (8 * sb); }
    }
    lo_w = __shfl_sync(0xffffffffu, lo_w, 0);
    hi_w = __shfl_sync(0xffffffffu, hi_w, 0);
#pragma unroll
    for (int sb = 0; sb < 8; sb++) bits[sb] = ((sb < 4 ? lo_w : hi_w) >> (8 * (sb & 3))) & 0xFF;
    int before = 0;                                                     // bits of the subbands before k in a block
#pragma unroll
    for (int sb = 0; sb < 8; sb++) before += sb < k ? bits[sb] : 0;
    const int L = bits[k];
    if (L) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const int b = (lane >> 3) + 4 * r;
            uint32_t q = (uint32_t)((((long long)v[r] + (1ll << (s + 16))) * ((1ll << L) - 1)) >> (s + 17));
            if (L == 16 && s == 15) q = min(q, 32767u);
            const int pos = b * bitpool + before, wd = pos >> 5, off = pos & 31;
            const int sh = 32 - off - L;                               // the value's place in its word, negative: it straddles
            if (sh >= 0) atomicOr(&sm.words[wd], q << sh);
            else { atomicOr(&sm.words[wd], q >> -sh); atomicOr(&sm.words[wd + 1], q << (32 + sh)); }
        }
    }
    __syncwarp();
    const int fbytes = 8 + 2 * bitpool;
    uint8_t* dst = out + (fr - frame0) * (uint64_t)fbytes;
    uint32_t hdr = 0;                                                   // bytes 0..3 little-endian in a word
    uint32_t sfw = 0;                                                   // bytes 4..7
    if (lane == 0) {
        const uint32_t b1 = (uint32_t)(frequency << 6) | 0x30u | (uint32_t)(allocation << 1) | 1u;
        uint32_t c = crc8_byte(crc8_byte(0x0F, b1), (uint32_t)bitpool);
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const uint32_t by = (uint32_t)(sf[2 * t] << 4 | sf[2 * t + 1]);
            c = crc8_byte(c, by);
            sfw |= by << (8 * t);
        }
        hdr = 0x9Cu | b1 << 8 | (uint32_t)bitpool << 16 | c << 24;
    }
    hdr = __shfl_sync(0xffffffffu, hdr, 0);
    sfw = __shfl_sync(0xffffffffu, sfw, 0);
    for (int t = lane; t < fbytes; t += 32) {
        uint32_t by;
        if (t < 4) by = hdr >> (8 * t);
        else if (t < 8) by = sfw >> (8 * (t - 4));
        else by = sm.words[(t - 8) >> 2] >> (8 * (3 - ((t - 8) & 3)));
        dst[t] = (uint8_t)by;
    }
}

}  // namespace

cudaError_t ef_sbc_encode_upload_tables()
{
    cudaError_t e = cudaMemcpyToSymbol(c_awin, ef_sbc_analysis_window, sizeof(ef_sbc_analysis_window));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_amat, ef_sbc_analysis_matrix, sizeof(ef_sbc_analysis_matrix));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_aoffset8, ef_sbc_offset8, sizeof(ef_sbc_offset8));
    return e;
}

// frames [frame0, frame0 + n_frames) into out (frame frame0 at out[0])
cudaError_t ef_sbc_launch_encode(const int16_t* pcm, uint64_t pcm_base, uint64_t pcm_len, const uint64_t* pcm_off, const uint64_t* frame_first,
                                 int n_streams, uint64_t frame0, uint64_t n_frames, int frequency, int allocation, int bitpool, uint8_t* out,
                                 cudaStream_t st)
{
    if (!n_frames) return cudaSuccess;
    ef_sbc_encode_kernel<<<(unsigned)((n_frames + kWarps - 1) / kWarps), kWarps * 32, 0, st>>>(pcm, pcm_base, pcm_len, pcm_off, frame_first,
        n_streams, frame0, n_frames, frequency, allocation, bitpool, out);
    return cudaGetLastError();
}
