// csrc/ef_encode.cu — a title's video.ts encoded on the device from raw pictures: what the reference's indexer makes with ffmpeg
// (make_video(), indexer/indexer.cpp:306). GOPs of an I picture (ef_trick_encode_kernel, unchanged) and P pictures predicted from the
// decoder's own reconstruction of the picture before them (the frame store K1b wrote). The rule, byte for byte, is
// tests/encode_cases.py; the host side (GOP batches, the rounds, the reconstruction, the mux) is ef_encode_build in ef_capi.cu.
// Kernels:
//   ef_encode_tile_kernel      I420 pictures -> the macroblock-tiled frame layout, one 16-byte store per thread
//   ef_encode_search_kernel    one warp per macroblock: the source macroblock and the reference window in shared memory, full-pel
//                              candidates split over the lanes (packed SADs, one warp minimum at the end), then the 3 x 3 half-pel
//                              neighbours and the intra decision
//   ef_encode_p_kernel         one warp per slice of a P picture: prediction, FDCT, quantiser, then the macroblock header and block
//                              codes placed by a warp prefix sum in a shared window, flushed to a per-slice region of kEncSliceBytes
//   ef_encode_census_kernel    ef_encode_build_rate: one warp per slice, the slice's exact bytes at every candidate quantiser and as
//                              its fallback, from one FDCT per block
//   ef_encode_choose_kernel    ef_encode_build_rate: one thread per GOP, its bucket and the choice of the picture's quantiser
//   ef_encode_assemble_kernel  one CTA per P picture: its 9 header bytes and 12 slices at the picture's offset in the ES
#include <stdint.h>

#include "ef_vlc_put.cuh"

namespace {

constexpr int kEncWarps = 4;
constexpr int kZeroBias = 64;        // tests/encode_cases.ZERO_BIAS
constexpr int kIntraMargin = 512;    // tests/encode_cases.INTRA_MARGIN
constexpr int kWinW = 10, kWinH = 33;   // reference window: 33 rows of 40 bytes from (16 mx - 8, 16 my - 8)

struct EncTables {
    uint32_t mba[34];        // macroblock_address_increment 1..33: (code << 8) | length
    uint32_t type[32];       // P macroblock_type value -> (code << 8) | length
    uint32_t mv[33];         // motion code -16..16 at [code + 16] (f_code 1: no residual bits)
    uint32_t cbp[64];        // coded_block_pattern 1..63
};
__constant__ EncTables c_enc;

// efsynth's legal(): the prediction block inside the picture and the vector inside forward_f_code 1's range
__device__ __forceinline__ bool legal_mv(int mx, int my, int h, int v)
{
    const int hx = 32 * mx + h, hy = 32 * my + v;
    return hx >= 0 && hy >= 0 && (hx >> 1) + 16 + (hx & 1) <= EF_W && (hy >> 1) + 16 + (hy & 1) <= EF_H && h >= -16 && h <= 15 && v >= -16 &&
           v <= 15;
}

__device__ __forceinline__ int mc_pel(const uint8_t* p0, const uint8_t* p1, const uint8_t* p2, const uint8_t* p3, int xh, int yh)
{
    const int a = *p0;
    if (xh && yh) return (a + *p1 + *p2 + *p3 + 2) >> 2;
    if (xh) return (a + *p1 + 1) >> 1;
    if (yh) return (a + *p2 + 1) >> 1;
    return a;
}

__device__ __forceinline__ int quant_inter(int i, const int* F, int qscale)
{
    const int f = F[c_trick.zz[i]], a = (8 * (f < 0 ? -f : f)) / (16 * qscale);
    const int lv = a > 255 ? 255 : a;
    return f < 0 ? -lv : lv;
}

}  // namespace

__global__ void ef_encode_tile_kernel(const uint8_t* __restrict__ i420, const uint32_t* __restrict__ src, int count, uint8_t* __restrict__ tiled)
{
    constexpr uint32_t per = EF_FRAME / 16;
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t k = (uint32_t)(t / per), w = (uint32_t)(t % per);
    if (k >= (uint32_t)count) return;
    const uint8_t* pic = i420 + (size_t)src[k] * EF_FRAME;
    const uint32_t tile = w / 24, q = w % 24, mx = tile % EF_MBW_MAX, my = tile / EF_MBW_MAX;
    uint4 v;
    if (q < 16) v = *(const uint4*)(pic + (my * 16 + q) * EF_W + mx * 16);
    else {                                               // two 8-byte rows of block 4 (q 16..19) or block 5 (q 20..23)
        const uint32_t c = q - 16, row = (c & 3) * 2;
        const uint8_t* p = pic + EF_W * EF_H + (c >> 2) * (176 * 96) + (my * 8 + row) * 176 + mx * 8;
        const uint2 a = *(const uint2*)p, b = *(const uint2*)(p + 176);
        v = make_uint4(a.x, a.y, b.x, b.y);
    }
    ((uint4*)(tiled + (size_t)k * EF_FRAME))[w] = v;
}

// picture k of the list (tiled source src + k EF_FRAME) is predicted from the latest frame store of decoder stream streams[k];
// mbinfo[k * 264 + address] = h & 0xFF | (v & 0xFF) << 8 (half-pel vector), or 1 << 16 for an intra macroblock
__global__ void __launch_bounds__(kEncWarps * 32) ef_encode_search_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ streams, int count,
                                                                         const uint8_t* __restrict__ frames, const uint32_t* __restrict__ base_pics,
                                                                         const uint32_t* __restrict__ n_pics, int search, uint32_t* __restrict__ mbinfo)
{
    __shared__ uint32_t s_src[kEncWarps][64];
    __shared__ uint32_t s_win[kEncWarps][kWinH * kWinW];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * kEncWarps + warp;
    if (gw >= count * EF_MBW_MAX * EF_MBH_MAX) return;
    const int k = gw / (EF_MBW_MAX * EF_MBH_MAX), mb = gw % (EF_MBW_MAX * EF_MBH_MAX), mx = mb % EF_MBW_MAX, my = mb / EF_MBW_MAX;
    const int s = (int)streams[k];
    const uint8_t* ref = frames + ef_frame_offset(s, (int)((base_pics[s] + n_pics[s]) & 1u));
    const uint32_t* tile = (const uint32_t*)(src + (size_t)k * EF_FRAME + ef_tile_offset(mx, my));
    uint32_t* S = s_src[warp];
    uint32_t* Wn = s_win[warp];
    for (int i = lane; i < 64; i += 32) S[i] = tile[i];
    for (int i = lane; i < kWinH * kWinW; i += 32) {     // 4 pixels at x % 4 == 0 lie in one tile row: one aligned word
        const int y = my * 16 - 8 + i / kWinW, x = mx * 16 - 8 + 4 * (i % kWinW);
        Wn[i] = (y >= 0 && y < EF_H && x >= 0 && x < EF_W) ? *(const uint32_t*)(ref + ef_luma_offset(x, y)) : 0u;
    }
    __syncwarp();
    // the zero vector: lane = (row lane / 2, half lane & 1)
    const int yr = lane >> 1, xo = (lane & 1) * 8;
    const int sad0 = __reduce_add_sync(0xFFFFFFFFu, (int)(__vsadu4(Wn[(8 + yr) * kWinW + 2 + (lane & 1) * 2], S[yr * 4 + (lane & 1) * 2]) +
                                                          __vsadu4(Wn[(8 + yr) * kWinW + 3 + (lane & 1) * 2], S[yr * 4 + (lane & 1) * 2 + 1])));
    // full-pel candidates c = (dy + search) n + dx + search in raster order, lane c % 32; key = sad << 10 | c, so the warp minimum is the
    // first candidate of the lowest sad
    const int n = 2 * search + 1, nc = n * n;
    uint32_t key = 0xFFFFFFFFu;
    for (int c = lane; c < nc; c += 32) {
        const int dx = c % n - search, dy = c / n - search;
        if (!legal_mv(mx, my, 2 * dx, 2 * dy)) continue;            // legal: -8 <= dx, dy <= 7
        const int o = dx + 8, wi = o >> 2, sh = (o & 3) * 8;
        uint32_t sad = 0;
        #pragma unroll 4
        for (int y = 0; y < 16; y++) {
            const uint32_t* w = Wn + (dy + 8 + y) * kWinW + wi;
            const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4];
            sad = __vsadu4(__funnelshift_r(w0, w1, sh), S[y * 4]) + sad;
            sad = __vsadu4(__funnelshift_r(w1, w2, sh), S[y * 4 + 1]) + sad;
            sad = __vsadu4(__funnelshift_r(w2, w3, sh), S[y * 4 + 2]) + sad;
            sad = __vsadu4(__funnelshift_r(w3, w4, sh), S[y * 4 + 3]) + sad;
        }
        key = min(key, (sad << 10) | (uint32_t)c);
    }
    key = __reduce_min_sync(0xFFFFFFFFu, key);
    int best = sad0 - kZeroBias, bh = 0, bv = 0;
    if (key != 0xFFFFFFFFu && (int)(key >> 10) < best) {
        const int c = (int)(key & 1023);
        best = (int)(key >> 10); bh = 2 * (c % n - search); bv = 2 * (c / n - search);
    }
    // half-pel neighbours, the decoder's averaging; lane = 8 pixels of row yr
    const uint8_t* Wb = (const uint8_t*)Wn;
    const uint8_t* Sb = (const uint8_t*)S;
    const int ch = bh, cv = bv;
    for (int b = -1; b <= 1; b++)
        for (int a = -1; a <= 1; a++) {
            const int h = ch + a, v = cv + b;
            if (!legal_mv(mx, my, h, v)) continue;
            const int ry = v + 16 + 2 * yr, py = ry >> 1, yh = ry & 1;
            int acc = 0;
            #pragma unroll
            for (int i = 0; i < 8; i++) {
                const int rx = h + 16 + 2 * (xo + i), px = rx >> 1, xh = rx & 1;
                const uint8_t* p = Wb + py * (kWinW * 4) + px;
                const int d = (int)Sb[yr * 16 + xo + i] - mc_pel(p, p + 1, p + kWinW * 4, p + kWinW * 4 + 1, xh, yh);
                acc += d < 0 ? -d : d;
            }
            const int sad = __reduce_add_sync(0xFFFFFFFFu, acc);
            if (sad < best) { best = sad; bh = h; bv = v; }
        }
    // intra when the best prediction is worse than the source's own mean absolute deviation by more than the margin
    int sum = 0;
    #pragma unroll
    for (int i = 0; i < 8; i++) sum += Sb[yr * 16 + xo + i];
    const int mean = (__reduce_add_sync(0xFFFFFFFFu, sum) + 128) >> 8;
    int dev = 0;
    #pragma unroll
    for (int i = 0; i < 8; i++) { const int d = (int)Sb[yr * 16 + xo + i] - mean; dev += d < 0 ? -d : d; }
    const int mad = __reduce_add_sync(0xFFFFFFFFu, dev);
    if (lane == 0) mbinfo[gw] = best > mad + kIntraMargin ? (1u << 16) : ((uint32_t)(bh & 0xFF) | ((uint32_t)(bv & 0xFF) << 8));
}

__global__ void __launch_bounds__(kEncWarps * 32) ef_encode_p_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ streams, int count,
                                                                    const uint8_t* __restrict__ frames, const uint32_t* __restrict__ base_pics,
                                                                    const uint32_t* __restrict__ n_pics, const uint32_t* __restrict__ mbinfo, int qscale_all,
                                                                    const uint8_t* __restrict__ qpic, uint32_t* __restrict__ slots, uint32_t* __restrict__ slice_len)
{
    __shared__ uint32_t s_ac[32 * 41];
    __shared__ int s_t[kEncWarps][64], s_f[kEncWarps][64];
    __shared__ uint32_t s_win[kEncWarps][kWin + 2];
    for (int i = threadIdx.x; i < 32 * 41; i += blockDim.x) s_ac[i] = c_trick.ac[i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * kEncWarps + warp;
    if (gw >= count * EF_MBH_MAX) return;
    const int k = gw / EF_MBH_MAX, row = gw % EF_MBH_MAX;
    const int qv = qpic ? (int)qpic[k] : qscale_all, qscale = qv & 31;
    const bool fallback = qv & kQFallback;               // every macroblock not coded: vector (0, 0), no levels
    const int s = (int)streams[k];
    const uint8_t* ref = frames + ef_frame_offset(s, (int)((base_pics[s] + n_pics[s]) & 1u));
    const uint8_t* frame = src + (size_t)k * EF_FRAME;
    const uint32_t* info_row = mbinfo + (size_t)k * EF_MBW_MAX * EF_MBH_MAX + row * EF_MBW_MAX;
    uint32_t* out = slots + (size_t)gw * (kEncSliceBytes / 4);
    uint32_t* win = s_win[warp];
    int* T = s_t[warp];
    int* F = s_f[warp];
    for (int i = lane; i < kWin + 2; i += 32) win[i] = 0;
    __syncwarp();
    if (lane == 0) { win[0] = 0x00000100u | (uint32_t)(row + 1); win[1] = (uint32_t)qscale << 27; }
    uint32_t P = 38, wbase = 0;
    int pred[3] = { 128, 128, 128 }, mvp[2] = { 0, 0 }, pending = 0;
    const int r = lane >> 2, k0 = (lane & 3) * 2;
    auto flush = [&]() {                                 // the complete words out, the partial one kept
        __syncwarp();
        const uint32_t full = (P >> 5) - wbase;
        for (uint32_t i = lane; i < full; i += 32) out[wbase + i] = __byte_perm(win[i], 0, 0x0123);
        __syncwarp();
        const uint32_t carry = win[full];
        __syncwarp();
        for (int i = lane; i < kWin + 2; i += 32) win[i] = 0;
        __syncwarp();
        if (lane == 0) win[0] = carry;
        wbase += full;
    };
    for (int mx = 0; mx < EF_MBW_MAX; mx++) {
        const uint32_t info = fallback ? 0u : info_row[mx];
        const bool intra = (info >> 16) & 1;
        const int h = (int8_t)(info & 0xFF), v = (int8_t)((info >> 8) & 0xFF);
        const uint8_t* tile = frame + ef_tile_offset(mx, row);
        int lv0[6], lv1[6];
        uint32_t cbp = intra ? 63u : 0u;
        #pragma unroll
        for (int b = 0; b < 6; b++) {
            const int po = b < 4 ? ((b >> 1) * 8 + r) * 16 + (b & 1) * 8 : 256 + (b - 4) * 64 + r * 8;
            const uint2 px = *(const uint2*)(tile + po);
            int x[8];
            #pragma unroll
            for (int n = 0; n < 4; n++) { x[n] = (px.x >> (8 * n)) & 0xFF; x[n + 4] = (px.y >> (8 * n)) & 0xFF; }
            if (!intra) {                                // minus the prediction of row r of block b
                if (b < 4) {
                    const int X = 2 * (mx * 16 + (b & 1) * 8) + h, Y = 2 * (row * 16 + (b >> 1) * 8 + r) + v;
                    const int x0 = X >> 1, y0 = Y >> 1, xh = X & 1, yh = Y & 1;
                    #pragma unroll
                    for (int n = 0; n < 8; n++)
                        x[n] -= mc_pel(ref + ef_luma_offset(x0 + n, y0), ref + ef_luma_offset(x0 + n + xh, y0), ref + ef_luma_offset(x0 + n, y0 + yh),
                                       ref + ef_luma_offset(x0 + n + xh, y0 + yh), xh, yh);
                } else {                                 // quirk Q3: the chroma position is the floor of the halved luma vector
                    const int hx = (32 * mx + h) >> 1, hy = (32 * row + v) >> 1, p = b - 4;
                    const int x0 = hx >> 1, y0 = (hy >> 1) + r, xh = hx & 1, yh = hy & 1;
                    #pragma unroll
                    for (int n = 0; n < 8; n++)
                        x[n] -= mc_pel(ref + ef_chroma_offset(p, x0 + n, y0), ref + ef_chroma_offset(p, x0 + n + xh, y0),
                                       ref + ef_chroma_offset(p, x0 + n, y0 + yh), ref + ef_chroma_offset(p, x0 + n + xh, y0 + yh), xh, yh);
                }
            }
            fdct_block(x, T, F, r, k0);
            lv0[b] = intra ? quant(2 * lane, F, qscale) : quant_inter(2 * lane, F, qscale);
            lv1[b] = intra ? quant(2 * lane + 1, F, qscale) : quant_inter(2 * lane + 1, F, qscale);
            if (fallback) lv0[b] = lv1[b] = 0;
            if (!intra && __any_sync(0xFFFFFFFFu, lv0[b] != 0 || lv1[b] != 0)) cbp |= 0x20u >> b;
            __syncwarp();
        }
        const bool zero = h == 0 && v == 0;
        if (!intra && zero && !cbp && mx > 0 && mx < EF_MBW_MAX - 1) { pending++; continue; }
        if (pending) { pred[0] = pred[1] = pred[2] = 128; mvp[0] = mvp[1] = 0; }
        // macroblock header: increment, type, vector, pattern (warp-uniform lengths, lane 0 writes)
        uint32_t e = c_enc.mba[pending + 1];
        if (lane == 0) put_bits(win, P - wbase * 32, e >> 8, e & 0xFF);
        P += e & 0xFF;
        pending = 0;
        const int type = intra ? 0x01 : !zero ? (cbp ? 0x0A : 0x08) : (cbp ? 0x02 : 0x08);
        e = c_enc.type[type];
        if (lane == 0) put_bits(win, P - wbase * 32, e >> 8, e & 0xFF);
        P += e & 0xFF;
        if (intra) mvp[0] = mvp[1] = 0;
        else {
            pred[0] = pred[1] = pred[2] = 128;
            if (type & 0x08) {
                #pragma unroll
                for (int c = 0; c < 2; c++) {
                    const int val = c ? v : h;
                    int d = val - mvp[c];
                    d = d < -16 ? d + 32 : d > 15 ? d - 32 : d;
                    e = c_enc.mv[d + 16];
                    if (lane == 0) put_bits(win, P - wbase * 32, e >> 8, e & 0xFF);
                    P += e & 0xFF;
                    mvp[c] = val;
                }
            } else mvp[0] = mvp[1] = 0;
            if (type & 0x02) {
                e = c_enc.cbp[cbp];
                if (lane == 0) put_bits(win, P - wbase * 32, e >> 8, e & 0xFF);
                P += e & 0xFF;
            }
        }
        flush();
        #pragma unroll
        for (int b = 0; b < 6; b++) {
            if (!(cbp & (0x20u >> b))) continue;
            const int a0 = lv0[b], a1 = lv1[b];
            const uint32_t ev = __ballot_sync(0xFFFFFFFFu, (intra && lane == 0) || a0 != 0), od = __ballot_sync(0xFFFFFFFFu, a1 != 0);
            const uint64_t mask = spread_bits(ev) | (spread_bits(od) << 1);
            uint32_t c0, n0, c1, n1;
            code_of(2 * lane, a0, mask, s_ac, &c0, &n0);
            code_of(2 * lane + 1, a1, mask, s_ac, &c1, &n1);
            if (lane == 0) {
                if (intra) {                             // DC difference: size code, then the difference bits
                    const int comp = b < 4 ? 0 : b - 3;
                    const int diff = a0 - pred[comp], a = diff < 0 ? -diff : diff;
                    const uint32_t size = 32 - __clz(a);
                    const uint32_t d = c_trick.dc[comp ? 1 : 0][size];
                    c0 = ((d >> 8) << size) | (uint32_t)(diff > 0 ? diff : diff + (1 << size) - 1);
                    n0 = (d & 0xFF) + size;
                } else if (a0 == 1 || a0 == -1) { c0 = 2u | (a0 < 0 ? 1u : 0u); n0 = 2; }    // the first coefficient's "1s"
                else if (a0) code_of(1, a0, 1, s_ac, &c0, &n0);   // run 0 (index 1 after a coded index 0): the table or an escape
            }
            if (intra) pred[b < 4 ? 0 : b - 3] = __shfl_sync(0xFFFFFFFFu, a0, 0);
            const uint32_t sum = n0 + n1;
            uint32_t incl = sum;
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
                if (lane >= d) incl += t;
            }
            const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
            const uint32_t q = P - wbase * 32 + incl - sum;
            put_bits(win, q, c0, n0);
            put_bits(win, q + n0, c1, n1);
            if (lane == 0) put_bits(win, P - wbase * 32 + total, 2u, 2);     // end of block "10"
            P += total + 2;
            flush();
        }
    }
    __syncwarp();
    const uint32_t words = ((P + 31) >> 5) - wbase;
    for (uint32_t i = lane; i < words; i += 32) out[wbase + i] = __byte_perm(win[i], 0, 0x0123);
    if (lane == 0) slice_len[gw] = (P + 7) >> 3;
}

// the exact bytes of slice `row` of picture k of the round coded at every candidate q = qmin + lane (lane < nq) and as its fallback
// (lane kCensusFallback): census[(k * 32 + lane) * 12 + row]. One warp per slice; the FDCT of a block does not depend on q, so each
// block is transformed once and then quantised and its codes counted at every candidate, the lanes splitting the coefficients as
// ef_encode_p_kernel does. Lane q then walks the slice's macroblock headers for its own q: address increments and skips (they depend
// on q through the coded block pattern), the predictor resets, vector, type and pattern codes, DC differences. ipic: the round's
// pictures are I pictures (every macroblock intra, the trick encoder's 2-bit header); else P pictures with their search's mbinfo.
__global__ void __launch_bounds__(kEncWarps * 32) ef_encode_census_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ streams, int count,
                                                                         const uint8_t* __restrict__ frames, const uint32_t* __restrict__ base_pics,
                                                                         const uint32_t* __restrict__ n_pics, const uint32_t* __restrict__ mbinfo, int ipic,
                                                                         int qmin, int nq, uint32_t* __restrict__ census)
{
    __shared__ uint32_t s_ac[32 * 41];
    __shared__ int s_t[kEncWarps][64], s_f[kEncWarps][64];
    for (int i = threadIdx.x; i < 32 * 41; i += blockDim.x) s_ac[i] = c_trick.ac[i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * kEncWarps + warp;
    if (gw >= count * EF_MBH_MAX) return;
    const int k = gw / EF_MBH_MAX, row = gw % EF_MBH_MAX;
    const uint8_t* frame = src + (size_t)k * EF_FRAME;
    const uint8_t* ref = nullptr;
    const uint32_t* info_row = nullptr;
    if (!ipic) {
        const int s = (int)streams[k];
        ref = frames + ef_frame_offset(s, (int)((base_pics[s] + n_pics[s]) & 1u));
        info_row = mbinfo + (size_t)k * EF_MBW_MAX * EF_MBH_MAX + row * EF_MBW_MAX;
    }
    int* T = s_t[warp];
    int* F = s_f[warp];
    const int r = lane >> 2, k0 = (lane & 3) * 2;
    const bool fb_lane = lane == kCensusFallback;
    const int my_q = qmin + lane;                        // this lane's candidate (lanes nq .. 30 count nothing of use)
    uint32_t P = 38;
    int pred[3] = { 128, 128, 128 }, mvp[2] = { 0, 0 }, pending = 0;
    for (int mx = 0; mx < EF_MBW_MAX; mx++) {
        const uint32_t info = ipic ? (1u << 16) : info_row[mx];
        const bool intra = (info >> 16) & 1;
        const int h = (int8_t)(info & 0xFF), v = (int8_t)((info >> 8) & 0xFF);
        const uint8_t* tile = frame + ef_tile_offset(mx, row);
        uint32_t cbp = 0, blk = 0;                       // this lane's q: coded blocks, their run / level and end-of-block bits
        int dcl[6];
        #pragma unroll 1
        for (int b = 0; b < 6; b++) {
            const int po = b < 4 ? ((b >> 1) * 8 + r) * 16 + (b & 1) * 8 : 256 + (b - 4) * 64 + r * 8;
            const uint2 px = *(const uint2*)(tile + po);
            int x[8];
            #pragma unroll
            for (int n = 0; n < 4; n++) { x[n] = (px.x >> (8 * n)) & 0xFF; x[n + 4] = (px.y >> (8 * n)) & 0xFF; }
            if (!intra) {
                if (b < 4) {
                    const int X = 2 * (mx * 16 + (b & 1) * 8) + h, Y = 2 * (row * 16 + (b >> 1) * 8 + r) + v;
                    const int x0 = X >> 1, y0 = Y >> 1, xh = X & 1, yh = Y & 1;
                    #pragma unroll
                    for (int n = 0; n < 8; n++)
                        x[n] -= mc_pel(ref + ef_luma_offset(x0 + n, y0), ref + ef_luma_offset(x0 + n + xh, y0), ref + ef_luma_offset(x0 + n, y0 + yh),
                                       ref + ef_luma_offset(x0 + n + xh, y0 + yh), xh, yh);
                } else {
                    const int hx = (32 * mx + h) >> 1, hy = (32 * row + v) >> 1, p = b - 4;
                    const int x0 = hx >> 1, y0 = (hy >> 1) + r, xh = hx & 1, yh = hy & 1;
                    #pragma unroll
                    for (int n = 0; n < 8; n++)
                        x[n] -= mc_pel(ref + ef_chroma_offset(p, x0 + n, y0), ref + ef_chroma_offset(p, x0 + n + xh, y0),
                                       ref + ef_chroma_offset(p, x0 + n, y0 + yh), ref + ef_chroma_offset(p, x0 + n + xh, y0 + yh), xh, yh);
                }
            }
            fdct_block(x, T, F, r, k0);
            dcl[b] = intra ? quant(0, F, 1) : 0;         // an intra DC level does not depend on q
            // every candidate, lowest first; levels only shrink as q grows, so once a block has no level left (intra: no AC
            // level) it has none at any later candidate
            int qi = 0;
            for (; qi < nq; qi++) {
                const int q = qmin + qi;
                const int a0 = intra ? (lane ? quant(2 * lane, F, q) : 0) : quant_inter(2 * lane, F, q);
                const int a1 = intra ? quant(2 * lane + 1, F, q) : quant_inter(2 * lane + 1, F, q);
                const uint32_t ev = __ballot_sync(0xFFFFFFFFu, (intra && lane == 0) || a0 != 0), od = __ballot_sync(0xFFFFFFFFu, a1 != 0);
                if (!(od | (intra ? ev & ~1u : ev))) break;
                const uint64_t mask = spread_bits(ev) | (spread_bits(od) << 1);
                uint32_t c0, n0, c1, n1;
                code_of(2 * lane, a0, mask, s_ac, &c0, &n0);
                code_of(2 * lane + 1, a1, mask, s_ac, &c1, &n1);
                if (lane == 0 && !intra) {
                    if (a0 == 1 || a0 == -1) n0 = 2;
                    else if (a0) code_of(1, a0, 1, s_ac, &c0, &n0);
                }
                const uint32_t bits = (uint32_t)__reduce_add_sync(0xFFFFFFFFu, (int)(n0 + n1));
                if (lane == qi) { blk += bits + 2; cbp |= 0x20u >> b; }
            }
            if (intra && lane >= qi && !fb_lane) { blk += 2; cbp |= 0x20u >> b; }
            __syncwarp();
        }
        // the fallback: P every macroblock not coded; I the DC levels and end of block of every block
        const bool my_intra = intra && !(fb_lane && !ipic);
        const bool zero = (h == 0 && v == 0) || fb_lane;
        if (fb_lane) { cbp = ipic ? 63u : 0u; blk = ipic ? 12u : 0u; }
        if (!my_intra && zero && !cbp && mx > 0 && mx < EF_MBW_MAX - 1) { pending++; continue; }
        if (pending) { pred[0] = pred[1] = pred[2] = 128; mvp[0] = mvp[1] = 0; }
        P += c_enc.mba[pending + 1] & 0xFF;
        pending = 0;
        const int type = my_intra ? 0x01 : !zero ? (cbp ? 0x0A : 0x08) : (cbp ? 0x02 : 0x08);
        P += ipic ? 1 : c_enc.type[type] & 0xFF;
        if (my_intra) {
            mvp[0] = mvp[1] = 0;
            #pragma unroll
            for (int b = 0; b < 6; b++) {
                const int comp = b < 4 ? 0 : b - 3;
                const int diff = dcl[b] - pred[comp], size = 32 - __clz(diff < 0 ? -diff : diff);
                P += (c_trick.dc[comp ? 1 : 0][size] & 0xFF) + size;
                pred[comp] = dcl[b];
            }
        } else {
            pred[0] = pred[1] = pred[2] = 128;
            if (type & 0x08) {
                #pragma unroll
                for (int c = 0; c < 2; c++) {
                    const int val = fb_lane ? 0 : c ? v : h;
                    int d = val - mvp[c];
                    d = d < -16 ? d + 32 : d > 15 ? d - 32 : d;
                    P += c_enc.mv[d + 16] & 0xFF;
                    mvp[c] = val;
                }
            } else mvp[0] = mvp[1] = 0;
            if (type & 0x02) P += c_enc.cbp[cbp] & 0xFF;
        }
        P += blk;
    }
    if (lane < nq || fb_lane) census[((size_t)k * 32 + lane) * EF_MBH_MAX + row] = (P + 7) >> 3;
}

// one thread per GOP of the round: the GOP's bucket (fullness in 1/90000 bit, bucket[g]) and the choice of picture j's quantiser from
// the census (tests/rate_cases.py): the smallest candidate within the soft target and the hard bound, else the smallest within the
// hard bound, else the fallback. gop_n[g] = pictures of GOP g | 1 << 16 when it is its title's last (it must end at 0, not full).
// qpic[k] receives the choice, pic_bytes[k] its ES bytes.
__global__ void ef_encode_choose_kernel(const uint32_t* __restrict__ census, const uint32_t* __restrict__ streams, int count, int j, int qmin, int nq,
                                        int qmax, EfRateBucket rb, const uint32_t* __restrict__ gop_n, int64_t* __restrict__ bucket,
                                        uint8_t* __restrict__ qpic, uint32_t* __restrict__ pic_bytes)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const int g = (int)streams[k];
    const int n = (int)(gop_n[g] & 0xFFFF);
    const int64_t E = (gop_n[g] >> 16) ? 0 : rb.full;
    int64_t need = E;                                    // need_{j + 1}: every picture after j is a P picture
    for (int m = n - 1; m > j; m--) need = max(rb.fb_p, rb.fb_p + need - rb.r);
    const int64_t f = j ? bucket[g] : rb.full;
    const int64_t hard = min(f, f + rb.r - need);
    const int64_t L = f + (int64_t)(n - j) * rb.r - E;
    const int64_t soft = j ? L / (n - j) : L * kIWeight / (kIWeight + n - 1);
    const uint32_t hb = j ? kEncPHeaderBytes : kTrickHeaderBytes;
    const uint32_t* c = census + (size_t)k * 32 * EF_MBH_MAX;
    auto bytes = [&](int slot) {
        uint32_t s = hb;
        for (int row = 0; row < EF_MBH_MAX; row++) s += c[slot * EF_MBH_MAX + row];
        return s;
    };
    int pick = -1;
    uint32_t s = 0;
    for (int pass = 0; pass < 2 && pick < 0; pass++) {
        const int64_t cap = pass ? hard : min(soft, hard);
        for (int qi = 0; qi < nq; qi++) {
            s = bytes(qi);
            if ((int64_t)s * 8 * kRateUnit <= cap) { pick = qi; break; }
        }
    }
    if (pick < 0) s = bytes(kCensusFallback);
    qpic[k] = (uint8_t)(pick < 0 ? (qmax | kQFallback) : qmin + pick);
    pic_bytes[k] = s;
    bucket[g] = min(rb.full, f - (int64_t)s * 8 * kRateUnit + rb.r);
}

// one CTA per P picture: the round's header (all pictures of a round share their temporal reference), then its 12 slices
__global__ void ef_encode_assemble_kernel(const uint32_t* __restrict__ slots, const uint32_t* __restrict__ slice_len, const uint64_t* __restrict__ pic_dst,
                                          const uint8_t* __restrict__ header, uint8_t* __restrict__ es)
{
    const int p = blockIdx.x;
    __shared__ uint32_t off[EF_MBH_MAX + 1];
    if (threadIdx.x == 0) {
        off[0] = kEncPHeaderBytes;
        for (int s = 0; s < EF_MBH_MAX; s++) off[s + 1] = off[s] + slice_len[p * EF_MBH_MAX + s];
    }
    __syncthreads();
    uint8_t* dst = es + pic_dst[p];
    for (int i = threadIdx.x; i < kEncPHeaderBytes; i += blockDim.x) dst[i] = header[i];
    for (int s = 0; s < EF_MBH_MAX; s++) {
        const uint8_t* src = (const uint8_t*)(slots + (size_t)(p * EF_MBH_MAX + s) * (kEncSliceBytes / 4));
        const uint32_t n = off[s + 1] - off[s];
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[off[s] + i] = src[i];
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------------------------
cudaError_t ef_encode_upload_tables()
{
    cudaError_t e = upload_trick_tables();
    if (e != cudaSuccess) return e;
    EncTables t;
    memset(&t, 0, sizeof(t));
    for (int i = 0; i < EF_VLC_MBA_COUNT; i++) if (ef_vlc_mba[i].value >= 1 && ef_vlc_mba[i].value <= 33) t.mba[ef_vlc_mba[i].value] = vlc_entry(ef_vlc_mba[i].code);
    for (int i = 0; i < EF_VLC_MBTYPE_P_COUNT; i++) t.type[ef_vlc_mbtype_p[i].value] = vlc_entry(ef_vlc_mbtype_p[i].code);
    for (int i = 0; i < EF_VLC_MV_COUNT; i++) t.mv[ef_vlc_mv[i].value + 16] = vlc_entry(ef_vlc_mv[i].code);
    for (int i = 0; i < EF_VLC_CBP_COUNT; i++) t.cbp[ef_vlc_cbp[i].value] = vlc_entry(ef_vlc_cbp[i].code);
    return cudaMemcpyToSymbol(c_enc, &t, sizeof(t));
}

cudaError_t ef_encode_launch_tile(const uint8_t* i420, const uint32_t* src, int count, uint8_t* tiled, cudaStream_t st)
{
    if (!count) return cudaSuccess;
    const uint64_t threads = (uint64_t)count * (EF_FRAME / 16);
    ef_encode_tile_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(i420, src, count, tiled);
    return cudaGetLastError();
}

cudaError_t ef_encode_launch_search(const uint8_t* src, const uint32_t* streams, int count, const uint8_t* frames, const uint32_t* base_pics,
                                    const uint32_t* n_pics, int search, uint32_t* mbinfo, cudaStream_t st)
{
    const int warps = count * EF_MBW_MAX * EF_MBH_MAX;
    ef_encode_search_kernel<<<(warps + kEncWarps - 1) / kEncWarps, kEncWarps * 32, 0, st>>>(src, streams, count, frames, base_pics, n_pics, search, mbinfo);
    return cudaGetLastError();
}

cudaError_t ef_encode_launch_p(const uint8_t* src, const uint32_t* streams, int count, const uint8_t* frames, const uint32_t* base_pics,
                               const uint32_t* n_pics, const uint32_t* mbinfo, int qscale, const uint8_t* qpic, uint32_t* slots, uint32_t* slice_len,
                               cudaStream_t st)
{
    const int warps = count * EF_MBH_MAX;
    ef_encode_p_kernel<<<(warps + kEncWarps - 1) / kEncWarps, kEncWarps * 32, 0, st>>>(src, streams, count, frames, base_pics, n_pics, mbinfo, qscale,
                                                                                      qpic, slots, slice_len);
    return cudaGetLastError();
}

cudaError_t ef_encode_launch_census(const uint8_t* src, const uint32_t* streams, int count, const uint8_t* frames, const uint32_t* base_pics,
                                    const uint32_t* n_pics, const uint32_t* mbinfo, int ipic, int qmin, int nq, uint32_t* census, cudaStream_t st)
{
    const int warps = count * EF_MBH_MAX;
    ef_encode_census_kernel<<<(warps + kEncWarps - 1) / kEncWarps, kEncWarps * 32, 0, st>>>(src, streams, count, frames, base_pics, n_pics, mbinfo, ipic,
                                                                                           qmin, nq, census);
    return cudaGetLastError();
}

cudaError_t ef_encode_launch_choose(const uint32_t* census, const uint32_t* streams, int count, int j, int qmin, int qmax, const EfRateBucket& rb,
                                    const uint32_t* gop_n, int64_t* bucket, uint8_t* qpic, uint32_t* pic_bytes, cudaStream_t st)
{
    ef_encode_choose_kernel<<<(count + 127) / 128, 128, 0, st>>>(census, streams, count, j, qmin, qmax - qmin + 1, qmax, rb, gop_n, bucket, qpic,
                                                                 pic_bytes);
    return cudaGetLastError();
}

cudaError_t ef_encode_launch_assemble(const uint32_t* slots, const uint32_t* slice_len, const uint64_t* pic_dst, const uint8_t* header, int n_pics,
                                      uint8_t* es, cudaStream_t st)
{
    ef_encode_assemble_kernel<<<n_pics, 256, 0, st>>>(slots, slice_len, pic_dst, header, es);
    return cudaGetLastError();
}
