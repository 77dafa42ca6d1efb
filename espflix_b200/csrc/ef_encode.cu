// csrc/ef_encode.cu — the picture encoders, every kernel that codes MPEG-1 pictures: a title's video.ts encoded on the device from
// raw pictures (what the reference's indexer makes with ffmpeg, make_video(), indexer/indexer.cpp:306) and the intra pictures of the
// trick streams (its two re-encodes, indexer.cpp:308-309). A title's GOPs are an I picture and P pictures predicted from the
// decoder's own reconstruction of the picture before them (the frame store K1b wrote). The rules, byte for byte, are
// tests/encode_cases.py, tests/rate_cases.py and tests/trick_cases.py; the host sides are ef_encode_build and ef_trick_build in
// ef_capi.cu. Kernels:
//   ef_encode_tile_kernel      I420 pictures -> the macroblock-tiled frame layout, one 16-byte store per thread
//   ef_encode_search_kernel    one warp per macroblock: the source macroblock and the reference window in shared memory, full-pel
//                              candidates split over the lanes (packed SADs, one warp minimum at the end), then the 3 x 3 half-pel
//                              neighbours and the intra decision
//   ef_encode_slice_kernel     one warp per slice (macroblock row) of an I picture (every macroblock intra, coded block by block) or
//                              a P picture (its search's mbinfo; the six blocks quantised before the header for the coded block
//                              pattern): prediction, FDCT, quantiser, codes placed by a warp prefix sum in a shared window, flushed
//                              to a per-slice region of kTrickSliceBytes
//   ef_encode_census_kernel    ef_encode_build_rate: one warp per slice, the slice's exact bytes at every candidate quantiser and as
//                              its fallback, from one FDCT per block, with the slice coder's own pieces
//   ef_encode_choose_kernel    ef_encode_build_rate: one thread per GOP, its bucket and the choice of the picture's quantiser
//   ef_encode_assemble_kernel  one CTA per picture: its header and its 12 slices at the picture's offset in the ES
#include <stdint.h>
#include <string.h>

#include "ef_common.cuh"
#include "ef_iso11172_tables.h"

namespace {

constexpr int kEncWarps = 4;
constexpr int kZeroBias = 64;        // tests/encode_cases.ZERO_BIAS
constexpr int kIntraMargin = 512;    // tests/encode_cases.INTRA_MARGIN
constexpr int kWinW = 10, kWinH = 33;   // reference window: 33 rows of 40 bytes from (16 mx - 8, 16 my - 8)

// FDCT_C of tests/trick_cases.py: round(4096 c_k cos((2n + 1) k pi / 16)); rows sum to at most 11,585 in magnitude, so with pixels
// 0..255 the row pass stays below 2^22 and the column pass below 2^28 (int32); residuals of -255..255 keep the same bounds.
__constant__ int c_fdct[64] = {
    1448, 1448, 1448, 1448, 1448, 1448, 1448, 1448,
    2009, 1703, 1138, 400, -400, -1138, -1703, -2009,
    1892, 784, -784, -1892, -1892, -784, 784, 1892,
    1703, -400, -2009, -1138, 1138, 2009, 400, -1703,
    1448, -1448, -1448, 1448, 1448, -1448, -1448, 1448,
    1138, -2009, 400, 1703, -1703, -400, 2009, -1138,
    784, -1892, 1892, -784, -784, 1892, -1892, 784,
    400, -1138, 1703, -2009, 2009, -1703, 1138, -400,
};

struct CodeTables {            // filled by ef_encode_upload_tables()
    uint32_t ac[32 * 41];      // run 0..31 x level 0..40: (code << 8) | length, without the sign bit; 0 = escape
    uint32_t dc[2][9];         // luma / chroma dct_dc_size: (code << 8) | length
    uint8_t zz[64];            // zig-zag index -> raster index
    uint8_t q[64];             // default intra matrix, raster index
    uint32_t mba[34];          // macroblock_address_increment 1..33: (code << 8) | length
    uint32_t type[32];         // P macroblock_type value -> (code << 8) | length
    uint32_t mv[33];           // motion code -16..16 at [code + 16] (f_code 1: no residual bits)
    uint32_t cbp[64];          // coded_block_pattern 1..63
};
__constant__ CodeTables c_tab;

constexpr int kWin = 64;       // window words: one block's codes (intra at most 1,784 bits, non-intra 1,794) plus 31 carried bits
static_assert(kWin * 32 >= 31 + 2 + 16 + 63 * 28 + 2, "window holds an intra macroblock header and a worst-case intra block");
static_assert(kWin * 32 >= 31 + 64 * 28 + 2, "window holds a worst-case non-intra block");

__device__ __forceinline__ void put_bits(uint32_t* win, uint32_t q, uint32_t code, uint32_t len)
{
    if (!len) return;
    const uint32_t w = q >> 5, off = q & 31;
    if (off + len <= 32) atomicOr(&win[w], code << (32 - off - len));
    else {
        atomicOr(&win[w], code >> (off + len - 32));
        atomicOr(&win[w + 1], code << (64 - off - len));
    }
}

__device__ __forceinline__ void code_of(int i, int lv, uint64_t mask, const uint32_t* ac, uint32_t* code, uint32_t* len)
{
    *code = 0; *len = 0;
    if (i == 0 || lv == 0) return;
    const int prev = 63 - __clzll((long long)(mask & ((1ull << i) - 1)));
    const int run = i - prev - 1, a = lv < 0 ? -lv : lv;
    const uint32_t e = (a <= 40 && run <= 31) ? ac[run * 41 + a] : 0u;
    if (e & 0xFF) { *code = ((e >> 8) << 1) | (lv < 0 ? 1u : 0u); *len = (e & 0xFF) + 1; return; }
    uint32_t L, bits;
    if (lv >= -127 && lv <= 127) { L = 8; bits = (uint32_t)lv & 0xFF; }
    else if (lv > 0) { L = 16; bits = (uint32_t)lv; }
    else { L = 16; bits = (128u << 8) | ((uint32_t)(lv + 256) & 0xFF); }
    *code = (1u << (6 + L)) | ((uint32_t)run << L) | bits;
    *len = 12 + L;
}

// bit i of m -> bit 2 i
__device__ __forceinline__ uint64_t spread_bits(uint32_t m)
{
    uint64_t x = m;
    x = (x | (x << 16)) & 0x0000FFFF0000FFFFull;
    x = (x | (x << 8)) & 0x00FF00FF00FF00FFull;
    x = (x | (x << 4)) & 0x0F0F0F0F0F0F0F0Full;
    x = (x | (x << 2)) & 0x3333333333333333ull;
    return (x | (x << 1)) & 0x5555555555555555ull;
}

__device__ __forceinline__ int quant(int i, const int* F, int qscale)
{
    const int z = c_tab.zz[i], f = F[z];
    if (i == 0) { const int dc = (f + 4) >> 3; return dc > 255 ? 255 : dc; }
    const int den = qscale * c_tab.q[z], num = 8 * (f < 0 ? -f : f);
    int lv = (2 * num + den) / (2 * den);
    lv = lv > 255 ? 255 : lv;
    return f < 0 ? -lv : lv;
}

__device__ __forceinline__ int quant_inter(int i, const int* F, int qscale)
{
    const int f = F[c_tab.zz[i]], a = (8 * (f < 0 ? -f : f)) / (16 * qscale);
    const int lv = a > 255 ? 255 : a;
    return f < 0 ? -lv : lv;
}

// FDCT of one 8 x 8 block by a warp: lane = (row r, outputs k0, k0 + 1) holds the samples x of row r; T and F are the warp's
// 64-entry scratch, F receives the coefficients (raster)
__device__ __forceinline__ void fdct_block(const int (&x)[8], int* T, int* F, int r, int k0)
{
    #pragma unroll
    for (int kk = 0; kk < 2; kk++) {
        int acc = 0;
        #pragma unroll
        for (int n = 0; n < 8; n++) acc += c_fdct[(k0 + kk) * 8 + n] * x[n];
        T[r * 8 + k0 + kk] = (acc + 128) >> 8;
    }
    __syncwarp();
    // column pass: lane = (column r, outputs k0, k0 + 1)
    #pragma unroll
    for (int kk = 0; kk < 2; kk++) {
        int acc = 0;
        #pragma unroll
        for (int n = 0; n < 8; n++) acc += c_fdct[(k0 + kk) * 8 + n] * T[n * 8 + r];
        F[(k0 + kk) * 8 + r] = (acc + 32768) >> 16;
    }
    __syncwarp();
}

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

// the frame store that holds the decoder's latest picture of stream s: the reference of the picture predicted from it
__device__ __forceinline__ const uint8_t* latest_frame(const uint8_t* frames, const uint32_t* base_pics, const uint32_t* n_pics, int s)
{
    return frames + ef_frame_offset(s, (int)((base_pics[s] + n_pics[s]) & 1u));
}

// the samples of row r of block b (0..3 luma, 4 Cb, 5 Cr) of a macroblock tile
__device__ __forceinline__ void load_row(const uint8_t* tile, int b, int r, int (&x)[8])
{
    const int po = b < 4 ? ((b >> 1) * 8 + r) * 16 + (b & 1) * 8 : 256 + (b - 4) * 64 + r * 8;
    const uint2 px = *(const uint2*)(tile + po);
    #pragma unroll
    for (int n = 0; n < 4; n++) { x[n] = (px.x >> (8 * n)) & 0xFF; x[n + 4] = (px.y >> (8 * n)) & 0xFF; }
}

// x minus the prediction of row r of block b of macroblock (mx, my) from ref at the half-pel vector (h, v)
__device__ __forceinline__ void sub_prediction(const uint8_t* ref, int mx, int my, int b, int r, int h, int v, int (&x)[8])
{
    if (b < 4) {
        const int X = 2 * (mx * 16 + (b & 1) * 8) + h, Y = 2 * (my * 16 + (b >> 1) * 8 + r) + v;
        const int x0 = X >> 1, y0 = Y >> 1, xh = X & 1, yh = Y & 1;
        #pragma unroll
        for (int n = 0; n < 8; n++)
            x[n] -= mc_pel(ref + ef_luma_offset(x0 + n, y0), ref + ef_luma_offset(x0 + n + xh, y0), ref + ef_luma_offset(x0 + n, y0 + yh),
                           ref + ef_luma_offset(x0 + n + xh, y0 + yh), xh, yh);
    } else {                                             // quirk Q3: the chroma position is the floor of the halved luma vector
        const int hx = (32 * mx + h) >> 1, hy = (32 * my + v) >> 1, p = b - 4;
        const int x0 = hx >> 1, y0 = (hy >> 1) + r, xh = hx & 1, yh = hy & 1;
        #pragma unroll
        for (int n = 0; n < 8; n++)
            x[n] -= mc_pel(ref + ef_chroma_offset(p, x0 + n, y0), ref + ef_chroma_offset(p, x0 + n + xh, y0),
                           ref + ef_chroma_offset(p, x0 + n, y0 + yh), ref + ef_chroma_offset(p, x0 + n + xh, y0 + yh), xh, yh);
    }
}

// The coded indices of a block whose lanes hold the levels a0, a1 of zig-zag indices 2 lane, 2 lane + 1 (bit i: index i); an intra
// block's DC counts as coded
__device__ __forceinline__ uint64_t level_mask(int lane, int a0, int a1, bool intra)
{
    const uint32_t ev = __ballot_sync(0xFFFFFFFFu, (intra && lane == 0) || a0 != 0), od = __ballot_sync(0xFFFFFFFFu, a1 != 0);
    return spread_bits(ev) | (spread_bits(od) << 1);
}

// the run / level codes of this lane's two indices; a non-intra block's first coefficient by its own rule. Lane 0's first code of an
// intra block is its DC difference (dc_code).
__device__ __forceinline__ void ac_codes(int lane, int a0, int a1, bool intra, uint64_t mask, const uint32_t* ac, uint32_t* c0, uint32_t* n0,
                                         uint32_t* c1, uint32_t* n1)
{
    code_of(2 * lane, a0, mask, ac, c0, n0);
    code_of(2 * lane + 1, a1, mask, ac, c1, n1);
    if (lane == 0 && !intra) {
        if (a0 == 1 || a0 == -1) { *c0 = 2u | (a0 < 0 ? 1u : 0u); *n0 = 2; }   // the first coefficient's "1s"
        else if (a0) code_of(1, a0, 1, ac, c0, n0);     // run 0 (index 1 after a coded index 0): the table or an escape
    }
}

// an intra block's DC difference from its component's predictor: the size code, then the difference bits
__device__ __forceinline__ void dc_code(int comp, int diff, uint32_t* code, uint32_t* len)
{
    const int a = diff < 0 ? -diff : diff;
    const uint32_t size = 32 - __clz(a);
    const uint32_t e = c_tab.dc[comp ? 1 : 0][size];
    *code = ((e >> 8) << size) | (uint32_t)(diff > 0 ? diff : diff + (1 << size) - 1);
    *len = (e & 0xFF) + size;
}

// The header of macroblock mx of a slice, one walk for the coder (emit puts a code (code << 8) | length) and the census (emit adds
// its length): false when the macroblock is skipped (pending counts it), else its address increment, type, vector and pattern codes
// and the predictor resets. An I picture's macroblocks are all intra and none is skipped: increment 1 and type "1", 2 bits.
template <typename Emit>
__device__ __forceinline__ bool mb_header(bool ipic, int mx, bool intra, int h, int v, uint32_t cbp, int& pending, int (&pred)[3], int (&mvp)[2],
                                          Emit emit)
{
    if (ipic) { emit((3u << 8) | 2u); return true; }
    const bool zero = h == 0 && v == 0;
    if (!intra && zero && !cbp && mx > 0 && mx < EF_MBW_MAX - 1) { pending++; return false; }
    if (pending) { pred[0] = pred[1] = pred[2] = 128; mvp[0] = mvp[1] = 0; }
    emit(c_tab.mba[pending + 1]);
    pending = 0;
    const int type = intra ? 0x01 : !zero ? (cbp ? 0x0A : 0x08) : (cbp ? 0x02 : 0x08);
    emit(c_tab.type[type]);
    if (intra) { mvp[0] = mvp[1] = 0; return true; }
    pred[0] = pred[1] = pred[2] = 128;
    if (type & 0x08) {
        #pragma unroll
        for (int c = 0; c < 2; c++) {
            const int val = c ? v : h;
            int d = val - mvp[c];
            d = d < -16 ? d + 32 : d > 15 ? d - 32 : d;
            emit(c_tab.mv[d + 16]);
            mvp[c] = val;
        }
    } else mvp[0] = mvp[1] = 0;
    if (type & 0x02) emit(c_tab.cbp[cbp]);
    return true;
}

// A warp's slice being coded: bit P of the slice lies at bit P - 32 wbase of the shared window win (kWin + 2 words); the words before
// wbase are in out, the slice's region
struct SliceOut {
    uint32_t* win;
    uint32_t* out;
    uint32_t P, wbase;
    int lane;

    // the slice start code, the quantiser and the extra bit
    __device__ __forceinline__ SliceOut(uint32_t* win_, uint32_t* out_, int lane_, int row, int qscale) : win(win_), out(out_), P(38), wbase(0), lane(lane_)
    {
        for (int i = lane; i < kWin + 2; i += 32) win[i] = 0;
        __syncwarp();
        if (lane == 0) { win[0] = 0x00000100u | (uint32_t)(row + 1); win[1] = (uint32_t)qscale << 27; }
    }

    // a code of warp-uniform length, (code << 8) | length; lane 0 writes it
    __device__ __forceinline__ void put(uint32_t e)
    {
        if (lane == 0) put_bits(win, P - wbase * 32, e >> 8, e & 0xFF);
        P += e & 0xFF;
    }

    // one block's codes: levels a0, a1 of zig-zag indices 2 lane, 2 lane + 1, placed by a warp prefix sum, then the end of block; an
    // intra block's DC as its difference from pred[comp]
    __device__ __forceinline__ void block(int a0, int a1, bool intra, int comp, int (&pred)[3], const uint32_t* ac)
    {
        uint32_t c0, n0, c1, n1;
        ac_codes(lane, a0, a1, intra, level_mask(lane, a0, a1, intra), ac, &c0, &n0, &c1, &n1);
        if (intra) {
            if (lane == 0) dc_code(comp, a0 - pred[comp], &c0, &n0);
            pred[comp] = __shfl_sync(0xFFFFFFFFu, a0, 0);
        }
        const uint32_t sum = n0 + n1;
        const uint32_t incl = ef_warp_inclusive_scan(sum);
        const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
        const uint32_t q = P - wbase * 32 + incl - sum;
        put_bits(win, q, c0, n0);
        put_bits(win, q + n0, c1, n1);
        if (lane == 0) put_bits(win, P - wbase * 32 + total, 2u, 2);     // end of block "10"
        P += total + 2;
    }

    // the complete words out, the partial one kept
    __device__ __forceinline__ void flush()
    {
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
    }

    // the rest of the slice, which ends on a byte boundary, zero-padded; *len receives its bytes
    __device__ __forceinline__ void finish(uint32_t* len)
    {
        __syncwarp();
        const uint32_t words = ((P + 31) >> 5) - wbase;
        for (uint32_t i = lane; i < words; i += 32) out[wbase + i] = __byte_perm(win[i], 0, 0x0123);
        if (lane == 0) *len = (P + 7) >> 3;
    }
};

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
    const uint8_t* ref = latest_frame(frames, base_pics, n_pics, (int)streams[k]);
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

// Slice `row` of picture k of the list (tiled source src + k EF_FRAME), at the quantiser qpic[k] (or qscale_all without qpic), to
// slots + (k * 12 + row) kTrickSliceBytes and its bytes to slice_len[k * 12 + row]. A quantiser with kQFallback codes the fallback: an I
// picture's DC levels alone, a P picture with every macroblock not coded. An I picture codes each block as it is transformed; a P
// picture (predicted from the latest frame store of decoder stream streams[k], with mbinfo as ef_encode_search_kernel wrote it)
// quantises a macroblock's six blocks first, as its header carries their coded block pattern.
template <bool kIntraPicture>
__global__ void __launch_bounds__(kEncWarps * 32) ef_encode_slice_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ streams, int count,
                                                                        const uint8_t* __restrict__ frames, const uint32_t* __restrict__ base_pics,
                                                                        const uint32_t* __restrict__ n_pics, const uint32_t* __restrict__ mbinfo,
                                                                        int qscale_all, const uint8_t* __restrict__ qpic, uint32_t* __restrict__ slots,
                                                                        uint32_t* __restrict__ slice_len)
{
    __shared__ uint32_t s_ac[32 * 41];
    __shared__ int s_t[kEncWarps][64], s_f[kEncWarps][64];
    __shared__ uint32_t s_win[kEncWarps][kWin + 2];
    for (int i = threadIdx.x; i < 32 * 41; i += blockDim.x) s_ac[i] = c_tab.ac[i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * kEncWarps + warp;
    if (gw >= count * EF_MBH_MAX) return;
    const int k = gw / EF_MBH_MAX, row = gw % EF_MBH_MAX;
    const int qv = qpic ? (int)qpic[k] : qscale_all, qscale = qv & 31;
    const bool fallback = qv & kQFallback;
    const uint8_t* frame = src + (size_t)k * EF_FRAME;
    int* T = s_t[warp];
    int* F = s_f[warp];
    SliceOut w(s_win[warp], slots + (size_t)gw * (kTrickSliceBytes / 4), lane, row, qscale);
    int pred[3] = { 128, 128, 128 }, mvp[2] = { 0, 0 }, pending = 0;
    const int r = lane >> 2, k0 = (lane & 3) * 2;
    const auto put = [&](uint32_t e) { w.put(e); };
    if (kIntraPicture) {
        for (int mx = 0; mx < EF_MBW_MAX; mx++) {
            const uint8_t* tile = frame + ef_tile_offset(mx, row);
            __syncwarp();
            mb_header(true, mx, true, 0, 0, 63u, pending, pred, mvp, put);
            for (int b = 0; b < 6; b++) {
                int x[8];
                load_row(tile, b, r, x);
                fdct_block(x, T, F, r, k0);
                // quantise zig-zag indices 2 lane and 2 lane + 1 (so the lanes' codes follow each other in bitstream order)
                int a0 = quant(2 * lane, F, qscale), a1 = quant(2 * lane + 1, F, qscale);
                if (fallback) { a1 = 0; if (lane) a0 = 0; }
                w.block(a0, a1, true, b < 4 ? 0 : b - 3, pred, s_ac);
                w.flush();
            }
        }
    } else {
        const uint8_t* ref = latest_frame(frames, base_pics, n_pics, (int)streams[k]);
        const uint32_t* info_row = mbinfo + (size_t)k * EF_MBW_MAX * EF_MBH_MAX + row * EF_MBW_MAX;
        for (int mx = 0; mx < EF_MBW_MAX; mx++) {
            const uint32_t info = fallback ? 0u : info_row[mx];
            const bool intra = (info >> 16) & 1;
            const int h = (int8_t)(info & 0xFF), v = (int8_t)((info >> 8) & 0xFF);
            const uint8_t* tile = frame + ef_tile_offset(mx, row);
            int lv0[6], lv1[6];
            uint32_t cbp = intra ? 63u : 0u;
            #pragma unroll
            for (int b = 0; b < 6; b++) {
                int x[8];
                load_row(tile, b, r, x);
                if (!intra) sub_prediction(ref, mx, row, b, r, h, v, x);
                fdct_block(x, T, F, r, k0);
                lv0[b] = intra ? quant(2 * lane, F, qscale) : quant_inter(2 * lane, F, qscale);
                lv1[b] = intra ? quant(2 * lane + 1, F, qscale) : quant_inter(2 * lane + 1, F, qscale);
                if (fallback) lv0[b] = lv1[b] = 0;
                if (!intra && __any_sync(0xFFFFFFFFu, lv0[b] != 0 || lv1[b] != 0)) cbp |= 0x20u >> b;
                __syncwarp();
            }
            if (!mb_header(false, mx, intra, h, v, cbp, pending, pred, mvp, put)) continue;
            w.flush();
            #pragma unroll
            for (int b = 0; b < 6; b++) {
                if (!(cbp & (0x20u >> b))) continue;
                w.block(lv0[b], lv1[b], intra, b < 4 ? 0 : b - 3, pred, s_ac);
                w.flush();
            }
        }
    }
    w.finish(slice_len + gw);
}

// the exact bytes of slice `row` of picture k of the round coded at every candidate q = qmin + lane (lane < nq) and as its fallback
// (lane kCensusFallback): census[(k * 32 + lane) * 12 + row]. One warp per slice; the FDCT of a block does not depend on q, so each
// block is transformed once and then quantised and its codes counted at every candidate, the lanes splitting the coefficients as
// the slice coder does. Lane q then walks the slice's macroblock headers for its own q with the coder's walk: address increments and
// skips (they depend on q through the coded block pattern), the predictor resets, vector, type and pattern codes, DC differences.
// ipic: the round's pictures are I pictures; else P pictures with their search's mbinfo.
__global__ void __launch_bounds__(kEncWarps * 32) ef_encode_census_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ streams, int count,
                                                                         const uint8_t* __restrict__ frames, const uint32_t* __restrict__ base_pics,
                                                                         const uint32_t* __restrict__ n_pics, const uint32_t* __restrict__ mbinfo, int ipic,
                                                                         int qmin, int nq, uint32_t* __restrict__ census)
{
    __shared__ uint32_t s_ac[32 * 41];
    __shared__ int s_t[kEncWarps][64], s_f[kEncWarps][64];
    for (int i = threadIdx.x; i < 32 * 41; i += blockDim.x) s_ac[i] = c_tab.ac[i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * kEncWarps + warp;
    if (gw >= count * EF_MBH_MAX) return;
    const int k = gw / EF_MBH_MAX, row = gw % EF_MBH_MAX;
    const uint8_t* frame = src + (size_t)k * EF_FRAME;
    const uint8_t* ref = nullptr;
    const uint32_t* info_row = nullptr;
    if (!ipic) {
        ref = latest_frame(frames, base_pics, n_pics, (int)streams[k]);
        info_row = mbinfo + (size_t)k * EF_MBW_MAX * EF_MBH_MAX + row * EF_MBW_MAX;
    }
    int* T = s_t[warp];
    int* F = s_f[warp];
    const int r = lane >> 2, k0 = (lane & 3) * 2;
    const bool fb_lane = lane == kCensusFallback;
    uint32_t P = 38;
    int pred[3] = { 128, 128, 128 }, mvp[2] = { 0, 0 }, pending = 0;
    const auto count_bits = [&](uint32_t e) { P += e & 0xFF; };
    for (int mx = 0; mx < EF_MBW_MAX; mx++) {
        const uint32_t info = ipic ? (1u << 16) : info_row[mx];
        const bool intra = (info >> 16) & 1;
        const int h = (int8_t)(info & 0xFF), v = (int8_t)((info >> 8) & 0xFF);
        const uint8_t* tile = frame + ef_tile_offset(mx, row);
        uint32_t cbp = 0, blk = 0;                       // this lane's q: coded blocks, their run / level and end-of-block bits
        int dcl[6];
        #pragma unroll 1
        for (int b = 0; b < 6; b++) {
            int x[8];
            load_row(tile, b, r, x);
            if (!intra) sub_prediction(ref, mx, row, b, r, h, v, x);
            fdct_block(x, T, F, r, k0);
            dcl[b] = intra ? quant(0, F, 1) : 0;         // an intra DC level does not depend on q
            // every candidate, lowest first; levels only shrink as q grows, so once a block has no level left (intra: no AC
            // level) it has none at any later candidate
            int qi = 0;
            for (; qi < nq; qi++) {
                const int q = qmin + qi;
                const int a0 = intra ? (lane ? quant(2 * lane, F, q) : 0) : quant_inter(2 * lane, F, q);
                const int a1 = intra ? quant(2 * lane + 1, F, q) : quant_inter(2 * lane + 1, F, q);
                const uint64_t mask = level_mask(lane, a0, a1, intra);
                if (!(intra ? mask & ~1ull : mask)) break;
                uint32_t c0, n0, c1, n1;
                ac_codes(lane, a0, a1, intra, mask, s_ac, &c0, &n0, &c1, &n1);
                const uint32_t bits = (uint32_t)__reduce_add_sync(0xFFFFFFFFu, (int)(n0 + n1));
                if (lane == qi) { blk += bits + 2; cbp |= 0x20u >> b; }
            }
            if (intra && lane >= qi && !fb_lane) { blk += 2; cbp |= 0x20u >> b; }
            __syncwarp();
        }
        // the fallback: P every macroblock not coded (vector (0, 0)); I the DC levels and end of block of every block
        const bool my_intra = intra && !(fb_lane && !ipic);
        if (fb_lane) { cbp = ipic ? 63u : 0u; blk = ipic ? 12u : 0u; }
        if (!mb_header(ipic, mx, my_intra, fb_lane ? 0 : h, fb_lane ? 0 : v, cbp, pending, pred, mvp, count_bits)) continue;
        if (my_intra) {
            #pragma unroll
            for (int b = 0; b < 6; b++) {
                const int comp = b < 4 ? 0 : b - 3;
                uint32_t code, len;
                dc_code(comp, dcl[b] - pred[comp], &code, &len);
                P += len;
                pred[comp] = dcl[b];
            }
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

// one CTA per picture: its header of hb bytes (headers + p hb with per_picture, else the one header at headers), then its 12 slices,
// at pic_dst[p] in es
__global__ void ef_encode_assemble_kernel(const uint32_t* __restrict__ slots, const uint32_t* __restrict__ slice_len, const uint64_t* __restrict__ pic_dst,
                                          const uint8_t* __restrict__ headers, int hb, bool per_picture, uint8_t* __restrict__ es)
{
    const int p = blockIdx.x;
    __shared__ uint32_t off[EF_MBH_MAX + 1];
    if (threadIdx.x == 0) {
        off[0] = (uint32_t)hb;
        for (int s = 0; s < EF_MBH_MAX; s++) off[s + 1] = off[s] + slice_len[p * EF_MBH_MAX + s];
    }
    __syncthreads();
    uint8_t* dst = es + pic_dst[p];
    const uint8_t* header = headers + (per_picture ? (size_t)p * hb : 0);
    for (int i = threadIdx.x; i < hb; i += blockDim.x) dst[i] = header[i];
    for (int s = 0; s < EF_MBH_MAX; s++) {
        const uint8_t* src = (const uint8_t*)(slots + (size_t)(p * EF_MBH_MAX + s) * (kTrickSliceBytes / 4));
        const uint32_t n = off[s + 1] - off[s];
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[off[s] + i] = src[i];
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------------------------
namespace {

uint32_t vlc_entry(const char* code)
{
    uint32_t v = 0, n = 0;
    for (; *code; code++, n++) v = (v << 1) | (uint32_t)(*code == '1');
    return (v << 8) | n;
}

}  // namespace

cudaError_t ef_encode_upload_tables()
{
    CodeTables t;
    memset(&t, 0, sizeof(t));
    for (int i = 0; i < EF_VLC_DCT_COUNT; i++) {
        const int run = ef_vlc_dct[i].value >> 8, level = ef_vlc_dct[i].value & 0xFF;
        if (run <= 31 && level <= 40) t.ac[run * 41 + level] = vlc_entry(ef_vlc_dct[i].code);
    }
    for (int i = 0; i < EF_VLC_DC_LUMA_COUNT; i++) t.dc[0][ef_vlc_dc_luma[i].value] = vlc_entry(ef_vlc_dc_luma[i].code);
    for (int i = 0; i < EF_VLC_DC_CHROMA_COUNT; i++) t.dc[1][ef_vlc_dc_chroma[i].value] = vlc_entry(ef_vlc_dc_chroma[i].code);
    memcpy(t.zz, ef_zigzag, 64);
    memcpy(t.q, ef_default_intra_q, 64);
    for (int i = 0; i < EF_VLC_MBA_COUNT; i++) if (ef_vlc_mba[i].value >= 1 && ef_vlc_mba[i].value <= 33) t.mba[ef_vlc_mba[i].value] = vlc_entry(ef_vlc_mba[i].code);
    for (int i = 0; i < EF_VLC_MBTYPE_P_COUNT; i++) t.type[ef_vlc_mbtype_p[i].value] = vlc_entry(ef_vlc_mbtype_p[i].code);
    for (int i = 0; i < EF_VLC_MV_COUNT; i++) t.mv[ef_vlc_mv[i].value + 16] = vlc_entry(ef_vlc_mv[i].code);
    for (int i = 0; i < EF_VLC_CBP_COUNT; i++) t.cbp[ef_vlc_cbp[i].value] = vlc_entry(ef_vlc_cbp[i].code);
    return cudaMemcpyToSymbol(c_tab, &t, sizeof(t));
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

cudaError_t ef_encode_launch_slices(bool ipic, const uint8_t* src, const uint32_t* streams, int count, const uint8_t* frames, const uint32_t* base_pics,
                                    const uint32_t* n_pics, const uint32_t* mbinfo, int qscale, const uint8_t* qpic, uint32_t* slots, uint32_t* slice_len,
                                    cudaStream_t st)
{
    const int warps = count * EF_MBH_MAX;
    auto kernel = ipic ? ef_encode_slice_kernel<true> : ef_encode_slice_kernel<false>;
    kernel<<<(warps + kEncWarps - 1) / kEncWarps, kEncWarps * 32, 0, st>>>(src, streams, count, frames, base_pics, n_pics, mbinfo, qscale, qpic, slots,
                                                                        slice_len);
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

cudaError_t ef_encode_launch_assemble(const uint32_t* slots, const uint32_t* slice_len, const uint64_t* pic_dst, const uint8_t* headers, int hb,
                                      bool per_picture, int n_pics, uint8_t* es, cudaStream_t st)
{
    ef_encode_assemble_kernel<<<n_pics, 256, 0, st>>>(slots, slice_len, pic_dst, headers, hb, per_picture, es);
    return cudaGetLastError();
}
