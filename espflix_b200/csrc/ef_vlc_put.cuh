// csrc/ef_vlc_put.cuh — the picture encoders' shared parts (ef_trick.cu's intra pictures, ef_encode.cu's predicted ones): the
// integer FDCT, the intra quantiser, the run / level and DC code tables, and the warp's bit window. Every translation unit that
// includes it holds its own copy of the constant tables and fills it with upload_trick_tables().
#pragma once
#include <stdint.h>
#include <string.h>

#include "ef_common.cuh"
#include "ef_iso11172_tables.h"

namespace {

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

struct TrickTables {
    uint32_t ac[32 * 41];      // run 0..31 x level 0..40: (code << 8) | length, without the sign bit; 0 = escape
    uint32_t dc[2][9];         // luma / chroma dct_dc_size: (code << 8) | length
    uint8_t zz[64];            // zig-zag index -> raster index
    uint8_t q[64];             // default intra matrix, raster index
};
__constant__ TrickTables c_trick;

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
    const int z = c_trick.zz[i], f = F[z];
    if (i == 0) { const int dc = (f + 4) >> 3; return dc > 255 ? 255 : dc; }
    const int den = qscale * c_trick.q[z], num = 8 * (f < 0 ? -f : f);
    int lv = (2 * num + den) / (2 * den);
    lv = lv > 255 ? 255 : lv;
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

// ---- host side ----------------------------------------------------------------------------------------------------------------------
static uint32_t vlc_entry(const char* code)
{
    uint32_t v = 0, n = 0;
    for (; *code; code++, n++) v = (v << 1) | (uint32_t)(*code == '1');
    return (v << 8) | n;
}

static cudaError_t upload_trick_tables()
{
    TrickTables t;
    memset(&t, 0, sizeof(t));
    for (int i = 0; i < EF_VLC_DCT_COUNT; i++) {
        const int run = ef_vlc_dct[i].value >> 8, level = ef_vlc_dct[i].value & 0xFF;
        if (run <= 31 && level <= 40) t.ac[run * 41 + level] = vlc_entry(ef_vlc_dct[i].code);
    }
    for (int i = 0; i < EF_VLC_DC_LUMA_COUNT; i++) t.dc[0][ef_vlc_dc_luma[i].value] = vlc_entry(ef_vlc_dc_luma[i].code);
    for (int i = 0; i < EF_VLC_DC_CHROMA_COUNT; i++) t.dc[1][ef_vlc_dc_chroma[i].value] = vlc_entry(ef_vlc_dc_chroma[i].code);
    memcpy(t.zz, ef_zigzag, 64);
    memcpy(t.q, ef_default_intra_q, 64);
    return cudaMemcpyToSymbol(c_trick, &t, sizeof(t));
}

}  // namespace
