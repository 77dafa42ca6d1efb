// espflix_b200/csrc/ef_coef_step.cuh — one step of K1a's coefficient parser, shared by the kernel (ef_decode.cu)
// and by the host-side model test (tests/k1a_step_model.cpp), so the exact code the GPU runs is checked on the CPU
// against a symbol-by-symbol restatement of get_vlc_dct()/block() (player.cpp:549-644, 1068-1121).
//
// ef_coef_sym decodes ONE symbol from the next 32 bits of the slice (`w`, MSB first) through the clz-indexed table
// (EfTables::dct): a (run, level) code with its sign bit or escape payload, an end of block, or not a code. The kernel
// folds a '10' that follows a coefficient into the same step. ef_coef_entry dequantises a coefficient and packs it into
// its list entry.
#pragma once
#include "ef_common.cuh"

// plain C on both sides (the __byte_perm intrinsic masks the sign-replicate bit of its selector: a hand-picked PRMT
// would differ between the kernel and the host model; the compiler finds PRMT / SGXT itself)
#if defined(__CUDA_ARCH__)
#define EF_CLZ(x) __clz((int)(x))
#else
#define EF_CLZ(x) ((x) ? __builtin_clz((unsigned)(x)) : 32)
#endif
#define EF_BYTE1(x) ((int)(((x) >> 8) & 255u))                    // bits 8-15, zero-extended

// One coefficient of block(), player.cpp:1106-1121, from its signed level to its list entry. Dequantisation in
// magnitude form: v = 2*level (+-1 when not intra, k = 1); v = (v * qscale * q) / 16 with C truncation, i.e. on the
// magnitude; oddify towards zero, except that 0 becomes +1 whatever the sign was (Q2); clamp to [-2048, 2047];
// b[zz] = v * scale_dct_q[zz]. z = the table word of scan position n (quantiser | prescale << 8 | zz << 18).
// List entry = (block << 24 | zz << 18) + b[zz] (two's complement add): |b[zz]| < 2^17, so the reader takes the value
// from the low 18 bits (sign-extended) and block / position from (entry + 2^17) >> 18.
static __host__ __device__ __forceinline__ uint32_t ef_coef_entry(uint32_t z, int level, int qscale, int k, uint32_t blk24)
{
    const int mag = level < 0 ? -level : level;
    int neg = level < 0;
    int m = ((2 * mag + k) * (qscale * (int)(z & 255u))) >> 4;
    if (m == 0) neg = 0;
    m = ((m > 1 ? m : 1) - 1) | 1;
    m = m < 2047 + neg ? m : 2047 + neg;
    const int v = neg ? -m : m;
    return (uint32_t)(v * EF_BYTE1(z) + (int)((z & 0x00FC0000u) | blk24));
}

#define EF_SYM_COEF 0u
#define EF_SYM_EOB 1u         // '10' on its own (an intra block without AC coefficients)
#define EF_SYM_DERAIL 2u      // not a code: nothing consumed

struct EfSym {
    uint32_t kind;
    int len, run, lvl;        // bits consumed (sign / escape payload included), zero run, signed level
};

static __host__ __device__ __forceinline__ EfSym ef_coef_sym(uint32_t w, bool first, const uint16_t* __restrict__ dct)
{
    EfSym r;
    // row (context, leading zeros), column = the five bits after the leading one. Branch-free: the row saturates at 12
    // (all-invalid: >= 12 leading zeros is not a code) and the leading-one column bit is forced, so that a window with
    // more than 12 zeros cannot slide back into row 11
    const int lz = EF_CLZ(w), row = lz < 12 ? lz : 12;
    const int idx = (first ? 13 * 32 - 32 : -32) + row * 32 + (int)(((w << row) >> 26) | 32u);
    const uint32_t t = dct[idx];
    r.len = (int)(t & 31u); r.run = (int)((t >> 5) & 31u);
    const int mag = (int)(t >> 10);
    r.kind = EF_SYM_COEF;
    r.lvl = ((w >> ((32 - r.len) & 31)) & 1u) ? -mag : mag;          // sign = last bit of a regular code
    if (mag == 0) {
        if (r.len == 2) r.kind = EF_SYM_EOB;                          // player.cpp:1075
        else if (r.len == 6) {                                        // escape: 6-bit run, 8- or 16-bit level (player.cpp:1092)
            r.run = (int)((w >> 20) & 63u);
            const int b = (int)((w >> 12) & 255u);
            r.lvl = (int)(int8_t)b; r.len = 20;
            if ((b & 127) == 0) { r.lvl = (int)((w >> 4) & 255u) - 2 * b; r.len = 28; }      // b = 0: 0..255, b = 128: -256..-1
        } else r.kind = EF_SYM_DERAIL;
    }
    return r;
}
