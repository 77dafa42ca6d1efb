// espflix_b200/csrc/ef_tables.cpp — host-side construction of the kernels' lookup tables from the
// ISO 11172-2 Annex B code lists (ef_iso11172_tables.h). The reference decodes the same codes
// with binary-tree walks (get_vlc, player.cpp:516) and a nested-prefix decoder (get_vlc_dct,
// player.cpp:549); here every table is re-shaped for "count leading zeros, take the next five
// bits, one load".
#include <stdio.h>
#include <string.h>

#include "ef_common.cuh"
#include "ef_iso11172_tables.h"

namespace {

// Place `entry` at every index (lz, next5) matched by `code` (code = lz zeros, a one, k more bits).
// max_lz = number of lz classes. Returns false if the code does not fit the (lz, 5-bit) shape.
bool place(uint16_t* tab, int max_lz, const char* code, uint16_t entry)
{
    int len = (int)strlen(code), lz = 0;
    while (lz < len && code[lz] == '0') lz++;
    if (lz >= len || lz >= max_lz) return false;
    int k = len - lz - 1;
    if (k > 5) return false;
    unsigned rest = 0;
    for (int i = 0; i < k; i++) rest = (rest << 1) | (unsigned)(code[lz + 1 + i] == '1');
    for (unsigned fill = 0; fill < (1u << (5 - k)); fill++) {
        unsigned idx = (unsigned)lz * 32 + ((rest << (5 - k)) | fill);
        if (tab[idx]) return false;
        tab[idx] = entry;
    }
    return true;
}

}  // namespace

// combined per-scan-position entry of the parser: quantiser byte | AAN prescale << 8 | raster index << 18
uint32_t ef_qz_entry(unsigned q, int n) { return (q & 255u) | ((uint32_t)ef_aan_prescale[ef_zigzag[n]] << 8) | ((uint32_t)ef_zigzag[n] << 18); }

// returns 0 on success, else the number of the table that failed
int ef_build_tables(EfTables* t)
{
    memset(t, 0, sizeof(*t));
    for (int i = 0; i < EF_VLC_DCT_COUNT; i++) {
        int run = ef_vlc_dct[i].value >> 8, level = ef_vlc_dct[i].value & 0xFF;
        int len = (int)strlen(ef_vlc_dct[i].code) + 1;                 // + sign bit
        // (0,1) is "11s" as dct_coeff_next: lives in row 0 next to end-of-block "10"
        if (!place(t->dct, 12, ef_vlc_dct[i].code, (uint16_t)(len | (run << 5) | (level << 10)))) return 1;
    }
    if (!place(t->dct, 12, "10", (uint16_t)2)) return 1;               // end of block: level 0, length 2
    if (!place(t->dct, 12, "000001", (uint16_t)(6 | (1 << 5)))) return 1;   // escape: level 0, run 1
    memcpy(t->dct + 13 * 32, t->dct, 13 * 32 * sizeof(uint16_t));      // first-coefficient context = same table ...
    for (int i = 0; i < 32; i++) t->dct[13 * 32 + i] = (uint16_t)(2 | (0 << 5) | (1 << 10));   // ... except "1s" = (0,1) instead of "10"/"11s"
    for (int i = 0; i < EF_VLC_MBA_COUNT; i++) {
        int len = (int)strlen(ef_vlc_mba[i].code);
        if (!place(t->mba, 8, ef_vlc_mba[i].code, (uint16_t)(len | (ef_vlc_mba[i].value << 4)))) return 2;
    }
    for (int i = 0; i < EF_VLC_MV_COUNT; i++) {
        int len = (int)strlen(ef_vlc_mv[i].code);
        if (!place(t->mv, 7, ef_vlc_mv[i].code, (uint16_t)(len | ((ef_vlc_mv[i].value + 16) << 4)))) return 3;
    }
    for (int i = 0; i < EF_VLC_CBP_COUNT; i++) {
        const char* c = ef_vlc_cbp[i].code;
        int len = (int)strlen(c);
        unsigned v = 0;
        for (int k = 0; k < len; k++) v = (v << 1) | (unsigned)(c[k] == '1');
        for (unsigned fill = 0; fill < (1u << (9 - len)); fill++) {
            unsigned idx = (v << (9 - len)) | fill;
            if (t->cbp[idx]) return 4;
            t->cbp[idx] = (uint16_t)(len | (ef_vlc_cbp[i].value << 4));
        }
    }
    for (int i = 0; i < EF_VLC_MBTYPE_P_COUNT; i++) {
        const char* c = ef_vlc_mbtype_p[i].code;
        int len = (int)strlen(c);
        unsigned v = 0;
        for (int k = 0; k < len; k++) v = (v << 1) | (unsigned)(c[k] == '1');
        for (unsigned fill = 0; fill < (1u << (6 - len)); fill++) {
            unsigned idx = (v << (6 - len)) | fill;
            if (t->ptype[idx]) return 5;
            t->ptype[idx] = (uint8_t)(len | (ef_vlc_mbtype_p[i].value << 3));
        }
    }
    for (int i = 0; i < 64; i++) t->izz[ef_zigzag[i]] = (uint8_t)i;
    memcpy(t->prescale, ef_aan_prescale, 64);
    memcpy(t->zigzag, ef_zigzag, 64);
    for (int n = 0; n < 64; n++) { t->qdef[n] = ef_default_intra_q[ef_zigzag[n]]; t->qdef[64 + n] = 16; }
    for (int n = 0; n < 64; n++) t->zp[n] = (uint16_t)(ef_zigzag[n] | (ef_aan_prescale[ef_zigzag[n]] << 8));
    for (int n = 0; n < 128; n++) t->qz[n] = ef_qz_entry(t->qdef[n], n & 63);
    return 0;
}

// ---- composite LUTs (video.cpp:335-507 data tables; derivation espflix.cpp:1091-1180) ----------
// 4 subcarrier phases per entry: p_i = round(w_i * (128-c) * (24/33)) + 48, clamped to [0,127],
// bytes swizzled 0123 -> 0213 to match the blitter's sample order.
#include <math.h>
static int round_half_away(float v) { return v < 0 ? -(int)(-v + 0.5) : (int)(v + 0.5); }

static void chroma_lut(uint32_t* dst, int use_cos, int negate)
{
    const int black = 24;                     // IRE(7.5) >> 8, video.cpp:520-525
    const float scale = (float)black / 33;
    for (int c = 0; c < 256; c++) {
        int u = 128 - c;
        uint32_t v = 0;
        for (int i = 0; i < 4; i++) {
            double w = use_cos ? cos(2 * M_PI * i / 4) : sin(2 * M_PI * i / 4);
            if (negate) w = -w;
            int p = round_half_away((float)(w * u * scale)) + 2 * black;
            p = p < 0 ? 0 : (p < 127 ? p : 127);
            v = (v << 8) | (uint32_t)p;
        }
        dst[c] = (v & 0xFF0000FFu) | ((v >> 8) & 0xFF00u) | ((v << 8) & 0xFF0000u);
    }
}

void ef_build_color_tab(uint32_t* tab768, int ntsc)
{
    chroma_lut(tab768, 0, 0);                 // NTSC uv_tab[u] / PAL sin_u
    chroma_lut(tab768 + 256, 1, 0);           // NTSC uv_tab[v] / PAL cos_v
    chroma_lut(tab768 + 512, 1, ntsc ? 0 : 1);   // NTSC uv_tab[v] again / PAL cos_v_neg (video.cpp:584-591)
}

// PAL burst tables (video.cpp:619-629): BLANKING + sin(phase +- 3pi/4) * BLANKING / 1.5, phase = pi + k*pi/2
void ef_build_pal_burst(int16_t* b0, int16_t* b1, int width)
{
    const unsigned blanking = 0x1400;
    float phase = 2 * M_PI / 2;
    for (int i = 0; i < width; i++) {
        b0[i] = (int16_t)(blanking + sin(phase + 3 * M_PI / 4) * blanking / 1.5);
        b1[i] = (int16_t)(blanking + sin(phase - 3 * M_PI / 4) * blanking / 1.5);
        phase += 2 * M_PI / 4;
    }
}
