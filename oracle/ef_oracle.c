/* oracle/ef_oracle.c — CPU restatement of the espflix hot path. TEST INFRASTRUCTURE ONLY
 * (see ef_oracle.h). Plain C; every function cites the reference lines it follows
 * (paths relative to the reference's src/). Validated against the unmodified reference built in
 * oracle/_ref and against the pins in tests/golden/.
 */
#include "ef_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "../espflix_b200/csrc/ef_iso11172_tables.h"   /* ISO 11172-2 Annex B tables (shared data, not logic) */

/* ------------------------------------------------------------------------------------------
 * VLC tries built from the ISO code strings; decoded one bit at a time like get_vlc
 * (player.cpp:516-530).
 * ---------------------------------------------------------------------------------------- */
typedef struct { int16_t next[2]; int32_t value; int8_t leaf; } trie_node;
typedef struct { trie_node n[512]; int count; } trie;

static void trie_add(trie* t, const char* code, int value)
{
    int s = 0;
    for (const char* c = code; *c; c++) {
        int b = *c == '1';
        if (t->n[s].next[b] < 0) {
            int k = t->count++;
            t->n[k].next[0] = t->n[k].next[1] = -1;
            t->n[k].leaf = 0;
            t->n[s].next[b] = (int16_t)k;
        }
        s = t->n[s].next[b];
    }
    t->n[s].leaf = 1;
    t->n[s].value = value;
}

static void trie_build(trie* t, const ef_vlc_code* codes, int n)
{
    t->count = 1;
    t->n[0].next[0] = t->n[0].next[1] = -1;
    t->n[0].leaf = 0;
    for (int i = 0; i < n; i++) trie_add(t, codes[i].code, codes[i].value);
}

static trie T_mba, T_type_i, T_type_p, T_cbp, T_mv, T_dct;
static int tables_ready = 0;

static void tables_init(void)
{
    if (tables_ready) return;
    trie_build(&T_mba, ef_vlc_mba, EF_VLC_MBA_COUNT);
    trie_build(&T_type_i, ef_vlc_mbtype_i, EF_VLC_MBTYPE_I_COUNT);
    trie_build(&T_type_p, ef_vlc_mbtype_p, EF_VLC_MBTYPE_P_COUNT);
    trie_build(&T_cbp, ef_vlc_cbp, EF_VLC_CBP_COUNT);
    trie_build(&T_mv, ef_vlc_mv, EF_VLC_MV_COUNT);
    trie_build(&T_dct, ef_vlc_dct, EF_VLC_DCT_COUNT);
    trie_add(&T_dct, "000001", 0);          /* escape: level 0, run follows (player.cpp:611-615) */
    tables_ready = 1;
}

/* coverage counters (test assertions only): which decoder paths an input exercised */
static efo_stats g_stats;
void efo_stats_reset(void) { memset(&g_stats, 0, sizeof(g_stats)); }
void efo_stats_get(efo_stats* s) { *s = g_stats; }

/* ------------------------------------------------------------------------------------------
 * TS demux — MpegDecoder::more / demux / parse_pts (player.cpp:294-307, 381-436, 459-493)
 * ---------------------------------------------------------------------------------------- */
static int be16(const uint8_t* d) { return (d[0] << 8) | d[1]; }

static int64_t pes_pts(const uint8_t* d, int flags)      /* player.cpp:299 */
{
    flags = (flags >> 2) & 0x30;
    if ((d[0] & 0xF0) != flags) return -1;
    int64_t n = ((int64_t)(d[0] & 0x0E)) << 29;
    n += (int64_t)(be16(d + 1) >> 1) << 15;
    return n + (be16(d + 3) >> 1);
}

size_t efo_demux_ts(const uint8_t* ts, size_t len, uint8_t* es, size_t es_cap,
                    uint64_t* pes_off, int64_t* pes_ptsv, size_t pes_cap, size_t* n_pes)
{
    size_t out = 0, np = 0;
    for (size_t pos = 0; pos + 188 <= len; pos += 188) {
        const uint8_t* d = ts + pos;
        if (d[0] != 0x47) break;                               /* "ts lost sync" (player.cpp:477) */
        int pid = ((d[1] << 8) + d[2]) & 0x1fff;
        const uint8_t* data = d + 4;
        if (d[3] & 0x20) data = d + 5 + d[4];                  /* adaptation field */
        if (!(d[3] & 0x10)) continue;                          /* no payload */
        const uint8_t* end = d + 188;
        const uint8_t* payload = data;
        int64_t pts = -1;
        int pus = d[1] & 0x40;
        if (pus) {                                             /* PES header (player.cpp:387-406) */
            const uint8_t* p = data + 6;
            int flags = be16(p);
            payload = p + 3 + p[2];
            if (flags & 0x0080) pts = pes_pts(p + 3, flags);
        }
        if (pid != 0x100) continue;
        if (pus) {
            if (np < pes_cap) {
                if (pes_off) pes_off[np] = out;
                if (pes_ptsv) pes_ptsv[np] = pts;
            }
            np++;
        }
        if (payload < end) {
            size_t n = (size_t)(end - payload);
            if (out + n <= es_cap) memcpy(es + out, payload, n);
            out += n;
        }
    }
    if (n_pes) *n_pes = np;
    return out;
}

/* ------------------------------------------------------------------------------------------
 * Decoder state
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    const uint8_t* es; size_t len; size_t bitpos;    /* flat ES + eos padding (player.cpp:456) */

    uint8_t* fb[2];            /* two striped frame stores, strips contiguous (video.h:36) */
    int fb_index;
    uint8_t* reference; uint8_t* current;
    int have_pts; int64_t last_pts;                    /* -1 = none (Q10) */

    int horizontal_size, vertical_size, mb_width, mb_height;
    uint8_t intra_q[64], non_intra_q[64];
    int picture_coding_type, full_pel_forward, forward_r_size, quantizer_scale;
    int mb_x, mb_y;
    uint8_t *y_addr, *cr_addr, *cb_addr;
    int y_dc, cr_dc, cb_dc, forward_motion_h, forward_motion_v;

    uint8_t* out; size_t cap; size_t n_out;
    int ended;
} dec_t;

/* bit reader: MSB-first over the byte stream; FILL_BITS/get_bits/peek_bits (player.cpp:348-352,
 * 495-514) only ever expose "the next n bits", which is what these two functions return. */
static const uint8_t EOS[8] = { 0x00, 0x00, 0x01, 0xB7, 0x00, 0x00, 0x01, 0xB7 };

static int es_byte(const dec_t* d, size_t i)
{
    if (i < d->len) return d->es[i];
    i -= d->len;
    return i < 8 ? EOS[i] : 0;
}

static uint32_t peek_bits(const dec_t* d, int n)       /* n <= 25 */
{
    size_t byte = d->bitpos >> 3;
    int sh = (int)(d->bitpos & 7);
    uint64_t w = 0;
    for (int i = 0; i < 5; i++) w = (w << 8) | (uint64_t)es_byte(d, byte + i);
    return (uint32_t)((w >> (40 - sh - n)) & ((1u << n) - 1));
}
static uint32_t get_bits(dec_t* d, int n) { uint32_t v = n ? peek_bits(d, n) : 0; d->bitpos += n; return v; }
static int get_bit(dec_t* d) { return (int)get_bits(d, 1); }

static int get_vlc(dec_t* d, const trie* t)            /* player.cpp:516 */
{
    int s = 0;
    do {
        s = t->n[s].next[get_bit(d)];
        if (s < 0) return 0;            /* invalid code: reference walks out of its table (UB) */
    } while (!t->n[s].leaf);
    return t->n[s].value;
}

/* frame address map (player.cpp:33-46) on contiguous strips: strip s at s*8448 */
static uint8_t* get_y(uint8_t* f, int y) { return f + (y >> 4) * 8448 + (y & 15) * 528; }
static uint8_t* get_cr(uint8_t* f, int y) { return f + (y >> 3) * 8448 + (y & 7) * 528 + 352; }
static uint8_t* get_cb(uint8_t* f, int y) { return f + (y >> 3) * 8448 + ((y & 7) + 8) * 528 + 352; }

void efo_i420_to_strips(const uint8_t* s, uint8_t* f)
{
    for (int y = 0; y < 192; y++, s += 352) memcpy(get_y(f, y), s, 352);
    for (int y = 0; y < 96; y++, s += 176) memcpy(get_cr(f, y), s, 176);
    for (int y = 0; y < 96; y++, s += 176) memcpy(get_cb(f, y), s, 176);
}
void efo_strips_to_i420(const uint8_t* f, uint8_t* d)
{
    for (int y = 0; y < 192; y++, d += 352) memcpy(d, get_y((uint8_t*)f, y), 352);
    for (int y = 0; y < 96; y++, d += 176) memcpy(d, get_cr((uint8_t*)f, y), 176);
    for (int y = 0; y < 96; y++, d += 176) memcpy(d, get_cb((uint8_t*)f, y), 176);
}

static int pin(int x)   /* _pin LUT, player.cpp:183-236 (Q1); the table covers -256..511, outside is undefined in the reference */
{
    if (x < -256 || x > 511) g_stats.pin_out_of_domain++;
    return x < 0 ? 0 : x > 248 ? 248 : x;
}

/* ------------------------------------------------------------------------------------------
 * headers — sequence/gop/picture/flush_picture (player.cpp:646-724)
 * ---------------------------------------------------------------------------------------- */
static void push_frame(dec_t* d, const uint8_t* f)
{
    if (d->out && d->n_out < d->cap) efo_strips_to_i420(f, d->out + d->n_out * EFO_I420_BYTES);
    d->n_out++;
}

static void flush_picture(dec_t* d, int mode)          /* player.cpp:692 */
{
    if (d->last_pts != -1 || mode) {
        push_frame(d, d->fb[d->fb_index & 1]);
        d->reference = d->fb[d->fb_index++ & 1];
        d->current = d->fb[d->fb_index & 1];
    }
    if (!mode) d->last_pts = d->have_pts ? 1 : -1;     /* _last_pts = _pts */
}

static void sequence(dec_t* d)                         /* player.cpp:658 */
{
    d->horizontal_size = (int)get_bits(d, 12);
    d->vertical_size = (int)get_bits(d, 12);
    get_bits(d, 4); get_bits(d, 4); get_bits(d, 18); get_bits(d, 12);
    if (get_bit(d)) { for (int i = 0; i < 64; i++) d->intra_q[i] = (uint8_t)get_bits(d, 8); }   /* Q4: stored in stream order */
    else memcpy(d->intra_q, ef_default_intra_q, 64);
    if (get_bit(d)) { for (int i = 0; i < 64; i++) d->non_intra_q[i] = (uint8_t)get_bits(d, 8); }
    else memset(d->non_intra_q, 16, 64);
    d->mb_width = (d->horizontal_size + 15) >> 4;
    d->mb_height = (d->vertical_size + 15) >> 4;
}

static void gop(dec_t* d) { get_bits(d, 25); get_bits(d, 7); }   /* player.cpp:680 (Q9: values unused) */

/* which macroblocks each of the first EFO_COV_PICTURES pictures of the last efo_decode_es call wrote: 2 decoded from its own
   codes, 1 copied by a skip (the last write counts), 0 not written (tests of ef_trick_build's segment rule) */
#define EFO_COV_PICTURES 8
static uint8_t g_cov[EFO_COV_PICTURES][264];
static int g_cov_n;

static void cover(const dec_t* d, uint8_t how)
{
    if (g_cov_n >= 1 && g_cov_n <= EFO_COV_PICTURES && d->mb_x < 22 && d->mb_y < 12) g_cov[g_cov_n - 1][d->mb_y * 22 + d->mb_x] = how;
}

int efo_coverage(uint8_t* out, int max_pictures)
{
    const int n = g_cov_n < max_pictures ? g_cov_n : max_pictures;
    memcpy(out, g_cov, (size_t)(n < EFO_COV_PICTURES ? n : EFO_COV_PICTURES) * 264);
    return g_cov_n;
}

static void picture(dec_t* d)                          /* player.cpp:704 */
{
    flush_picture(d, 0);
    g_cov_n++;
    get_bits(d, 10);
    d->picture_coding_type = (int)get_bits(d, 3);
    g_stats.pictures[d->picture_coding_type & 7]++;
    if (d->picture_coding_type != 1 && d->picture_coding_type != 2) return;
    get_bits(d, 16);
    if (d->picture_coding_type == 2) {
        d->full_pel_forward = get_bit(d);
        d->forward_r_size = (int)get_bits(d, 3) - 1;
        g_stats.f_code[(d->forward_r_size + 1) & 7]++;
    }
}

/* ------------------------------------------------------------------------------------------
 * motion compensation — mocomp/blit/predict_zero/predict (player.cpp:732-889)
 * ---------------------------------------------------------------------------------------- */
static const uint8_t* ref_row(dec_t* d, int c, int y)
{
    switch (c) {
        case 1: return get_cr(d->reference, y);
        case 2: return get_cb(d->reference, y);
        default: return get_y(d->reference, y);
    }
}

static void mocomp(dec_t* d, uint8_t* dst, int pos_x, int pos_y, int size, int c)   /* player.cpp:733 */
{
    int xh = pos_x & 1, yh = pos_y & 1;
    if (size == 16) g_stats.mocomp_xy[(yh << 1) | xh]++;
    pos_y >>= 1; pos_x >>= 1;
    dst += size * d->mb_x;
    for (int y = 0; y < size; y++) {
        const uint8_t* a = ref_row(d, c, pos_y + y) + pos_x;
        const uint8_t* b = yh ? ref_row(d, c, pos_y + y + 1) + pos_x : a;
        for (int x = 0; x < size; x++) {
            int v;
            if (!xh && !yh) v = a[x];
            else if (xh && !yh) v = (a[x] + a[x + 1] + 1) >> 1;
            else if (!xh) v = (a[x] + b[x] + 1) >> 1;
            else v = (a[x] + a[x + 1] + b[x] + b[x + 1] + 2) >> 2;
            dst[x] = (uint8_t)v;
        }
        dst += 528;
    }
}

static void predict_zero(dec_t* d)                     /* player.cpp:861 */
{
    const uint8_t* ref = get_y(d->reference, d->mb_y << 4);
    for (int i = 0; i < 16; i++) memcpy(d->y_addr + d->mb_x * 16 + i * 528, ref + d->mb_x * 16 + i * 528, 16);
    for (int i = 0; i < 8; i++) memcpy(d->cr_addr + d->mb_x * 8 + i * 528, ref + 352 + d->mb_x * 8 + i * 528, 8);
    for (int i = 0; i < 8; i++) memcpy(d->cb_addr + d->mb_x * 8 + i * 528, ref + 352 + 528 * 8 + d->mb_x * 8 + i * 528, 8);
}

static void predict(dec_t* d)                          /* player.cpp:870 */
{
    int h = d->forward_motion_h, v = d->forward_motion_v;
    if (h == 0 && v == 0) { predict_zero(d); return; }
    if (d->full_pel_forward) { h <<= 1; v <<= 1; }
    int x = (d->mb_x << 5) + h, y = (d->mb_y << 5) + v;
    mocomp(d, d->y_addr, x, y, 16, 0);
    x >>= 1; y >>= 1;                                  /* Q3: floor */
    mocomp(d, d->cr_addr, x, y, 8, 1);
    mocomp(d, d->cb_addr, x, y, 8, 2);
}

static int motion_vector(dec_t* d, int m, int r_size)  /* player.cpp:891 */
{
    int dd, scale = 1 << r_size;
    int code = get_vlc(d, &T_mv);
    if (code != 0 && scale != 1) {
        dd = ((abs(code) - 1) << r_size) + (int)get_bits(d, r_size) + 1;
        if (code < 0) dd = -dd;
    } else dd = code;
    m += dd;
    if (m > (scale << 4) - 1) m -= scale << 5;
    else if (m < -(scale << 4)) m += scale << 5;
    return m;
}

/* ------------------------------------------------------------------------------------------
 * IDCT (player.cpp:922-996): 8-point AAN butterflies on prescaled ints, columns then rows
 * ---------------------------------------------------------------------------------------- */
static void idct_1d(int32_t* v, int stride, int final_shift)
{
    int32_t in0 = v[0], in1 = v[stride], in2 = v[2 * stride], in3 = v[3 * stride];
    int32_t in4 = v[4 * stride], in5 = v[5 * stride], in6 = v[6 * stride], in7 = v[7 * stride];
    int32_t b1 = in4, b3 = in2 + in6, b4 = in5 - in3;
    int32_t t1 = in1 + in7, t2 = in3 + in5, b6 = in1 - in7, b7 = t1 + t2, m0 = in0;
    int32_t x4 = ((b6 * 473 - b4 * 196 + 128) >> 8) - b7;
    int32_t x0 = x4 - (((t1 - t2) * 362 + 128) >> 8);
    int32_t x1 = m0 - b1;
    int32_t x2 = (((in2 - in6) * 362 + 128) >> 8) - b3;
    int32_t x3 = m0 + b1;
    int32_t y3 = x1 + x2, y4 = x3 + b3, y5 = x1 - x2, y6 = x3 - b3;
    int32_t y7 = -x0 - ((b4 * 473 + b6 * 196 + 128) >> 8);
    int32_t o[8] = { b7 + y4, x4 + y3, y5 - x0, y6 - y7, y6 + y7, x0 + y5, y3 - x4, y4 - b7 };
    for (int i = 0; i < 8; i++) v[i * stride] = final_shift ? (o[i] + 128) >> 8 : o[i];
}

void efo_idct(int32_t* b)
{
    for (int i = 0; i < 8; i++) idct_1d(b + i, 8, 0);
    for (int i = 0; i < 64; i += 8) idct_1d(b + i, 1, 1);
}

/* ------------------------------------------------------------------------------------------
 * block (player.cpp:999-1148) and the four store flavours (player.cpp:1150-1236)
 * ---------------------------------------------------------------------------------------- */
static int leading_ones(uint32_t v, int width)
{
    int n = 0;
    while (n < width && (v >> (width - 1 - n)) & 1) n++;
    return n;
}

static int block(dec_t* d, int blk, int intra)
{
    const uint8_t* q = d->non_intra_q;
    int n = 0;
    int32_t b[64];
    memset(b, 0, sizeof(b));

    if (intra) {
        uint32_t pb = peek_bits(d, 10);
        int dc_size, used;
        if (blk < 4) {                                 /* B.5a as decoded at player.cpp:1014-1034 */
            b[0] = d->y_dc;
            uint32_t p9 = pb >> 1;
            if (!(p9 & 0x100)) { dc_size = 1 + (int)((p9 >> 7) & 1); used = 2; }
            else if (!(p9 & 0x80)) { dc_size = (p9 & 0x40) ? 3 : 0; used = 3; }
            else { int ones = leading_ones(p9, 9); dc_size = ones + 2; used = dc_size - 1; }
        } else {                                       /* B.5b, player.cpp:1035-1049 */
            b[0] = blk == 4 ? d->cr_dc : d->cb_dc;
            if (!(pb & 0x200)) { dc_size = (int)(pb >> 8); used = 2; }
            else { int ones = leading_ones(pb, 10); dc_size = ones + 1; used = dc_size < 10 ? dc_size : 10; }
        }
        d->bitpos += used;
        if (dc_size) {
            int delta = (int)get_bits(d, dc_size);
            if (delta & (1 << (dc_size - 1))) b[0] += delta;
            else b[0] += (int32_t)((0xFFFFFFFFu << dc_size) | (uint32_t)(delta + 1));
            if (blk == 4) d->cr_dc = b[0]; else if (blk == 5) d->cb_dc = b[0]; else d->y_dc = b[0];
        }
        b[0] = (int32_t)((uint32_t)b[0] << 8);
        q = d->intra_q;
        n = 1;
    }

    for (;;) {
        int run, v;
        uint32_t p = peek_bits(d, 2);
        if (n && p == 2) { d->bitpos += 2; break; }    /* end of block */
        if (p >> 1) {                                  /* '1s' first / '11s' next: run 0 level 1 */
            d->bitpos += n ? 2 : 1;
            run = 0; v = 1;
            if (get_bit(d)) v = -v;
        } else {
            int rl = get_vlc(d, &T_dct);
            run = rl >> 8; v = rl & 0xFF;
            if (v == 0) {                              /* escape (player.cpp:1092-1099) */
                run = (int)get_bits(d, 6);
                v = (int)get_bits(d, 8);
                g_stats.escapes++;
                if (v == 0 || v == 128) g_stats.escapes16++;
                if (v == 0) v = (int)get_bits(d, 8);
                else if (v == 128) v = (int)get_bits(d, 8) - 256;
                else if (v > 128) v -= 256;
            } else if (get_bit(d)) v = -v;
        }
        n += run;
        if (n >= 64) return -1;
        int zz = ef_zigzag[n++];
        v <<= 1;
        if (!intra) v += v < 0 ? -1 : 1;
        v = (v * d->quantizer_scale * q[zz]) / 16;
        if (v == 0) g_stats.q2_zero++;
        if ((v & 1) == 0) v -= v > 0 ? 1 : -1;         /* Q2 */
        if (v > 2047 || v < -2048) g_stats.saturated++;
        if (v > 2047) v = 2047; else if (v < -2048) v = -2048;
        b[zz] = v * ef_aan_prescale[zz];
    }

    uint8_t* dst = d->y_addr + (d->mb_x << 4);
    switch (blk) {
        case 1: dst += 8; break;
        case 2: dst += 528 * 8; break;
        case 3: dst += 528 * 8 + 8; break;
        case 4: dst = d->cr_addr + (d->mb_x << 3); break;
        case 5: dst = d->cb_addr + (d->mb_x << 3); break;
    }

    g_stats.blocks++;
    if (n == 1) {                                      /* Q5: DC-only blocks bypass the IDCT */
        int dc = b[0] >> 8;
        g_stats.blocks_dc_only++;
        if (intra) {                                   /* copy_block_dc: no clamp (Q7) */
            uint32_t w = (uint32_t)dc; w |= w << 8; w |= w << 16;
            for (int i = 0; i < 8; i++, dst += 528) { memcpy(dst, &w, 4); memcpy(dst + 4, &w, 4); }
        } else {
            for (int i = 0; i < 8; i++, dst += 528)
                for (int x = 0; x < 8; x++) dst[x] = (uint8_t)pin(dc + dst[x]);
        }
        return 0;
    }
    efo_idct(b);
    for (int i = 0; i < 8; i++, dst += 528)
        for (int x = 0; x < 8; x++) dst[x] = (uint8_t)pin(b[i * 8 + x] + (intra ? 0 : dst[x]));
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * slice (player.cpp:1238-1316)
 * ---------------------------------------------------------------------------------------- */
static void inc_mb(dec_t* d)                           /* player.cpp:823 (argument ignored, Q6) */
{
    d->mb_x += 1;
    while (d->mb_x >= d->mb_width) {
        d->mb_x -= d->mb_width;
        d->mb_y++;
        d->y_addr = get_y(d->current, d->mb_y << 4);
        d->cr_addr = d->y_addr + 352;
        d->cb_addr = d->cr_addr + 528 * 8;
    }
}

static void reset_predictors(dec_t* d) { d->y_dc = d->cr_dc = d->cb_dc = 128; d->forward_motion_h = d->forward_motion_v = 0; }

static int slice(dec_t* d, int s)
{
    d->mb_y = s - 2;
    d->mb_x = d->mb_width - 1;
    if (d->mb_y >= d->mb_height) return -1;            /* player.cpp:1257 */
    reset_predictors(d);
    d->quantizer_scale = (int)get_bits(d, 5);
    while (get_bit(d)) get_bits(d, 8);
    g_stats.slices++;

    for (int mb = 0; peek_bits(d, 23) != 0; mb++) {    /* slice_done (player.cpp:1238) */
        int increment = 0;
        int i = get_vlc(d, &T_mba);
        while (i == 34) i = get_vlc(d, &T_mba);
        while (i == 35) { increment += 33; i = get_vlc(d, &T_mba); }
        increment += i;

        if (mb == 0) inc_mb(d);
        else {
            if (increment > 1) reset_predictors(d);
            while (increment > 1) {
                inc_mb(d);
                if (d->mb_y >= 12) return -1;             /* past the frame's 12 strips: the reference writes out of bounds */
                g_stats.skipped++;
                predict_zero(d);
                cover(d, 1);
                increment--;
            }
            inc_mb(d);
        }
        if (d->mb_y >= 12) return -1;                  /* past the frame's 12 strips: the reference writes out of bounds */
        cover(d, 2);

        int mb_type = get_vlc(d, d->picture_coding_type == 1 ? &T_type_i : &T_type_p);
        int intra = mb_type & 0x01;
        g_stats.mb_type[mb_type & 31]++;
        if (d->picture_coding_type == 2 && d->full_pel_forward) g_stats.full_pel_mbs++;
        if (mb_type & 0x10) d->quantizer_scale = (int)get_bits(d, 5);
        if (intra) d->forward_motion_h = d->forward_motion_v = 0;
        else {
            d->y_dc = d->cr_dc = d->cb_dc = 128;
            if (mb_type & 0x08) {
                d->forward_motion_h = motion_vector(d, d->forward_motion_h, d->forward_r_size);
                d->forward_motion_v = motion_vector(d, d->forward_motion_v, d->forward_r_size);
            } else d->forward_motion_h = d->forward_motion_v = 0;
            predict(d);
        }
        int cbp = (mb_type & 0x02) ? get_vlc(d, &T_cbp) : intra ? 63 : 0;
        for (int k = 0, mask = 0x20; k < 6; k++, mask >>= 1)
            if (cbp & mask) block(d, k, intra);
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * run / marker (player.cpp:1318-1367)
 * ---------------------------------------------------------------------------------------- */
/* efo_walk's record of the markers efo_decode_es dispatches (NULL: not recording) */
static uint64_t* g_walk_pos;
static uint8_t* g_walk_code;
static size_t g_walk_cap, g_walk_n;

long efo_decode_es(const uint8_t* es, size_t len, int has_pts,
                   uint8_t* out_i420, size_t cap_frames, uint8_t* strips_out)
{
    tables_init();
    g_cov_n = 0;
    memset(g_cov, 0, sizeof(g_cov));
    dec_t* d = (dec_t*)calloc(1, sizeof(dec_t));
    d->es = es; d->len = len;
    d->fb[0] = (uint8_t*)calloc(1, EFO_FRAME_BYTES + 64);   /* Frame::init zero-fills (player.cpp:25) */
    d->fb[1] = (uint8_t*)calloc(1, EFO_FRAME_BYTES + 64);
    d->reference = d->fb[d->fb_index++ & 1];                /* ctor, player.cpp:354 */
    d->current = d->fb[d->fb_index & 1];
    d->have_pts = has_pts; d->last_pts = -1;
    d->out = out_i420; d->cap = cap_frames;
    d->mb_width = 22; d->mb_height = 12;
    memcpy(d->intra_q, ef_default_intra_q, 64); memset(d->non_intra_q, 16, 64);

    size_t limit = (len + 16) * 8;
    while (!d->ended && d->bitpos < limit) {
        while (peek_bits(d, 24) == 0 && d->bitpos < limit) d->bitpos++;
        const size_t at = d->bitpos;
        get_bits(d, 24);
        int m = (int)get_bits(d, 8);
        if (g_walk_n < g_walk_cap) { g_walk_pos[g_walk_n] = at; g_walk_code[g_walk_n] = (uint8_t)m; }
        g_walk_n++;
        switch (m) {
            case 0xB3: sequence(d); break;
            case 0xB8: gop(d); break;
            case 0x00: picture(d); break;
            case 0xB7: d->ended = 1; break;             /* pause() */
            case 0xB2: case 0xB5: break;
            default: if (m >= 0x01 && m <= 0xAF) slice(d, m);
        }
    }
    flush_picture(d, 1);                                    /* harness: last picture (Q10) */
    if (strips_out) { memcpy(strips_out, d->fb[0], EFO_FRAME_BYTES); memcpy(strips_out + EFO_FRAME_BYTES, d->fb[1], EFO_FRAME_BYTES); }
    long n = (long)d->n_out;
    free(d->fb[0]); free(d->fb[1]); free(d);
    return n;
}

long efo_walk(const uint8_t* es, size_t len, uint64_t* pos, uint8_t* code, size_t cap, long counts[3])
{
    g_walk_pos = pos; g_walk_code = code; g_walk_cap = pos && code ? cap : 0; g_walk_n = 0;
    efo_decode_es(es, len, 1, NULL, 0, NULL);
    const long n = (long)g_walk_n;
    if (counts) {
        counts[0] = counts[1] = counts[2] = 0;
        for (size_t i = 0; i < g_walk_n && i < g_walk_cap; i++) {
            const uint8_t m = code[i];
            counts[0] += m == 0x00; counts[1] += m >= 0x01 && m <= 0xAF; counts[2] += m == 0xB3;
        }
    }
    g_walk_pos = NULL; g_walk_code = NULL; g_walk_cap = 0; g_walk_n = 0;
    return n;
}

long efo_decode_ts(const uint8_t* ts, size_t len, uint8_t* out_i420, size_t cap_frames)
{
    uint8_t* es = (uint8_t*)malloc(len + 16);
    int64_t pts0 = -1; size_t np = 0;
    size_t n = efo_demux_ts(ts, len, es, len, NULL, &pts0, 1, &np);
    long r = efo_decode_es(es, n, np > 0 && pts0 != -1, out_i420, cap_frames, NULL);
    free(es);
    return r;
}

/* ------------------------------------------------------------------------------------------
 * Composite synthesis (video.cpp)
 * ---------------------------------------------------------------------------------------- */
#define IRE_LEVEL(x) ((uint32_t)(((x) + 40) * 255 / 3.3 / 147.5) << 8)     /* video.cpp:520 */
#define SYNC_LEVEL      IRE_LEVEL(-40)
#define BLANKING_LEVEL  IRE_LEVEL(0)
#define BLACK_LEVEL     IRE_LEVEL(7.5)

static int usec_samples(float us, float sample_rate, int spc)             /* video.cpp:554 */
{
    uint32_t r = (uint32_t)(us * sample_rate);
    return (int)(((r + spc) / (spc << 1)) * (spc << 1));
}

static int rup(float v) { if (v < 0) return -rup(-v); return (int)(v + 0.5); }           /* espflix.cpp:1071 */
static uint32_t swizzle(uint32_t uv) { return (uv & 0xFF0000FFu) | ((uv >> 8) & 0xFF00u) | ((uv << 8) & 0xFF0000u); }

/* chroma LUTs as gen_palettes derives them (espflix.cpp:1091-1180): 4 subcarrier phases per entry */
static void chroma_lut(uint32_t* dst, int use_cos, int negate)
{
    int black = (int)(BLACK_LEVEL >> 8);
    float scale = (float)black / 33;
    for (int c = 0; c < 256; c++) {
        int u = 128 - c;
        uint32_t v = 0;
        for (int i = 0; i < 4; i++) {
            double w = use_cos ? cos(2 * M_PI * i / 4) : sin(2 * M_PI * i / 4);
            if (negate) w = -w;
            int p = rup((float)(w * u * scale)) + 2 * black;
            p = p < 0 ? 0 : (p < 127 ? p : 127);
            v = (v << 8) | (uint32_t)p;
        }
        dst[c] = swizzle(v);
    }
}

void efo_video_init(efo_video* v, int ntsc)            /* video.cpp:572-630 */
{
    memset(v, 0, sizeof(*v));
    v->ntsc = ntsc;
    int spc = 4;
    if (ntsc) {
        float rate = 315.0 / 88 * spc;
        v->line_width = 228 * spc; v->line_count = 262;
        v->hsync_long = usec_samples(63.555 - 4.7, rate, spc);
        v->active_start = usec_samples(10, rate, spc);
        v->hsync = usec_samples(4.7, rate, spc);
        chroma_lut(v->color_tab, 0, 0);                /* uv_tab u */
        chroma_lut(v->color_tab + 256, 1, 0);          /* uv_tab v */
        chroma_lut(v->color_tab + 512, 1, 0);
    } else {
        float rate = 4433618.75 * spc / 1000000.0;
        v->line_width = 284 * spc; v->line_count = 312;
        v->hsync_short = usec_samples(2, rate, spc);
        v->hsync_long = usec_samples(30, rate, spc);
        v->hsync = usec_samples(4.7, rate, spc);
        v->burst_start = usec_samples(5.6, rate, spc);
        v->burst_width = (int)(10 * spc + 4) & 0xFFFE;
        v->active_start = usec_samples(10.4, rate, spc);
        float phase = 2 * M_PI / 2;
        for (int i = 0; i < v->burst_width; i++) {
            v->burst0[i] = (int16_t)(BLANKING_LEVEL + sin(phase + 3 * M_PI / 4) * BLANKING_LEVEL / 1.5);
            v->burst1[i] = (int16_t)(BLANKING_LEVEL + sin(phase - 3 * M_PI / 4) * BLANKING_LEVEL / 1.5);
            phase += 2 * M_PI / spc;
        }
        chroma_lut(v->color_tab, 0, 0);                /* sin_u */
        chroma_lut(v->color_tab + 256, 1, 0);          /* cos_v */
        chroma_lut(v->color_tab + 512, 1, 1);          /* cos_v_neg */
    }
}

static const uint32_t DITHER[8] = {                    /* video.cpp:673: 4 lines x 2 field phases */
    0x00020301, 0x03010002, 0x02030100, 0x01000203, 0x03010002, 0x00020301, 0x01000203, 0x02030100 };

static uint32_t ld32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
static void st32(uint16_t* p, uint32_t v) { memcpy(p, &v, 4); }

/* four luma pixels + two chroma samples -> eight composite samples (video.cpp:716-733) */
static uint8_t quad(uint16_t* dst, uint32_t y4, uint32_t dither, uint32_t ca, uint32_t cb, uint8_t lum)
{
    uint32_t p0 = (y4 + dither) & 0xFCFCFCFCu;
    uint32_t p1 = ((p0 >> 1) + (p0 >> 9)) & 0xFCFCFCFCu;
    p0 >>= 2; p1 >>= 2;
    lum = (uint8_t)(((uint8_t)p0 + lum) >> 1);
    st32(dst + 0, (((uint32_t)lum << 24) | ((p0 & 0xFF) << 8)) + ca);
    st32(dst + 2, ((p1 << 24) | (p0 & 0xFF00)) + (ca << 8));
    st32(dst + 4, ((p1 << 16) | (p0 >> 8)) + cb);
    st32(dst + 6, (((p1 << 8) & 0xFF000000u) | (p0 >> 16)) + (cb << 8));
    return (uint8_t)(p0 >> 24);
}

void efo_blit(const efo_video* v, const uint8_t* f, uint16_t* dst, int line, int x, int width, int frame_counter)
{
    x &= ~3;
    const uint8_t* yp = get_y((uint8_t*)f, line) + x;
    const uint8_t* up = get_cr((uint8_t*)f, line >> 1) + (x >> 1);
    const uint8_t* vp = get_cb((uint8_t*)f, line >> 1) + (x >> 1);
    if (!v->ntsc) dst += 80;
    uint32_t dither = DITHER[(line & 3) + ((frame_counter & 1) << 2)];
    int odd = line & 1;
    int n = (line >> 1) + (line == 191 ? 0 : 1);
    const uint8_t* up2 = get_cr((uint8_t*)f, n) + (x >> 1);
    const uint8_t* vp2 = get_cb((uint8_t*)f, n) + (x >> 1);
    const uint32_t* tab = v->color_tab;
    int vt = odd ? 512 : 256;                          /* CHROMA_EVEN / CHROMA_ODD */
    uint8_t lum = 0;
    for (int i = 0; i < width; i += 8) {
        uint32_t u4 = ld32(up), v4 = ld32(vp);
        if (odd) {
            u4 = ((u4 >> 1) & 0x7F7F7F7Fu) + ((ld32(up2) >> 1) & 0x7F7F7F7Fu);
            v4 = ((v4 >> 1) & 0x7F7F7F7Fu) + ((ld32(vp2) >> 1) & 0x7F7F7F7Fu);
        }
        uint32_t c[4];
        for (int k = 0; k < 4; k++)
            c[k] = ((tab[(u4 >> (8 * k)) & 0xFF] + tab[vt + ((v4 >> (8 * k)) & 0xFF)]) & 0xFCFCFCFCu) >> 2;
        lum = quad(dst, ld32(yp), dither, c[0], c[1], lum);
        lum = quad(dst + 8, ld32(yp + 4), dither, c[2], c[3], lum);
        dst += 16; yp += 8; up += 4; vp += 4; up2 += 4; vp2 += 4;
    }
}

static void fill16(uint16_t* p, uint16_t v, int n) { for (int i = 0; i < n; i++) p[i] = v; }

static void burst(const efo_video* v, uint16_t* line, int line_counter_after)   /* video.cpp:619, 806 */
{
    if (!v->ntsc) {
        const int16_t* b = (line_counter_after & 1) ? v->burst0 : v->burst1;
        for (int i = 0; i < v->burst_width; i++) line[v->burst_start + (i ^ 1)] = (uint16_t)b[i];
        return;
    }
    for (int i = v->hsync; i < v->hsync + 40; i += 4) {
        line[i + 1] = (uint16_t)BLANKING_LEVEL;
        line[i + 0] = (uint16_t)(BLANKING_LEVEL + BLANKING_LEVEL / 2);
        line[i + 3] = (uint16_t)BLANKING_LEVEL;
        line[i + 2] = (uint16_t)(BLANKING_LEVEL - BLANKING_LEVEL / 2);
    }
}

static void blanking(const efo_video* v, uint16_t* line, int vbl, int lc)        /* video.cpp:904 */
{
    int sw = vbl ? v->hsync_long : v->hsync;
    fill16(line, (uint16_t)SYNC_LEVEL, sw);
    fill16(line + sw, (uint16_t)(vbl ? BLANKING_LEVEL : BLACK_LEVEL), v->line_width - sw);
    if (!vbl) burst(v, line, lc);
}

static void pal_sync_half(const efo_video* v, uint16_t* line, int width, int lng)  /* video.cpp:917 */
{
    int sw = lng ? v->hsync_long : v->hsync_short;
    fill16(line, (uint16_t)SYNC_LEVEL, sw);
    fill16(line + sw, (uint16_t)BLANKING_LEVEL, width - sw);
}

/* composite(), video.cpp:845-887: overlay bitmap scaled into the black level, progress bar on lines 3..8 */
static void overlay(const efo_video* v, uint16_t* dst, int line, const uint8_t* bitmap, int blend, int progress)
{
    if (!blend) return;
    if (!v->ntsc) dst += 80;
    dst += 16;
    const uint8_t* src = bitmap + line * 80;
    int scale = 255 / 4;
    if (blend != -1 && blend < 32) scale = (scale * blend) >> 5;
    for (int n = 0; n < 80; n++) {
        uint32_t p = BLACK_LEVEL + src[n] * scale;
        st32(dst, (p << 16) | p);
        dst += 2;
    }
    if (line < 3 || line > 8) return;
    dst += 16;
    uint32_t c0 = BLACK_LEVEL + (scale << 8), c1 = BLACK_LEVEL + (scale << 7);
    for (int i = 0; i < 352 - 80 - 32; i += 2) {
        uint32_t c = i < progress ? c0 : c1;
        st32(dst, (c << 16) | c); st32(dst + 2, (c << 16) | c);
        dst += 4;
    }
}

void efo_field_ex(const efo_video* v, const uint8_t* strips_a, const uint8_t* strips_b, int frame_counter, int hscroll,
                  const uint8_t* bitmap, int blend, int progress, uint16_t* out)   /* video_isr, video.cpp:1122 */
{
    static const uint8_t sync_type[8] = { 0, 0, 0, 3, 3, 2, 0, 0 };
    uint16_t* lb[2];
    lb[0] = (uint16_t*)calloc((size_t)v->line_width + 64, 2);
    lb[1] = (uint16_t*)calloc((size_t)v->line_width + 64, 2);
    int top = 32 + (v->ntsc ? 0 : 32), bottom = top + 192;
    int vsync_start = v->line_count - (v->ntsc ? 3 : 8);
    for (int i = 0; i < v->line_count; i++) {
        uint16_t* buf = lb[i & 1];
        int lc = i + 1;                                 /* _line_counter after the increment */
        if (i >= top && i < bottom) {
            fill16(buf, (uint16_t)SYNC_LEVEL, v->hsync);
            burst(v, buf, lc);
            uint16_t* dst = buf + v->active_start + 16;
            const uint8_t* f = strips_a; const uint8_t* g = strips_b;
            int h = hscroll;
            if (h < 0) { h += 352; f = strips_b; g = strips_a; }       /* video.cpp:1148-1151 */
            efo_blit(v, f, dst, i - top, h, 352 - h, frame_counter);
            if (h) efo_blit(v, g, dst + (352 - h) * 2, i - top, 0, h, frame_counter);
        } else if (i >= vsync_start) {
            if (!v->ntsc) {
                uint8_t t = sync_type[i - 304];
                pal_sync_half(v, buf, v->line_width / 2, t & 2);
                pal_sync_half(v, buf + v->line_width / 2, v->line_width / 2, t & 1);
            } else blanking(v, buf, 1, lc);
        } else {
            blanking(v, buf, 0, lc);
            int ptop = bottom + 2;
            if (i >= ptop && i < ptop + 16) overlay(v, buf + v->active_start + 16, i - ptop, bitmap, blend, progress);
        }
        memcpy(out + (size_t)i * v->line_width, buf, (size_t)v->line_width * 2);
    }
    free(lb[0]); free(lb[1]);
}

void efo_field(const efo_video* v, const uint8_t* strips, int frame_counter, uint16_t* out)
{
    efo_field_ex(v, strips, strips, frame_counter, 0, NULL, 0, 0, out);
}


/* ================================================================================================
 * Trick-mode index (indexer/indexer.cpp). TEST INFRASTRUCTURE like the rest of this file.
 * ================================================================================================ */
static uint32_t idx_byte(const uint8_t* ts, size_t len, size_t i) { return i < len ? ts[i] : 0u; }
static uint32_t idx_be16(const uint8_t* ts, size_t len, size_t i) { return (idx_byte(ts, len, i) << 8) | idx_byte(ts, len, i + 1); }

/* parse_pts(), indexer.cpp:43-51 */
static int64_t idx_parse_pts(const uint8_t* ts, size_t len, size_t d, int flags)
{
    flags = (flags >> 2) & 0x30;
    if ((int)(idx_byte(ts, len, d) & 0xF0) != flags) return -1;
    int64_t n = ((int64_t)(idx_byte(ts, len, d) & 0x0E)) << 29;
    n += (int64_t)((idx_be16(ts, len, d + 1) >> 1) << 15);
    return n + (int64_t)(idx_be16(ts, len, d + 3) >> 1);
}

/* parse(), indexer.cpp:53-75: returns the 4th payload byte (the start-code value), sets pts */
static int idx_parse(const uint8_t* ts, size_t len, size_t d, int64_t* pts)
{
    *pts = 0;
    d += 6;
    const int flags = (int)idx_be16(ts, len, d);
    const size_t payload = d + 3 + idx_byte(ts, len, d + 2);
    d += 3;
    if (flags & 0x0080) *pts = idx_parse_pts(ts, len, d, flags);
    return (int)idx_byte(ts, len, payload + 3);
}

int efo_make_index(const uint8_t* ts, size_t len, int64_t* pts_out, uint32_t* pos_out, int cap, int64_t* first_pts, int64_t* last_pts)
{
    int n = 0;
    int64_t origin = -1, video_pts = -1;
    uint32_t packet = 0;
    for (size_t i = 0; i + 188 <= len; i += 188, packet++) {          /* indexer.cpp:121-171 */
        const uint8_t* d = ts + i;
        const int pid = ((d[1] << 8) + d[2]) & 0x1fff;
        size_t data = i + 4;
        if (d[3] & 0x20) data = i + 5 + d[4];                          /* adaptation field */
        if ((d[3] & 0x10) && (d[1] & 0x40) && pid == 0x100) {          /* payload present, PES starts here, video PID */
            int64_t pts;
            const int m = idx_parse(ts, len, data, &pts);
            if (m == 0xB3) {                                           /* payload begins with a sequence header */
                if (origin == -1) origin = pts;
                if (n < cap) { pts_out[n] = pts; pos_out[n] = packet; }
                n++;
            }
            video_pts = pts;
        }
    }
    *first_pts = origin; *last_pts = video_pts;
    return n;
}

int efo_pts2seq(const int64_t* pts, const uint32_t* pos188, int n, int64_t first_pts, int64_t last_pts, uint32_t bin_size,
                uint32_t* samples, int cap)
{
    if (n <= 0 || bin_size == 0) return 0;
    const int64_t end = last_pts - first_pts;
    int count = 0;
    for (int64_t t = 0; t <= end; t += bin_size, count++) {            /* indexer.cpp:211-216 */
        const int64_t want = t + first_pts;
        int mini = 0, mine = 0x7FFFFFF;                                /* pts2pos(), indexer.cpp:193-207 */
        for (int i = 0; i < n; i++) {
            int64_t diff = pts[i] - want;
            if (diff < 0) diff = -diff;
            const int e = (int)diff;
            if (e < mine) { mine = e; mini = i; }
        }
        if (count < cap) samples[count] = pos188[mini];
    }
    return count;
}

size_t efo_build_idx(const uint8_t* const ts[3], const size_t len[3], uint8_t* out, size_t cap)
{
    /* idx_hdr (indexer.cpp:22-36): sig, len, then three idx_rec {i64 first, i64 last, u32 bin, u32 speed, u32 count, pad} */
    size_t total = 104;
    uint32_t counts[3];
    for (int k = 0; k < 3; k++) {
        const int np = (int)(len[k] / 188) + 1;
        int64_t* pts = (int64_t*)malloc(sizeof(int64_t) * (size_t)np);
        uint32_t* pos = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)np);
        int64_t first, last;
        const int n = efo_make_index(ts[k], len[k], pts, pos, np, &first, &last);
        const uint32_t bin = 90000 / 12, speed = k == 0 ? 1u : 15u;
        const int cnt = efo_pts2seq(pts, pos, n, first, last, bin, NULL, 0);
        counts[k] = (uint32_t)cnt;
        if (total + 4 * (size_t)cnt <= cap) {
            efo_pts2seq(pts, pos, n, first, last, bin, (uint32_t*)(out + total), cnt);
            uint8_t* r = out + 8 + 32 * k;
            memset(r, 0, 32);
            memcpy(r, &first, 8); memcpy(r + 8, &last, 8); memcpy(r + 16, &bin, 4); memcpy(r + 20, &speed, 4); memcpy(r + 24, &counts[k], 4);
        }
        total += 4 * (size_t)cnt;
        free(pts); free(pos);
    }
    if (total > cap) return 0;
    const uint32_t sig = ('I' << 0) | ('D' << 8) | ('X' << 16), three = 3;
    memcpy(out, &sig, 4); memcpy(out + 4, &three, 4);
    return total;
}


/* ================================================================================================
 * PTS -> field pacing (video.cpp:1023-1057, 1122-1198), instant-decoder model.
 * ================================================================================================ */
static const int16_t efo_easd[16] = { 0, 8, 16, 24, 48, 72, 104, 136, 176, 216, 248, 280, 304, 328, 336, 344 };   /* _easd, video.cpp:1077 */

long efo_paced_schedule_ex(const int64_t* pts, const int* modes, int n_frames, int ntsc, uint32_t frame_counter0, long max_fields, long tail_fields,
                           uint32_t* flip_field, int* flip_line, int16_t* field_hscroll)
{
    const int line_count = ntsc ? 262 : 312;
    const int active_top = 32 + (ntsc ? 0 : 32), active_bottom = active_top + 192;      /* video.cpp:1135-1137 */
    const int vsync_start = line_count - (ntsc ? 3 : 8);
    uint32_t frame_counter = frame_counter0;
    uint32_t video_pts, pts_origin = 0, fc_origin = 0, next_time = 0;
    int current = -1, next = -1, k = 0;
    int animate = 0, animate_index = 0, hscroll = 0;                  /* _animate, _animate_index, _hscroll (video.cpp:939-942) */
    long fields = 0, tail = -1;
    while (fields < max_fields) {
        for (int i = 0; i < line_count; i++) {
            if (next == -1 && k < n_frames) {                         /* push_video(k), video.cpp:1023 */
                int64_t p = pts[k] / (ntsc ? 1500 : 1800);
                video_pts = (uint32_t)p;
                if (fc_origin == 0) { pts_origin = video_pts; fc_origin = frame_counter; }
                uint32_t d = (video_pts - pts_origin) + fc_origin;
                if (modes && modes[k]) { d = frame_counter; animate = modes[k]; }   /* non-zero mode: due now; 2 / 3 start the poster scroll, video.cpp:1039-1042 */
                if (d < frame_counter) {
                    const int late = (int)(frame_counter - d);
                    if (late > 2) fc_origin = 0;                       /* more than two fields late: re-latch the origin at the next push */
                }
                next_time = d; next = k & 1;
            }
            if (i == active_top && field_hscroll) field_hscroll[fields] = (int16_t)hscroll;
            const int active = i >= active_top && i < active_bottom && current != -1;
            if (!active && i < vsync_start) {                          /* the else branch of video_isr: flip buffers in blanking */
                if (next != -1 && frame_counter >= next_time) {
                    current = next; next = -1;
                    if (animate == 2) animate_index = -16; else if (animate == 3) animate_index = 16;     /* video.cpp:1168-1171 */
                    animate = 0;
                    /* animate(), video.cpp:1078-1088 */
                    if (animate_index == 0) hscroll = 0; else if (animate_index < 0) hscroll = -efo_easd[-(++animate_index)]; else hscroll = efo_easd[--animate_index];
                    flip_field[k] = frame_counter; flip_line[k] = i;
                    k++;
                }
            }
        }
        frame_counter++;
        fields++;
        if (animate_index == 0) hscroll = 0; else if (animate_index < 0) hscroll = -efo_easd[-(++animate_index)]; else hscroll = efo_easd[--animate_index];   /* animate() at the end of every field, video.cpp:1195 */
        if (k >= n_frames && next == -1) {
            if (tail < 0) tail = tail_fields;
            if (tail-- <= 0) break;
        }
    }
    return fields;
}

long efo_paced_schedule(const int64_t* pts, const int* modes, int n_frames, int ntsc, uint32_t frame_counter0, long max_fields,
                        uint32_t* flip_field, int* flip_line)
{
    return efo_paced_schedule_ex(pts, modes, n_frames, ntsc, frame_counter0, max_fields, 0, flip_field, flip_line, NULL);
}
