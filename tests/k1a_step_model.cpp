// tests/k1a_step_model.cpp — CPU model test of K1a's coefficient step (espflix_b200/csrc/ef_coef_step.cuh): the
// SAME header the kernel compiles is driven here on the host over encoded and random bit strings and compared,
// block by block, with a symbol-by-symbol restatement of the reference's block() loop (player.cpp:1068-1121) that
// reads the ISO code list directly (independent of the lookup table). Built and run by tests/test_k1a_step_model.py.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../espflix_b200/csrc/ef_coef_step.cuh"
#include "../espflix_b200/csrc/ef_iso11172_tables.h"

int ef_build_tables(EfTables* t);

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (uint32_t)(rng_state >> 16); }

struct Bits {
    std::vector<uint8_t> b;       // one bit per entry
    void put(uint32_t v, int n) { for (int i = n - 1; i >= 0; i--) b.push_back((v >> i) & 1); }
    void puts(const char* s) { for (; *s; s++) b.push_back(*s == '1'); }
    uint32_t window(size_t pos) const { uint32_t w = 0; for (int i = 0; i < 32; i++) w = (w << 1) | (pos + i < b.size() ? b[pos + i] : 0); return w; }
};

struct Coef { int pos, level; };
struct Result { std::vector<Coef> c; size_t bits; int end; };   // end: 0 end of block, 1 abort (position >= 64), 2 derail

// the reference's loop: first = non-intra block (n starts at 0), else n starts at 1
static Result ref_block(const Bits& B, size_t pos, bool nonintra)
{
    Result r; r.end = 2;
    int n = nonintra ? 0 : 1;
    for (;;) {
        const uint32_t w = B.window(pos);
        int run, level, len = 0;
        if (n && (w >> 30) == 2) { pos += 2; r.end = 0; break; }
        if (!n && (w >> 31)) { run = 0; level = ((w >> 30) & 1) ? -1 : 1; len = 2; }
        else if ((w >> 26) == 1) {                                           // escape
            run = (w >> 20) & 63;
            const int b = (w >> 12) & 255;
            if (b == 0) { level = (w >> 4) & 255; len = 28; }
            else if (b == 128) { level = (int)((w >> 4) & 255) - 256; len = 28; }
            else { level = (int)(int8_t)b; len = 20; }
        } else {
            for (int i = 0; i < EF_VLC_DCT_COUNT && !len; i++) {
                const char* c = ef_vlc_dct[i].code;
                const int l = (int)strlen(c);
                if (!n && l == 2) continue;
                bool ok = true;
                for (int k = 0; k < l && ok; k++) ok = (int)((w >> (31 - k)) & 1) == (c[k] == '1');
                if (!ok) continue;
                run = ef_vlc_dct[i].value >> 8; level = ef_vlc_dct[i].value & 255;
                if ((w >> (31 - l)) & 1) level = -level;
                len = l + 1;
            }
            if (!len) { r.end = 2; break; }                                  // not a code
        }
        n += run;
        pos += len;
        if (n >= 64) { r.end = 1; break; }
        r.c.push_back({ n, level });
        n++;
    }
    r.bits = pos;
    return r;
}

// K1a: one symbol per step (ef_coef_sym), a following '10' folded in by the caller exactly as the kernel does
static Result model_block(const EfTables& T, const Bits& B, size_t pos, bool nonintra)
{
    Result r; r.end = 2;
    int n = nonintra ? 0 : 1;
    bool first = nonintra;
    for (int guard = 0; guard < 200; guard++) {
        const uint32_t w = B.window(pos);
        const EfSym s = ef_coef_sym(w, first, T.dct);
        first = false;
        if (s.kind == EF_SYM_DERAIL) { r.end = 2; break; }
        int len = s.len;
        bool done = s.kind == EF_SYM_EOB;
        if (s.kind == EF_SYM_COEF) {
            n += s.run;
            if (n > 63) { pos += len; r.end = 1; break; }
            r.c.push_back({ n, s.lvl });
            n++;
            if (len <= 30 && ((w << len) >> 30) == 2u) { len += 2; done = true; }
        }
        pos += len;
        if (done) { r.end = 0; break; }
    }
    r.bits = pos;
    return r;
}

static long n_blocks = 0, n_coefs = 0;
static int compare(const EfTables& T, const Bits& B, size_t pos, bool nonintra, const char* what)
{
    const Result a = ref_block(B, pos, nonintra), m = model_block(T, B, pos, nonintra);
    n_blocks++; n_coefs += (long)a.c.size();
    bool ok = a.end == m.end && a.c.size() == m.c.size() && (a.end == 2 || a.bits == m.bits);
    for (size_t i = 0; ok && i < a.c.size(); i++) ok = a.c[i].pos == m.c[i].pos && a.c[i].level == m.c[i].level;
    if (!ok) {
        fprintf(stderr, "MISMATCH (%s, %s): ref end %d coefs %zu bits %zu / model end %d coefs %zu bits %zu\n", what, nonintra ? "non-intra" : "intra",
                a.end, a.c.size(), a.bits - pos, m.end, m.c.size(), m.bits - pos);
        for (size_t i = 0; i < a.c.size() || i < m.c.size(); i++)
            fprintf(stderr, "  %2zu: ref (%d,%d) model (%d,%d)\n", i, i < a.c.size() ? a.c[i].pos : -1, i < a.c.size() ? a.c[i].level : 0,
                    i < m.c.size() ? m.c[i].pos : -1, i < m.c.size() ? m.c[i].level : 0);
        return 1;
    }
    return 0;
}

int main()
{
    static EfTables T;
    if (ef_build_tables(&T)) { fprintf(stderr, "table build failed\n"); return 2; }
    int bad = 0;
    // 1. encoded blocks: random (run, level) sequences drawn with a bias to the short codes, escapes mixed in,
    //    ending with '10'; sometimes running past position 63 (abort) or cut by garbage (derail)
    for (int it = 0; it < 200000 && bad < 5; it++) {
        Bits B;
        const bool nonintra = rnd() & 1;
        int n = nonintra ? 0 : 1;
        const int want = 1 + rnd() % 24;
        for (int k = 0; k < want; k++) {
            const uint32_t pick = rnd() % 100;
            if (pick < 4) {                                                   // escape
                const int run = rnd() % 20, lv = (int)(rnd() % 511) - 255;
                B.puts("000001"); B.put((uint32_t)run, 6);
                if (lv > -128 && lv < 128 && lv != 0 && (rnd() & 3)) B.put((uint32_t)lv & 255, 8);
                else if (lv >= 0) { B.put(0, 8); B.put((uint32_t)lv & 255, 8); }
                else { B.put(128, 8); B.put((uint32_t)(lv + 256) & 255, 8); }
                n += run + 1;
            } else {
                const int idx = pick < 70 ? (int)(rnd() % 8) : pick < 92 ? (int)(rnd() % 31) : (int)(rnd() % EF_VLC_DCT_COUNT);
                const char* c = ef_vlc_dct[idx].code;
                if (k == 0 && nonintra && strlen(c) == 2) B.puts("1"); else B.puts(c);
                B.put(rnd() & 1, 1);
                n += (ef_vlc_dct[idx].value >> 8) + 1;
            }
            if (n > 70) break;
        }
        if (rnd() % 50) B.puts("10");
        B.put(rnd(), 32); B.put(rnd(), 32);                                    // whatever follows
        bad += compare(T, B, 0, nonintra, "encoded");
    }
    // 2. garbage: random bits, zero runs, all ones
    for (int it = 0; it < 200000 && bad < 5; it++) {
        Bits B;
        for (int k = 0; k < 12; k++) B.put((rnd() % 7 == 0) ? 0u : rnd(), 32);
        bad += compare(T, B, rnd() % 32, rnd() & 1, "random");
    }
    // 3. every 10-bit prefix, both contexts, followed by zeros, ones or random bits
    for (int ctx = 0; ctx < 2 && bad < 5; ctx++)
        for (uint32_t p = 0; p < 1024 && bad < 5; p++)
            for (int fill = 0; fill < 4 && bad < 5; fill++) {
                Bits B; B.put(p, 10); B.put(fill == 0 ? 0u : fill == 1 ? 0xFFFFFFFFu : rnd(), 32); B.put(rnd(), 32); B.put(rnd(), 32);
                bad += compare(T, B, 0, ctx == 1, "prefix");
            }
    // 4. list entry: pack/unpack round trip over the whole value range, as K1b reads it
    for (int n = 0; n < 128 && bad < 5; n++)
        for (int level = -255; level <= 255; level += 1)
            for (int qs = 1; qs <= 31; qs += 5) {
                const int intra = n < 64, k = intra ? 0 : 1;
                const uint32_t z = T.qz[n];
                const int zz = ef_zigzag[n & 63], q = (int)(z & 255);
                int v = 2 * level; if (!intra) v += (v < 0 ? -1 : (level == 0 ? 1 : 1)) * (level == 0 ? 1 : 1);
                if (!intra && level == 0) v = 1;                              // v = 0 -> +1 (the reference's v < 0 ? -1 : 1)
                v = (v * qs * q) / 16;
                if ((v & 1) == 0) v -= v > 0 ? 1 : -1;
                if (v > 2047) v = 2047; else if (v < -2048) v = -2048;
                const int want = v * ef_aan_prescale[zz];
                const uint32_t blk = (uint32_t)(n % 6);
                const uint32_t ent = ef_coef_entry(z, level, qs, k, blk << 24);
                const uint32_t hi = ent + 0x20000u;
                const int got = ((int)(ent << 14)) >> 14, gb = (hi >> 24) & 7, gp = (hi >> 18) & 63;
                if (got != want || gb != (int)blk || gp != zz) {
                    fprintf(stderr, "ENTRY MISMATCH n %d level %d qs %d: want %d blk %u pos %d, got %d blk %d pos %d\n", n, level, qs, want, blk, zz, got, gb, gp);
                    bad++;
                }
            }
    printf("{\"blocks\": %ld, \"coefficients\": %ld, \"bad\": %d}\n", n_blocks, n_coefs, bad);
    return bad ? 1 : 0;
}
