// espflix_b200/csrc/ef_composite.cu — K2, the composite field kernel: one launch synthesises a whole
// NTSC (262 x 912) or PAL (312 x 1136) field of uint16 DAC samples for every stream.
//
// Replaces one field's worth of video_isr() calls (video.cpp:1122-1198): sync(), burst() /
// burst_pal(), blit() (video.cpp:690-804), blanking(), pal_sync(). The reference rewrites only part
// of a two-entry ping-pong line buffer on active lines; the closed form of what the DAC sees is
// (SURVEY.md §8a a19):
//   NTSC active line: sync [0,64) | burst [64,104) | BLACK [104,160) | blit [160,864) | BLACK [864,912)
//   PAL  active line: sync [0,80) | BLACK [80,96) | burst [96,140) | BLACK [140,280) | blit [280,984) | BLACK [984,1136)
// Pure streaming, HBM bound: each thread produces 8 samples (one 16-byte store) from 4 luma pixels
// and 2+2 chroma bytes; the packed 4x8-bit expressions of blit() are reproduced verbatim because
// the low byte of every sample carries deterministic carry "junk" that parity depends on.
// Paced presentation can also emit what the DAC plays instead of the line buffer: one byte per sample (EF_FIELD_DAC8, dac_word).
#include <type_traits>

#include "ef_common.cuh"

namespace {

__device__ __forceinline__ uint32_t chroma_word(const uint32_t* tab, uint32_t u, uint32_t v, int vt)
{
    return ((tab[u & 255] + tab[vt + (v & 255)]) & 0xFCFCFCFCu) >> 2;      // CHROMA_EVEN / CHROMA_ODD, video.cpp:670
}

// The chroma LUTs have a closed form (tests/test_tables.py::test_chroma_lut_closed_form checks all 768 entries of
// both standards): the four subcarrier phases of a table entry are 48, 48 +- r(c) with
//   r(c) = sgn(128 - c) * ((16 |128 - c| + 11) / 22)          [= round_half_away((128 - c) * 24 / 33), espflix.cpp:1091-1180]
// clamped to [0, 127]: U rides on the sine phases (bytes 1, 0), V on the cosine phases (bytes 3, 2; swapped on the PAL
// lines that use cos_v_neg).

// compile-time geometry of the two standards (video_init / pal_init, video.cpp:572-630; values
// probe-verified against the reference in tests/golden/composite_pins.json)
template <bool kNtsc> struct Geo;
template <> struct Geo<true> {
    static constexpr int W = 912, LINES = 262, HSYNC = 64, HSYNC_LONG = 840, HSYNC_SHORT = 0, BURST_START = 64, BURST_W = 40,
                         TOP = 32, VSYNC = 259, BLIT = 160;
};
template <> struct Geo<false> {
    static constexpr int W = 1136, LINES = 312, HSYNC = 80, HSYNC_LONG = 536, HSYNC_SHORT = 32, BURST_START = 96, BURST_W = 44,
                         TOP = 64, VSYNC = 304, BLIT = 280;
};

template <bool kNtsc>
__device__ __forceinline__ uint32_t blank_sample(const int16_t* pal_burst, int line, int x)
{
    using G = Geo<kNtsc>;
    const uint32_t SYNC = 0x0000, BLANKING = 0x1400, BLACK = 0x1800;       // IRE(-40), IRE(0), IRE(7.5): video.cpp:520-525
    if (line >= G::VSYNC) {
        if (kNtsc) return x < G::HSYNC_LONG ? SYNC : BLANKING;             // blanking(buf, true)
        const uint32_t types = 0x00233000u;                                // _sync_type[8] = {0,0,0,3,3,2,0,0}, one nibble each
        const int t = (types >> ((line - G::VSYNC) * 4)) & 15;
        const int half = G::W >> 1;
        const int second = x >= half;
        const int xx = second ? x - half : x;
        const int lng = second ? (t & 1) : (t & 2);
        return xx < (lng ? G::HSYNC_LONG : G::HSYNC_SHORT) ? SYNC : BLANKING; // pal_sync2
    }
    if (x < G::HSYNC) return SYNC;
    const int i = x - G::BURST_START;
    if (i >= 0 && i < G::BURST_W) {
        if (kNtsc) return (i & 1) ? BLANKING : ((i & 2) ? 0x0A00u : 0x1E00u);   // burst(), video.cpp:806: 10 cycles of [1E00 1400 0A00 1400]
        return (uint16_t)pal_burst[(((line + 1) & 1) ? 0 : 64) + (i ^ 1)];     // burst_pal(): pair-swapped, table chosen by (_line_counter after ++) & 1
    }
    return BLACK;
}

__constant__ uint32_t c_dither[8] = {                                     // dither4x4, video.cpp:673
    0x00020301, 0x03010002, 0x02030100, 0x01000203, 0x03010002, 0x00020301, 0x01000203, 0x02030100 };

}  // namespace

// eight samples (one 16-byte chunk) of a blank / vsync line, or of an active line outside the blit span
// (which still shows what blanking() last left in the ping-pong buffer: sync, burst, BLACK). Most chunks lie
// wholly inside one constant region: decide per chunk, go per sample only at the burst, on the vsync lines
// and under the overlay.
template <bool kNtsc>
__device__ __forceinline__ uint4 blank_chunk(const EfDev& D, const EfPresent& pr, int line, int x0)
{
    using G = Geo<kNtsc>;
    const uint32_t SYNC2 = 0x00000000u, BLACK2 = 0x18001800u;
    uint32_t w[4];
    const int ol = line - (G::TOP + EF_H + 2);                             // overlay line 0..15 (video.cpp:1183-1189)
    if (pr.blend != 0 && ol >= 0 && ol < 16 && x0 >= G::BLIT + 16 && x0 < G::BLIT + 16 + 160 + 16 + 480) {
        // composite(), video.cpp:845-887: 80 bitmap bytes -> 160 samples, then (lines 3..8) a 480-sample progress bar
        int scale = 255 / 4;
        if (pr.blend != -1 && pr.blend < 32) scale = (scale * pr.blend) >> 5;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int s = x0 + 2 * i - (G::BLIT + 16);                     // both samples of a word share the source byte / bar step
            uint32_t v = 0x1800u;
            if (s < 160) v = 0x1800u + (uint32_t)pr.bitmap[ol * 80 + (s >> 1)] * (uint32_t)scale;
            else if (s >= 176 && ol >= 3 && ol <= 8) v = 0x1800u + ((uint32_t)scale << ((((s - 176) >> 2) * 2 < pr.progress) ? 8 : 7));
            w[i] = (v & 0xFFFFu) | (v << 16);
        }
    } else if (line < G::VSYNC && x0 + 8 <= G::HSYNC) w[0] = w[1] = w[2] = w[3] = SYNC2;
    else if (line < G::VSYNC && (x0 >= G::BURST_START + G::BURST_W || (x0 >= G::HSYNC && x0 + 8 <= G::BURST_START))) w[0] = w[1] = w[2] = w[3] = BLACK2;
    else {
#pragma unroll
        for (int i = 0; i < 4; i++)
            w[i] = blank_sample<kNtsc>(D.pal_burst, line, x0 + 2 * i) | (blank_sample<kNtsc>(D.pal_burst, line, x0 + 2 * i + 1) << 16);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// four luma pixels + two chroma phase words -> eight samples (video.cpp:716-733, verbatim packed arithmetic)
__device__ __forceinline__ uint4 blit_quad(uint32_t y4, uint32_t dither, uint32_t ca, uint32_t cb, uint32_t& lum)
{
    uint32_t p0 = (y4 + dither) & 0xFCFCFCFCu;
    uint32_t p1 = ((p0 >> 1) + (p0 >> 9)) & 0xFCFCFCFCu;
    p0 >>= 2; p1 >>= 2;
    const uint32_t l = (((p0 & 0xFF) + lum) >> 1) & 0xFF;
    lum = p0 >> 24;
    return make_uint4(((l << 24) | ((p0 & 0xFF) << 8)) + ca, ((p1 << 24) | (p0 & 0xFF00)) + (ca << 8),
                      ((p1 << 16) | (p0 >> 8)) + cb, (((p1 << 8) & 0xFF000000u) | (p0 >> 16)) + (cb << 8));
}

// EF_FIELD_DAC8: what the video DAC plays. The I2S unit sends the two 16-bit halves of each word in swapped order (burst_pal()
// writes line[i ^ 1] = b[i], video.cpp:640-644; blit() stores each pixel before the sample interpolated ahead of it,
// video.cpp:727-733), so buffer sample t ^ 1 plays at time t, and only its high byte drives the 8-bit DAC. Two words holding
// samples 0..3 give the bytes played as samples 1, 0, 3, 2: one byte permute per pair of words.
__device__ __forceinline__ uint32_t dac_word(uint32_t w0, uint32_t w1) { return __byte_perm(w0, w1, 0x5713); }
__device__ __forceinline__ uint2 dac_chunk(uint4 c) { return make_uint2(dac_word(c.x, c.y), dac_word(c.z, c.w)); }   // 8 samples -> 8 bytes

template <bool kDac8> using K2Out = std::conditional_t<kDac8, uint8_t, uint16_t>;   // one output sample

// ---- K2 v6: a CTA synthesises a BAND of 16 consecutive lines of one stream in shared memory and hands the finished
// rows to the TMA engine (cp.async.bulk.global.shared::cta): the field leaves the SM as bulk stores instead of 16-byte
// STG, which took the output off the L1/TEX pipe - the v4 kernel was bound there (86 % busy at 42 % DRAM throughput,
// profiles/r01_k2_details.txt). Bands coincide with macroblock rows of the tiled frame (the active area starts at
// line 32 / 64), so the loads follow the tile layout: a warp takes two 8-pixel groups x 16 rows = 256 contiguous luma
// bytes and 2 x 64 contiguous chroma bytes of ONE tile (2 + 1 + 1 L1 wavefronts instead of 8 + 8 + 8 when its lanes
// ran along a scan line). What is NOT picture is constant and is not recomputed per line (v5 did, and was bound by
// instruction issue: profiles/r02_k2v5_ncu.txt):
//   * a blank band synthesises each DISTINCT line once (NTSC: one; PAL: two burst phases; the vertical sync types; the
//     overlay lines) and bulk-stores that one shared-memory row to every field line that shows it;
//   * an active band synthesises sync / burst / black margins for two rows (the two PAL burst phases) and stores every
//     line as three bulk copies: left margin and right margin from the template row, the blit span from the line's own.
// Shared-memory rows are padded by 16 bytes: the 16-byte stores of 8 consecutive rows then hit 32 distinct banks.
// grid: x = band (17 NTSC / 20 PAL), y = stream; 352 threads = 11 warps x 2 tile columns = the 22 macroblocks of a row.
#ifndef EF_K2_THREADS
#define EF_K2_THREADS 352
#endif
constexpr int kK2Threads = EF_K2_THREADS;             // 352 (2 tile-column tasks per warp) or 704 (1)
constexpr int kK2Tasks = 22 / (kK2Threads / 32);
static_assert(kK2Tasks * (kK2Threads / 32) == 22, "the 22 macroblock columns of a row must divide over the warps");

__device__ __forceinline__ void bulk_store(void* gdst, const void* ssrc, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gdst), "r"((uint32_t)__cvta_generic_to_shared(ssrc)), "r"(bytes) : "memory");
}

// which blank lines look alike: lines of one class are sample-identical
template <bool kNtsc>
__device__ __forceinline__ int blank_class(const EfPresent& pr, int line)
{
    using G = Geo<kNtsc>;
    if (line >= G::VSYNC) return kNtsc ? 1 : 16 + (int)((0x00233000u >> ((line - G::VSYNC) * 4)) & 15u);   // _sync_type[], as in blank_sample()
    const int ol = line - (G::TOP + EF_H + 2);
    if (pr.blend != 0 && ol >= 0 && ol < 16) return 64 + ol;              // overlay rows differ line by line
    return kNtsc ? 0 : ((line + 1) & 1) + 2;                              // PAL: the burst table alternates (burst_pal())
}

// kPaced (ef_present_*): y = the field's slot; stream, frame store, frame counter and hscroll come from desc[y], the field goes
// to dst + y * LINES * W, and the overlay is off. Otherwise y = stream and the field goes to the stream's field buffer.
// kOverlay (paced only): the overlay is on, with blend, progress and bitmap slot from fovl[y]; pr.bitmap is the base of the
// bitmap slots, two per stream.
// kGated (paced only, ef_present_*_async): the grid follows the caller's capacity, not the call's fields; a CTA whose output slot
// slot0 + y is at or past *total (ef_pace_size_kernel: the call's fields, 0 when its chain failed) exits at once.
// kDac8 (paced only, ef_present_format EF_FIELD_DAC8): rows are built as DAC bytes in playback order (dac_word), and the field is
// one byte per sample. An active line's own row then spans X0..X1: PAL's blit span [280, 984) is 8 mod 16 at both ends and bulk
// copies move 16-byte aligned runs, so PAL rows also carry the black margin bytes 272..279 and 984..991 and a line is cut at
// [0, 272) | [272, 992) | [992, 1136).
template <bool kNtsc, bool kPaced, bool kOverlay = false, bool kGated = false, bool kDac8 = false>
__global__ void __launch_bounds__(kK2Threads)
ef_composite_kernel(const EfDev* __restrict__ Dp, int fb_sel, int frame_counter, const EfPresent pr, const EfFieldDesc* __restrict__ desc,
                    K2Out<kDac8>* __restrict__ dst, const EfFieldOverlay* __restrict__ fovl = nullptr, const uint64_t* __restrict__ total = nullptr,
                    uint64_t slot0 = 0)
{
    static_assert(kPaced || !kOverlay, "the per-field overlay is a paced variant");
    static_assert(kPaced || !kGated, "the gate is on the paced variant");
    static_assert(kPaced || !kDac8, "the DAC byte format is a paced variant");
    if constexpr (kGated) {
        if (slot0 + blockIdx.y >= *total) return;
    }
    using G = Geo<kNtsc>;
    constexpr int OB = kDac8 ? 1 : 2;                                      // bytes per output sample
    constexpr int CPL = G::W / 8;                                          // 8-sample chunks per line
    constexpr int LB = G::W * OB, LS = LB + 16;                            // bytes per line in the field / in shared memory
    constexpr int BLIT_C = G::BLIT / 8, BLIT_N = 2 * EF_W / 8;             // the blit span in chunks: [BLIT_C, BLIT_C + 88)
    constexpr int MARGIN_N = CPL - BLIT_N;                                 // chunks of a line outside it
    constexpr int X0 = (G::BLIT * OB) % 16 ? G::BLIT - 8 : G::BLIT;        // the samples a line takes from its own row: [X0, X1)
    constexpr int X1 = (G::BLIT * OB) % 16 ? G::BLIT + 2 * EF_W + 8 : G::BLIT + 2 * EF_W;
    static_assert(X0 * OB % 16 == 0 && X1 * OB % 16 == 0 && LB % 16 == 0, "bulk copies move 16-byte aligned runs");
    __shared__ __align__(128) uint8_t sm[16 * LS];
    __shared__ int s_src[16], s_distinct[16], s_n;
    const EfDev& D = *Dp;
    const uint32_t* tab = D.color_tab;                                     // 3 KB chroma LUT through L1
    const int line0 = (int)blockIdx.x * 16;
    int stream = (int)blockIdx.y;
    EfPresent p = pr;
    K2Out<kDac8>* out0;
    if constexpr (kPaced) {
        const EfFieldDesc f = desc[blockIdx.y];
        stream = (int)f.stream; fb_sel = f.fb; frame_counter = (int)f.frame_counter; p.hscroll = f.hscroll;
        if constexpr (kOverlay) {
            const EfFieldOverlay v = fovl[blockIdx.y];
            p.blend = v.blend; p.progress = v.progress;
            p.bitmap = pr.bitmap + ((size_t)stream * 2 + v.slot) * EF_OVERLAY_BYTES;
        } else {
            p.blend = 0;
        }
        out0 = dst + (size_t)blockIdx.y * (G::LINES * G::W) + (size_t)line0 * G::W;
    } else {
        out0 = D.fields + (size_t)stream * D.field_stride + (size_t)line0 * G::W;
    }
    const int nlines = min(16, G::LINES - line0);
    const int fl0 = line0 - G::TOP;                                        // frame line of the band's first line (bands = macroblock rows)
    const bool active = fl0 >= 0 && fl0 < EF_H && fb_sel != -2;            // -2: no frame presented yet (video.cpp:1140)

    if (!active) {
        // ---- blank band: every distinct line once ------------------------------------------------------------------
        if (threadIdx.x == 0) {
            int n = 0;
            for (int l = 0; l < nlines; l++) {
                const int c = blank_class<kNtsc>(p, line0 + l);
                int src = l;
                for (int k = 0; k < l; k++) if (blank_class<kNtsc>(p, line0 + k) == c) { src = k; break; }
                s_src[l] = src;
                if (src == l) s_distinct[n++] = l;
            }
            s_n = n;
        }
        __syncthreads();
        const int n = s_n;
        for (int i = (int)threadIdx.x; i < n * CPL; i += kK2Threads) {
            const int l = s_distinct[i / CPL], c = i % CPL;
            if constexpr (kDac8) *(uint2*)(sm + l * LS + c * 8) = dac_chunk(blank_chunk<kNtsc>(D, p, line0 + l, c * 8));
            else *(uint4*)(sm + l * LS + c * 16) = blank_chunk<kNtsc>(D, p, line0 + l, c * 8);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> async proxy
        __syncthreads();
        if ((int)threadIdx.x < nlines) {
            bulk_store(out0 + (size_t)threadIdx.x * G::W, sm + s_src[threadIdx.x] * LS, LB);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); // shared memory must stay valid until the engine has read it
        }
        return;
    }

    // ---- active band: margins of the two template rows (rows 0 and 1: even / odd field line) ----------------------------
    for (int i = (int)threadIdx.x; i < 2 * MARGIN_N; i += kK2Threads) {
        const int l = i / MARGIN_N, k = i % MARGIN_N;
        const int c = k >= BLIT_C ? k + BLIT_N : k;
        if constexpr (kDac8) *(uint2*)(sm + l * LS + c * 8) = dac_chunk(blank_chunk<kNtsc>(D, p, line0 + l, c * 8));
        else *(uint4*)(sm + l * LS + c * 16) = blank_chunk<kNtsc>(D, p, line0 + l, c * 8);
    }
    if constexpr (X0 != G::BLIT) {                                         // the margin chunks of rows 2..15 that their lines copy
        for (int i = (int)threadIdx.x; i < 2 * 14; i += kK2Threads) {
            const int l = 2 + (i >> 1), c = (i & 1) ? BLIT_C + BLIT_N : BLIT_C - 1;
            *(uint2*)(sm + l * LS + c * 8) = dac_chunk(blank_chunk<kNtsc>(D, p, line0 + l, c * 8));
        }
    }
    {
        const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
        const int row = lane & 15, fl = fl0 + row;                         // frame line 0..191
        int fb0 = fb_sel >= 0 ? fb_sel : (int)((D.base_pics[stream] + D.n_pics[stream]) & 1u);
        // two-frame horizontal scroll (video.cpp:1146-1154): blit(f, dst, i, h, 352-h) then blit(f^1, dst + (352-h)*2, i, 0, h)
        int h = p.hscroll;
        if (h < 0) { h += EF_W; fb0 ^= 1; }
        const int split = (EF_W - h) >> 3;                                 // first 8-pixel group drawn by the second blit
        const uint32_t dither = c_dither[(fl & 3) + ((frame_counter & 1) << 2)];
        const int cy = fl >> 1, ncy = cy + (fl == 191 ? 0 : 1);            // odd lines average with the next chroma row (video.cpp:704-716)
        const int yoff = (fl >> 4) * EF_MBW_MAX * EF_TILE + (fl & 15) * 16;
        const int coff = (cy >> 3) * EF_MBW_MAX * EF_TILE + (cy & 7) * 8 + 256;      // get_cr(line>>1); get_cb is the next 64-byte plane
        const int noff = (fl & 1) ? (ncy >> 3) * EF_MBW_MAX * EF_TILE + (ncy & 7) * 8 + 256 : coff;
        const int vt = (fl & 1) ? 512 : 256;
        const uint8_t* fbase = D.frames + ef_frame_offset(stream, 0);
        // the warp's two tasks (destination groups gd and gd + 22): all loads first, then the arithmetic
        uint32_t u4[kK2Tasks], v4[kK2Tasks], un[kK2Tasks], vn[kK2Tasks], lumw[kK2Tasks];
        uint2 y8[kK2Tasks];
        bool cstart[kK2Tasks];
#pragma unroll
        for (int t = 0; t < kK2Tasks; t++) {
            const int gd = warp * 2 + (lane >> 4) + t * (44 / kK2Tasks);   // destination group 0..43
            const bool second = gd >= split;
            const int g = second ? gd - split : gd + (h >> 3);             // 8-pixel group of the source frame
            cstart[t] = second ? g == 0 : gd == 0;                         // blit() starts its luma carry at 0
            const uint8_t* f = fbase + (size_t)(fb0 ^ (int)second) * EF_FRAME;
            const int tcol = (g >> 1) * EF_TILE, sub = g & 1;
            u4[t] = *(const uint32_t*)(f + coff + tcol + sub * 4);
            v4[t] = *(const uint32_t*)(f + coff + tcol + sub * 4 + 64);
            un[t] = *(const uint32_t*)(f + noff + tcol + sub * 4);
            vn[t] = *(const uint32_t*)(f + noff + tcol + sub * 4 + 64);
            y8[t] = *(const uint2*)(f + yoff + tcol + sub * 8);
            const int q = cstart[t] ? 0 : 2 * g - 1;                       // previous 4-pixel group
            lumw[t] = *(const uint32_t*)(f + yoff + (q >> 2) * EF_TILE + (q & 3) * 4);
        }
#pragma unroll
        for (int t = 0; t < kK2Tasks; t++) {
            const int gd = warp * 2 + (lane >> 4) + t * (44 / kK2Tasks);
            uint32_t u = u4[t], v = v4[t];
            if (fl & 1) {
                u = ((u >> 1) & 0x7F7F7F7Fu) + ((un[t] >> 1) & 0x7F7F7F7Fu);
                v = ((v >> 1) & 0x7F7F7F7Fu) + ((vn[t] >> 1) & 0x7F7F7F7Fu);
            }
            uint32_t lum = cstart[t] ? 0u : ((((lumw[t] + dither) & 0xFCFCFCFCu) >> 2) >> 24);   // carry = last pixel of the previous group
            const uint4 o0 = blit_quad(y8[t].x, dither, chroma_word(tab, u, v, vt), chroma_word(tab, u >> 8, v >> 8, vt), lum);
            const uint4 o1 = blit_quad(y8[t].y, dither, chroma_word(tab, u >> 16, v >> 16, vt), chroma_word(tab, u >> 24, v >> 24, vt), lum);
            uint8_t* o = sm + row * LS + (G::BLIT + gd * 16) * OB;
            if constexpr (kDac8) {                                         // 16 samples -> 16 bytes
                const uint4 b = make_uint4(dac_word(o0.x, o0.y), dac_word(o0.z, o0.w), dac_word(o1.x, o1.y), dac_word(o1.z, o1.w));
                if constexpr (G::BLIT % 16 == 0) *(uint4*)o = b;
                else {                                                     // PAL: 8 mod 16
                    *(uint2*)o = make_uint2(b.x, b.y);
                    *(uint2*)(o + 8) = make_uint2(b.z, b.w);
                }
            } else {
                *(uint4*)o = o0;
                *(uint4*)(o + 16) = o1;
            }
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x < 16) {
        const int l = (int)threadIdx.x;
        K2Out<kDac8>* out = out0 + (size_t)l * G::W;
        const uint8_t* tmpl = sm + (l & 1) * LS;
        bulk_store(out, tmpl, X0 * OB);
        bulk_store(out + X0, sm + l * LS + X0 * OB, (X1 - X0) * OB);
        bulk_store(out + X1, tmpl + X1 * OB, (G::W - X1) * OB);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
}

// single blit() call into a device buffer (line-blit entry point; used by ef_blit): one thread per 4 luma pixels
__global__ void ef_blit_kernel(const EfDev* __restrict__ Dp, int stream, int fb, int fl, int x, int width, int frame_counter, uint16_t* __restrict__ dst)
{
    const EfDev& D = *Dp;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;                   // group index relative to x
    x &= ~3;
    if (q * 4 >= width) return;
    const uint8_t* f = D.frames + ef_frame_offset(stream, fb);
    const uint32_t dither = c_dither[(fl & 3) + ((frame_counter & 1) << 2)];
    const int g = (x >> 2) + q;                                            // absolute 4-pixel group index
    const int cy = fl >> 1;
    const int ycol = (g >> 2) * EF_TILE + (g & 3) * 4, ccol = (g >> 2) * EF_TILE + 256 + (g & 3) * 2;
    const uint8_t* yrow = f + (fl >> 4) * EF_MBW_MAX * EF_TILE + (fl & 15) * 16;
    const uint8_t* crow = f + (cy >> 3) * EF_MBW_MAX * EF_TILE + (cy & 7) * 8;
    uint32_t u2 = *(const uint16_t*)(crow + ccol);
    uint32_t v2 = *(const uint16_t*)(crow + ccol + 64);
    int vt = 256;
    if (fl & 1) {
        const int n = cy + (fl == 191 ? 0 : 1);
        const uint8_t* nrow = f + (n >> 3) * EF_MBW_MAX * EF_TILE + (n & 7) * 8;
        const uint32_t ub = *(const uint16_t*)(nrow + ccol);
        const uint32_t vb = *(const uint16_t*)(nrow + ccol + 64);
        u2 = ((u2 >> 1) & 0x7F7Fu) + ((ub >> 1) & 0x7F7Fu);
        v2 = ((v2 >> 1) & 0x7F7Fu) + ((vb >> 1) & 0x7F7Fu);
        vt = 512;
    }
    const uint32_t* tab = D.color_tab;
    const uint32_t ca = chroma_word(tab, u2, v2, vt), cb = chroma_word(tab, u2 >> 8, v2 >> 8, vt);
    uint32_t lum = 0;
    if (q > 0) lum = ((((*(const uint32_t*)(yrow + ((g - 1) >> 2) * EF_TILE + ((g - 1) & 3) * 4) + dither) & 0xFCFCFCFCu) >> 2) >> 24);
    uint32_t p0 = (*(const uint32_t*)(yrow + ycol) + dither) & 0xFCFCFCFCu;
    uint32_t p1 = ((p0 >> 1) + (p0 >> 9)) & 0xFCFCFCFCu;
    p0 >>= 2; p1 >>= 2;
    lum = (((p0 & 0xFF) + lum) >> 1) & 0xFF;
    uint32_t* o = (uint32_t*)(dst + q * 8);
    o[0] = ((lum << 24) | ((p0 & 0xFF) << 8)) + ca;
    o[1] = ((p1 << 24) | (p0 & 0xFF00)) + (ca << 8);
    o[2] = ((p1 << 16) | (p0 >> 8)) + cb;
    o[3] = (((p1 << 8) & 0xFF000000u) | (p0 >> 16)) + (cb << 8);
}

cudaError_t ef_launch_composite(const EfDev* dev, int n_streams, const EfGeometry& g, int fb, int frame_counter, const EfPresent& pr, cudaStream_t stream)
{
    const dim3 bands((unsigned)(g.line_count + 15) / 16, (unsigned)n_streams);
    if (g.ntsc) ef_composite_kernel<true, false><<<bands, kK2Threads, 0, stream>>>(dev, fb, frame_counter, pr, nullptr, nullptr);
    else ef_composite_kernel<false, false><<<bands, kK2Threads, 0, stream>>>(dev, fb, frame_counter, pr, nullptr, nullptr);
    return cudaGetLastError();
}

// ---- paced presentation (ef_present_*): push_video's PTS -> field schedule (video.cpp:1023-1057) against the flip of video_isr
// (video.cpp:1122-1198), instant-decoder model, one thread per stream. A push runs push_video's arithmetic at the display's
// position, then "draws" lines up to the flip: the first line below vsync_start that is not an active line of a presented
// frame, once the frame counter has reached _next_frame_time. Closed form: the flip is in the current field or at line 0 of a
// later one, so no loop walks lines or fields (a PTS jump of 2^33 ticks costs nothing here; the caller then lacks the room).
// The fields a call emits are those whose line active_bottom - 1 it draws; animate() (video.cpp:1076-1088) runs at every field
// end and at the flip. The state is written to `next` and committed by ef_pace_fill_kernel once the output fits.
namespace {
__constant__ int16_t c_easd[16] = { 0, 8, 16, 24, 48, 72, 104, 136, 176, 216, 248, 280, 304, 328, 336, 344 };   // _easd, video.cpp:1077

__device__ __forceinline__ int pace_animate(int ai, uint64_t n)            // _animate_index after n animate() calls
{
    const uint64_t a = (uint64_t)abs(ai);
    return a <= n ? 0 : ai > 0 ? ai - (int)n : ai + (int)n;
}
__device__ __forceinline__ int pace_hscroll(int ai) { return ai < 0 ? -c_easd[-ai] : c_easd[ai]; }   // _hscroll once animate() left ai
}  // namespace

// pic >= 0: every stream with a picture `pic` pushes it (pts from pic_pts, modes[s] or 0); pic < 0: every stream idles until
// it has emitted idle_n[s] fields. lib_modes (NULL unless the context has library posters): the poster mode the current submit
// carries for each stream (ef_library_submit), used for the stream's last picture of the submit where modes[s] is 0. ovl (NULL
// unless the context stages overlays): the staged overlay changes latch, into ovl_next, when the call draws line 0 of their latch field
__global__ void ef_pace_kernel(const EfPaceState* __restrict__ st, EfPaceState* __restrict__ next, EfPaceRun* __restrict__ run, EfPaceOut* __restrict__ out,
                               const int64_t* __restrict__ pic_pts, const uint32_t* __restrict__ n_pics, const uint32_t* __restrict__ base_pics,
                               const uint8_t* __restrict__ modes, const uint8_t* __restrict__ lib_modes, const uint32_t* __restrict__ idle_n, int pic,
                               int max_pictures, int n_streams, int ntsc, const EfOverlayState* __restrict__ ovl, EfOverlayState* __restrict__ ovl_next)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams) return;
    const uint32_t top = ntsc ? 32 : 64, bottom = top + EF_H, vsync = ntsc ? 259 : 304;   // video.cpp:1135-1137
    EfPaceState q = st[s];
    const uint32_t F = q.fc;
    const uint32_t first = q.line <= bottom - 1 ? 0u : 1u;                 // does this call draw line active_bottom - 1 of field F?
    EfPaceRun r = { F + first, q.cur, pace_animate(q.ai, first), 0 };
    EfPaceOut o = { 0, 0, F + first, 0, -1, 0 };
    uint64_t n = 0;
    if (pic < 0) {
        n = idle_n[s];
        if (n) {
            const uint64_t end = first + n - 1;                            // stop right after line active_bottom - 1 of the last field
            q.ai = pace_animate(q.ai, end);
            q.fc = F + (uint32_t)end; q.line = bottom;
        }
    } else if ((uint32_t)pic < n_pics[s]) {
        const int64_t pts = pic_pts[(size_t)s * max_pictures + pic];
        int mode = modes ? modes[s] : 0;
        if (!mode && lib_modes && (uint32_t)pic + 1u == n_pics[s]) mode = lib_modes[s];   // load_poster's flush_picture(mode)
        if (pts == -1 && mode == 0) q.flags |= 1u;                         // flush_picture() pushes nothing (player.cpp:692-702)
        else {
            const uint32_t vp = (uint32_t)(pts / (ntsc ? 1500 : 1800));
            if (q.fc_origin == 0) { q.pts_origin = vp; q.fc_origin = F; }
            uint32_t d = vp - q.pts_origin + q.fc_origin;
            if (mode) d = F;                                               // due now (video.cpp:1039-1042)
            if (d < F && (int)(F - d) > 2) q.fc_origin = 0;                // late by more than two fields: re-latch at the next push
            uint32_t ff = 0, fl = 0;                                       // fields from F to the flip, flip line
            if (d <= F) {
                uint32_t l = q.line;
                if (q.cur >= 0 && l >= top && l < bottom) l = bottom;      // not on an active line of a presented frame
                if (l < vsync) fl = l; else ff = 1;
            } else ff = d - F;
            const int64_t last = (int64_t)ff - (fl >= bottom - 1 ? 0 : 1);
            n = last >= (int64_t)first ? (uint64_t)(last - (int64_t)first + 1) : 0;
            int ai = pace_animate(q.ai, ff);
            if (mode == 2) ai = -16; else if (mode == 3) ai = 16;          // load_poster: the scroll starts at the flip (video.cpp:1168-1171)
            q.ai = pace_animate(ai, 1);
            q.fc = F + ff; q.line = fl + 1;
            q.cur = (int)((base_pics[s] + (uint32_t)pic + 1u) & 1u);       // the store flush_picture() gave picture `pic` (player.cpp:692)
            o.flip_field = q.fc; o.flip_line = (int)fl;
        }
    }
    r.n = o.n_fields = n > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)n;
    o.flags = (int)q.flags;
    next[s] = q; run[s] = r; out[s] = o;
    if (ovl) {
        // latch field G: F when the call starts at line 0, else F + 1. The changes latch if the call draws line 0 of G, i.e. it
        // ends past (G, 0); otherwise they stay pending and latch at the same field with the next call's.
        EfOverlayState v = ovl[s];
        const uint32_t need = st[s].line == 0 ? 0u : 1u, adv = q.fc - F;
        v.latch_fc = F + need;
        if (v.pending && (adv > need || (adv == need && q.line > 0))) {
            if (v.pending & 1u) v.slot ^= 1u;
            if (v.pending & 2u) { v.blend = v.p_blend; v.blend_fc = v.latch_fc; }
            if (v.pending & 4u) v.progress = v.p_progress;
            v.pending = 0;
        }
        ovl_next[s] = v;
    }
}

// once the fields fit: one descriptor per emitted field, at the stream's offset `first` in the output; commits the state. ovl: also
// the overlay each field is drawn with (fields before the latch field show the state latched before this call), and its commit.
// kGated (ef_present_*_async, where only the device knows whether the fields fit): nothing at all once chain[0] says a call of the
// chain did not fit.
template <bool kGated>
__global__ void ef_pace_fill_kernel(EfPaceState* __restrict__ st, const EfPaceState* __restrict__ next, const EfPaceRun* __restrict__ run,
                                    const uint64_t* __restrict__ first, EfFieldDesc* __restrict__ desc,
                                    EfOverlayState* __restrict__ ovl, const EfOverlayState* __restrict__ ovl_next, EfFieldOverlay* __restrict__ fovl,
                                    const int* __restrict__ chain)
{
    if (kGated && *chain) return;
    const int s = blockIdx.x;
    const EfPaceRun r = run[s];
    const uint64_t base = first[s];
    for (uint32_t j = threadIdx.x; j < r.n; j += blockDim.x)
        desc[base + j] = { (uint32_t)s, r.cur < 0 ? -2 : r.cur, r.fc0 + j, pace_hscroll(pace_animate(r.ai, j)) };
    if (ovl) {
        const EfOverlayState a = ovl[s], b = ovl_next[s];
        const uint32_t k = b.latch_fc - r.fc0;                             // 0 or 1 fields drawn before the latch
        for (uint32_t j = threadIdx.x; j < r.n; j += blockDim.x) {
            const bool old = j < k;
            fovl[base + j] = { ef_overlay_blend(old ? a.blend : b.blend, old ? a.blend_fc : b.blend_fc, r.fc0 + j), old ? a.progress : b.progress,
                               old ? a.slot : b.slot, 0u };
        }
        __syncthreads();                                                   // every thread has read ovl[s]
        if (threadIdx.x == 0) ovl[s] = b;
    }
    if (threadIdx.x == 0) st[s] = next[s];
}

cudaError_t ef_launch_pace_fill(EfPaceState* st, const EfPaceState* next, const EfPaceRun* run, const uint64_t* first, EfFieldDesc* desc, EfOverlayState* ovl,
                                const EfOverlayState* ovl_next, EfFieldOverlay* fovl, int n_streams, const int* chain, cudaStream_t stream)
{
    if (chain) ef_pace_fill_kernel<true><<<n_streams, 128, 0, stream>>>(st, next, run, first, desc, ovl, ovl_next, fovl, chain);
    else ef_pace_fill_kernel<false><<<n_streams, 128, 0, stream>>>(st, next, run, first, desc, ovl, ovl_next, fovl, nullptr);
    return cudaGetLastError();
}

// ef_present_*_async: one CTA of 1,024 threads sizes a call on the device. The output offset of every stream's fields (an exclusive
// prefix of out[].n_fields, tile by tile with the carry of the tiles before) goes to first[] and, with the rest of the schedule's row,
// to the caller's info[]; *total gets the call's fields, or 0 when they exceed cap or an earlier call of the chain did not fit. The
// verdict is ANDed into the chain: chain[0] turns 1 at the first call that does not fit and stays so, chain[1] counts the calls that
// took effect. A call that does not take effect marks its info rows with flag bit 1 (the failing call keeps its counts and offsets,
// so it doubles as a sizing call; later calls carry none) and zeroes the mb_info slots `rec` of its record picture (NULL for an
// idle call): K1b then leaves every macroblock, and so the frame stores, as they are.
__global__ void __launch_bounds__(1024)
ef_pace_size_kernel(const EfPaceOut* __restrict__ out, int n_streams, uint64_t cap, uint64_t* __restrict__ first, EfPaceOut* __restrict__ info,
                    uint64_t* __restrict__ total, int* __restrict__ chain, uint32_t* __restrict__ rec)
{
    __shared__ EfBlockScan<uint64_t, 1024> scan;
    __shared__ int skip;
    if (threadIdx.x == 0) skip = *chain;
    scan.init();
    for (int base = 0; base < n_streams; base += 1024) {
        const int k = base + threadIdx.x;
        const uint64_t e = scan.exclusive(k < n_streams ? out[k].n_fields : 0);
        if (k < n_streams) first[k] = e;
    }
    const bool fits = !skip && scan.carry <= cap;
    for (int k = threadIdx.x; k < n_streams; k += 1024) {   // the same thread wrote first[k] above
        EfPaceOut o = out[k];
        o.first = skip ? 0 : first[k];
        if (skip) o.n_fields = 0;
        if (!fits) o.flags |= 2;
        info[k] = o;
    }
    if (!fits && rec) {
        uint4* r = (uint4*)rec;
        const size_t n = (size_t)n_streams * (EF_MBW_MAX * EF_MBH_MAX / 4);
        for (size_t i = threadIdx.x; i < n; i += 1024) r[i] = make_uint4(0, 0, 0, 0);
    }
    if (threadIdx.x == 0) {
        *total = fits ? scan.carry : 0;
        if (fits) chain[1] += 1; else chain[0] = 1;
    }
}

// ef_present_overlay: stream first + i takes cmd[i]; a bitmap goes to the slot that is not latched. One CTA per stream.
__global__ void ef_overlay_stage_kernel(EfOverlayState* __restrict__ ovl, uint8_t* __restrict__ slots, const EfOverlayCmd* __restrict__ cmd,
                                        const uint8_t* __restrict__ bitmaps, int first)
{
    const int i = blockIdx.x, s = first + i;
    const EfOverlayCmd c = cmd[i];
    if (c.set & 1u) {
        uint4* d = (uint4*)(slots + ((size_t)s * 2 + (ovl[s].slot ^ 1u)) * EF_OVERLAY_BYTES);
        const uint4* src = (const uint4*)(bitmaps + (size_t)i * EF_OVERLAY_BYTES);
        for (int k = (int)threadIdx.x; k < EF_OVERLAY_BYTES / 16; k += blockDim.x) d[k] = src[k];
    }
    __syncthreads();                                                       // every thread has read ovl[s].slot
    if (threadIdx.x == 0) {
        EfOverlayState v = ovl[s];
        if (c.set & 2u) v.p_blend = c.blend;
        if (c.set & 4u) v.p_progress = c.progress;
        v.pending |= c.set;
        ovl[s] = v;
    }
}

// ---- the clock of paced presentation (ef_present_clock): update_progress() (espflix.cpp:862-874) at the start of a present call ----
namespace {
// sprintf's "%d" (two = false) or "%02d" (two = true) of v at b + n; returns the new length
__device__ int clock_put_int(char* b, int n, int v, bool two)
{
    uint32_t u = v < 0 ? 0u - (uint32_t)v : (uint32_t)v;
    char d[10];
    int k = 0;
    do { d[k++] = (char)('0' + u % 10u); u /= 10u; } while (u);
    if (two && v >= 0 && k < 2) d[k++] = '0';                              // a sign counts towards the width
    if (v < 0) b[n++] = '-';
    while (k) b[n++] = d[--k];
    return n;
}
}  // namespace

// One CTA per stream. Every stream gets ovl_clk[s] = its committed overlay state; a stream whose clock is on also stages there the
// progress and, when the whole second changed, the bitmap that show_time() draws, rendered into its scratch bm[s]. ef_pace_kernel
// takes ovl_clk as the staged state; nothing committed changes here (ef_clock_commit_kernel does that once the call takes effect).
// The text: show_time()'s format (espflix.cpp:163-174) drawn from x = 0 into the erased 80 x 16 bitmap, glyph c - 0x18 being columns
// [rights[c - 0x19], rights[c - 0x18]) of the atlas; rows are contiguous, so column x >= 80 lands at x - 80 of the next row and
// what passes row 15 is dropped. Each byte folds the pixels that land on it in the order the reference writes them (glyph, then row,
// then column) through p32() with _color 240 (espflix.cpp:87-96).
__global__ void __launch_bounds__(128)
ef_clock_kernel(EfClockState* __restrict__ clk, const EfOverlayState* __restrict__ ovl, EfOverlayState* __restrict__ ovl_clk, uint8_t* __restrict__ bm,
                const int64_t* __restrict__ pic_pts, const uint32_t* __restrict__ n_pics, const int64_t* __restrict__ pts_last, int pic, int max_pictures,
                const uint8_t* __restrict__ font, const int16_t* __restrict__ rights)
{
    __shared__ char text[24];
    __shared__ int x0[25];                                                 // text column where each glyph starts; x0[len] = the width
    __shared__ int16_t col[EF_OVERLAY_BYTES];                              // text column X < 1280 -> atlas column, -1 past the text
    __shared__ uint8_t glyph[EF_OVERLAY_BYTES];                            // and the glyph it belongs to
    __shared__ int s_len, s_draw;
    const int s = blockIdx.x;
    if (threadIdx.x == 0) {
        EfClockState k = clk[s];
        EfOverlayState v = ovl[s];
        int draw = 0;
        if (k.flags & 1u) {
            const int64_t pts = pic >= 0 && (uint32_t)pic < n_pics[s] ? pic_pts[(size_t)s * max_pictures + pic] : pts_last[s];
            const int64_t main = ef_pts2pts(pts, k.speed, k.v_first, k.v_last, k.f_first, k.f_last, k.r_first, k.r_last);
            const int seconds = (int)(main / 90000);
            draw = seconds != k.last_seconds;
            v.p_progress = (int)(main * 240 / k.v_last);                   // VIDEO_COMPOSITE_PROGRESS_WIDTH
            v.pending |= draw ? 5u : 4u;
            if (draw) {
                const int m = seconds / 60, h = m / 60;
                const char icon = k.speed == 0 ? ((k.flags & 2u) ? 0x19 : 0x1A) : (k.speed == 1 ? 0x1B : 0x1C);   // PAUSE PLAY FFWD RWND
                int n = 0;
                text[n++] = icon;
                text[n++] = ' ';
                if (h) {
                    n = clock_put_int(text, n, h, false);
                    text[n++] = ':';
                } else {
                    text[n++] = ' '; text[n++] = ' ';
                }
                n = clock_put_int(text, n, m % 60, true);
                text[n++] = ':';
                n = clock_put_int(text, n, seconds % 60, true);
                int x = 0;
                for (int i = 0; i < n; i++) {
                    x0[i] = x;
                    const int g = text[i] - 0x18;
                    x += rights[g] - rights[g - 1];
                }
                x0[n] = x;
                s_len = n;
            }
            clk[s].seconds = seconds;
        }
        clk[s].draw = (uint32_t)draw;
        ovl_clk[s] = v;
        s_draw = draw;
    }
    __syncthreads();
    if (!s_draw) return;
    const int len = s_len;
    for (int X = (int)threadIdx.x; X < EF_OVERLAY_BYTES; X += blockDim.x) {
        int i = 0;
        while (i < len && x0[i + 1] <= X) i++;
        col[X] = i < len ? (int16_t)(rights[text[i] - 0x18 - 1] + X - x0[i]) : (int16_t)-1;
        glyph[X] = (uint8_t)i;
    }
    __syncthreads();
    uint8_t* out = bm + (size_t)s * EF_OVERLAY_BYTES;
    for (int L = (int)threadIdx.x; L < EF_OVERLAY_BYTES; L += blockDim.x) {
        const int y = L / 80, x = L % 80;
        int ks[16], n = 0;                                                 // pixel (row y - k, column x + 80 k) lands on byte L
        for (int k = 0; k <= y && x + 80 * k < EF_OVERLAY_BYTES && col[x + 80 * k] >= 0; k++) ks[n++] = k;
        uint32_t v = 0;
        for (int a = 0; a < n;) {                                          // glyph by glyph; inside a glyph, row by row
            int b = a;
            while (b + 1 < n && glyph[x + 80 * ks[b + 1]] == glyph[x + 80 * ks[a]]) b++;
            for (int j = b; j >= a; j--) {
                const int k = ks[j];
                const uint32_t p = font[(y - k) * EF_FONT_W + col[x + 80 * k]];
                if (p) v = (240u * p + (255u - p) * v) >> 8;
            }
            a = b + 1;
        }
        out[L] = (uint8_t)v;
    }
}

// Once the call takes effect (after ef_pace_fill_kernel, before the paced K2): the rendered bitmap goes to the slot that was not
// latched when the call began (ovl_clk[s].slot ^ 1, where ef_present_overlay stages), and last_seconds advances. kGated
// (ef_present_*_async): nothing once chain[0] says a call of the chain did not fit.
template <bool kGated>
__global__ void __launch_bounds__(96) ef_clock_commit_kernel(EfClockState* __restrict__ clk, const EfOverlayState* __restrict__ ovl_clk,
                                                             const uint8_t* __restrict__ bm, uint8_t* __restrict__ slots, const int* __restrict__ chain)
{
    if (kGated && *chain) return;
    const int s = blockIdx.x;
    const uint32_t flags = clk[s].flags, draw = clk[s].draw;
    if (!(flags & 1u)) return;
    if (draw) {
        uint4* d = (uint4*)(slots + ((size_t)s * 2 + (ovl_clk[s].slot ^ 1u)) * EF_OVERLAY_BYTES);
        const uint4* src = (const uint4*)(bm + (size_t)s * EF_OVERLAY_BYTES);
        for (int k = (int)threadIdx.x; k < EF_OVERLAY_BYTES / 16; k += blockDim.x) d[k] = src[k];
    }
    if (threadIdx.x == 0) clk[s].last_seconds = clk[s].seconds;
}

cudaError_t ef_launch_clock_commit(EfClockState* clk, const EfOverlayState* ovl_clk, const uint8_t* bm, uint8_t* slots, int n_streams, const int* chain,
                                   cudaStream_t stream)
{
    if (chain) ef_clock_commit_kernel<true><<<n_streams, 96, 0, stream>>>(clk, ovl_clk, bm, slots, chain);
    else ef_clock_commit_kernel<false><<<n_streams, 96, 0, stream>>>(clk, ovl_clk, bm, slots, nullptr);
    return cudaGetLastError();
}

// one launch of the paced K2 in the standard and output format of the instantiation; the overlay and gated variants as
// ef_launch_composite_paced picks them
template <bool kNtsc, bool kDac8>
static void launch_paced(dim3 grid, cudaStream_t stream, const EfDev* dev, const EfFieldDesc* desc, uint8_t* dst, const EfFieldOverlay* fovl,
                         const uint8_t* bitmaps, const uint64_t* total, uint64_t f0)
{
    K2Out<kDac8>* d = (K2Out<kDac8>*)dst;
    const EfPresent pr = { 0, 0, 0, bitmaps };
    if (total && fovl) ef_composite_kernel<kNtsc, true, true, true, kDac8><<<grid, kK2Threads, 0, stream>>>(dev, 0, 0, pr, desc, d, fovl, total, f0);
    else if (total) ef_composite_kernel<kNtsc, true, false, true, kDac8><<<grid, kK2Threads, 0, stream>>>(dev, 0, 0, pr, desc, d, nullptr, total, f0);
    else if (fovl) ef_composite_kernel<kNtsc, true, true, false, kDac8><<<grid, kK2Threads, 0, stream>>>(dev, 0, 0, pr, desc, d, fovl);
    else ef_composite_kernel<kNtsc, true, false, false, kDac8><<<grid, kK2Threads, 0, stream>>>(dev, 0, 0, EfPresent{}, desc, d);
}

// the paced K2: fields [0, n_fields) of desc into dst, at most 65,535 per launch (grid y). fovl != NULL: the overlay variant, with
// the per-field overlay fovl and the bitmap slots `bitmaps`. total != NULL: the gated variant, n_fields is the capacity of dst and
// only the slots below *total are drawn. dac8: EF_FIELD_DAC8 fields (line_count x line_width bytes), else uint16 samples.
cudaError_t ef_launch_composite_paced(const EfDev* dev, const EfGeometry& g, const EfFieldDesc* desc, uint64_t n_fields, uint8_t* dst, bool dac8,
                                      cudaStream_t stream, uint64_t* launches, const EfFieldOverlay* fovl, const uint8_t* bitmaps, const uint64_t* total)
{
    const size_t per = (size_t)g.line_count * g.line_width * (dac8 ? 1 : 2);   // bytes per field
    for (uint64_t f0 = 0; f0 < n_fields; f0 += 65535) {
        const dim3 grid((unsigned)(g.line_count + 15) / 16, (unsigned)(n_fields - f0 < 65535 ? n_fields - f0 : 65535));
        const EfFieldOverlay* fo = fovl ? fovl + f0 : nullptr;
        if (g.ntsc && dac8) launch_paced<true, true>(grid, stream, dev, desc + f0, dst + f0 * per, fo, bitmaps, total, f0);
        else if (g.ntsc) launch_paced<true, false>(grid, stream, dev, desc + f0, dst + f0 * per, fo, bitmaps, total, f0);
        else if (dac8) launch_paced<false, true>(grid, stream, dev, desc + f0, dst + f0 * per, fo, bitmaps, total, f0);
        else launch_paced<false, false>(grid, stream, dev, desc + f0, dst + f0 * per, fo, bitmaps, total, f0);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        ++*launches;
    }
    return cudaSuccess;
}

cudaError_t ef_launch_blit(const EfDev* dev, int stream_index, int fb, int line, int x, int width, int frame_counter, uint16_t* dst, cudaStream_t stream)
{
    const int groups = (width + 3) / 4;
    ef_blit_kernel<<<(groups + 63) / 64, 64, 0, stream>>>(dev, stream_index, fb, line, x, width, frame_counter, dst);
    return cudaGetLastError();
}
