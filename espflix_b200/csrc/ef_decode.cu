// espflix_b200/csrc/ef_decode.cu — K1, the macroblock decoder, as a pair of kernels.
//
// Replaces, for every stream at once, MpegDecoder::slice() and everything under it
// (player.cpp:733-1316): macroblock-header VLC, motion vectors, block() coefficient VLC +
// dequantisation, idct(), mocomp()/predict_zero(), copy_block/add_block with the [0,248] clamp.
//
// The reference interleaves bitstream parsing and pixel reconstruction macroblock by macroblock.
// The two halves have opposite shapes on a GPU, so they are separate kernels here:
//
//   K1a ef_parse_kernel   bitstream -> macroblock records. VLC parsing is serial inside a slice and
//       needs NO pixel data, so every slice of EVERY picture of the submit is independent: one launch
//       covers pictures x streams x slices (589,824 slices for the BASELINE batch), one slice per
//       LANE, lanes pulling new slices from a global cursor as they finish. Per macroblock a lane
//       emits (i) a 48-byte record (type, coded-block pattern, motion vector, intra DCs, skip run,
//       list position) in the slot of its macroblock ADDRESS and (ii) its coefficients as 32-bit
//       entries (block, raster position, dequantised + AAN-prescaled value), appended to the slice's
//       list in HBM. A VLC symbol is one CLZ + one shared-memory table load; dequantisation
//       (quirk Q2 included) happens on the spot. The list of a slice starts at entry 3 x (byte offset
//       of the slice in the ES blob): every coefficient costs at least 3 bits of bitstream, so lists
//       can never run into each other and no allocation or prefix sum is needed.
//       A global-memory instruction whose lanes point into 32 different slices costs the load/store
//       unit a cycle per lane, and the round-1 parser issued two of them per symbol step; so the
//       bitstream comes in as 16-byte cp.async.cg chunks (one per lane per 128 bits) and list entries
//       are staged in a per-lane ring in shared memory and written out by the whole warp, one list run
//       per store instruction, independently of macroblock boundaries (DESIGN.md 4).
//   K1b ef_recon_kernel   records -> pixels, one launch per picture index (P pictures read the
//       previous picture of their stream). One HALF-WARP per macroblock record (a warp = two
//       consecutive slots), all 1,081,344 of a BASELINE picture batch independent: scatter the list
//       into a dense 6x64 scratch, the reference's integer AAN IDCT in place (3 column passes, then 3
//       row passes of 16 lanes), half-pel motion compensation from reference tiles staged by TMA bulk
//       copies, the clamped add, 8-byte stores. Records are prefetched one iteration ahead; work
//       comes from a global cursor.
//
//   * frame stores are MACROBLOCK-TILED in HBM (ef_common.cuh): a macroblock is 384 contiguous
//     bytes, so a half-warp stores one full 128-byte line per row pass, no partial sectors;
//     motion-compensated reads touch <= 4 tiles.
// Bit-exactness notes (SURVEY.md §8a-Q): Q1 clamp [0,248]; Q2 oddification maps 0 -> +1; Q3 chroma
// vector = floor(luma position / 2); Q4 matrices indexed in raster order (done at index time);
// Q5 single-coefficient blocks bypass the IDCT with floor; Q6 first macroblock of a slice lands in
// column 0; Q7 intra DC-only blocks are replicated unclamped.
#include "ef_common.cuh"
#include "ef_coef_step.cuh"

namespace {

constexpr int kParseThreads = EF_K1A_THREADS;   // per CTA
constexpr int kParseCtasPerSm = EF_K1A_CTAS;
constexpr int kHdrBatch = EF_K1A_HDR_BATCH;        // waiting lanes that end a symbol loop early
constexpr int kReconWarps = EF_K1B_WARPS;       // per CTA
constexpr int kReconCtasPerSm = EF_K1B_CTAS;

// macroblock info word (EfDev::mb_info): bit0 valid, 1 intra, 2-7 coded blocks, 8-13 n==1 mask,
// 14-19 abort mask (bit b = block b), 20-24 mb_width of the stream, 25 destination frame store
constexpr int kDenseStride = 72;                // words per block in the dense scratch: 64 + 8 pad -> the 4 luma blocks hit distinct banks
constexpr int kDenseWords = 6 * kDenseStride;   // int32 [6][72] prescaled coefficients, raster order, also the IDCT transpose buffer; 432 = 16 mod 32: the two halves of a warp hit disjoint banks
constexpr int kDenseBytes = kDenseWords * 4;
constexpr int kStageBytes = 4 * EF_TILE;        // motion-compensation staging: up to 2 x 2 reference tiles per macroblock
constexpr int kWarpBytes = 2 * (kDenseBytes + kStageBytes) + 16;   // two macroblocks per warp + their mbarriers
constexpr int kReconQzBytes = EF_K1B_DEQUANT ? 128 * 4 : 0;             // K1b dequantises (v3): the default matrices' table words, once per CTA

struct SharedTables {                           // same layout as the head of EfTables
    uint16_t dct[26 * 32];
    uint16_t mba[8 * 32];
    uint16_t mv[7 * 32];
    uint16_t cbp[512];
    uint8_t ptype[64];
    uint8_t qdef[128];
    uint16_t zp[64];                            // scan position -> raster index | AAN prescale << 8
    uint32_t qz[128];                           // default matrices: quantiser | prescale << 8 | raster index << 18
};
constexpr int kTableBytes = (sizeof(SharedTables) + 15) & ~15;
constexpr int kLutBits = EF_K1A_LUT_BITS;       // the two-symbol table (EfTables::lut2) is indexed by the next kLutBits bits
constexpr int kLutSize = 1 << kLutBits;         // entries per context
constexpr int kLutBytes = kLutBits > 0 ? 2 * kLutSize * (int)sizeof(uint2) : 0;

// ---------------------------------------------------------------------------------------------
// bit reader (FILL_BITS/peek_bits/get_bits, player.cpp:348-352, 495-514): MSB-first. `hi` holds the
// current 32-bit word, `lo` the next one, pos = bits of `hi` already consumed; peek() is a single funnel
// shift. The words after `lo` come through a per-lane ring of 8 words in shared memory filled by 4-byte
// cp.async copies issued 7 words ahead: a register scoreboard is warp-wide, so a plain look-ahead load
// into a register stalls ALL lanes at the next refill of ANY lane (that was 1/3 of K1a's stall samples);
// the asynchronous copies involve no register. Reads run at most 12 bytes past the slice plus the 28
// prefetched ones (into the next start code); the ES blob carries 256 bytes of zero padding at its end.
// ---------------------------------------------------------------------------------------------
#if EF_K1A_ES16
constexpr int kRingStride = kParseThreads * 16;         // bytes between the 16-byte chunk slots of one lane (4 slots)
constexpr int kRingBytes = 4 * kRingStride;
#else
constexpr int kRingStride = kParseThreads * 4;          // bytes between ring slots of one lane: slot-major, conflict-free
constexpr int kRingBytes = 8 * kRingStride;
#endif
// List entries not yet written to HBM: a ring of kStage words per lane in shared memory (entry e of the slice's list in
// word e % kStage). They go out coalesced, one list run per store instruction, before any lane's ring could overflow:
// the symbol loop flushes when a lane holds more than kStageHigh entries, which leaves room for one pass of steps.
constexpr int kStage = 32;
constexpr int kStageHigh = kStage - (EF_K1A_V3 ? EF_K1A_UNROLL : 2);   // a pass adds at most one entry per step (v3) or two (one two-symbol step)
static_assert(kStageHigh > 0, "a pass of the symbol loop must fit in the staging ring");
// bytes per staging row: with the 16-byte bitstream slots a multiple of 16 (36 words for 32 entries), so that a lane's row
// address is a multiple of its ring address (one IMAD where the compiler otherwise re-derives it from the thread index at
// every store); else an odd number of words
constexpr int kStageRow = EF_K1A_ES16 ? ((kStage * 4 + 16 + 15) & ~15) : (kStage + 1) * 4;
constexpr int kStageBytesA = kParseThreads * kStageRow;

struct BitReader {
    const uint32_t* words;   // the whole ES blob as aligned 32-bit words (cudaMalloc alignment)
    uint32_t rp;             // index of the next word to take from the ring
    uint32_t sring;          // shared-window address of this lane's ring slot 0
    uint32_t hi, lo;
#if EF_K1A_RING_AHEAD || EF_K1A_ES16
    uint32_t nx;             // raw word after `lo` (its ring load is issued one refill before it is needed: off the dependent chain)
#endif
    int pos;

#if EF_K1A_ES16
    // 16-byte chunks: chunk c of the blob lives in slot c & 3. hi, lo, nx = words rp - 2, rp - 1, rp; the next word taken
    // from the ring is rp + 1, in chunk (rp + 1) >> 2, and the chunks in flight always reach 3 past that one.
    __device__ __forceinline__ void copy_chunk(uint32_t cidx)
    {
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sring + (cidx & 3u) * kRingStride), "l"((const uint4*)words + cidx) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    __device__ __forceinline__ void init(const uint8_t* blob, uint64_t byte_off)
    {
        words = (const uint32_t*)blob;
        const uint32_t w0 = (uint32_t)(byte_off >> 2);
        pos = (int)(byte_off & 3) * 8;
        asm volatile("cp.async.wait_all;" ::: "memory");      // copies of the previous slice must not land in the new ring
        rp = w0 + 2;
        const uint32_t c0 = (rp + 1) >> 2;
#pragma unroll
        for (int k = 0; k < 4; k++) copy_chunk(c0 + k);
        hi = __byte_perm(__ldg(words + w0), 0, 0x0123); lo = __byte_perm(__ldg(words + w0 + 1), 0, 0x0123);
        nx = __ldg(words + w0 + 2);
    }
    __device__ __forceinline__ uint32_t peek() const { return __funnelshift_l(lo, hi, pos); }
    __device__ __forceinline__ void skip(int n)
    {
        pos += n;
        if (pos >= 32) {
            pos -= 32; hi = lo;
            lo = __byte_perm(nx, 0, 0x0123);
            rp++;
            asm volatile("cp.async.wait_group 3;" ::: "memory");          // the chunk of word rp has landed (4 chunks in flight, one group each)
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(nx) : "r"(sring + ((rp >> 2) & 3u) * kRingStride + (rp & 3u) * 4) : "memory");
            if ((rp & 3u) == 3u) copy_chunk((rp >> 2) + 4);               // its last word: the slot takes the chunk 4 further on
        }
    }
#else
    __device__ __forceinline__ void copy_in(uint32_t widx)
    {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sring + (widx & 7u) * kRingStride), "l"(words + widx) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    __device__ __forceinline__ void init(const uint8_t* blob, uint64_t byte_off)
    {
        words = (const uint32_t*)blob;
        const uint32_t w0 = (uint32_t)(byte_off >> 2);
        pos = (int)(byte_off & 3) * 8;
        asm volatile("cp.async.wait_all;" ::: "memory");      // copies of the previous slice must not land in the new ring
        rp = w0 + 2;
#pragma unroll
        for (int k = 0; k < 7; k++) copy_in(rp + k);
        hi = __byte_perm(__ldg(words + w0), 0, 0x0123); lo = __byte_perm(__ldg(words + w0 + 1), 0, 0x0123);
#if EF_K1A_RING_AHEAD
        nx = __ldg(words + w0 + 2);
#endif
    }
    __device__ __forceinline__ uint32_t peek() const { return __funnelshift_l(lo, hi, pos); }
    __device__ __forceinline__ void skip(int n)
    {
        pos += n;
        if (pos >= 32) {
            pos -= 32; hi = lo;
#if EF_K1A_RING_AHEAD
            lo = __byte_perm(nx, 0, 0x0123);
            asm volatile("cp.async.wait_group 5;" ::: "memory");          // word rp + 1 has landed (7 copies in flight, one group each)
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(nx) : "r"(sring + ((rp + 1) & 7u) * kRingStride) : "memory");
            copy_in(rp + 7);                                              // slot (rp - 1) & 7: read one refill ago
#else
            asm volatile("cp.async.wait_group 6;" ::: "memory");          // word rp has landed (7 copies in flight, one group each)
            uint32_t raw;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(raw) : "r"(sring + (rp & 7u) * kRingStride) : "memory");
            lo = __byte_perm(raw, 0, 0x0123);
            copy_in(rp + 7);                                              // into the slot that was read one refill ago
#endif
#if EF_K1A_PF_L2
            if ((rp & 7u) == 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(words + rp + 32));   // 128 bytes ahead of this slice's read position
#endif
            rp++;
        }
    }
#endif
    __device__ __forceinline__ uint32_t get(int n)     // 1 <= n <= 32
    {
        uint32_t v = peek() >> (32 - n);
        skip(n);
        return v;
    }
};

// per-lane slice parser state
struct SliceState {
    BitReader br;
    uint32_t* list;          // the slice's coefficient list in HBM (entry 3 x byte offset of the slice)
    uint32_t slot_base;      // record slot of macroblock (0,0) of this slice's picture | destination frame store << 31
    uint32_t seqi;           // index of the slice's sequence state in the stream's EfSeq table (K1a v3: handed to K1b for streams with their own matrices)
    const uint32_t* qzp;     // generic pointer to the table words in use: T.qz in shared memory (default matrices) or the stream's own in HBM
    const uint32_t* qz;      // scan-order quantiser | prescale | raster index tables [intra 64 | non-intra 64] of a stream with its OWN matrices (global memory); nullptr = the defaults, served from shared memory
    int mbw;
    int mb_x, mb_y;          // last macroblock handled
    int first;               // next macroblock is the first of the slice (Q6)
    int ptype, full_pel, r_size;
    int qscale;
    int dc_y, dc_cr, dc_cb;  // reference names: cr = block 4, cb = block 5 (player.cpp:728)
    int mv_h, mv_v;
};

// Headers are parsed from a 32-bit WINDOW (w = br.peek(), `used` bits consumed so far) and the bit reader
// is advanced once per window: every br.skip() site carries the ring-refill code, and the header phase runs
// with most lanes diverged, so fewer sites is what counts. Window budgets are noted at each use.
__device__ __forceinline__ int motion_component(uint32_t w, int& used, const uint16_t* mvtab, int m, int r_size, bool& bad)
{
    // motion_vector(), player.cpp:891; at most 11 + 6 bits
    const uint32_t bits = w << used;
    int lz = __clz(bits);
    if (lz > 6) { bad = true; return m; }
    uint32_t e = mvtab[lz * 32 + ((bits << (lz + 1)) >> 27)];
    int len = e & 15;
    if (!len) { bad = true; return m; }
    int code = (int)(e >> 4) - 16;
    used += len;
    int d = code;
    if (code != 0 && r_size != 0) {
        d = ((abs(code) - 1) << r_size) + (int)((w << used) >> (32 - r_size)) + 1;
        used += r_size;
        if (code < 0) d = -d;
    }
    int scale = 1 << r_size;
    m += d;
    if (m > (scale << 4) - 1) m -= scale << 5;
    else if (m < -(scale << 4)) m += scale << 5;
    return m;
}

// One 8-point pass of the reference IDCT (player.cpp:938-995), on registers.
template <bool kFinal>
__device__ __forceinline__ void idct8(int (&v)[8])
{
    int b1 = v[4];
    int b3 = v[2] + v[6];
    int b4 = v[5] - v[3];
    int t1 = v[1] + v[7];
    int t2 = v[3] + v[5];
    int b6 = v[1] - v[7];
    int b7 = t1 + t2;
    int m0 = kFinal ? v[0] + 128 : v[0];            // every output carries m0 exactly once: the final (x + 128) >> 8 needs one add
    int x4 = ((b6 * 473 - b4 * 196 + 128) >> 8) - b7;
    int x0 = x4 - (((t1 - t2) * 362 + 128) >> 8);
    int x1 = m0 - b1;
    int x2 = (((v[2] - v[6]) * 362 + 128) >> 8) - b3;
    int x3 = m0 + b1;
    int y3 = x1 + x2, y4 = x3 + b3, y5 = x1 - x2, y6 = x3 - b3;
    int y7 = -x0 - ((b4 * 473 + b6 * 196 + 128) >> 8);
    v[0] = b7 + y4; v[1] = x4 + y3; v[2] = y5 - x0; v[3] = y6 - y7;
    v[4] = y6 + y7; v[5] = x0 + y5; v[6] = y3 - x4; v[7] = y4 - b7;
    // kFinal: the outputs are left scaled by 256 (the reference's final >> 8 is folded into pin4)
}

__device__ __forceinline__ uint32_t pin4(uint32_t pred, int r0, int r1, int r2, int r3)
{
    // PIN(b + (s >> 8)) for four pixels (add_block, player.cpp:1189; _pin clamps to [0,248], Q1), with the residuals r
    // still scaled by 256. Two pixels per DPX instruction: PRMT cuts (r >> 8) out of bytes 1-2 of two residuals as a pair
    // of int16 (|r >> 8| < 30,500 for any coefficients within +-2048: the 64 basis amplitudes sum to 14.85), another PRMT
    // spreads two prediction bytes to halfwords, VIADDMNMX.S16x2.RELU computes max(min(pred + res, 248), 0) on both.
#if EF_K1B_PIN16
    const uint32_t s01 = __viaddmin_s16x2_relu(__byte_perm(pred, 0, 0x4140), __byte_perm((uint32_t)r0, (uint32_t)r1, 0x6521), 0x00F800F8u);
    const uint32_t s23 = __viaddmin_s16x2_relu(__byte_perm(pred, 0, 0x4342), __byte_perm((uint32_t)r2, (uint32_t)r3, 0x6521), 0x00F800F8u);
    return __byte_perm(s01, s23, 0x6420);
#else
    // one pixel per instruction: t = max(min(pred * 256 + r, 248 * 256 + 255), 0), floor(t / 256) = its byte 1
    const int p0 = __viaddmin_s32_relu((int)__byte_perm(pred, 0, 0x4404), r0, 0xF8FF);
    const int p1 = __viaddmin_s32_relu((int)__byte_perm(pred, 0, 0x4414), r1, 0xF8FF);
    const int p2 = __viaddmin_s32_relu((int)__byte_perm(pred, 0, 0x4424), r2, 0xF8FF);
    const int p3 = __viaddmin_s32_relu((int)__byte_perm(pred, 0, 0x4434), r3, 0xF8FF);
    return __byte_perm(__byte_perm(p0, p1, 0x0051), __byte_perm(p2, p3, 0x0051), 0x5410);
#endif
}

// (a+b+1)>>1 on four packed bytes (mocomp cases 1 and 2, player.cpp:777-805)
__device__ __forceinline__ uint32_t avg2x4(uint32_t a, uint32_t b) { return (a | b) - (((a ^ b) >> 1) & 0x7F7F7F7Fu); }

// (a+b+c+d+2)>>2 on four packed bytes (mocomp case 3, player.cpp:806)
__device__ __forceinline__ uint32_t avg4x4(uint32_t a, uint32_t b, uint32_t c, uint32_t d)
{
    const uint32_t m = 0x00FF00FFu;
    uint32_t e = (a & m) + (b & m) + (c & m) + (d & m) + 0x00020002u;
    uint32_t o = ((a >> 8) & m) + ((b >> 8) & m) + ((c >> 8) & m) + ((d >> 8) & m) + 0x00020002u;
    return ((e >> 2) & m) | (((o >> 2) & m) << 8);
}

// ---- motion-compensation source: TMA-engine bulk copies of whole reference tiles into shared memory ----
// A macroblock's prediction window (17 x 17 luma + 2 x 9 x 9 chroma at a half-pel vector) lies in at
// most 2 x 2 tiles of the reference frame, and a tile (384 B: Y, block-4, block-5 chroma) is contiguous
// in HBM, so one elected lane issues 1, 2 or 4 cp.async.bulk copies per macroblock, completion is
// signalled on a per-warp mbarrier, and all lanes then read their pixels from shared memory. The copies
// are issued before the IDCT work of the macroblock and waited for after it.
struct PredWords { uint32_t a0, a1, a2, b0, b1, b2; };

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t sbar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sbar), "r"(bytes) : "memory");
}
// one or two horizontally adjacent reference tiles (384 / 768 contiguous bytes) HBM -> shared memory
// through the TMA engine; sdst / sbar are shared-window addresses
__device__ __forceinline__ void bulk_tiles(uint32_t sdst, const uint8_t* gsrc, uint32_t bytes, uint32_t sbar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(sdst), "l"(gsrc), "r"(bytes), "r"(sbar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t sbar, uint32_t parity)
{
    uint32_t ok;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(ok) : "r"(sbar), "r"(parity) : "memory");
    } while (!ok);
}

// Words of this lane's 8-pixel segment from the staged tiles. (x, y) = first pixel in plane
// coordinates, (tx0, ty0) = tile of the window's top-left corner. kLuma: 16-pixel tile rows, else
// 8-pixel chroma tile rows of plane 0/1.
template <bool kLuma>
__device__ __forceinline__ void pred_words_staged(const uint8_t* st, int plane, int x, int y, int tx0, int ty0, bool yh, PredWords& w)
{
    constexpr int TS = kLuma ? 16 : 8, SH = kLuma ? 4 : 3;
    const int xa = x & ~3, xi = xa & (TS - 1), yi = y & (TS - 1);
    // word 0, then +4 bytes each, hopping to the next staged tile column (+384) at the end of a tile row;
    // a hop out of the 2 x 2 window can only happen for the third word when it is not used: keep it inside
    const int o0 = ((y >> SH) - ty0) * (2 * EF_TILE) + ((xa >> SH) - tx0) * EF_TILE + (kLuma ? 0 : 256 + plane * 64) + yi * TS + xi;
    const int o1 = o0 + (xi + 4 < TS ? 4 : EF_TILE + 4 - TS);
    const int xj = (xi + 4) & (TS - 1);
    int o2 = o1 + (xj + 4 < TS ? 4 : EF_TILE + 4 - TS);
    if (((xa + 8) >> SH) - tx0 > 1) o2 = o1;
    w.a0 = *(const uint32_t*)(st + o0); w.a1 = *(const uint32_t*)(st + o1); w.a2 = *(const uint32_t*)(st + o2);
    if (yh) {
        const int d = yi == TS - 1 ? 2 * EF_TILE - (TS - 1) * TS : TS;    // next row: same tile, or the tile below
        w.b0 = *(const uint32_t*)(st + o0 + d); w.b1 = *(const uint32_t*)(st + o1 + d); w.b2 = *(const uint32_t*)(st + o2 + d);
    }
}

// Same words straight from HBM with coordinates clamped into the frame: only for vectors that
// point outside the picture, where the reference reads whatever lies there (plain byte semantics of mocomp()).
template <bool kLuma>
__device__ __forceinline__ void pred_words_clamped(const uint8_t* ref, int plane, int x, int y, bool yh, PredWords& w)
{
    constexpr int W = kLuma ? EF_W : EF_W / 2, H = kLuma ? EF_H : EF_H / 2, TS = kLuma ? 16 : 8, SH = kLuma ? 4 : 3;
    const int plane_off = kLuma ? 0 : 256 + plane * 64;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        if (r == 1 && !yh) break;
        const int yy = max(0, min(H - 1, y + r));
        const int xa = max(0, min(W - 4, x & ~3)), xb = min(W - 4, xa + 4), xc = min(W - 4, xa + 8);
        const int rowbase = (yy >> SH) * EF_MBW_MAX * EF_TILE + plane_off + (yy & (TS - 1)) * TS;
        const uint32_t v0 = *(const uint32_t*)(ref + rowbase + (xa >> SH) * EF_TILE + (xa & (TS - 1)));
        const uint32_t v1 = *(const uint32_t*)(ref + rowbase + (xb >> SH) * EF_TILE + (xb & (TS - 1)));
        const uint32_t v2 = *(const uint32_t*)(ref + rowbase + (xc >> SH) * EF_TILE + (xc & (TS - 1)));
        if (r == 0) { w.a0 = v0; w.a1 = v1; w.a2 = v2; } else { w.b0 = v0; w.b1 = v1; w.b2 = v2; }
    }
}

// eight predicted pixels from the loaded words (the four cases of mocomp(), player.cpp:767-820)
__device__ __forceinline__ void pred_finish(const PredWords& w, int x, int xh, int yh, uint32_t& o0, uint32_t& o1)
{
    const int sh = (x & 3) * 8;
    const uint32_t p0 = __funnelshift_r(w.a0, w.a1, sh), p1 = __funnelshift_r(w.a1, w.a2, sh);
    if (xh) {
        const uint32_t q0 = __funnelshift_rc(w.a0, w.a1, sh + 8), q1 = __funnelshift_rc(w.a1, w.a2, sh + 8);
        if (yh) {
            o0 = avg4x4(p0, q0, __funnelshift_r(w.b0, w.b1, sh), __funnelshift_rc(w.b0, w.b1, sh + 8));
            o1 = avg4x4(p1, q1, __funnelshift_r(w.b1, w.b2, sh), __funnelshift_rc(w.b1, w.b2, sh + 8));
        } else {
            o0 = avg2x4(p0, q0);
            o1 = avg2x4(p1, q1);
        }
    } else if (yh) {
        o0 = avg2x4(p0, __funnelshift_r(w.b0, w.b1, sh));
        o1 = avg2x4(p1, __funnelshift_r(w.b1, w.b2, sh));
    } else {
        o0 = p0; o1 = p1;
    }
}

// ---------------------------------------------------------------------------------------------
// macroblock header of this lane's slice (player.cpp:1266-1307). Returns false when the slice
// ended. On success: `cbp` = blocks to parse (bit b = block b), `intra`, the skip run before this
// macroblock and its motion vector in half-pel units ((int16 h) | (int16 v) << 16).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool parse_header(SliceState& s, const SharedTables& T, int& cbp_out, int& intra_out, uint32_t& skip_out, uint32_t& mv_out)
{
    BitReader& br = s.br;
    uint32_t bits = br.peek();
    if ((bits >> 9) == 0) return false;             // slice_done(): next 23 bits are zero (player.cpp:1238)

    // window A: address increment (<= 11 bits) + macroblock_type (<= 6) + quantiser_scale (5)
    int increment = 0, used;                        // macroblock_address_increment (player.cpp:1267-1275)
    uint32_t w;
    for (;;) {
        w = br.peek();
        int lz = __clz(w);
        if (lz > 7) return false;
        uint32_t e = T.mba[lz * 32 + ((w << (lz + 1)) >> 27)];
        int len = e & 15, val = (int)(e >> 4);
        if (!len) return false;
        if (val == 35 || (val == 34 && !increment)) {     // escape, or stuffing before the first escape: consume and look again
            br.skip(len);
            if (val == 35) increment += 33;
            continue;
        }
        increment += val;                           // stuffing after an escape ends the address: + 34 (player.cpp:1269-1275)
        used = len;
        break;
    }
    int skip_before = 0;
    if (s.first) { s.first = 0; increment = 1; }    // inc_mb ignores its argument for the first macroblock (Q6)
    else if (increment > 1) { s.dc_y = s.dc_cr = s.dc_cb = 128; s.mv_h = s.mv_v = 0; skip_before = increment - 1; }
    s.mb_x += increment;
    while (s.mb_x >= s.mbw) { s.mb_x -= s.mbw; s.mb_y++; }     // inc_mb(), player.cpp:823
    if (s.mb_y >= EF_MBH_MAX) return false;         // past the frame's 12 strips: the reference would write out of bounds

    int mb_type;                                    // macroblock_type (player.cpp:1292)
    bits = w << used;
    if (s.ptype == 1) {
        if (bits >> 31) { mb_type = 0x01; used += 1; }
        else if (bits >> 30) { mb_type = 0x11; used += 2; }
        else return false;
    } else {
        uint32_t e = T.ptype[bits >> 26];
        if (!(e & 7)) return false;
        mb_type = (int)(e >> 3);
        used += e & 7;
    }
    const int intra = mb_type & 1;
    if (mb_type & 0x10) { s.qscale = (int)((w << used) >> 27); used += 5; }
    br.skip(used);                                  // <= 22 bits

    int mvh = 0, mvv = 0;
    used = 0;
    if (intra) { s.mv_h = s.mv_v = 0; }
    else {
        s.dc_y = s.dc_cr = s.dc_cb = 128;
        if (mb_type & 0x08) {
            bool bad = false;
            w = br.peek();                          // window B: horizontal component (<= 17 bits)
            s.mv_h = motion_component(w, used, T.mv, s.mv_h, s.r_size, bad);
            br.skip(used);
            used = 0;
            w = br.peek();                          // window C: vertical component (<= 17) + coded_block_pattern (<= 9)
            s.mv_v = motion_component(w, used, T.mv, s.mv_v, s.r_size, bad);
            if (bad) return false;
        } else s.mv_h = s.mv_v = 0;
        mvh = s.mv_h << s.full_pel;                 // predict(), player.cpp:878
        mvv = s.mv_v << s.full_pel;
    }
    int cbp = intra ? 63 : 0;
    if (mb_type & 0x02) {
        if (!used) w = br.peek();
        uint32_t e = T.cbp[(w << used) >> 23];
        if (!(e & 15)) return false;
        cbp = (int)(e >> 4);
        used += e & 15;
    }
    if (used) br.skip(used);
    cbp_out = (int)(__brev((unsigned)cbp) >> 26);   // bit b = block b (the VLC value has block 0 in bit 5)
    intra_out = intra;
    skip_out = (uint32_t)skip_before;
    mv_out = ((uint32_t)mvh & 0xFFFFu) | ((uint32_t)mvv << 16);
    return true;
}

// dct_dc_size + differential of an intra block (player.cpp:1010-1068); returns the DC (pixel scale)
__device__ __forceinline__ int parse_dc(SliceState& s, int blk)
{
    BitReader& br = s.br;
    const uint32_t bits = br.peek();                // one window: size code (<= 10 bits) + differential (<= 11)
    int dc_size, used, dc;
    if (blk < 4) {
        dc = s.dc_y;
        if (!(bits >> 31)) { dc_size = 1 + (int)((bits >> 30) & 1); used = 2; }
        else if (!((bits >> 30) & 1)) { dc_size = ((bits >> 29) & 1) ? 3 : 0; used = 3; }
        else { int ones = min(9, __clz(~bits)); dc_size = ones + 2; used = dc_size - 1; }
    } else {
        dc = blk == 4 ? s.dc_cr : s.dc_cb;
        if (!(bits >> 31)) { dc_size = (int)((bits >> 30) & 1); used = 2; }
        else { int ones = min(10, __clz(~bits)); dc_size = ones + 1; used = min(dc_size, 10); }
    }
    if (dc_size) {
        int delta = (int)((bits << used) >> (32 - dc_size));
        if (delta & (1 << (dc_size - 1))) dc += delta;
        else dc += (int)((0xFFFFFFFFu << dc_size) | (uint32_t)(delta + 1));
        if (blk < 4) s.dc_y = dc; else if (blk == 4) s.dc_cr = dc; else s.dc_cb = dc;
    }
    br.skip(used + dc_size);
    return dc;
}

}  // namespace

// =================================================================================================
// K1a: bitstream -> macroblock records, every slice of pictures [pic0, pic0 + n_pics) in one launch
//
// Lane states: no slice (idle / exhausted), WAITING for the header of its next macroblock, BUSY in the
// coefficient state machine. Header phases (flush finished records, refill idle lanes, parse headers)
// alternate with symbol loops (per busy lane and step: one run/level symbol with a following end of block folded in -
// or, with EF_K1A_V3 = 0, up to two coefficients and an end of block from one look-up in the two-symbol table); a
// symbol loop ends when no lane is busy or when kHdrBatch lanes are waiting.
// =================================================================================================
__global__ void __launch_bounds__(kParseThreads, kParseCtasPerSm)
ef_parse_kernel(const __grid_constant__ EfDev D, int pic0, int n_pics)   // the context by value: every D.field is a constant-bank operand (no register, no load)
{
    extern __shared__ __align__(16) uint8_t smem[];           // tables | two-symbol table | bitstream rings | staged list entries
    SharedTables& T = *(SharedTables*)smem;
    const uint2* lut = (const uint2*)(smem + kTableBytes);
    {   // stage the tables (the first sizeof(SharedTables) bytes of EfTables have the same layout)
        const uint32_t* src = (const uint32_t*)D.tables;
        uint32_t* dst = (uint32_t*)smem;
        for (int i = threadIdx.x; i < (int)(sizeof(SharedTables) / 4); i += blockDim.x) dst[i] = src[i];
        const uint4* lsrc = (const uint4*)D.tables->lut2;
        uint4* ldst = (uint4*)(smem + kTableBytes);
        for (int i = threadIdx.x; i < kLutBytes / 16; i += blockDim.x) ldst[i] = lsrc[i];
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;

    // the work lists of consecutive picture indices are contiguous (ef_prefix_kernel)
    uint32_t total = 0;
    for (int p = pic0; p < pic0 + n_pics; p++) total += D.pic_total[p];
    const EfWork* work = D.work + D.pic_base[pic0];
    const uint32_t n_slots = (uint32_t)D.n_streams * (EF_MBW_MAX * EF_MBH_MAX);

    SliceState s;
    s.first = 0; s.list = D.coef; s.slot_base = 0; s.qz = nullptr; s.mbw = 0; s.mb_x = s.mb_y = 0;
    s.br.sring = smem_u32(smem + kTableBytes + kLutBytes) + threadIdx.x * (EF_K1A_ES16 ? 16 : 4);
    // staged list entries: one ring row per lane
    const uint32_t sstage_warp = smem_u32(smem + kTableBytes + kLutBytes + kRingBytes) + (threadIdx.x & ~31u) * kStageRow;
#if EF_K1A_ES16
    const uint32_t sstage_bias = smem_u32(smem + kTableBytes + kLutBytes + kRingBytes) - (kStageRow / 16) * smem_u32(smem + kTableBytes + kLutBytes);
#define EF_SSTAGE (s.br.sring * (kStageRow / 16) + sstage_bias)      /* = stage base + thread * kStageRow (sring = ring base + thread * 16) */
#else
    const uint32_t sstage = sstage_warp + lane * kStageRow;
#define EF_SSTAGE sstage
#endif
    bool active = false, exhausted = false, busy = false;
    // the slice's list: `tot` entries so far, the first `done` of them in HBM, the rest in the lane's ring.
    // The macroblock in flight: info word under construction (bit 0 set = a record is owed), its first list entry,
    // skip run, motion vector, record slot
    uint32_t tot = 0, done = 0;
    uint32_t info_acc = 0, mb0 = 0, skipw = 0, mvw = 0, slot = 0;
    uint32_t blk24 = 0, blkbit = 0;                           // current block: number << 24 (v3: token head = number << 27 | quantiser_scale << 16), 0x100 << number
    int cbp_rem = 0, n = 0, intra = 0, ctx = 0;               // n = scan position of the block in flight; ctx = 1: the next symbol is the first coefficient of a non-intra block
    // next coded block of the macroblock in flight (cbp_rem != 0): block number, contexts, intra DC
    auto start_block = [&]() {
        const int blk = __ffs(cbp_rem) - 1;
#if EF_K1B_DEQUANT
        blk24 = ((uint32_t)blk << 27) | ((uint32_t)s.qscale << 16);
#else
        blk24 = (uint32_t)blk << 24;
#endif
        blkbit = 0x100u << blk;
        cbp_rem &= cbp_rem - 1;
        n = 0; ctx = 1;                                       // dct_coeff_first: no end of block, '1s' = (0, 1)
        if (intra) { D.mb_rec[slot].dc[blk] = parse_dc(s, blk); n = 1; ctx = 0; }
    };
    // next list entry of the slice: into the lane's ring
    auto put_entry = [&](uint32_t ent) {
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(EF_SSTAGE + (tot % kStage) * 4), "r"(ent) : "memory");
        tot++;
    };
    // warp-wide (all lanes converged): every lane's entries still in its ring go to the list in HBM. Lane j stores
    // entry j of one lane's pending run, so each store instruction writes one contiguous run of one list
    auto flush = [&]() {
        __syncwarp();                                                 // the ring words of other lanes are read below, and rewritten after
#if !EF_PROBE_NOSTORE                                                 /* bottleneck probe (wrong output): no list stores */
        const uint32_t pend = tot - done;                             // <= kStage
        const uint64_t dst = (uint64_t)(s.list + done);
        const uint32_t key = pend | (done << 8);                      // run length | ring position of its first entry
        unsigned owed = __ballot_sync(0xFFFFFFFFu, pend != 0);
        while (owed) {
            const int src = __ffs(owed) - 1;
            owed &= owed - 1;
            const uint32_t k = __shfl_sync(0xFFFFFFFFu, key, src);
            uint32_t* const d = (uint32_t*)((uint64_t)__shfl_sync(0xFFFFFFFFu, (uint32_t)dst, src) | ((uint64_t)__shfl_sync(0xFFFFFFFFu, (uint32_t)(dst >> 32), src) << 32));
            if ((uint32_t)lane < (k & 255u)) {
                uint32_t v;
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(sstage_warp + (uint32_t)src * kStageRow + (((k >> 8) + lane) % kStage) * 4) : "memory");
                d[lane] = v;
            }
        }
#endif
        __syncwarp();
        done = tot;
    };
    // first round: thread t takes slice t; afterwards lanes whose slice ended pull from the cursor
    const uint32_t first_round = gridDim.x * blockDim.x;
    bool first_fill = true;

    for (;;) {
        // ---- header phase: records of finished macroblocks ------------------------------------------
        if (!busy && (info_acc & 1u)) {
            const uint64_t li = (uint64_t)(s.list - D.coef) + mb0;
            *(uint4*)(D.mb_rec + slot) = make_uint4((tot - mb0) | (skipw << 16), mvw, (uint32_t)li, (uint32_t)(li >> 32));
#if EF_K1B_DEQUANT
            if (s.qz) { info_acc |= 1u << 26; D.mb_rec[slot].pad[0] = s.seqi; }     // K1b dequantises with the stream's own matrices
#endif
            D.mb_info[slot] = info_acc | ((uint32_t)s.mbw << 20) | ((s.slot_base >> 31) << 25);
            info_acc = 0;
        }
        // ---- refill lanes without a slice, parse the header of every waiting lane -------------------
        do {
            if (__any_sync(0xFFFFFFFFu, !active && tot != done)) flush();   // a lane's ring is emptied before it takes its next slice
            unsigned need = __ballot_sync(0xFFFFFFFFu, !active && !exhausted);
            if (need) {
                uint32_t base;
                if (first_fill) {
                    base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u;
                    first_fill = false;
                } else {
                    base = 0;
                    int leader = __ffs(need) - 1;
                    if (lane == leader) base = first_round + atomicAdd(D.parse_cursor, (uint32_t)__popc(need));
                    base = __shfl_sync(0xFFFFFFFFu, base, leader);
                }
                if (!active && !exhausted) {
                    uint32_t idx = base + (uint32_t)__popc(need & ((1u << lane) - 1));
                    if (idx >= total) exhausted = true;
                    else {
                        const EfWork w = work[idx];
                        const int code = w.info & 255;
                        s.ptype = (w.info >> 8) & 7; s.full_pel = (w.info >> 11) & 1; s.r_size = (w.info >> 12) & 7;
                        const EfSeq* seq = D.seq + (size_t)w.stream * (D.max_seq + 1) + (w.info >> 16);
                        s.mbw = min((int)seq->mb_width, EF_MBW_MAX);
                        s.qz = seq->custom ? (const uint32_t*)seq->qz : nullptr;
                        s.seqi = w.info >> 16;
                        s.qzp = s.qz ? s.qz : T.qz;
                        const uint64_t byte_off = D.es_off[w.stream] + w.es_off;
                        s.slot_base = (w.pic - (uint32_t)pic0) * n_slots + w.stream * (uint32_t)(EF_MBW_MAX * EF_MBH_MAX);
                        s.slot_base |= ((D.base_pics[w.stream] + w.pic + 1u) & 1u) << 31;      // destination frame store: flush_picture(), player.cpp:692
                        s.list = D.coef + 3 * byte_off;          // >= 3 bits of bitstream per coefficient: lists cannot collide
                        tot = done = 0;
                        s.br.init(D.es, byte_off);
                        s.mb_y = code - 2; s.mb_x = s.mbw - 1;   // slice(), player.cpp:1255: the first increment lands on column 0 of row code-1
                        s.first = 1;
                        s.dc_y = s.dc_cr = s.dc_cb = 128; s.mv_h = s.mv_v = 0;
                        active = code >= 1 && code - 2 < (int)seq->mb_height && s.mbw > 0 && seq->valid;     // player.cpp:1257
                        if (active) {
                            s.qscale = (int)s.br.get(5);
                            while (s.br.get(1)) s.br.skip(8);    // extra_information_slice
                        }
                    }
                }
            }
            if (active && !busy && !(info_acc & 1u)) {
                if (parse_header(s, T, cbp_rem, intra, skipw, mvw)) {
                    slot = (s.slot_base & 0x7FFFFFFFu) + (uint32_t)(s.mb_y * EF_MBW_MAX + s.mb_x);
                    info_acc = 1u | ((uint32_t)intra << 1) | ((uint32_t)cbp_rem << 2);
                    mb0 = tot;
                    busy = cbp_rem != 0;
                    if (busy) start_block();
                } else active = false;
            }
        } while (__any_sync(0xFFFFFFFFu, !active && !exhausted));
        const unsigned amask = __ballot_sync(0xFFFFFFFFu, active);
        if (!amask) break;

        // ---- symbol loop: each lane runs through its own macroblock; a lane whose macroblock is complete waits (its
        // record is owed) until the loop ends, when no lane is busy or when kHdrBatch lanes are waiting. Per pass, every
        // busy lane takes EF_K1A_UNROLL steps (v3) or one two-symbol step
        const int qoff = intra ? 0 : 64, kq = intra ? 0 : 1;
#if EF_K1A_V3
        const uint32_t* const qrow = s.qzp + qoff;               // table words of this macroblock's matrix, by scan position
#else
        // table word of scan position n: shared memory for the default matrices (no global-load latency in the symbol
        // chain), the stream's own table in HBM otherwise (sequence headers that load matrices are rare)
        auto qword = [&](int pos) -> uint32_t { return s.qz ? __ldg(s.qz + qoff + pos) : T.qz[qoff + pos]; };
#endif
        for (;;) {
            const unsigned bmask = __ballot_sync(0xFFFFFFFFu, busy);
            if (!bmask || __popc(amask & ~bmask) >= kHdrBatch) break;
            if (__any_sync(0xFFFFFFFFu, tot - done > (uint32_t)kStageHigh)) flush();
#if EF_K1A_V3
            // per step ONE run/level symbol through the clz-indexed table, a following end of block folded in;
            // dequantised on the spot (table word of the scan position: shared memory for the default matrices, the
            // stream's own table in HBM otherwise) or, with EF_K1B_DEQUANT, stored as a raw token
#pragma unroll
            for (int u_ = 0; u_ < EF_K1A_UNROLL; u_++)
            if (busy) {
                BitReader& br = s.br;
                const uint32_t w = br.peek();
                const EfSym sy = ef_coef_sym(w, ctx != 0, T.dct);
                ctx = 0;
                int len = sy.len;
                bool block_done = sy.kind == EF_SYM_EOB;
                if (sy.kind == EF_SYM_DERAIL) {                  // give up on this and the remaining blocks, end the slice
                    info_acc |= (blkbit << 6) | ((uint32_t)cbp_rem << 14);
                    s.mb_y = EF_MBH_MAX;
                    busy = false;
                } else {
                    if (sy.kind == EF_SYM_COEF) {
                        n += sy.run;
                        if (n > 63) { info_acc |= blkbit << 6; block_done = true; }      // block() returns -1: nothing of the block is stored; the symbol is consumed
                        else {
#if EF_K1B_DEQUANT
                            put_entry(blk24 | ((uint32_t)n << 21) | ((uint32_t)sy.lvl & 0xFFFFu));
#else
                            put_entry(ef_coef_entry(qrow[n], sy.lvl, s.qscale, kq, blk24));
#endif
                            n++;
                            if (len <= 30 && ((w << len) >> 30) == 2u) { len += 2; block_done = true; }   // '10' follows: end of block
                        }
                    }
                    br.skip(len);
                    if (block_done) {
                        if (n == 1) info_acc |= blkbit;          // Q5 (an aborted block has n >= 64)
                        busy = cbp_rem != 0;
                        if (busy) start_block();
                    }
                }
            }
#else
            // per step up to two coefficients and an end of block. Fast path: the next kLutBits bits index the
            // two-symbol table; everything that lies wholly inside them (one or two run/level codes with their sign
            // bits, a closing '10') is taken in one step. Long codes, the escape, invalid prefixes and symbols that
            // would run past scan position 63 decode one symbol through the clz-indexed table (and fold a following
            // end of block in).
            if (busy) {
                BitReader& br = s.br;
                const uint32_t w = br.peek();
                const EfCoefStep st = ef_coef_step(w, ctx != 0, n, lut, T.dct);
                const uint32_t fl = st.fl;
                const int len = st.len;
                ctx = 0;
                if (fl & EF_STEP_COEF1) { n += st.run1; put_entry(ef_coef_entry(qword(n), st.lvl1, s.qscale, kq, blk24)); n++; }
                if (fl & EF_STEP_COEF2) { n += st.run2; put_entry(ef_coef_entry(qword(n), st.lvl2, s.qscale, kq, blk24)); n++; }
                if (fl & 16u) {                                // give up on this and the remaining blocks, end the slice
                    info_acc |= (blkbit << 6) | ((uint32_t)cbp_rem << 14);
                    s.mb_y = EF_MBH_MAX;
                    busy = false;
                } else {
                    br.skip(len);
                    if (fl & 12u) {
                        if (fl & 8u) info_acc |= blkbit << 6;
                        else if (n == 1) info_acc |= blkbit;   // Q5
                        busy = cbp_rem != 0;
                        if (busy) start_block();
                    }
                }
            }
#endif
        }
    }
#undef EF_SSTAGE
}

// =================================================================================================
// K1b: macroblock records -> pixels, one launch per picture index. A HALF-WARP rebuilds one
// macroblock (a warp = two consecutive macroblock slots): its 48 eight-pixel row segments are 3 passes
// of 16 lanes, so every lane is busy in every pass, and the per-macroblock bookkeeping (record decode,
// TMA issue, list expansion) is paid once per two macroblocks.
//   lane hl = lane & 15 of a half:  column pass p (p = 0..2): block 2p + hl/8, column hl%8
//                                   row pass 0, 1: luma row 8p + hl/2, 8-pixel half hl%2 (block 2p + hl%2)
//                                   row pass 2:    chroma plane hl/8 (block 4 + hl/8), row hl%8
// =================================================================================================
__global__ void __launch_bounds__(kReconWarps * 32, kReconCtasPerSm)
ef_recon_kernel(const __grid_constant__ EfDev D, int pic_rel)
{
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int hl = lane & 15, hb = lane & 16, half = lane >> 4;
    uint8_t* wbase = smem + (size_t)warp * kWarpBytes;
    int* dense = (int*)wbase + half * kDenseWords;
    uint8_t* stage = wbase + 2 * kDenseBytes + half * kStageBytes;
    uint64_t* bar = (uint64_t*)(wbase + 2 * kDenseBytes + 2 * kStageBytes) + half;
    const uint32_t sstage = smem_u32(stage), sbar = smem_u32(bar);
    uint32_t bar_phase = 0;
    if (hl == 0) mbar_init(bar, 1);
    for (int i = hl; i < kDenseWords; i += 16) dense[i] = 0;
#if EF_K1B_DEQUANT
    const uint32_t* qzs = (const uint32_t*)(smem + (size_t)kReconWarps * kWarpBytes);   // default matrices: quantiser | prescale << 8 | raster index << 18 per scan position
    for (int i = threadIdx.x; i < 128; i += blockDim.x) ((uint32_t*)qzs)[i] = D.tables->qz[i];
    __syncthreads();
#endif
    __syncwarp();

    constexpr uint32_t kMbs = EF_MBW_MAX * EF_MBH_MAX;
    const uint32_t n_slots = (uint32_t)D.n_streams * kMbs;            // even
    const uint32_t* infos = D.mb_info + (size_t)pic_rel * n_slots;
    const uint32_t* recs = (const uint32_t*)(D.mb_rec + (size_t)pic_rel * n_slots);

    const int ccol = hl & 7, cpb = hl >> 3;         // column pass: column, block within the pair
    const int prow = hl >> 1, phalf = hl & 1;       // luma row passes
    const int crow = hl & 7, cplane = hl >> 3;      // chroma row pass

    // one load per lane fetches a record: lanes 0-9 of the half its words, lane 12 the info word
    auto fetch = [&](uint32_t slot) -> uint32_t {
        uint32_t v = 0;
        if (slot < n_slots && (hl < (EF_K1B_DEQUANT ? 11 : 10) || hl == 12)) v = __ldg(hl == 12 ? infos + slot : recs + (size_t)slot * (sizeof(EfMbRec) / 4) + hl);
        return v;
    };

    // Work distribution: the first two pairs of a warp are static, later ones come from a global cursor
    // (the warp schedulers do not share the issue slots evenly, so a static split leaves a long tail). The
    // atomic is issued two iterations ahead of its use and the record one iteration ahead.
    const uint32_t n_warps = gridDim.x * kReconWarps;
    uint32_t* cursor = D.recon_cursor + pic_rel;
    uint32_t pair = blockIdx.x * kReconWarps + warp, pair_next = pair + n_warps, pair_fut = 0;
    uint32_t pre = fetch(pair * 2 + half);
    for (;; pair = pair_next, pair_next = __shfl_sync(0xFFFFFFFFu, pair_fut, 0)) {
        if (pair * 2 >= n_slots) break;
        const uint32_t slot = pair * 2 + half;
        const uint32_t recw = pre;
        pre = fetch(pair_next * 2 + half);
        if (lane == 0) pair_fut = 2 * n_warps + atomicAdd(cursor, 1u);
        const uint32_t info = __shfl_sync(0xFFFFFFFFu, recw, hb + 12);
        const bool valid = info & 1u;
        if (!__any_sync(0xFFFFFFFFu, valid)) continue;
        const uint32_t cntw = __shfl_sync(0xFFFFFFFFu, recw, hb);
        const uint32_t mvw = __shfl_sync(0xFFFFFFFFu, recw, hb + 1);
        const uint64_t li = (uint64_t)__shfl_sync(0xFFFFFFFFu, recw, hb + 2) | ((uint64_t)__shfl_sync(0xFFFFFFFFu, recw, hb + 3) << 32);
        const uint32_t stream = slot / kMbs, mb = slot - stream * kMbs;
        const int my = (int)(mb / EF_MBW_MAX), mx = (int)(mb - (uint32_t)my * EF_MBW_MAX);
        const uint32_t fb = (info >> 25) & 1u;                                      // flush_picture(), player.cpp:692
        uint8_t* cur = D.frames + ef_frame_offset((int)stream, (int)fb);
        const uint8_t* ref = D.frames + ef_frame_offset((int)stream, (int)(fb ^ 1u));
        const bool intra_r = (info >> 1) & 1;
        const int cbp = valid ? (info >> 2) & 63 : 0, n1m = (info >> 8) & 63;
        const int abm = ((info >> 14) & 63) | 0xC0;                                 // block numbers 6, 7 (damaged record): dropped
        const int mbw = (info >> 20) & 31;
        const int entries = valid ? min((int)(cntw & 0xFFFF), 384) : 0, skip_before = valid ? (int)(cntw >> 16) : 0;
        const int live = cbp & ~abm;
        const bool do_mc = valid && !intra_r;

        // coefficient list: issue the loads first
        const uint32_t* rl = D.coef + li;
        uint32_t e0 = 0, e1 = 0, e2 = 0;
        if (hl < entries) e0 = __ldg(rl + hl);
        if (hl + 16 < entries) e1 = __ldg(rl + hl + 16);
        if (hl + 32 < entries) e2 = __ldg(rl + hl + 32);

        const int mvh = (int)(int16_t)(mvw & 0xFFFF), mvv = (int)(int16_t)(mvw >> 16);
        const int tile = ef_tile_offset(mx, my);
        const int hx = mx * 32 + mvh, hy = my * 32 + mvv;                       // predict(), player.cpp:882
        const int cx = hx >> 1, cy = hy >> 1;                                   // Q3: floor
        const int X0 = hx >> 1, Y0 = hy >> 1, tx0 = X0 >> 4, ty0 = Y0 >> 4;
        // whole prediction window inside the picture (always, for streams the reference accepts)
        const bool inside = hx >= 0 && hy >= 0 && X0 + 16 + (hx & 1) <= EF_W && Y0 + 16 + (hy & 1) <= EF_H;
        if (do_mc && inside && hl == 0) {
            // reference tiles by TMA bulk copy: the prediction window lies in at most 2 x 2 tiles, tiles of
            // one row are contiguous in HBM. (The staging area is only written by these copies and read with
            // plain loads that have all completed before the __syncwarp() that ended the previous iteration.)
            const bool two_x = ((X0 + 15 + (hx & 1)) >> 4) != tx0, two_y = ((Y0 + 15 + (hy & 1)) >> 4) != ty0;
            const uint8_t* src = ref + ef_tile_offset(tx0, ty0);
            const uint32_t row_bytes = two_x ? 2 * EF_TILE : EF_TILE;
            mbar_expect_tx(sbar, row_bytes << (int)two_y);
            bulk_tiles(sstage, src, row_bytes, sbar);
            if (two_y) bulk_tiles(sstage + 2 * EF_TILE, src + EF_MBW_MAX * EF_TILE, row_bytes, sbar);
        }

        // skipped macroblocks: predict_zero() copies them from the reference frame (player.cpp:1283-1288)
        if (skip_before) {
            int sx = mx, sy = my;
            for (int k = 0; k < skip_before; k++) {
                if (--sx < 0) { sx = mbw - 1; sy--; }
                if (sy < 0) break;
                const int to = ef_tile_offset(sx, sy);
                *(uint4*)(cur + to + hl * 16) = *(const uint4*)(ref + to + hl * 16);
                *(uint2*)(cur + to + 256 + hl * 8) = *(const uint2*)(ref + to + 256 + hl * 8);
            }
        }

        // expand the coefficient list into the dense scratch (entries of aborted blocks are dropped)
#if EF_K1B_DEQUANT
        // token = block << 27 | scan position << 21 | quantiser_scale << 16 | (int16) level: dequantise here (block(),
        // player.cpp:1106-1121), with the table word of the scan position from shared memory (default matrices) or from
        // the stream's sequence state (info bit 26; record word 10 = its index)
        const int qoff = intra_r ? 0 : 64, kq = intra_r ? 0 : 1;
        const uint32_t seqi = __shfl_sync(0xFFFFFFFFu, recw, hb + 10);
        const uint32_t* cqz = nullptr;
        if (valid && ((info >> 26) & 1u)) cqz = D.seq[(size_t)stream * (D.max_seq + 1) + min(seqi, (uint32_t)D.max_seq)].qz;
#define EF_EXPAND(ent) { const uint32_t t_ = (ent); const int eb = (t_ >> 27) & 7; if (!((abm >> eb) & 1)) { const int n_ = qoff + ((t_ >> 21) & 63); \
            const uint32_t z_ = cqz ? __ldg(cqz + n_) : qzs[n_]; dense[eb * kDenseStride + ((z_ >> 18) & 63)] = ef_dequant(z_, (int)(int16_t)(t_ & 0xFFFFu), (int)((t_ >> 16) & 31u), kq); } }
#else
        // entry = (block << 24 | raster position << 18) + value, |value| < 2^17: adding 2^17 undoes the borrow of a negative value
#define EF_EXPAND(ent) { const uint32_t hi_ = (ent) + 0x20000u; const int eb = (hi_ >> 24) & 7; if (!((abm >> eb) & 1)) dense[eb * kDenseStride + ((hi_ >> 18) & 63)] = ((int)((ent) << 14)) >> 14; }
#endif
        if (hl < entries) EF_EXPAND(e0)
        if (hl + 16 < entries) EF_EXPAND(e1)
        if (hl + 32 < entries) EF_EXPAND(e2)
        for (int j = hl + 48; j < entries; j += 16) { const uint32_t ent = __ldg(rl + j); EF_EXPAND(ent) }
#undef EF_EXPAND
        __syncwarp();                                                           // dense[] complete

        // ---- column passes, in place: lane (block, column) owns the 8 words dense[block][0..7][column]
        unsigned pass_on = 0;
#pragma unroll
        for (int p = 0; p < 3; p++) {
            if (!__any_sync(0xFFFFFFFFu, live & (3 << (2 * p)))) continue;       // warp-uniform
            pass_on |= 1u << p;
            const int bk = 2 * p + cpb;
            const int dc_col = (int)__shfl_sync(0xFFFFFFFFu, recw, hb + 4 + bk);  // intra DC of that block
            int* db = dense + bk * kDenseStride + ccol;
            int v[8];
#pragma unroll
            for (int rr = 0; rr < 8; rr++) v[rr] = db[rr * 8];
            if (intra_r && ccol == 0) v[0] = (int)((uint32_t)dc_col << 8);       // b[0] <<= 8, player.cpp:1065
            idct8<false>(v);
#pragma unroll
            for (int rr = 0; rr < 8; rr++) db[rr * 8] = v[rr];
        }
        __syncwarp();

        if (do_mc && inside) { mbar_wait(sbar, bar_phase); bar_phase ^= 1; }

        // ---- row passes: residual row, prediction, clamped add, store ---------------------------------
#pragma unroll
        for (int p = 0; p < 3; p++) {
            const bool luma = p < 2;
            const int oblk = luma ? 2 * p + phalf : 4 + cplane;
            const int orow = luma ? prow : crow;
            int w[8], dcv = 0;
#pragma unroll
            for (int i = 0; i < 8; i++) w[i] = 0;
            if (pass_on & (1u << p)) {                                           // warp-uniform
                const int dc_row = (int)__shfl_sync(0xFFFFFFFFu, recw, hb + 4 + oblk);
                int4* rowp = (int4*)(dense + oblk * kDenseStride + orow * 8);
                const int4 a = rowp[0], b = rowp[1];
                rowp[0] = make_int4(0, 0, 0, 0); rowp[1] = make_int4(0, 0, 0, 0);    // leave the scratch zeroed for the next macroblock
                w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
                if ((live >> oblk) & 1) {
                    if (!((n1m >> oblk) & 1)) idct8<true>(w);        // residuals scaled by 256
                    else {                                           // n == 1: dc = b[0] >> 8 (Q5); after the column pass every row holds b[0] in column 0
                        dcv = intra_r ? dc_row : w[0] >> 8;
#pragma unroll
                        for (int i = 0; i < 8; i++) w[i] = dcv * 256;
                    }
                }
            }
            // prediction: the four cases of mocomp()
            uint32_t q0 = 0, q1 = 0;
            if (do_mc) {
                PredWords pw;
                if (luma) {
                    const int lx = (hx >> 1) + phalf * 8, ly = (hy >> 1) + p * 8 + prow;
                    if (inside) pred_words_staged<true>(stage, 0, lx, ly, tx0, ty0, hy & 1, pw);
                    else pred_words_clamped<true>(ref, 0, lx, ly, hy & 1, pw);
                    pred_finish(pw, lx, hx & 1, hy & 1, q0, q1);
                } else {
                    const int kx = cx >> 1, ky = (cy >> 1) + crow;
                    if (inside) pred_words_staged<false>(stage, cplane, kx, ky, tx0, ty0, cy & 1, pw);
                    else pred_words_clamped<false>(ref, cplane, kx, ky, cy & 1, pw);
                    pred_finish(pw, kx, cx & 1, cy & 1, q0, q1);
                }
            }
            // combine + store (copy_block / copy_block_dc / add_block / add_block_dc)
            const bool coded = (cbp >> oblk) & 1, aborted = (abm >> oblk) & 1, n1 = (n1m >> oblk) & 1;
            uint32_t o0 = q0, o1 = q1;
            bool store = valid;
            if (coded && !aborted) {
                if (intra_r && n1) {                                 // copy_block_dc: replicated, not clamped (Q7)
                    uint32_t d = (uint32_t)dcv; d |= d << 8; d |= d << 16;
                    o0 = o1 = d;
                } else {
                    o0 = pin4(q0, w[0], w[1], w[2], w[3]);
                    o1 = pin4(q1, w[4], w[5], w[6], w[7]);
                }
            } else if (intra_r) store = false;                        // aborted intra block: destination untouched
            uint8_t* dst = cur + tile + (luma ? (p * 8 + prow) * 16 + phalf * 8 : 256 + cplane * 64 + crow * 8);
            if (store) *(uint2*)dst = make_uint2(o0, o1);
        }
        __syncwarp();
    }
}

// host-side launch helpers -----------------------------------------------------------------------
size_t ef_recon_smem_bytes() { return (size_t)kReconWarps * kWarpBytes + kReconQzBytes; }
static constexpr size_t kParseSmemBytes = (size_t)kTableBytes + kLutBytes + kRingBytes + kStageBytesA;

static int g_parse_ctas = kParseCtasPerSm, g_recon_ctas = kReconCtasPerSm;   // resident CTAs per SM, measured by the occupancy API

cudaError_t ef_decode_configure()
{
    cudaError_t e = cudaFuncSetAttribute(ef_recon_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ef_recon_smem_bytes());
    if (e != cudaSuccess) return e;
    // K1b wants shared memory (two macroblock scratch areas per warp), not L1
    e = cudaFuncSetAttribute(ef_recon_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    int n = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, ef_recon_kernel, kReconWarps * 32, ef_recon_smem_bytes());
    if (e != cudaSuccess) return e;
    if (n >= 1) g_recon_ctas = n;
    e = cudaFuncSetAttribute(ef_parse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kParseSmemBytes);
    if (e != cudaSuccess) return e;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, ef_parse_kernel, kParseThreads, kParseSmemBytes);
    if (e != cudaSuccess) return e;
    if (n >= 1) g_parse_ctas = n;
    return cudaSuccess;
}

int ef_decode_resident_ctas(int which) { return which == 0 ? g_parse_ctas : g_recon_ctas; }

// parse every slice of picture indices [pic0, pic0 + n_pics) into record pictures 0 .. n_pics-1
// (grids are persistent - one wave of resident CTAs - but never larger than the work: a one-stream context of the
// level-1 drop-in launches a handful of CTAs, not 592 that each stage 20 KB of tables first)
cudaError_t ef_launch_parse(const EfDev& dev, int pic0, int n_pics, int sm_count, size_t max_slices, cudaStream_t stream)
{
    size_t grid = (size_t)sm_count * g_parse_ctas, need = (max_slices + kParseThreads - 1) / kParseThreads;
    if (need < 1) need = 1;
    if (need < grid) grid = need;
    ef_parse_kernel<<<(unsigned)grid, kParseThreads, kParseSmemBytes, stream>>>(dev, pic0, n_pics);
    return cudaGetLastError();
}

// rebuild one picture index of every stream from record picture `pic_rel`
cudaError_t ef_launch_recon(const EfDev& dev, int pic_rel, int sm_count, size_t n_slots, cudaStream_t stream)
{
    size_t grid = (size_t)sm_count * g_recon_ctas, need = (n_slots / 2 + kReconWarps - 1) / kReconWarps;
    if (need < 1) need = 1;
    if (need < grid) grid = need;
    ef_recon_kernel<<<(unsigned)grid, kReconWarps * 32, ef_recon_smem_bytes(), stream>>>(dev, pic_rel);
    return cudaGetLastError();
}
