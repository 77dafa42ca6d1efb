// espflix_b200/csrc/ef_index.cu — K1a: start-code scan, header parse and slice work lists, done
// once per submit for the whole batch, entirely on the device.
//
// Replaces the serial start-code search of MpegDecoder::run() (player.cpp:1360-1363), the marker
// dispatch (player.cpp:1318-1340) and the header parsers sequence()/gop()/picture()
// (player.cpp:658-724). The reference walks the stream bit by bit from one start code to the next;
// start codes are byte aligned in every stream it accepts (Q8), so here a warp sweeps 512 bytes of
// one stream per step with 128-bit loads, finds "00 00 01 xx" with byte permutes, and orders the
// hits with a ballot + popcount prefix so the picture/slice tables come out in stream order.
//   ef_scan_kernel    one warp per stream   -> seq[], pics[], slice_off[], slice_code[], n_pics[]
//   ef_prefix_kernel  one CTA               -> per picture index: exclusive prefix over streams
//   ef_fill_kernel    one thread per (picture, stream) -> flat EfWork list per picture index
// TS input (the reference's wire format) is first compacted to an elementary stream by
//   ef_ts_len_kernel / ef_ts_copy_kernel    one thread per 188-byte packet (more()/demux(),
//                                           player.cpp:381-493)
// and, after ef_pts_enable, the presentation timestamp of every picture by
//   ef_pts_packet_kernel (per TS submit, one CTA per stream) / ef_pts_resolve_kernel (per ef_index, one warp per stream)
#include "ef_common.cuh"
#include "ef_iso11172_tables.h"

namespace {

__device__ __forceinline__ uint32_t ld_byte(const uint8_t* es, uint64_t len, uint64_t i) { return i < len ? es[i] : 0u; }

// read `n` (<= 24) bits at bit offset `bit` of the stream
__device__ __forceinline__ uint32_t bits_at(const uint8_t* es, uint64_t len, uint64_t bit, int n)
{
    uint64_t byte = bit >> 3;
    uint32_t w = (ld_byte(es, len, byte) << 24) | (ld_byte(es, len, byte + 1) << 16) | (ld_byte(es, len, byte + 2) << 8) | ld_byte(es, len, byte + 3);
    return (w << (bit & 7)) >> (32 - n);
}

__constant__ uint8_t c_default_intra_q[64];

}  // namespace

cudaError_t ef_index_upload_constants()
{
    return cudaMemcpyToSymbol(c_default_intra_q, ef_default_intra_q, 64);
}

__global__ void __launch_bounds__(128)
ef_scan_kernel(EfDev* __restrict__ Dp)
{
    EfDev& D = *Dp;
    const int lane = threadIdx.x & 31;
    const int s = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (s >= D.n_streams) return;

    EfSeq* seqs = D.seq + (size_t)s * (D.max_seq + 1);
    EfPic* pics = D.pics + (size_t)s * D.max_pictures;
    uint32_t* soff = D.slice_off + (size_t)s * D.max_slices;
    uint8_t* scode = D.slice_code + (size_t)s * D.max_slices;

    // roll the state of the previous submit: ping-pong phase, the last sequence header and the forward-vector
    // parameters of the last P picture header (decoder members in the reference, player.cpp:716-722)
    uint32_t fp_rs = seqs[0].fp_rs;
    __syncwarp();
    {
        const uint32_t prev_seq = min(D.n_seq[s], (uint32_t)D.max_seq);
        if (prev_seq) {
            const uint32_t* src = (const uint32_t*)(seqs + prev_seq);
            uint32_t* dst = (uint32_t*)seqs;
            for (int i = lane; i < (int)(sizeof(EfSeq) / 4); i += 32) dst[i] = src[i];
        }
        if (lane == 0) { D.base_pics[s] += D.n_pics[s]; }
        __syncwarp();
    }

    const uint8_t* es = D.es + D.es_off[s];
    const uint64_t len = D.es_off[s + 1] - D.es_off[s];
    const uintptr_t misalign = (uintptr_t)es & 15;
    const uint8_t* abase = es - misalign;                 // 16-byte aligned sweep origin
    const uint64_t span = len + misalign;

    uint32_t n_pic = 0, n_slice = 0, n_seq = 0;           // warp-uniform running counts
    // fp_rs: full_pel | r_size << 1 of the last P header (stale state a B/D picture would see)
    bool stop = false;

    // the sweep is latency bound (one warp per stream): keep the loads of the next two 512-byte chunks in flight
    auto load_chunk = [&](uint64_t chunk, uint4& v, uint32_t& nxt) {
        const uint64_t o = chunk + (uint64_t)lane * 16;
        v = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
        nxt = 0xFFFFFFFFu;
        if (o < span) v = __ldg((const uint4*)(abase + o));
        if (o + 16 < span) nxt = __ldg((const uint32_t*)(abase + o + 16));
    };
    uint4 v, v1, v2;
    uint32_t nxt, nxt1, nxt2;
    load_chunk(0, v, nxt);
    load_chunk(512, v1, nxt1);
    for (uint64_t chunk = 0; chunk < span && !stop; chunk += 512, v = v1, nxt = nxt1, v1 = v2, nxt1 = nxt2) {
        const uint64_t o = chunk + (uint64_t)lane * 16;
        load_chunk(chunk + 1024, v2, nxt2);
        const uint32_t w[5] = { v.x, v.y, v.z, v.w, nxt };
        // "00 00 01" at byte i of the lane's 20-byte window, all 16 positions at once: exact per-byte masks of the zero
        // bytes and of the bytes equal to 1 (0x80 in the byte), shifted against each other across the word boundaries
        // (about 3 integer operations per stream byte; the per-position compare it replaces took 10 and made the scan
        // ALU bound: profiles/r02_k0_ncu.txt). Positions before the stream or within 4 bytes of its end are dropped below.
        uint32_t zm[5], om[5];
#pragma unroll
        for (int k = 0; k < 5; k++) {
            const uint32_t x = w[k] ^ 0x01010101u;
            zm[k] = ~(((w[k] & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | w[k]) & 0x80808080u;
            om[k] = ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
        }
        uint32_t hits = 0;
        uint32_t any = 0, hm[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            hm[k] = zm[k] & __funnelshift_r(zm[k], zm[k + 1], 8) & __funnelshift_r(om[k], om[k + 1], 16);
            any |= hm[k];
        }
        if (any) {                                                            // bit 7 of byte j of word k -> bit 4k + j
#pragma unroll
            for (int k = 0; k < 4; k++) hits |= ((((hm[k] >> 7) * 0x00204081u) >> 21) & 15u) << (4 * k);
        }
        unsigned lanes = __ballot_sync(0xFFFFFFFFu, hits != 0);
        while (lanes && !stop) {
            const int src = __ffs(lanes) - 1;
            uint32_t h = __shfl_sync(0xFFFFFFFFu, hits, src);
            const uint64_t obase = chunk + (uint64_t)src * 16;
            while (h && !stop) {
                const int i = __ffs(h) - 1;
                h &= h - 1;
                if (obase + i < misalign || obase + i - misalign + 4 > len) continue;   // window bytes outside the stream (alignment slack, tail)
                const uint64_t pos = obase + i - misalign;                    // first 00 of the start code
                // the start-code value is byte i + 3 of the owning lane's 20-byte window: a shuffle, not another
                // dependent global load per start code (the sweep is latency bound, ~170 start codes per stream)
                const int bi = i + 3;
                const uint32_t wsel = bi < 4 ? w[0] : bi < 8 ? w[1] : bi < 12 ? w[2] : bi < 16 ? w[3] : w[4];
                const uint32_t code = __shfl_sync(0xFFFFFFFFu, (wsel >> ((bi & 3) * 8)) & 0xFFu, src);
                if (code == 0x00) {                                           // picture(), player.cpp:704
                    const uint32_t idx = n_pic++;
                    const uint64_t hb = (pos + 4) * 8;
                    const uint32_t type = bits_at(es, len, hb + 10, 3);
                    if (type == 2) {
                        const uint32_t fp = bits_at(es, len, hb + 29, 1);
                        const uint32_t fc = bits_at(es, len, hb + 30, 3);
                        fp_rs = fp | (((fc - 1u) & 7u) << 1);
                    }
                    if (idx < (uint32_t)D.max_pictures && lane == 0) {
                        EfPic p;
                        p.first_slice = n_slice; p.n_slices = 0; p.type = (uint8_t)type; p.fp_rsize = (uint8_t)fp_rs;
                        p.seq = (uint16_t)min(n_seq, (uint32_t)D.max_seq); p.code_off = (uint32_t)(pos + 3);
                        pics[idx] = p;
                    }
                } else if (code >= 0x01 && code <= 0xAF) {                    // slice start code
                    if (n_pic > 0 && n_pic <= (uint32_t)D.max_pictures) {     // slices of pictures beyond max_pictures are dropped with them (info[3] flags the overflow)
                        const uint32_t j = n_slice++;
                        if (j < (uint32_t)D.max_slices && lane == 0) { soff[j] = (uint32_t)(pos + 4); scode[j] = (uint8_t)code; }
                    }
                } else if (code == 0xB3) {                                    // sequence(), player.cpp:658
                    const uint32_t k = ++n_seq;
                    if (k <= (uint32_t)D.max_seq) {
                        const uint64_t hb = (pos + 4) * 8;
                        const uint32_t hsize = bits_at(es, len, hb, 12), vsize = bits_at(es, len, hb + 12, 12);
                        const uint32_t load_intra = bits_at(es, len, hb + 62, 1);
                        const uint64_t after_intra = hb + 63 + (load_intra ? 512 : 0);
                        const uint32_t load_inter = bits_at(es, len, after_intra, 1);
                        EfSeq* q = seqs + k;
                        for (int n = lane; n < 64; n += 32) {
                            // Q4: the decoder keeps the 64 bytes in stream order and indexes them with the raster
                            // index zz = zigzag[n]; the tables here are stored per scan position n
                            const int zz = D.tables->zigzag[n];
                            const uint32_t qi = load_intra ? bits_at(es, len, hb + 63 + 8 * zz, 8) : c_default_intra_q[zz];
                            const uint32_t qn = load_inter ? bits_at(es, len, after_intra + 1 + 8 * zz, 8) : 16u;
                            const uint32_t hi = ((uint32_t)D.tables->prescale[zz] << 8) | ((uint32_t)zz << 18);     // EfTables::qz form
                            q->qz[n] = (qi & 255u) | hi;
                            q->qz[64 + n] = (qn & 255u) | hi;
                        }
                        if (lane == 0) {
                            q->mb_width = (uint16_t)((hsize + 15) >> 4);
                            q->mb_height = (uint16_t)((vsize + 15) >> 4);
                            q->valid = 1; q->custom = (uint16_t)((load_intra || load_inter) ? 1 : 0);
                        }
                    }
                } else if (code == 0xB7) {                                    // sequence end: the reference decoder parks in pause()
                    stop = true;
                }
            }
            lanes &= lanes - 1;
        }
    }
    __syncwarp();

    // fix-up: slice counts per picture = difference of consecutive first_slice
    const uint32_t np = min(n_pic, (uint32_t)D.max_pictures);
    const uint32_t ns = min(n_slice, (uint32_t)D.max_slices);
    for (uint32_t i = lane; i < np; i += 32) {
        const uint32_t first = min(pics[i].first_slice, ns);
        const uint32_t next = i + 1 < np ? min(pics[i + 1].first_slice, ns) : ns;
        pics[i].n_slices = next - first;
    }
    if (lane == 0) {
        seqs[0].fp_rs = fp_rs;                                  // both the carried entry and the one the next submit rolls into it
        seqs[min(n_seq, (uint32_t)D.max_seq)].fp_rs = fp_rs;
        D.n_pics[s] = np;
        D.n_seq[s] = n_seq;
        atomicMax(&D.info[0], np);
        atomicAdd(&D.info[1], np);
        atomicAdd(&D.info[2], ns);
        if (n_pic > (uint32_t)D.max_pictures || n_slice > (uint32_t)D.max_slices || n_seq > (uint32_t)D.max_seq) atomicOr(&D.info[3], 1u);
    }
}

// exclusive prefix of slices-per-stream, one CTA of 1024 threads per picture index (grid = max_pictures); the
// base of a picture index in the flat work list (sum of the totals before it) is taken in ef_fill_kernel
__global__ void __launch_bounds__(1024)
ef_prefix_kernel(EfDev* __restrict__ Dp)
{
    EfDev& D = *Dp;
    __shared__ uint32_t warp_sum[32];
    __shared__ uint32_t carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int p = blockIdx.x;
    const int pmax = min((int)D.info[0], D.max_pictures);
    if (p >= pmax) {
        if (threadIdx.x == 0) { D.pic_total[p] = 0; D.cursor[p] = 0; }
        return;
    }
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < D.n_streams; base += 1024) {
        const int s = base + threadIdx.x;
        uint32_t v = 0;
        if (s < D.n_streams && (uint32_t)p < D.n_pics[s]) v = D.pics[(size_t)s * D.max_pictures + p].n_slices;
        uint32_t x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= d) x += y; }
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint32_t t = warp_sum[lane], z = t;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xFFFFFFFFu, z, d); if (lane >= d) z += y; }
            warp_sum[lane] = z - t;                   // exclusive offsets of the warps
        }
        __syncthreads();
        const uint32_t excl = carry + warp_sum[warp] + x - v;
        if (s < D.n_streams) D.pic_pref[(size_t)p * D.n_streams + s] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) { D.pic_total[p] = carry; D.cursor[p] = 0; }
}

__global__ void __launch_bounds__(256)
ef_fill_kernel(EfDev* __restrict__ Dp)
{
    EfDev& D = *Dp;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int p = (int)(t / D.n_streams), s = (int)(t % D.n_streams);
    if (p >= D.max_pictures) return;
    if ((uint32_t)p >= D.n_pics[s]) {
        if (s == 0) { uint32_t b = 0; for (int q = 0; q < p; q++) b += D.pic_total[q]; D.pic_base[p] = b; }
        return;
    }
    const EfPic pic = D.pics[(size_t)s * D.max_pictures + p];
    const uint32_t first = pic.first_slice, seq_idx = pic.seq;
    uint32_t pbase = 0;                                      // work lists of consecutive picture indices are contiguous
    for (int q = 0; q < p; q++) pbase += D.pic_total[q];
    if (s == 0) D.pic_base[p] = pbase;
    const size_t dst = (size_t)pbase + D.pic_pref[(size_t)p * D.n_streams + s];
    // picture types other than I are parsed with the P tables (picture() ignores B/D headers but
    // their slices still reach slice(), player.cpp:716, 1292)
    const uint32_t type = pic.type == 1 ? 1u : 2u;
    for (uint32_t j = 0; j < pic.n_slices; j++) {
        if (dst + j >= D.work_capacity) { atomicOr(&D.info[3], 2u); return; }
        EfWork w;
        w.stream = (uint32_t)s;
        w.es_off = D.slice_off[(size_t)s * D.max_slices + first + j];
        w.info = (uint32_t)D.slice_code[(size_t)s * D.max_slices + first + j] | (type << 8) | ((uint32_t)(pic.fp_rsize & 15) << 11) | (seq_idx << 16);
        w.pic = (uint32_t)p;
        D.work[dst + j] = w;
    }
}

// ---- TS -> ES compaction -------------------------------------------------------------------------
// One thread per 188-byte packet: payload start/length for PID 0x100 following more()/demux()
// (player.cpp:381-493): sync byte, adaptation field, PES header skipped on payload_unit_start.
__device__ __forceinline__ void ts_payload(const uint8_t* d, int& start, int& n)
{
    start = 188; n = 0;
    if (d[0] != 0x47) return;
    const int pid = ((d[1] << 8) | d[2]) & 0x1FFF;
    if (pid != 0x100 || !(d[3] & 0x10)) return;
    int o = 4;
    if (d[3] & 0x20) o = 5 + d[4];
    if (d[1] & 0x40) { if (o + 9 > 188) return; o = o + 9 + d[o + 8]; }      // payload = d + 6 + 3 + header_data_length
    if (o < 188) { start = o; n = 188 - o; }
}

// pass 1: per-packet payload length; pass 2: exclusive scan of the lengths INSIDE every stream (one CTA per stream,
// streams are independent) + the stream totals; pass 3: scan of the totals -> ES offset of every stream; pass 4: copy.
__global__ void ef_ts_len_kernel(const uint8_t* __restrict__ ts, uint64_t n_packets, uint32_t* __restrict__ out_len)
{
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_packets) return;
    int start, n;
    ts_payload(ts + k * 188, start, n);
    out_len[k] = (uint32_t)n;
}

// one warp per packet: lanes copy the payload bytes to es_off[stream] + offset inside the stream
__global__ void ef_ts_copy_kernel(const uint8_t* __restrict__ ts, uint64_t n_packets, const uint32_t* __restrict__ local_off, const uint16_t* __restrict__ pkt_stream,
                                  const uint64_t* __restrict__ es_off, uint8_t* __restrict__ es)
{
    const uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (k >= n_packets) return;
    const uint8_t* d = ts + k * 188;
    int start, n;
    ts_payload(d, start, n);
    uint8_t* dst = es + es_off[pkt_stream[k]] + local_off[k];
    for (int i = lane; i < n; i += 32) dst[i] = d[start + i];
}

// exclusive scan of the payload lengths of ONE stream's packets per CTA (grid = n_streams)
__global__ void __launch_bounds__(256)
ef_ts_scan_kernel(const uint32_t* __restrict__ len, const uint64_t* __restrict__ ts_off, uint32_t* __restrict__ local_off, uint16_t* __restrict__ pkt_stream,
                  uint64_t* __restrict__ stream_total)
{
    __shared__ uint32_t warp_sum[8];
    __shared__ uint32_t carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, s = blockIdx.x;
    const uint64_t p0 = ts_off[s] / 188, p1 = ts_off[s + 1] / 188;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint64_t base = p0; base < p1; base += 256) {
        const uint64_t k = base + threadIdx.x;
        const uint32_t v = k < p1 ? len[k] : 0;
        uint32_t x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= d) x += y; }
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        uint32_t before = carry;
        for (int w = 0; w < warp; w++) before += warp_sum[w];
        if (k < p1) { local_off[k] = before + x - v; pkt_stream[k] = (uint16_t)s; }
        __syncthreads();
        if (threadIdx.x == 255) carry = before + x;
        __syncthreads();
    }
    if (threadIdx.x == 0) stream_total[s] = carry;
}

// ES offset of every stream = exclusive scan of the stream totals (n_streams <= 65,535: one CTA), zero padding behind the ES
__global__ void __launch_bounds__(1024)
ef_ts_offsets_kernel(const uint64_t* __restrict__ stream_total, int n_streams, uint64_t* __restrict__ es_off, uint8_t* __restrict__ es)
{
    __shared__ uint64_t warp_sum[32];
    __shared__ uint64_t carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n_streams; base += 1024) {
        const int k = base + threadIdx.x;
        const uint64_t v = k < n_streams ? stream_total[k] : 0;
        uint64_t x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint64_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= d) x += y; }
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint64_t t = warp_sum[lane], z = t;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint64_t y = __shfl_up_sync(0xFFFFFFFFu, z, d); if (lane >= d) z += y; }
            warp_sum[lane] = z - t;
        }
        __syncthreads();
        const uint64_t excl = carry + warp_sum[warp] + x - v;
        if (k < n_streams) es_off[k] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) es_off[n_streams] = carry;
    // K1's bit reader runs a few bytes past the last slice: zero the 256 bytes behind the elementary stream
    if (threadIdx.x < 256) es[carry + threadIdx.x] = 0;
}

// ---- presentation timestamps of the pictures of TS submits (ef_pts_enable) ------------------------------------------
// The reference latches _pts in demux() when a video PES start carries a valid PTS (player.cpp:399-419; parse_pts()'s prefix
// check, player.cpp:299-306) and hands it to the picture whose header is parsed next: picture() -> flush_picture() sets
// _last_pts = _pts (player.cpp:692-702) and pushes it with that picture one header later. demux() runs when the bit reader
// fetches the packet's first payload byte (more(), player.cpp:459-493), and FILL_BITS keeps 24 bits buffered (player.cpp:348-352),
// so when picture() runs after the 24-bit prefix and the 8-bit code (player.cpp:1360-1363) the reader has fetched the code byte
// and the 2 bytes after it. Hence: pts(picture) = PTS of the last valid video PES start whose first payload byte lies at ES
// offset <= code byte + 2, else the value carried from earlier submits (-1 if none; reset() does not clear _pts).

// PTS of a video (PID 0x100) packet that starts a PES with a non-empty payload and a PTS with the right prefix; -1 otherwise
__device__ __forceinline__ int64_t ts_video_pes_pts(const uint8_t* d)
{
    if (d[0] != 0x47 || !(d[1] & 0x40) || !(d[3] & 0x10)) return -1;
    if ((((d[1] << 8) | d[2]) & 0x1FFF) != 0x100) return -1;
    const int o = (d[3] & 0x20) ? 5 + d[4] : 4;
    if (o + 9 > 188 || o + 9 + d[o + 8] >= 188) return -1;        // no PES payload reaches the ES (as ts_payload())
    const int flags = (d[o + 6] << 8) | d[o + 7];
    if (!(flags & 0x0080) || o + 14 > 188) return -1;             // PES_PTS
    const uint8_t* q = d + o + 9;
    if ((q[0] & 0xF0) != ((flags >> 2) & 0x30)) return -1;        // parse_pts(): '0010' for PTS only, '0011' with DTS
    int64_t n = ((int64_t)(q[0] & 0x0E)) << 29;
    n += (int64_t)((((uint32_t)q[1] << 8) | q[2]) >> 1) << 15;
    return n + ((((uint32_t)q[3] << 8) | q[4]) >> 1);
}

// Packet pass, one CTA per stream, one thread per packet: the stream's video PES starts with a valid PTS, in packet order, as
// (stream-local ES offset of the first payload byte, pts) at list_*[first packet of the stream ...]; span[s] = (that index, count).
// local_off comes from ef_ts_scan_kernel. The lists belong to one ES buffer: the shared packet tables are overwritten by the next
// submit while the compute stream may still resolve this one.
__global__ void __launch_bounds__(256)
ef_pts_packet_kernel(const uint8_t* __restrict__ ts, const uint64_t* __restrict__ ts_off, const uint32_t* __restrict__ local_off,
                     uint32_t* __restrict__ list_off, int64_t* __restrict__ list_pts, uint2* __restrict__ span)
{
    __shared__ uint32_t warp_cnt[8];
    __shared__ uint32_t carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, s = blockIdx.x;
    const uint64_t p0 = ts_off[s] / 188, p1 = ts_off[s + 1] / 188;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint64_t base = p0; base < p1; base += 256) {
        const uint64_t k = base + threadIdx.x;
        const int64_t pts = k < p1 ? ts_video_pes_pts(ts + k * 188) : -1;
        const unsigned m = __ballot_sync(0xFFFFFFFFu, pts >= 0);
        if (lane == 0) warp_cnt[warp] = __popc(m);
        __syncthreads();
        uint32_t before = carry;
        for (int w = 0; w < warp; w++) before += warp_cnt[w];
        if (pts >= 0) {
            const uint64_t j = p0 + before + __popc(m & ((1u << lane) - 1u));
            list_off[j] = local_off[k];
            list_pts[j] = pts;
        }
        __syncthreads();
        if (threadIdx.x == 255) carry = before + __popc(m);
        __syncthreads();
    }
    if (threadIdx.x == 0) span[s] = make_uint2((uint32_t)p0, carry);
}

// Resolve pass after ef_fill_kernel, one warp per stream, lanes over pictures: upper-bound search for code byte + 2 in the
// stream's list, else the carried PTS. pic_pts[s][p] (-1 past the stream's pictures); carry[s] becomes the submit's last valid
// PTS and last[s] the PTS of its most recent picture (get_pts(), player.cpp:653-656). Indexing the same submit again rolls
// both as if the input followed itself.
__global__ void __launch_bounds__(128)
ef_pts_resolve_kernel(const EfDev* __restrict__ Dp, const uint2* __restrict__ span, const uint32_t* __restrict__ list_off,
                      const int64_t* __restrict__ list_pts, int64_t* __restrict__ carry, int64_t* __restrict__ last, int64_t* __restrict__ pic_pts)
{
    const EfDev& D = *Dp;
    const int lane = threadIdx.x & 31;
    const int s = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (s >= D.n_streams) return;
    const uint2 sp = span[s];
    const uint32_t* lo = list_off + sp.x;
    const int64_t* lp = list_pts + sp.x;
    const int64_t carried = carry[s];
    const uint32_t np = D.n_pics[s];
    const EfPic* pics = D.pics + (size_t)s * D.max_pictures;
    int64_t* out = pic_pts + (size_t)s * D.max_pictures;
    int64_t newest = last[s];
    for (uint32_t p0 = 0; p0 < (uint32_t)D.max_pictures; p0 += 32) {
        const uint32_t p = p0 + lane;
        int64_t v = -1;
        if (p < np) {
            const uint64_t latch = (uint64_t)pics[p].code_off + 2;
            uint32_t a = 0, b = sp.y;                                  // first entry with offset > latch
            while (a < b) {
                const uint32_t m = (a + b) >> 1;
                if (lo[m] <= latch) a = m + 1; else b = m;
            }
            v = a ? lp[a - 1] : carried;
        }
        if (p < (uint32_t)D.max_pictures) out[p] = v;
        const int64_t at_last = __shfl_sync(0xFFFFFFFFu, v, (np - 1) & 31);
        if (np && (np - 1) / 32 == p0 / 32) newest = at_last;
    }
    if (lane == 0) {
        carry[s] = sp.y ? lp[sp.y - 1] : carried;
        last[s] = newest;
    }
}
