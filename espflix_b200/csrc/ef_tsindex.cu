// espflix_b200/csrc/ef_tsindex.cu — trick-mode index of transport streams (SURVEY.md §8f-4).
//
// Replaces make_index() / pts2pos() / pts2seq() of the reference's offline tool (indexer/indexer.cpp:90-228)
// for a batch of transport-stream files resident in HBM:
//   ef_tsidx_packet_kernel   one thread per 188-byte packet: PID, payload-unit-start, PES header -> pts and
//                            "payload starts with a sequence header" (parse()/parse_pts(), indexer.cpp:43-75)
//   ef_tsidx_compact_kernel  one CTA per file: ordered compaction of the sequence-header packets into the
//                            (pts, packet number) table, first / last pts (block-wide exclusive scan of the flags)
//   ef_tsidx_sample_kernel   one thread per 1/12 s bin: nearest table entry in pts with the reference's exact
//                            tie-breaking and its int-cast distance (pts2pos(), indexer.cpp:193-207)
// All integer; the table and the samples are bit-identical to the reference's vectors.
#include "ef_common.cuh"

namespace {

__device__ __forceinline__ uint32_t tb(const uint8_t* ts, uint64_t len, uint64_t i) { return i < len ? ts[i] : 0u; }
__device__ __forceinline__ uint32_t tb16(const uint8_t* ts, uint64_t len, uint64_t i) { return (tb(ts, len, i) << 8) | tb(ts, len, i + 1); }

}  // namespace

// kind: 0 nothing, 1 video PES start, 2 video PES start whose payload begins with a sequence header
__global__ void ef_tsidx_packet_kernel(const uint8_t* __restrict__ ts, const uint64_t* __restrict__ pkt_off, int n_files, uint64_t n_packets,
                                       int64_t* __restrict__ pkt_pts, uint8_t* __restrict__ pkt_kind)
{
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_packets) return;
    const uint64_t i = k * 188;
    const uint32_t b1 = ts[i + 1], b2 = ts[i + 2], b3 = ts[i + 3];
    const uint32_t pid = ((b1 << 8) + b2) & 0x1fff;
    uint8_t kind = 0;
    int64_t pts = 0;
    if ((b3 & 0x10) && (b1 & 0x40) && pid == 0x100) {                    // payload present, PES starts here, video PID
        // a PES header cut short by the packet is read on into the following packets of the SAME file (as the
        // reference's buffer would give), zeros behind the end of the file: find the file of this packet
        int lo = 0, hi = n_files;
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pkt_off[mid] <= k) lo = mid; else hi = mid; }
        const uint64_t total_bytes = pkt_off[lo + 1] * 188;
        uint64_t d = i + 4;
        if (b3 & 0x20) d = i + 5 + ts[i + 4];                             // skip the adaptation field
        d += 6;                                                           // parse(), indexer.cpp:53
        const int flags = (int)tb16(ts, total_bytes, d);
        const uint64_t payload = d + 3 + tb(ts, total_bytes, d + 2);
        d += 3;
        if (flags & 0x0080) {                                             // parse_pts(), indexer.cpp:43
            const int want = (flags >> 2) & 0x30;
            const uint32_t p0 = tb(ts, total_bytes, d);
            if ((int)(p0 & 0xF0) != want) pts = -1;
            else pts = ((int64_t)(p0 & 0x0E) << 29) + (int64_t)((tb16(ts, total_bytes, d + 1) >> 1) << 15) + (int64_t)(tb16(ts, total_bytes, d + 3) >> 1);
        }
        kind = tb(ts, total_bytes, payload + 3) == 0xB3 ? 2 : 1;
    }
    pkt_pts[k] = pts;
    pkt_kind[k] = kind;
}

// info per file: [0] first_pts, [1] last_pts, [2] number of table entries
__global__ void __launch_bounds__(256)
ef_tsidx_compact_kernel(const uint64_t* __restrict__ pkt_off /* [n_files + 1], in packets */, const int64_t* __restrict__ pkt_pts,
                        const uint8_t* __restrict__ pkt_kind, int64_t* __restrict__ seq_pts, uint32_t* __restrict__ seq_pos,
                        int64_t* __restrict__ info)
{
    __shared__ EfBlockScan<uint32_t, 256> scan;
    __shared__ unsigned long long last_video;                             // 1 + packet index of the last video PES start
    const int f = blockIdx.x;
    const uint64_t p0 = pkt_off[f], p1 = pkt_off[f + 1];
    if (threadIdx.x == 0) last_video = 0;
    scan.init();
    unsigned long long my_last = 0;
    for (uint64_t c = p0; c < p1; c += 256) {
        const uint64_t k = c + threadIdx.x;
        const uint32_t kind = k < p1 ? pkt_kind[k] : 0u;
        if (kind) my_last = k - p0 + 1;
        const uint32_t j = scan.exclusive(kind == 2);
        if (kind == 2) {
            seq_pts[p0 + j] = pkt_pts[k];                                 // the table of a file lives at its packet offset (n_seq <= n_packets)
            seq_pos[p0 + j] = (uint32_t)(k - p0);
        }
    }
    atomicMax(&last_video, my_last);
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t n = scan.carry;
        int64_t origin = -1;                                              // "if (origin == -1) origin = pts" (indexer.cpp:136): the first
        for (uint32_t j = 0; j < n && origin == -1; j++) origin = seq_pts[p0 + j];   // entry whose pts is not -1 (a malformed PTS reads as -1)
        info[f * 3 + 0] = origin;
        info[f * 3 + 1] = last_video ? pkt_pts[p0 + last_video - 1] : -1; // video_pts
        info[f * 3 + 2] = (int64_t)n;
    }
}

__global__ void ef_tsidx_sample_kernel(const int64_t* __restrict__ seq_pts, const uint32_t* __restrict__ seq_pos, int n,
                                       int64_t first_pts, uint32_t bin_size, uint32_t n_samples, uint32_t* __restrict__ samples)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_samples) return;
    const int64_t want = (int64_t)b * bin_size + first_pts;
    int mini = 0, mine = 0x7FFFFFF;                                       // pts2pos(), indexer.cpp:196-197
    for (int i = 0; i < n; i++) {
        int64_t diff = seq_pts[i] - want;
        if (diff < 0) diff = -diff;
        const int e = (int)diff;                                          // the reference keeps the distance in an int
        if (e < mine) { mine = e; mini = i; }
    }
    samples[b] = seq_pos[mini];
}
