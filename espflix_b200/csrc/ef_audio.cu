// espflix_b200/csrc/ef_audio.cu — the audio half of a transport-stream program (SURVEY.md §8f-3), batched over streams.
//
// Replaces, for every stream at once (paths relative to the reference's checkout):
//   MpegDecoder::demux() for PID 0x101 / 0x102 -> push_audio()      src/player.cpp:381-432, src/video.cpp:1007
//   decode_audio() -> sbc_decoder(): get_samples(), bit_allocation(), IQUANT(), synthesize8()
//                                                                    src/video.cpp:964-986, src/sbc_decoder.cpp:70-373
//   write_pcm_16() -> pdm_second_order()                             espflix.ino:73-136
// The reference decodes one 128-sample frame at a time through a 170-word ring shared by 16 sliding windows. The
// ring is only a delay line: V_t[i] = (sum_j matrix[i][j] * S_t[j]) >> 15 for block t, and
//   pcm_t[i] = clip((sum_{d=0..9} window[d][i] * V_{t-d}[d even ? i : (i + 8) & 15]) >> 15),
// so every frame - and every block - is independent once the V rows are in HBM:
//   ef_sbc_probe_kernel   one thread per stream: the frame size decode_audio() learns from the first 64 bytes
//   ef_sbc_matrix_kernel  one warp per frame: header, scale factors, bit allocation (12.6.3), 128 samples cut out of
//                         the bit field at computed offsets (no serial bit reader), IQUANT, matrixing -> V[16][16]
//   ef_sbc_window_kernel  one thread per PCM sample: 10 taps over the V rows of this and the nine blocks before
//   ef_pdm_kernel         one thread per stream: the second-order delta-sigma modulator is a serial non-linear
//                         recurrence (32 one-bit samples per PCM sample); streams run side by side
//   ef_audio_ts_*         TS -> audio bytes on the device (one thread per packet; the "PES without PTS mutes the
//                         stream" gate of demux() is walked per stream, from the gate the previous submit left)
// A call decodes every stream's held-back bytes followed by its new bytes and leaves in EfAudioState
// (ef_common.cuh) what the next call needs: frame size, the bytes of the first frame not yet decodable, the last
// accepted frame's subband samples, the last 9 V rows and the modulator state. The whole-stream ef_audio_decode is
// the same kernels with a zeroed state and every stream ended (DESIGN.md §4).
// Quirks kept: decode_audio() decodes the first frame twice (once to learn the frame size, video.cpp:971), so the
// filter memory already holds it when the real decode starts; a frame it rejects (bad sync byte, joint stereo,
// 4 subbands) re-synthesises the previous frame's samples; 32-bit wrap-around of the accumulators. Domain: mono,
// 8 subbands, 16 blocks (write_pcm_16(mono,128,1) passes 128 samples whatever the header says); a frame size that
// does not divide the reference's 4 KB ring makes it read past the ring on the straddling frame (undefined there;
// here the stream is simply linear).
#include "ef_common.cuh"
#include "ef_sbc_tables.h"

namespace {

__constant__ int c_matrix[16][8];
__constant__ int c_window[10][8];
__constant__ signed char c_offset8[4][8];

// header + scale factors + bit allocation of one frame (get_samples / bit_allocation, sbc_decoder.cpp:141-305).
// Returns the sum of bits over the 8 subbands, or -1 for a frame the reference rejects, -2 outside its domain.
__device__ int sbc_frame_bits(const uint8_t* d, uint64_t avail, int* bits, int* sf)
{
    if (avail < 4 || d[0] != 0x9C) return -1;
    const uint32_t b1 = d[1];
    const int frequency = (b1 >> 6) & 3, blocks = 4 * (((b1 >> 4) & 3) + 1), mode = (b1 >> 2) & 3;
    const int allocation = (b1 >> 1) & 1, subbands = (b1 & 1) ? 8 : 4, bitpool = avail > 2 ? d[2] : 0;
    if (mode == 3 || subbands == 4) return -1;
    if (mode != 0 || blocks != 16) return -2;
    int bitneed[8], max_bitneed = 0;
#pragma unroll
    for (int sb = 0; sb < 8; sb++) {
        const uint32_t byte = 4 + (sb >> 1) < (int)avail ? d[4 + (sb >> 1)] : 0u;
        const int s = (sb & 1) ? (byte & 15) : (byte >> 4);
        sf[sb] = s;
        int need;
        if (allocation) need = s;
        else if (s == 0) need = -5;
        else { need = s - c_offset8[frequency][sb]; if (need > 0) need /= 2; }
        bitneed[sb] = need;
        max_bitneed = max(max_bitneed, need);
    }
    int bitcount = 0, slicecount = 0, bitslice = max_bitneed + 1;
    do {
        bitslice--;
        bitcount += slicecount;
        slicecount = 0;
#pragma unroll
        for (int sb = 0; sb < 8; sb++) {
            if (bitneed[sb] > bitslice + 1 && bitneed[sb] < bitslice + 16) slicecount++;
            else if (bitneed[sb] == bitslice + 1) slicecount += 2;
        }
    } while (bitcount + slicecount < bitpool);
    if (bitcount + slicecount == bitpool) { bitcount += slicecount; bitslice--; }
    int total = 0;
#pragma unroll
    for (int sb = 0; sb < 8; sb++) bits[sb] = bitneed[sb] < bitslice + 2 ? 0 : min(bitneed[sb] - bitslice, 16);
#pragma unroll
    for (int sb = 0; sb < 8; sb++) {
        if (bitcount < bitpool) {
            if (bits[sb] >= 2 && bits[sb] < 16) { bits[sb]++; bitcount++; }
            else if (bitneed[sb] == bitslice + 1 && bitpool > bitcount + 1) { bits[sb] = 2; bitcount += 2; }
        }
    }
#pragma unroll
    for (int sb = 0; sb < 8; sb++) {
        if (bitcount < bitpool && bits[sb] < 16) { bits[sb]++; bitcount++; }
        total += bits[sb];
    }
    return total;
}

}  // namespace

cudaError_t ef_audio_upload_constants()
{
    cudaError_t e = cudaMemcpyToSymbol(c_matrix, ef_sbc_matrix, sizeof(ef_sbc_matrix));
    if (e != cudaSuccess) return e;
    e = cudaMemcpyToSymbol(c_window, ef_sbc_window, sizeof(ef_sbc_window));
    if (e != cudaSuccess) return e;
    return cudaMemcpyToSymbol(c_offset8, ef_sbc_offset8, sizeof(ef_sbc_offset8));
}

// ---- one decode call over a blob: every stream's held-back bytes followed by its new bytes, off[n_streams + 1] --------
// plan[s]: .x frame size after this call (0: not learned yet, -1 first frame rejected, -2 outside the domain), .y 1 when
// the probe decode of frame 0 runs in this call, .z frames decoded in this call.

// blob length of every stream: held-back bytes + the new bytes of this call (new_off == nullptr: none). A stream ended
// while a demuxed submit was already queued behind the current one drops that submit's bytes before its first PES start
// (skip[s], lead[s]): they passed the demux gate only because it was still open.
__global__ void ef_audio_len_kernel(const EfAudioState* __restrict__ st, const uint64_t* __restrict__ new_off, const uint32_t* __restrict__ lead,
                                    const uint8_t* __restrict__ skip, int n_streams, uint64_t* __restrict__ len)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams) return;
    uint64_t n = 0;
    if (new_off) n = new_off[s + 1] - new_off[s] - (skip[s] ? lead[s] : 0u);
    len[s] = (uint64_t)st[s].carry_len + n;
}

// one CTA per stream: held-back bytes, then the new bytes, to blob + blob_off[s]
__global__ void ef_audio_assemble_kernel(const EfAudioState* __restrict__ st, const uint8_t* __restrict__ src, const uint64_t* __restrict__ new_off,
                                         const uint32_t* __restrict__ lead, const uint8_t* __restrict__ skip, const uint64_t* __restrict__ blob_off, uint8_t* __restrict__ blob)
{
    const int s = blockIdx.x;
    const int carry = st[s].carry_len;
    uint8_t* dst = blob + blob_off[s];
    for (int i = threadIdx.x; i < carry; i += blockDim.x) dst[i] = st[s].carry[i];
    if (!new_off) return;
    const uint64_t a = new_off[s] + (skip[s] ? lead[s] : 0u), n = blob_off[s + 1] - blob_off[s] - (uint64_t)carry;
    for (uint64_t i = threadIdx.x; i < n; i += blockDim.x) dst[carry + i] = src[a + i];
}

// one thread per stream: the frame size decode_audio() learns from the first 64 bytes (video.cpp:971). It runs once the
// stream holds the header and scale factors (8 bytes) and, for an accepted frame, all 8 + 2 * total bytes the probe
// decode of frame 0 reads; at the end of the stream on whatever is there.
__global__ void ef_sbc_probe_kernel(const uint8_t* __restrict__ es, const uint64_t* __restrict__ off, const EfAudioState* __restrict__ st,
                                    const uint8_t* __restrict__ ended, int n_streams, int4* __restrict__ plan)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams) return;
    const uint64_t len = off[s + 1] - off[s];
    int fs = st[s].frame_size, probe = 0;
    if (fs == 0 && len && (ended[s] || len >= 8)) {
        int bits[8], sf[8];
        const int total = sbc_frame_bits(es + off[s], len < 64 ? len : 64, bits, sf);   // decode_audio() hands sbc_decoder 64 bytes
        const int f = total < 0 ? total : 8 + 2 * total;  // the lazy byte loader has consumed header + scale factors + 16 * total bits
        if (f < 0 || ended[s] || len >= (uint64_t)f) { fs = f; probe = f > 0; }
    }
    plan[s] = make_int4(fs, probe, 0, 0);
}

// one warp per stream: frames decodable in this call. Before the end of the stream a frame is decoded only when every
// byte its bit loader reads is present: its own frame_size bytes and, for an accepted frame, its 8 + 2 * total bytes
// (more than frame_size when its scale factors differ from frame 0's). The first frame that fails holds back itself and
// everything after it. At the end of the stream every whole frame is decoded and missing bytes read as 0.
__global__ void ef_sbc_count_kernel(const uint8_t* __restrict__ es, const uint64_t* __restrict__ off, const uint8_t* __restrict__ ended,
                                    int n_streams, int4* __restrict__ plan)
{
    const int s = (int)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (s >= n_streams) return;                            // whole warps leave together
    const int fs = plan[s].x;
    const uint64_t len = off[s + 1] - off[s];
    uint64_t n = fs > 0 ? len / (uint64_t)fs : 0;
    if (n && !ended[s]) {
        const uint8_t* d = es + off[s];
        for (uint64_t base = 0; base < n; base += 32) {
            const uint64_t f = base + lane;
            bool bad = false;
            if (f < n) {
                int bits[8], sf[8];
                const uint64_t a = f * (uint64_t)fs;
                const int total = sbc_frame_bits(d + a, len - a, bits, sf);
                bad = total >= 0 && a + 8 + 2 * (uint64_t)total > len;
            }
            const unsigned m = __ballot_sync(0xFFFFFFFFu, bad);
            if (m) { n = base + (uint64_t)(__ffs(m) - 1); break; }
        }
    }
    if (lane == 0) plan[s].z = (int)n;
}

// One warp per frame slot. Slots of stream s (slot_base[s] ..): 0 = the V rows of its last 9 blocks before this call
// (rows 7..15), then, when plan[s].y, the probe decode of frame 0 (video.cpp:971), then frame f of this call at slot
// f + 1 + plan[s].y. V rows go to vrows[(16 slot + blk) * 16 + i]. The last slot of a stream also leaves its subband
// samples in sb_last[s] for the next call.
__global__ void __launch_bounds__(128)
ef_sbc_matrix_kernel(const uint8_t* __restrict__ es, const uint64_t* __restrict__ off, const int4* __restrict__ plan, const EfAudioState* __restrict__ st,
                     const uint64_t* __restrict__ slot_base /* [n_streams + 1] */, int n_streams, int32_t* __restrict__ vrows, int32_t* __restrict__ sb_last)
{
    __shared__ int32_t sb_s[4][16][8];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint64_t slot = (uint64_t)blockIdx.x * 4 + w;
    const uint64_t total_slots = slot_base[n_streams];
    int s = 0;
    bool history = false;
    if (slot < total_slots) {                              // (no early return: the warp reaches __syncwarp below either way)
        int lo = 0, hi = n_streams;                        // stream of this slot
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (slot_base[mid] <= slot) lo = mid; else hi = mid; }
        s = lo;
        const uint64_t ls = slot - slot_base[s];
        history = ls == 0;
        if (!history) {
            const int4 p = plan[s];
            const int fs = p.x;
            const uint64_t base = off[s], len = off[s + 1] - off[s];
            const bool probe = p.y && ls == 1;
            const long f = probe ? 0 : (long)ls - 1 - p.y;
            // a rejected frame re-synthesises the samples of the last accepted one (sb_sample[] is simply left as it was);
            // when that one was decoded by an earlier call, its samples come from the stream's state
            int bits[8], sf[8], total = -1;
            const uint8_t* d = nullptr;
            uint64_t avail = 0;
            for (long g = f; g >= 0 && total < 0; g--) {
                d = es + base + (uint64_t)g * (uint64_t)fs;
                avail = len - (uint64_t)g * (uint64_t)fs;  // the bit loader may run on into the next frame; bytes behind the stream read as 0
                total = sbc_frame_bits(d, avail, bits, sf);
                if (probe) break;
            }
            // lane -> block lane/2, subbands 4 (lane & 1) .. + 3
            const int blk = lane >> 1, sb0 = (lane & 1) * 4;
            if (total < 0 && !probe) {
#pragma unroll
                for (int k = 0; k < 4; k++) sb_s[w][blk][sb0 + k] = st[s].sb[blk][sb0 + k];
            } else {
                int pre = 0;
#pragma unroll
                for (int sb = 0; sb < 8; sb++) if (sb < sb0) pre += bits[sb];
                uint32_t bitpos = (uint32_t)(blk * max(total, 0) + pre);
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int sb = sb0 + k, level = total < 0 ? 0 : bits[sb];
                    int32_t sample = 0;
                    if (level) {
                        const uint64_t byte = 8 + (bitpos >> 3);
                        uint32_t win = 0;                  // 24 bits starting at that byte cover <= 7 + 16 bits
#pragma unroll
                        for (int q = 0; q < 3; q++) win = (win << 8) | (byte + q < avail ? d[byte + q] : 0u);
                        const uint32_t raw = (win >> (24 - (bitpos & 7) - level)) & ((1u << level) - 1);
                        sample = (int32_t)((uint32_t)((raw << 1) | 1) << sf[sb]) / (int32_t)((1u << level) - 1);   // IQUANT, sbc_decoder.cpp:262
                        sample -= 1 << sf[sb];
                        bitpos += (uint32_t)level;
                    }
                    sb_s[w][blk][sb] = sample;
                }
            }
        }
    }
    __syncwarp();
    if (slot < total_slots) {
        if (history) {
            int32_t* out = vrows + slot * 256;
            for (int i = lane; i < 256; i += 32) out[i] = i >= 7 * 16 ? st[s].vhist[(i >> 4) - 7][i & 15] : 0;
        } else {
            // matrixing: lane -> block lane/2, outputs 8 (lane & 1) .. + 7
            const int blk = lane >> 1, i0 = (lane & 1) * 8;
            int32_t src[8];
#pragma unroll
            for (int j = 0; j < 8; j++) src[j] = sb_s[w][blk][j];
            int32_t* out = vrows + (slot * 16 + blk) * 16 + i0;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                uint32_t acc = 0;
#pragma unroll
                for (int j = 0; j < 8; j++) acc += (uint32_t)c_matrix[i0 + i][j] * (uint32_t)src[j];
                out[i] = (int32_t)acc >> 15;
            }
            if (slot + 1 == slot_base[s + 1]) {
#pragma unroll
                for (int k = 0; k < 4; k++) sb_last[(size_t)s * 128 + blk * 8 + (lane & 1) * 4 + k] = sb_s[w][blk][(lane & 1) * 4 + k];
            }
        }
    }
}

// one thread per PCM sample. The first output row of a stream follows its history slot (and the probe decode); the
// 10 taps reach back at most 9 rows, into the history slot at worst.
__global__ void ef_sbc_window_kernel(const int32_t* __restrict__ vrows, const uint64_t* __restrict__ slot_base, const uint64_t* __restrict__ pcm_off,
                                     int n_streams, int16_t* __restrict__ pcm)
{
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= pcm_off[n_streams]) return;
    int lo = 0, hi = n_streams;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pcm_off[mid] <= k) lo = mid; else hi = mid; }
    const int s = lo;
    const uint64_t local = k - pcm_off[s];
    const int i = (int)(local & 7);
    const uint64_t frames = (pcm_off[s + 1] - pcm_off[s]) >> 7;
    const uint64_t t = 16 * (slot_base[s + 1] - slot_base[s] - frames) + (local >> 3);   // block index inside the stream's rows
    const int32_t* rows = vrows + slot_base[s] * 16 * 16;
    uint32_t acc = 0;
#pragma unroll
    for (int d = 0; d < 10; d++) acc += (uint32_t)rows[(t - d) * 16 + ((d & 1) ? ((i + 8) & 15) : i)] * (uint32_t)c_window[d][i];
    int32_t v = (int32_t)acc >> 15;
    v = max(-0x7FFF, min(0x7FFF, v));
    pcm[k] = (int16_t)v;
}

// pdm_second_order (espflix.ino:73-107) over this call's PCM of a stream, the modulator continuing from the stream's
// state (all 16 bits of every output word are new, so only i0, i1, i2 carry over)
__global__ void ef_pdm_kernel(const int16_t* __restrict__ pcm, const uint64_t* __restrict__ pcm_off, int n_streams, EfAudioState* __restrict__ st,
                              uint16_t* __restrict__ pdm)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams) return;
    const int32_t a1 = (int32_t)(0x7FFF * 1.18940), a2 = (int32_t)(0x7FFF * 2.12340);
    int32_t i0 = st[s].i0, i1 = st[s].i1, i2 = st[s].i2;
    uint32_t b = 0;
    const uint64_t p0 = pcm_off[s], p1 = pcm_off[s + 1];
    for (uint64_t k = p0; k < p1; k++) {
        const int32_t smp = (int32_t)pcm[k] * 2;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            i0 = (i0 + smp) >> 1;                          // low pass
#pragma unroll 4
            for (int j = 0; j < 16; j++) {
                b <<= 1;
                if (i2 >= 0) { i1 += i0 - a1 - (i2 >> 7); i2 += i1 - a2; b |= 1; }
                else { i1 += i0 + a1 - (i2 >> 7); i2 += i1 + a2; }
            }
            pdm[2 * k + h] = (uint16_t)b;
        }
    }
    st[s].i0 = i0; st[s].i1 = i1; st[s].i2 = i2;
}

// one warp per stream, after the call's kernels: hold back the bytes of the first frame not decoded (all bytes while
// the frame size is unknown, none once the first frame was rejected), keep the last accepted frame's subband samples
// and the last 9 V rows. An ended stream starts over from zero (MpegDecoder::reset(), player.cpp:439).
__global__ void ef_audio_commit_kernel(EfAudioState* __restrict__ st, const uint8_t* __restrict__ blob, const uint64_t* __restrict__ blob_off,
                                       const int4* __restrict__ plan, const uint64_t* __restrict__ slot_base, const int32_t* __restrict__ vrows,
                                       const int32_t* __restrict__ sb_last, const uint8_t* __restrict__ ended, int n_streams)
{
    const int s = (int)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (s >= n_streams) return;
    EfAudioState& a = st[s];
    if (ended[s]) {
        int32_t* w = (int32_t*)&a;
        for (int i = lane; i < (int)(sizeof(EfAudioState) / 4); i += 32) w[i] = 0;
        return;
    }
    const int4 p = plan[s];
    const uint64_t len = blob_off[s + 1] - blob_off[s];
    const uint64_t used = p.x > 0 ? (uint64_t)p.z * (uint64_t)p.x : p.x < 0 ? len : 0;
    const int keep = (int)(len - used);                    // < EF_AUDIO_CARRY (ef_sbc_count_kernel, ef_sbc_probe_kernel)
    for (int i = lane; i < keep; i += 32) a.carry[i] = blob[blob_off[s] + used + i];
    if (p.z) {
        for (int i = lane; i < 128; i += 32) a.sb[i >> 3][i & 7] = sb_last[(size_t)s * 128 + i];
        const int32_t* rows = vrows + (slot_base[s + 1] * 16 - 9) * 16;
        for (int i = lane; i < 9 * 16; i += 32) a.vhist[i >> 4][i & 15] = rows[i];
    }
    if (lane == 0) { a.frame_size = p.x; a.carry_len = keep; }
}

// ---- TS -> audio bytes --------------------------------------------------------------------------------------
// per packet: payload start (0 = none) and length of PID 0x101 / 0x102, and for PES starts whether the PTS parses
__global__ void ef_audio_ts_packet_kernel(const uint8_t* __restrict__ ts, uint64_t n_packets, uint8_t* __restrict__ start, uint8_t* __restrict__ kind)
{
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_packets) return;
    const uint8_t* d = ts + k * 188;
    uint8_t st = 0, kd = 0;                                // kind: 0 continuation, 1 PES start with PTS, 2 PES start without
    const int pid = ((d[1] << 8) | d[2]) & 0x1FFF;
    if (d[0] == 0x47 && (pid == 0x101 || pid == 0x102) && (d[3] & 0x10)) {
        int o = 4;
        if (d[3] & 0x20) o = 5 + d[4];
        if (d[1] & 0x40) {
            kd = 2;
            if (o + 9 <= 188) {
                const int flags = (d[o + 6] << 8) | d[o + 7];
                const int p = o + 9;
                if ((flags & 0x80) && p < 188 && (d[p] & 0xF0) == ((flags >> 2) & 0x30)) kd = 1;   // parse_pts(), player.cpp:299
                o = o + 9 + d[o + 8];
            } else o = 188;
        }
        if (o < 188) st = (uint8_t)o;
    }
    start[k] = st;
    kind[k] = kd;                                          // a packet without the sync byte is skipped (more(), player.cpp:476-479)
}

// One thread per file walks its packets in order (a few thousand): byte offsets of the payloads that reach push_audio().
// ts_off: byte offsets of the files (multiples of 188). The demux gate (_audio_pts != -1) of a file starts as gate_in
// and ends as gate_out: 0 shut, 1 opened by a PES with PTS, 2 still open from before this walk (no PES started in it).
// lead[f] = bytes that passed before the first PES start; skip[f] is cleared (ef_audio_end_kernel sets it).
__global__ void ef_audio_ts_scan_kernel(const uint64_t* __restrict__ ts_off, int n_files, const uint8_t* __restrict__ start, const uint8_t* __restrict__ kind,
                                        const uint8_t* __restrict__ gate_in, uint8_t* __restrict__ gate_out, uint32_t* __restrict__ lead, uint8_t* __restrict__ skip,
                                        uint32_t* __restrict__ out_pos /* per packet, 0xFFFFFFFF = dropped */, uint64_t* __restrict__ es_len)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_files) return;
    uint32_t gate = gate_in[f] ? 2 : 0;
    uint64_t out = 0, first = ~0ull;
    for (uint64_t k = ts_off[f] / 188; k < ts_off[f + 1] / 188; k++) {
        const uint32_t kd = kind[k];
        if (kd) { if (first == ~0ull) first = out; gate = kd == 1 ? 1 : 0; }
        const uint32_t st = start[k];
        if (gate && st) { out_pos[k] = (uint32_t)out; out += 188 - st; }
        else out_pos[k] = 0xFFFFFFFFu;
    }
    es_len[f] = out;
    gate_out[f] = (uint8_t)gate;
    lead[f] = (uint32_t)(first == ~0ull ? out : first);
    skip[f] = 0;
}

__global__ void ef_audio_ts_copy_kernel(const uint8_t* __restrict__ ts, const uint64_t* __restrict__ ts_off, int n_files, uint64_t n_packets,
                                        const uint8_t* __restrict__ start, const uint32_t* __restrict__ out_pos, const uint64_t* __restrict__ es_off, uint8_t* __restrict__ es)
{
    const uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (k >= n_packets || out_pos[k] == 0xFFFFFFFFu) return;
    int lo = 0, hi = n_files;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (ts_off[mid] / 188 <= k) lo = mid; else hi = mid; }
    const uint8_t* d = ts + k * 188;
    const int st = start[k];
    uint8_t* dst = es + es_off[lo] + out_pos[k];
    for (int i = st + lane; i < 188; i += 32) dst[i - st] = d[i];
}

// ef_decode_audio ended these streams: their demux gate shuts (MpegDecoder::reset()). A TS submit already demuxed
// behind the current one saw the gate open: its bytes before its first PES start are dropped (skip) and a gate it only
// inherited shuts. An ES submit queued there copied the gate: it shuts too.
__global__ void ef_audio_end_kernel(const uint8_t* __restrict__ ended, int n_streams, uint8_t* __restrict__ gate_cur, uint8_t* __restrict__ gate_next,
                                    uint8_t* __restrict__ skip_next, int next_is_ts)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams || !ended[s]) return;
    gate_cur[s] = 0;
    if (!gate_next) return;
    if (!next_is_ts) gate_next[s] = 0;
    else { if (gate_next[s] == 2) gate_next[s] = 0; skip_next[s] = 1; }
}

