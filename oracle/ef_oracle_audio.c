/* oracle/ef_oracle_audio.c — CPU restatement of the espflix audio path. TEST INFRASTRUCTURE ONLY (see ef_oracle.h).
 *
 * Follows, function by function (paths relative to the reference's checkout):
 *   efo_demux_audio_ts   MpegDecoder::more() / demux() for PID 0x101 / 0x102   src/player.cpp:381-432, 451-493
 *   efo_sbc_frame        get_samples() + bit_allocation() + IQUANT()          src/sbc_decoder.cpp:141-341
 *   efo_sbc_synth        synthesize8() with its 170-word ring and 16 offsets   src/sbc_decoder.cpp:70-139
 *   efo_sbc_decode       decode_audio() driving sbc_decoder()                  src/video.cpp:964-986, sbc_decoder.cpp:343-373
 *   efo_pdm              pdm_second_order()                                    espflix.ino:73-107
 * Parity status: PINNED against the unmodified reference (oracle/_ref/efref_audio) on the audio of the reference's
 * own splash.ts / vmedia.ts (tests/golden/audio_pins.json), on synthetic SBC streams (tests/test_audio.py) and on
 * directed frames across the whole header domain (tests/golden/sbc_pins.json, tests/test_sbc_domain.py).
 * Domain: mono, 8 subbands, 16 blocks, bit pool <= 128 (what the reference's ffmpeg line produces; write_pcm_16(mono,
 * 128,1) passes 128 samples whatever the header says, so other shapes read uninitialised stack there, and the bit
 * allocation never ends above 128); joint stereo is outside it, since the reference synthesises two channels' blocks
 * for such a frame; first audio payload >= 64 bytes
 * (decode_audio probes the frame size on the first 64 bytes of its ring). Constant tables: espflix_b200/csrc/ef_sbc_tables.h
 * (spec constants, checked against the reference's arrays by tests/test_tables.py). */
#include <stdlib.h>
#include <string.h>

#include "ef_oracle.h"
#include "../espflix_b200/csrc/ef_sbc_tables.h"

static int be16a(const uint8_t* p) { return (p[0] << 8) | p[1]; }

/* parse_pts (player.cpp:299): a malformed marker nibble reads as -1, which mutes the audio like a missing PTS */
static int64_t pes_pts_a(const uint8_t* d, int flags)
{
    flags = (flags >> 2) & 0x30;
    if ((d[0] & 0xF0) != flags) return -1;
    int64_t n = ((int64_t)(d[0] & 0x0E)) << 29;
    n += (int64_t)(be16a(d + 1) >> 1) << 15;
    return n + (be16a(d + 3) >> 1);
}

size_t efo_demux_audio_ts(const uint8_t* ts, size_t len, uint8_t* es, size_t cap)
{
    size_t out = 0;
    int64_t audio_pts = -1;                                    /* MpegDecoder::reset(), player.cpp:449 */
    for (size_t pos = 0; pos + 188 <= len; pos += 188) {
        const uint8_t* d = ts + pos;
        if (d[0] != 0x47) continue;                            /* "ts lost sync": more() drops the packet and goes on (player.cpp:476-479) */
        int pid = ((d[1] << 8) + d[2]) & 0x1fff;
        const uint8_t* data = d + 4;
        if (d[3] & 0x20) data = d + 5 + d[4];
        if (!(d[3] & 0x10)) continue;
        const uint8_t* end = d + 188;
        const uint8_t* payload = data;
        int64_t pts = -1;
        int pus = d[1] & 0x40;
        if (pus) {
            const uint8_t* p = data + 6;
            int flags = be16a(p);
            payload = p + 3 + p[2];
            if (flags & 0x0080) pts = pes_pts_a(p + 3, flags);
        }
        if (pid != 0x101 && pid != 0x102) continue;
        if (pus) audio_pts = pts;                              /* a PES without PTS mutes the stream until the next one with */
        if (audio_pts != -1 && payload < end) {
            size_t n = (size_t)(end - payload);
            if (out + n <= cap) memcpy(es + out, payload, n);
            out += n;
        }
    }
    return out;
}

/* ---- one SBC frame -> 16 x 8 subband samples (sbc_decoder.cpp:141-341). Returns the bytes the bit loader consumed
 * (what the reference uses as the frame size), or sbc_header's -1 / -2. */
#define EFO_SBC_MAX_BITPOOL 128                            /* EF_SBC_MAX_BITPOOL of espflix_b200/csrc/ef_common.cuh */

static void bit_allocation8(int frequency, int allocation, int bitpool, const uint8_t* sf, int* bits)
{
    int bitneed[8], max_bitneed = 0;
    for (int sb = 0; sb < 8; sb++) {
        int s = sf[sb];
        if (allocation) bitneed[sb] = s;                       /* SNR */
        else if (s == 0) bitneed[sb] = -5;                     /* loudness */
        else {
            int loudness = s - ef_sbc_offset8[frequency][sb];
            if (loudness > 0) loudness /= 2;
            bitneed[sb] = loudness;
        }
        if (bitneed[sb] > max_bitneed) max_bitneed = bitneed[sb];
    }
    int bitcount = 0, slicecount = 0, bitslice = max_bitneed + 1;
    do {
        bitslice--;
        bitcount += slicecount;
        slicecount = 0;
        for (int sb = 0; sb < 8; sb++) {
            if (bitneed[sb] > bitslice + 1 && bitneed[sb] < bitslice + 16) slicecount++;
            else if (bitneed[sb] == bitslice + 1) slicecount += 2;
        }
    } while (bitcount + slicecount < bitpool);
    if (bitcount + slicecount == bitpool) { bitcount += slicecount; bitslice--; }
    for (int sb = 0; sb < 8; sb++) {
        if (bitneed[sb] < bitslice + 2) bits[sb] = 0;
        else { bits[sb] = bitneed[sb] - bitslice; if (bits[sb] > 16) bits[sb] = 16; }
    }
    for (int sb = 0; bitcount < bitpool && sb < 8; sb++) {
        if (bits[sb] >= 2 && bits[sb] < 16) { bits[sb]++; bitcount++; }
        else if (bitneed[sb] == bitslice + 1 && bitpool > bitcount + 1) { bits[sb] = 2; bitcount += 2; }
    }
    for (int sb = 0; bitcount < bitpool && sb < 8; sb++)
        if (bits[sb] < 16) { bits[sb]++; bitcount++; }
}

/* header + scale factors + bit allocation: the sum of the 8 widths, or -1 for a frame the reference rejects (bad sync,
 * 4 subbands), -2 outside its domain (see the header comment): not mono / 16 blocks, joint stereo (the reference sets
 * two channels and the header's block count before it rejects such a frame, then synthesises both channels), or a bit
 * pool above EFO_SBC_MAX_BITPOOL, which bit_allocation8's slice loop never reaches (each subband adds 16 over the whole
 * descent: only the signed overflow of bitslice would end it) */
static int sbc_header(const uint8_t* data, size_t len, uint8_t sf[8], int bits[8])
{
    if (len < 4 || data[0] != 0x9C) return -1;
    const int frequency = (data[1] >> 6) & 3, blocks = 4 * (((data[1] >> 4) & 3) + 1), mode = (data[1] >> 2) & 3;
    const int allocation = (data[1] >> 1) & 1, subbands = (data[1] & 1) ? 8 : 4, bitpool = data[2];
    if (subbands == 4) return -1;
    if (mode != 0 || blocks != 16 || bitpool > EFO_SBC_MAX_BITPOOL) return -2;
    for (int sb = 0; sb < 8; sb += 2) { uint8_t a = 4 + (size_t)(sb >> 1) < len ? data[4 + (sb >> 1)] : 0; sf[sb] = a >> 4; sf[sb + 1] = a & 15; }
    bit_allocation8(frequency, allocation, bitpool, sf, bits);
    int total = 0;
    for (int sb = 0; sb < 8; sb++) total += bits[sb];
    return total;
}

int efo_sbc_bits(const uint8_t* data, size_t len, int bits[8])
{
    uint8_t sf[8];
    for (int sb = 0; sb < 8; sb++) bits[sb] = 0;
    return sbc_header(data, len, sf, bits);
}

int efo_sbc_frame(const uint8_t* data, size_t len, int32_t sb_sample[16][8])
{
    uint8_t sf[8];
    int bits[8];
    const int total = sbc_header(data, len, sf, bits);
    if (total < 0) return total;
    const uint8_t* p = data + 8;
    uint32_t acc = 0;
    int have = 0;
    for (int blk = 0; blk < 16; blk++)
        for (int sb = 0; sb < 8; sb++) {
            int32_t sample = 0;
            const int level = bits[sb];
            if (level) {
                while (have < level) { acc = (acc << 8) | (p < data + len ? *p : 0); p++; have += 8; }   /* bytes behind the stream read as 0 */
                have -= level;
                uint32_t raw = (acc >> have) & ((1u << level) - 1);
                /* IQUANT (sbc_decoder.cpp:262): ((2 raw + 1) << scale) / (2^level - 1), then minus 2^scale; 32-bit wrap as compiled */
                sample = (int32_t)((uint32_t)((raw << 1) | 1) << sf[sb]) / (int32_t)((1u << level) - 1);
                sample -= 1 << sf[sb];
            }
            sb_sample[blk][sb] = sample;
        }
    return (int)(p - data);
}

/* ---- synthesis filterbank state, exactly the reference's: one 170-word ring shared by 16 sliding windows */
typedef struct { int32_t v[170]; uint8_t offset[16]; } efo_sbc_state;

static void sbc_state_init(efo_sbc_state* s)
{
    memset(s, 0, sizeof(*s));
    for (int i = 0; i < 16; i++) s->offset[i] = (uint8_t)((i + 1) * 10);
}

static void efo_sbc_synth(efo_sbc_state* s, const int32_t* src, int16_t* dst)
{
    for (int i = 0; i < 16; i++) {                             /* matrixing into the ring (sbc_decoder.cpp:74-99) */
        if (!s->offset[i]) { for (int j = 0; j < 9; j++) s->v[j + 160] = s->v[j]; s->offset[i] = 160; }
        int k = --s->offset[i];
        uint32_t acc = 0;
        for (int j = 0; j < 8; j++) acc += (uint32_t)ef_sbc_matrix[i][j] * (uint32_t)src[j];
        s->v[k] = (int32_t)acc >> 15;
    }
    for (int i = 0; i < 8; i++) {                              /* windowing (sbc_decoder.cpp:102-138) */
        const int32_t* p0 = s->v + s->offset[i];
        const int32_t* p1 = s->v + s->offset[(i + 8) & 15] + 1;
        uint32_t acc = 0;
        for (int d = 0; d < 10; d += 2) {
            acc += (uint32_t)p0[d] * (uint32_t)ef_sbc_window[d][i];
            acc += (uint32_t)p1[d] * (uint32_t)ef_sbc_window[d + 1][i];
        }
        int32_t v = (int32_t)acc >> 15;
        if (v < -0x7FFF) v = -0x7FFF; else if (v > 0x7FFF) v = 0x7FFF;
        dst[i] = (int16_t)v;
    }
}

/* decode_audio() over everything push_audio() received (video.cpp:964-986), "instant audio thread": the first call
 * decodes the first 64 bytes once to learn the frame size (and leaves that frame in the filter memory), then whole
 * frames are decoded in order; a rejected frame re-synthesises the previous frame's subband samples. Frame 0 outside
 * the domain: -2, nothing decoded; a later frame outside it re-synthesises like a rejected frame. */
long efo_sbc_decode(const uint8_t* es, size_t len, int16_t* pcm, size_t cap_samples)
{
    if (!len) return 0;
    efo_sbc_state st;
    sbc_state_init(&st);
    int32_t sb[16][8];
    memset(sb, 0, sizeof(sb));
    int16_t scratch[8];
    int frame_size = efo_sbc_frame(es, len, sb);               /* the probe: sbc_decoder(&_sbc, _sbc_buf, 64, ...) reads what it needs from the ring */
    if (frame_size == -2) return -2;
    for (int blk = 0; blk < 16; blk++) efo_sbc_synth(&st, sb[blk], scratch);
    if (frame_size <= 0) return frame_size == 0 ? 0 : -1;      /* the reference stalls / misbehaves here: outside the domain */
    long n = 0;
    for (size_t r = 0; r + (size_t)frame_size <= len; r += (size_t)frame_size) {
        efo_sbc_frame(es + r, len - r, sb);                    /* a rejected or out-of-domain frame leaves sb[] as it was */
        for (int blk = 0; blk < 16; blk++) {
            int16_t out[8];
            efo_sbc_synth(&st, sb[blk], out);
            if ((size_t)n + 8 <= cap_samples) memcpy(pcm + n, out, sizeof(out));
            n += 8;
        }
    }
    return n;
}

/* pdm_second_order (espflix.ino:73-107) over a whole PCM stream, modulator state starting at zero: every PCM sample
 * becomes 2 x 16 one-bit samples; a1 = (int32)(0x7FFF * 1.18940), a2 = (int)(0x7FFF * 2.12340). */
void efo_pdm(const int16_t* pcm, size_t n, uint16_t* out)
{
    const int32_t a1 = (int32_t)(0x7FFF * 1.18940), a2 = (int32_t)(0x7FFF * 2.12340);
    int32_t i0 = 0, i1 = 0, i2 = 0, s = 0;
    uint32_t b = 0;
    for (size_t k = 0; k < 2 * n; k++) {
        if (!(k & 1)) s = pcm[k >> 1] * 2;                     /* "if (len & 1)" with len counting down from 2n */
        i0 = (i0 + s) >> 1;
        for (int j = 0; j < 16; j++) {
            b <<= 1;
            if (i2 >= 0) { i1 += i0 - a1 - (i2 >> 7); i2 += i1 - a2; b |= 1; }
            else { i1 += i0 + a1 - (i2 >> 7); i2 += i1 + a2; }
        }
        out[k] = (uint16_t)b;
    }
}
