"""tests/sbc_encode_cases.py — a title's audio encoded from PCM (ef_sbc_encode) and interleaved into its video.ts (ef_mux_audio),
restated in numpy. The device must equal this byte for byte.

The reference's make_video() (indexer/indexer.cpp:306-309) gives ffmpeg "-codec:a sbc -ar 48000 -b:a 192k -ac 1 -streamid 1:258
-pes_payload_size 512": mono SBC, 16 blocks, 8 subbands, on PID 0x102. Here the caller gives mono 16-bit PCM at the header's rate.

SBC (ef_sbc_encode). Parameters: frequency code 0..3 (16, 32, 44.1, 48 kHz), allocation 0 loudness / 1 SNR, bit pool 2..128.
  Frames:      a stream of n samples makes ceil(n / 128) frames; frame f covers samples 128 f .. 128 f + 127; samples outside
               0..n-1 read as zero.
  Analysis:    block b of frame f takes X[j] = x[128 f + 8 b + 7 - j], j = 0..79 (X[0] the newest; A2DP 12.5.1), in integers:
                 Y[i] = sum_{m<5} WINDOW[i + 16 m] * X[i + 16 m]           WINDOW: ef_sbc_analysis_window, C[.] in Q18
                 acc[k] = sum_{i<16} MATRIX[k][i] * Y[i]                   MATRIX: ef_sbc_analysis_matrix, Q15; int64 throughout
                 v[b][k] = clamp((acc[k] + 2^17) >> 18, -2^31, 2^31 - 1)    the subband sample in the decoder's units, Q16
               The decoder (sbc_decoder.cpp, ef_audio.cu) synthesises with twice the spec's gain, so the analysis carries 1/2:
               acc is Q33 of the spec's sample, and >> 18 leaves Q16 of half of it. tests/test_sbc_encode.py measures the
               round trip's gain on sines.
  Scale factor of subband k: the smallest s in 0..15 with |v[b][k]| < 2^(s + 16) for all 16 blocks, else 15.
  Bit allocation: sbc_cases.alloc(frequency, allocation, bitpool, scale factors), once per frame. Its total is always the bit
               pool here (tests/test_sbc_encode.py asserts it per frame), so every frame is 8 + 2 * bitpool bytes.
  Quantiser:   a subband of width L > 0: q = ((v + 2^(s + 16)) * (2^L - 1)) >> (s + 17), in 0 .. 2^L - 2. The decoder's IQUANT
               (sbc_decoder.cpp:257) gives back 2^s ((2q + 1) / (2^L - 1) - 1). At L = 16 and s = 15, q is clamped to 32767 so
               that (2q + 1) << 15 stays below 2^31: the reference's int wraps above that (sbc_cases.iquant_wraps).
  Frame:       9C, (frequency << 6) | 0x30 | (allocation << 1) | 1 (16 blocks, mono, 8 subbands), bit pool, CRC-8, the eight
               scale factors as nibbles (subband 0 high), then q of every (block, subband) in that order, MSB first, at its width.
               CRC-8: polynomial x^8 + x^4 + x^3 + x^2 + 1 (0x1D), initial value 0x0F, MSB first, over byte 1, byte 2 and bytes
               4..7 (ffmpeg checks it; the reference's decoder ignores it).

Mux (ef_mux_audio). Parameters: frames_per_pes F (0: floor(512 / frame bytes), ffmpeg's -pes_payload_size 512), pts0.
  PES k carries frames kF .. kF + F - 1 (the last may hold fewer): 00 00 01 BD, PES_packet_length = 8 + payload bytes, 80 80 05,
  the PTS a_k = pts0 + floor(k F 128 90000 / fs) with the 0x21 prefix; packetised as trick_cases.mux does on PID 0x102 (full
  184-byte payloads, the last packet stuffed by its adaptation field), one continuity counter per title from 0.
  Interleave: PES k goes immediately before the first packet of the first video PES start (PID 0x100 with
  payload_unit_start) in file order whose pts v_j >= a_k; after the last packet when there is none. Every input packet keeps its
  bytes and order. Rejected: an input with PID 0x101 or 0x102, a video PES start without a PTS, a last a_k >= 2^33."""
import os
import re

import numpy as np

from tests import sbc_cases as sc
from tests import trick_cases as tc

ROOT = tc.ROOT
FS_HZ = (16000, 32000, 44100, 48000)
DEFAULTS = dict(frequency=3, allocation=0, bitpool=28, frames_per_pes=0, pts0=0)
FRAC = 16                                     # fractional bits of the subband samples


def _table(name):
    src = open(os.path.join(ROOT, "espflix_b200", "csrc", "ef_sbc_analysis_tables.h")).read()
    body = re.search(name + r"\[[^=]*=\s*\{(.*?)\};", src, re.S).group(1)
    return np.array([int(v) for v in re.findall(r"-?\d+", body)], dtype=np.int64)


WINDOW = _table("ef_sbc_analysis_window")
MATRIX = _table("ef_sbc_analysis_matrix").reshape(8, 16)


def frame_bytes(bitpool):
    return 8 + 2 * bitpool


def n_frames(n_samples):
    return (n_samples + 127) // 128


def analysis(pcm):
    """int16 PCM -> the subband samples v[frame][block][subband] (int64, Q16 of the decoder's units)"""
    x = np.asarray(pcm, dtype=np.int64)
    nf = n_frames(x.size)
    if not nf:
        return np.zeros((0, 16, 8), dtype=np.int64)
    xp = np.concatenate([np.zeros(72, np.int64), x, np.zeros(nf * 128 - x.size, np.int64)])
    newest = 72 + 128 * np.arange(nf)[:, None] + 8 * np.arange(16)[None, :] + 7         # [f][b]
    X = xp[newest[:, :, None] - np.arange(80)[None, None, :]]                          # [f][b][80]
    Y = (X * WINDOW).reshape(nf, 16, 5, 16).sum(axis=2)                                # [f][b][16]
    acc = np.einsum("fbi,ki->fbk", Y, MATRIX)
    return np.clip((acc + (1 << 17)) >> 18, -(1 << 31), (1 << 31) - 1)


def scale_factors(v):
    """[frame][block][subband] -> [frame][subband] in 0..15"""
    m = np.abs(v).max(axis=1)
    s = np.zeros(m.shape, dtype=np.int64)
    for k in range(15):
        s += m >= (1 << (k + FRAC))
    return s


def quantise(v, s, bits):
    """v [16][8], s [8], bits [8] -> q [16][8] (0 where a width is 0)"""
    L = np.asarray(bits, dtype=np.int64)
    s = np.asarray(s, dtype=np.int64)
    q = ((v + (1 << (s + FRAC))) * ((1 << L) - 1)) >> (s + FRAC + 1)
    q = np.where((L == 16) & (s == 15), np.minimum(q, 32767), q)
    return np.where(L > 0, q, 0)


def crc8(data):
    c = 0x0F
    for b in data:
        for i in range(7, -1, -1):
            bit = ((b >> i) & 1) ^ (c >> 7)
            c = (c << 1) & 0xFF
            if bit:
                c ^= 0x1D
    return c


def header(frequency, allocation, bitpool):
    return bytes([0x9C, (frequency << 6) | 0x30 | (allocation << 1) | 1, bitpool])


def pack_frame(frequency, allocation, bitpool, sf, bits, q):
    h = header(frequency, allocation, bitpool)
    sfb = bytes([(int(sf[k]) << 4) | int(sf[k + 1]) for k in range(0, 8, 2)])
    w = np.tile(np.asarray(bits, dtype=np.int64), 16)
    vals = np.asarray(q, dtype=np.int64).reshape(-1)
    j = np.arange(16)
    sel = j[None, :] < w[:, None]
    b = (vals[:, None] >> np.clip(w[:, None] - 1 - j[None, :], 0, 15)) & 1
    payload = np.packbits(b[sel].astype(np.uint8)).tobytes()
    assert len(payload) == 2 * bitpool, (len(payload), bitpool)
    return h + bytes([crc8(h[1:3] + sfb)]) + sfb + payload


def encode(pcm, frequency=3, allocation=0, bitpool=28, info=None):
    """int16 PCM -> SBC bytes; `info` (a list) receives (scale factors, alloc(), q) per frame"""
    v = analysis(pcm)
    sfs = scale_factors(v)
    out = bytearray()
    for f in range(v.shape[0]):
        sf = [int(x) for x in sfs[f]]
        a = sc.alloc(frequency, allocation, bitpool, sf)
        q = quantise(v[f], sfs[f], a["bits"])
        if info is not None:
            info.append((sf, a, q))
        out += pack_frame(frequency, allocation, bitpool, sf, a["bits"], q)
    return bytes(out)


# ---- mux --------------------------------------------------------------------------------------------------------------------------
def frames_per_pes(bitpool, frames_per_pes=0):
    return frames_per_pes or 512 // frame_bytes(bitpool)


def audio_pts(k, frequency, fpp, pts0):
    return pts0 + (k * fpp * 128 * 90000) // FS_HZ[frequency]


def audio_pes(sbc, bitpool=28, frequency=3, frames_per_pes=0, pts0=0, **_):
    """[(pts, PES bytes)] of one title's SBC"""
    fb = frame_bytes(bitpool)
    fpp = globals()["frames_per_pes"](bitpool, frames_per_pes)
    out = []
    for k, o in enumerate(range(0, len(sbc), fpp * fb)):
        pay = bytes(sbc[o:o + fpp * fb])
        pts = audio_pts(k, frequency, fpp, pts0)
        n = 8 + len(pay)
        out.append((pts, bytes([0, 0, 1, 0xBD, n >> 8, n & 0xFF, 0x80, 0x80, 5]) + tc.pes_header(pts)[9:] + pay))
    return out


def packetise(pes_list, pid, cc=0):
    """trick_cases.mux's packetisation on any PID: -> (list of packets of each PES, next continuity counter)"""
    out = []
    for pes in pes_list:
        pk, pos = [], 0
        while pos < len(pes):
            left = len(pes) - pos
            b1 = (0x40 if pos == 0 else 0) | (pid >> 8)
            if left >= 184:
                pk.append(bytes([0x47, b1, pid & 0xFF, 0x10 | (cc & 15)]) + pes[pos:pos + 184])
                pos += 184
            else:
                af = 184 - left
                stuff = bytes([af - 1]) + (bytes([0]) + b"\xff" * (af - 2) if af > 1 else b"")
                pk.append(bytes([0x47, b1, pid & 0xFF, 0x30 | (cc & 15)]) + stuff + pes[pos:])
                pos = len(pes)
            cc += 1
        out.append(pk)
    return out, cc


def video_starts(ts):
    """[(packet index, pts)] of every video PES start; ValueError for audio PIDs or a start without a PTS"""
    ts = bytes(ts)
    if len(ts) % 188:
        raise ValueError("not whole packets")
    out = []
    for k in range(len(ts) // 188):
        d = ts[188 * k:188 * k + 188]
        pid = ((d[1] << 8) | d[2]) & 0x1FFF
        if pid in (0x101, 0x102):
            raise ValueError("packet %d is on audio PID 0x%x" % (k, pid))
        if pid != 0x100 or not d[1] & 0x40 or not d[3] & 0x10:          # more() demuxes only packets with a payload
            continue
        o = 5 + d[4] if d[3] & 0x20 else 4
        if o + 14 > 188 or d[o:o + 3] != b"\x00\x00\x01" or not d[o + 7] & 0x80 or (d[o + 9] & 0xF0) != ((d[o + 7] >> 2) & 0x30):
            raise ValueError("video PES start at packet %d without a PTS" % k)
        p = d[o + 9:o + 14]
        out.append((k, ((p[0] >> 1) & 7) << 30 | p[1] << 22 | (p[2] >> 1) << 15 | p[3] << 7 | p[4] >> 1))
    return out


def mux(ts, sbc, **params):
    """video.ts + SBC -> video.ts with audio; ValueError where ef_mux_audio returns EF_EINVAL"""
    p = dict(DEFAULTS, **params)
    ts = bytes(ts)
    starts = video_starts(ts)
    if len(sbc) % frame_bytes(p["bitpool"]):
        raise ValueError("SBC is not whole frames")
    pes = audio_pes(sbc, **p)
    if pes and pes[-1][0] >= 1 << 33:
        raise ValueError("audio pts beyond 2^33")
    pkts, _ = packetise([b for _, b in pes], 0x102)
    n = len(ts) // 188
    at = [[] for _ in range(n + 1)]                         # audio packets to go before input packet i (n: the end)
    j = 0                                                   # a_k rises, so the first start with v_j >= a_k never moves back
    for (a, _), pk in zip(pes, pkts):
        while j < len(starts) and starts[j][1] < a:
            j += 1
        at[starts[j][0] if j < len(starts) else n] += pk
    out = bytearray()
    for i in range(n + 1):
        out += b"".join(at[i])
        if i < n:
            out += ts[188 * i:188 * i + 188]
    return bytes(out)


# ---- cases -------------------------------------------------------------------------------------------------------------------------
BITPOOLS = (2, 7, 20, 28, 60, 97, 128)


def sine(n, freq, fs, amp, phase=0.0):
    t = np.arange(n)
    return np.round(amp * np.sin(2 * np.pi * freq / fs * t + phase)).astype(np.int16)


def centre(k, fs):
    """centre frequency of subband k"""
    return (k + 0.5) * fs / 16


def pcm_cases(fs=48000):
    """name -> int16 PCM of the directed signals"""
    rng = np.random.default_rng(20261017)
    c = {"silence": np.zeros(1280, np.int16), "one": np.array([12345], np.int16), "empty": np.zeros(0, np.int16)}
    for n in (127, 128, 129):
        c["len%d" % n] = rng.integers(-20000, 20000, n).astype(np.int16)
    for k in range(8):
        c["centre%d" % k] = sine(2048, centre(k, fs), fs, 12000)
    for k in range(9):
        c["edge%d" % k] = sine(2048, min(k * fs / 16, fs / 2 - 1), fs, 9000, 0.3)
    t = np.arange(4096)
    c["chirp"] = np.round(16000 * np.sin(2 * np.pi * (20 + (fs / 2 - 20) * t / (2 * t.size)) * t / fs)).astype(np.int16)
    c["noise"] = rng.normal(0, 6000, 3000).clip(-32768, 32767).astype(np.int16)
    c["square"] = np.where((np.arange(2560) // 37) % 2, 32767, -32768).astype(np.int16)
    clip = rng.integers(-32768, 32768, 2560).astype(np.int16)
    clip[300:900] = 32767
    clip[1200:1700] = -32768
    clip[2000:2200:2] = -32768
    clip[2001:2200:2] = 32767
    c["clipped"] = clip
    return c


def fixture_pcm(name, oracle):
    """the fixture's own audio, decoded by the oracle"""
    ts = tc.fixture(name)
    es = oracle.demux_audio_ts(np.frombuffer(ts, np.uint8))
    return np.asarray(oracle.sbc_decode(es), dtype=np.int16), bytes(es)


def sweep():
    """(frequency, allocation, bitpool) of the parameter sweep"""
    return [(f, a, b) for f in range(4) for a in (0, 1) for b in BITPOOLS]


def sweep_pcm(frequency, seed=7):
    """the sweep's signal: a sine per subband centre over noise, 10 frames"""
    fs = FS_HZ[frequency]
    rng = np.random.default_rng(seed + frequency)
    x = rng.normal(0, 1500, 1280)
    for k in range(8):
        x += sine(1280, centre(k, fs), fs, 2500 / (k + 1), k)
    return x.clip(-32768, 32767).astype(np.int16)
