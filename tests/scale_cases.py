"""tests/scale_cases.py — the benchmark-sized batch of transport streams the batch-scale tests run on.

4,096 streams (bench.STREAMS_PER_GPU) of 12 pictures each, from D = 67 distinct streams built with the benchmark's generator
parameters. Stream k carries distinct stream k % 67, packetised in variant k % 5, so the batch has period 335: coprime to
1,024, the tile width of ef_ts_offsets_kernel's scan, so stream k and stream k + 1,024 never share their bytes, and TS lengths
and ES offsets differ from stream to stream. Replicas of one distinct stream (k = d + 67 j) differ in their PES cut positions,
PES header kinds and stuffing, adaptation fields, and the places of the interleaved audio and PSI packets, but carry the same
video ES, the same PTS for every picture, the same audio ES, the same presentation modes and the same frame-counter parity:
their decoded pictures, PTS, audio and composite fields must be equal, so every stream can be checked against its original."""
import bisect
import functools
import math

import numpy as np

from tests import audio_cases, pts_cases

N = 4096                            # bench.STREAMS_PER_GPU
D = 67                              # distinct streams (prime)
V = 5                               # packetisation variants
PERIOD = D * V
PICTURES = 12
SEED_INDEX = 9000                   # synth seeds SEED0 + SEED_INDEX + d


def pts_of(d):
    """pts of the 12 pictures of distinct stream d: its own base and one of five step patterns"""
    base = 400000 + 12347 * d
    kind = d % 5
    j = 1 + d % 11                                   # where the late frame or the jump happens
    if kind == 2:                                    # irregular steps
        steps = [1501, 3003, 4505, 3003]
        return [base + sum(steps[m % 4] for m in range(i)) for i in range(PICTURES)]
    p = [base + 3003 * i for i in range(PICTURES)]
    if kind == 1:                                    # one frame four frames late: more than two fields late, re-latch
        p[j] -= 4 * 3003
    elif kind == 3:                                  # a forward jump of ten frames
        p = [v + (30030 if i >= j else 0) for i, v in enumerate(p)]
    elif kind == 4:                                  # a backward jump of three seconds
        p = [v - (270000 if i >= j else 0) for i, v in enumerate(p)]
    return p


def frame_counter0(d):
    """first field of distinct stream d's display; d = 0 starts at frame counter 0 (no origin latched at the first push).
    The others start at 1,000 or later: push_video's unsigned arithmetic puts a picture whose pts lies before the origin's
    by more than the origin's frame counter 2^32 fields ahead, so a backward jump must stay within it."""
    return 0 if d == 0 else 1000 + (d * 7919) % 1000


def modes_of(d):
    """push_video mode of each of the 12 pictures: one mode-1, -2 or -3 push for three streams in four"""
    m = [0] * PICTURES
    if d % 4:
        m[(d * 5) % PICTURES] = d % 4
    return m


def idle_fields(d):
    return 1 + d % 3


def extra_pictures(d):
    """pictures of the short ES submit that follows the batch in the composite test: the latest frame store then differs
    from stream to stream"""
    return d % 3


def audio_params(d):
    return {"n_frames": 100 + (d * 37) % 61, "bitpool": [12, 19, 28, 35, 53][d % 5], "allocation": (d >> 1) & 1,
            "frequency": d % 4, "consistent": d % 3 != 0}


def audio_pid(d):
    return 0x101 if d & 1 else 0x102


def _psi_packet(v, j):
    return pts_cases._packet(0x000, True, b"\x00\x00\xb0\x0d" + bytes([v, j & 0xFF]) + b"\x00" * 18)


def _mux(d, v, es, codes, pts, audio_ts):
    """distinct stream d in packetisation variant v: a video PES per picture starting 4 bytes before to 2 bytes after its
    picture start code's code byte (every third exactly at the start code, so that the TS can be cut there), PES 0 at ES
    offset 0; audio packets and PSI packets between the video packets at seeded places"""
    shift = [-4, -2, -1, 0, 1, 2]
    starts = [0] + [codes[i] + (-3 if (i + v) % 3 == 0 else shift[(5 * v + i) % 6]) for i in range(1, PICTURES)]
    kinds = ["dts" if (i + v) % 4 == 3 else "pts" for i in range(PICTURES)]
    video = pts_cases.wrap(es, starts, kinds, pts, seed=1000 * d + v, adapt=0.05 + 0.1 * v, others=0.0)
    vp = [video[i:i + 188] for i in range(0, len(video), 188)]
    ap = [bytes(audio_ts[i:i + 188]) for i in range(0, len(audio_ts), 188)]
    rng = np.random.default_rng(5000 + 100 * d + v)
    after = np.sort(rng.integers(0, len(vp), size=len(ap)))           # audio packet j goes after video packet after[j]
    psi = set(rng.choice(len(vp), size=3 + v, replace=False).tolist())
    out, j = [], 0
    for i, p in enumerate(vp):
        out.append(p)
        while j < len(ap) and after[j] == i:
            out.append(ap[j])
            j += 1
        if i in psi:
            out.append(_psi_packet(v, i))
    return b"".join(out)


def _cuts(ts, codes):
    """[(packet index, pictures before it)] of the packets the TS can be cut before so that both parts hold whole pictures"""
    out = []
    for c in pts_cases.cut_points(ts):
        es = pts_cases.demux(ts[:188 * c])[0]
        out.append((c, bisect.bisect_left(codes, len(es))))
    return out


class Batch:
    """the batch; stream k is distinct stream k % D in variant k % V"""

    def __init__(self):
        from espflix_b200 import synth
        gen = synth.generate_many(D, first_index=SEED_INDEX, n_pictures=PICTURES, gop=PICTURES, slices=12)
        self.es = [bytes(e) for e, _ in gen]
        self.codes = [pts_cases.picture_codes(e) for e in self.es]
        assert all(len(c) == PICTURES for c in self.codes)
        self.pts = [pts_of(d) for d in range(D)]
        self.audio = [audio_cases.sbc_stream(8000 + d, **audio_params(d)) for d in range(D)]
        aud_ts = [audio_cases.mux_audio_ts(self.audio[d], pid=audio_pid(d), pes_bytes=[333, 1024, 700][d % 3], first_pts=self.pts[d][0])
                  for d in range(D)]
        self.var = {}
        self.var_cuts = {}
        for d in range(D):
            for v in range(V):
                t = _mux(d, v, self.es[d], self.codes[d], self.pts[d], aud_ts[d])
                self.var[d, v] = t
                self.var_cuts[d, v] = _cuts(t, self.codes[d])
        self.n = N

    @staticmethod
    def distinct(k):
        return k % D

    def ts(self, k):
        return self.var[k % D, k % V]

    def cuts(self, k):
        return self.var_cuts[k % D, k % V]

    def cut(self, k, salt=0):
        """one picture-boundary cut of stream k, chosen with k: (packet index, pictures before it)"""
        c = self.cuts(k)
        return c[(k // PERIOD + 3 * salt) % len(c)]

    def fc0(self, k):
        return frame_counter0(k % D)

    def modes(self, k):
        return modes_of(k % D)

    def all_ts(self):
        return [self.ts(k) for k in range(self.n)]


def period_is_coprime_to_tiles():
    return math.gcd(PERIOD, 1024) == 1


@functools.lru_cache(maxsize=1)
def batch():
    return Batch()
