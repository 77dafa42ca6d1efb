"""tests/ts_cases.py — small synthetic transport streams for the trick-mode index tests: PES starts with and
without a sequence header, PTS present / absent / malformed, adaptation fields, audio and PSI packets in
between, non-monotonic PTS (so the nearest-entry search has ties and far entries)."""
import os

import numpy as np

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FUZZ_SEEDS = range(40, 52)


def _pts_bytes(pts, prefix=0x20):
    return bytes([prefix | (((pts >> 30) & 7) << 1) | 1, (pts >> 22) & 0xFF, (((pts >> 15) & 0x7F) << 1) | 1, (pts >> 7) & 0xFF, ((pts & 0x7F) << 1) | 1])


def _packet(pid, pusi, payload, adapt=0, cc=0):
    hdr = bytearray([0x47, (0x40 if pusi else 0) | (pid >> 8), pid & 0xFF, (0x30 if adapt else 0x10) | (cc & 15)])
    body = bytearray()
    if adapt:
        body += bytes([adapt - 1]) + (bytes([0x00]) + b"\xff" * (adapt - 2) if adapt > 1 else b"")
    room = 188 - 4 - len(body)
    body += payload[:room]
    body += b"\xff" * (188 - 4 - len(body))
    return bytes(hdr + body)


def make_ts(seed, n_pes=120, monotonic=True, ref_domain=True):
    """ref_domain: keep every sequence-header PES on a well-formed PTS at least 90 ticks away from the previous
    sequence header's (the reference tool divides by (pts - previous) / 90 for a printed statistic and dies on 0)."""
    rng = np.random.default_rng(seed)
    out, pts, last_seq = [], 129003 + int(rng.integers(0, 5000)), None
    for k in range(n_pes):
        seq = k == 0 or rng.random() < 0.25
        es = (b"\x00\x00\x01\xb3" if seq else b"\x00\x00\x01\x00") + bytes(rng.integers(0, 256, 40, dtype=np.uint8))
        mode = rng.random()
        if ref_domain and seq:
            mode = 0.0
            if last_seq is not None and abs(pts - last_seq) < 90:
                pts = last_seq + 90 + int(rng.integers(0, 500))
            last_seq = pts
        if mode < 0.85:
            flags, hdr = 0x8080, _pts_bytes(pts)
        elif mode < 0.92:
            flags, hdr = 0x80C0, _pts_bytes(pts, 0x30) + _pts_bytes(max(pts - 3003, 0), 0x10)      # PTS + DTS
        elif mode < 0.96:
            flags, hdr = 0x8000, b""                                                              # no PTS: pts = 0
        else:
            flags, hdr = 0x8080, _pts_bytes(pts, 0x30)                                            # wrong prefix: pts = -1
        stuffing = bytes([0xFF] * int(rng.integers(0, 4)))
        pes = b"\x00\x00\x01\xe0\x00\x00" + bytes([flags >> 8, flags & 0xFF, len(hdr) + len(stuffing)]) + hdr + stuffing + es
        out.append(_packet(0x100, True, pes, adapt=int(rng.integers(0, 20)) if rng.random() < 0.3 else 0, cc=k))
        for _ in range(int(rng.integers(0, 6))):
            kind = rng.random()
            if kind < 0.6:
                out.append(_packet(0x100, False, bytes(rng.integers(0, 256, 184, dtype=np.uint8))))
            elif kind < 0.85:
                out.append(_packet(0x102, rng.random() < 0.5, b"\x00\x00\x01\xc0\x00\x10\x80\x80\x05" + _pts_bytes(pts) + b"\x9c" * 32))
            else:
                out.append(_packet(0x000, True, b"\x00\x00\xb0\x0d" + b"\x00" * 20))
        step = int(rng.integers(1500, 9000))
        pts = pts + step if monotonic or rng.random() < 0.88 else max(0, pts - int(rng.integers(0, 30000)))
    return b"".join(out)


def fuzzed_stream(seed):
    return make_ts(seed, n_pes=90, monotonic=seed % 3 != 0)


def fuzzed_image_files():
    return [make_ts(s, monotonic=s != 61) for s in (60, 61, 62)]


def files_of(key):
    """the files of a pinned video.idx image, keyed 'fixture:<names>' or 'fuzz:<seeds>:<monotonic>'"""
    kind, rest = key.split(":", 1)
    if kind == "fixture":
        return [open(os.path.join(G, n + ".ts"), "rb").read() for n in rest.split(",")]
    seeds, mono = rest.split(":")
    return [make_ts(int(s), monotonic=bool(int(mono))) for s in seeds.split(",")]
