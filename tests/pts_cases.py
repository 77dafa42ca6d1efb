"""tests/pts_cases.py — the presentation-timestamp rule restated in Python, and the transport streams it is pinned on.

The rule (include/espflix_b200.h, ef_picture_pts): a picture gets the PTS of the last video PES start with a valid PTS whose
first payload byte lies at ES offset <= (offset of the picture start code's 0x00 code byte) + 2, over the whole stream; -1 if
there is none. It follows the reference decoder: demux() latches _pts only from a PTS with the right prefix nibble
(player.cpp:299-306, 399-419), more() demuxes a packet when the bit reader fetches its first payload byte (player.cpp:459-493),
FILL_BITS keeps 24 bits buffered (player.cpp:348-352), and picture() runs after the 24-bit prefix and the code byte
(player.cpp:1360-1363) and hands _pts on through flush_picture() (player.cpp:692-702).

cases() builds the programs the pins cover (tests/golden/pts_pins.json, written by tools/make_pts_golden.py from the
unmodified reference): synthetic ES from espflix_b200.synth and the fixtures' own ES, re-wrapped with PES boundaries a few
bytes around the picture start codes, PES without PTS, with a malformed prefix and with PTS + DTS, adaptation fields, audio
and PSI packets in between, decreasing PTS, PES starts in mid-slice and on every packet, and one program outside the
reference's domain (its first PES has no PTS, so the reference pushes nothing until a PTS arrives)."""
import bisect
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FIXTURES = ("splash", "vmedia")


# -- the restatement --------------------------------------------------------------------------------------------------
def parse_pts(d, flags):
    """parse_pts() (player.cpp:299-306): -1 unless the prefix nibble is '0010' (PTS only) or '0011' (PTS + DTS)"""
    if (d[0] & 0xF0) != ((flags >> 2) & 0x30):
        return -1
    n = (d[0] & 0x0E) << 29
    n += (((d[1] << 8) | d[2]) >> 1) << 15
    return n + (((d[3] << 8) | d[4]) >> 1)


def demux(ts):
    """more() / demux() for PID 0x100 (player.cpp:381-493) -> (video ES bytes, [(ES offset of the first payload byte, pts or
    -1)] of every video PES start). Raises ValueError outside the reference's domain (lost sync, an empty video payload)."""
    ts = bytes(ts)
    es, pes = bytearray(), []
    for k in range(0, len(ts) - 187, 188):
        d = ts[k:k + 188]
        if d[0] != 0x47:
            raise ValueError("packet %d: lost sync" % (k // 188))
        pid = ((d[1] << 8) | d[2]) & 0x1FFF
        if pid != 0x100 or not d[3] & 0x10:
            continue
        o = 5 + d[4] if d[3] & 0x20 else 4
        if d[1] & 0x40:
            flags = (d[o + 6] << 8) | d[o + 7]
            pts = parse_pts(d[o + 9:o + 14], flags) if flags & 0x80 else -1
            o += 9 + d[o + 8]
            pes.append((len(es), pts))
        if o >= 188:
            raise ValueError("packet %d: video packet without payload bytes" % (k // 188))
        es += d[o:]
    return bytes(es), pes


def picture_codes(es):
    """ES offset of the code byte of every picture start code, up to a sequence end code (K0's byte-aligned scan)"""
    out, i = [], 0
    while True:
        i = es.find(b"\x00\x00\x01", i)
        if i < 0 or i + 4 > len(es) or es[i + 3] == 0xB7:
            return out
        if es[i + 3] == 0x00:
            out.append(i + 3)
        i += 1


def picture_pts(ts):
    """pts of every picture of a whole program, by the rule"""
    es, pes = demux(ts)
    valid = [(o, p) for o, p in pes if p >= 0]
    offs = [o for o, _ in valid]
    out = []
    for x in picture_codes(es):
        j = bisect.bisect_right(offs, x + 2)
        out.append(valid[j - 1][1] if j else -1)
    return out


def in_domain(ts):
    """the reference pushes every picture only when the first one latches a valid PTS (else quirk Q10)"""
    p = picture_pts(ts)
    return bool(p) and p[0] >= 0


# -- building programs --------------------------------------------------------------------------------------------------
def pts_bytes(pts, prefix):
    return bytes([prefix | (((pts >> 30) & 7) << 1) | 1, (pts >> 22) & 0xFF, (((pts >> 15) & 0x7F) << 1) | 1, (pts >> 7) & 0xFF,
                  ((pts & 0x7F) << 1) | 1])


def pes_header(kind, pts, stuffing=0):
    """kind: 'pts', 'none' (no PTS), 'bad' (PTS with the DTS-form prefix: reads -1), 'dts' (PTS + DTS), 'bad_dts' (PTS + DTS
    flags with the PTS-only prefix: reads -1)"""
    flags, body = {
        "pts": (0x8080, lambda: pts_bytes(pts, 0x20)),
        "none": (0x8000, lambda: b""),
        "bad": (0x8080, lambda: pts_bytes(pts, 0x30)),
        "dts": (0x80C0, lambda: pts_bytes(pts, 0x30) + pts_bytes(max(pts - 3003, 0), 0x10)),
        "bad_dts": (0x80C0, lambda: pts_bytes(pts, 0x20) + pts_bytes(max(pts - 3003, 0), 0x10)),
    }[kind]
    h = body() + b"\xff" * stuffing
    return b"\x00\x00\x01\xe0\x00\x00" + bytes([flags >> 8, flags & 0xFF, len(h)]) + h


def _packet(pid, pusi, payload, af=None, cc=0):
    """one 188-byte packet carrying exactly `payload`; the room left over goes into the adaptation field (af = its minimum
    total size, None: only when needed), never into the payload"""
    room = 184 - len(payload)
    assert room >= 0 and (af is None or af <= room)
    need = room if room or af else 0
    hdr = bytes([0x47, (0x40 if pusi else 0) | (pid >> 8), pid & 0xFF, (0x30 if need else 0x10) | (cc & 15)])
    a = b""
    if need:
        a = bytes([need - 1]) + (b"\x00" + b"\xff" * (need - 2) if need > 1 else b"")
    return hdr + a + payload


def _other_packet(rng, pts):
    if rng.random() < 0.6:            # audio PES on PID 0x102 (demuxed and dropped by the video path)
        p = b"\x00\x00\x01\xc0\x00\x10\x80\x80\x05" + pts_bytes(pts, 0x20) + b"\x9c" * 40
        return _packet(0x102, rng.random() < 0.5, p)
    return _packet(0x000, True, b"\x00\x00\xb0\x0d" + b"\x00" * 20)


def wrap(es, starts, kinds, pts, seed, adapt=0.0, others=0.0):
    """video ES -> TS with a video PES starting at every ES offset in `starts` (sorted, starts[0] == 0), PES i with header
    kind kinds[i] and PTS pts[i]; a random adaptation field on a fraction `adapt` of the video packets and an audio or PSI
    packet after a fraction `others` of them"""
    es = bytes(es)
    rng = np.random.default_rng(seed)
    assert starts[0] == 0 and all(a < b for a, b in zip(starts, starts[1:])) and starts[-1] < len(es)
    edges = list(starts) + [len(es)]
    out, cc = [], 0
    for i in range(len(starts)):
        data = es[edges[i]:edges[i + 1]]
        hdr = pes_header(kinds[i], int(pts[i]), int(rng.integers(0, 4)))
        pos, first = 0, True
        while pos < len(data):
            room = 184 - (len(hdr) if first else 0)
            af = int(rng.integers(1, 24)) if rng.random() < adapt else None
            m = min(len(data) - pos, room - (af or 0))
            out.append(_packet(0x100, first, (hdr if first else b"") + data[pos:pos + m], af, cc))
            cc += 1
            pos += m
            first = False
            if rng.random() < others:
                out.append(_other_packet(rng, int(pts[i])))
    return b"".join(out)


def fixture_es(name):
    return demux(open(os.path.join(GOLDEN, name + ".ts"), "rb").read())[0]


def _synth_es(seed, n_pictures, gop):
    from espflix_b200 import synth
    return bytes(synth.generate(synth.SEED0 + seed, n_pictures=n_pictures, gop=gop)[0])


def _shifted(es, shift, kind_of, pts_of, seed, **kw):
    """a PES boundary at every picture's code byte + shift(k); the first PES starts at 0"""
    starts = sorted({0} | {x + shift(k) for k, x in enumerate(picture_codes(es)) if 0 < x + shift(k) < len(es)})
    n = len(starts)
    return wrap(es, starts, [kind_of(i) for i in range(n)], [pts_of(i) for i in range(n)], seed, **kw)


def _rising(base, step=3003):
    return lambda i: base + i * step


def cases():
    """[(name, ts bytes)] in a fixed order; every program but 'ood_first_without_pts' is inside the reference's domain"""
    out = []
    # the fixtures' ES: boundary at code byte + (k mod 9) - 4, every 7th PES without PTS
    for j, name in enumerate(FIXTURES):
        es = fixture_es(name)
        out.append(("%s_shift" % name, _shifted(es, lambda k: k % 9 - 4, lambda i: "none" if i % 7 == 6 else "pts", _rising(900000 + j),
                                                 seed=10 + j)))
    # the fixtures' ES with every header kind, adaptation fields and other PIDs in between
    kinds = ["pts", "dts", "bad", "pts", "none", "bad_dts", "pts", "dts"]
    for j, name in enumerate(FIXTURES):
        es = fixture_es(name)
        out.append(("%s_kinds" % name, _shifted(es, lambda k: (3 * k + 1) % 9 - 4, lambda i: "pts" if i == 0 else kinds[i % 8],
                                                 _rising((1 << 32) + 12345 * j, 1501), seed=20 + j, adapt=0.3, others=0.2)))
    # synthetic programs of different lengths, each shift -4..+4 and each header kind
    for j, (n, gop) in enumerate([(5, 5), (9, 3), (12, 12), (14, 7), (20, 10)]):
        es = _synth_es(j, n, gop)
        out.append(("synth%d_shift" % n, _shifted(es, lambda k, j=j: (k + j) % 9 - 4, lambda i: "pts" if i == 0 else kinds[(i + j) % 8],
                                                   _rising(5000 * j + 1), seed=30 + j, adapt=0.25, others=0.15)))
    # decreasing and jumping PTS
    es = _synth_es(7, 16, 8)
    rng = np.random.default_rng(41)
    vals = [int(v) for v in rng.integers(0, 1 << 33, size=64)]
    out.append(("synth_decreasing", _shifted(es, lambda k: -(k % 5), lambda i: "pts" if i % 4 else ("pts" if i == 0 else "bad"),
                                             lambda i: (1 << 33) - 1 - 4000 * i if i < 8 else vals[i], seed=42)))
    # PES starts in mid-slice: 3 boundaries per picture at random offsets
    es = _synth_es(8, 12, 6)
    rng = np.random.default_rng(43)
    starts = sorted({0} | {int(x) for x in rng.integers(1, len(es), size=36)})
    out.append(("synth_midslice", wrap(es, starts, ["pts" if i == 0 or i % 6 else "none" for i in range(len(starts))],
                                       [777777 + 1001 * i for i in range(len(starts))], seed=44, adapt=0.2, others=0.1)))
    # a PES start on every packet (120 to 149 ES bytes each)
    es = _synth_es(9, 6, 3)
    rng = np.random.default_rng(45)
    starts, p = [0], 0
    while True:
        p += int(rng.integers(120, 150))
        if p >= len(es):
            break
        starts.append(p)
    out.append(("synth_every_packet", wrap(es, starts, [["pts", "pts", "dts", "none", "bad"][i % 5] if i else "pts" for i in range(len(starts))],
                                           [3 * i + 17 for i in range(len(starts))], seed=46)))
    # outside the domain: the first PES has no PTS (pictures before the first PTS read -1)
    es = _synth_es(10, 10, 5)
    out.append(("ood_first_without_pts", _shifted(es, lambda k: 2 if k < 4 else -3, lambda i: "none" if i < 3 else "pts", _rising(60000),
                                                  seed=47)))
    return out


def cut_points(ts):
    """indices of the packets a TS may be cut before so that every submit holds whole pictures: video packets whose payload
    starts exactly at a sequence, GOP or picture start code"""
    ts = bytes(ts)
    es, _ = demux(ts)
    cuts, off = [], 0
    for k in range(0, len(ts) - 187, 188):
        d = ts[k:k + 188]
        if ((d[1] << 8 | d[2]) & 0x1FFF) != 0x100 or not d[3] & 0x10:
            continue
        o = 5 + d[4] if d[3] & 0x20 else 4
        if d[1] & 0x40:
            o += 9 + d[o + 8]
        if off and es[off:off + 3] == b"\x00\x00\x01" and es[off + 3:off + 4] in (b"\x00", b"\xb3", b"\xb8"):
            cuts.append(k // 188)
        off += 188 - o
    return cuts
