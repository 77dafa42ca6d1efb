"""tests/carry_cases.py — the hold-back rule of TS submits cut at any packet boundary (ef_carry_enable), restated in Python.

A stream's part of a submit is the bytes it held after the previous submit followed by the submit's new video ES. An access
unit (an optional sequence header, an optional GOP header, a picture header and its slices) is complete once all four bytes of
a later sequence (B3), GOP (B8), picture (00) or sequence-end (B7) start code are present. The complete units are decoded; from
the first byte of the first incomplete unit on, everything is held (with no unit open, the last 3 bytes, which may begin a start
code; after a sequence-end code, nothing). At the end of a stream the last unit counts as complete.

Presentation timestamps follow the rule of tests/pts_cases.py over the whole ES. Per submit, the PES starts of the new packets
sit behind the held bytes; a picture whose latch (code byte + 2) lies inside the held bytes takes the pts resolved for it by the
submit before (over everything received then), and every other picture without a PES start at or before its latch takes the
last valid PTS received so far. That is what ef_pts_resolve_kernel carries: no PES entry travels with the held bytes."""
import bisect

import numpy as np

from tests import pts_cases, scan_cases

UNIT_CODES = (0x00, 0xB3, 0xB8, 0xB7)


def scan(region, end=False):
    """K0 with carry over one stream's region -> (code byte offsets of the complete pictures, held bytes, code byte offset of
    the held picture or None)"""
    pics, c_pic, open_, unit, unit_code, stop = [], 0, 0, 0, None, False
    for i, code in scan_cases.start_codes(region):
        if code in UNIT_CODES:
            if open_ == 2 or code == 0xB7:
                c_pic = len(pics)
            if code == 0xB7:
                stop = True
                break
            if open_ != 1:
                unit = i
            if code == 0x00:
                open_, unit_code = 2, i + 3
            else:
                open_ = 1
        if code == 0x00:
            pics.append(i + 3)
    if stop or end:
        return pics, 0, None
    if open_:
        return pics[:c_pic], len(region) - unit, unit_code if open_ == 2 else None
    return pics, min(len(region), 3), None


class Stream:
    """one stream of a carrying context: feed() one submit's TS bytes at a time"""

    def __init__(self):
        self.held = b""
        self.base = 0                 # whole-stream ES offset of the held bytes
        self.carried = -1             # the last valid PTS received so far (_pts)
        self.hold_pts = -1            # pts of the held picture, resolved over the bytes received so far
        self.codes, self.pts, self.counts, self.held_sizes = [], [], [], []

    def feed(self, ts, end=False):
        es, pes = pts_cases.demux(ts)
        hin = len(self.held)
        region = self.held + es
        entries = [(o + hin, p) for o, p in pes if p >= 0]
        offs = [o for o, _ in entries]

        def resolve(latch):
            j = bisect.bisect_right(offs, latch)
            return entries[j - 1][1] if j else (self.hold_pts if latch < hin else self.carried)

        pics, hold, hcode = scan(region, end)
        self.codes += [self.base + x for x in pics]
        self.pts += [resolve(x + 2) for x in pics]
        if hcode is not None:
            self.hold_pts = resolve(hcode + 2)
        if entries:
            self.carried = entries[-1][1]
        self.base += len(region) - hold
        self.held = region[len(region) - hold:]
        self.counts.append(len(pics))
        self.held_sizes.append(hold)
        return pics, hold


def packets(ts):
    ts = bytes(ts)
    return [ts[i:i + 188] for i in range(0, len(ts), 188)]


def cut(ts, cuts):
    """TS bytes -> the submits cut before the packets in `cuts` (sorted, repeats give empty submits)"""
    pk = packets(ts)
    edges = [0] + list(cuts) + [len(pk)]
    return [b"".join(pk[a:b]) for a, b in zip(edges[:-1], edges[1:])]


def seeded_cuts(ts, seed, max_packets=40):
    """cut points of submits of 0..max_packets packets each"""
    n = len(ts) // 188
    r = np.random.RandomState(seed)
    cuts, p = [], 0
    while True:
        p += int(r.randint(0, max_packets + 1))
        if p >= n:
            return cuts
        cuts.append(p)


def run(ts, cuts):
    """feed a whole program cut before `cuts`, ending it with the last submit -> Stream"""
    st = Stream()
    chunks = cut(ts, cuts)
    for k, c in enumerate(chunks):
        st.feed(c, end=k == len(chunks) - 1)
    return st


def es_cut_offsets(ts, cuts):
    """whole-stream ES offset at which every cut falls, and the ES offsets of every video PES start"""
    es, pes = pts_cases.demux(ts)
    pk = packets(ts)
    offs, o = [], 0
    cut_set = set(cuts)
    for k, d in enumerate(pk):
        if k in cut_set:
            offs.append(o)
        o += len(pts_cases.demux(d)[0])
    return offs, [x for x, _ in pes]


def matrices_program(seed=3):
    """a synthetic program with custom quantiser matrices in every sequence header, a PES start every 40 to 90 ES bytes
    (so cuts land inside the 128 matrix bytes)"""
    from espflix_b200 import synth
    es = bytes(synth.generate(synth.SEED0 + 500 + seed, n_pictures=8, gop=2, flags=synth.MATRICES)[0])
    r = np.random.default_rng(seed)
    starts, p = [0], 0
    while True:
        p += int(r.integers(40, 90))
        if p >= len(es):
            break
        starts.append(p)
    return pts_cases.wrap(es, starts, ["pts"] * len(starts), [90000 + 3003 * i for i in range(len(starts))], seed=600 + seed)


def headers_tail_program():
    """a synthetic program followed by a lone sequence header (a headers-only unit the end of the stream drops)"""
    from espflix_b200 import synth
    es = bytes(synth.generate(synth.SEED0 + 700, n_pictures=5, gop=5)[0])
    seq = es[es.find(b"\x00\x00\x01\xb3"):]
    seq = seq[:seq.find(b"\x00\x00\x01", 4)]
    es = es + seq
    codes = pts_cases.picture_codes(es)
    starts = sorted({0} | {x - 1 for x in codes[1:]} | {len(es) - len(seq)})
    return pts_cases.wrap(es, starts, ["pts"] * len(starts), [45000 + 3003 * i for i in range(len(starts))], seed=701)


def programs():
    """[(name, ts)]: every program of pts_cases.cases(), both fixtures, custom matrices and a headers-only tail"""
    out = list(pts_cases.cases())
    for name in pts_cases.FIXTURES:
        with open("%s/%s.ts" % (pts_cases.GOLDEN, name), "rb") as f:
            out.append((name, f.read()))
    out.append(("matrices", matrices_program()))
    out.append(("headers_tail", headers_tail_program()))
    return out
