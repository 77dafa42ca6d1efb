"""Streams with start codes placed on purpose, for K0's start-code scan (ef_scan_kernel, ef_prefix_kernel, ef_fill_kernel).

K0's rule, restated by start_codes(): every byte-aligned 00 00 01 xx whose four bytes lie in the stream is a start code, up to
and including a sequence end code, except a hit inside a sequence header's 8 / 72 / 136 bytes (code included: 12 + 64 per
loaded matrix). The reference reads the matrices with get_bits and searches on from the end of the header
(player.cpp:658-676, 1355-1366), so zero matrix entries can make byte patterns there that are no start code: the non-intra
matrix starts byte aligned (entries 0, 0, 1, c are the bytes 00 00 01 c), the intra matrix one bit early (entries {0|128}, 0,
0, e >= 128 give the code ((e & 0x7F) << 1) | (next >> 7)).

The pictures come from the syntax generator (tests/syntax_cases.py) with knobs that keep every sample independent of the
matrices (intra blocks carry only their DC, non-intra macroblocks only a vector), so a matrix with zero entries stays inside
the reference's defined domain. The cases:
  geometry   the start code of a picture (or, where no room is left before it, the stream's first sequence header) with its
             first 00 at every offset 0-511 of its 512-byte chunk, in chunk 0, 1, 2 or a later one, at every stream-base
             misalignment 0-15 (the sweep rounds the base down to 16 bytes): zero bytes in front of the code place it
  zeros      runs of 2-40 zero bytes in front of a 01
  tails      streams ending 00, 00 00 or 00 00 01, a start code as the last 4 bytes, empty streams and streams of 1-3 bytes,
             and pairs of streams whose bytes form a start code only across the boundary between them
  matrix     zero-entry matrices holding 00 00 01 c for c in 00 01 05 AF B3 B7 B8 (non-intra) and picture / slice codes
             (intra), at stream start and mid-stream, with and without the other matrix, straddling a lane and a chunk edge
  limits     pictures, slices and sequence headers at the index's limits and one past them, a sequence end mid-stream

Every stream is a bytes object; a case also names the stream-base misalignment it needs (pack() places it) and carries a
census of the edge it reaches."""
import functools

import numpy as np

from tests import syntax_cases as sx

CHUNK = 512
# pictures whose samples do not depend on the matrices: DC-only intra blocks, non-intra macroblocks with a vector and no
# coefficients
SAFE = dict(p_dc_only=1.0, p_intra_in_p=0.0, p_mf=1.0, p_coded=0.0, p_mquant=0.0, p_skip=0.2, skip_max=3, p_zero_slices=0.0)
SIZE = (32, 32)                 # 2 x 2 macroblocks: every picture is a few dozen bytes, two slices
# the index limits the limit cases are built for: max_pictures, max_slices_per_picture (max_seq = max_pictures)
LIMIT_PICTURES, LIMIT_SLICES = 4, 3
EMULATED = (0x00, 0x01, 0x05, 0xAF, 0xB3, 0xB7, 0xB8)


# ---- K0's rule ---------------------------------------------------------------------------------------------------------
def header_bytes(es, i):
    """bytes of the sequence header whose code starts at i, code included (bytes past the stream read as 0, as K0's reader)"""
    def bit(b):
        k = i + 4 + (b >> 3)
        return (es[k] >> (7 - (b & 7))) & 1 if k < len(es) else 0
    li = bit(62)
    ln = bit(63 + 512 * li)
    return 12 + 64 * li + 64 * ln


def start_codes(es):
    """[(offset of the first 00, code)] of every start code K0 dispatches, up to and including a sequence end"""
    es = bytes(es)
    out, i, skip = [], 0, 0
    while True:
        i = es.find(b"\x00\x00\x01", i)
        if i < 0 or i + 4 > len(es):
            return out
        if i >= skip:
            c = es[i + 3]
            out.append((i, c))
            if c == 0xB7:
                return out
            if c == 0xB3:
                skip = i + header_bytes(es, i)
        i += 1


def raw_hits(es):
    """every byte-aligned 00 00 01 xx with its four bytes in the stream (the rule without the sequence-header exception)"""
    es = bytes(es)
    out, i = [], 0
    while True:
        i = es.find(b"\x00\x00\x01", i)
        if i < 0 or i + 4 > len(es):
            return out
        out.append((i, es[i + 3]))
        i += 1


def census_of(es):
    """(pictures, slices of pictures, sequence headers) K0 counts before its limits"""
    n_pic = n_slice = n_seq = 0
    for _, c in start_codes(es):
        if c == 0x00:
            n_pic += 1
        elif 0x01 <= c <= 0xAF and n_pic:
            n_slice += 1
        elif c == 0xB3:
            n_seq += 1
    return n_pic, n_slice, n_seq


# ---- building blocks ---------------------------------------------------------------------------------------------------
def _bits_to_bytes(s):
    assert len(s) % 8 == 0
    return int(s, 2).to_bytes(len(s) // 8, "big") if s else b""


def sequence(size=SIZE, intra=None, inter=None):
    """a sequence header; intra / inter: 64 matrix entries to load (None: the default matrix)"""
    w, h = size
    s = sx._b(w, 12) + sx._b(h, 12) + sx._b(1, 4) + sx._b(3, 4) + sx._b(0x3FFFF, 18) + "1" + sx._b(20, 10) + "0"
    for m in (intra, inter):
        s += "0" if m is None else "1" + "".join(sx._b(v, 8) for v in m)
    return b"\x00\x00\x01\xb3" + _bits_to_bytes(s)


def gop(n=0):
    return b"\x00\x00\x01\xb8" + _bits_to_bytes(sx._b((1 << 12) | (n & 63), 25) + "1" + "0" * 6)


SEQ_END = b"\x00\x00\x01\xb7"


@functools.lru_cache(maxsize=None)
def pictures(seed, n, size=SIZE, ptypes=None):
    """n pictures (picture header and slices, each a bytes object) from the syntax generator: I first, then I / P"""
    knobs = dict(SAFE, sizes=[size], n_pictures=(n, n), p_i=0.2)
    if ptypes:
        knobs["ptypes"] = list(ptypes)
    es, off, _, _ = sx.generate(seed, knobs)
    es = bytes(es)
    first = es.find(b"\x00\x00\x01\x00")
    cuts = [first] + [int(x) for x in off[1:]]
    return tuple(es[a:b] for a, b in zip(cuts[:-1], cuts[1:]))


def with_slices(pic, n_slices):
    """a picture with its slices replaced by n_slices copies of its first slice at rows 0, 1, ... (n_slices <= 12 rows of
    the picture's first slice body; rows past the picture's height stay inside the frame's 12 strips)"""
    hits = [i for i, c in raw_hits(pic) if 0x01 <= c <= 0xAF]
    head = pic[:hits[0]] if hits else pic
    if not hits:
        return head
    body = pic[hits[0] + 4:hits[1]] if len(hits) > 1 else pic[hits[0] + 4:]
    return head + b"".join(b"\x00\x00\x01" + bytes([r + 1]) + body for r in range(n_slices))


def base_stream(seed=1, n=3):
    return sequence() + gop() + b"".join(pictures(seed, n))


# ---- cases -------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, name, es, misalign=0, census=None, pinned=True, eos_code=False):
        self.name, self.es, self.misalign = name, bytes(es), misalign
        self.census = dict(census or {})
        # tools/make_scan_pins.py pins it: the reference defines the decode, and its harness can finish the stream. It
        # cannot when the stream holds a sequence end code (the decoder parks in pause() there) or ends in a GOP code (gop()
        # reads the first half of the end padding, and the reader then waits for bytes after the second)
        self.pinned = pinned
        self.eos_code = eos_code        # the reference reads a picture code from the padding behind the stream


def _place(prefix, target, suffix, o, m, chunk):
    """prefix + zeros + target + suffix with target's first byte at offset o of chunk `chunk` of a stream based at misalign
    m; None when the prefix does not fit in front of it"""
    at = chunk * CHUNK + o - m
    if at < len(prefix):
        return None
    return prefix + b"\x00" * (at - len(prefix)) + target + suffix


def geometry_base():
    """the stream every geometry case decodes to: the geometry cases only add zero bytes in front of a start code"""
    return sequence() + gop() + b"".join(pictures(2, 3))


def geometry_cases():
    """the first 00 of a start code at every chunk offset x every misalignment; chunk index 0, 1, 2 or later"""
    pics = pictures(2, 3)
    head, mid = sequence() + gop() + pics[0], pics[1]
    later = [0, 1, 2, 3, 6]
    out = []
    for m in range(16):
        for o in range(CHUNK):
            chunk = later[(o + 3 * m) % 5]
            es = _place(head, mid, pics[2], o, m, chunk)
            what = "picture"
            if es is None:                      # no room for the headers in front: place the sequence header itself
                while True:
                    es = _place(b"", head + mid, pics[2], o, m, chunk)
                    if es is not None:
                        break
                    chunk += 1
                what = "sequence"
            at = (chunk * CHUNK + o - m)
            assert (at + m) % CHUNK == o and (at + m) // CHUNK == chunk
            out.append(Case("geo_o%03d_m%02d" % (o, m), es, m, dict(offset=o, misalign=m, chunk=chunk, code=what, at=at,
                                                                    lane_straddle=o % 16 >= 13, chunk_straddle=o >= CHUNK - 3)))
    return out


def zero_run_cases():
    pics = pictures(3, 3)
    out = []
    for k in range(2, 41):
        es = sequence() + gop() + pics[0] + b"\x00" * (k - 2) + pics[1] + b"\x00" * (k - 2) + pics[2]
        out.append(Case("zeros_%02d" % k, es, k % 16, dict(zero_run=k)))
    return out


def tail_cases():
    base = base_stream(4)
    out = [Case("tail_00", base + b"\x00", 5, dict(ends=b"\x00")),
           Case("tail_0000", base + b"\x00\x00", 7, dict(ends=b"\x00\x00")),
           Case("tail_000001", base + b"\x00\x00\x01", 9, dict(ends=b"\x00\x00\x01"), pinned=False, eos_code=True),
           Case("tail_code_b7", base + SEQ_END, 11, dict(ends=SEQ_END, last4=0xB7), pinned=False),
           Case("tail_code_b8", base + b"\x00\x00\x01\xb8", 13, dict(ends=b"\x00\x00\x01\xb8", last4=0xB8), pinned=False)]
    # the reference reads past a stream's end into the padding its reader appends (00 00 01 B7 twice, player.cpp:456): these
    # end the walk there, while a stream of 1-3 bytes that does not start with zeros, or 00 00 01, makes it read a picture
    # code from the padding
    for n, b in enumerate([b"", b"\x00", b"\xff", b"\x00\x00", b"\x00\x00\x00"]):
        out.append(Case("short_%d" % n, b, n * 5 % 16, dict(short=len(b)), pinned=False))
    for n, b in enumerate([b"\x00\x00\x01", b"\x01\x02", b"\x00\x01\x00", b"\xff\x00\x00"]):
        out.append(Case("short_eos_%d" % n, b, n * 3 % 16, dict(short=len(b)), pinned=False, eos_code=True))
    # across two streams: A ends 00 00 and B starts 01 xx, A ends 00 and B starts 00 01 xx. B's first four bytes are one
    # marker to the reference (prefix, then FF: no marker), so B is a valid stream on its own; xx = 00 would be a picture
    # if the sweep joined the streams. B's misalignment puts A's last bytes in its alignment slack.
    a = base_stream(5)
    b = base_stream(6)
    # pack() puts no filler between A and B: B's misalignment follows from A's
    for tag_a, tail, tag_b, head, mb in (("0000", b"\x00\x00", "01", b"\x01\x00\xff\xff", 5), ("00", b"\x00", "0001", b"\x00\x01\x00\xff", 11)):
        ea = a + tail
        out.append(Case("pair_a_" + tag_a, ea, (mb - len(ea)) % 16, dict(pair="A", ends=tail)))
        out.append(Case("pair_b_" + tag_b, head + b, mb, dict(pair="B", starts=head[:4 - len(tail)])))
    return out


def _entries(r, n):
    return [r.int(1, 255) for _ in range(n)]


def _inter_with(c, j, r):
    m = _entries(r, 64)
    m[j:j + 4] = [0, 0, 1, c]
    return m


def _intra_with(code, k, r):
    """intra entries with the byte pattern 00 00 01 code starting at header byte 8 + k"""
    m = _entries(r, 64)
    e = 128 | (code >> 1)
    nxt = r.int(128, 255) if code & 1 else r.int(1, 127)
    m[k:k + 5] = [r.pick([0, 128]), 0, 0, e, nxt]
    return m


def matrix_cases():
    """zero-entry matrices whose bytes hold a start-code pattern the reference never sees"""
    out = []
    r = sx.Rng(0x5CA7)
    pics = pictures(7, 4)
    for c in EMULATED:
        for where in ("start", "mid"):
            for other in (False, True):
                for j in (0, 9, 60):
                    inter = _inter_with(c, j, r)
                    intra = _entries(r, 64) if other else None
                    hdr = sequence(intra=intra, inter=inter)
                    es = (hdr + gop() + b"".join(pics) if where == "start" else
                          sequence() + gop() + pics[0] + pics[1] + hdr + gop(2) + pics[2] + pics[3])
                    out.append(Case("mat_inter_%02x_%s_%s_%d" % (c, where, "both" if other else "one", j), es, (j * 7 + c) % 16,
                                    dict(kind="inter", code=c, where=where, other=other)))
    for code, tag in ((0x00, "picture"), (0x01, "slice01"), (0x05, "slice05")):
        for where in ("start", "mid"):
            for other in (False, True):
                for k in (0, 30, 59):
                    intra = _intra_with(code, k, r)
                    inter = _entries(r, 64) if other else None
                    hdr = sequence(intra=intra, inter=inter)
                    es = (hdr + gop() + b"".join(pics) if where == "start" else
                          sequence() + gop() + pics[0] + pics[1] + hdr + gop(2) + pics[2] + pics[3])
                    out.append(Case("mat_intra_%s_%s_%s_%d" % (tag, where, "both" if other else "one", k), es, (k * 3 + code) % 16,
                                    dict(kind="intra", code=code, where=where, other=other)))
    # the emulated code straddling a lane (first 00 at 13-15 mod 16) and a chunk (509-511): zeros in front of the header
    for c in (0x00, 0xB3, 0xB7):
        for o in (13, 14, 15, CHUNK - 3, CHUNK - 2, CHUNK - 1):
            m = (o * 5 + c) % 16
            inter = _inter_with(c, 20, r)
            hdr = sequence(inter=inter)
            lead = sequence() + gop() + pics[0]
            at = CHUNK + o - m - 12 - 20                    # the header's offset that puts its pattern at o of chunk 1
            es = lead + b"\x00" * (at - len(lead)) + hdr + gop(1) + pics[1] + pics[2]
            out.append(Case("mat_straddle_%02x_%03d" % (c, o), es, m, dict(kind="inter", code=c, where="mid", other=False, offset=o)))
    return out


def limit_cases():
    """counts at the limits of a context with max_pictures = LIMIT_PICTURES, max_slices_per_picture = LIMIT_SLICES"""
    P, S = LIMIT_PICTURES, LIMIT_SLICES
    size = (32, 96)                     # slices on rows 0..S are rows of the picture (player.cpp:1257)
    raw = pictures(8, P + 1, size, (1,))    # intra only: a slice's copy on another row predicts nothing
    pics = [with_slices(p, 2) for p in raw]
    seq = functools.partial(sequence, size)
    out = []

    def case(name, es, **census):
        out.append(Case(name, es, len(out) % 16, census))

    case("lim_pictures_at", seq() + gop() + b"".join(pics[:P]), over=False)
    case("lim_pictures_past", seq() + gop() + b"".join(pics[:P + 1]), over=True)
    full = [with_slices(p, S) for p in raw[:P]]
    case("lim_slices_at", seq() + gop() + b"".join(full), over=False)
    # one picture over max_slices_per_picture, the stream's total still inside P * S
    case("lim_slices_one_picture_over", seq() + gop() + with_slices(raw[0], S + 1) + with_slices(raw[1], S - 1)
         + b"".join(full[2:]), over=False)
    case("lim_slices_past", seq() + gop() + b"".join(full[:P - 1]) + with_slices(raw[P - 1], S + 1), over=True)
    case("lim_seq_at", b"".join(seq() + gop(k) + pics[k] for k in range(P)), over=False)
    case("lim_seq_past", seq() + b"".join(seq() + gop(k) + pics[k] for k in range(P)), over=True)
    case("lim_seq_end_mid", seq() + gop() + pics[0] + pics[1] + SEQ_END + seq() + gop(2) + pics[2] + pics[3],
         over=False, seq_end=True)
    out[-1].pinned = False
    case("lim_no_slices", seq() + gop() + pics[0] + with_slices(pics[1], 0) + pics[2] + with_slices(pics[3], 0), over=False)
    return out


@functools.lru_cache(maxsize=None)
def all_cases():
    return geometry_cases() + zero_run_cases() + tail_cases() + matrix_cases() + limit_cases()


def directed_cases():
    """every case but the geometry sweep"""
    return [c for c in all_cases() if not c.name.startswith("geo_")]


def pack(streams, misaligns):
    """streams placed at the given base misalignments: a filler stream of zero bytes (no start code, no picture) in front of
    each stream that needs one -> (blob, offsets, index of each stream). Zero bytes, because K1a reads a stream's last
    slice on into the bytes behind the stream, where the reference reads the 00 00 01 B7 of its end padding: the two agree
    when those bytes start with at least 23 zero bits, as a stream that starts with a start code or a filler of zeros does."""
    parts, idx, at = [], [], 0
    for s, m in zip(streams, misaligns):
        pad = (m - at) % 16
        if pad or not parts:
            parts.append(b"\x00" * pad)
            at += pad
        idx.append(len(parts))
        parts.append(bytes(s))
        at += len(s)
    off = np.zeros(len(parts) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(p) for p in parts])
    blob = np.frombuffer(b"".join(parts), dtype=np.uint8).copy() if int(off[-1]) else np.zeros(1, np.uint8)
    return blob, off, idx


def batch_pool():
    """streams for the batch shapes: 0 to LIMIT_PICTURES pictures each, some pictures without slices"""
    out = []
    for k in range(67):
        n = k % (LIMIT_PICTURES + 1)
        pics = list(pictures(100 + k % 11, max(n, 1)))[:n]
        if k % 3 == 0 and n > 1:
            pics[1] = with_slices(pics[1], 0)
        es = (sequence() + gop() + b"".join(pics)) if n else (sequence() + gop() if k % 2 else b"")
        out.append(es)
    return out


def unit_offsets(es):
    """ES offsets of the access units (a picture with the sequence and GOP headers in front of it) and the end: where
    synth.wrap_ts starts a PES"""
    out, start = [], None
    for i, c in start_codes(es):
        if c in (0xB3, 0xB8) and start is None:
            start = i
        elif c == 0x00:
            out.append(start if start is not None else i)
            start = None
    if not out:
        return np.array([0, len(es)], dtype=np.uint32)
    out[0] = 0
    return np.array(out + [len(es)], dtype=np.uint32)
