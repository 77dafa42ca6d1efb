"""tests/trick_scale_cases.py — mains that take ef_trick_build past its first batch and into the encoder's rare codes, an independent
reading of the trick pictures it writes, and plan(): the host side of ef_trick_build (segment cuts, batches, selection, encode
flushes) restated, so that every scenario can show which path it reaches.

Mains here are built from I420 frames with the trick encoder itself (trick_cases.encode_picture): every picture is intra, carries
its own sequence header and starts a PES with a PTS, so every picture may start a segment. The encoder of the trick files sees the
frames the oracle decodes from such a main, not the frames it was built from; every coverage claim below is checked on the levels
trick_cases computes from that decode."""
import functools
import os
import re

import numpy as np

from tests import pts_cases, trick_cases as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Y_BYTES, C_BYTES = 352 * 192, 176 * 96
FRAME = Y_BYTES + 2 * C_BYTES
P = 3003                                   # 29.97 Hz picture period in 90 kHz ticks
NULL = bytes([0x47, 0x1F, 0xFF, 0x10]) + b"\xff" * 184      # a null packet (PID 0x1FFF)

# ef_trick_build's host constants (csrc/ef_capi.cu) and the encoder's per-slice region (csrc/ef_common.cuh), read from the source
_CAPI = open(os.path.join(ROOT, "espflix_b200", "csrc", "ef_capi.cu")).read()
CHUNK_STREAMS = int(re.search(r"kTrickChunkStreams = (\d+);", _CAPI).group(1))
CHUNK_BYTES = int(re.search(r"kTrickChunkBytes = (\d+)u << (\d+);", _CAPI).group(1)) << int(re.search(r"kTrickChunkBytes = (\d+)u << (\d+);", _CAPI).group(2))
ENCODE_BATCH = int(re.search(r"kTrickEncodeBatch = (\d+);", _CAPI).group(1))
MAX_PICTURES = int(re.search(r"std::min<uint64_t>\(max_pusi, (\d+)\)", _CAPI).group(1))
SLICE_BYTES = int(re.search(r"kTrickSliceBytes = (\d+);", open(os.path.join(ROOT, "espflix_b200", "csrc", "ef_common.cuh")).read()).group(1))


# -- frames -----------------------------------------------------------------------------------------------------------------------
def flat(y, cb=128, cr=128):
    return bytes([y]) * Y_BYTES + bytes([cb]) * C_BYTES + bytes([cr]) * C_BYTES


def planes(y, cb, cr):
    return np.asarray(y, np.uint8).tobytes() + np.asarray(cb, np.uint8).tobytes() + np.asarray(cr, np.uint8).tobytes()


_C = np.array([[(np.sqrt(1 / 8) if k == 0 else 0.5) * np.cos((2 * n + 1) * k * np.pi / 16) for n in range(8)] for k in range(8)])


def basis_block(raster, amp, dc=128):
    """an 8 x 8 block of mean `dc` whose only AC energy is about `amp` at coefficient `raster` (orthonormal DCT scale)"""
    u, v = divmod(raster, 8)
    return np.clip(np.rint(dc + amp * np.outer(_C[u], _C[v])), 0, 255).astype(np.uint8)


def _tile(blocks, rows, cols, fill=128):
    """blocks (a list of 8 x 8 arrays) laid out row by row on a rows x cols grid of blocks, the rest `fill`"""
    out = np.full((rows * 8, cols * 8), fill, np.uint8)
    for k, b in enumerate(blocks[:rows * cols]):
        r, c = divmod(k, cols)
        out[r * 8:r * 8 + 8, c * 8:c * 8 + 8] = b
    return out


def sweep_frame():
    """zig-zag 1 (raster 1, matrix entry 16) swept across levels 36..45 and 122..133 of both signs at qscale 1 (8 F / 16 = F / 2),
    single coefficients at zig-zag 32, 33 and 63 (runs 31, 32 and 62 after the DC) at several amplitudes, and DC steps of 255 in
    luma (an 8-pixel 0 / 255 checkerboard row) and chroma (macroblocks alternating 0 and 255)"""
    blocks = []
    for lv in (40, 41, 127, 128):
        for s in (1, -1):
            for amp in np.arange(2 * lv - 3, 2 * lv + 3, 0.25):
                for dc in (96, 128, 160):
                    blocks.append(basis_block(1, s * amp, dc))
    for zz in (3, 4, 5):                      # matrix entries 19, 22, 22: other rounding grids reach 128 where 16 does not
        raster = int(tc.ZIGZAG[zz])
        for s in (1, -1):
            for amp in np.arange(-6, 6, 0.5) + 128 * int(tc.INTRA_Q[raster]) / 8:
                blocks.append(basis_block(raster, s * amp))
    for zz in (32, 33, 63):
        for amp in (12, 20, 28, 40, 60, 90, 140, 200, 260, 320, -12, -20, -40, -90, -200):
            blocks.append(basis_block(int(tc.ZIGZAG[zz]), amp))
    y = _tile(blocks, 24, 44)
    y[176:192] = ((np.arange(352)[None, :] // 8 + np.arange(16)[:, None] // 8) % 2 * 255).astype(np.uint8)
    cb = np.full((96, 176), 128, np.uint8)
    cr = np.full((96, 176), 128, np.uint8)
    alt = (np.arange(176) // 8 % 2 * 255).astype(np.uint8)
    cb[88:96] = alt[None, :]
    cr[88:96] = 255 - alt[None, :]
    return planes(y, cb, cr)


def clamp_frame():
    """+-max basis patterns (0 / 255 by the sign of a low-frequency basis function): F far past 255 q Q / 8 at qscale 1"""
    blocks = []
    for raster in (1, 8, 9, 2, 16, 10, 17):
        u, v = divmod(raster, 8)
        pat = (np.outer(_C[u], _C[v]) > 0).astype(np.uint8) * 255
        blocks += [pat, 255 - pat]
    return planes(_tile(blocks * 76, 24, 44), _tile(blocks * 19, 12, 22), _tile(blocks[::-1] * 19, 12, 22))


def noise_frame(seed):
    """full-range uniform noise: the largest slices the encoder writes"""
    return np.random.default_rng(seed).integers(0, 256, FRAME, dtype=np.uint8).tobytes()


def sparse_frame(seed, count):
    """flat grey with `count` 8 x 8 blocks set to random flat levels: DC-only pictures whose coded size moves with the seed"""
    rng = np.random.default_rng(seed)
    fr = np.frombuffer(flat(128), np.uint8).copy()
    y = fr[:Y_BYTES].reshape(192, 352)
    for _ in range(count):
        r, c = rng.integers(0, 24), rng.integers(0, 44)
        y[r * 8:r * 8 + 8, c * 8:c * 8 + 8] = rng.integers(0, 256)
    return fr.tobytes()


# -- mains ------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4096)
def _picture(frame, qscale, aspect, rate, seq):
    """frame: I420 bytes, or an int for flat(frame) (kept small in the cache)"""
    es = tc.encode_picture(flat(frame) if isinstance(frame, int) else frame, qscale, tc.header_bytes(aspect, rate))
    return es if seq else es[12:]                 # without its sequence header: the picture continues the segment before it


def intra_main(frames, pts=None, qscale=1, aspect=1, rate=3, seq=True, edit=None, pes=None):
    """a main of intra pictures from I420 frames (an int y stands for flat(y)), one PES with a PTS per picture (`pes`: pictures per PES instead); qscale and
    seq (a sequence header before the picture) may be lists; edit: {picture index: function(picture ES) -> ES}"""
    n = len(frames)
    pts = [90000 + P * k for k in range(n)] if pts is None else list(pts)
    q = qscale if isinstance(qscale, (list, tuple)) else [qscale] * n
    s = seq if isinstance(seq, (list, tuple)) else [seq] * n
    pics = [_picture(frames[k] if isinstance(frames[k], int) else bytes(frames[k]), q[k], aspect, rate, bool(s[k])) for k in range(n)]
    for k, fn in (edit or {}).items():
        pics[k] = fn(pics[k])
    if pes is None:
        return tc.mux(pics, pts)
    groups = [(b"".join(pics[k:k + pes]), pts[k]) for k in range(0, n, pes)]
    return tc.mux([g for g, _ in groups], [p for _, p in groups])


def pad(ts, after, packets):
    """null packets (PID 0x1FFF) inserted after the PES of picture `after` (mains from intra_main)"""
    starts = [k for k in range(len(ts) // 188) if ts[k * 188 + 1] & 0x40] + [len(ts) // 188]
    cut = starts[after + 1] * 188
    return ts[:cut] + NULL * packets + ts[cut:]


def slices(es):
    """picture ES -> (bytes before the first slice, [(vertical position, slice bytes)])"""
    at = [m.start() for m in re.finditer(b"\x00\x00\x01", es)]
    body = [i for i in at if 0x01 <= es[i + 3] <= 0xAF]
    return es[:body[0]], [(es[i + 3], es[i:j]) for i, j in zip(body, body[1:] + [len(es)])]


def drop_slice(vpos):
    def fn(es):
        head, sl = slices(es)
        return head + b"".join(b for v, b in sl if v != vpos)
    return fn


_MBA = tc._vlc("ef_vlc_mba")


def flat_slice(vpos, first_col, y, qscale=1):
    """a slice of flat macroblocks of luma `y` (chroma 128) from column first_col to the end of its row: first address increment
    first_col + 1, then DC-only blocks"""
    bits = format(qscale, "05b") + "0"
    pred = [128, 128, 128]
    for col in range(first_col, 22):
        bits += _MBA[first_col + 1] if col == first_col else "1"
        bits += "1"                                               # intra
        for b, v in enumerate([y] * 4 + [128, 128]):
            comp = 0 if b < 4 else b - 3
            d = v - pred[comp]
            pred[comp] = v
            size = abs(d).bit_length()
            bits += tc.DC_CODES[min(comp, 1)][size] + (format(d if d > 0 else d + (1 << size) - 1, "0%db" % size) if size else "")
            bits += "10"
    bits += "0" * (-len(bits) % 8)
    return bytes([0, 0, 1, vpos]) + int(bits, 2).to_bytes(len(bits) // 8, "big")


def restart_row(vpos, first_col, y):
    """the slice of row vpos replaced by flat_slice(vpos, first_col, y): written to start mid-row. The decoder puts a slice's first
    macroblock at column 0 whatever its increment (player.cpp:823), so the picture writes columns 0 .. 21 - first_col of the row
    and leaves the rest as the frame store held it"""
    def fn(es):
        head, sl = slices(es)
        return head + b"".join(flat_slice(vpos, first_col, y) if v == vpos else b for v, b in sl)
    return fn


# -- the cases --------------------------------------------------------------------------------------------------------------------
ADV_PICTURES = (0, 15, 30)                 # the selected pictures of adversarial_main()


def adversarial_main():
    """main pictures 0, 15 and 30 (the selected ones) carry the sweep, clamp and noise frames, flat pictures in between; the clamp
    picture is coded at qscale 4 in the main so that its decode saturates (levels at qscale 1 would stop at 255 exactly)"""
    frames = [16 + 7 * k for k in range(31)]
    frames[0], frames[15], frames[30] = sweep_frame(), clamp_frame(), noise_frame(5)
    q = [1] * 31
    q[15] = 4
    return intra_main(frames, qscale=q)


# (14 + ES length) % 184 of a fwd picture sets how the mux ends its PES: 0 no adaptation field, 183 a length byte only, 182 a
# length byte and the flags byte, 1 the longest stuffing. (seed, blocks) of sparse_frame at RESIDUE_QSCALE, found by
# residue_search(); each block adds about 3 bytes to a picture of 2,384 bytes.
RESIDUE_QSCALE = 8
RESIDUE_FRAMES = {0: (1, 3), 1: (7, 3), 182: (1, 2), 183: (13, 2)}


def residue_search(want, qscale=RESIDUE_QSCALE):
    """the first (seed, blocks) whose sparse_frame picture ends its PES on residue `want` (how RESIDUE_FRAMES was found)"""
    hdr = tc.header_bytes(1, 3)
    for blocks in range(12):
        for seed in range(30):
            if (14 + len(tc.encode_picture(sparse_frame(seed, blocks), qscale, hdr))) % 184 == want:
                return seed, blocks
    return None


def residue_main():
    """fwd pictures 0..3 end their PES on residues 0, 1, 182 and 183 at RESIDUE_QSCALE"""
    frames = [100] * 46
    for k, r in enumerate(sorted(RESIDUE_FRAMES)):
        frames[15 * k] = sparse_frame(*RESIDUE_FRAMES[r])
    return intra_main(frames)


def dropped_slice_main():
    """20 flat intra pictures of luma 10 k, each with a sequence header; picture 15 (fwd picture 1) lacks slice 5, so its row 4
    keeps what the frame store held: picture 13's 130 in a continuous decode, 0 after a reset"""
    return intra_main([10 * k for k in range(20)], edit={15: drop_slice(5)})


def mid_row_main():
    """as dropped_slice_main, but picture 15's slice 5 is written to start at column 6 (first address increment 7): its 16
    macroblocks land at columns 0..15, and columns 16..21 of row 4 keep what the frame store held"""
    return intra_main([10 * k for k in range(20)], edit={15: restart_row(5, 6, 150)})


def next_picture_main():
    """picture 14 is whole but picture 15 lacks slice 9: a segment that starts at 14 decodes 15 into a frame store fresh from the
    reset (the picture before 14 never wrote it), so the cut at 14 must go too"""
    return intra_main([10 * k for k in range(20)], edit={15: drop_slice(9)})


# -- an independent reading of trick pictures ---------------------------------------------------------------------------------------
class _Bits:
    def __init__(self, data):
        self.s = "".join(format(b, "08b") for b in data)
        self.i = 0

    def read(self, n):
        v = int(self.s[self.i:self.i + n], 2) if n else 0
        assert len(self.s[self.i:self.i + n]) == n, "read past the end"
        self.i += n
        return v

    def vlc(self, table, longest=17):
        for n in range(1, longest + 1):
            c = self.s[self.i:self.i + n]
            if c in table:
                self.i += n
                return table[c]
        raise AssertionError("no code at bit %d" % self.i)


_DCT_BY_CODE = {c: v for v, c in tc._DCT.items()}
_DC_BY_CODE = [{c: v for v, c in t.items()} for t in tc.DC_CODES]
_MBA_BY_CODE = {c: v for v, c in _MBA.items()}
_TABLE_PAIRS = {(v >> 8, v & 0xFF) for v in tc._DCT}     # (run, level) pairs the table codes: never escaped


def parse_picture(es):
    """an intra trick picture (trick_cases' layout: headers, then slices 1..12 of 22 macroblocks) -> levels int64 [12, 22, 6, 64]
    in zig-zag order, read with ISO 11172-2's tables (Annex B) and its escape forms; non-canonical or forbidden forms fail"""
    head, sl = slices(es)
    assert head[:4] == b"\x00\x00\x01\xb3" and b"\x00\x00\x01\x00" in head
    pic = head.index(b"\x00\x00\x01\x00")
    assert (head[pic + 5] >> 3) & 7 == 1, "not an I picture"
    assert [v for v, _ in sl] == list(range(1, 13)), [v for v, _ in sl]
    out = np.zeros((12, 22, 6, 64), np.int64)
    for row, (_, data) in enumerate(sl):
        r = _Bits(data[4:])
        qscale = r.read(5)
        assert r.read(1) == 0, "extra_bit_slice"
        pred = [128, 128, 128]
        for mb in range(22):
            assert r.vlc(_MBA_BY_CODE, 11) == 1, "address increment"
            assert r.read(1) == 1, "macroblock type"
            for b in range(6):
                comp = 0 if b < 4 else b - 3
                size = r.vlc(_DC_BY_CODE[min(comp, 1)], 8)
                d = r.read(size)
                if size and not d >> (size - 1):
                    d -= (1 << size) - 1
                pred[comp] += d
                assert 0 <= pred[comp] <= 255
                out[row, mb, b, 0] = pred[comp]
                i = 0
                while True:
                    if r.s[r.i:r.i + 2] == "10":
                        r.i += 2
                        break
                    if r.s[r.i:r.i + 6] == "000001":
                        r.i += 6
                        run, lv = r.read(6), r.read(8)
                        if lv == 0:
                            lv = r.read(8)
                            assert lv >= 128, "16-bit escape of a level that fits 8 bits"
                        elif lv == 128:
                            lv = r.read(8) - 256
                            assert lv <= -128, "16-bit escape of a level that fits 8 bits"
                            assert lv >= -255, "16-bit escape of -256"
                        elif lv > 128:
                            lv -= 256
                        assert (run, abs(lv)) not in _TABLE_PAIRS, "escape of a pair the table codes"
                    else:
                        v = r.vlc(_DCT_BY_CODE)
                        run, lv = v >> 8, v & 0xFF
                        if r.read(1):
                            lv = -lv
                    i += run + 1
                    assert i < 64, "past the end of the block"
                    out[row, mb, b, i] = lv
        rest = r.s[r.i:]
        assert len(rest) < 8 and set(rest) <= {"0"}, "slice ends on a zero-padded byte"
        assert qscale >= 1
    return out



def fwd_pictures(ts):
    """the picture ES of every PES of a trick file, in order"""
    es, pes = pts_cases.demux(ts)
    offs = [o for o, _ in pes] + [len(es)]
    return [es[a:b] for a, b in zip(offs, offs[1:])]


def trick_levels(frame, qscale):
    return tc.quantise(tc.fdct(tc.picture_blocks(frame)), qscale)


# -- the host plan ------------------------------------------------------------------------------------------------------------------
def _video_packets(ts):
    """(packet numbers of video packets with payload, ES offset where each one's payload starts, the video ES, {packet: PTS ok})"""
    a = np.frombuffer(bytes(ts), np.uint8).reshape(-1, 188)
    pid = ((a[:, 1].astype(np.int64) << 8) | a[:, 2]) & 0x1FFF
    vid = np.nonzero((a[:, 0] == 0x47) & (pid == 0x100) & ((a[:, 3] & 0x10) != 0))[0]
    es, at, pts_ok = bytearray(), [], {}
    for k in vid:
        d = a[k]
        o = 5 + int(d[4]) if d[3] & 0x20 else 4
        if d[1] & 0x40 and o + 14 <= 188:
            flags = (int(d[o + 6]) << 8) | int(d[o + 7])
            pts_ok[int(k)] = bool(flags & 0x80) and (int(d[o + 9]) & 0xF0) == ((flags >> 2) & 0x30)
            o += 9 + int(d[o + 8])
        at.append(len(es))
        if o < 188:
            es += d[o:].tobytes()
    return vid, np.array(at, np.int64), bytes(es), pts_ok


def _pictures(es):
    """[(ES offset of the picture start code, picture_coding_type)] of a video ES, up to a sequence end code"""
    return [(o - 3, (es[o + 2] >> 3) & 7 if o + 2 < len(es) else 0) for o in pts_cases.picture_codes(es)]


def starts_whole(es, oracle):
    """whether a segment may start at es (a sequence header, then pictures): its first picture is intra and the oracle's decode
    of it writes every macroblock of the picture from its own codes; its second, intra or predicted, writes every macroblock,
    coded or skipped. The sizes are the sequence header's, at most the 22 x 12 frame store."""
    pics = _pictures(es)[:3]
    if not pics or pics[0][1] != 1 or (len(pics) > 1 and pics[1][1] not in (1, 2)):
        return False
    body = es[:pics[2][0]] if len(pics) > 2 else es
    oracle.decode_es(body, max_frames=4)
    cov = oracle.coverage(2)[:min(len(pics), 2)].reshape(-1, 12, 22)
    w, h = ((es[4] << 4) | (es[5] >> 4)), (((es[5] & 15) << 8) | es[6])
    cov = cov[:, :min((h + 15) >> 4, 12), :min((w + 15) >> 4, 22)]
    return bool((cov[0] == 2).all() and (len(cov) < 2 or (cov[1] > 0).all()))


def plan(mains, oracle, rec_pics=None):
    """ef_trick_build's host plan for `mains`:
    segs     [(main, first packet, end packet, pictures)]: a main is cut before each sequence header of make_index's table whose
             PES has a PTS parse_pts() accepts and where starts_whole() holds (so a decode from reset frame stores gives the
             frames of a continuous one)
    batches  [(first segment, end segment, reason of the cut after it: 'count', 'bytes' or 'end')]
    selected [[(main, main picture)] of every batch]
    events   [('ctx', batch, max_pictures) | ('grow_in', batch, capacity) | ('flush', batch, pictures, 'room' / 'full' / 'end')]
    pieces   [decode_range calls of every batch] when rec_pics is given"""
    segs, guess = [], 1
    for f, ts in enumerate(mains):
        vid, at, es, pts_ok = _video_packets(ts)
        pic_at = np.array([o for o, _ in _pictures(es)], np.int64)
        npk = len(ts) // 188

        def es_at(pkt):
            j = np.searchsorted(vid, pkt)
            return int(at[j]) if j < len(vid) else len(es)

        cuts = [0]
        for p in oracle.make_index(ts)["seq_pos"][1:]:
            p = int(p)
            if p <= cuts[-1] or not pts_ok.get(p, False):
                continue
            if not starts_whole(es[es_at(p):], oracle):
                continue
            cuts.append(p)
        for a, b in zip(cuts, cuts[1:] + [npk]):
            n = int(np.searchsorted(pic_at, es_at(b)) - np.searchsorted(pic_at, es_at(a)))
            segs.append((f, a, b, n))
            pusi = sum(1 for k in vid[(vid >= a) & (vid < b)] if ts[int(k) * 188 + 1] & 0x40)
            guess = max(guess, pusi + 1)
    base = np.cumsum([0] + [len(m) // 188 for m in mains])
    g0 = lambda s: int(base[segs[s][0]] + segs[s][1])            # noqa: E731
    g1 = lambda s: int(base[segs[s][0]] + segs[s][2])            # noqa: E731
    starts, why = [0], []
    for s in range(len(segs)):
        c0 = starts[-1]
        if s > c0 and (s - c0 >= CHUNK_STREAMS or (g1(s) - g0(c0)) * 188 > CHUNK_BYTES):
            why.append("count" if s - c0 >= CHUNK_STREAMS else "bytes")
            starts.append(s)
    batches = [(a, b, w) for a, b, w in zip(starts, starts[1:] + [len(segs)], why + ["end"])]
    maxp_ctx = min(guess, MAX_PICTURES)
    seen = [0] * len(mains)
    selected, events, pieces = [], [], []
    pending, in_cap = 0, 0
    for c, (a, b, _) in enumerate(batches):
        need = max(segs[s][3] for s in range(a, b))
        grew = c == 0
        while need > maxp_ctx and maxp_ctx < MAX_PICTURES:
            maxp_ctx, grew = min(MAX_PICTURES, maxp_ctx * 2), True
        if grew:
            events.append(("ctx", c, maxp_ctx))
        sel = []
        for s in range(a, b):
            f = segs[s][0]
            for _ in range(segs[s][3]):
                if seen[f] % tc.SPEED == 0:
                    sel.append((f, seen[f]))
                seen[f] += 1
        selected.append(sel)
        if pending + len(sel) > in_cap:
            if pending:
                events.append(("flush", c, pending, "room"))
            pending = 0
            if len(sel) > in_cap:
                in_cap = max(len(sel), ENCODE_BATCH)
                events.append(("grow_in", c, in_cap))
        if rec_pics is not None:
            rp = min(rec_pics, maxp_ctx)
            pieces.append(-(-need // rp) if sel else 0)
        pending += len(sel)
        if pending >= ENCODE_BATCH:
            events.append(("flush", c, pending, "full"))
            pending = 0
    if pending:
        events.append(("flush", len(batches), pending, "end"))
    return {"segs": segs, "batches": batches, "selected": selected, "events": events, "pieces": pieces, "guess": min(guess, MAX_PICTURES)}


# -- scenarios: mains that reach each path of the host plan (tests/test_trick_scale.py checks each one's plan) -----------------------
def flat_run(n, seed):
    """n flat pictures (ints for intra_main) whose luma steps by 37 from a seed-dependent start"""
    return [(seed * 53 + 37 * k) % 256 for k in range(n)]


def many_segments():
    """one main of 600 one-picture segments: batches cut at 256 segments, and the every-15th selection runs across the cuts"""
    return [intra_main(flat_run(600, 1))]


def many_mains():
    """150 mains of 1..3 one-picture segments, 100 mains of one 31-picture segment, 150 short mains again: more than 256 selected
    pictures, so encodes flush with pictures pending from earlier batches, the ES buffer grows keeping what it holds, and a batch
    selects more pictures than the encoder's input holds"""
    out = []
    for j in range(400):
        if 150 <= j < 250:
            out.append(intra_main(flat_run(31, j), seq=[True] + [False] * 30))
        else:
            out.append(intra_main(flat_run(1 + j % 3, j)))
    return out


def padded_main():
    """40 one-picture segments; null packets after pictures 3 and 8 (40 MB each) cut batches by bytes before 256 segments, and
    70 MB after picture 16 make a segment longer than a batch, which selects nothing (main picture 16 is not a 15th)"""
    ts = intra_main(flat_run(40, 2))
    for after, mb in ((16, 70), (8, 40), (3, 40)):
        ts = pad(ts, after, (mb << 20) // 188)
    return ts


def multi_pes_mains():
    """a main of 260 one-picture segments (so the first guess is 2 pictures per segment), then one of 40 pictures, 10 per PES:
    its segments hold 10 pictures, so the second batch rebuilds the decode context with more pictures"""
    return [intra_main(flat_run(260, 3)), intra_main(flat_run(40, 4), pes=10)]


def cut_cases():
    return {"dropped_slice": dropped_slice_main(), "mid_row": mid_row_main(), "next_picture": next_picture_main()}


# what each scenario's plan must show (tests/test_trick_scale.py on the CPU, tests/test_trick_scale_gpu.py beside the build)
def check_many_segments(p):
    assert [w for _, _, w in p["batches"]] == ["count", "count", "end"]
    assert [len(s) for s in p["selected"]] == [18, 17, 5]                   # 256 is not a multiple of 15
    assert [(f, j) for s in p["selected"] for f, j in s] == [(0, 15 * k) for k in range(40)]
    assert not [e for e in p["events"] if e[0] == "flush" and e[3] != "end"]   # pending pictures carried across batches


def check_many_mains(p):
    flushes = [e for e in p["events"] if e[0] == "flush"]
    assert flushes[0][3] == "room" and len(flushes) >= 3                    # flushed partway; d_es grows twice, keeping
    assert [e[0] for e in p["events"]].count("grow_in") == 2                 # d_in reserved again after a flush
    assert sum(len(s) for s in p["selected"]) > ENCODE_BATCH


def check_padded(p):
    assert [w for _, _, w in p["batches"]] == ["bytes", "bytes", "bytes", "end"]
    assert p["batches"][2][1] - p["batches"][2][0] == 1 and p["selected"][2] == []


def check_multi_pes(p):
    ctx = [e for e in p["events"] if e[0] == "ctx"]
    assert ctx[0] == ("ctx", 0, 2) and ctx[-1][1] == 1 and ctx[-1][2] >= 10    # a later batch needs more pictures


def long_main(copies=60):
    """the vmedia fixture back to back `copies` times: 4,320 pictures of ffmpeg's mpeg1video slices (5 a picture, each running
    across rows), more than one segment may hold, so it builds only when it is cut at its I pictures"""
    return tc.fixture("vmedia") * copies


def check_long(p):
    assert max(n for _, _, _, n in p["segs"]) <= 12 and sum(n for _, _, _, n in p["segs"]) > MAX_PICTURES
