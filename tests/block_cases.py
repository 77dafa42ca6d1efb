"""Block-level MPEG-1 streams for K1b's arithmetic: each macroblock's contents are chosen, not drawn. The writer pieces
(bit output, start codes, VLC tables, coefficient, DC, address and vector codes) are those of tests/syntax_cases.py, and
so are its rules: only valid codes, no run of 23 zero bits inside a slice, slices never share a row, every prediction
window inside the 352 x 192 frame.

  basis_*      every raster position alone, intra and non-intra, at small levels and at the dequantised extremes
               +2047 / -2048 (quantiser 31, matrix entries 255, 16-bit escapes); position 0 alone (Q5, n == 1) and
               position 0 plus one more (full IDCT)
  edges        pre-clamp samples of exactly -256, -1, 0, 248, 249 and 511: intra, and non-intra over predictions of
               0, 248 and 255
  signs_*      for each output sample, the coefficients +-2048 * sign(L[o][i]) in both signs (the largest samples the
               transform can produce), non-intra over every prediction byte, and intra
  dc_*         intra DC predictors climbing past +32,768 and below -32,768 in +-255 steps, with plateaus at 16k-20k,
               each level with DC-only blocks (Q7), one small AC coefficient and a saturated AC sign pattern
  pred_*       P pictures whose vectors cover every luma (hx mod 32, hy mod 32) and so every chroma (cx mod 16, cy mod 16)
               alignment of the staged prediction words, windows on all four frame edges with each half-pel flag, over
               a reference holding bytes 249..255 and the mixed bytes of Q7, with no, a small and a clamping residual
  pairs        every ordered pair of macroblock kinds in the two slots (2k, 2k + 1) that one K1b warp rebuilds

Each case records a census of what it reached; tests/test_blocks.py asserts it. Which cases leave the reference's
clamp-table domain is decided by the restatement (UNPINNED)."""
import os
import re
from collections import Counter

import numpy as np

from tests import idct_linear
from tests import syntax_cases as sc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _table(name):
    hdr = open(os.path.join(ROOT, "espflix_b200", "csrc", "ef_iso11172_tables.h")).read()
    i = hdr.index(name + "[64]")
    return [int(x) for x in re.findall(r"\d+", hdr[hdr.index("{", i):hdr.index("};", i)])]


ZIGZAG = _table("ef_zigzag")                 # scan index -> raster position
SCAN = [ZIGZAG.index(p) for p in range(64)]  # raster position -> scan index
PRESCALE = _table("ef_aan_prescale")
INTRA_Q = _table("ef_default_intra_q")
L = idct_linear.matrix()                     # [output][input], raster


# ---- integer port of the reference IDCT (player.cpp:922-996) ---------------------------------------------------------
def _pass(v):
    b1, b3, b4 = v[..., 4], v[..., 2] + v[..., 6], v[..., 5] - v[..., 3]
    t1, t2, b6 = v[..., 1] + v[..., 7], v[..., 3] + v[..., 5], v[..., 1] - v[..., 7]
    b7, m0 = t1 + t2, v[..., 0]
    x4 = ((b6 * 473 - b4 * 196 + 128) >> 8) - b7
    x0 = x4 - (((t1 - t2) * 362 + 128) >> 8)
    x1, x2, x3 = m0 - b1, (((v[..., 2] - v[..., 6]) * 362 + 128) >> 8) - b3, m0 + b1
    y3, y4, y5, y6 = x1 + x2, x3 + b3, x1 - x2, x3 - b3
    y7 = -x0 - ((b4 * 473 + b6 * 196 + 128) >> 8)
    return np.stack([b7 + y4, x4 + y3, y5 - x0, y6 - y7, y6 + y7, x0 + y5, y3 - x4, y4 - b7], axis=-1)


def idct(b):
    """prescaled coefficients [..., 64] (raster) -> pre-clamp samples [..., 64], columns then rows, (x + 128) >> 8"""
    b = np.asarray(b, dtype=np.int64)
    m = b.reshape(b.shape[:-1] + (8, 8))
    cols = np.swapaxes(_pass(np.swapaxes(m, -1, -2)), -1, -2)
    return ((_pass(cols) + 128) >> 8).reshape(b.shape)


def dequant(level, q, m, intra):
    """dequantised coefficient (player.cpp:1105-1125, Q2, saturation)"""
    v = 2 * level
    if not intra:
        v += -1 if v < 0 else 1
    t = v * q * m
    v = abs(t) // 16 * (1 if t >= 0 else -1)
    if v & 1 == 0:
        v -= 1 if v > 0 else -1
    return max(-2048, min(2047, v))


def samples(blk, q, mat, intra, dc=0):
    """pre-clamp samples of a block {coefs: [(raster, level)]} (intra: with DC `dc`)"""
    b = np.zeros(64, dtype=np.int64)
    for p, lv in blk.get("coefs", ()):
        b[p] = dequant(lv, q, mat[p], intra) * PRESCALE[p]
    if intra:
        b[0] = dc << 8
    return idct(b)


# ---- the writer ------------------------------------------------------------------------------------------------------
def _b(v, n):
    return sc._b(v, n)


class Writer(sc._Stream):
    """A stream whose macroblocks are given. Macroblock: dict(intra, q (mquant) or None, mv (stored units) or None
    (no motion_forward), blocks: six entries of None (not coded) or {dc (intra, absolute), coefs: [(raster, level)],
    abort}, skip: macroblocks skipped before it)."""

    def __init__(self, intra_q=None, non_intra_q=None):
        super().__init__(0, dict(sc.BASE, p_wrap=0.0))
        self.mats = (intra_q, non_intra_q)
        self.mat = [list(INTRA_Q) if intra_q is None else list(intra_q), [16] * 64 if non_intra_q is None else list(non_intra_q)]
        self.n_pic = 0

    def sequence_header(self, intra_q=None, non_intra_q=None):
        self.start_code(0xB3)
        self.put(_b(352, 12) + _b(192, 12) + _b(1, 4) + _b(3, 4) + _b(0x3FFFF, 18) + "1" + _b(20, 10) + "0")
        for i, m in enumerate((intra_q, non_intra_q)):
            if m is None:
                self.put("0")
                self.mat[i] = list(INTRA_Q) if i == 0 else [16] * 64
            else:
                self.put("1" + "".join(_b(v, 8) for v in m))
                self.mat[i] = list(m)
        self.mbw, self.mbh = 22, 12
        self.gop(0)

    def start_picture(self, ptype, fp=0, f_code=1):
        self.pic_off.append(self.nbits // 8 + (1 if self.nbits % 8 else 0))
        if self.n_pic == 0:
            self.sequence_header(*self.mats)
        self.start_code(0x00)
        self.put(_b(self.n_pic, 10) + _b(ptype, 3) + _b(0xFFFF, 16))
        if ptype == 2:
            self.fp, self.rs = fp, f_code - 1
            self.put(_b(fp, 1) + _b(f_code, 3))
        self.ptype = ptype
        self.n_pic += 1

    def _coefs(self, blk, intra):
        s, n = "", 1 if intra else 0
        for p, lv in sorted(blk.get("coefs", ()), key=lambda c: SCAN[c[0]]):
            k = SCAN[p]
            assert k >= n and lv != 0, (p, lv)
            s += self.coef(k - n, lv, n == 0, self.census)
            n = k + 1
        if blk.get("abort"):
            assert n > 0
            self.census["abort_" + ("intra" if intra else "inter")] += 1
            return s + self.coef(64 - n, 1, False, self.census, force_escape=True)
        return s + "10"

    def slice(self, row, q, mbs):
        st = {"dc": [128, 128, 128], "mv": (0, 0), "q": q}
        s = _b(q, 5) + "0"
        addr = row * 22 - 1
        for i, mb in enumerate(mbs):
            inc = 1 if i == 0 else mb.get("skip", 0) + 1
            assert i > 0 or not mb.get("skip")
            s += self.address(inc, i == 0, self.census)
            if inc > 1:
                st["dc"], st["mv"] = [128, 128, 128], (0, 0)
            addr += inc
            s += self._macroblock(mb, st, addr % 22, addr // 22)
        if "0" * 23 in s:
            raise RuntimeError("start-code emulation in a slice of row %d" % row)
        self.start_code(row + 1)
        self.put(s)
        self.census["slices"] += 1

    def _macroblock(self, mb, st, mx, my):
        intra = mb["intra"]
        blocks = mb["blocks"]
        cbp = sum(32 >> b for b in range(6) if blocks[b] is not None)
        if intra:
            assert cbp == 63
            mb_type = 0x01
        else:
            mb_type = (0x08 if mb.get("mv") is not None else 0) | (0x02 if cbp else 0)
            assert mb_type
        if mb.get("q") is not None:
            assert intra or cbp
            mb_type |= 0x10
        s = (sc.TYPE_I if self.ptype == 1 else sc.TYPE_P)[mb_type]
        if mb_type & 0x10:
            st["q"] = mb["q"]
            s += _b(mb["q"], 5)
        if intra:
            st["mv"] = (0, 0)
        else:
            st["dc"] = [128, 128, 128]
            if mb_type & 0x08:
                t = mb["mv"]
                h, v = t[0] << self.fp, t[1] << self.fp
                assert self.window_ok(mx, my, h, v), (mx, my, t)
                s += self.mv_component(st["mv"][0], t[0], self.census) + self.mv_component(st["mv"][1], t[1], self.census)
                st["mv"] = t
            else:
                st["mv"] = (0, 0)
            if mb_type & 0x02:
                s += sc.CBP[cbp]
        for b in range(6):
            blk = blocks[b]
            if blk is None:
                continue
            if intra:
                comp = 0 if b < 4 else b - 3
                diff = blk["dc"] - st["dc"][comp]
                assert -255 <= diff <= 255, (blk["dc"], st["dc"][comp])
                size = abs(diff).bit_length()
                s += (sc.LUMA_DC if b < 4 else sc.CHROMA_DC)[size]
                if size:
                    s += _b(diff if diff > 0 else diff + (1 << size) - 1, size)
                st["dc"][comp] = blk["dc"]
            s += self._coefs(blk, intra)
        return s

    def result(self):
        es = self.es()
        return es, np.array(self.pic_off + [es.size], dtype=np.uint32), self.census


def _flat_i_picture(w, value_of):
    """an I picture of DC-only macroblocks: value_of(mx, my) -> DC of all six blocks (reached from 128 within one step)"""
    w.start_picture(1)
    for row in range(12):
        w.slice(row, 8, [dict(intra=True, blocks=[{"dc": value_of(mx, row)} for _ in range(6)]) for mx in range(22)])


class _IntraFill:
    """Intra macroblocks from queues of wanted blocks per component (luma, Cr, Cb): a block whose DC is out of reach of
    the predictor is preceded by DC-only walker blocks in +-255 steps; an empty queue fills with DC-only blocks"""

    def __init__(self, luma, cr, cb):
        self.q = [list(luma), list(cr), list(cb)]

    def empty(self):
        return not any(self.q)

    def slice_mbs(self, n):
        pred, out = [128, 128, 128], []
        for _ in range(n):
            blocks = []
            for b in range(6):
                comp = 0 if b < 4 else b - 3
                q = self.q[comp]
                if q and abs(q[0]["dc"] - pred[comp]) <= 255:
                    blk = q.pop(0)
                elif q:
                    blk = {"dc": pred[comp] + max(-255, min(255, q[0]["dc"] - pred[comp]))}
                else:
                    blk = {"dc": pred[comp]}
                pred[comp] = blk["dc"]
                blocks.append(blk)
            out.append(dict(intra=True, blocks=blocks))
        return out


def _intra_pictures(w, fill, q):
    """I pictures of one slice per row until the fill is empty"""
    while not fill.empty():
        w.start_picture(1)
        for row in range(12):
            w.slice(row, q, fill.slice_mbs(22))
            if fill.empty():
                break


def _non_intra_picture(w, blocks, q):
    """a P picture of coded macroblocks without motion (prediction = the co-sited reference bytes), six of `blocks`
    per macroblock in raster order from (0, 0)"""
    w.start_picture(2)
    mbs = [dict(intra=False, blocks=(blocks[i:i + 6] + [None] * 6)[:6]) for i in range(0, len(blocks), 6)]
    for row in range(0, len(mbs), 22):
        w.slice(row // 22, q, mbs[row:row + 22])


# ---- a. basis sweep ---------------------------------------------------------------------------------------------------
def case_basis(extreme):
    w = Writer([255] * 64, [255] * 64) if extreme else Writer()
    c = w.census
    if extreme:
        levels, q = [255, -255], 31
    else:
        levels, q = [1, -1, 3, -3], 2
    # non-intra over a flat 128 reference: each position alone, and position 0 plus each other position
    _flat_i_picture(w, lambda mx, my: 128)
    blocks = []
    for p in range(64):
        for lv in levels:
            blocks.append({"coefs": [(p, lv)]})
            v = dequant(lv, q, w.mat[1][p], False)
            c["inter_pos%d_%s" % (p, "max" if v == 2047 else "min" if v == -2048 else "small")] += 1
    for p in range(1, 64):
        for lv in levels[:2]:
            blocks.append({"coefs": [(0, lv), (p, -lv)]})
            c["inter_pos0_plus%d" % p] += 1
    _non_intra_picture(w, blocks, q)
    # intra: DC only, and the DC plus each position
    luma, chroma = [], []
    for p in range(1, 64):
        for lv in levels:
            v = dequant(lv, q, w.mat[0][p], True)
            (luma if (p + lv) % 3 else chroma).append({"dc": 128 + lv, "coefs": [(p, lv)]})
            c["intra_pos%d_%s" % (p, "max" if v == 2047 else "min" if v == -2048 else "small")] += 1
    for dc in (0, 128, 248, 255):
        luma.append({"dc": dc})
        chroma.append({"dc": dc})
        c["intra_dc_only"] += 2
    _intra_pictures(w, _IntraFill(luma, chroma[::2], chroma[1::2]), q)
    return w.result()


# ---- b. exact domain edges ---------------------------------------------------------------------------------------------
EDGE_TARGETS = (-256, -1, 0, 248, 249, 511)
EDGE_PREDS = (0, 248, 255)


def _edge_intra_blocks(c):
    """DC + one AC coefficient, the DC chosen so that the block's minimum (targets <= 0) or maximum (targets >= 248) is
    exactly the target"""
    out = []
    for t in EDGE_TARGETS:
        for p, lv in ((1, 2), (9, -3), (18, 1), (63, 5)):
            a = samples({"coefs": [(p, lv)]}, 4, INTRA_Q, True)
            dc = t - (int(a.min()) if t <= 0 else int(a.max()))
            s = a + dc
            assert (s.min() == t if t <= 0 else s.max() == t) and s.min() >= -256 and s.max() <= 511
            out.append({"dc": dc, "coefs": [(p, lv)]})
            c["intra_edge_%d" % t] += 1
    return out


def _edge_inter_block(pred, t):
    """a non-intra block (position 0 and one more, shared quantiser, flat matrix 16) whose samples over a flat
    prediction `pred` reach exactly `t` at their minimum (t <= 0) or maximum, all inside [-256, 511]: -> (q, block)"""
    for q in range(1, 32):
        vals = {}
        for lv in range(-255, 256):
            if lv:
                vals.setdefault(dequant(lv, q, 16, False), lv)
        for p in (1, 8, 9, 2, 16, 10):
            for l1 in sorted(vals.values(), key=abs):
                b = np.zeros(64, dtype=np.int64)
                b[p] = dequant(l1, q, 16, False) * PRESCALE[p]
                a = idct(b)
                anchor = int(a.min()) if t <= 0 else int(a.max())
                need = t - pred - anchor                       # wanted DC term, dc = (32 v0 + rounding) >> 8
                for v0, l0 in vals.items():
                    if (v0 * 32 + 128) >> 8 != need and abs(((v0 * 32 + 128) >> 8) - need) > 1:
                        continue
                    s = samples({"coefs": [(0, l0), (p, l1)]}, q, [16] * 64, False) + pred
                    if (s.min() == t if t <= 0 else s.max() == t) and s.min() >= -256 and s.max() <= 511:
                        return q, {"coefs": [(0, l0), (p, l1)]}
    raise RuntimeError("no block reaches %d over %d" % (t, pred))


def case_edges():
    w = Writer()
    c = w.census
    fill = _IntraFill(_edge_intra_blocks(c), [], [])
    fill.q[1] = [dict(b) for b in fill.q[0][::2]]
    fill.q[2] = [dict(b) for b in fill.q[0][1::2]]
    _intra_pictures(w, fill, 4)
    # reference: rows 0-3 flat 0, rows 4-7 flat 248, rows 8-11 flat 255
    _flat_i_picture(w, lambda mx, my: EDGE_PREDS[my // 4])
    w.start_picture(2)
    for band, pred in enumerate(EDGE_PREDS):
        mbs = []
        for t in EDGE_TARGETS:
            q, blk = _edge_inter_block(pred, t)
            mbs.append(dict(intra=False, q=q, blocks=[blk] * 6))
            c["inter_edge_%d_over_%d" % (t, pred)] += 1
        w.slice(band * 4, 8, mbs)
    return w.result()


# ---- c. worst-case sign patterns --------------------------------------------------------------------------------------
def _sign_block(o, sign, intra, dc=128):
    coefs = [(i, 255 * sign * (1 if L[o][i] > 0 else -1)) for i in range(1 if intra else 0, 64) if L[o][i] != 0]
    blk = {"coefs": coefs}
    if intra:
        blk["dc"] = dc
    return blk


def case_signs(intra):
    w = Writer([255] * 64, [255] * 64)
    c = w.census
    if intra:
        luma = [_sign_block(o, s, True) for o in range(64) for s in (1, -1)]
        for o in range(64):
            c["intra_sign_sample%d" % o] += 2
        chroma = [_sign_block(o, s, True) for o in (0, 7, 27, 63) for s in (1, -1)]
        _intra_pictures(w, _IntraFill(luma, chroma, chroma[::-1]), 31)
        return w.result()
    # reference: block b of macroblock m flat at byte (6 m + b) mod 256, so the 258 blocks of the first 43
    # macroblocks lie over every byte (those above 248 through Q7)
    _flat_blocks = lambda mx, my, b: (6 * (my * 22 + mx) + b) % 256
    w.start_picture(1)
    for row in range(12):
        w.slice(row, 8, [dict(intra=True, blocks=[{"dc": _flat_blocks(mx, row, b)} for b in range(6)]) for mx in range(22)])
    blocks, preds = [], set()
    for j in range(258):
        o, s = (j // 2) % 64, 1 if j % 2 == 0 else -1
        blocks.append(_sign_block(o, s, False))
        preds.add(_flat_blocks(j // 6 % 22, j // 6 // 22, j % 6))
        c["inter_sign_sample%d" % o] += 1
    c["pred_bytes"] = len(preds)
    _non_intra_picture(w, blocks, 31)
    return w.result()


# ---- d. large intra DC predictors -------------------------------------------------------------------------------------
def _dc_levels(sign, plateaus=(16000, 18500, 20000), top=36000, hold=12):
    """DC levels in +-255 steps from 128, holding `hold` blocks at each plateau and past +-32,768"""
    out, v = [], 128
    for target in list(plateaus) + [top]:
        while abs(v) < target:
            v += 255 * sign
            out.append(v)
        out += [v] * hold
    return out


def _dc_blocks(levels, c, plane):
    """each level with a DC-only block, one small AC coefficient and a saturated AC sign pattern, in turn"""
    out = []
    for i, dc in enumerate(levels):
        kind = ("dc_only", "ac_small", "ac_saturated")[i % 3]
        if kind == "dc_only":
            blk = {"dc": dc}
        elif kind == "ac_small":
            blk = {"dc": dc, "coefs": [(1 + i % 9, 1 if i % 2 else -1)]}
        else:
            blk = _sign_block(i % 64, 1 if i % 2 else -1, True, dc)
        band = "ge32768" if dc >= 32768 else "le-32768" if dc <= -32768 else "16k_20k" if 16000 <= abs(dc) <= 20500 else "other"
        c["%s_dc_%s_%s" % (plane, band, kind)] += 1
        out.append(blk)
    return out


def case_dc(span):
    """I pictures of slices `span` rows long whose luma (span 3) or chroma (span 6) DC predictors climb past +32,768 in
    one slice and fall below -32,768 in the next"""
    w = Writer([255] * 64)
    c = w.census
    per = 22 * span
    for sign in (1, -1):
        if span == 3:
            luma, chroma = _dc_blocks(_dc_levels(sign), c, "luma"), _dc_blocks(_dc_levels(sign, top=15000)[:per], c, "chroma")
        else:
            luma, chroma = _dc_blocks(_dc_levels(sign, top=20000)[:4 * per], c, "luma"), _dc_blocks(_dc_levels(sign, (16000,), top=33500, hold=0)[:per], c, "chroma")
        assert len(luma) <= 4 * per and len(chroma) <= per
        fill = _IntraFill(luma, chroma, [dict(b) for b in chroma])
        if sign == 1:
            w.start_picture(1)
        w.slice(0 if sign == 1 else span, 31, fill.slice_mbs(per))
    return w.result()


# ---- e. prediction sweep ----------------------------------------------------------------------------------------------
def _reference_picture(w, rng, c):
    """an I picture over every byte value: textured blocks (clamped to 0..248) and DC-only blocks at 249..255 and at DCs
    outside 0..255 (Q7 keeps their low byte)"""
    w.start_picture(1)
    special = list(range(249, 256)) + list(range(256, 300, 3)) + list(range(-40, 0, 3))
    for row in range(12):
        pred, mbs = [128, 128, 128], []
        for mx in range(22):
            blocks = []
            for b in range(6):
                comp = 0 if b < 4 else b - 3
                k = rng.int(0, 9)
                if k < 4:
                    want = rng.pick(special)
                    dc = pred[comp] + max(-255, min(255, want - pred[comp]))
                    blk = {"dc": dc}
                    c["ref_dc_byte_%d" % (dc & 255)] += 1
                else:
                    dc = pred[comp] + max(-255, min(255, rng.int(20, 228) - pred[comp]))
                    blk = {"dc": dc, "coefs": [(rng.int(1, 63), rng.pick([-3, -2, -1, 1, 2, 3])) for _ in range(rng.int(2, 6))]}
                    seen = {}
                    for p, lv in blk["coefs"]:
                        seen[p] = lv
                    blk["coefs"] = sorted(seen.items())
                pred[comp] = dc
                blocks.append(blk)
            mbs.append(dict(intra=True, blocks=blocks))
        w.slice(row, 4, mbs)


EDGES = {"left": lambda hx, hy: (hx >> 1) == 0, "top": lambda hx, hy: (hy >> 1) == 0,
         "right": lambda hx, hy: (hx >> 1) + 16 + (hx & 1) == 352, "bottom": lambda hx, hy: (hy >> 1) + 16 + (hy & 1) == 192}


def _edge_vector(mx, my, edge, xh, yh):
    """absolute half-pel window position (hx, hy) of macroblock (mx, my) touching `edge` with half-pel flags (xh, yh)"""
    hx, hy = mx * 32 + xh, my * 32 + yh
    if edge == "left":
        hx = xh
    elif edge == "right":
        hx = 2 * (336 - xh) + xh
    elif edge == "top":
        hy = yh
    else:
        hy = 2 * (176 - yh) + yh
    return hx, hy


def _residual(kind, k):
    if kind == 0:
        return [None] * 6
    if kind == 1:
        return [{"coefs": [((k + 3 * b) % 64, 1 if (k + b) % 2 else -1)]} for b in range(6)]
    return [{"coefs": [(0, 33 if b % 2 == 0 else -33)]} for b in range(6)]    # +-2048 -> DC term +255 / -256


def case_pred(kind, full_pel=False):
    """I, P, I, P, ... : the P macroblocks' vectors walk through the (hx mod 32, hy mod 32) alignments (even ones for
    full-pel pictures), the first and last columns and rows put windows on the frame edges"""
    w = Writer()
    c = w.census
    rng = sc.Rng(0xB10C + kind)
    f_code = 3                                                  # vectors -64..63 half pels
    aligns = [(a, b) for b in range(0, 32, 2 if full_pel else 1) for a in range(0, 32, 2 if full_pel else 1)]
    edge_jobs = [(e, xh, yh) for e in EDGES for xh in ((0,) if full_pel else (0, 1)) for yh in ((0,) if full_pel else (0, 1))]
    k = 0
    while aligns or edge_jobs:
        _reference_picture(w, rng, c)
        w.start_picture(2, fp=1 if full_pel else 0, f_code=f_code)
        for row in range(12):
            mbs = []
            for mx in range(22):
                hxy = None
                for j, (e, xh, yh) in enumerate(edge_jobs):
                    hx, hy = _edge_vector(mx, row, e, xh, yh)
                    h, v = hx - mx * 32, hy - row * 32
                    if -64 <= h <= 63 and -64 <= v <= 63 and w.window_ok(mx, row, h, v):
                        hxy = (h, v)
                        del edge_jobs[j]
                        break
                if hxy is None:
                    for j, (a, b) in enumerate(aligns):
                        opts = [(h, v) for h in (a, a - 32, a + 32, a - 64) for v in (b, b - 32, b + 32, b - 64)
                                if -64 <= h <= 63 and -64 <= v <= 63 and w.window_ok(mx, row, h, v)]
                        if opts:
                            hxy = opts[(mx + row) % len(opts)]
                            del aligns[j]
                            break
                if hxy is None:
                    hxy = (2 * rng.int(-8, 8), 2 * rng.int(-8, 8)) if full_pel else (rng.int(-16, 16), rng.int(-16, 16))
                    if not w.window_ok(mx, row, *hxy):
                        hxy = (0, 0)
                h, v = hxy
                hx, hy = mx * 32 + h, row * 32 + v
                c["luma_align_%d_%d" % (hx % 32, hy % 32)] += 1
                c["chroma_align_%d_%d" % ((hx >> 1) % 16, (hy >> 1) % 16)] += 1
                c["negative_vector"] += h < 0 or v < 0
                for e, f in EDGES.items():
                    if f(hx, hy):
                        c["edge_%s_xy%d" % (e, (hx & 1) | (hy & 1) << 1)] += 1
                mv = (h >> 1, v >> 1) if full_pel else (h, v)
                mbs.append(dict(intra=False, mv=mv, q=31 if kind == 2 else None, blocks=_residual(kind, k)))
                k += 1
            w.slice(row, 4, mbs)
    return w.result()


# ---- f. warp pairs ----------------------------------------------------------------------------------------------------
KINDS = ["none", "skip", "intra_dc", "intra_ac", "ni_luma", "ni_chroma", "ni_one", "ni_all", "mc_cbp0", "aborted"]
CODED = KINDS[2:]
# the pairs a stream can hold: a slice starts at column 0 and ends on a coded macroblock, a skip run ends on one
PAIRS = [(a, b) for a in CODED + ["skip"] for b in CODED + ["skip"]] + [(a, "none") for a in CODED] + [("none", "none")]


def _mb_of_kind(kind, mx, my, k):
    small = lambda b: {"coefs": [((k + 5 * b) % 63 + 1, 1 if (k + b) % 2 else -1)]}
    if kind in ("intra_dc", "intra_ac"):
        return dict(intra=True, blocks=[{"dc": 128 + (k % 7) * 10, **({"coefs": [(1 + b, 2)]} if kind == "intra_ac" else {})} for b in range(6)])
    h = 3 if mx < 21 else -3
    v = 1 if my < 11 else -1
    coded = {"ni_luma": (0, 1, 2, 3), "ni_chroma": (4, 5), "ni_one": (3,), "ni_all": range(6), "mc_cbp0": (), "aborted": range(6)}[kind]
    blocks = [small(b) if b in coded else None for b in range(6)]
    if kind == "aborted":
        blocks[2] = dict(blocks[2], abort=True)
    return dict(intra=False, mv=(h, v), blocks=blocks)


def case_pairs():
    w = Writer()
    c = w.census
    _reference_picture(w, sc.Rng(0xFA12), Counter())
    todo = [p for p in PAIRS if p != ("none", "none")]
    w.start_picture(2)
    for row in range(12):
        kinds = []
        for j in range(11):
            ok = [p for p in todo if (j > 0 or p[0] != "skip") and (j < 10 or p[1] != "skip")
                  and (p[1] != "none" or j == 9 or not any(q[1] != "none" for q in todo))
                  and (p[1] == "none" or j < 9 or not any(q[1] == "none" for q in todo) or j == 10)]
            if j == 9 and any(p[1] == "none" for p in ok):
                ok = [p for p in ok if p[1] == "none"]
            p = ok[0] if ok else ("ni_all", "intra_dc")
            if p in todo:
                todo.remove(p)
            kinds += list(p)
            if p[1] == "none":
                kinds += ["none"] * (22 - len(kinds))
                break
        mbs, skip = [], 0
        for mx, kind in enumerate(kinds):
            if kind == "none":
                break
            if kind == "skip":
                skip += 1
                continue
            mb = _mb_of_kind(kind, mx, row, len(mbs) + 22 * row)
            if skip:
                mb["skip"] = skip
                c["skip_run_ends_half%d" % (mx & 1)] += 1
            skip = 0
            mbs.append(mb)
        assert not skip
        for j in range(11):
            c["pair_%s_%s" % (kinds[2 * j], kinds[2 * j + 1])] += 1
        w.slice(row, 6, mbs)
        if not todo:
            break
    assert not todo, todo
    return w.result()


# ---- the case list ----------------------------------------------------------------------------------------------------
CASES = {
    "basis_small": lambda: case_basis(False),
    "basis_extreme": lambda: case_basis(True),
    "edges": case_edges,
    "signs_inter": lambda: case_signs(False),
    "signs_intra": lambda: case_signs(True),
    "dc_luma": lambda: case_dc(3),
    "dc_chroma": lambda: case_dc(6),
    "pred_none": lambda: case_pred(0),
    "pred_small": lambda: case_pred(1),
    "pred_clamp": lambda: case_pred(2),
    "pred_fullpel": lambda: case_pred(1, full_pel=True),
    "pairs": case_pairs,
}
# Outside the reference's defined domain (samples leave [-256, 511]): compared with the restatement only.
UNPINNED = ["basis_extreme", "signs_inter", "signs_intra", "dc_luma", "dc_chroma"]


def case_names():
    return list(CASES)


def make(name):
    """-> (es uint8 array, picture offsets uint32[n+1], census Counter)"""
    return CASES[name]()
