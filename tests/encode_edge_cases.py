"""tests/encode_edge_cases.py — titles whose encoder decisions are chosen, not drawn, a census of what their codes reach, and a
model of what a decoder must make of the decisions.

The encoder tests of tests/encode_cases.py and tests/rate_cases.py run natural and synthetic pictures; nothing says which syntax
they reach. The titles here are built through the restatement so that its decisions land on the edges of the slice syntax:

  intra_dc      flat blocks whose DC differences take every size 0..8 in both DC tables with both signs, carried across
                macroblocks (DC-only intra blocks: the reference's unclamped copy, Q7)
  intra_q1      AC levels at index 1 (run 0) of +-40 / 41 (table / 8-bit escape), +-127 / 128 (8- / 16-bit escape), +-255 and
                clamped to 255, at quantiser 1
  intra_q8      every run 0..31 at its table's largest level and one beyond it (an escape), both signs; runs 32..62, and a
                block whose only AC coefficient is zig-zag 63
  intra_q31     the table boundaries reachable at quantiser 31, and zig-zag 63 alone
  p_vectors     a P picture whose vectors walk every motion code -16..15 with wrapped deltas, between first / last
                macroblocks of type 0x08 with vector (0, 0)
  p_blocks      every coded block pattern 1..63 (types 0x02 and 0x0A), non-intra first coefficients of +-1 ("1s"), +-2 and
                escapes, and every ordered pair of skip, 0x01, 0x02, 0x08 and 0x0A neighbours
  p_skips       every address increment 1..21
  domain_q*     intra blocks from the domain search below, tiled

A P picture is predicted from the restatement's reconstruction R of the picture before (a textured, mid-range I picture): each
macroblock is mc(R, target vector) plus a designed residual, or a flat patch far from R that the mode rule makes intra.

census() reads what each title reached from the restatement's own code arrays (trick_cases.slice_codes in its MB_SLOTS layout) and
decisions, not from the builders' intentions: if the search picks another vector than a builder aimed for, the census shows it.
model_decode() computes the pictures a decoder must produce from the decisions alone (vectors, modes, skips and levels), without
reading the bitstream; equal to the oracle's decode of the file, it shows the codes mean what the encoder decided.
domain_search() is a seeded, bounded hill climb for single blocks whose pre-clamp decode moves furthest toward the ends of the
reference's clamp table (-256..511): a search, not a bound."""
import functools

import numpy as np

from tests import block_cases as bc
from tests import encode_cases as ec
from tests import trick_cases as tc

W, H = ec.W, ec.H
ZZ = tc.ZIGZAG
PRESCALE = np.array(bc.PRESCALE, np.int64)
W_INTRA = tc.INTRA_Q[ZZ]                       # intra weight of each zig-zag index
TABLE_MAX = [int(max(a for a in range(1, 256) if tc.AC_LEN[r, a])) for r in range(32)]   # the run / level table's largest level per run
P_PARAMS = dict(qscale_i=2, qscale_p=4)        # the P titles: a detailed reference, a quantiser where a flat residual d has level d


# -- pictures from blocks -----------------------------------------------------------------------------------------------------------
def from_blocks(B):
    """[264, 6, 8, 8] blocks in macroblock address order -> an I420 picture (the inverse of encode_cases.mb_blocks)"""
    B = np.asarray(B, np.int64)
    assert B.min() >= 0 and B.max() <= 255, (B.min(), B.max())
    y = B[:, :4].reshape(12, 22, 2, 2, 8, 8).transpose(0, 2, 4, 1, 3, 5).reshape(H, W)
    c = [B[:, k].reshape(12, 22, 8, 8).transpose(0, 2, 1, 3).reshape(H // 2, W // 2) for k in (4, 5)]
    return np.concatenate([y.ravel()] + [x.ravel() for x in c]).astype(np.uint8)


def _basis(i):
    """the orthonormal DCT basis function of zig-zag index i, [8, 8]"""
    u, v = divmod(int(ZZ[i]), 8)
    c = lambda k: np.sqrt(1 / 8) if k == 0 else 0.5
    n = np.arange(8)
    return c(u) * c(v) * np.outer(np.cos((2 * n + 1) * u * np.pi / 16), np.cos((2 * n + 1) * v * np.pi / 16))


def tuned(i, level, q, base=128):
    """an intra 8 x 8 block base + A basis_i whose level at zig-zag index i at quantiser q is `level` (a |level| above 255 asks
    for one that quantise clamps to 255), A tuned against trick_cases.quantise(trick_cases.fdct(...)); None when out of reach"""
    a = abs(level)
    amp = np.sign(level) * (a + 0.5) * q * W_INTRA[i] / 8 * np.linspace(0.8, 1.25, 512)
    blk = np.rint(amp[:, None, None] * _basis(i)).astype(np.int64) + base
    ok = (blk.min(axis=(1, 2)) >= 0) & (blk.max(axis=(1, 2)) <= 255)
    F = tc.fdct(blk).reshape(-1, 64)[:, ZZ]
    raw = (2 * 8 * np.abs(F[:, i]) + W_INTRA[i] * q) // (2 * W_INTRA[i] * q)
    got = np.where(a > 255, raw > 255, raw == a) & (np.sign(F[:, i]) == np.sign(level))
    k = np.flatnonzero(ok & got)
    return blk[k[len(k) // 2]] if len(k) else None


def _fill(blocks, filler=128):
    """blocks [..., 8, 8] into a picture's 1,584 block slots in order, the rest flat `filler`"""
    B = np.full((264 * 6, 8, 8), filler, np.int64)
    blocks = list(blocks)
    assert len(blocks) <= 264 * 6
    if blocks:
        B[:len(blocks)] = np.stack(blocks)
    return from_blocks(B.reshape(264, 6, 8, 8))


# -- I pictures --------------------------------------------------------------------------------------------------------------------
def _dc_walk(n, rng, start=0):
    """n values 0..255 whose differences (from 128) take every DC size 0..8 with both signs, each at its smallest and largest
    magnitude (the list rotated by `start`), then random ones"""
    want = [0] + [s * m for k in range(1, 9) for s in (1, -1) for m in (1 << (k - 1), (1 << k) - 1)]
    want = want[start % len(want):] + want[:start % len(want)]
    out, c = [], 128
    while len(out) < n:
        if not want:
            want = [int(d) for d in rng.integers(-255, 256, 16)]
        d = next((d for d in want if 0 <= c + d <= 255), None)
        if d is None:                                   # step to where the first pending difference fits
            d0 = want[0]
            c = 255 - d0 if d0 > 0 else -d0
        else:
            want.remove(d)
            c += d
        out.append(c)
    return out


def intra_dc():
    """flat blocks: every row's luma and both chroma chains walk every DC size and sign"""
    rng = np.random.default_rng(11)
    B = np.zeros((12, 22, 6), np.int64)
    for row in range(12):
        B[row, :, :4] = np.array(_dc_walk(88, rng)).reshape(22, 4)
        B[row, :, 4] = _dc_walk(22, rng, 11 * row)
        B[row, :, 5] = _dc_walk(22, rng, 11 * row + 5)
    return from_blocks(np.broadcast_to(B.reshape(264, 6)[..., None, None], (264, 6, 8, 8)))


def _intra_targets(q):
    """(zig-zag index, level) targets of the intra_q* pictures"""
    if q == 1:
        return [(1, s * a) for a in (40, 41, 127, 128, 255, 300) for s in (1, -1)] + [(2, s * a) for a in (40, 41, 127, 128) for s in (1, -1)]
    out = [(r + 1, s * a) for r in range(32) for a in (TABLE_MAX[r], TABLE_MAX[r] + 1) for s in (1, -1)]
    return out + [(i, s * a) for i in range(33, 64) for a in (1, 2) for s in (1, -1)]


def intra_targets(q):
    """the I picture of intra_q<q>: one block per reachable target, each with DC 128"""
    blocks = [b for b in (tuned(i, lv, q) for i, lv in _intra_targets(q)) if b is not None]
    return _fill(blocks)


# -- P pictures --------------------------------------------------------------------------------------------------------------------
def reference(seed=3):
    """a textured, mid-range picture (luma 48..208): the I picture every P title predicts from"""
    y, cb, cr = ec.textured(seed, grain=14.0)
    mid = lambda p: np.rint(48 + np.clip(p, 0, 255) * 160 / 255).astype(np.int64)
    return np.concatenate([mid(y)[32:32 + H, 32:32 + W].ravel(), mid(cb)[16:16 + H // 2, 16:16 + W // 2].ravel(),
                           mid(cr)[16:16 + H // 2, 16:16 + W // 2].ravel()]).astype(np.uint8)


@functools.lru_cache(maxsize=None)
def _recon_reference(qscale_i):
    """the restatement's reconstruction R of reference() coded at qscale_i (the oracle's decode of it)"""
    from tests.oracle_lib import Oracle
    es = tc.encode_picture(reference(), qscale_i, tc.header_bytes(1, 2))
    return Oracle().decode_es(es, max_frames=1)[0]


def p_source(R, mbs):
    """the P picture of per-macroblock specs over reconstruction R: ("mc", h, v, residual [6, 8, 8] or None) is the prediction
    mc(R, h, v) plus the residual; ("intra", [6] values) is a flat patch per block"""
    h = np.array([m[1] if m[0] == "mc" else 0 for m in mbs])
    v = np.array([m[2] if m[0] == "mc" else 0 for m in mbs])
    assert ec.legal(ec._MX, ec._MY, h, v).all()
    B = ec.predictions(ec.planes(R), h, v).copy()
    for k, m in enumerate(mbs):
        if m[0] == "intra":
            B[k] = np.asarray(m[1])[:, None, None]
        elif m[3] is not None:
            B[k] = B[k] + m[3]
    return from_blocks(B)


def _flat_residual(values):
    """[6, 8, 8] residual of flat blocks"""
    return np.broadcast_to(np.asarray(values, np.int64)[:, None, None], (6, 8, 8)).copy()


def _residual63(level, q):
    """a non-intra residual block whose only level at quantiser q is `level` at zig-zag index 63"""
    for amp in np.linspace(1.0, 4.0, 61) * abs(level) * 2 * q:
        blk = np.rint(np.sign(level) * amp * _basis(63)).astype(np.int64)
        lv = ec.inter_levels(tc.fdct(blk), q)
        if lv[63] == level and not lv[:63].any():
            return blk
    raise AssertionError("no residual for level %d at zig-zag 63" % level)


def _wrap(x):
    return (x + 16) % 32 - 16


def p_vectors(R):
    """rows 1..10, columns 1..20: vectors whose deltas (with wraps) walk every motion code, the h and v walks independent;
    first and last macroblocks of each slice 0x08 with vector (0, 0), rows 0 and 11 skipped between them"""
    rng = np.random.default_rng(5)
    mbs = [("mc", 0, 0, None)] * 264
    qh, qv = [], []
    for row in range(1, 11):
        h = v = 0
        for mx in range(1, 21):
            if len(qh) < 8:
                qh += list(rng.permutation(32) - 16)
            if len(qv) < 8:
                qv += list(rng.permutation(32) - 16)
            # the next pending deltas that keep the vector inside -15..15 (the search reaches no -16) and not (0, 0)
            dh = next(d for d in qh if _wrap(h + d) != -16)
            dv = next((d for d in qv if _wrap(v + d) != -16 and (_wrap(h + dh), _wrap(v + d)) != (0, 0)), None)
            if dv is None:
                dv = 1 if _wrap(v + 1) != -16 else 2
            else:
                qv.remove(dv)
            qh.remove(dh)
            h, v = _wrap(h + dh), _wrap(v + dv)
            mbs[row * 22 + mx] = ("mc", int(h), int(v), None)
    return p_source(R, mbs)


_KINDS = ["skip", "intra", "0x02", "0x08", "0x0A"]


def _vector(rng, mx, row):
    """a random vector other than (0, 0), legal at macroblock (mx, row)"""
    vec = (0, 0)
    while vec == (0, 0):
        vec = (int(rng.integers(0 if mx == 0 else -12, (0 if mx == 21 else 12) + 1)),
               int(rng.integers(0 if row == 0 else -12, (0 if row == 11 else 12) + 1)))
    return vec


def p_blocks(R):
    """patterns 1..63 alternating between vector (0, 0) (0x02) and vectors (0x0A); first coefficients; kind pairs"""
    rng = np.random.default_rng(7)
    mbs = [None] * 264
    # rows 0..2: coded block patterns 1..63 (columns 1..21), luma residuals of level +-1..3, chroma escapes of +-41
    for c in range(1, 64):
        row, mx = (c - 1) // 21, (c - 1) % 21 + 1
        lv = [(1 + (c + b) % 3) * (1 if (c >> b) & 1 else -1) for b in range(4)] + [41 * (1 if c & 1 else -1), -41 * (1 if c & 2 else -1)]
        res = _flat_residual([lv[b] if c & (0x20 >> b) else 0 for b in range(6)])
        if c % 3 == 0 and c & 1:                    # block 5's only coefficient at zig-zag 63: run 63
            res[5] = _residual63(1 if c & 4 else -1, P_PARAMS["qscale_p"])
        vec = (0, 0) if c % 2 else _vector(rng, mx, row)
        mbs[row * 22 + mx] = ("mc", vec[0], vec[1], res)
    # rows 3..11: kinds, each next kind chosen to close a not-yet-seen ordered pair
    seen = set()
    for row in range(3, 12):
        prev = "start"
        for mx in range(22):
            options = [k for k in _KINDS if not (k == "skip" and mx in (0, 21))]
            fresh = [k for k in options if (prev, k) not in seen]
            kind = fresh[int(rng.integers(len(fresh)))] if fresh else options[int(rng.integers(len(options)))]
            seen.add((prev, kind))
            prev = kind
            vec = _vector(rng, mx, row)
            a = int(rng.integers(1, 3)) * (1 if rng.integers(2) else -1)
            res = _flat_residual([a, 0, 0, -a, 0, 41 if rng.integers(2) else -41])
            if kind == "skip":
                mbs[row * 22 + mx] = ("mc", 0, 0, None)
            elif kind == "intra":                   # one luma value far from R's 48..208, chroma anywhere: the mode rule's intra
                y = int(rng.choice([int(rng.integers(0, 24)), int(rng.integers(232, 256))]))
                mbs[row * 22 + mx] = ("intra", [y] * 4 + [int(x) for x in rng.integers(0, 256, 2)])
            elif kind == "0x02":
                mbs[row * 22 + mx] = ("mc", 0, 0, res)
            elif kind == "0x08":
                mbs[row * 22 + mx] = ("mc", vec[0], vec[1], None)
            else:
                mbs[row * 22 + mx] = ("mc", vec[0], vec[1], res)
    for k in range(264):
        if mbs[k] is None:
            mbs[k] = ("mc", 0, 0, None)
    return p_source(R, mbs)


def p_skips(R):
    """row r < 11: one 0x02 macroblock at column r + 1 between skip runs; row 11 all skipped between its first and last"""
    mbs = [("mc", 0, 0, None)] * 264
    for row in range(11):
        mbs[row * 22 + row + 1] = ("mc", 0, 0, _flat_residual([2, 0, 0, 0, 0, 0]))
    return p_source(R, mbs)


# -- the domain search ---------------------------------------------------------------------------------------------------------------
def _dequant(L, q, m, intra):
    """block_cases.dequant over arrays (Q2 and saturation); m broadcasts as the weight of each coefficient"""
    v = 2 * L + (0 if intra else np.sign(L))
    t = v * q * m
    v = np.sign(t) * (np.abs(t) // 16)
    v = np.where((v & 1) == 0, v - np.where(v > 0, 1, -1), v)
    return np.clip(v, -2048, 2047)


def block_samples(levels, q, intra, pred=0):
    """zig-zag levels [..., 64] -> the reference's samples [..., 64] (raster) before its clamp: DC-only blocks by Q5 / Q7 (an intra
    one is its DC level, copied without the clamp), the rest through the IDCT; non-intra ones over `pred`"""
    L = np.asarray(levels, np.int64)
    m = W_INTRA if intra else 16
    c = np.where(L != 0, _dequant(L, q, m, intra) * PRESCALE[ZZ], 0)
    if intra:
        c[..., 0] = L[..., 0] << 8
    b = np.zeros(L.shape, np.int64)
    b[..., ZZ] = c
    only_dc = ~(L[..., 1:] != 0).any(axis=-1, keepdims=True)
    dc_value = L[..., :1] if intra else (b[..., :1] >> 8)
    return np.where(only_dc, dc_value, bc.idct(b)) + pred


def _block_eval(x, q, intra, pred):
    """pixel blocks [n, 8, 8] -> pre-clamp samples [n, 64] of the encoder's coding at q and the decode"""
    if intra:
        return block_samples(tc.quantise(tc.fdct(x), q), q, True)
    return block_samples(ec.inter_levels(tc.fdct(x - pred), q), q, False, pred)


def domain_search(q, intra, pred=0, toward=511, seed=0, chains=64, steps=400):
    """-> (most extreme pre-clamp sample toward `toward`, blocks evaluated, the block that reached it): a hill climb from random
    blocks, each step setting 1..3 pixels of every chain to 0, 255 or a random value and keeping the change unless it is worse"""
    rng = np.random.default_rng(seed)
    sign = 1 if toward > 0 else -1
    x = rng.integers(0, 256, (chains, 8, 8))
    score = lambda s: sign * s.max(axis=-1) if sign > 0 else -s.min(axis=-1)
    cur = score(_block_eval(x, q, intra, pred))
    n = chains
    for _ in range(steps):
        y = x.copy()
        for _ in range(int(rng.integers(1, 4))):
            i, j = rng.integers(0, 8, (2, chains))
            pick = rng.integers(0, 3, chains)
            y[np.arange(chains), i, j] = np.where(pick == 0, 0, np.where(pick == 1, 255, rng.integers(0, 256, chains)))
        s = score(_block_eval(y, q, intra, pred))
        n += chains
        keep = s >= cur
        x[keep], cur[keep] = y[keep], s[keep]
    best = int(np.argmax(cur))
    return sign * int(cur[best]), n, x[best]


DOMAIN_RUNS = [(q, True, 0) for q in (16, 31)] + [(q, False, p) for q in (16, 31) for p in (0, 248)]


@functools.lru_cache(maxsize=None)
def domain_results():
    """{(q, intra, pred, toward): (sample, blocks evaluated, block)} of every domain search"""
    return {(q, intra, p, t): domain_search(q, intra, p, t, seed=q * 7 + p + (t > 0)) for q, intra, p in DOMAIN_RUNS for t in (-256, 511)}


def domain_picture(q):
    """an I picture tiled with the intra blocks the domain search found at q"""
    blocks = [b for (qq, intra, _, _), (_, _, b) in sorted(domain_results().items()) if qq == q and intra]
    return _fill(blocks * (264 * 6 // len(blocks)))


# -- the directed titles -------------------------------------------------------------------------------------------------------------
NAMES = ["intra_dc", "intra_q1", "intra_q8", "intra_q31", "p_vectors", "p_blocks", "p_skips", "domain_q16", "domain_q31"]


@functools.lru_cache(maxsize=None)
def title(name):
    """-> (pictures uint8 [n, PICTURE_BYTES], encode parameters): the directed title `name`, coded with one GOP"""
    if name == "intra_dc":
        return np.stack([intra_dc()]), dict(qscale_i=8, qscale_p=8)
    if name.startswith("intra_q"):
        q = int(name[7:])
        return np.stack([intra_targets(q)]), dict(qscale_i=q, qscale_p=q)
    if name.startswith("domain_q"):
        q = int(name[8:])
        return np.stack([domain_picture(q)]), dict(qscale_i=q, qscale_p=q)
    R = _recon_reference(P_PARAMS["qscale_i"])
    build = {"p_vectors": p_vectors, "p_blocks": p_blocks, "p_skips": p_skips}[name]
    return np.stack([reference(), build(R)]), dict(P_PARAMS)


# -- the decisions, the census and the model ------------------------------------------------------------------------------------------
def encode(pictures, oracle, rate=False, **params):
    """encode_cases.encode_title (rate_cases.encode_title with rate) of a title, and the restatement's decisions for every picture:
    -> (the encoder's result, [dict(p, q, intra, h, v, skipped [264], levels [264, 6, 64], codes (values, lengths) [12, slots], F)]).
    Each P picture's analysis is the one the encoder made (encode_cases.analyse, recorded as it runs)."""
    from tests import rate_cases as rc
    seen, analyse = [], ec.analyse

    def recording(*a, **k):
        seen.append(analyse(*a, **k))
        return seen[-1]
    ec.analyse = recording
    try:
        res = rc.encode_title(pictures, oracle, **params) if rate else ec.encode_title(pictures, oracle, **params)
    finally:
        ec.analyse = analyse
    p = dict(ec.DEFAULT_PARAMS, **(rc.RATE_DEFAULTS if rate else {}))
    p.update(params)
    pictures = np.asarray(pictures).reshape(-1, ec.PICTURE_BYTES)
    ans = iter(seen)
    out = []
    for k, pic in enumerate(pictures):
        ipic = k % p["gop"] == 0
        q = res[3][k] if rate else p["qscale_i" if ipic else "qscale_p"]
        fb = q == 0
        q = p["qmax"] if fb else q
        if ipic:
            F = tc.fdct(tc.picture_blocks(pic))
            codes = tc.i_codes(F, [q], [fb])
            L = tc.quantise(F, q).reshape(264, 6, 64)
            if fb:
                L[..., 1:] = 0
            d = dict(p=False, intra=np.ones(264, bool), h=np.zeros(264, np.int64), v=np.zeros(264, np.int64), levels=L,
                     F=F.reshape(264, 6, 8, 8))
        else:
            an = next(ans)
            codes = ec.p_codes(an, [q], [fb])
            z = np.zeros(264, np.int64)
            d = dict(p=True, intra=an["intra"] & (not fb), h=z if fb else an["h"], v=z if fb else an["v"],
                     levels=0 * ec.p_levels(an, q) if fb else ec.p_levels(an, q), F=an["Fi"])
        d.update(q=q, codes=(codes[0][0], codes[1][0]), skipped=codes[1][0, :, 2::tc.MB_SLOTS].ravel() == 0)
        out.append(d)
    return res, out


def model_picture(d, ref):
    """the picture (I420) a decoder must produce from one picture's decisions d, predicting from ref (I420, the model's previous
    picture): skipped macroblocks copy, the rest predict with encode_cases.predictions (chroma by Q3); coded blocks add the
    reference's dequantisation and IDCT (DC-only blocks by Q5, intra ones by Q7); samples clamp to 0..248 (Q1)"""
    intra = d["intra"]
    L = d["levels"]
    if d["p"]:
        h, v = np.where(d["skipped"], 0, d["h"]), np.where(d["skipped"], 0, d["v"])
        pred = ec.predictions(ec.planes(ref), h, v).reshape(264, 6, 64)
    else:
        pred = np.zeros((264, 6, 64), np.int64)
    coded = intra[:, None] | (L != 0).any(axis=-1)
    s_intra = block_samples(L, d["q"], True)
    s_inter = block_samples(L, d["q"], False, pred)
    only_dc = ~(L[..., 1:] != 0).any(axis=-1, keepdims=True)
    s_intra = np.where(only_dc, s_intra, np.clip(s_intra, 0, 248))              # Q7: an intra DC-only block is not clamped
    out = np.where(intra[:, None, None], s_intra, np.where(coded[..., None], np.clip(s_inter, 0, 248), pred))
    return from_blocks(out.reshape(264, 6, 8, 8))


def model_decode(decs):
    """the decoder's pictures of a title from its decisions, each P picture predicted from the model's own previous one"""
    out = []
    for d in decs:
        out.append(model_picture(d, out[-1] if out else None))
    return np.stack(out)


def _inverse(table):
    return {(int(c, 2), len(c)): v for v, c in table.items()}


_MBA_INV, _MV_INV, _CBP_INV = _inverse(tc.MBA), _inverse(tc.MV), _inverse(tc.CBP)
_TYPE_INV = [_inverse(t) for t in tc.MBTYPE]
_AC_INV = {(int(tc.AC_CODE[r, a]) << 1 | s, int(tc.AC_LEN[r, a]) + 1): (r, -a if s else a)
           for r in range(64) for a in range(1, 256) if tc.AC_LEN[r, a] for s in (0, 1)}
_DC_INV = [{(int(c, 2), len(c)): s for s, c in t.items()} for t in tc.DC_CODES]


def _dc_of(val, n, table):
    """a DC difference code -> (size, difference)"""
    for s in range(9):
        key = (val >> s, n - s)
        if _DC_INV[table].get(key) == s:
            bits = val & ((1 << s) - 1)
            return s, (0 if s == 0 else bits if bits >> (s - 1) else bits - (1 << s) + 1)
    raise AssertionError("no DC code (%x, %d)" % (val, n))


def _level_of(val, n, first):
    """a coefficient code -> (kind, run, level): "1s", "table", "esc8" or "esc16" """
    if first and n == 2:
        return "1s", 0, -1 if val & 1 else 1
    if (n == 20 or n == 28) and val >> (n - 6) == 1:
        run = (val >> (n - 12)) & 63
        if n == 20:
            b = val & 0xFF
            return "esc8", run, b - 256 if b > 128 else b
        hi, lo = (val >> 8) & 0xFF, val & 0xFF
        assert hi in (0, 0x80), hex(val)
        return "esc16", run, lo if hi == 0 else lo - 256
    kind = _AC_INV[(val, n)]
    return "table", kind[0], kind[1]


def empty_census():
    return dict(mv_codes=set(), mv_wrapped=set(), cbp=set(), inc=set(), types=set(), pairs=set(), dc=set(), dc_carried=set(),
                levels=set(), first=set(), clamped=set(), intra_ac_only63=0, max_zero_run=0, mv_decoded_ok=True)


def census(decs, into=None):
    """what one title's codes reach, read back from the restatement's code arrays; each P slice walked with the reference's
    predictor rules (ef_oracle.c slice()) to find wrapped vector deltas and to check the vectors decode to the decisions"""
    c = into if into is not None else empty_census()
    for d in decs:
        vals, lens = d["codes"]
        p = d["p"]
        for row in range(12):
            bits_v, bits_l = vals[row], lens[row]
            c["max_zero_run"] = max(c["max_zero_run"], _max_zero_run(bits_v[1:], bits_l[1:]))
            mv_v = bits_v[2:].reshape(22, tc.MB_SLOTS)
            mv_l = bits_l[2:].reshape(22, tc.MB_SLOTS)
            prev, mvp, dcp = "start", [0, 0], [128, 128, 128]
            for mx in range(22):
                a = row * 22 + mx
                if not mv_l[mx, 0]:
                    continue
                inc = _MBA_INV[(int(mv_v[mx, 0]), int(mv_l[mx, 0]))]
                t = _TYPE_INV[p][(int(mv_v[mx, 1]), int(mv_l[mx, 1]))]
                c["inc"].add(inc)
                c["types"].add((p, mx == 0, mx == 21, t))
                if inc > 1:
                    prev, mvp, dcp = "skip", [0, 0], [128, 128, 128]
                c["pairs"].add((prev, t))
                if t & 1:
                    mvp = [0, 0]
                    if prev == 0x01:
                        c["dc_carried"].add(p)
                else:
                    dcp = [128, 128, 128]
                    if t & 8:
                        for k in (0, 1):
                            delta = _MV_INV[(int(mv_v[mx, 2 + k]), int(mv_l[mx, 2 + k]))]
                            c["mv_codes"].add(delta)
                            m = mvp[k] + delta
                            if m > 15 or m < -16:
                                c["mv_wrapped"].add((k, delta))
                            mvp[k] = _wrap(m)
                    else:
                        mvp = [0, 0]
                    if p and (mvp[0], mvp[1]) != (int(d["h"][a]), int(d["v"][a])):
                        c["mv_decoded_ok"] = False
                cbp = _CBP_INV[(int(mv_v[mx, 4]), int(mv_l[mx, 4]))] if t & 2 else 63 if t & 1 else 0
                if not t & 1:
                    c["cbp"].add((cbp, t))
                blk_v, blk_l = mv_v[mx, 5:].reshape(6, 65), mv_l[mx, 5:].reshape(6, 65)
                for b in range(6):
                    if not cbp & (0x20 >> b):
                        continue
                    at = np.flatnonzero(blk_l[b, :64])
                    if t & 1:
                        comp = 0 if b < 4 else b - 3
                        size, diff = _dc_of(int(blk_v[b, 0]), int(blk_l[b, 0]), 0 if b < 4 else 1)
                        c["dc"].add((0 if b < 4 else 1, size, int(np.sign(diff))))
                        dcp[comp] += diff
                        assert dcp[comp] == d["levels"][a, b, 0], (a, b)
                        at = at[at > 0]
                        if list(at) == [63]:
                            c["intra_ac_only63"] += 1
                    for i in at:
                        kind, run, lv = _level_of(int(blk_v[b, i]), int(blk_l[b, i]), i == 0 and not t & 1)
                        assert lv == d["levels"][a, b, i], (a, b, i, kind, run, lv)
                        if i == 0 and not t & 1:
                            c["first"].add((kind, lv))
                        else:
                            c["levels"].add((run, lv, kind))
                            if t & 1:
                                raw = (16 * abs(int(d["F"][a, b].reshape(64)[ZZ[i]])) + W_INTRA[i] * d["q"]) // (2 * W_INTRA[i] * d["q"])
                                if raw > 255:
                                    c["clamped"].add(lv)
                prev = t
    return c


def _max_zero_run(vals, lens):
    """the longest run of zero bits in a slice's codes after its start code"""
    keep = lens > 0
    vals, lens = vals[keep], lens[keep]
    total = int(lens.sum())
    rep = np.repeat(np.arange(len(lens)), lens)
    j = np.arange(total) - np.repeat(np.cumsum(lens) - lens, lens)
    bits = (vals[rep] >> (lens[rep] - 1 - j)) & 1
    ones = np.flatnonzero(np.concatenate([[1], bits, [1]]))
    return int(np.diff(ones).max() - 1)


@functools.lru_cache(maxsize=None)
def restated(name):
    """(video.ts, ES of every picture, reconstructions, decisions) of the directed title `name`"""
    from tests.oracle_lib import Oracle
    pics, params = title(name)
    (ts, es, rec, _), decs = encode(pics, Oracle(), **params)
    return ts, es, rec, decs
