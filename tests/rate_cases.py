"""tests/rate_cases.py — a title's video.ts encoded to a bit rate and a buffer size (ef_encode_build_rate), restated in numpy.

The reference's indexer encodes with "-b:v 1500k -maxrate 1500k -bufsize 0.25M -qmin 3" (make_video(), indexer/indexer.cpp:307), so
that a title streams over the player's link. ef_encode_build_rate does the same on the device; this module is the rule it must equal
byte for byte.

Everything of tests/encode_cases.py holds (GOP layout, motion search, mode decision, block coding, the mux) except the quantiser of
each picture and two sequence-header fields.
Parameters: encode_cases' gop, search, aspect, rate, pts0, pts_step (its qscale_i / qscale_p are not read) and bit_rate R (bits/s,
400 .. 400 * 0x3FFFE), vbv_bits B (1 .. 1023 * 16384), qmin (1..31), qmax (qmin..31).
Headers: every sequence header carries bit_rate = ceil(R / 400) and vbv_buffer_size = ceil(B / 16384); vbv_delay stays 0xFFFF.
Bucket, per GOP, in int64 units of 1/90000 bit (U = 90000): picture j of a GOP of n has s_j = its ES bytes * 8 * U (from its first
header byte up to the next picture's); the refill per picture is r = R * pts_step; f_0 = B U; s_j <= f_j; f_{j+1} = min(B U, f_j - s_j
+ r); f_n >= E, E = B U for every GOP but a title's last, E = 0 for the last.
Fallbacks: P: every macroblock not coded (the skip rule with empty blocks: the first and last of each slice as 0x08 with vector (0, 0),
the rest skipped), slices at qmax, exactly P_MIN bytes. I: every block's DC level, every AC level 0, slices at qmax; its worst case is
D_MAX bytes (every DC difference at the longest size-8 code).
Feasibility: fb_j = D_MAX * 8 U for j = 0, P_MIN * 8 U otherwise; need_n = E, need_j = max(fb_j, fb_j + need_{j+1} - r); the hard
bound is h_j = min(f_j, f_j + r - need_{j+1}).
Soft target: L_j = f_j + (n - j) r - E; t_j = L_j // (n - j) for P pictures, t_0 = L_0 * I_WEIGHT // (I_WEIGHT + n - 1).
Choice, with s(q) the exact size of the picture coded at q: the smallest q in qmin..qmax with s(q) <= min(t_j, h_j); else the smallest
with s(q) <= h_j; else the fallback. Every candidate is evaluated (sizes are not monotone in q).
Validation: EF_EINVAL when D_MAX * 8 U > min(B U, B U + r - need_1) for a full GOP with E = B U."""
import numpy as np

from tests import encode_cases as ec
from tests import trick_cases as tc

U = 90000
RATE_DEFAULTS = dict(bit_rate=1500000, vbv_bits=250000, qmin=3, qmax=31)
# The I picture's share of a GOP's budget against one P picture's, chosen on the two fixtures' decoded pictures: the weight of 2, 3, 4, 6
# and 8 with the highest mean PSNR on vmedia both at the defaults and at 300 kbit/s. At the defaults 3 and above give identical files
# (vmedia 44.73 dB mean, 33.72 dB lowest; 2 gives 44.47 dB) and splash stays at qmin 3 throughout for every weight; at 300 kbit/s vmedia
# gives 37.91, 38.08, 37.62 and 37.70 dB mean at 2, 3, 4 and 6. Larger weights let the I picture meet its own target more often and
# leave less to the P pictures after it.
I_WEIGHT = 3

MBA_LEN = np.array([len(ec.MBA.get(i, "")) for i in range(34)], np.int64)
TYPE_LEN = {k: len(v) for k, v in ec.MBTYPE_P.items()}
MV_LEN = np.array([len(ec.MV[d]) for d in range(-16, 16)] + [len(ec.MV[16])], np.int64)   # [d + 16]
CBP_LEN = np.array([len(ec.CBP.get(c, "")) for c in range(64)], np.int64)
DC_LEN = [np.array([len(tc.DC_CODES[c][s]) + s for s in range(9)], np.int64) for c in (0, 1)]


def _slice_bytes(bits):
    return (bits + 7) // 8


def _p_min_slice_bits():
    return 38 + 2 * (MBA_LEN[1] + TYPE_LEN[8] + 2 * MV_LEN[16]) + MBA_LEN[21] - MBA_LEN[1]


P_MIN = ec.P_HEADER_BYTES + 12 * int(_slice_bytes(_p_min_slice_bits()))
D_MAX = tc.HEADER_BYTES + 12 * int(_slice_bytes(38 + 22 * (2 + 4 * (DC_LEN[0][8] + 2) + 2 * (DC_LEN[1][8] + 2))))


def header_bytes(aspect, rate, bit_rate, vbv_bits):
    """tc.header_bytes with the rate fields: bit_rate ceil(R / 400), vbv_buffer_size ceil(B / 16384)"""
    seq = tc.pack([352, 192, aspect, rate, -(-bit_rate // 400), 1, -(-vbv_bits // 16384), 0, 0, 0], [12, 12, 4, 4, 18, 1, 10, 1, 1, 1])
    return b"\x00\x00\x01\xb3" + seq + tc.header_bytes(aspect, rate)[12:]


# -- sizes at every q ----------------------------------------------------------------------------------------------------------------
def ac_bits(L, intra):
    """[..., 64] zig-zag levels -> [...] bits of their run / level codes (intra: from index 1, the DC counted as coded; non-intra:
    from index 0, a first coefficient of +-1 as "1s")"""
    idx = np.arange(64)
    nz = L != 0
    if intra:
        nz[..., 0] = True
    mark = np.where(nz, idx, -1)
    prev = np.concatenate([np.full(L.shape[:-1] + (1,), -1), np.maximum.accumulate(mark, axis=-1)[..., :-1]], axis=-1)
    run = idx - prev - 1
    a = np.minimum(np.abs(L), 255)
    alen = tc.AC_LEN[np.clip(run, 0, 63), a]
    n = np.where((a <= 40) & (alen > 0), alen + 1, np.where(a <= 127, 20, 28))
    if not intra:
        n[..., 0] = np.where(a[..., 0] == 1, 2, n[..., 0])
    else:
        nz[..., 0] = False
    return np.where(nz, n, 0).sum(axis=-1)


def i_sizes(i420, qs):
    """-> {q: ES bytes of the I picture coded at q}, and its fallback's bytes"""
    F = tc.fdct(tc.picture_blocks(i420))                           # [12, 22, 6, 8, 8], the same at every q
    L0 = tc.quantise(F, 1)
    dc = L0[..., 0]
    dcb = np.zeros(12, np.int64)
    comp = [0, 0, 0, 0, 1, 2]
    for row in range(12):
        pred = [128, 128, 128]
        for mb in range(22):
            for b in range(6):
                c = comp[b]
                dcb[row] += DC_LEN[min(c, 1)][abs(int(dc[row, mb, b]) - pred[c]).bit_length()]
                pred[c] = int(dc[row, mb, b])
    fixed = 38 + 22 * 2 + dcb + 132 * 2
    out = {}
    for q in qs:
        out[q] = tc.HEADER_BYTES + int(_slice_bytes(fixed + ac_bits(tc.quantise(F, q), True).sum(axis=(1, 2))).sum())
    return out, tc.HEADER_BYTES + int(_slice_bytes(fixed).sum())


def p_analysis(src, ref, search_px):
    """the q-independent part of a P picture: the search and both transforms"""
    y, cb, cr = src
    h, v, best, intra = ec.search(y, ref[0], search_px)
    h, v = np.where(intra, 0, h), np.where(intra, 0, v)
    blocks = ec.mb_blocks(y, cb, cr)
    return dict(h=h, v=v, intra=intra, Fi=tc.fdct(blocks), Fp=tc.fdct(blocks - ec.predictions(ref, h, v)))


def p_levels(an, q):
    return np.where(an["intra"][:, None, None], tc.quantise(an["Fi"], q), ec.inter_levels(an["Fp"], q))


def p_sizes(an, qs):
    """-> {q: ES bytes of the P picture coded at q}: the slice walk of encode_cases.p_picture counting bits, vectorised over q"""
    qs = list(qs)
    nq = len(qs)
    L = np.stack([p_levels(an, q) for q in qs])                     # [nq, 264, 6, 64]
    intra, h, v = an["intra"], an["h"], an["v"]
    coded = (L != 0).any(axis=3)                                    # [nq, 264, 6]
    coded[:, intra] = True
    cbp = (coded * (0x20 >> np.arange(6))).sum(axis=2)
    blk = np.where(intra[None, :, None], ac_bits(L, True), ac_bits(L, False)) + 2
    blk = np.where(coded, blk, 0).sum(axis=2)                       # [nq, 264]: run / level and end-of-block bits
    dcl = L[:, :, :, 0]
    total = np.full(nq, ec.P_HEADER_BYTES, np.int64)
    for row in range(12):
        bits = np.full(nq, 38, np.int64)
        pending = np.zeros(nq, np.int64)
        dcp = np.full((nq, 3), 128, np.int64)
        mvp = np.zeros((nq, 2), np.int64)
        for mx in range(22):
            a = row * 22 + mx
            zero = h[a] == 0 and v[a] == 0
            c = cbp[:, a]
            skip = (not intra[a]) & zero & (c == 0) & (0 < mx < 21)
            go = ~skip
            reset = go & (pending > 0)
            dcp[reset] = 128
            mvp[reset] = 0
            bits += np.where(go, MBA_LEN[np.minimum(pending + 1, 33)], 0)
            pending = np.where(go, 0, pending + 1)
            if intra[a]:
                t = np.full(nq, 0x01)
            elif not zero:
                t = np.where(c != 0, 0x0A, 0x08)
            else:
                t = np.where(c != 0, 0x02, 0x08)
            bits += np.where(go, [TYPE_LEN[int(x)] for x in t], 0)
            if intra[a]:
                mvp[go] = 0
                for b in range(6):
                    cp = 0 if b < 4 else b - 3
                    d = np.abs(dcl[:, a, b] - dcp[:, cp])
                    nb = DC_LEN[min(cp, 1)][np.array([int(x).bit_length() for x in d])]
                    bits += np.where(go, nb, 0)
                    dcp[go, cp] = dcl[go, a, b]
            else:
                dcp[go] = 128
                mv = go & ((t & 0x08) != 0)
                for cc, val in enumerate((int(h[a]), int(v[a]))):
                    d = val - mvp[:, cc]
                    d = np.where(d < -16, d + 32, np.where(d > 15, d - 32, d))
                    bits += np.where(mv, MV_LEN[d + 16], 0)
                    mvp[mv, cc] = val
                mvp[go & ~mv] = 0
                bits += np.where(go & ((t & 0x02) != 0), CBP_LEN[c], 0)
            bits += np.where(go, blk[:, a], 0)
        total += _slice_bytes(bits)
    return {q: int(total[i]) for i, q in enumerate(qs)}


# -- the coder at one q --------------------------------------------------------------------------------------------------------------
def i_picture(i420, q, hdr, fallback):
    levels = tc.quantise(tc.fdct(tc.picture_blocks(i420)), q)
    if fallback:
        levels[..., 1:] = 0
    return hdr + b"".join(tc.slice_codes(levels[r], r, q) for r in range(12))


def p_picture(an, k, gop, q, fallback):
    """encode_cases.p_picture from a precomputed analysis; the fallback codes every macroblock as not coded"""
    if fallback:
        z = np.zeros(264, np.int64)
        h, v, intra, L = z, z, np.zeros(264, bool), np.zeros((264, 6, 64), np.int64)
    else:
        h, v, intra, L = an["h"], an["v"], an["intra"], p_levels(an, q)
    cbp = np.where(intra, 63, ((L != 0).any(axis=2) * (0x20 >> np.arange(6))).sum(axis=1))
    out = [b"\x00\x00\x01\x00" + tc.pack([k % gop, 2, 0xFFFF, 0, 1, 0], [10, 3, 16, 1, 3, 1])]
    for row in range(12):
        bw = ec.Bits()
        bw.put(q << 1, 6)
        pending, dcp, mvp = 0, [128, 128, 128], [0, 0]
        for mx in range(22):
            a = row * 22 + mx
            zero = h[a] == 0 and v[a] == 0
            if not intra[a] and zero and cbp[a] == 0 and 0 < mx < 21:
                pending += 1
                continue
            if pending:
                dcp, mvp = [128, 128, 128], [0, 0]
            bw.code(ec.MBA[pending + 1])
            pending = 0
            t = 0x01 if intra[a] else (0x0A if cbp[a] else 0x08) if not zero else (0x02 if cbp[a] else 0x08)
            bw.code(ec.MBTYPE_P[t])
            if intra[a]:
                mvp = [0, 0]
            else:
                dcp = [128, 128, 128]
                if t & 0x08:
                    for c, val in enumerate((int(h[a]), int(v[a]))):
                        d = val - mvp[c]
                        d = d + 32 if d < -16 else d - 32 if d > 15 else d
                        bw.code(ec.MV[d])
                        mvp[c] = val
                else:
                    mvp = [0, 0]
                if t & 0x02:
                    bw.code(ec.CBP[int(cbp[a])])
            for b in range(6):
                if cbp[a] & (0x20 >> b):
                    comp = 0 if b < 4 else b - 3
                    dcp[comp] = ec.put_block(bw, L[a, b], bool(intra[a]), comp, dcp[comp])
        out.append(bytes([0, 0, 1, row + 1]) + tc.pack(bw.v, bw.n))
    return b"".join(out)


# -- the bucket ----------------------------------------------------------------------------------------------------------------------
def refill(bit_rate, pts_step):
    return bit_rate * pts_step


def needs(n, r, E):
    """need_0 .. need_n of a GOP of n pictures"""
    need = [0] * (n + 1)
    need[n] = E
    for j in range(n - 1, -1, -1):
        fb = (D_MAX if j == 0 else P_MIN) * 8 * U
        need[j] = max(fb, fb + need[j + 1] - r)
    return need


def check(gop, bit_rate, vbv_bits, qmin, qmax, pts_step, **_):
    """None when the parameters are valid, else the reason for EF_EINVAL"""
    if not 400 <= bit_rate <= 400 * 0x3FFFE or not 1 <= vbv_bits <= 1023 * 16384 or not 1 <= qmin <= qmax <= 31:
        return "rate field out of range"
    r, BU = refill(bit_rate, pts_step), vbv_bits * U
    need = needs(gop, r, BU)
    need1 = need[1] if gop > 1 else BU
    if D_MAX * 8 * U > min(BU, BU + r - need1):
        return "no encode can be guaranteed"
    return None


def choose(sizes, fb_bytes, f, j, n, r, E, need_next, qmin, qmax):
    """-> (q, 0 for the fallback; ES bytes)"""
    h = min(f, f + r - need_next)
    L = f + (n - j) * r - E
    t = L * I_WEIGHT // (I_WEIGHT + n - 1) if j == 0 else L // (n - j)
    for cap in (min(t, h), h):
        for q in range(qmin, qmax + 1):
            if sizes[q] * 8 * U <= cap:
                return q, sizes[q]
    assert fb_bytes * 8 * U <= h, (fb_bytes, f, h)
    return 0, fb_bytes


def encode_title(pictures, oracle, **params):
    """pictures uint8 [n, PICTURE_BYTES] -> (video.ts bytes, ES of every picture, reconstructions, chosen q per picture (0: fallback),
    census {q: bytes} per picture)"""
    p = dict(ec.DEFAULT_PARAMS, **RATE_DEFAULTS)
    p.update(params)
    why = check(**p)
    assert why is None, why
    pictures = np.asarray(pictures, dtype=np.uint8).reshape(-1, ec.PICTURE_BYTES)
    gop, qmin, qmax = p["gop"], p["qmin"], p["qmax"]
    qs = range(qmin, qmax + 1)
    hdr = header_bytes(p["aspect"], p["rate"], p["bit_rate"], p["vbv_bits"])
    r, BU = refill(p["bit_rate"], p["pts_step"]), p["vbv_bits"] * U
    N = len(pictures)
    pics, recon, chosen, census = [], [], [], []
    gop_es = b""
    for k in range(N):
        j = k % gop
        if j == 0:
            n = min(gop, N - k)
            E = 0 if k + n == N else BU
            need, f, gop_es = needs(n, r, E), BU, b""
            sizes, fb = i_sizes(pictures[k], qs)
        else:
            an = p_analysis(ec.planes(pictures[k]), ec.planes(recon[-1]), p["search"])
            sizes, fb = p_sizes(an, qs), P_MIN
        q, s = choose(sizes, fb, f, j, n, r, E, need[j + 1], qmin, qmax)
        es = i_picture(pictures[k], q or qmax, hdr, not q) if j == 0 else p_picture(an, k, gop, q or qmax, not q)
        assert len(es) == s, (k, q, len(es), s)
        f = min(BU, f - s * 8 * U + r)
        gop_es += es
        frames = oracle.decode_es(gop_es, max_frames=gop)
        assert len(frames) == j + 1, (k, len(frames))
        recon.append(frames[-1].copy())
        pics.append(es)
        chosen.append(q)
        census.append(sizes)
    pts = [p["pts0"] + k * p["pts_step"] for k in range(N)]
    return tc.mux(pics, pts), pics, np.array(recon), chosen, census


# -- an independent bucket check -----------------------------------------------------------------------------------------------------
def pictures_of(ts):
    """the ES of PID 0x100 cut at picture starts: a sequence header opens a picture (and a GOP), so does a picture start code not
    preceded by one -> [(bytes, opens a GOP)]"""
    es = bytearray()
    for o in range(0, len(ts), 188):
        pk = ts[o:o + 188]
        assert pk[0] == 0x47
        if ((pk[1] & 0x1F) << 8 | pk[2]) != 0x100:
            continue
        s = 4 + (pk[4] + 1 if pk[3] & 0x20 else 0)
        if pk[1] & 0x40:
            s += 9 + pk[s + 8]
        es += pk[s:]
    es = bytes(es)
    cuts, i = [], 0
    while True:
        i = es.find(b"\x00\x00\x01", i)
        if i < 0 or i + 3 >= len(es):
            break
        c = es[i + 3]
        if c == 0xB3:
            cuts.append((i, True))
        elif c == 0x00 and not (cuts and cuts[-1][1] and i - cuts[-1][0] < 32):
            cuts.append((i, False))
        i += 3
    ends = [c[0] for c in cuts[1:]] + [len(es)]
    return [(es[c[0]:e], c[1]) for c, e in zip(cuts, ends)]


def bucket_violations(ts, bit_rate, vbv_bits, pts_step):
    """-> (violations, largest draw in bits): a picture larger than the buffer holds, or a GOP but the last not handing on a full
    buffer; counted in exact integers from the file's own picture boundaries"""
    pics = pictures_of(ts)
    r, BU = bit_rate * pts_step, vbv_bits * U
    bad, draw, f = [], 0, None
    gops = [i for i, (_, g) in enumerate(pics) if g] + [len(pics)]
    for gi in range(len(gops) - 1):
        f = BU
        for j in range(gops[gi], gops[gi + 1]):
            s = len(pics[j][0]) * 8 * U
            draw = max(draw, BU - (f - s))
            if s > f:
                bad.append(("underflow", j))
            f = min(BU, f - s + r)
        if gi + 2 < len(gops) and f < BU:
            bad.append(("not full", gops[gi + 1]))
    return bad, draw // U


PIN_NAMES = ["vmedia/default", "vmedia/300k", "splash/400k", "cut", "noise/fallback", "checker", "gop1", "gop13"]


def pin_cases(oracle):
    """name -> (pictures, parameters) of tests/golden/rate_pins.json: vmedia at the reference's rate and at 300 kbit/s (where the fixed
    q8 file overflows), splash in a small bucket, a scene cut with a short last GOP, noise that forces both fallbacks, checkerboards
    over the whole q range, GOP 1 and GOP 13 over mixed content with a short last GOP"""
    vm = ec.fixture_pictures("vmedia", oracle)
    mixed = np.concatenate([ec.translated(9, 14, (2, 1)), ec.noise(5, 4), ec.translated(12, 12, (-3, 2))])
    return {
        "vmedia/default": (vm, {}),
        "vmedia/300k": (vm, dict(bit_rate=300000)),
        "splash/400k": (ec.fixture_pictures("splash", oracle)[:30], dict(bit_rate=400000, vbv_bits=40000)),
        "cut": (ec.scene_cut(4, 14, 5), dict(bit_rate=700000, vbv_bits=40000, qmin=1, qmax=31)),
        "noise/fallback": (ec.noise(3, 5), dict(gop=12, bit_rate=1000000, vbv_bits=40000, qmin=30, qmax=31)),
        "checker": (np.concatenate([ec.checkerboard(4, cell=1), ec.checkerboard(4, cell=8, phase=1)]),
                    dict(gop=5, bit_rate=2000000, vbv_bits=500000, qmin=1, qmax=31)),
        "gop1": (ec.translated(3, 4, (1, 3)), dict(gop=1)),
        "gop13": (mixed, dict(gop=13, bit_rate=900000, vbv_bits=200000)),
    }


def rate_weight_table(oracle, weights=(2, 3, 4, 6, 8)):
    """the measurement behind I_WEIGHT: (fixture, weight) -> (mean PSNR, lowest PSNR) at the defaults"""
    global I_WEIGHT
    keep, out = I_WEIGHT, {}
    try:
        for name in ("vmedia", "splash"):
            pics = ec.fixture_pictures(name, oracle)
            for w in weights:
                I_WEIGHT = w
                rec = encode_title(pics, oracle)[2]
                ps = ec.psnr_list(pics, rec)
                out[(name, w)] = (float(np.mean(ps)), float(np.min(ps)))
    finally:
        I_WEIGHT = keep
    return out
