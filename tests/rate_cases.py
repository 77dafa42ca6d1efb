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

# The fallbacks' sizes from the code tables: P_MIN, every slice (start code and quantiser, 38 bits) two 0x08 macroblocks of vector (0, 0)
# around a skip run of 20; D_MAX, the worst I fallback: 22 intra macroblocks a slice, every DC difference at the longest size-8 code.
P_MIN = ec.P_HEADER_BYTES + 12 * ((38 + 2 * (len(tc.MBTYPE[1][8]) + 2 * len(tc.MV[0])) + len(tc.MBA[1]) + len(tc.MBA[21]) + 7) // 8)
D_MAX = tc.HEADER_BYTES + 12 * ((38 + 22 * (2 + sum(len(tc.DC_CODES[c][8]) + 8 + 2 for c in (0, 0, 0, 0, 1, 1))) + 7) // 8)


def header_bytes(aspect, rate, bit_rate, vbv_bits):
    """tc.header_bytes with the rate fields: bit_rate ceil(R / 400), vbv_buffer_size ceil(B / 16384)"""
    seq = tc.pack([352, 192, aspect, rate, -(-bit_rate // 400), 1, -(-vbv_bits // 16384), 0, 0, 0], [12, 12, 4, 4, 18, 1, 10, 1, 1, 1])
    return b"\x00\x00\x01\xb3" + seq + tc.header_bytes(aspect, rate)[12:]


# -- sizes at every q ----------------------------------------------------------------------------------------------------------------
def take_census(code, x, qs, head_bytes):
    """(codes, bytes) of a picture at every candidate q of qs and, last, at its fallback (slices at qs[-1]), from one coder call:
    code is tc.i_codes (x: the coefficients) or ec.p_codes (x: the analysis)"""
    qs = list(qs)
    codes = code(x, qs + qs[-1:], [False] * len(qs) + [True])
    return codes, tc.picture_bytes(head_bytes, codes)


def i_sizes(i420, qs):
    """-> {q: ES bytes of the I picture coded at q}, and its fallback's bytes"""
    size = take_census(tc.i_codes, tc.fdct(tc.picture_blocks(i420)), qs, tc.HEADER_BYTES)[1].tolist()
    return dict(zip(qs, size)), size[-1]


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
            head, code, x = hdr, tc.i_codes, tc.fdct(tc.picture_blocks(pictures[k]))
        else:
            head, code, x = ec.p_header(j), ec.p_codes, ec.analyse(ec.planes(pictures[k]), ec.planes(recon[-1]), p["search"])
        codes, size = take_census(code, x, qs, len(head))
        sizes = dict(zip(qs, size.tolist()))
        q, s = choose(sizes, int(size[-1]), f, j, n, r, E, need[j + 1], qmin, qmax)
        es = tc.picture(head, [c[q - qmin if q else -1] for c in codes])
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
