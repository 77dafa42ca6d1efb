"""tests/encode_cases.py — a title's video.ts encoded from raw pictures (ef_encode_build), restated in numpy.

The reference's indexer makes video.ts with ffmpeg (make_video(), indexer/indexer.cpp:306): MPEG-1 at GOP 12 without B pictures.
ef_encode_build makes it on the device; this module is the rule it must equal byte for byte.

Input: a title's pictures in display order, 352 x 192 I420 (PICTURE_BYTES each); parameters gop, qscale_i, qscale_p, search,
aspect, rate, pts0, pts_step.
GOPs: picture k of the title opens a GOP when k % gop == 0. A GOP is trick_cases.header_bytes(aspect, rate) (sequence header,
closed GOP header, I picture header with temporal reference 0) and the I picture's 12 slices exactly as trick_cases encodes them
at qscale_i; then up to gop - 1 P pictures. A P picture is a 9-byte header (picture start code, temporal reference k % gop,
type 2, vbv_delay 0xFFFF, full_pel_forward 0, forward_f_code 1, extra bit 0, zero padding) and 12 slices, one per macroblock row
(slice code row + 1, quantiser qscale_p, extra bit 0), each starting at column 0. No user data, extensions or sequence end code.
Reference picture of P picture k: the decoder's reconstruction of picture k - 1 (here: the oracle's decode of the GOP so far).
Motion search, per macroblock (mx, my), vectors (h, v) in half-pel units:
  legal(h, v): hx = 32 mx + h >= 0, hy = 32 my + v >= 0, (hx >> 1) + 16 + (hx & 1) <= 352, (hy >> 1) + 16 + (hy & 1) <= 192,
               -16 <= h, v <= 15 (forward_f_code 1);
  sad(h, v):   sum over the 16 x 16 luma of |source - mc(ref.y, hx, hy)|, mc the decoder's half-pel averaging (mc_block());
  best = sad(0, 0) - ZERO_BIAS, vector (0, 0); then every full-pel (h, v) = (2 dx, 2 dy), dy outer and dx inner, each from
  -search to search, in raster order: a legal candidate replaces the best when its sad is strictly lower; then the 3 x 3
  half-pel neighbours (bh + a, bv + b), b outer and a inner from -1 to 1, the same way (the centre never replaces itself).
Mode: intra when best > mad + INTRA_MARGIN, mad = sum |y - ((sum y + 128) >> 8)| over the source luma; all integers.
Prediction: luma mc(ref.y, hx, hy, 16); chroma mc(ref.cb / ref.cr, hx >> 1, hy >> 1, 8) (quirk Q3: the floor of the halved
vector). Residual: source - prediction through trick_cases.fdct; level = sign(F) min(floor(8 |F| / (16 qscale_p)), 255) at every
coefficient (the non-intra dead zone, flat matrix 16). Intra macroblocks: trick_cases.quantise(F, qscale_p).
Coded block pattern: bit 0x20 >> b when block b has a non-zero level (intra: all six).
Macroblock type: intra 0x01; else vector != 0: 0x0A with coded blocks, 0x08 without; vector 0: 0x02 with coded blocks; without,
the macroblock is skipped unless it is the first or last of its slice, which is coded as 0x08 with vector (0, 0).
Predictors: the motion-vector predictor is (0, 0) at slice start and after an intra macroblock, a skip or a 0x02; the vector
delta is wrapped into -16..15 and coded with the motion VLC (f_code 1: no residual bits). DC predictors are 128 at slice start
and after a skipped or non-intra macroblock. Blocks: non-intra blocks code every level from zig-zag index 0, a first
coefficient of run 0 and level +-1 as "1s", the rest as trick_cases codes AC levels (table, 8- and 16-bit escapes); intra
blocks as trick_cases; every coded block ends with "10". An address increment counts the skipped macroblocks before a coded
one plus 1.
Mux: trick_cases.mux(pictures of a title, pts0 + k pts_step): PID 0x100, one PES per picture, one continuity counter per file."""
import hashlib
import os

import numpy as np

from tests import trick_cases as tc

ROOT = tc.ROOT
W, H = 352, 192
MBW, MBH = 22, 12
PICTURE_BYTES = 101376
ZERO_BIAS = 64             # the zero vector's head start, so that static areas skip
INTRA_MARGIN = 512         # 2 per luma sample beyond the source's own deviation before a macroblock goes intra
P_HEADER_BYTES = 9
# ef_encode_build's defaults (espflix_b200/capi.ENCODE_DEFAULTS). The quantisers were chosen on the two fixtures' decoded pictures
# as trick_cases.DEFAULT_QSCALE was: the largest of 8 and 16 whose worst picture stays at or above 35 dB on both. At 8 / 8 vmedia
# gives 1,936 bytes per picture, PSNR 36.1 dB lowest and 38.1 dB mean (ffmpeg's vmedia.ts: 6,104 bytes per picture), splash 797
# bytes and 42.5 dB lowest; at 16 / 16 vmedia's worst picture falls to 31.6 dB.
DEFAULT_PARAMS = dict(gop=12, qscale_i=8, qscale_p=8, search=7, aspect=1, rate=2, pts0=0, pts_step=3750)


def planes(i420):
    f = np.frombuffer(bytes(i420), dtype=np.uint8).astype(np.int64)
    return f[:67584].reshape(H, W), f[67584:84480].reshape(H // 2, W // 2), f[84480:].reshape(H // 2, W // 2)


def legal(mx, my, h, v):
    hx, hy = 32 * mx + h, 32 * my + v
    return ((hx >= 0) & (hy >= 0) & ((hx >> 1) + 16 + (hx & 1) <= W) & ((hy >> 1) + 16 + (hy & 1) <= H) &
            (h >= -16) & (h <= 15) & (v >= -16) & (v <= 15))


def mc(plane, hx, hy, size):
    """the decoder's prediction of one size x size block at half-pel position (hx, hy); arrays broadcast over blocks"""
    hx, hy = np.asarray(hx), np.asarray(hy)
    x0, y0, xh, yh = hx >> 1, hy >> 1, hx & 1, hy & 1
    pad = np.pad(plane, 1, mode="edge")                       # reads of illegal positions are discarded by the caller
    r = np.arange(size)
    ys = np.clip(y0[..., None] + r, -1, plane.shape[0]) + 1
    xs = np.clip(x0[..., None] + r, -1, plane.shape[1]) + 1
    ys1 = np.clip(y0[..., None] + r + 1, -1, plane.shape[0]) + 1
    xs1 = np.clip(x0[..., None] + r + 1, -1, plane.shape[1]) + 1
    a = pad[ys[..., :, None], xs[..., None, :]]
    b = pad[ys[..., :, None], xs1[..., None, :]]
    c = pad[ys1[..., :, None], xs[..., None, :]]
    d = pad[ys1[..., :, None], xs1[..., None, :]]
    xh, yh = xh[..., None, None], yh[..., None, None]
    return np.where(xh & yh, (a + b + c + d + 2) >> 2, np.where(xh, (a + b + 1) >> 1, np.where(yh, (a + c + 1) >> 1, a)))


_MX, _MY = np.meshgrid(np.arange(MBW), np.arange(MBH))
_MX, _MY = _MX.ravel(), _MY.ravel()                           # macroblock address order


def search(src_y, ref_y, search_px):
    """-> (h, v, best, intra) per macroblock, [264] each"""
    S = src_y.reshape(MBH, 16, MBW, 16).transpose(0, 2, 1, 3).reshape(264, 16, 16)
    z = np.zeros(264, np.int64)

    def sad(h, v):
        return np.abs(S - mc(ref_y, 32 * _MX + h, 32 * _MY + v, 16)).sum(axis=(1, 2))

    best, bh, bv = sad(z, z) - ZERO_BIAS, z.copy(), z.copy()
    pad = np.pad(ref_y, 16)                                   # full-pel: the whole picture shifted at once, summed per macroblock
    for dy in range(-search_px, search_px + 1):
        for dx in range(-search_px, search_px + 1):
            h, v = np.full(264, 2 * dx), np.full(264, 2 * dy)
            ok = legal(_MX, _MY, h, v)
            if not ok.any():
                continue
            d = np.abs(src_y - pad[16 + dy:16 + dy + H, 16 + dx:16 + dx + W])
            s = d.reshape(MBH, 16, MBW, 16).sum(axis=(1, 3)).ravel()
            w = ok & (s < best)
            best, bh, bv = np.where(w, s, best), np.where(w, h, bh), np.where(w, v, bv)
    ch, cv = bh.copy(), bv.copy()
    for b in (-1, 0, 1):
        for a in (-1, 0, 1):
            h, v = ch + a, cv + b
            ok = legal(_MX, _MY, h, v)
            s = sad(h, v)
            w = ok & (s < best)
            best, bh, bv = np.where(w, s, best), np.where(w, h, bh), np.where(w, v, bv)
    tot = S.sum(axis=(1, 2))
    mad = np.abs(S - ((tot + 128) >> 8)[:, None, None]).sum(axis=(1, 2))
    return bh, bv, best, best > mad + INTRA_MARGIN


def mb_blocks(y, cb, cr):
    """planes -> int64 [264, 6, 8, 8] in macroblock address order, MPEG block order"""
    Y = y.reshape(MBH, 2, 8, MBW, 2, 8).transpose(0, 3, 1, 4, 2, 5).reshape(264, 4, 8, 8)
    C = [p.reshape(MBH, 8, MBW, 8).transpose(0, 2, 1, 3).reshape(264, 1, 8, 8) for p in (cb, cr)]
    return np.concatenate([Y] + C, axis=1)


def predictions(ref, h, v):
    """[264, 6, 8, 8] prediction blocks of vectors (h, v)"""
    hx, hy = 32 * _MX + h, 32 * _MY + v
    py = mc(ref[0], hx, hy, 16).reshape(264, 2, 8, 2, 8).transpose(0, 1, 3, 2, 4).reshape(264, 4, 8, 8)
    pc = [mc(ref[k], hx >> 1, hy >> 1, 8)[:, None] for k in (1, 2)]
    return np.concatenate([py] + pc, axis=1)


def inter_levels(F, qscale):
    f = F.reshape(F.shape[:-2] + (64,))[..., tc.ZIGZAG]
    return np.sign(f) * np.minimum((8 * np.abs(f)) // (16 * qscale), 255)


def p_header(tref):
    """a P picture's header (P_HEADER_BYTES) of temporal reference tref"""
    return b"\x00\x00\x01\x00" + tc.pack([tref, 2, 0xFFFF, 0, 1, 0], [10, 3, 16, 1, 3, 1])


def analyse(src, ref, search_px):
    """the quantiser-independent part of a P picture: the search, the mode decision and both transforms"""
    y, cb, cr = src
    h, v, best, intra = search(y, ref[0], search_px)
    h, v = np.where(intra, 0, h), np.where(intra, 0, v)
    blocks = mb_blocks(y, cb, cr)
    return dict(h=h, v=v, intra=intra, Fi=tc.fdct(blocks), Fp=tc.fdct(blocks - predictions(ref, h, v)))


def p_levels(an, q):
    """[264, 6, 64] zig-zag levels at quantiser q"""
    return np.where(an["intra"][:, None, None], tc.quantise(an["Fi"], q), inter_levels(an["Fp"], q))


def p_codes(an, qs, fallback):
    """a P picture's slice codes [candidates, 12, slots] at each candidate quantiser of qs; fallback [candidates]: every macroblock not
    intra, with vector (0, 0) and all levels zero"""
    fb = np.asarray(fallback, bool)
    L = np.stack([p_levels(an, q) for q in qs])
    L[fb] = 0
    intra, h, v = (np.where(fb[:, None], d, an[k]).reshape(-1, MBH, MBW) for k, d in (("intra", False), ("h", 0), ("v", 0)))
    return tc.slice_codes(True, tc.ROWS, intra, h, v, L.reshape(-1, MBH, MBW, 6, 64), np.asarray(qs)[:, None])


def p_picture(an, tref, qscale):
    """-> (picture bytes, per-macroblock (h, v, intra, skipped, cbp)); skipped: the slice writes no address increment for it"""
    codes = p_codes(an, [qscale], [False])
    skipped = codes[1][0, :, 2::tc.MB_SLOTS].ravel() == 0
    cbp = np.where(an["intra"], 63, ((p_levels(an, qscale) != 0).any(axis=2) * (0x20 >> np.arange(6))).sum(axis=1))
    return tc.picture(p_header(tref), codes), dict(h=an["h"], v=an["v"], intra=an["intra"], skipped=skipped, cbp=cbp)


def encode_title(pictures, oracle, **params):
    """pictures uint8 [n, PICTURE_BYTES] -> (video.ts bytes, ES of every picture, reconstructions [n, PICTURE_BYTES], infos)"""
    p = dict(DEFAULT_PARAMS, **params)
    pictures = np.asarray(pictures, dtype=np.uint8).reshape(-1, PICTURE_BYTES)
    gop = p["gop"]
    pics, recon, infos = [], [], []
    gop_es = b""
    for k in range(len(pictures)):
        if k % gop == 0:
            es, info = tc.encode_picture(pictures[k], p["qscale_i"], tc.header_bytes(p["aspect"], p["rate"])), None
            gop_es = b""
        else:
            es, info = p_picture(analyse(planes(pictures[k]), planes(recon[-1]), p["search"]), k % gop, p["qscale_p"])
        gop_es += es
        frames = oracle.decode_es(gop_es, max_frames=gop)
        assert len(frames) == k % gop + 1, (k, len(frames))
        recon.append(frames[-1].copy())
        pics.append(es)
        infos.append(info)
    pts = [p["pts0"] + k * p["pts_step"] for k in range(len(pictures))]
    return tc.mux(pics, pts), pics, np.array(recon), infos


# -- synthetic sources -------------------------------------------------------------------------------------------------------------
def textured(seed, w=W + 64, h=H + 64, grain=6.0):
    """a smooth random texture larger than the picture (so shifted crops stay inside it), uint8 planes (y, cb, cr)"""
    rng = np.random.default_rng(seed)
    def field(hh, ww, cell):
        g = rng.integers(16, 240, size=(hh // cell + 2, ww // cell + 2)).astype(np.float64)
        yy, xx = np.mgrid[0:hh, 0:ww] / cell
        y0, x0 = yy.astype(int), xx.astype(int)
        fy, fx = yy - y0, xx - x0
        v = (g[y0, x0] * (1 - fx) * (1 - fy) + g[y0, x0 + 1] * fx * (1 - fy) + g[y0 + 1, x0] * (1 - fx) * fy + g[y0 + 1, x0 + 1] * fx * fy)
        return v
    y = field(h, w, 8) + rng.normal(0, grain, size=(h, w))
    return np.clip(y, 0, 255), np.clip(field(h // 2, w // 2, 8), 0, 255), np.clip(field(h // 2, w // 2, 8), 0, 255)


def crop(tex, x2, y2):
    """picture whose luma sample (x, y) is the texture at (x + x2 / 2 + 32, y + y2 / 2 + 32): a half-pel crop (averaged as the
    decoder averages, so a half-pel translation of the previous crop is exactly representable)"""
    def sub(p, hx, hy, ww, hh):
        x0, y0, xh, yh = hx >> 1, hy >> 1, hx & 1, hy & 1
        a = p[y0:y0 + hh, x0:x0 + ww]
        b = p[y0:y0 + hh, x0 + 1:x0 + ww + 1]
        c = p[y0 + 1:y0 + hh + 1, x0:x0 + ww]
        d = p[y0 + 1:y0 + hh + 1, x0 + 1:x0 + ww + 1]
        if xh and yh:
            return (a + b + c + d + 2) >> 2
        if xh:
            return (a + b + 1) >> 1
        if yh:
            return (a + c + 1) >> 1
        return a
    y, cb, cr = [np.asarray(t, dtype=np.int64) for t in tex]
    Y = sub(y, 64 + x2, 64 + y2, W, H)
    C = [sub(c, 32 + (x2 // 2) // 2 * 2, 32 + (y2 // 2) // 2 * 2, W // 2, H // 2) for c in (cb, cr)]
    return np.concatenate([Y.ravel()] + [c.ravel() for c in C]).astype(np.uint8)


def halfpel_chain(seed, n, step):
    """n pictures where picture k is the decoder's half-pel prediction of picture k - 1's source moved by step (half-pels, each
    component -1, 0 or 1): exactly what a vector of -step predicts from an exact reference"""
    y, cb, cr = [np.asarray(t, dtype=np.int64) for t in textured(seed, grain=20.0)]
    out = []
    for k in range(n):
        if k:
            y = _shift_half(y, step)
        out.append(np.concatenate([y[32:32 + H, 32:32 + W].ravel(), cb[16:16 + H // 2, 16:16 + W // 2].ravel(),
                                   cr[16:16 + H // 2, 16:16 + W // 2].ravel()]).astype(np.uint8))
    return np.stack(out)


def _shift_half(p, step):
    """the plane sampled at (x + step[0] / 2, y + step[1] / 2) with the decoder's rounding (edges repeated)"""
    q = np.pad(p, 1, mode="edge")
    ox, oy = (step[0] >> 1) + 1, (step[1] >> 1) + 1
    hh, ww = p.shape
    a = q[oy:oy + hh, ox:ox + ww]
    b = q[oy:oy + hh, ox + 1:ox + ww + 1]
    c = q[oy + 1:oy + hh + 1, ox:ox + ww]
    d = q[oy + 1:oy + hh + 1, ox + 1:ox + ww + 1]
    xh, yh = step[0] & 1, step[1] & 1
    return (a + b + c + d + 2) >> 2 if xh and yh else (a + b + 1) >> 1 if xh else (a + c + 1) >> 1 if yh else a


def translated(seed, n, step, grain=6.0):
    """n pictures moving by (step[0], step[1]) half-pels per picture"""
    tex = textured(seed, grain=grain)
    return np.stack([crop(tex, -k * step[0], -k * step[1]) for k in range(n)])


def noise(seed, n):
    return np.random.default_rng(seed).integers(0, 256, size=(n, PICTURE_BYTES), dtype=np.uint8)


def checkerboard(n, cell=1, phase=0):
    out = []
    for k in range(n):
        y, x = np.mgrid[0:H, 0:W]
        Y = np.where(((x // cell + y // cell + k + phase) & 1) == 1, 255, 0)
        yc, xc = np.mgrid[0:H // 2, 0:W // 2]
        C = np.where(((xc // cell + yc // cell + k) & 1) == 1, 255, 0)
        out.append(np.concatenate([Y.ravel(), C.ravel(), (255 - C).ravel()]).astype(np.uint8))
    return np.stack(out)


def scene_cut(seed, n, cut):
    """a static texture, then from picture `cut` on a darker, flatter one"""
    a, b = translated(seed, n, (0, 0)), translated(seed + 1, n, (0, 0)) // 4 + 8
    return np.concatenate([a[:cut], b[cut:]])


def fixture_pictures(name, oracle):
    return oracle.decode_ts(tc.fixture(name), max_frames=256)


def pin_cases(oracle):
    """(name, pictures, parameters) of tests/golden/encode_pins.json: both fixtures at the defaults and at qscale 1 and 31, and the
    synthetic cases that reach every P macroblock kind, half-pel vectors, escapes and +-255 levels"""
    out = []
    for name in ("vmedia", "splash"):
        pics = fixture_pictures(name, oracle)
        for q in (DEFAULT_PARAMS["qscale_p"], 1, 31):
            out.append(("%s/q%d" % (name, q), pics, dict(qscale_i=q, qscale_p=q)))
    out += [("static", translated(1, 6, (0, 0), grain=0.0), {}), ("halfpel", halfpel_chain(20, 6, (1, -1)), {}),
            ("cut", scene_cut(4, 6, 3), {}), ("noise/q1", noise(7, 3), dict(qscale_i=1, qscale_p=1)),
            ("checker/q31", checkerboard(3, cell=8, phase=1), dict(qscale_i=31, qscale_p=31))]
    return out


def digest(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def psnr_list(src, rec):
    return [tc.psnr(a, b) for a, b in zip(src, rec)]
