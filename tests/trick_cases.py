"""tests/trick_cases.py — the fast-forward and rewind trick streams (video_fwd.ts, video_rwd.ts) restated in numpy.

The reference's indexer makes them with two ffmpeg re-encodes of video.ts (indexer/indexer.cpp:308-309): fwd = setpts=PTS/15,
rwd = fwd played backwards. ef_trick_build makes them on the device; this module is the rule it must equal byte for byte.

Source pictures: the main's pictures in decode order (the streams have no B pictures, so that is display order), each the frame
a continuous decode of the whole video.ts gives, with p_j = the pts ef_picture_pts reports for picture j.
Selection: fwd picture k is main picture 15 k, k = 0 .. n - 1, n = (N - 1) // 15 + 1; its pts is p_0 + (p_15k - p_0) / 15, a
C division (truncated toward zero). rwd picture j is fwd picture n - 1 - j with pts f_0 + (f_{n-1} - f_{n-1-j}): the spacing
kept, the order reversed.
Pictures: every picture is a random-access point: a sequence header (352 x 192, the aspect and picture-rate codes of the main's
first sequence header, bit_rate 0x3FFFF, vbv 20, default matrices), a closed GOP header and an I picture header, then 12
slices (codes 1 .. 12) of 22 intra macroblocks (address increment 1, type 1), DC differences with the size tables, AC
coefficients with the run / level table, 8- and 16-bit escapes and "10" as the end of block. No sequence end code.
Transform: FDCT_C, an integer separable DCT with fixed rounding (fdct()); quantiser: DC level = round(F00 / 8) clamped to
0 .. 255, AC level = round-half-away-from-zero of 8 F / (qscale q_intra[zz]) clamped to +-255, both in integers.
Mux: efs_wrap_ts's layout with these pts: PID 0x100, one PES per picture (stream id 0xE0, flags 0x8080, a 5-byte PTS), every
PES starts a packet and its last packet is padded with adaptation-field stuffing, one continuity counter through the file."""
import collections
import hashlib
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_TABLES = os.path.join(ROOT, "espflix_b200", "csrc", "ef_iso11172_tables.h")
SPEED = 15                 # merge_index's trick_speed: one fwd picture per 15 main pictures
# ef_trick_build's default, chosen on the two fixtures (tests/golden/trick_pins.json): the largest of qscale 4, 8 and 16 whose worst
# fwd picture stays at or above 35 dB on both (35.8 / 43.1 dB at 8, 31.7 / 39.3 dB at 16); 8 takes a third off the bytes of 4.
DEFAULT_QSCALE = 8
HEADER_BYTES = 28          # sequence (12) + GOP (8) + picture (8) header bytes of every trick picture

# FDCT_C[k][n] = round(4096 c_k cos((2n + 1) k pi / 16)), c_0 = sqrt(1/8), c_k = 1/2: the orthonormal DCT-II in 12-bit fixed
# point. Row pass: (x C^T + 2^7) >> 8 (4 fractional bits kept); column pass: (C t + 2^15) >> 16. Pixels are 0..255, every row of
# C sums to at most 11,585 in magnitude, so the row pass stays within 255 x 11,585 < 2^22 and its output within 11,539; the
# column pass within 11,585 x 11,539 < 2^28: int32 throughout (FDCT_BOUNDS below; tests/test_trick.py checks them).
FDCT_C = np.array([
    [1448, 1448, 1448, 1448, 1448, 1448, 1448, 1448],
    [2009, 1703, 1138, 400, -400, -1138, -1703, -2009],
    [1892, 784, -784, -1892, -1892, -784, 784, 1892],
    [1703, -400, -2009, -1138, 1138, 2009, 400, -1703],
    [1448, -1448, -1448, 1448, 1448, -1448, -1448, 1448],
    [1138, -2009, 400, 1703, -1703, -400, 2009, -1138],
    [784, -1892, 1892, -784, -784, 1892, -1892, 784],
    [400, -1138, 1703, -2009, 2009, -1703, 1138, -400]], dtype=np.int64)
_ROWSUM = int(np.abs(FDCT_C).sum(axis=1).max())
FDCT_BOUNDS = {"row_acc": 255 * _ROWSUM, "row_out": (255 * _ROWSUM + 128) >> 8, "col_acc": _ROWSUM * ((255 * _ROWSUM + 128) >> 8)}


def _vlc(name):
    s = open(_TABLES).read()
    i = s.index("static const ef_vlc_code %s[]" % name)
    body = s[i:s.index("};", i)]
    return {int(m.group(2), 0): m.group(1) for m in re.finditer(r'\{"([01]+)", (-?(?:0x)?[0-9A-Fa-f]+)\}', body)}


def _u8(name):
    s = open(_TABLES).read()
    i = s.index("static const unsigned char %s[" % name)
    return np.array([int(x) for x in re.findall(r"\d+", s[s.index("{", i):s.index("};", i)])], dtype=np.int64)


ZIGZAG = _u8("ef_zigzag")                  # zig-zag index -> raster index
INTRA_Q = _u8("ef_default_intra_q")        # indexed by the raster index, as efsynth and the decoder index it
_DCT = _vlc("ef_vlc_dct")
DC_CODES = [_vlc("ef_vlc_dc_luma"), _vlc("ef_vlc_dc_chroma")]
# run / level table: code and length without the sign bit, length 0 = escape
AC_CODE = np.zeros((64, 256), dtype=np.int64)
AC_LEN = np.zeros((64, 256), dtype=np.int64)
for _v, _c in _DCT.items():
    AC_CODE[_v >> 8, _v & 0xFF], AC_LEN[_v >> 8, _v & 0xFF] = int(_c, 2), len(_c)


# -- selection and timestamps --------------------------------------------------------------------------------------------------
def c_div(a, b):
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def select(pts):
    """main pts p_0 .. p_{N-1} -> (fwd source picture indices, fwd pts, rwd pts); rwd picture j is fwd picture n - 1 - j"""
    N = len(pts)
    if N == 0:
        return [], [], []
    src = list(range(0, N, SPEED))
    f = [int(pts[0]) + c_div(int(pts[j]) - int(pts[0]), SPEED) for j in src]
    n = len(f)
    r = [f[0] + (f[n - 1] - f[n - 1 - j]) for j in range(n)]
    return src, f, r


# -- transform and quantiser ----------------------------------------------------------------------------------------------------
def fdct(blocks):
    """int64 [..., 8, 8] pixels -> [..., 8, 8] coefficients (raster)"""
    x = np.asarray(blocks, dtype=np.int64)
    t = (x @ FDCT_C.T + 128) >> 8
    return (FDCT_C @ t + 32768) >> 16


def quantise(F, qscale):
    """[..., 8, 8] coefficients -> [..., 64] levels in zig-zag order"""
    f = F.reshape(F.shape[:-2] + (64,))[..., ZIGZAG]
    den = qscale * INTRA_Q[ZIGZAG]
    num = 8 * np.abs(f)
    lv = np.minimum((2 * num + den) // (2 * den), 255) * np.sign(f)
    lv[..., 0] = np.minimum((f[..., 0] + 4) >> 3, 255)
    return lv


def picture_blocks(i420):
    """I420 frame -> int64 [12 rows, 22 macroblocks, 6 blocks, 8, 8] in MPEG block order"""
    fr = np.frombuffer(bytes(i420), dtype=np.uint8).astype(np.int64)
    y = fr[:67584].reshape(12, 2, 8, 22, 2, 8).transpose(0, 3, 1, 4, 2, 5).reshape(12, 22, 4, 8, 8)
    cb = fr[67584:84480].reshape(12, 8, 22, 8).transpose(0, 2, 1, 3)[:, :, None]
    cr = fr[84480:].reshape(12, 8, 22, 8).transpose(0, 2, 1, 3)[:, :, None]
    return np.concatenate([y, cb, cr], axis=2)


# -- bitstream -------------------------------------------------------------------------------------------------------------------
def pack(vals, lens):
    """MSB-first bit packing of codes, zero-padded to a byte"""
    vals, lens = np.asarray(vals, dtype=np.int64), np.asarray(lens, dtype=np.int64)
    total = int(lens.sum())
    rep = np.repeat(np.arange(len(lens)), lens)
    j = np.arange(total) - np.repeat(np.cumsum(lens) - lens, lens)
    bits = (vals[rep] >> (lens[rep] - 1 - j)) & 1
    return np.packbits(np.concatenate([bits, np.zeros((-total) % 8, dtype=np.int64)]).astype(np.uint8)).tobytes()


def _dc_code(comp, diff):
    size = int(abs(diff)).bit_length()
    c = DC_CODES[comp][size]
    return (int(c, 2) << size) | (diff if diff > 0 else diff + (1 << size) - 1), len(c) + size


def slice_codes(levels, row, qscale):
    """levels int64 [22, 6, 64] of macroblock row `row` -> the slice's bytes"""
    L = levels.reshape(132, 64)
    keys, vals, lens = [], [], []
    # macroblock headers: address increment 1 ("1") and intra type ("1") before block 0
    mb = np.arange(0, 132, 6)
    keys += [mb * 128, mb * 128 + 1]; vals += [np.ones(22, np.int64)] * 2; lens += [np.ones(22, np.int64)] * 2
    # DC differences: one predictor per component, 128 at the start of the slice
    comp = np.tile([0, 0, 0, 0, 1, 2], 22)
    pred, dvals, dlens = [128, 128, 128], [], []
    for b in range(132):
        d = int(L[b, 0]) - pred[comp[b]]
        pred[comp[b]] = int(L[b, 0])
        v, n = _dc_code(min(comp[b], 1), d)
        dvals.append(v); dlens.append(n)
    keys.append(np.arange(132) * 128 + 2); vals.append(np.array(dvals, np.int64)); lens.append(np.array(dlens, np.int64))
    # AC: run since the previous coded coefficient (the DC counts as coded)
    b, i = np.nonzero(L[:, 1:])
    i = i + 1
    same = np.concatenate([[False], b[1:] == b[:-1]])
    prev = np.where(same, np.concatenate([[0], i[:-1]]), 0)
    run = i - prev - 1
    lv = L[b, i]
    a = np.abs(lv)
    alen = AC_LEN[run, np.minimum(a, 255)]
    coded = (a <= 40) & (alen > 0)
    sign = (lv < 0).astype(np.int64)
    esc8 = (lv >= -127) & (lv <= 127)
    esc_level = np.where(esc8, lv & 0xFF, np.where(lv > 0, lv, (128 << 8) | ((lv + 256) & 0xFF)))
    esc_len = np.where(esc8, 8, 16)
    v = np.where(coded, (AC_CODE[run, np.minimum(a, 255)] << 1) | sign, (1 << (6 + esc_len)) | (run << esc_len) | esc_level)
    n = np.where(coded, alen + 1, 12 + esc_len)
    keys.append(b * 128 + 2 + i); vals.append(v); lens.append(n)
    # end of block
    keys.append(np.arange(132) * 128 + 127); vals.append(np.full(132, 2, np.int64)); lens.append(np.full(132, 2, np.int64))
    keys, vals, lens = np.concatenate(keys), np.concatenate(vals), np.concatenate(lens)
    o = np.argsort(keys, kind="stable")
    head = [(qscale << 1), ]
    body = pack(np.concatenate([head, vals[o]]), np.concatenate([[6], lens[o]]))
    return bytes([0, 0, 1, row + 1]) + body


def header_bytes(aspect, rate):
    """sequence header, closed GOP header and I picture header of every trick picture (HEADER_BYTES)"""
    seq = pack([352, 192, aspect, rate, 0x3FFFF, 1, 20, 0, 0, 0], [12, 12, 4, 4, 18, 1, 10, 1, 1, 1])
    gop = pack([1 << 12, 1, 0, 0], [25, 1, 1, 5])
    pic = pack([0, 1, 0xFFFF, 0], [10, 3, 16, 1])
    return b"\x00\x00\x01\xb3" + seq + b"\x00\x00\x01\xb8" + gop + b"\x00\x00\x01\x00" + pic


def encode_picture(i420, qscale, header):
    F = fdct(picture_blocks(i420))
    levels = quantise(F, qscale)
    return header + b"".join(slice_codes(levels[r], r, qscale) for r in range(12))


def main_codes(es):
    """(aspect, picture-rate) codes of the first sequence header of a video ES"""
    i = es.find(b"\x00\x00\x01\xb3")
    if i < 0 or i + 8 > len(es):
        raise ValueError("no sequence header")
    return es[i + 7] >> 4, es[i + 7] & 15


# -- mux -------------------------------------------------------------------------------------------------------------------------
def pes_header(pts):
    return bytes([0, 0, 1, 0xE0, 0, 0, 0x80, 0x80, 5, 0x21 | ((pts >> 29) & 0x0E), (pts >> 22) & 0xFF, 0x01 | ((pts >> 14) & 0xFE),
                  (pts >> 7) & 0xFF, 0x01 | ((pts << 1) & 0xFE)])


def mux(pictures, pts):
    out, cc = bytearray(), 0
    for es, p in zip(pictures, pts):
        pes = pes_header(int(p) & ((1 << 33) - 1)) + es
        pos, first = 0, True
        while pos < len(pes):
            left = len(pes) - pos
            if left >= 184:
                pkt = bytes([0x47, (0x40 if first else 0) | 0x01, 0x00, 0x10 | (cc & 15)]) + pes[pos:pos + 184]
                pos += 184
            else:
                af = 184 - left
                stuff = bytes([af - 1]) + (bytes([0]) + b"\xff" * (af - 2) if af > 1 else b"")
                pkt = bytes([0x47, (0x40 if first else 0) | 0x01, 0x00, 0x30 | (cc & 15)]) + stuff + pes[pos:]
                pos = len(pes)
            out += pkt
            cc += 1
            first = False
    return bytes(out)


# -- the whole rule ----------------------------------------------------------------------------------------------------------------
def source(ts, oracle):
    """(frames of every main picture from the plain-C oracle, their pts, the main's (aspect, rate) codes)"""
    from tests import pts_cases
    pts = pts_cases.picture_pts(ts)
    frames = oracle.decode_ts(ts, max_frames=max(len(pts), 1))
    assert len(frames) == len(pts), (len(frames), len(pts))
    es, _ = pts_cases.demux(ts)
    return frames, pts, main_codes(es)


_ENCODED = collections.OrderedDict()        # (frame digest, qscale, header) -> picture: mains repeat frames, the encoder is slow


def _encode_cached(frame, qscale, header):
    key = (hashlib.sha256(bytes(frame)).digest(), qscale, header)
    if key in _ENCODED:
        _ENCODED.move_to_end(key)
    else:
        _ENCODED[key] = encode_picture(frame, qscale, header)
        if len(_ENCODED) > 512:
            _ENCODED.popitem(last=False)
    return _ENCODED[key]


def restate(ts, oracle, qscale=DEFAULT_QSCALE, src=None):
    """video.ts -> (video_fwd.ts, video_rwd.ts, fwd source picture indices)"""
    frames, pts, codes = src if src is not None else source(ts, oracle)
    sel, f, r = select(pts)
    hdr = header_bytes(*codes)
    pics = [_encode_cached(frames[j], qscale, hdr) for j in sel]
    return mux(pics, f), mux(pics[::-1], r), sel


def psnr(a, b):
    d = np.frombuffer(bytes(a), np.uint8).astype(np.float64) - np.frombuffer(bytes(b), np.uint8).astype(np.float64)
    mse = float((d * d).mean())
    return float("inf") if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


def fixture(name):
    return open(os.path.join(ROOT, "tests", "golden", name + ".ts"), "rb").read()
