"""The rate-controlled title rule (tests/rate_cases.py) on the CPU: its files hold the bucket by a checker that reads only the file,
each picture gets the smallest quantiser that fits its target, the fallbacks take over when nothing else fits and still decode, the
fixed quantisers' files overflow where these do not, quality at the reference's rate beats the fixed q8, an unlimited budget gives
encode_cases' file, the validation boundary is D_MAX against need_1, and the pins of tests/golden/rate_pins.json hold."""
import functools
import hashlib
import json
import os

import numpy as np
import pytest

from tests import encode_cases as ec
from tests import rate_cases as rc
from tests import trick_cases as tc
from tests.oracle_lib import Oracle, have_ref, ref_decode_ts


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@functools.lru_cache(maxsize=None)
def _restated(name):
    pics, params = rc.pin_cases(Oracle())[name]
    return pics, params, rc.encode_title(pics, Oracle(), **params)


def _bucket(params):
    p = dict(ec.DEFAULT_PARAMS, **rc.RATE_DEFAULTS)
    p.update(params)
    return p["bit_rate"], p["vbv_bits"], p["pts_step"]


@pytest.mark.parametrize("name", rc.PIN_NAMES)
def test_bucket_holds_by_the_file(name):
    pics, params, (ts, es, rec, chosen, census) = _restated(name)
    bad, draw = rc.bucket_violations(ts, *_bucket(params))
    assert bad == [] and draw <= _bucket(params)[1]
    assert [len(e) for e, _ in rc.pictures_of(ts)] == [len(e) for e in es]


@pytest.mark.parametrize("name", rc.PIN_NAMES)
def test_smallest_quantiser_that_fits(name):
    """the bucket state re-derived from the file's own picture sizes: every chosen q is the first candidate within min(t_j, h_j),
    else within h_j, else the fallback"""
    pics, params, (ts, es, rec, chosen, census) = _restated(name)
    p = dict(ec.DEFAULT_PARAMS, **rc.RATE_DEFAULTS)
    p.update(params)
    R, B, step = _bucket(params)
    r, BU, U = R * step, B * rc.U, rc.U
    sizes = [len(e) * 8 * U for e, _ in rc.pictures_of(ts)]
    N, gop = len(sizes), p["gop"]
    qs = range(p["qmin"], p["qmax"] + 1)
    for g0 in range(0, N, gop):
        n = min(gop, N - g0)
        E = 0 if g0 + n == N else BU
        f = BU
        for j in range(n):
            need = E
            for m in range(n - 1, j, -1):
                need = max(rc.P_MIN * 8 * U, rc.P_MIN * 8 * U + need - r)
            hard = min(f, f + r - need)
            L = f + (n - j) * r - E
            soft = L * rc.I_WEIGHT // (rc.I_WEIGHT + n - 1) if j == 0 else L // (n - j)
            s = census[g0 + j]
            fit = [q for q in qs if s[q] * 8 * U <= min(soft, hard)] or [q for q in qs if s[q] * 8 * U <= hard] or [0]
            assert chosen[g0 + j] == fit[0], (name, g0 + j)
            if fit[0]:
                assert s[fit[0]] * 8 * U == sizes[g0 + j]
            f = min(BU, f - sizes[g0 + j] + r)


def test_census_is_every_candidate_not_a_bisection():
    """every candidate is sized, and the choice scans them all: with sizes that are not monotone in q it still takes the smallest q
    that fits, where a bisection would miss it"""
    for name in ("cut", "checker", "gop13"):
        p = dict(rc.RATE_DEFAULTS, **rc.pin_cases(Oracle())[name][1])
        assert all(sorted(s) == list(range(p["qmin"], p["qmax"] + 1)) for s in _restated(name)[2][4])
    U8 = 8 * rc.U
    sizes = {q: 5000 for q in range(3, 32)}
    sizes.update({4: 900, 20: 1000})                            # only q 4 fits below, q 5..19 do not
    r = 1500000 * 3750
    f = 1000 * U8                                               # the last P picture of a title's last GOP with 1,000 bytes left
    q, s = rc.choose(sizes, rc.P_MIN, f, 11, 12, r, 0, 0, 3, 31)
    assert (q, s) == (4, 900)


def test_fallbacks_are_forced_and_decode(oracle):
    pics, params, (ts, es, rec, chosen, census) = _restated("noise/fallback")
    assert chosen[0] == 0 and 0 in chosen[1:]
    for k, e in enumerate(es):
        if chosen[k] == 0 and k % params["gop"]:
            assert len(e) == rc.P_MIN
        if chosen[k] == 0 and k % params["gop"] == 0:
            assert len(e) <= rc.D_MAX
    frames = oracle.decode_ts(ts, max_frames=len(pics) + 1)
    assert len(frames) == len(pics) and np.array_equal(frames, rec)
    for k in range(1, len(pics)):                              # a P fallback is a copy of the picture before it
        if chosen[k] == 0 and k % params["gop"]:
            assert np.array_equal(rec[k], rec[k - 1])


def test_fixed_q8_overflows_where_the_rate_encode_holds(oracle):
    pics, params, (ts, es, rec, chosen, census) = _restated("vmedia/300k")
    fixed = ec.encode_title(pics, oracle)[0]
    assert rc.bucket_violations(fixed, 300000, 250000, 3750)[0] != []
    assert rc.bucket_violations(ts, 300000, 250000, 3750)[0] == []


def test_quality_at_the_reference_rate(oracle):
    pics, params, (ts, es, rec, chosen, census) = _restated("vmedia/default")
    rate_psnr = np.mean(ec.psnr_list(pics, rec))
    fixed_psnr = np.mean(ec.psnr_list(pics, ec.encode_title(pics, oracle)[2]))
    assert rate_psnr > fixed_psnr and rate_psnr > 38.1


@pytest.mark.parametrize("q", [1, 8, 31])
@pytest.mark.parametrize("case", ["cut", "noise", "checker"])
def test_unlimited_budget_is_the_fixed_quantiser_file(oracle, case, q):
    pics = {"cut": lambda: ec.scene_cut(4, 6, 3), "noise": lambda: ec.noise(7, 3), "checker": lambda: ec.checkerboard(3, cell=1)}[case]()
    R, B = 400 * 0x3FFFE, 1023 * 16384
    es = rc.encode_title(pics, oracle, bit_rate=R, vbv_bits=B, qmin=q, qmax=q)[1]
    want = ec.encode_title(pics, oracle, qscale_i=q, qscale_p=q)[1]
    hdr = rc.header_bytes(1, 2, R, B)
    for k, (a, b) in enumerate(zip(es, want)):
        if k % 12:
            assert a == b
        else:
            assert a[:28] == hdr and a[28:] == b[28:] and a[:28] != b[:28]


def test_header_fields():
    h = rc.header_bytes(1, 2, 1500000, 250000)
    bits = int.from_bytes(h[4:12], "big")
    assert (bits >> 14) & 0x3FFFF == 3750 and (bits >> 3) & 0x3FF == 16
    h = rc.header_bytes(1, 2, 1500001, 1)
    bits = int.from_bytes(h[4:12], "big")
    assert (bits >> 14) & 0x3FFFF == 3751 and (bits >> 3) & 0x3FF == 1
    assert h[12:] == tc.header_bytes(1, 2)[12:] and len(h) == tc.HEADER_BYTES


def test_fallback_sizes_from_the_tables():
    """P_MIN: 12 slices of start code, quantiser, two 0x08 macroblocks and an increment of 21; D_MAX: 22 macroblocks of 106 bits"""
    assert 2 + 4 * (len(tc.DC_CODES[0][8]) + 8 + 2) + 2 * (len(tc.DC_CODES[1][8]) + 8 + 2) == 106
    assert rc.D_MAX == 28 + 12 * ((38 + 22 * 106 + 7) // 8) == 3592
    assert rc.P_MIN == 9 + 12 * ((38 + 2 * (1 + 3 + 1 + 1) + len(tc.MBA[21]) + 7) // 8)
    # the I fallback of a picture of 8 x 8 blocks alternating 0 and 255: many DC differences take the size-8 code
    i420 = np.zeros(ec.PICTURE_BYTES, np.uint8)
    i420[:67584] = np.kron((np.add.outer(np.arange(24), np.arange(44)) & 1) * 255, np.ones((8, 8), np.int64)).ravel()
    c = np.kron((np.add.outer(np.arange(12), np.arange(22)) & 1) * 255, np.ones((8, 8), np.int64))
    i420[67584:84480], i420[84480:] = c.ravel(), (255 - c).ravel()
    _, fb = rc.i_sizes(i420, [31])
    assert rc.D_MAX // 2 < fb <= rc.D_MAX


@pytest.mark.parametrize("gop", [1, 2, 12, 13, 1024])
def test_validation_boundary(gop):
    """EF_EINVAL exactly when D_MAX does not fit min(B, B + r - need_1) of a full GOP that ends full"""
    for R in (400, 300000, 689664, 689665, 1500000, 400 * 0x3FFFE):
        for B in (1, 28735, 28736, 40000, 250000, 1023 * 16384):
            r, BU = R * 3750, B * rc.U
            need1 = rc.needs(gop, r, BU)[1] if gop > 1 else BU
            ok = rc.D_MAX * 8 * rc.U <= min(BU, BU + r - need1)
            assert (rc.check(gop, R, B, 3, 31, 3750) is None) == ok
    assert rc.check(1, 689664, 250000, 3, 31, 3750) is None and rc.check(1, 689663, 250000, 3, 31, 3750) is not None
    for bad in [dict(bit_rate=399), dict(bit_rate=400 * 0x3FFFE + 1), dict(vbv_bits=0), dict(vbv_bits=1023 * 16384 + 1), dict(qmin=0),
                dict(qmax=32), dict(qmin=9, qmax=8)]:
        p = dict(gop=12, bit_rate=1500000, vbv_bits=250000, qmin=3, qmax=31, pts_step=3750)
        p.update(bad)
        assert rc.check(**p) is not None, bad


def test_pins():
    """tests/golden/rate_pins.json: the restated files, their quantisers and bytes per picture, and the unmodified reference decoder's
    frames of each file, which the oracle's decode must equal"""
    with open(os.path.join(ec.ROOT, "tests", "golden", "rate_pins.json")) as f:
        pins = json.load(f)
    assert sorted(pins) == sorted(rc.PIN_NAMES)
    o = Oracle()
    for name in rc.PIN_NAMES:
        pics, params, (ts, es, rec, chosen, census) = _restated(name)
        pin = pins[name]
        assert hashlib.sha256(ts).hexdigest() == pin["ts_sha256"], name
        assert chosen == pin["pic_q"] and [len(e) for e in es] == pin["pic_bytes"], name
        frames = o.decode_ts(ts, max_frames=len(pics) + 1)
        assert hashlib.sha256(frames.tobytes()).hexdigest() == pin["ref_decode_sha256"], name
        if have_ref():
            _, ref = ref_decode_ts(ts)
            assert hashlib.sha256(ref.tobytes()).hexdigest() == pin["ref_decode_sha256"], name
