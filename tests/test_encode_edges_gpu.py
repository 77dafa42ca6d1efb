"""The device encoders on the directed titles of tests/encode_edge_cases.py, and the rate census at every candidate quantiser:
ef_encode_build and ef_trick_build against the restatement byte for byte, and ef_encode_build_rate's choice probed at each candidate's
exact size, so that a census entry wrong at any q (not only the chosen one) changes the choice."""
import functools

import numpy as np
import pytest

from tests import encode_cases as ec
from tests import encode_edge_cases as ee
from tests import rate_cases as rc
from tests import trick_cases as tc
from tests.oracle_lib import Oracle

pytestmark = pytest.mark.gpu


def _capi():
    from espflix_b200 import capi
    return capi


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def _first_difference(a, b):
    return next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), min(len(a), len(b)))


@functools.lru_cache(maxsize=None)
def _mixed():
    """every directed title's pictures, three times over: 39 pictures whose P pictures follow other titles' pictures"""
    return np.concatenate([ee.title(n)[0] for n in ee.NAMES] * 3)


def _titles():
    return [ee.title(n)[0] for n in ee.NAMES] + [_mixed()]


@pytest.mark.parametrize("params", [dict(qscale_i=q, qscale_p=q, gop=g) for q in (1, 8, 31) for g in (2, 12)] + [dict(ee.P_PARAMS)],
                         ids=lambda p: "-".join("%s%d" % (k[0], v) for k, v in sorted(p.items())))
def test_fixed_quantiser(oracle, params):
    """ef_encode_build of every directed title and of one title mixing them all, in one call, equals the restatement"""
    titles = _titles()
    got = _capi().encode_build(titles, **params)
    for name, pics, ts in zip(ee.NAMES + ["mixed"], titles, got):
        want = ec.encode_title(pics, oracle, **params)[0]
        assert ts == want, "%s (%s): first difference at byte %d" % (name, params, _first_difference(ts, want))


def test_trick_build(oracle):
    """ef_trick_build of the mixed title's video.ts (and of a directed one's) equals trick_cases.restate"""
    mains = [_capi().encode_build([_mixed()], gop=12)[0], _capi().encode_build([ee.title("p_blocks")[0]], **ee.P_PARAMS)[0]]
    got = _capi().trick_build(mains)
    for main, (fwd, rwd) in zip(mains, got):
        want_fwd, want_rwd, sel = tc.restate(main, oracle)
        assert fwd == want_fwd and rwd == want_rwd
    assert len(tc.restate(mains[0], oracle)[2]) == 3


# -- the census at every candidate -----------------------------------------------------------------------------------------------------
BIG_RATE = 400 * 0x3FFFE                     # a refill so large that the only cap on a probe picture is the buffer, vbv_bits U
VBV_MAX = 1023 * 16384


def _flat(v):
    return np.full((1, ec.PICTURE_BYTES), v, np.uint8)


# (name, title, gop): the probe picture is the title's last. A flat I picture is the same size with the same reconstruction at every
# q, so the P picture after it has the same census in every call. Noise after flat grey is non-intra in every macroblock; after flat
# 16 its macroblocks all go intra.
PROBES = [("I", lambda: ec.noise(1, 1), 1), ("P", lambda: np.concatenate([_flat(128), ec.noise(3, 1)]), 2),
          ("P intra", lambda: np.concatenate([_flat(16), ec.noise(3, 1)]), 2)]


def _rate(vbv):
    return dict(bit_rate=BIG_RATE, vbv_bits=vbv, qmin=1, qmax=31)


@functools.lru_cache(maxsize=None)
def _probe_census(name):
    """(pictures, gop, the restatement's census {q: bytes} of every picture, fallback bytes of every picture, the probe's analysis)"""
    make, gop = next((m, g) for n, m, g in PROBES if n == name)
    pics = make()
    oracle = Oracle()
    res, decs = ee.encode(pics, oracle, rate=True, gop=gop, **_rate(VBV_MAX))
    fb = []
    for k, pic in enumerate(pics):
        if k % gop == 0:
            fb.append(rc.take_census(tc.i_codes, tc.fdct(tc.picture_blocks(pic)), [31], tc.HEADER_BYTES)[1][-1])
        else:
            an = ec.analyse(ec.planes(pic), ec.planes(res[2][k - 1]), ec.DEFAULT_PARAMS["search"])
            fb.append(rc.take_census(ec.p_codes, an, [31], ec.P_HEADER_BYTES)[1][-1])
    return pics, gop, res[4], [int(x) for x in fb], decs[-1]


def _predict(census, fb, gop, vbv):
    """rate_cases' choice for every picture of a one-GOP probe title at buffer vbv: [(q, bytes)]"""
    n, r, BU = len(census), rc.refill(BIG_RATE, ec.DEFAULT_PARAMS["pts_step"]), vbv * rc.U
    assert n <= gop
    need, f, out = rc.needs(n, r, 0), BU, []
    for j in range(n):
        q, s = rc.choose(census[j], fb[j], f, j, n, r, 0, need[j + 1], 1, 31)
        out.append((q, s))
        f = min(BU, f - s * 8 * rc.U + r)
    return out


@pytest.mark.parametrize("name", [n for n, _, _ in PROBES])
def test_census_at_every_candidate(oracle, name):
    """for every candidate q whose size is below every smaller candidate's, a buffer of exactly s(q) must choose q and one byte less
    must not: the device's choice and bytes equal rate_cases.choose on the restatement's census at both, for every q 1..31"""
    capi = _capi()
    pics, gop, census, fb, dec = _probe_census(name)
    if name == "P":
        assert not dec["intra"].any() and dec["p"]
    if name == "P intra":
        assert dec["intra"].all() and dec["p"]
    s = census[-1]
    probed = [q for q in range(1, 32) if all(s[q] < s[p] for p in range(1, q))]
    assert probed == list(range(1, 32)), probed                 # every candidate, lanes 0..30 of the census warp
    assert min(s.values()) - 1 > rc.D_MAX                        # every bucket below is one the rule accepts
    for q in probed:
        for vbv in (8 * s[q], 8 * s[q] - 8):
            assert rc.check(gop, BIG_RATE, vbv, 1, 31, ec.DEFAULT_PARAMS["pts_step"]) is None
            ts, qs, nb = capi.encode_build_rate([pics], gop=gop, **_rate(vbv))[0]
            want = _predict(census, fb, gop, vbv)
            assert [(int(a), int(b)) for a, b in zip(qs, nb)] == want, (name, q, vbv)
            if vbv == 8 * s[q]:
                assert want[-1] == (q, s[q])
            else:
                assert want[-1][0] != q
    vbv = 8 * s[probed[len(probed) // 2]]
    ts = capi.encode_build_rate([pics], gop=gop, **_rate(vbv))[0][0]
    want = rc.encode_title(pics, oracle, gop=gop, **_rate(vbv))[0]
    assert ts == want, "first difference at byte %d" % _first_difference(ts, want)
