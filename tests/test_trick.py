"""The trick-stream restatement (tests/trick_cases.py) on the CPU: the integer FDCT's range and accuracy, the selection and its
timestamps, the restated files decoded back by the plain-C oracle (and the unmodified reference decoder when it is built), the
index the reference's arithmetic builds over them, and the pinned hashes (tests/golden/trick_pins.json)."""
import hashlib
import json
import math
import os

import numpy as np
import pytest

from tests import library_cases, pts_cases, trick_cases
from tests.oracle_lib import Oracle, RefIndexer, have_ref, have_ref_index, ref_decode_ts

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trick_pins.json")
MAX_FDCT_ERROR = 0.75         # largest |integer FDCT - float DCT| on 100,000 random blocks, measured with this test


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@pytest.fixture(scope="module")
def sources(oracle):
    return {n: trick_cases.source(trick_cases.fixture(n), oracle) for n in ("vmedia", "splash")}


def test_fdct_fits_int32():
    b = trick_cases.FDCT_BOUNDS
    assert b["row_acc"] < 2 ** 22 and b["col_acc"] < 2 ** 28
    rng = np.random.default_rng(7)
    blocks = np.concatenate([rng.integers(0, 256, (20000, 8, 8)), np.zeros((1, 8, 8), np.int64), np.full((1, 8, 8), 255),
                             (np.indices((8, 8)).sum(axis=0)[None] % 2) * 255])
    t = blocks @ trick_cases.FDCT_C.T
    assert np.abs(t).max() <= b["row_acc"]
    t = (t + 128) >> 8
    assert np.abs(t).max() <= b["row_out"]
    assert np.abs(trick_cases.FDCT_C @ t).max() <= b["col_acc"]


def test_fdct_error_against_float_dct():
    C = np.array([[(math.sqrt(1 / 8) if k == 0 else 0.5) * math.cos((2 * n + 1) * k * math.pi / 16) for n in range(8)] for k in range(8)])
    x = np.random.default_rng(1).integers(0, 256, (100000, 8, 8))
    err = np.abs(trick_cases.fdct(x) - C @ x @ C.T).max()
    assert err <= MAX_FDCT_ERROR + 1e-9, err


def test_quantiser_rounds_half_away_from_zero():
    F = np.zeros((8, 8), np.int64)
    F[0, 1] = 11          # 8 * 11 / (2 * 16) = 2.75 -> 3 at qscale 2, zig-zag 1 is raster 1 (matrix entry 16)
    F[1, 0] = -6          # 8 * -6 / (2 * 16) = -1.5 -> -2 (half away from zero)
    F[0, 0] = 1020        # DC 127.5 -> 128
    lv = trick_cases.quantise(F, 2)
    assert lv[0] == 128 and lv[1] == 3 and lv[2] == -2
    F[0, 0] = 2047
    assert trick_cases.quantise(F, 2)[0] == 255


@pytest.mark.parametrize("N", list(range(1, 47)))
def test_selection_every_residue(N):
    rng = np.random.default_rng(N)
    gaps = rng.choice([3003, 3754, 1, 0, -3003, 90000], size=max(N - 1, 0))
    pts = np.concatenate([[129003], 129003 + np.cumsum(gaps)]).astype(np.int64)
    src, f, r = trick_cases.select(pts)
    n = (N - 1) // 15 + 1
    assert src == [15 * k for k in range(n)] and len(f) == len(r) == n
    for k, j in enumerate(src):
        d = int(pts[j]) - int(pts[0])
        assert f[k] == int(pts[0]) + int(d / 15)                     # setpts=PTS/15, truncated toward zero
    assert r[0] == f[0] and r[-1] == f[-1]
    assert [r[j + 1] - r[j] for j in range(n - 1)] == [f[n - 1 - j] - f[n - 2 - j] for j in range(n - 1)]


def test_selection_negative_gap_truncates():
    assert trick_cases.select([1000, 993] + [993] * 13 + [986])[1] == [1000, 1000]


@pytest.mark.parametrize("name", ["vmedia", "splash"])
@pytest.mark.parametrize("qscale", [4, trick_cases.DEFAULT_QSCALE, 16])
def test_restated_files_decode_to_the_source(oracle, sources, name, qscale):
    pin = json.load(open(PINS))["%s/q%d" % (name, qscale)]
    frames, pts, _ = sources[name]
    fwd, rwd, sel = trick_cases.restate(trick_cases.fixture(name), oracle, qscale, sources[name])
    df = oracle.decode_ts(fwd, max_frames=len(sel) + 1)
    dr = oracle.decode_ts(rwd, max_frames=len(sel) + 1)
    assert len(df) == len(dr) == len(sel) == pin["pictures"]
    for k, j in enumerate(sel):
        assert trick_cases.psnr(df[k], frames[j]) >= pin["min_psnr_db"] - 0.005
        assert np.array_equal(dr[len(sel) - 1 - k], df[k])
    _, f, r = trick_cases.select(pts)
    assert pts_cases.picture_pts(fwd) == f and pts_cases.picture_pts(rwd) == r
    if have_ref():
        for ts, dec in ((fwd, df), (rwd, dr)):
            _, ref = ref_decode_ts(ts)
            assert ref.shape[0] == dec.shape[0] and np.array_equal(ref, dec)


@pytest.mark.parametrize("name", ["vmedia", "splash"])
@pytest.mark.parametrize("qscale", [4, trick_cases.DEFAULT_QSCALE, 16])
def test_pins(oracle, sources, name, qscale):
    pin = json.load(open(PINS))["%s/q%d" % (name, qscale)]
    fwd, rwd, _ = trick_cases.restate(trick_cases.fixture(name), oracle, qscale, sources[name])
    assert hashlib.sha256(fwd).hexdigest() == pin["fwd_sha256"] and hashlib.sha256(rwd).hexdigest() == pin["rwd_sha256"]
    assert len(fwd) == pin["fwd_bytes"]


@pytest.mark.parametrize("name", ["vmedia", "splash"])
def test_index_navigates_to_the_nearest_fwd_picture(oracle, sources, name):
    """video.idx of (main, fwd, rwd), by the reference's indexer when it is built (else the oracle's restatement of it): FAST_FORWARD
    from main position x starts at the fwd picture whose pts is nearest x / 15 on the fwd clock (a sequence header every picture)."""
    main = trick_cases.fixture(name)
    fwd, rwd, sel = trick_cases.restate(main, oracle, trick_cases.DEFAULT_QSCALE, sources[name])
    idx = RefIndexer().build_idx([main, fwd, rwd]) if have_ref_index() else oracle.build_idx([main, fwd, rwd])
    h = library_cases.parse(idx)
    _, f, _ = trick_cases.select(sources[name][1])
    starts = [k for k in range(len(fwd) // 188) if fwd[k * 188 + 1] & 0x40]     # packet of every fwd picture's PES start
    ff, fl, fbin, ftrick, _ = h["fwd"]
    assert (ff, fl, ftrick) == (f[0], f[-1], 15)
    vf, vl = h["video"][:2]
    for x in np.linspace(vf, vl, 25).astype(np.int64):
        _, pkt = library_cases.get_index(idx, int(x), 1)
        target = ff + (int(x) - vf) // 15 // fbin * fbin          # the fwd bin pts2offset reads at speed 1
        k = starts.index(pkt)
        assert abs(f[k] - target) == min(abs(v - target) for v in f), (int(x), k)
