"""The block-level streams of tests/block_cases.py: the restatement against what the UNMODIFIED reference computed
(pinned by tools/make_block_pins.py in tests/golden/block_pins.json), which cases leave the clamp table's domain, and
the census that shows each case reaches every combination it targets."""
import functools
import json
import os

import numpy as np
import pytest

from tests import block_cases as bc
from tests.harness import sha

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "block_pins.json")))
PINNED = [n for n in bc.case_names() if n not in bc.UNPINNED]


@functools.lru_cache(maxsize=None)
def case(name):
    return bc.make(name)


@pytest.mark.parametrize("name", PINNED)
def test_restatement_equals_reference_pins(oracle, name):
    es = case(name)[0]
    pin = PINS[name]
    assert sha(es) == pin["es_sha256"], "%s: the generator no longer writes the pinned stream" % name
    oracle.stats_reset()
    got = oracle.decode_es(es)
    assert oracle.stats().pin_out_of_domain == 0, "%s left the clamp table's domain" % name
    assert got.shape[0] == pin["frames"], name
    for k in range(got.shape[0]):
        assert sha(got[k]) == pin["frame_sha256"][k], "%s picture %d" % (name, k)


def test_pinned_cases_are_exactly_the_in_domain_ones(oracle):
    assert sorted(PINS) == sorted(PINNED)
    for name in bc.UNPINNED:
        oracle.stats_reset()
        oracle.decode_es(case(name)[0])
        assert oracle.stats().pin_out_of_domain > 0, "%s is inside the domain: pin it" % name


def test_integer_idct_port_equals_the_restatement(oracle):
    rng = np.random.RandomState(7)
    pre = np.array(bc.PRESCALE)
    for _ in range(200):
        b = (rng.randint(-2048, 2048, 64) * (rng.rand(64) < 0.3)) * pre
        assert np.array_equal(bc.idct(b), oracle.idct(b)), b


def test_sign_patterns_are_the_transform_extremes():
    """the +2047 / -2048 sign pattern of each output sample gives that sample the largest magnitude the linear transform
    allows (rounding moves it by less than one), and no sample of any of them exceeds the 14,314 pin4 relies on"""
    worst = 0
    for o in range(64):
        for s in (1, -1):
            b = np.array([(2047 if s * bc.L[o][i] > 0 else -2048) if bc.L[o][i] else 0 for i in range(64)]) * np.array(bc.PRESCALE)
            out = bc.idct(b)
            lin = float((bc.L[o] * b).sum())
            assert abs(out[o] - lin) < 1 and abs(lin) > 14000, (o, s, out[o], lin)
            worst = max(worst, int(np.abs(out).max()))
    assert 14000 < worst <= 14314


def test_basis_sweep_census():
    for name, ext in (("basis_small", False), ("basis_extreme", True)):
        c = case(name)[2]
        for p in range(64):
            for path in ("inter", "intra") if p else ("inter",):
                keys = ["%s_pos%d_max" % (path, p), "%s_pos%d_min" % (path, p)] if ext else ["%s_pos%d_small" % (path, p)]
                assert all(c[k] > 0 for k in keys), (name, keys)
            if p:
                assert c["inter_pos0_plus%d" % p] > 0, (name, p)
        assert c["intra_dc_only"] > 0 and c["escape16"] > 0 if ext else True


def test_edge_census():
    c = case("edges")[2]
    for t in bc.EDGE_TARGETS:
        assert c["intra_edge_%d" % t] > 0, t
        for p in bc.EDGE_PREDS:
            assert c["inter_edge_%d_over_%d" % (t, p)] > 0, (t, p)


def test_sign_census():
    ci, cn = case("signs_intra")[2], case("signs_inter")[2]
    for o in range(64):
        assert ci["intra_sign_sample%d" % o] == 2 and cn["inter_sign_sample%d" % o] > 0, o
    assert cn["pred_bytes"] == 256


def test_dc_census():
    for name, plane in (("dc_luma", "luma"), ("dc_chroma", "chroma")):
        c = case(name)[2]
        for band in ("ge32768", "le-32768", "16k_20k"):
            for kind in ("dc_only", "ac_small", "ac_saturated"):
                assert c["%s_dc_%s_%s" % (plane, band, kind)] > 0, (name, band, kind)


def test_prediction_sweep_census():
    for name in ("pred_none", "pred_small", "pred_clamp"):
        c = case(name)[2]
        missing = [(a, b) for a in range(32) for b in range(32) if not c["luma_align_%d_%d" % (a, b)]]
        assert not missing, (name, missing[:8])
        assert all(c["chroma_align_%d_%d" % (a, b)] for a in range(16) for b in range(16)), name
        assert all(c["edge_%s_xy%d" % (e, xy)] for e in bc.EDGES for xy in range(4)), name
        assert c["negative_vector"] > 0
        ref = [k for k in c if k.startswith("ref_dc_byte_")]
        assert all(c["ref_dc_byte_%d" % v] for v in range(249, 256)) and len(ref) > 40, name
    c = case("pred_fullpel")[2]
    assert all(c["luma_align_%d_%d" % (a, b)] for a in range(0, 32, 2) for b in range(0, 32, 2))
    assert all(c["edge_%s_xy0" % e] for e in bc.EDGES)


def test_warp_pair_census():
    c = case("pairs")[2]
    missing = [p for p in bc.PAIRS if not c["pair_%s_%s" % p]]
    assert not missing, missing
    assert c["skip_run_ends_half0"] > 0 and c["skip_run_ends_half1"] > 0 and c["abort_inter"] > 0
