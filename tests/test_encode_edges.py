"""The picture encoders' restatement at its syntax edges (tests/encode_edge_cases.py), on the CPU: the directed titles reach every
target their census names, the decision-level model of the decode equals the oracle's decode of every directed title and of every
encode and rate pin, the files keep the reference's clamp domain and slice rules, and the restated files are pinned."""
import functools
import hashlib
import json
import os

import numpy as np
import pytest

from tests import encode_cases as ec
from tests import encode_edge_cases as ee
from tests import rate_cases as rc
from tests import trick_cases as tc
from tests.oracle_lib import Oracle, have_ref, ref_decode_ts


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@functools.lru_cache(maxsize=None)
def _census(names):
    c = ee.empty_census()
    for name in names:
        ee.census(ee.restated(name)[3], c)
    return c


def _levels(c):
    return {(r, lv): k for r, lv, k in c["levels"]}


def test_census_motion_codes():
    """every motion code -16..15 in both components, and deltas that wrap (|raw delta| > 15) in both directions"""
    c = _census(("p_vectors",))
    assert c["mv_codes"] == set(range(-16, 16))
    for k in (0, 1):
        wrapped = {d for kk, d in c["mv_wrapped"] if kk == k}
        assert min(wrapped) < 0 < max(wrapped) and -16 in wrapped and 15 in wrapped, (k, sorted(wrapped))
    assert c["mv_decoded_ok"]


def test_census_patterns_increments_and_types():
    c = _census(("p_blocks",))
    assert {cbp for cbp, t in c["cbp"] if t & 0x02} == set(range(1, 64))
    assert {t for cbp, t in c["cbp"] if cbp} == {0x02, 0x0A} and {t for cbp, t in c["cbp"] if not cbp} == {0x08}
    assert _census(("p_skips",))["inc"] == set(range(1, 22))
    types = _census(("p_vectors", "p_blocks", "p_skips"))["types"]
    assert {t for p, _, _, t in types if p} == {0x01, 0x02, 0x08, 0x0A}
    assert (True, True, False, 0x08) in types and (True, False, True, 0x08) in types      # first and last of a slice, vector (0, 0)
    # every ordered pair of neighbours: slice start, a skip or a coded macroblock of each type before each coded type
    assert c["pairs"] >= {(a, b) for a in ("start", "skip", 0x01, 0x02, 0x08, 0x0A) for b in (0x01, 0x02, 0x08, 0x0A)}
    assert True in c["dc_carried"] and c["mv_decoded_ok"]                  # an intra macroblock after an intra one in a P picture


def test_census_dc_sizes():
    """every DC size 0..8 in the luma and the chroma table with both signs, carried from macroblock to macroblock"""
    c = _census(("intra_dc",))
    assert c["dc"] == {(t, s, g) for t in (0, 1) for s in range(9) for g in ((0,) if s == 0 else (1, -1))}
    assert c["dc_carried"] == {False}


def test_census_escape_boundaries_q1():
    """run 0 at +-40 (table) / 41 (8-bit escape), +-127 / 128 (8- / 16-bit escape), +-255, and levels quantise clamped to 255"""
    lv = _levels(_census(("intra_q1",)))
    for s in (1, -1):
        assert lv[(0, 40 * s)] == "table" and lv[(0, 41 * s)] == "esc8"
        assert lv[(0, 127 * s)] == "esc8" and lv[(0, 128 * s)] == "esc16" and lv[(0, 255 * s)] == "esc16"
    assert _census(("intra_q1",))["clamped"] == {255, -255}


@pytest.mark.parametrize("q, runs", [(8, range(32)), (31, range(2, 32))])
def test_census_table_boundaries(q, runs):
    """each run at its table's largest level (a table code) and one beyond it (an escape), both signs; at q 31 runs 0 and 1 cannot
    reach them"""
    c = _census(("intra_q%d" % q,))
    lv = _levels(c)
    for r in runs:
        for s in (1, -1):
            assert lv.get((r, s * ee.TABLE_MAX[r])) == "table" and lv.get((r, s * (ee.TABLE_MAX[r] + 1))) == "esc8", (q, r, s)
    assert c["intra_ac_only63"] > 0                           # a block whose only AC coefficient is zig-zag 63


def test_census_long_runs_and_first_coefficients():
    """runs 32..63 (escapes only), and a non-intra block's first coefficient as "1s", as a table code and as an escape"""
    c = _census(tuple(ee.NAMES))
    assert {r for r, _, k in c["levels"] if r >= 32} == set(range(32, 64))
    assert all(k in ("esc8", "esc16") for r, _, k in c["levels"] if r >= 32)
    first = c["first"]
    assert {("1s", 1), ("1s", -1), ("table", 2), ("table", -2)} <= first
    assert any(k == "esc8" and lv > 0 for k, lv in first) and any(k == "esc8" and lv < 0 for k, lv in first)


@pytest.mark.parametrize("name", ee.NAMES)
def test_directed_title_decodes_as_decided(oracle, name):
    """the oracle's decode equals the decision-level model and the reconstruction, inside the clamp domain; no slice holds 23 zero
    bits; the marker walk finds 12 slices a picture; the oracle's coverage shows exactly the restatement's skips"""
    ts, es, rec, decs = ee.restated(name)
    oracle.stats_reset()
    frames = oracle.decode_ts(ts, max_frames=len(es) + 1)
    assert oracle.stats().pin_out_of_domain == 0
    assert np.array_equal(frames, rec)
    model = ee.model_decode(decs)
    bad = [k for k in range(len(es)) if not np.array_equal(model[k], frames[k])]
    assert not bad, "pictures %s differ from the decision-level model" % bad
    cov = oracle.coverage(8)
    for k, d in enumerate(decs[:8]):
        assert np.array_equal(cov[k], np.where(d["skipped"], 1, 2)), k
    assert ee.census(decs)["max_zero_run"] < 23
    markers, _ = oracle.walk(b"".join(es))
    slices, per = [], None
    for _, code in markers:
        if code == 0x00:
            per = []
            slices.append(per)
        elif 0x01 <= code <= 0xAF:
            per.append(code)
    assert slices == [list(range(1, 13))] * len(es)


_ENCODE_PINS = sorted(json.load(open(os.path.join(tc.ROOT, "tests", "golden", "encode_pins.json"))))


@pytest.mark.parametrize("name", _ENCODE_PINS)
def test_model_on_encode_pins(oracle, name):
    """the model, from the restatement's decisions alone, equals the oracle's decode of every pinned encode"""
    pics, params = {n: (p, q) for n, p, q in ec.pin_cases(oracle)}[name]
    (ts, _, rec, _), decs = ee.encode(pics, oracle, **params)
    assert np.array_equal(ee.model_decode(decs), rec)


@pytest.mark.parametrize("name", rc.PIN_NAMES)
def test_model_on_rate_pins(oracle, name):
    """the same for every pinned rate encode, each picture at its chosen quantiser or its fallback"""
    pics, params = rc.pin_cases(oracle)[name]
    res, decs = ee.encode(pics, oracle, rate=True, **params)
    assert np.array_equal(ee.model_decode(decs), res[2])


def test_domain_search():
    """the furthest pre-clamp samples the domain search found stay inside -256..511 (a search, not a bound); the largest
    excursions are reported"""
    res = ee.domain_results()
    lo = min(s for (_, _, _, t), (s, _, _) in res.items() if t < 0)
    hi = max(s for (_, _, _, t), (s, _, _) in res.items() if t > 0)
    n = sum(k for _, k, _ in res.values())
    print("domain search: %d blocks, pre-clamp samples %d .. %d" % (n, lo, hi))
    for key, (s, _, _) in sorted(res.items()):
        print("  q %d %s pred %d toward %d: %d" % (key[0], "intra" if key[1] else "non-intra", key[2], key[3], s))
    assert -256 <= lo and hi <= 511
    for (q, intra, pred, t), (s, _, blk) in res.items():       # the found blocks decode as the search scored them
        got = ee._block_eval(blk[None], q, intra, pred)[0]
        assert (got.min() if t < 0 else got.max()) == s


_PINS = json.load(open(os.path.join(tc.ROOT, "tests", "golden", "encode_edge_pins.json")))


@pytest.mark.parametrize("name", ee.NAMES)
def test_restatement_equals_pins(oracle, name):
    """the restated file and its picture sizes are pinned (tools/make_encode_edge_golden.py), and the oracle decodes it to the frames
    the unmodified reference decoder gave for it"""
    pin = _PINS[name]
    ts, es, rec, _ = ee.restated(name)
    assert hashlib.sha256(ts).hexdigest() == pin["ts_sha256"]
    assert [len(e) for e in es] == pin["picture_bytes"]
    assert hashlib.sha256(rec.tobytes()).hexdigest() == pin["ref_decode_sha256"]


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref (the unmodified reference) is not built")
@pytest.mark.parametrize("name", ["intra_dc", "intra_q1", "p_blocks", "domain_q31"])
def test_reference_decodes_as_decided(name):
    ts, _, rec, decs = ee.restated(name)
    _, frames = ref_decode_ts(ts)
    assert np.array_equal(frames, rec) and np.array_equal(frames, ee.model_decode(decs))
