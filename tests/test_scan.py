"""K0's start-code rule (tests/scan_cases.py) against the restatement's marker walk (efo_walk) on every start-code case, the
census of what the cases reach, and the restatement against what the unmodified reference computed on them
(tests/golden/scan_pins.json)."""
import json
import os

import numpy as np
import pytest

from tests import scan_cases as sc
from tests.harness import sha

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "scan_pins.json")))
DISPATCHING = {0x00, 0xB3, 0xB7, 0xB8} | set(range(0x01, 0xB0))


def test_rule_equals_the_marker_walk(oracle):
    """the walk's markers whose prefix is 00 00 01 inside the stream are the rule's start codes; every other marker it takes
    inside the stream dispatches nothing, and only the eos_code cases read a picture code from the padding behind it"""
    for c in sc.all_cases():
        es = c.es
        walk, counts = oracle.walk(es)
        assert counts == (sum(m == 0 for _, m in walk), sum(1 <= m <= 0xAF for _, m in walk), sum(m == 0xB3 for _, m in walk))
        inside = [(p // 8, m) for p, m in walk if p % 8 == 0 and p // 8 + 4 <= len(es) and es[p // 8:p // 8 + 3] == b"\x00\x00\x01"]
        assert inside == sc.start_codes(es), c.name
        others = [m for p, m in walk if p + 32 <= 8 * len(es) and (p // 8, m) not in inside]
        assert not DISPATCHING & set(others), c.name
        padding = [m for p, m in walk if p + 32 > 8 * len(es)]
        assert (0x00 in padding) == c.eos_code, c.name


def test_census():
    cases = sc.all_cases()
    geo = [c.census for c in cases if c.name.startswith("geo_")]
    assert {(g["offset"], g["misalign"]) for g in geo} == {(o, m) for o in range(sc.CHUNK) for m in range(16)}
    for o in range(sc.CHUNK):                   # chunk 0 needs the base's slack in front of offset o: misalign <= o
        assert len({min(g["chunk"], 3) for g in geo if g["offset"] == o}) >= 3, o
    assert {g["chunk"] for g in geo} == {0, 1, 2, 3, 6} and sum(g["chunk"] == 0 for g in geo) > 1000
    assert sum(g["lane_straddle"] for g in geo) == 3 * 32 * 16 and sum(g["chunk_straddle"] for g in geo) == 3 * 16
    assert {g["code"] for g in geo} == {"picture", "sequence"}
    for c in cases:
        if c.name.startswith("geo_"):          # the placed code is where the census says, and it is a start code
            g = c.census
            assert (g["at"], 0x00 if g["code"] == "picture" else 0xB3) in sc.start_codes(c.es), c.name
    assert {c.census["zero_run"] for c in cases if c.name.startswith("zeros_")} == set(range(2, 41))
    for c in cases:
        if "ends" in c.census:
            assert c.es.endswith(c.census["ends"]), c.name
    by = {c.name: c for c in cases}
    assert {len(c.es) for c in cases if c.name.startswith("short")} == {0, 1, 2, 3}
    # the pairs: A's last bytes and B's first bytes form a start code only together
    for a, b in (("pair_a_0000", "pair_b_01"), ("pair_a_00", "pair_b_0001")):
        joined = by[a].es + by[b].es
        assert (len(by[a].es) - 2 + (a == "pair_a_00"), 0x00) in sc.raw_hits(joined) and by[b].misalign >= 2
    # every emulation: a raw hit with the intended code inside a sequence header, which the rule drops
    emul = [c for c in cases if c.name.startswith("mat_")]
    seen = set()
    for c in emul:
        rule = sc.start_codes(c.es)
        hidden = [h for h in sc.raw_hits(c.es) if h not in rule]
        assert [m for _, m in hidden] == [c.census["code"]], c.name
        if "offset" in c.census:
            assert (hidden[0][0] + c.misalign) % sc.CHUNK == c.census["offset"], c.name
        seen.add((c.census["kind"], c.census["code"], c.census["where"], c.census["other"]))
    assert {(k, w, o) for k, _, w, o in seen} == {(k, w, o) for k in ("inter", "intra") for w in ("start", "mid") for o in (False, True)}
    assert {x for k, x, _, _ in seen if k == "inter"} == set(sc.EMULATED)
    assert {x for k, x, _, _ in seen if k == "intra"} == {0x00, 0x01, 0x05}
    # the limits
    P, S = sc.LIMIT_PICTURES, sc.LIMIT_SLICES
    for c in cases:
        if c.name.startswith("lim_"):
            n_pic, n_slice, n_seq = sc.census_of(c.es)
            over = n_pic > P or n_slice > P * S or n_seq > P
            assert over == c.census["over"], c.name
            assert n_pic == P + 1 or n_slice == P * S + 1 or n_seq == P + 1 or not over, c.name
    assert sc.census_of(by["lim_pictures_at"].es)[0] == P and sc.census_of(by["lim_slices_at"].es)[1] == P * S
    assert sc.census_of(by["lim_seq_at"].es)[2] == P
    assert sc.census_of(by["lim_seq_end_mid"].es)[0] == 2


@pytest.mark.parametrize("name", sorted(PINS))
def test_restatement_equals_the_reference_pins(oracle, name):
    es = sc.geometry_base() if name == "geo_base" else {c.name: c for c in sc.directed_cases()}[name].es
    assert sha(es) == PINS[name]["es_sha256"], "the case generator changed"
    oracle.stats_reset()
    got = oracle.decode_es(np.frombuffer(es, dtype=np.uint8))
    assert not oracle.stats().pin_out_of_domain
    assert got.shape[0] == PINS[name]["frames"]
    assert [sha(f) for f in got] == PINS[name]["frame_sha256"], name


def test_every_directed_in_domain_case_is_pinned():
    assert {c.name for c in sc.directed_cases() if c.pinned} | {"geo_base"} == set(PINS)


def test_geometry_cases_decode_to_the_base(oracle):
    """the zero bytes the geometry cases add change no picture (a sample of them; the GPU test checks all)"""
    want = oracle.decode_es(np.frombuffer(sc.geometry_base(), dtype=np.uint8))
    for c in sc.geometry_cases()[::97]:
        got = oracle.decode_es(np.frombuffer(c.es, dtype=np.uint8))
        assert np.array_equal(got, want), c.name
