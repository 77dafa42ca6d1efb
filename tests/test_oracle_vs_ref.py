"""The oracle restatement against the UNMODIFIED reference on the synthetic coverage streams, plus assertions that
those streams really exercise the paths the reference's fixtures lack. What the reference computed for the same
inputs is pinned in tests/golden/ref_pins.json (SHA-256 of its outputs, tools/make_ref_pins.py)."""
import json
import os

import numpy as np
import pytest

from tests.harness import sha
from tests.synth_cases import COVERAGE, coverage_stream, make, presentation_cases, video_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_pins.json")))


@pytest.mark.parametrize("idx", range(len(COVERAGE)), ids=[c[0] for c in COVERAGE])
def test_port_equals_reference_on_synthetic(oracle, idx):
    name, kw = COVERAGE[idx]
    es, ts = coverage_stream(idx)
    ref = PINS["decode"][name]
    got = oracle.decode_ts(ts)
    assert ref["frames"] == kw["n_pictures"] == got.shape[0]
    assert sha(got) == ref["sha256"], name
    assert sha(oracle.decode_es(es)) == ref["sha256"], "ES path"
    assert np.array_equal(oracle.demux_ts(ts), es), "TS wrapper round trip"


def test_coverage_set_reaches_the_missing_paths(oracle):
    oracle.stats_reset()
    for idx, (name, kw) in enumerate(COVERAGE):
        oracle.decode_es(make(idx, kw)[0])
    s = oracle.stats()
    t = list(s.mb_type)
    assert t[0x11] > 0 and t[0x12] > 0 and t[0x1A] > 0, "macroblock-level quantiser changes"
    assert t[0x01] > 0 and t[0x02] > 0 and t[0x08] > 0 and t[0x0A] > 0
    assert s.full_pel_mbs > 0
    assert s.f_code[3] > 0 and s.f_code[1] > 0
    assert s.escapes16 > 0
    assert s.q2_zero > 0, "quirk Q2 (zero coefficient becomes +1)"
    assert all(v > 0 for v in s.mocomp_xy), "all four half-pel cases"
    assert s.skipped > 0 and s.blocks_dc_only > 0
    assert s.pictures[1] > 0 and s.pictures[2] > 0
    assert s.pin_out_of_domain == 0, "coverage streams must stay inside the reference's defined clamp domain"


def test_reference_video_equals_port_on_random_frames(oracle):
    pins = PINS["video"]
    keys = []
    for key, call in video_cases():
        assert sha(call(oracle)) == pins[key], key
        keys.append(key)
    assert sorted(keys) == sorted(pins)


def test_presentation_extras_port_equals_reference(oracle):
    """SURVEY.md 8f-2: _hscroll two-frame scroll and the composite() overlay / progress bar / fade."""
    pins = PINS["presentation"]
    keys = []
    for key, call in presentation_cases():
        assert sha(call(oracle)) == pins[key], key
        keys.append(key)
    assert sorted(keys) == sorted(pins)
