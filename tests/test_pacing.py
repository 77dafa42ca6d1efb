"""PTS -> field pacing of push_video (SURVEY.md 8f-2; video.cpp:1023-1057, 1165-1177), CPU side: the C restatement
of the schedule against the pins the unmodified reference produced (tools/make_pacing_golden.py) and against what the
reference itself (real push_video / video_isr on two threads) scheduled for irregular PTS (tests/golden/ref_pins.json,
tools/make_ref_pins.py)."""
import json
import os

import numpy as np
import pytest

from tests.oracle_lib import Oracle
from tests.present_cases import irregular_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "pacing_pins.json")))
IRREGULAR = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_pins.json")))["pacing_irregular"]


@pytest.mark.parametrize("name", sorted(PINS))
def test_schedule_matches_reference_pins(name):
    p = PINS[name]
    pts = 129003 + 3003 * np.arange(p["pictures"], dtype=np.int64)
    fields, ff, fl, hs = Oracle().paced_schedule(pts, p["ntsc"], p["frame_counter0"], p["max_fields"], modes=p["modes"], tail_fields=p["tail_fields"], want_hscroll=True)
    assert fields == p["fields"] and ff.tolist() == p["flip_field"] and fl.tolist() == p["flip_line"]
    assert hs.tolist() == p["hscroll"]                    # the poster scroll (_animate / _easd) field by field


def test_schedule_matches_reference_on_irregular_pts():
    o = Oracle()
    cases = list(irregular_cases())
    assert len(cases) == len(IRREGULAR)
    for case, ((pts, ntsc, fc0, modes, tail), want) in enumerate(zip(cases, IRREGULAR)):
        f, ff, fl, hs = o.paced_schedule(pts, ntsc, fc0, 400, modes=modes, tail_fields=tail, want_hscroll=True)
        assert (f, ff.tolist(), fl.tolist()) == (want["fields"], want["flip_field"], want["flip_line"]), (case, ntsc, fc0, pts.tolist())
        assert hs.tolist() == want["hscroll"], (case, modes.tolist())
