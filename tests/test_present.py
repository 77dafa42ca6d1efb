"""Paced presentation, CPU side: the push / idle restatement in tests/present_cases.py against the pacing pins of the
unmodified reference (tests/golden/pacing_pins.json: flips, per-field hscroll and the SHA-256 of the whole field stream
push_video + video_isr emitted; ref_pins.json["pacing_irregular"]) and against the C restatement of the schedule."""
import hashlib
import json
import os

import numpy as np
import pytest

from espflix_b200 import synth
from tests import present_cases as pc
from tests.oracle_lib import Oracle
from tests.present_cases import irregular_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "pacing_pins.json")))
IRREGULAR = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_pins.json")))["pacing_irregular"]


def pinned_pts(p):
    return 129003 + 3003 * np.arange(p["pictures"], dtype=np.int64)


def all_cases():
    """(pts, modes, ntsc, frame_counter0, tail_fields) of the 5 pinned and the 24 irregular schedules"""
    out = [(pinned_pts(p), p["modes"], p["ntsc"], p["frame_counter0"], p["tail_fields"]) for _, p in sorted(PINS.items())]
    return out + [(pts, modes.tolist(), ntsc, fc0, tail) for pts, ntsc, fc0, modes, tail in irregular_cases()]


def test_restatement_reproduces_the_reference_schedules():
    o = Oracle()
    wants = [PINS[n] for n in sorted(PINS)] + IRREGULAR
    cases = all_cases()
    assert len(cases) == 29
    for i, ((pts, modes, ntsc, fc0, tail), want) in enumerate(zip(cases, wants)):
        f, ff, fl, hs, per, fields = pc.schedule(pts, modes, ntsc, fc0, tail)
        assert (f, ff, fl, hs) == (want["fields"], want["flip_field"], want["flip_line"], want["hscroll"]), i
        cf, cff, cfl, chs = o.paced_schedule(pts, ntsc, fc0, 400, modes=np.array(modes, dtype=np.int32), tail_fields=tail, want_hscroll=True)
        assert (f, ff, fl, hs) == (cf, cff.tolist(), cfl.tolist(), chs.tolist()), i
        assert [fc for fc, _, _ in fields] == [(fc0 + j) & pc.M32 for j in range(f)], i   # consecutive frame counters, none twice


@pytest.mark.parametrize("name", sorted(PINS))
def test_rendered_fields_hash_to_the_reference_stream(name):
    """ties the attribution rule to the reference: every field K2 would render for the restatement's field list,
    concatenated, is the field stream the unmodified reference emitted"""
    p = PINS[name]
    o = Oracle()
    es, off = synth.generate(synth.SEED0 + p["seed"], n_pictures=p["pictures"])
    frames = o.decode_ts(synth.wrap_ts(es, off))
    assert frames.shape[0] == p["pictures"]
    d, r = pc.Display(p["ntsc"], p["frame_counter0"]), pc.Renderer(o, p["ntsc"])
    h, n = hashlib.sha256(), 0
    last = None
    for k, (pts, mode) in enumerate(zip(pinned_pts(p), p["modes"])):
        r.decoded(k, frames[k])
        fields, last, _ = d.push(int(pts), mode)
        for f in fields:
            h.update(r.field(f).tobytes())
            n += 1
    for f in d.idle(((last + 1 + p["tail_fields"] - p["frame_counter0"]) & pc.M32) - n):
        h.update(r.field(f).tobytes())
        n += 1
    assert n == p["fields"]
    assert h.hexdigest() == p["stream_sha256"]


def _run(pts, modes, ntsc, fc0, cuts):
    """pushes, with an idle(0) call at every submit boundary in `cuts` -> the concatenated field list, flips, display"""
    d = pc.Display(ntsc, fc0)
    out, flips = [], []
    for k, (p, m) in enumerate(zip(pts, modes)):
        if k in cuts:
            out += d.idle(0)
        f, a, b = d.push(int(p), int(m))
        out += f
        flips.append((a, b))
    return out, flips, d


def test_concatenation_does_not_depend_on_cuts_or_idle_splits():
    rng = np.random.default_rng(7)
    for i, (pts, modes, ntsc, fc0, tail) in enumerate(all_cases()):
        whole, flips, d = _run(pts, modes, ntsc, fc0, ())
        tail_whole = d.idle(tail + 3)
        for _ in range(3):
            cuts = sorted(set(int(x) for x in rng.integers(1, max(2, len(pts)), size=int(rng.integers(1, 4)))))
            got, gflips, g = _run(pts, modes, ntsc, fc0, cuts)
            assert (got, gflips) == (whole, flips), i
            a = int(rng.integers(0, tail + 4))
            assert g.idle(a) + g.idle(tail + 3 - a) == tail_whole, i


def test_idle_before_the_first_push_emits_blank_fields():
    d = pc.Display(1, 5)
    blank = d.idle(3)
    assert blank == [(5, -1, 0), (6, -1, 0), (7, -1, 0)]
    fields, ff, fl = d.push(129003)
    assert (fields, ff, fl) == ([], 7, 224)             # the idle run stopped at line active_bottom of field 7
    assert d.idle(1) == [(8, 1, 0)]                 # picture 0 lives in store 1


def test_unpushed_picture_is_flagged():
    d = pc.Display(0, 1)
    d.push(129003)
    assert d.push(-1, 0) == ([], None, None) and d.out_of_domain


def test_blank_field_matches_k2_lines():
    o = Oracle()
    for ntsc in (1, 0):
        lines, top, bottom, _ = pc.geometry(ntsc)
        z = np.zeros(101376, dtype=np.uint8)
        b = pc.blank_field(o.field_ex(z, z, ntsc, 0), ntsc).reshape(lines, -1)
        for i in range(top, bottom):
            assert np.array_equal(b[i], b[bottom + ((i - bottom) & 1)])    # same as the blanking lines below the picture
