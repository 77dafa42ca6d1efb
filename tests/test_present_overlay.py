"""The overlay of paced presentation, CPU side: the restatement in tests/overlay_cases.py, rendered by the C checker, against
the pins of the unmodified reference (tests/golden/overlay_pins.json: flips, the blend of every field and the SHA-256 of the
whole field stream push_video + video_isr + composite() emitted)."""
import json
import os

import numpy as np
import pytest

from tests import overlay_cases as oc
from tests.oracle_lib import Oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "overlay_pins.json")))
CASES = oc.cases()


@pytest.fixture(scope="module")
def frames():
    o = Oracle()
    return {name: [o.decode_ts(oc.segment_ts(seed, pts)) for seed, pts in c["segments"]] for name, c in CASES.items()}


def test_every_case_is_pinned():
    assert sorted(PINS) == sorted(CASES) and len(CASES) == 10


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_reproduces_the_pins(name, frames):
    case, pin = CASES[name], PINS[name]
    d, _ = oc.restate(case)
    whole, _, blend = oc.rendered(case, frames[name], Oracle())
    assert len(d.emitted) == pin["fields"]
    assert d.emitted == [(case["fc0"] + j) & oc.M32 for j in range(pin["fields"])]
    assert blend == pin["blend"]
    assert whole == pin["stream_sha256"]


def test_pins_tell_the_rule_from_the_rejected_ones(frames):
    """latching at the line where the call starts, or at the first field the call emits, gives other fields on some pinned case"""
    o = Oracle()
    for rule in ("start_line", "first_emitted"):
        differ = [n for n in sorted(CASES) if oc.rendered(CASES[n], frames[n], o, rule)[0] != PINS[n]["stream_sha256"]]
        assert differ, rule


def _tail(d, calls_sizes, stage_at=None):
    out = []
    for i, n in enumerate(calls_sizes):
        if stage_at is not None and i == stage_at:
            d.stage()                                       # an empty change
        out += d.idle(n)
    return out


def test_idle_splits_and_empty_changes_change_nothing():
    rng = np.random.default_rng(11)
    for name, case in sorted(CASES.items()):
        base, _ = oc.restate(dict(case, tail_cmds={}, tail_fields=0))
        want_fields = _tail(base, [40])
        want = base.overlays()
        for _ in range(3):
            d, _ = oc.restate(dict(case, tail_cmds={}, tail_fields=0))
            cuts = sorted(set(int(x) for x in rng.integers(0, 40, size=int(rng.integers(1, 5)))))
            sizes = [b - a for a, b in zip([0] + cuts, cuts + [40])]
            got = _tail(d, sizes, stage_at=int(rng.integers(0, len(sizes))))
            assert got == want_fields, name
            assert [(b, p, bm.tobytes()) for b, p, bm in d.overlays()] == [(b, p, bm.tobytes()) for b, p, bm in want], name


def test_blend_counts_down_modulo_2_32():
    assert oc.overlay_blend(5, 0xFFFFFFFE, 1) == 2
    assert oc.overlay_blend(5, 10, 15) == 0 and oc.overlay_blend(-1, 0, 1 << 31) == -1 and oc.overlay_blend(0, 0, 3) == 0


def test_overlay_band_restates_composite():
    """overlay_band, which checks the overlay lines of every stream at the benchmark's batch size, against the C checker"""
    import torch
    o = Oracle()
    z = np.zeros(101376, dtype=np.uint8)
    rng = np.random.default_rng(5)
    for ntsc in (1, 0):
        lines, _, bottom, _ = oc.pc.geometry(ntsc)
        w = 912 if ntsc else 1136
        band = slice((bottom + 2) * w, (bottom + 18) * w)
        template = torch.as_tensor(o.field_ex(z, z, ntsc, 0).astype(np.int32)[band].reshape(16, w))
        combos = [(b, p) for b in (-1, 0, 1, 5, 31, 32, 180) for p in (-(1 << 31), -1, 0, 1, 2, 239, 240, 241, 1 << 30)]
        bms = rng.integers(0, 256, size=(len(combos), 1280), dtype=np.uint8)
        got = oc.overlay_band(template, torch.as_tensor(bms), torch.tensor([b for b, _ in combos]), torch.tensor([p for _, p in combos]), ntsc)
        for i, (b, p) in enumerate(combos):
            want = o.field_ex(z, z, ntsc, 7, 0, bms[i], b, p).astype(np.int32)
            assert np.array_equal(got[i].numpy().reshape(-1), want[band]), (ntsc, b, p)
