"""The overlay clock's restatement (tests/clock_cases.py) against what the unmodified reference's update_progress() and show_time()
produced (tests/golden/clock_pins.json, tools/make_clock_golden.py), and its staging into the restated overlay display."""

import numpy as np

from tests import clock_cases as cc
from tests import overlay_cases as oc
from tests.harness import sha

PINS = cc.pins()
ATLAS, RIGHTS = cc.font()


def test_font_fixture():
    assert ATLAS.shape == (16, 1024) and len(RIGHTS) >= ord(":") - 0x18 + 1
    assert (np.diff(RIGHTS.astype(np.int64)) > 0).all() and 0 < RIGHTS[0] and RIGHTS[-1] <= 1024


def test_update_progress_pins():
    cases = cc.cases()
    assert sorted(cases) == sorted(PINS["update_progress"])
    for name, steps in cases.items():
        want = [(p["sha256"], p["progress"], p["last_seconds"]) for p in PINS["update_progress"][name]]
        assert cc.restate(steps, ATLAS, RIGHTS) == want, name


def test_show_time_pins():
    for p in PINS["show_time"]:
        text = cc.time_text(p["seconds"], p["icon"])
        assert cc.text_width(text, RIGHTS) == p["width"]
        assert sha(cc.render(text, ATLAS, RIGHTS)) == p["sha256"], text
    widths = {cc.text_width(cc.time_text(s, cc.PLAY), RIGHTS) for s in (3723, 36671)}
    assert widths == {68, 76}                                   # one- and two-digit hours fit in a row; three digits wrap
    assert any(p["width"] > 80 for p in PINS["show_time"])


def test_pins_reject_wrong_rules():
    """each rule below changes pinned output: Python's floor division, text clipped at the row's end instead of wrapping into
    the next row, and _last_seconds zeroed by every call"""
    steps = cc.cases()
    pins = {n: [(p["sha256"], p["progress"], p["last_seconds"]) for p in v] for n, v in PINS["update_progress"].items()}
    floor = cc.c_div
    try:
        cc.c_div = lambda a, b: a // b
        assert any(cc.restate(steps[n], ATLAS, RIGHTS) != pins[n] for n in steps)
    finally:
        cc.c_div = floor

    def clipped(text, atlas, rights):
        out, x = np.zeros((16, 80), np.uint8), 0
        for ch in text:
            c = ord(ch) - 0x18
            left, right = int(rights[c - 1]) if c else 0, int(rights[c])
            for j in range(right - left):
                if x + j < 80:
                    col = atlas[:, left + j].astype(np.int32)
                    out[:, x + j] = np.where(col > 0, (cc.COLOR * col) >> 8, 0)
            x += right - left
        return out.reshape(-1)
    assert any(sha(clipped(cc.time_text(p["seconds"], p["icon"]), ATLAS, RIGHTS)) != p["sha256"] for p in PINS["show_time"])
    assert all(sha(clipped(cc.time_text(p["seconds"], p["icon"]), ATLAS, RIGHTS)) == p["sha256"] for p in PINS["show_time"] if p["width"] <= 80)

    def zeroing(steps_):
        return cc.restate([(h, sp, pa, True, pts) for h, sp, pa, _, pts in steps_], ATLAS, RIGHTS)
    assert zeroing(steps["last_seconds_quirk"]) != pins["last_seconds_quirk"]


def test_clock_staging_in_the_restated_display():
    """the clock staged before every call of a pinned overlay case, after the case's own changes: every emitted field shows the
    time text of the latest second that changed, and the progress of the latest call, as of its latch field"""
    case = oc.cases()["ntsc_fade"]
    hdr = cc.header((129003, 129003 + 90000 * 30), (0, 1), (0, 1))
    clk = cc.Clock()
    clk.set(hdr, 0, 1)
    d = oc.OverlayDisplay(case["ntsc"], case["fc0"])
    pts = [129003 + 90000 * k // 4 for k in range(len(case["segments"][0][1]))]          # a second every fourth picture
    shown = []
    for k, p in enumerate(pts):
        oc.stage(d, case["cmds"][k])
        r = clk.step(p)
        d.stage(r[0], None, r[1])
        clk.commit(r)
        shown.append((r[0], r[1]))
        d.push(p, 0)
    d.idle(3)
    ovs = d.overlays()
    assert len(ovs) == len(d.emitted)
    seconds = sorted({p // 90000 for p in pts})
    assert seconds == [1, 2, 3, 4] and sum(1 for bm, _ in shown if bm is not None) == len(seconds)
    assert all(sha(bm) == sha(cc.render(cc.time_text(4, cc.PLAY), ATLAS, RIGHTS)) for _, _, bm in ovs[-3:])
    assert ovs[-1][1] == shown[-1][1] == (pts[-1] * 240) // (129003 + 90000 * 30)
