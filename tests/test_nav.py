"""The poster menu's restatement (tests/nav_cases.py) against what the unmodified reference's own nav(), menu(), set_state(),
load_poster(), play_pause() and save_pos(), with loop()'s pause branch, did on the same scripts (tests/golden/nav_pins.json,
tools/make_nav_golden.py), and the mistakes those pins catch. CPU only."""
import json

import pytest

from tests import library_cases as lc
from tests import nav_cases as nc

PINS = json.load(open(nc.PINS))
CASES = nc.pinned_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_equals_reference(name):
    idxs, steps = CASES[name]
    assert [list(s) for s in steps] == PINS[name]["steps"]
    assert nc.restate(idxs, steps) == PINS[name]["results"]


def _any_pin_changes(**kw):
    return any(nc.restate(idxs, steps, **dict(kw)) != PINS[name]["results"] for name, (idxs, steps) in CASES.items())


def test_pins_catch_the_opposite_scroll_direction():
    assert _any_pin_changes(flip_dir=True)


def test_pins_catch_an_nvs_write_on_pause_or_at_done():
    assert _any_pin_changes(nv_on_pause=True)


def test_pins_catch_an_out_of_range_step_that_moves():
    assert _any_pin_changes(step_clamp=True)


def test_pins_catch_a_poster_on_menu_in_trick_mode():
    assert _any_pin_changes(trick_menu_poster=True)


def test_pins_catch_a_poster_end_that_ends_the_stream():
    assert _any_pin_changes(poster_ends=True)


def _titles(n=3, poster_packets=5):
    idx = CASES["done"][0][0]
    return [nc.Title(idx, bytes(188 * 40), bytes(188 * 10), bytes(188 * 10), bytes(188 * poster_packets) if k != 1 else None) for k in range(n)]


def test_poster_submits_end_once_and_keep_the_stream():
    """a POSTER stream reads its poster in budget-sized runs; the last one carries the end flag and the mode, then nothing more"""
    titles = _titles()
    nv = nc.new_nv(3, 1)
    nv[2][0] = 12345
    st = nc.Stream()
    assert st.command(titles, nc.NAV, 0, nv=nv) == (1, True) and st.mode == 1
    assert st.command(titles, nc.NAV, 2, nv=nv) == (1, True) and st.mode == 2 and st.pos == 12345
    runs = []
    while True:
        r = st.submit(titles, 2)
        if r is None:
            break
        runs.append(r)
    assert [(r[1], r[2], r[3]) for r in runs] == [(0, 2, False), (376, 2, False), (752, 1, True)]
    assert [st.end_mode(r) for r in runs] == [0, 0, 2]
    assert st.state == nc.POSTER and st.pos == 12345 and st.file == nc.POSTER_FILE
    assert st.submit(titles, 2) is None


def test_command_checks_and_ops():
    titles = _titles()
    nv = nc.new_nv(3, 1)
    st = nc.Stream()
    assert nc.check_command(titles, st, nc.MENU) and nc.check_command(titles, st, nc.NAV_STEP, 0, 1)
    assert nc.check_command(titles, st, nc.NAV, 1) and nc.check_command(titles, st, nc.NAV, 3)    # no poster; unknown title
    assert not nc.check_command(titles, st, nc.NAV, 0)
    st.command(titles, nc.NAV, 0, nv=nv)
    assert nc.check_command(titles, st, nc.NAV_STEP, 0, 1)                                       # title 1 has no poster
    assert not nc.check_command(titles, st, nc.NAV_STEP, 0, -1) and not nc.check_command(titles, st, nc.NAV_STEP, 0, 7)
    assert nc.check_command(titles, st, nc.NAV_STEP, 0, 2 ** 31) and nc.check_command(titles, st, nc.RESUME)
    assert st.command(titles, nc.NAV_STEP, arg=-1, nv=nv) == (0, False) and st.title == 0       # nav()'s early return
    assert st.command(titles, nc.MENU, nv=nv) == (0, False) and st.command(titles, nc.PAUSE, nv=nv) == (0, False)
    assert st.state == nc.POSTER
    assert st.command(titles, nc.PLAY, nv=nv)[0] == 1 and st.state == nc.PLAYING and st.file == 1
    assert nc.check_command(titles, st, nc.NAV, 0) and nc.check_command(titles, st, nc.NAV_STEP, 0, 1)
    st.command(titles, nc.FAST_FORWARD, last_pts=lc.parse(titles[0].idx)["video"][0], nv=nv)
    assert st.command(titles, nc.MENU, last_pts=lc.parse(titles[0].idx)["fwd"][0], nv=nv) == (1, False)   # trick mode: play, no poster
    assert st.state == nc.PLAYING and st.speed == 0 and nv[0][0] == st.pos
    st.title = 1
    assert nc.check_command(titles, st, nc.MENU)                                                # speed 0 navs: title 1 has no poster
    assert nc.check_command(titles, st, nc.MENU + 1)


def test_loop_command_with_the_menu():
    """loop()'s pause branch with the poster menu: a pending NAV and DONE become MENU at every speed, the rest as library_cases"""
    for speed in (-1, 0, 1):
        assert nc.loop_command(lc.P_NAV, speed) == (nc.MENU, 0) and nc.loop_command(lc.P_DONE, speed) == (nc.MENU, 0)
        for p in (lc.P_NONE, lc.P_REWIND, lc.P_FAST_FORWARD, lc.P_SKIP_FORWARD, lc.P_SKIP_BACK):
            assert nc.loop_command(p, speed) == lc.loop_command(p, speed)
