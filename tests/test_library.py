"""The title library's restatement (tests/library_cases.py) against what the unmodified reference's own play(), skip(),
fast_forward(), rewind(), play_pause(), save_pos(), get_index() and pts2offset did on the same scripts
(tests/golden/library_pins.json, tools/make_library_golden.py), and the mistakes those pins catch. CPU only."""
import json

import pytest

from tests import library_cases as lc

PINS = json.load(open(lc.PINS))
CASES = lc.pinned_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_equals_reference(name):
    idx, steps = CASES[name]
    assert [list(s) for s in steps] == PINS[name]["steps"]
    assert lc.restate(idx, steps) == PINS[name]["results"]


def _any_pin_changes(**kw):
    return any(lc.restate(idx, steps, **kw) != PINS[name]["results"] for name, (idx, steps) in CASES.items())


def test_pins_catch_a_single_first_pts_subtraction():
    assert _any_pin_changes(single_first=True)


def test_pins_catch_a_signed_fwd_division():
    assert _any_pin_changes(signed_fwd=True)


def test_pins_catch_a_clamped_skip():
    assert _any_pin_changes(clamp_skip=True)


def test_submit_slices_and_end():
    """a stream's runs cover its file from the sample's packet in budget-sized slices; the last one ends it with pos 0 at speed 0
    and pts2pts(0, speed) in a trick file"""
    idx, _ = CASES["fixture_done"]
    main, fwd = bytes(188 * 50), bytes(188 * 20)
    titles = [lc.Title(idx, main, fwd, main)]
    st = lc.Stream()
    assert st.command(titles, lc.PLAY_AT, 0, 0) == (1, 104)
    start = st.cursor // 188
    runs = []
    while st.state == lc.PLAYING:
        runs.append(st.submit(titles, 7))
    assert [r[2] for r in runs] == [7] * ((50 - start) // 7) + [(50 - start) % 7]
    assert runs[-1][3] and not any(r[3] for r in runs[:-1]) and st.pos == 0 and st.state == lc.ENDED
    assert st.submit(titles, 7) is None
    st.command(titles, lc.FAST_FORWARD)
    while st.state == lc.PLAYING:
        st.submit(titles, 1000)
    assert st.pos == lc.pts2pts(titles[0].hdr, 0, 1) != 0


def test_command_checks_and_ops():
    idx, _ = CASES["fixture_done"]
    titles = [lc.Title(idx, bytes(188), None, bytes(188))]
    st = lc.Stream()
    assert lc.check_command(titles, st, lc.PLAY, 0) and lc.check_command(titles, st, lc.PLAY_AT, 1)
    st.command(titles, lc.PLAY_AT, 0, 0)
    assert lc.check_command(titles, st, lc.FAST_FORWARD) and not lc.check_command(titles, st, lc.REWIND)
    assert lc.check_command(titles, st, lc.RESUME) and lc.check_command(titles, st, lc.SKIP, 0, 2 ** 31)
    assert st.command(titles, lc.PAUSE, last_pts=5) == (0, None) and st.state == lc.PAUSED and st.pos == 5
    assert st.command(titles, lc.RESUME) == (2, None) and st.state == lc.PLAYING
    assert [lc.OP[c] for c in range(8)] == [1, 1, 1, 1, 1, 0, 2, 0]


def test_loop_pause_handshake():
    """loop()'s pause branch (espflix.cpp:906-939, the UI thread): in trick mode every pending key but DONE becomes PLAY"""
    for p in range(7):
        assert lc.loop_command(p, 1) == ((lc.STOP, 0) if p == lc.P_DONE else (lc.PLAY, 0))
        assert lc.loop_command(p, -1) == lc.loop_command(p, 1)
    assert lc.loop_command(lc.P_SKIP_FORWARD, 0) == (lc.SKIP, 30) and lc.loop_command(lc.P_SKIP_BACK, 0) == (lc.SKIP, -30)
    assert lc.loop_command(lc.P_NONE, 0) == (lc.PAUSE, 0) and lc.loop_command(lc.P_REWIND, 0) == (lc.REWIND, 0)
