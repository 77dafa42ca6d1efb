"""The remote's restatement (tests/keys_cases.py) against what the unmodified reference's own loop() and key_event() did on the same
scripts (tests/golden/keys_pins.json, tools/make_keys_golden.py), and the mistakes those pins catch. CPU only."""
import json

import pytest

from tests import keys_cases as kc
from tests import nav_cases as nc

PINS = json.load(open(kc.PINS))
SENTINEL = PINS["sentinel"]
CASES = kc.pinned_cases()


def test_every_case_is_pinned():
    assert sorted(CASES) == sorted(PINS["cases"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_equals_reference(name):
    idxs, steps = CASES[name]
    assert [list(s) for s in steps] == PINS["cases"][name]["steps"]
    assert kc.restate(idxs, steps, SENTINEL) == PINS["cases"][name]["results"]


def _any_pin_changes(**kw):
    return any(kc.restate(idxs, steps, SENTINEL, **kw) != PINS["cases"][name]["results"] for name, (idxs, steps) in CASES.items())


def test_pins_catch_right_in_fast_forward_continuing_it():
    assert _any_pin_changes(ff_continues=True)


def test_pins_catch_up_acting_while_paused():
    assert _any_pin_changes(up_paused=True)


def test_pins_catch_trick_play_showing_180():
    assert _any_pin_changes(trick_blend_180=True)


def test_pins_catch_last_seconds_kept_on_play():
    assert _any_pin_changes(no_zero_on_play=True)


def test_pins_catch_done_ignored_on_key_0():
    assert _any_pin_changes(done_needs_key=True)


def test_key_event_table():
    """the pins run every NEC code the scripts hold through key_event(); the restated table maps exactly the seven Apple codes"""
    assert {kc.key_of(n) for n in kc.NEC.values()} == set(kc.KEYS)
    assert kc.key_of(0) == 0 and kc.key_of(kc.NEC_OTHER) == 0
    assert all(kc.key_of(n ^ 0x8000) == kc.key_of(n) for n in kc.NEC.values())   # bit 15 is not part of the 7-bit code


def test_refusals_and_ignored_streams():
    """what ef_library_command would refuse does nothing; IDLE and a poster-less ENDED stream ignore every key"""
    idx = CASES["row_ends"][0][0]
    titles = [nc.Title(idx, bytes(188), None, None, bytes(188)), nc.Title(idx, bytes(188), bytes(188), bytes(188), None)]
    nv = nc.new_nv(2, 1)
    st = kc.Stream()
    assert st.key(titles, kc.KEY_PLAY, nv=nv)["done"] == kc.NOTHING and st.state == nc.IDLE
    st.command(titles, nc.NAV, 0, nv=nv)
    r = st.key(titles, kc.KEY_RIGHT, nv=nv)                                   # title 1 has no poster
    assert r["done"] == kc.NOTHING and st.title == 0 and r["op"] == 0
    assert st.key(titles, kc.KEY_PLAY, nv=nv)["done"] == nc.PLAY and st.state == nc.PLAYING
    assert st.key(titles, kc.KEY_RIGHT, 0, nv=nv)["done"] == kc.NOTHING        # no fast-forward file
    assert st.key(titles, kc.KEY_PLAY, 0, nv=nv)["done"] == nc.PAUSE and st.state == nc.PAUSED
    st.title = 1
    assert st.key(titles, kc.KEY_MENU, nv=nv)["done"] == kc.NOTHING            # its poster is missing
    st.state = nc.PLAYING
    st.end(titles)
    assert st.state == nc.ENDED and st.key(titles, kc.KEY_PLAY, nv=nv)["done"] == kc.NOTHING and st.state == nc.ENDED
    st.title = 0
    r = st.key(titles, 0, nv=nv)
    assert r["done"] == kc.ENDED_BIT | kc.NOTHING and st.state == nc.POSTER and r["op"] == 1 and r["blend"] == 0
