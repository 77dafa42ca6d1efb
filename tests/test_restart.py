"""The per-stream restart restated (tests/restart_cases.py) against what the unmodified reference produced on the same programs
(tests/golden/restart_pins.json, tools/make_restart_golden.py), and the tempting wrong rules that the pins reject: the carried
PTS reset to -1, the audio state zeroed as for end_of_stream, and frame stores zero-filled as ef_reset does."""
import json
import os

import pytest

from tests import overlay_cases as oc, restart_cases as rc
from tests.harness import sha
from tests.oracle_lib import Oracle

PINS = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "restart_pins.json")))


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@pytest.fixture(scope="module")
def frames(oracle):
    return {name: [oracle.decode_ts(oc.segment_ts(seed, pts)) for seed, pts in case["segments"]] for name, case in rc.paced_cases().items()}


def test_pins_cover_the_cases():
    assert sorted(PINS["decoder"]) == sorted(rc.decoder_cases())
    assert sorted(PINS["paced"]) == sorted(rc.paced_cases())
    assert {c["ntsc"] for c in rc.paced_cases().values()} == {0, 1} and {c["op"] for c in rc.paced_cases().values()} == {1, 2}


@pytest.mark.parametrize("name", sorted(rc.decoder_cases()))
def test_decoder_restatement_matches_pins(name, oracle):
    progs, pin = rc.decoder_cases()[name], PINS["decoder"][name]
    want = rc.decoder_restate(progs)
    assert want["pushes"] == pin["pushes"]
    assert want["last"] == pin["get_pts"]
    assert [len(p) for p in want["pic_pts"]] == pin["pictures"]
    pcms, pdm = rc.audio_restate(oracle, progs)
    assert [p.size for p in pcms] == pin["pcm_samples"]
    assert [sha(p) for p in pcms] == pin["pcm_sha256"]
    assert sha(pdm) == pin["pdm_sha256"]


@pytest.mark.parametrize("name", sorted(rc.paced_cases()))
def test_paced_restatement_matches_pins(name, oracle, frames):
    case, pin = rc.paced_cases()[name], PINS["paced"][name]
    n, flips, whole = rc.paced_restate(case, frames[name], oracle)
    assert (n, flips, whole) == (pin["fields"], pin["flip_field"], pin["stream_sha256"])


def test_pins_reject_carry_reset():
    """clearing the carried _pts as ef_reset does changes the pts the reference pushes"""
    bad = [n for n, progs in rc.decoder_cases().items() if rc.decoder_restate(progs, carry_reset=True)["pushes"] != PINS["decoder"][n]["pushes"]]
    assert "carry_no_pts" in bad


def test_pins_reject_zeroed_audio_state(oracle):
    """starting each program's audio from a zero state (filter memory, modulator) changes PCM and PDM"""
    changed = 0
    for n, progs in rc.decoder_cases().items():
        pcms, pdm = rc.audio_restate(oracle, progs, zero_state=True)
        changed += [sha(p) for p in pcms] != PINS["decoder"][n]["pcm_sha256"] or sha(pdm) != PINS["decoder"][n]["pdm_sha256"]
    assert changed == len(rc.decoder_cases())


def test_pins_reject_zero_filled_stores(oracle, frames):
    """zero-filling the frame stores and restarting the store phase at a restart changes some pinned field stream"""
    bad = [n for n, case in rc.paced_cases().items() if rc.paced_restate(case, frames[n], oracle, zero_stores=True)[2] != PINS["paced"][n]["stream_sha256"]]
    assert bad
