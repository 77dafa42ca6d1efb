"""The SBC decoder across its whole frame-header domain, on the CPU (tests/sbc_cases.py): the plain-Python bit allocation
against the oracle's (oracle/ef_oracle_audio.c, efo_sbc_bits) at every bit pool 0..255, what the directed streams reach,
the oracle against the pins the unmodified reference produced on them (tools/make_sbc_pins.py ->
tests/golden/sbc_pins.json), and the rule for frames outside the domain."""
import json
import os

import numpy as np
import pytest

from tests import sbc_cases as sc

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PINS = json.load(open(os.path.join(G, "sbc_pins.json")))


def _out(oracle, es):
    """(PCM or the negative code, PDM) of the oracle's whole-stream decode"""
    pcm = oracle.sbc_decode(es)
    return (pcm, None) if isinstance(pcm, int) else (pcm, oracle.pdm(pcm))


def _descent(frequency, allocation, sf):
    """iterations after which the slice loop has counted every slice: from bitslice max(0, max need) down to
    min need - 16, plus the one that adds the last slice count"""
    need = sc.bitneed(frequency, allocation, sf)
    return max(0, max(need)) - min(need) + 18


@pytest.mark.parametrize("allocation", sc.ALLOCATIONS)
@pytest.mark.parametrize("frequency", sc.FREQUENCIES)
def test_allocation_matches_oracle_at_every_bit_pool(oracle, frequency, allocation):
    """every bit pool 0..255 x every scale-factor set: sum and widths equal efo_sbc_bits; above 128 both say -2 at once"""
    for name, sf in sc.SF_SETS.items():
        for bp in range(256):
            a = sc.alloc(frequency, allocation, bp, sf)
            f = sc.frame(sf, frequency=frequency, allocation=allocation, bitpool=bp, size=8)
            total, bits = oracle.sbc_bits(f)
            assert (total, bits) == (a["total"], a["bits"]), (name, bp)
            if bp > sc.MAX_BITPOOL:
                assert total == -2
            else:
                assert 0 <= total <= 128 and a["iterations"] <= _descent(frequency, allocation, sf), (name, bp, a["iterations"])


def test_slice_loop_never_ends_above_128():
    """the reference's loop as written (no bound): every pool <= 128 ends within the descent over the bit needs (at most
    38 iterations), while 129, 200 and 255 are still running after 20,000"""
    for name, sf in sc.SF_SETS.items():
        for fq in sc.FREQUENCIES:
            for al in sc.ALLOCATIONS:
                for bp in (0, 1, 2, 64, 127, 128):
                    a = sc.alloc(fq, al, bp, sf, bounded=False)
                    assert a["total"] is not None and a["iterations"] <= _descent(fq, al, sf) <= 38, (name, fq, al, bp)
    for sf in (sc.SF_SETS["zero"], sc.SF_SETS["all15"], sc.SF_SETS["ascending"]):
        for bp in (129, 200, 255):
            a = sc.alloc(2, 0, bp, sf, bounded=False, cap=20000)
            assert a["total"] is None, bp


def test_census_of_the_directed_streams():
    c = sc.census()
    assert c["widths"] == set(range(17))
    assert c["branches"] >= {"exact", "overshoot", "plus1", "plus2", "plus2_refused", "raise0", "saturated16"}
    for w in range(1, 17):
        for s in sc.IQUANT_SCALES:
            for tag in ("0", "1", "top-1", "top"):
                assert (w, s, tag) in c["iquant"], (w, s, tag)
    assert c["wraps"] == {(16, 15)}                       # the wrap happens, and only at width 16 with scale factor 15
    assert 264 in c["frame_sizes"] and c["overruns"] >= 6 and c["past_end"] >= 3
    assert all(s.size <= sc.ES_LIMIT for s in sc.streams().values())
    # the streaming cases hold back 263 bytes of a 264-byte frame
    es = sc.streams()["max_snr_zero"]
    assert any(sc.held(es, cut) == 263 for cut in sc.PLACED_CUTS["max_snr_zero"])


def test_iquant_against_exact_arithmetic():
    """IQUANT as the reference computes it equals the exact quotient (rounded toward zero) wherever (2 raw + 1) << scale
    fits in 31 bits; where it does not, the 32-bit wrap gives a different, negative-numerator answer"""
    for w in range(1, 17):
        top = (1 << w) - 1
        for s in range(16):
            for raw in sorted({0, 1, max(top - 1, 0), top, top // 2, top // 2 + 1}):
                num = (2 * raw + 1) << s
                exact = num // top - (1 << s)
                got = sc.iquant(raw, w, s)
                if sc.iquant_wraps(raw, w, s):
                    assert (w, s) == (16, 15) and raw >= 32768 and got != exact, (w, s, raw)
                else:
                    assert got == exact, (w, s, raw)


@pytest.mark.parametrize("group", ["alloc", "iquant", "max", "overrun", "kind"])
def test_oracle_matches_reference_pins(oracle, group):
    """the oracle's PCM and PDM equal the reference's on every pinned stream (undefined frames masked); the mode-3 /
    8-block streams are pinned to show that the restatement does not do what the reference does (next test)"""
    ss = sc.streams()
    names = [n for n in PINS if n.startswith(group + "_")]
    assert names
    for n in names:
        pcm, pdm = _out(oracle, ss[n])
        if isinstance(pcm, int):
            assert PINS[n]["samples"] == 0 and pcm < 0, n
            continue
        got = sc.pin_of(pcm, pdm, sc.ref_undefined_frames(ss[n]))
        if n.startswith("kind_m3_b8_") and not n.endswith("_first"):
            assert got["pcm"] != PINS[n]["pcm"], n
        else:
            assert got == PINS[n], n


@pytest.mark.parametrize("place", ["middle", "last", "twice"])
def test_pins_reject_resynthesis_for_joint_stereo(oracle, place):
    """Treating a mode-3 frame with 8 blocks as a rejected frame (re-synthesising the previous 16 blocks, as a bad sync
    byte does) changes its pin: the reference synthesises 8 blocks of each of two channels there, and it does so
    deterministically. So mode 3 is outside the domain, not rejected."""
    ss = sc.streams()
    m3, sync = ss["kind_m3_b8_" + place], ss["kind_sync_" + place]
    resynth = oracle.sbc_decode(sync)                     # the bad-sync twin: the old rule's output for the mode-3 frame
    assert np.array_equal(oracle.sbc_decode(m3), resynth)
    assert sc.pin_of(resynth, oracle.pdm(resynth), []) == PINS["kind_sync_" + place]
    assert PINS["kind_m3_b8_" + place]["samples"] == resynth.size and not PINS["kind_m3_b8_" + place]["undefined"]
    assert PINS["kind_m3_b8_" + place]["pcm"] != PINS["kind_sync_" + place]["pcm"]


@pytest.mark.parametrize("kind", [k for k, _ in sc.KINDS])
def test_out_of_domain_rule(oracle, kind):
    """frame 0 outside the domain: -2 and nothing decoded. A later out-of-domain frame re-synthesises the previous
    accepted samples exactly like a rejected frame (bad sync): the streams then decode to the same PCM."""
    ss = sc.streams()
    code = oracle.sbc_decode(ss["kind_%s_first" % kind])
    if kind in ("sync", "sub4"):
        assert code == -1
        return
    assert code == -2
    for place in ("middle", "last", "twice"):
        got = oracle.sbc_decode(ss["kind_%s_%s" % (kind, place)])
        want = oracle.sbc_decode(ss["kind_sync_%s" % place])
        assert not isinstance(got, int) and np.array_equal(got, want), (kind, place)
        assert got.size == sc.KIND_FRAMES * 128
