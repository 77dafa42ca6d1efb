"""The presentation-timestamp rule, restated on the CPU (tests/pts_cases.py), against the pts the unmodified reference pushes
with every picture (tests/golden/pts_pins.json, tools/make_pts_golden.py)."""
import bisect
import json
import os

import pytest

from tests import pts_cases

PINS = os.path.join(pts_cases.GOLDEN, "pts_pins.json")


@pytest.fixture(scope="module")
def pins():
    return json.load(open(PINS))["programs"]


@pytest.fixture(scope="module")
def programs():
    progs = {n: open(os.path.join(pts_cases.GOLDEN, n + ".ts"), "rb").read() for n in pts_cases.FIXTURES}
    progs.update(dict(pts_cases.cases()))
    return progs


def test_restatement_equals_every_pin(pins, programs):
    in_domain = [n for n, ts in programs.items() if pts_cases.in_domain(ts)]
    assert sorted(in_domain) == sorted(pins)
    assert pins["splash"]["pictures"] == 99 and pins["vmedia"]["pictures"] == 72
    for name in in_domain:
        got = pts_cases.picture_pts(programs[name])
        assert len(got) == pins[name]["pictures"], name
        assert got == pins[name]["pts"], name


def _variant(ts, slack):
    """the rule with another latch point (code byte + slack)"""
    es, pes = pts_cases.demux(ts)
    valid = [(o, p) for o, p in pes if p >= 0]
    offs = [o for o, _ in valid]
    return [valid[j - 1][1] if j else -1 for j in (bisect.bisect_right(offs, x + slack) for x in pts_cases.picture_codes(es))]


def _mirror(ts):
    """the one-stream host mirror's latch: the last PES at or before the code byte, a PES without PTS keeps the previous
    picture's value"""
    es, pes = pts_cases.demux(ts)
    out, prev = [], -1
    for x in pts_cases.picture_codes(es):
        j = bisect.bisect_right([o for o, _ in pes], x)
        v = pes[j - 1][1] if j else -1
        prev = v if v >= 0 else prev
        out.append(prev)
    return out


def test_pins_tell_the_latch_point_apart(pins, programs):
    """the shifted programs put PES boundaries at code byte -4..+4: every other latch point, and the host mirror's rule,
    disagree with the reference somewhere"""
    for name in ("splash_shift", "vmedia_shift", "synth14_shift", "synth20_shift"):
        want = pins[name]["pts"]
        assert _variant(programs[name], 2) == want
        for slack in (0, 1, 3, 4):
            assert _variant(programs[name], slack) != want, (name, slack)
    assert any(_mirror(programs[n]) != pins[n]["pts"] for n in ("splash_shift", "vmedia_shift"))


def test_out_of_domain_program(programs):
    """the first PES has no PTS: the pictures before the first PTS read -1, later ones follow the rule; the reference pushes
    nothing there (Q10), so the program is not pinned"""
    ts = programs["ood_first_without_pts"]
    got = pts_cases.picture_pts(ts)
    assert not pts_cases.in_domain(ts)
    k = next(i for i, v in enumerate(got) if v >= 0)
    assert k >= 1 and all(v == -1 for v in got[:k]) and all(v >= 0 for v in got[k:])
    assert got == _variant(ts, 2)


def test_cases_cover_what_they_claim(programs):
    kinds = set()
    adapt = other = 0
    for name, ts in programs.items():
        for k in range(0, len(ts), 188):
            d = ts[k:k + 188]
            pid = ((d[1] << 8) | d[2]) & 0x1FFF
            if pid != 0x100:
                other += 1
                continue
            adapt += bool(d[3] & 0x20)
            if d[1] & 0x40:
                o = 5 + d[4] if d[3] & 0x20 else 4
                flags = (d[o + 6] << 8) | d[o + 7]
                v = pts_cases.parse_pts(d[o + 9:o + 14], flags) if flags & 0x80 else None
                kinds.add({None: "none", -1: "malformed"}.get(v, "dts" if flags & 0x40 else "pts"))
    assert kinds == {"none", "malformed", "dts", "pts"}
    assert adapt > 100 and other > 100
    dec = pts_cases.picture_pts(programs["synth_decreasing"])
    assert any(b < a for a, b in zip(dec, dec[1:]))
    # every PES start on its own packet; and PES starts that are not at picture boundaries
    es, pes = pts_cases.demux(programs["synth_every_packet"])
    ts = programs["synth_every_packet"]
    assert len(pes) == len(ts) // 188 and all(ts[k + 1] & 0x40 for k in range(0, len(ts), 188))
    es, pes = pts_cases.demux(programs["synth_midslice"])
    codes = pts_cases.picture_codes(es)
    assert sum(1 for o, _ in pes if all(abs(o - x) > 8 for x in codes)) > 20
    assert all(len(pts_cases.cut_points(programs[n])) >= 2 for n in ("splash", "vmedia", "splash_shift", "synth20_shift"))
