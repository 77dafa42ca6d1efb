"""The transport-stream parsers at the edges of the packet and PES header, on the CPU: the census of tests/ts_edge_cases.py, the
restatements (tests/pts_cases.py, the C oracle's decode, audio demux and index) against what the unmodified reference made of every
in-domain program (tests/golden/ts_edge_pins.json, tools/make_ts_edge_golden.py), the device's rule on the out-of-domain programs,
and ef_mux_audio's accept / reject decision (a host function) against what the video PES starts allow."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import audio_cases, pts_cases, ts_edge_cases as te
from tests.oracle_lib import Oracle

PINS = os.path.join(pts_cases.GOLDEN, "ts_edge_pins.json")


def _sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


@pytest.fixture(scope="module")
def pins():
    return json.load(open(PINS))


@pytest.fixture(scope="module")
def progs():
    return te.programs()


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def test_census_reaches_every_shape(progs):
    c = te.census(progs)
    groups = {}
    for k, v in sorted(c.items()):
        groups.setdefault(k.split(":")[0].rstrip("0123456789"), []).append("%s=%d" % (k, v))
    for g, items in groups.items():
        print("%-14s %d shapes, fewest %s" % (g, len(items), min(items, key=lambda s: int(s.rsplit("=", 1)[1]))))
    missing = [k for k in te.census_targets() if not c.get(k)]
    assert not missing, missing


def test_restatements_equal_every_pin(pins, progs, oracle):
    assert sorted(pins) == sorted(n for n in progs if te.in_domain(n))
    for name, p in pins.items():
        ts, roles = progs[name]
        assert te.device_demux(ts) == pts_cases.demux(ts), name            # inside the domain the device's rule is the reference's
        assert pts_cases.picture_pts(ts) == p["pts"] and len(p["pts"]) == p["pictures"], name
        assert len(set(p["pts"])) > p["pictures"] // 2, name
        frames = oracle.decode_ts(ts, max_frames=512)
        assert frames.shape[0] == p["pictures"] and _sha(frames.tobytes()) == p["frames_sha256"], name
        es = oracle.demux_audio_ts(ts)
        assert es.size == p["audio_es_bytes"] and _sha(es) == p["audio_es_sha256"], name
        assert te.device_audio_demux(ts) == bytes(es), name
        pcm = oracle.sbc_decode(es)
        assert pcm.size == p["pcm_samples"] > 0 and _sha(pcm) == p["pcm_sha256"], name
        assert _sha(oracle.pdm(pcm)) == p["pdm_sha256"], name
        if "main" in roles:
            assert te.index_in_domain(ts), name
            ix = oracle.make_index(ts)
            assert [int(v) for v in ix["seq_pts"]] == p["seq_pts"] and [int(v) for v in ix["seq_pos"]] == p["seq_pos"], name
            assert (ix["first_pts"], ix["last_pts"]) == (p["first_pts"], p["last_pts"]), name
            assert _sha(oracle.build_idx([ts, ts, ts])) == p["video_idx_sha256"], name


def test_main_titles_read_the_next_packet(pins, progs):
    """a sequence header's PES start whose header ends at 185..187: the indexer's payload[3] is the next packet's sync or PID
    byte, so the entry is there exactly when that byte is 0xB3"""
    for name in ("main0", "main1"):
        ts, _ = progs[name]
        seq = set(pins[name]["seq_pos"])
        seen = 0
        for k in range(len(ts) // 188 - 1):
            d = ts[188 * k:188 * k + 188]
            if ((d[1] << 8) | d[2]) & 0x1FFF != 0x100 or not d[1] & 0x40 or not d[3] & 0x10:
                continue
            o = 5 + d[4] if d[3] & 0x20 else 4
            pay = o + 9 + d[o + 8]
            if pay >= 185:
                seen += 1
                assert (k in seq) == (ts[188 * k + pay + 3] == 0xB3), (name, k, pay)
        assert seen > 0


def test_out_of_domain_programs(progs):
    """each ood program is a base program plus three packets the reference reads past; the device takes nothing from them, so
    its ES and PES list are the base's, and the three PTS they carry are never latched"""
    base = None
    for name in ("ood_empty_payload", "ood_header_past_end", "ood_adaptation_184", "ood_lost_sync"):
        ts, _ = progs[name]
        assert not te.in_domain(name)
        es, pes = te.device_demux(ts)
        if base is None:
            base = (es, pes)
        assert (es, pes) == base, name
        got = te.device_picture_pts(ts)
        assert len(got) == 8 and all(v >= 0 for v in got) and not any(v >= 7000100 for v in got), name
        assert [got[k] for k in (2, 3, 4, 5, 6, 7)] == [7000002, 7000002, 7000004, 7000004, 7000006, 7000006], name
    # audio: two payload_unit_start packets whose adaptation field or PES header runs past the packet give no bytes, but one
    # opens the demux gate inside a PES without PTS and the other shuts it inside a PES with one
    ts, _ = progs["ood_audio_past_end"]
    pk = [ts[i:i + 188] for i in range(0, len(ts), 188)]

    def past_end(d):
        if ((d[1] << 8) | d[2]) & 0x1FFF not in te.AUDIO_PIDS or not d[1] & 0x40 or not d[3] & 0x10:
            return False
        o = 5 + d[4] if d[3] & 0x20 else 4
        return o + 9 > 188 or o + 9 + d[o + 8] > 188

    assert sum(map(past_end, pk)) == 2
    without = b"".join(d for d in pk if not past_end(d))
    got, base_es = te.device_audio_demux(ts), te.device_audio_demux(without)
    assert got != base_es and len(got) > 0 and len(base_es) > 0
    assert te.device_demux(ts) == te.device_demux(without)
    with pytest.raises(ValueError):
        pts_cases.demux(progs["ood_lost_sync"][0])
    with pytest.raises(ValueError):
        pts_cases.demux(progs["ood_empty_payload"][0])


def _bad_prefix(ts):
    """ts with its second video PES start's PTS prefix nibble turned into the DTS form: parse_pts() reads it as -1"""
    ts = bytearray(ts)
    seen = 0
    for k in range(0, len(ts), 188):
        d = ts[k:k + 188]
        if ((d[1] << 8) | d[2]) & 0x1FFF == 0x100 and d[1] & 0x40 and d[3] & 0x10:
            seen += 1
            if seen == 2:
                o = 5 + d[4] if d[3] & 0x20 else 4
                ts[k + o + 9] ^= 0x10
                return bytes(ts)
    raise AssertionError("no second PES start")


def test_mux_audio_accepts_what_the_pes_starts_allow(progs):
    """ef_mux_audio takes a title whose every video PES start carries a PTS parse_pts() reads, and rejects one with a start
    without a PTS, with a malformed one or with a header cut off by the packet; packets with payload_unit_start but no payload
    (adaptation_field_control 0 or 2) are no PES start to the demux and are skipped"""
    from espflix_b200 import capi
    sbc = bytes(audio_cases.sbc_stream(5, 40))
    cases = [(n, te.video_only(ts)) for n, (ts, _) in progs.items()]
    cases.append(("main0_bad_prefix", _bad_prefix(te.video_only(progs["main0"][0]))))
    verdicts = {}
    for name, v in cases:
        want = te.mux_accepts(v)
        try:
            out = capi.mux_audio([v], [sbc])[0]
            got = True
        except capi.EspflixError as e:
            assert e.code == capi.EF_EINVAL, name
            got = False
        assert got == want, name
        verdicts[name] = got
        if got:                                                      # the input packets keep their bytes and order
            assert te.video_only(out) == v, name
    assert verdicts["main0"] and verdicts["main1"] and not verdicts["main0_bad_prefix"]
    assert not verdicts["synth_sweep"] and not verdicts["ood_adaptation_184"]
    # main0 has payload_unit_start packets on 0x100 without payload between its PES packets
    v = te.video_only(progs["main0"][0])
    assert any(((v[k + 1] << 8) | v[k + 2]) & 0x1FFF == 0x100 and v[k + 1] & 0x40 and not v[k + 3] & 0x10 for k in range(0, len(v), 188))
    assert np.frombuffer(v, np.uint8).size % 188 == 0
