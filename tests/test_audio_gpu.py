"""Audio path on the GPU (SURVEY.md 8f-3): ef_audio_demux_ts / ef_audio_decode through the C-ABI against the oracle
restatement and the pins the unmodified reference produced (tests/golden/audio_pins.json). Bit-exact: integer."""
import hashlib
import json
import os

import numpy as np
import pytest

import espflix_b200
from tests import audio_cases

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


def _masked(pcm, ranges):
    p = pcm.copy()
    for a, b in ranges:
        p[a:b] = 0
    return p


def test_reference_fixture_audio(oracle):
    """the audio of the reference's own embedded streams, both files in one batch: demux on the device, SBC -> PCM -> PDM"""
    pins = json.load(open(os.path.join(G, "audio_pins.json")))
    names = ["splash", "vmedia"]
    ts = [open(os.path.join(G, n + ".ts"), "rb").read() for n in names]
    es = espflix_b200.audio_demux_ts(ts)
    res = espflix_b200.audio_decode(es)
    for n, e, r in zip(names, es, res):
        p = pins[n]
        assert e.size == p["es_bytes"] and hashlib.sha256(e.tobytes()).hexdigest() == p["es_sha256"]
        assert r["frame_size"] == p["frame_size"] and r["n_frames"] == p["n_frames"]
        assert hashlib.sha256(_masked(r["pcm"], p["undefined"]).tobytes()).hexdigest() == p["pcm_sha256_masked"]
        assert hashlib.sha256(r["pdm"][:p["pdm_defined_words"]].tobytes()).hexdigest() == p["pdm_sha256_defined"]
        want = oracle.sbc_decode(e)                      # and sample for sample against the restatement, undefined ranges included (both linear)
        assert np.array_equal(r["pcm"], want)
        assert np.array_equal(r["pdm"], oracle.pdm(want))


def test_batch_of_synthetic_streams(oracle):
    """many streams of different shape in one call: both allocation modes, all frequencies, bit pools 2..120 (sample
    widths 0..16: the allocation's last loop gives width 1 too), inconsistent scale factors (the bit loader runs into the next frame / past the end), rejected
    frames (re-synthesis of the previous samples), empty and sub-frame streams, loud streams (32-bit wrap-around)."""
    streams = []
    for i in range(48):
        streams.append(audio_cases.sbc_stream(5000 + i, 3 + i % 11, bitpool=[2, 7, 12, 28, 31, 60, 97, 120][i % 8], allocation=i & 1, frequency=i % 4,
                                              consistent=i % 3 != 0, bad_frames=(2, 5) if i % 5 == 0 else (), loud=i % 7 == 0))
    streams.append(np.zeros(0, dtype=np.uint8))                          # empty
    streams.append(audio_cases.sbc_stream(1, 1)[:40].copy())             # shorter than its frame
    streams.append(np.full(200, 0x55, dtype=np.uint8))                   # no sync byte at all: rejected
    res = espflix_b200.audio_decode(streams)
    for i, (s, r) in enumerate(zip(streams, res)):
        want = oracle.sbc_decode(s)
        if isinstance(want, int):
            assert r["frame_size"] < 0 and r["n_frames"] == 0, i
            continue
        assert r["pcm"].size == want.size, (i, r["frame_size"], r["n_frames"], want.size)
        assert np.array_equal(r["pcm"], want), "stream %d: first diff at %s" % (i, np.nonzero(r["pcm"] != want)[0][:4])
        assert np.array_equal(r["pdm"], oracle.pdm(want)), i
    assert res[-3]["n_frames"] == 0 and res[-2]["n_frames"] == 0


def test_demux_gating_and_errors(oracle):
    es = audio_cases.sbc_stream(77, 40)
    a = audio_cases.mux_audio_ts(es, drop_pts_on=(1,))
    b = audio_cases.mux_audio_ts(es, pid=0x102)
    got = espflix_b200.audio_demux_ts([a, b])
    assert np.array_equal(got[0], oracle.demux_audio_ts(a)) and got[0].size == es.size - 1024
    assert np.array_equal(got[1], es)
    with pytest.raises(espflix_b200.EspflixError):
        espflix_b200.audio_demux_ts([a[:100]])                            # not a multiple of 188
