"""Audio path on the CPU (SURVEY.md 8f-3): the oracle restatement (oracle/ef_oracle_audio.c) against the pins the
unmodified reference produced on its own fixtures (tests/golden/audio_pins.json, tools/make_audio_golden.py) and on
synthetic transport streams (tests/golden/ref_pins.json, tools/make_ref_pins.py), and the constant tables."""
import json
import os

import numpy as np
import pytest

from tests.audio_cases import AUDIO_CASES, synthetic_case
from tests.harness import sha

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
REF_PINS = json.load(open(os.path.join(G, "ref_pins.json")))["audio"]


def _masked(pcm, ranges):
    p = pcm.copy()
    for a, b in ranges:
        p[a:b] = 0
    return p


@pytest.mark.parametrize("name", ["splash", "vmedia"])
def test_oracle_matches_reference_pins(oracle, name):
    pins = json.load(open(os.path.join(G, "audio_pins.json")))[name]
    es = oracle.demux_audio_ts(open(os.path.join(G, name + ".ts"), "rb").read())
    assert es.size == pins["es_bytes"] and sha(es) == pins["es_sha256"]
    pcm = oracle.sbc_decode(es)
    assert pcm.size == pins["n_frames"] * 128 and [int(x) for x in pcm[:16]] == pins["pcm_head"]
    assert sha(_masked(pcm, pins["undefined"])) == pins["pcm_sha256_masked"]
    pdm = oracle.pdm(pcm)
    k = pins["pdm_defined_words"]
    assert sha(pdm[:k]) == pins["pdm_sha256_defined"]


def test_sbc_tables_match_reference_arrays():
    """espflix_b200/csrc/ef_sbc_tables.h (closed-form matrix, embedded spec window, offsets) against the reference's
    arrays as committed by tools/make_audio_golden.py: SBC_syn_8[i][j] = matrix[i][j]; SBC_proto_8[i][t] = window[t][i]."""
    import re
    g = json.load(open(os.path.join(G, "sbc_tables.json")))
    hdr = open(os.path.join(ROOT, "espflix_b200", "csrc", "ef_sbc_tables.h")).read()

    def table(name):
        i = hdr.index(name)
        return [int(x) for x in re.findall(r"-?\d+", hdr[hdr.index("{", i):hdr.index("};", i)])]

    assert table("ef_sbc_matrix[16][8]") == g["SBC_syn_8"]
    w = np.array(table("ef_sbc_window[10][8]")).reshape(10, 8)
    assert w.T.reshape(-1).tolist() == g["SBC_proto_8"]
    assert table("ef_sbc_offset8[4][8]") == g["SBC_offset8"]


@pytest.mark.parametrize("case", AUDIO_CASES)
def test_oracle_matches_reference_on_synthetic_streams(oracle, case):
    es, ts = synthetic_case(case)
    ref = REF_PINS[case]
    got_es = oracle.demux_audio_ts(ts)
    assert got_es.size == ref["es_bytes"] and sha(got_es) == ref["es_sha256"]
    if case == "muted_pes":
        assert got_es.size == es.size - 1024              # the second PES (no PTS) is dropped whole; the third one opens the stream again
    pcm = oracle.sbc_decode(got_es)
    assert ref["pcm_samples"] > 0 and pcm.size == ref["pcm_samples"] and sha(pcm) == ref["pcm_sha256"]
    assert sha(oracle.pdm(pcm)) == ref["pdm_sha256"]
