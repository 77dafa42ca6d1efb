#!/usr/bin/env python3
"""tools/make_ref_pins.py — tests/golden/ref_pins.json: what the UNMODIFIED reference (oracle/_ref, built by
`make -C oracle ref REF=<checkout of the reference>`) computes on the synthetic inputs of the tests that compare the
C restatement with it: decoded coverage streams, composite fields / blits / presentation extras, SBC audio, irregular
PTS pacing and the trick-mode index of fuzzed streams. Inputs come from the case modules the tests draw on, so the pins
and the tests cannot drift apart; outputs are stored as SHA-256 (and short lists where they are small)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = os.path.join(ROOT, "tests", "golden", "ref_pins.json")
SECTIONS = ("decode", "video", "presentation", "audio", "pacing_irregular", "index_fuzzed")
sys.path.insert(0, ROOT)
from tests import audio_cases, oracle_lib, present_cases, synth_cases, ts_cases  # noqa: E402
from tests.harness import sha  # noqa: E402


def ref_audio(ts):
    """efref_audio: demuxed ES, PCM and PDM of one transport stream (one process per run: the reference keeps its state in globals)"""
    with tempfile.TemporaryDirectory() as d:
        p, out = os.path.join(d, "a.ts"), os.path.join(d, "a.bin")
        open(p, "wb").write(ts.tobytes())
        subprocess.run([os.path.join(ROOT, "oracle", "_ref", "efref_audio"), p, out], check=True, capture_output=True, timeout=120)
        raw = open(out, "rb").read()
    nes, npcm = [int(x) for x in np.frombuffer(raw[:16], dtype=np.uint64)]
    es = np.frombuffer(raw[16:16 + nes], dtype=np.uint8)
    pcm = np.frombuffer(raw[16 + nes:16 + nes + 2 * npcm], dtype=np.int16)
    pdm = np.frombuffer(raw[16 + nes + 2 * npcm:], dtype=np.uint16)
    return es, pcm, pdm


def main():
    assert oracle_lib.have_ref() and oracle_lib.have_ref_index(), "build oracle/_ref first: make -C oracle ref REF=<checkout of the reference>"
    pins = {"decode": {}, "video": {}, "presentation": {}, "audio": {}, "pacing_irregular": [], "index_fuzzed": {"tables": {}}}

    for idx, (name, kw) in enumerate(synth_cases.COVERAGE):
        _, ts = synth_cases.coverage_stream(idx)
        info, frames = oracle_lib.ref_decode_ts(ts)
        assert frames.shape[0] == info["frames"]
        pins["decode"][name] = {"frames": int(info["frames"]), "sha256": sha(frames)}

    rv = oracle_lib.RefVideo()
    for key, call in synth_cases.video_cases():
        pins["video"][key] = sha(call(rv))
    for key, call in synth_cases.presentation_cases():
        pins["presentation"][key] = sha(call(rv))

    for case in audio_cases.AUDIO_CASES:
        _, ts = audio_cases.synthetic_case(case)
        es, pcm, pdm = ref_audio(ts)
        pins["audio"][case] = {"es_bytes": int(es.size), "es_sha256": sha(es), "pcm_samples": int(pcm.size), "pcm_sha256": sha(pcm), "pdm_sha256": sha(pdm)}

    for pts, ntsc, fc0, modes, tail in present_cases.irregular_cases():
        frames = np.zeros((len(pts), 101376), dtype=np.uint8)             # content is irrelevant to the schedule
        f, ff, fl, _, hs = rv.paced(frames, pts, ntsc, fc0, 400, want_fields=False, modes=modes, tail_fields=tail, want_hscroll=True)
        pins["pacing_irregular"].append({"fields": int(f), "flip_field": [int(x) for x in ff], "flip_line": [int(x) for x in fl], "hscroll": [int(x) for x in hs]})

    ri = oracle_lib.RefIndexer()
    for seed in ts_cases.FUZZ_SEEDS:
        t = ri.make_index(ts_cases.fuzzed_stream(seed))
        pins["index_fuzzed"]["tables"][str(seed)] = {"first_pts": int(t["first_pts"]), "last_pts": int(t["last_pts"]), "entries": int(t["seq_pts"].size),
                                                     "seq_pts_sha256": sha(t["seq_pts"]), "seq_pos_sha256": sha(t["seq_pos"])}
    img = ri.build_idx(ts_cases.fuzzed_image_files())
    pins["index_fuzzed"]["image"] = {"bytes": len(img), "sha256": sha(img)}

    assert tuple(pins) == SECTIONS
    with open(PINS, "w") as f:
        json.dump(pins, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
