#!/usr/bin/env python3
"""tools/make_sbc_encode_golden.py — pins of the SBC encoder's restatement (tests/sbc_encode_cases.py): for every case of
tests/test_sbc_encode.py, the SHA-256 of the restated SBC and of the PCM the UNMODIFIED reference decoder gives for it
(oracle/_ref/efref_audio on the stream muxed alone into a transport stream by sbc_encode_cases.mux: the reference's demux ->
push_audio -> decode_audio -> sbc_decoder, one process per stream). Writes
tests/golden/sbc_encode_pins.json. Where the TS path leaves the PCM undefined (frames over the 64 bytes decode_audio() probes,
or frames straddling the end of its 4 KB ring), the stream's first frames that fit the ring are handed to the reference's decoder
directly (efref_audio -es) instead. It also pins the title with audio that ef_indexer_cli --encode --audio is checked on, played
through the reference's TS path. Needs oracle/_ref built (make -C oracle ref REF=<checkout>)."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import sbc_encode_cases as se  # noqa: E402
from tests import test_sbc_encode as t  # noqa: E402
from tests.oracle_lib import Oracle  # noqa: E402


REF = os.path.join(ROOT, "oracle", "_ref", "efref_audio")


def run_ref(ts):
    """the reference's PCM for a transport stream"""
    with tempfile.TemporaryDirectory() as d:
        p, out = os.path.join(d, "a.ts"), os.path.join(d, "a.bin")
        open(p, "wb").write(ts)
        subprocess.run([REF, p, out], check=True, capture_output=True, timeout=120)
        raw = open(out, "rb").read()
    nes, npcm = [int(x) for x in np.frombuffer(raw[:16], dtype=np.uint64)]
    return np.frombuffer(raw[16 + nes:16 + nes + 2 * npcm], dtype=np.int16)


def run_ref_es(sbc):
    """the reference's PCM for SBC bytes handed whole to push_audio() (efref_audio -es)"""
    with tempfile.TemporaryDirectory() as d:
        p, out = os.path.join(d, "a.sbc"), os.path.join(d, "a.bin")
        open(p, "wb").write(sbc)
        subprocess.run([REF, "-es", p, out], check=True, capture_output=True, timeout=120)
        raw = open(out, "rb").read()
    nes, npcm = [int(x) for x in np.frombuffer(raw[:16], dtype=np.uint64)]
    return np.frombuffer(raw[16 + nes:16 + nes + 2 * npcm], dtype=np.int16)


def main():
    oracle = Oracle()
    cases = t._all_cases(oracle)

    def one(item):
        name, (x, p) = item
        p = dict(se.DEFAULTS, **p)
        s = se.encode(x, p["frequency"], p["allocation"], p["bitpool"])
        pin = {"sbc": hashlib.sha256(s).hexdigest()[:32], "bytes": len(s)}
        if s and t.ref_defined(len(s), p["bitpool"]):
            pin["pcm"] = t._pin(run_ref(se.mux(b"", s, **p)))
        elif s:
            k = t.es_frames(len(s), p["bitpool"])
            pin["es_frames"] = k
            pin["pcm_es"] = t._pin(run_ref_es(s[:k * se.frame_bytes(p["bitpool"])]))
        return name, pin
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        pins = dict(ex.map(one, cases.items()))
    ts = t.cli_title_ts(oracle)
    pins["title_with_audio"] = {"ts": hashlib.sha256(ts).hexdigest()[:32], "pcm": t._pin(run_ref(ts))}
    with open(os.path.join(ROOT, "tests", "golden", "sbc_encode_pins.json"), "w") as f:
        json.dump(pins, f, sort_keys=True, indent=0)
        f.write("\n")
    print(len(pins), "cases pinned")


if __name__ == "__main__":
    main()
