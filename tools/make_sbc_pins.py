#!/usr/bin/env python3
"""tools/make_sbc_pins.py — pins of the directed SBC streams of tests/sbc_cases.py, generated HERE by the UNMODIFIED
reference (oracle/_ref/efref_audio -es: the real push_audio -> decode_audio -> sbc_decoder chain and pdm_second_order,
one process per stream). Writes tests/golden/sbc_pins.json. Needs oracle/_ref built (make -C oracle ref REF=<checkout>).

Only streams whose output the reference defines are handed to it (sbc_cases.ref_defined): never a bit pool above 128
(its bit allocation does not end) and never a mode other than mono with 12 or 16 blocks (256 samples into mono[128]).
A 4-subband frame, and a bad-sync frame while a 4-subband header is still in force, synthesise nothing and emit
mono[128] uninitialised: those frames are masked out of the PCM hash and the PDM is pinned up to the first of them."""
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import sbc_cases as sc  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "efref_audio")


def run_ref(es):
    with tempfile.TemporaryDirectory() as d:
        p, out = os.path.join(d, "a.sbc"), os.path.join(d, "a.bin")
        open(p, "wb").write(bytes(es))
        subprocess.run([REF, "-es", p, out], check=True, capture_output=True, timeout=60)
        raw = open(out, "rb").read()
    nes, npcm = [int(x) for x in np.frombuffer(raw[:16], dtype=np.uint64)]
    assert nes == len(es)
    pcm = np.frombuffer(raw[16 + nes:16 + nes + 2 * npcm], dtype=np.int16)
    pdm = np.frombuffer(raw[16 + nes + 2 * npcm:], dtype=np.uint16)
    return pcm, pdm


def main():
    ss = sc.streams()
    names = sc.pinned_names()
    assert all(sc.ref_defined(ss[n]) for n in names)

    def one(n):
        pcm, pdm = run_ref(ss[n])
        return n, sc.pin_of(pcm, pdm, sc.ref_undefined_frames(ss[n]))
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        pins = dict(ex.map(one, names))
    with open(os.path.join(ROOT, "tests", "golden", "sbc_pins.json"), "w") as f:
        json.dump(pins, f, sort_keys=True, separators=(",", ":"))
        f.write("\n")
    print(len(pins), "streams pinned,", sum(1 for p in pins.values() if p["undefined"]), "with undefined frames")


if __name__ == "__main__":
    main()
