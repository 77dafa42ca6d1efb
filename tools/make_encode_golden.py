"""tools/make_encode_golden.py — writes tests/golden/encode_pins.json: for the restated video.ts (tests/encode_cases.py) of both
fixtures' decoded pictures at the defaults and at qscale 1 and 31, and of the synthetic motion cases, the SHA-256 of the file, the
ES bytes of every picture and the PSNR of every reconstruction against its source (lowest and mean); and the SHA-256 of the frames
the UNMODIFIED reference decoder (oracle/_ref/efref_decode, built by `make -C oracle ref REF=<checkout>`) gives for the file, which
tests/test_encode.py holds the oracle's decode to. CPU only: python tools/make_encode_golden.py"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import encode_cases as ec  # noqa: E402
from tests.oracle_lib import Oracle, have_ref, ref_decode_ts  # noqa: E402


def pins():
    oracle = Oracle()
    if not have_ref():
        raise SystemExit("oracle/_ref is not built: make -C oracle ref REF=<checkout of the reference>")
    out = {}
    for name, pics, params in ec.pin_cases(oracle):
        ts, es, rec, _ = ec.encode_title(pics, oracle, **params)
        info, frames = ref_decode_ts(ts)
        assert frames.shape[0] == len(pics), (name, frames.shape)
        psnr = [min(ec.tc.psnr(a, b), 99.0) for a, b in zip(pics, rec)]
        out[name] = {"ts_sha256": hashlib.sha256(ts).hexdigest(), "picture_bytes": [len(e) for e in es],
                     "min_psnr_db": round(min(psnr), 2), "mean_psnr_db": round(float(np.mean(psnr)), 2),
                     "ref_decode_sha256": hashlib.sha256(frames.tobytes()).hexdigest()}
    return out


if __name__ == "__main__":
    path = os.path.join(ROOT, "tests", "golden", "encode_pins.json")
    with open(path, "w") as f:
        json.dump(pins(), f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path)
