"""tools/make_rate_golden.py — writes tests/golden/rate_pins.json: for every case of tests/rate_cases.pin_cases, the SHA-256 of the
restated video.ts, the quantiser (0: the fallback) and ES bytes of every picture, and the SHA-256 of the frames the UNMODIFIED reference
decoder (oracle/_ref/efref_decode, built by `make -C oracle ref REF=<checkout>`) gives for the file, which tests/test_rate.py holds the
oracle's decode to. CPU only: python tools/make_rate_golden.py"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import rate_cases as rc  # noqa: E402
from tests.oracle_lib import Oracle, have_ref, ref_decode_ts  # noqa: E402


def pins():
    oracle = Oracle()
    if not have_ref():
        raise SystemExit("oracle/_ref is not built: make -C oracle ref REF=<checkout of the reference>")
    out = {}
    for name, (pics, params) in rc.pin_cases(oracle).items():
        ts, es, rec, chosen, _ = rc.encode_title(pics, oracle, **params)
        info, frames = ref_decode_ts(ts)
        assert frames.shape[0] == len(pics), (name, frames.shape)
        assert (frames == rec).all(), name
        out[name] = {"ts_sha256": hashlib.sha256(ts).hexdigest(), "pic_q": chosen, "pic_bytes": [len(e) for e in es],
                     "ref_decode_sha256": hashlib.sha256(frames.tobytes()).hexdigest()}
    return out


if __name__ == "__main__":
    path = os.path.join(ROOT, "tests", "golden", "rate_pins.json")
    with open(path, "w") as f:
        json.dump(pins(), f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path)
