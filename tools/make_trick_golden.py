"""tools/make_trick_golden.py — writes tests/golden/trick_pins.json: the SHA-256 of the restated video_fwd.ts and video_rwd.ts
(tests/trick_cases.py) of both fixtures at three quantiser scales, with their sizes and the lowest PSNR of a fwd picture against
its source picture. CPU only: python tools/make_trick_golden.py"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import trick_cases  # noqa: E402
from tests.oracle_lib import Oracle  # noqa: E402

QSCALES = (4, trick_cases.DEFAULT_QSCALE, 16)


def pins():
    oracle = Oracle()
    out = {}
    for name in ("vmedia", "splash"):
        ts = trick_cases.fixture(name)
        src = trick_cases.source(ts, oracle)
        for q in QSCALES:
            fwd, rwd, sel = trick_cases.restate(ts, oracle, q, src)
            dec = oracle.decode_ts(fwd, max_frames=len(sel) + 1)
            psnr = min(trick_cases.psnr(dec[k], src[0][j]) for k, j in enumerate(sel))
            out["%s/q%d" % (name, q)] = {"fwd_sha256": hashlib.sha256(fwd).hexdigest(), "rwd_sha256": hashlib.sha256(rwd).hexdigest(),
                                         "fwd_bytes": len(fwd), "pictures": len(sel), "main_bytes": len(ts),
                                         "min_psnr_db": round(psnr, 2)}
    return out


if __name__ == "__main__":
    path = os.path.join(ROOT, "tests", "golden", "trick_pins.json")
    with open(path, "w") as f:
        json.dump(pins(), f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path)
