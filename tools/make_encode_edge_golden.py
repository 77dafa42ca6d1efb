"""tools/make_encode_edge_golden.py — writes tests/golden/encode_edge_pins.json: for the restated video.ts of every directed title of
tests/encode_edge_cases.py, the SHA-256 of the file and the ES bytes of every picture; and the SHA-256 of the frames the UNMODIFIED
reference decoder (oracle/_ref/efref_decode, built by `make -C oracle ref REF=<checkout>`) gives for the file, which
tests/test_encode_edges.py holds the oracle's decode and the decision-level model to. CPU only: python tools/make_encode_edge_golden.py"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import encode_edge_cases as ee  # noqa: E402
from tests.oracle_lib import have_ref, ref_decode_ts  # noqa: E402


def pins():
    if not have_ref():
        raise SystemExit("oracle/_ref is not built: make -C oracle ref REF=<checkout of the reference>")
    out = {}
    for name in ee.NAMES:
        ts, es, rec, _ = ee.restated(name)
        _, frames = ref_decode_ts(ts)
        assert frames.shape[0] == len(es), (name, frames.shape)
        out[name] = {"ts_sha256": hashlib.sha256(ts).hexdigest(), "picture_bytes": [len(e) for e in es],
                     "ref_decode_sha256": hashlib.sha256(frames.tobytes()).hexdigest()}
    return out


if __name__ == "__main__":
    path = os.path.join(ROOT, "tests", "golden", "encode_edge_pins.json")
    with open(path, "w") as f:
        json.dump(pins(), f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path)
