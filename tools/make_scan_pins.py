#!/usr/bin/env python3
"""tools/make_scan_pins.py — pins what the UNMODIFIED reference decoder computes on the start-code streams of
tests/scan_cases.py.

Runs oracle/_ref/efref_decode (built by `make -C oracle ref REF=<checkout>` or by build() with EF_REFERENCE=<checkout>) on
synth.wrap_ts() of every pinned directed case and of the one stream every geometry case decodes to (`geo_base`: the geometry
cases only add zero bytes in front of a start code), and writes tests/golden/scan_pins.json: per case the SHA-256 of the ES,
the frame count and the SHA-256 of every pushed picture. Cases where the restatement disagrees with the reference are
printed; what the reference computed is written either way.

  EF_REFERENCE=<checkout of the reference> python tools/make_scan_pins.py
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def sha(a):
    import numpy as np
    return hashlib.sha256(np.ascontiguousarray(a).tobytes() if not isinstance(a, bytes) else a).hexdigest()


def main():
    ref = os.environ.get("EF_REFERENCE")
    if not ref or not os.path.isdir(os.path.join(ref, "src")):
        raise SystemExit("make_scan_pins.py needs EF_REFERENCE=<checkout of the reference>")
    import __graft_entry__
    __graft_entry__.build()
    import numpy as np
    from espflix_b200 import synth
    from tests import oracle_lib, scan_cases
    if not oracle_lib.have_ref():
        raise SystemExit("oracle/_ref is not built: make -C oracle ref REF=$EF_REFERENCE")
    oracle = oracle_lib.Oracle()
    cases = [("geo_base", scan_cases.geometry_base())] + [(c.name, c.es) for c in scan_cases.directed_cases() if c.pinned]
    pins = {}
    for name, es in cases:
        a = np.frombuffer(es, dtype=np.uint8)
        oracle.stats_reset()
        port = oracle.decode_es(a)
        assert not oracle.stats().pin_out_of_domain, name
        _, frames = oracle_lib.ref_decode_ts(synth.wrap_ts(a, scan_cases.unit_offsets(es)))
        pins[name] = {"es_sha256": sha(es), "frames": int(frames.shape[0]), "frame_sha256": [sha(f) for f in frames]}
        if port.shape == frames.shape and all(sha(x) == sha(y) for x, y in zip(port, frames)):
            print("%-32s %2d pictures" % (name, frames.shape[0]))
        else:
            print("%-32s RESTATEMENT DIFFERS: %d / %d pictures" % (name, len(port), len(frames)))
    path = os.path.join(ROOT, "tests", "golden", "scan_pins.json")
    with open(path, "w") as f:
        json.dump(pins, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
