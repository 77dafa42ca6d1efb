#!/usr/bin/env python3
"""tools/make_syntax_pins.py — pins what the UNMODIFIED reference decoder computes on the syntax-level streams of
tests/syntax_cases.py.

Runs oracle/_ref/efref_decode (built by `make -C oracle ref REF=<checkout>` or by build() with EF_REFERENCE=<checkout>)
on synth.wrap_ts() of every case whose restatement decode stays inside the clamp table's domain (pin_out_of_domain == 0)
and writes tests/golden/syntax_pins.json: per case the SHA-256 of the generated ES (a change to the generator shows up as a
pin mismatch, not as silent drift), the frame count and the SHA-256 of every pushed picture. Cases where the restatement
disagrees with the reference are printed; what the reference computed is written either way.

  EF_REFERENCE=<checkout of the reference> python tools/make_syntax_pins.py
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
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    ref = os.environ.get("EF_REFERENCE")
    if not ref or not os.path.isdir(os.path.join(ref, "src")):
        raise SystemExit("make_syntax_pins.py needs EF_REFERENCE=<checkout of the reference>")
    import __graft_entry__
    __graft_entry__.build()
    from espflix_b200 import synth
    from tests import oracle_lib, syntax_cases
    if not oracle_lib.have_ref():
        raise SystemExit("oracle/_ref is not built: make -C oracle ref REF=$EF_REFERENCE")
    oracle = oracle_lib.Oracle()
    pins, unpinned = {}, []
    for name in syntax_cases.case_names():
        es, off, _, _ = syntax_cases.make(name)
        oracle.stats_reset()
        port = oracle.decode_es(es)
        if oracle.stats().pin_out_of_domain:
            unpinned.append(name)
            print("%-24s outside the clamp domain: restatement only" % name)
            continue
        _, frames = oracle_lib.ref_decode_ts(synth.wrap_ts(es, off))
        pins[name] = {"es_sha256": sha(es), "frames": int(frames.shape[0]), "frame_sha256": [sha(f) for f in frames]}
        same = port.shape == frames.shape and all(sha(a) == sha(b) for a, b in zip(port, frames))
        if not same:
            bad = [k for k in range(min(len(port), len(frames))) if sha(port[k]) != sha(frames[k])]
            print("%-24s RESTATEMENT DIFFERS: %d / %d pictures, first differences at %s" % (name, len(port), len(frames), bad[:8]))
        else:
            print("%-24s %2d pictures" % (name, frames.shape[0]))
    if unpinned != syntax_cases.UNPINNED:
        print("tests/syntax_cases.py UNPINNED should read", unpinned)
    path = os.path.join(ROOT, "tests", "golden", "syntax_pins.json")
    with open(path, "w") as f:
        json.dump(pins, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
