#!/usr/bin/env python3
"""tools/make_overlay_golden.py <reference checkout> — golden vectors of the paced overlay, generated HERE by the UNMODIFIED
reference: push_video + video_isr + composite() driven under the instant-decoder model by tools/ref_overlay_harness.cpp, with
the overlay globals written between pushes as tests/overlay_cases.py stages them. Builds the reference with the oracle's
recipe (make -C oracle ref), links the harness against those objects in a temporary directory, checks every case against the
restatement (tests/overlay_cases.py rendered by the C checker) and writes tests/golden/overlay_pins.json: per case the flips,
the blend every field was drawn with and the SHA-256 of the whole field stream."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import overlay_cases as oc  # noqa: E402
from tests.oracle_lib import Oracle  # noqa: E402


def build(ref, tmp):
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "ref", "REF=" + os.path.abspath(ref)], check=True, capture_output=True)
    objs = [os.path.join(ROOT, "oracle", "_ref", o + ".o") for o in ("video", "player", "streamer", "sbc_decoder", "ref_video_harness")]
    lib = os.path.join(tmp, "libefref_ovl.so")
    subprocess.run(["g++", "-std=c++14", "-O2", "-w", "-fpermissive", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-I" + os.path.join(ref, "src"),
                    "-o", lib, os.path.join(ROOT, "tools", "ref_overlay_harness.cpp")] + objs + ["-lpthread", "-lm"], check=True)
    L = ctypes.CDLL(lib)
    VP, I = ctypes.c_void_p, ctypes.c_int
    L.efref_paced_overlay.restype = ctypes.c_long
    L.efref_paced_overlay.argtypes = [VP, I, VP, VP, VP, I, I, I, VP, VP, VP, VP, I, VP, VP, VP, VP]
    L.efref_geometry.argtypes = [VP]
    return L


def run(L, case, frames):
    L.efref_video_init(case["ntsc"])
    g = (ctypes.c_int * 8)()
    L.efref_geometry(g)
    per_field = g[0] * g[1]
    allf = np.ascontiguousarray(np.concatenate(frames), dtype=np.uint8)
    pts = np.array([p for _, s in case["segments"] for p in s], dtype=np.int64)
    n = len(pts)
    modes = np.array(case["modes"], dtype=np.int32)
    reset = np.zeros(n, dtype=np.uint8)
    k = 0
    for si, (_, s) in enumerate(case["segments"]):
        reset[k] = 1 if si else 0
        k += len(s)
    n_tail = max(case["tail_cmds"], default=-1) + 1
    cmds = list(case["cmds"]) + [case["tail_cmds"].get(t) for t in range(n_tail)]
    cset = np.zeros(len(cmds), dtype=np.int32)
    cblend, cprog = np.zeros(len(cmds), dtype=np.int32), np.zeros(len(cmds), dtype=np.int32)
    cbm = np.zeros((len(cmds), 1280), dtype=np.uint8)
    for i, c in enumerate(cmds):
        if not c:
            continue
        if c["bitmap"] is not None:
            cset[i] |= 1
            cbm[i] = oc.bitmap(c["bitmap"])
        if c["blend"] is not None:
            cset[i] |= 2
            cblend[i] = c["blend"]
        if c["progress"] is not None:
            cset[i] |= 4
            cprog[i] = c["progress"]
    max_fields = 400
    out = np.zeros(max_fields * per_field, dtype=np.uint16)
    ff, fl = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.int32)
    blend = np.zeros(max_fields + 1, dtype=np.int32)
    r = L.efref_paced_overlay(allf.ctypes.data, n, pts.ctypes.data, modes.ctypes.data, reset.ctypes.data, case["fc0"], max_fields, case["tail_fields"],
                              cset.ctypes.data, cblend.ctypes.data, cprog.ctypes.data, cbm.ctypes.data, n_tail, out.ctypes.data, ff.ctypes.data,
                              fl.ctypes.data, blend.ctypes.data)
    assert 0 <= r < max_fields, r
    return int(r), ff.tolist(), fl.tolist(), out[:r * per_field], blend[:r].tolist()


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: tools/make_overlay_golden.py <reference checkout>")
    o = Oracle()
    pins = {}
    with tempfile.TemporaryDirectory() as tmp:
        L = build(sys.argv[1], tmp)
        for name, case in sorted(oc.cases().items()):
            frames = [o.decode_ts(oc.segment_ts(seed, pts)) for seed, pts in case["segments"]]
            assert [len(f) for f in frames] == [len(p) for _, p in case["segments"]]
            n, ff, fl, stream, blend = run(L, case, frames)
            d, _ = oc.restate(case)
            whole, _, want_blend = oc.rendered(case, frames, o)
            sha = hashlib.sha256(stream.tobytes()).hexdigest()
            assert len(d.emitted) == n, (name, len(d.emitted), n)
            assert blend == want_blend, (name, blend, want_blend)
            assert sha == whole, name
            pins[name] = {"fields": n, "flip_field": ff, "flip_line": fl, "blend": blend, "stream_sha256": sha}
            print(name, n, "fields; blends", sorted(set(blend)))
    json.dump(pins, open(os.path.join(ROOT, "tests", "golden", "overlay_pins.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
