#!/usr/bin/env python3
"""tools/make_nav_golden.py <reference checkout> — tests/golden/nav_pins.json, generated HERE by the UNMODIFIED reference.

tools/ref_nav_harness.cpp compiles espflix.cpp as it is; its own nav(), menu(), set_state(), load_poster(), play_pause() and save_pos(),
with loop()'s pause branch, run every case of tests/nav_cases.py's pinned scripts (nav_cases.pinned_cases()): per step the file and
byte offset Streamer::get() was asked for, the mode flush_picture() was given, the NVS writes, _nav, _speed, _state, pos and the saved
position of every title. Every result is checked against the restatement before it is written."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import nav_cases as nc  # noqa: E402


def build(ref, tmp):
    lib = os.path.join(tmp, "libefref_nav.so")
    subprocess.run(["g++", "-std=c++14", "-O2", "-w", "-fpermissive", "-fPIC", "-shared", "-I" + os.path.join(ref, "src"), "-o", lib,
                    os.path.join(ROOT, "tools", "ref_nav_harness.cpp")], check=True)
    L = ctypes.CDLL(lib)
    VP, I = ctypes.c_void_p, ctypes.c_int
    L.efref_nav_load.argtypes = [I, VP, VP]
    L.efref_nav_step.argtypes = [I, ctypes.c_int64, ctypes.c_int64]
    L.efref_nav_result.argtypes = [VP] * 9
    return L


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: tools/make_nav_golden.py <reference checkout>")
    ref = os.path.abspath(sys.argv[1])
    pins = {}
    with tempfile.TemporaryDirectory() as tmp:
        L = build(ref, tmp)
        f, o, m, w, t, s, st, p = (ctypes.c_int(), ctypes.c_uint32(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int(),
                                   ctypes.c_int(), ctypes.c_int64())
        for name, (idxs, steps) in sorted(nc.pinned_cases().items()):
            blob = np.frombuffer(b"".join(idxs), dtype=np.uint8).copy()
            off = np.concatenate([[0], np.cumsum([len(i) for i in idxs])]).astype(np.uint64)
            L.efref_nav_load(len(idxs), blob.ctypes.data, off.ctypes.data)
            nv = np.zeros(len(idxs), np.int64)
            got = []
            for cmd, arg, pts in steps:
                L.efref_nav_step(cmd, arg, pts)
                L.efref_nav_result(*[ctypes.byref(x) for x in (f, o, m, w, t, s, st, p)], nv.ctypes.data)
                got.append({"file": f.value, "offset": o.value if f.value >= 0 else 0, "mode": m.value, "writes": w.value, "title": t.value,
                            "speed": s.value, "state": st.value, "pos": p.value, "nv": [int(x) for x in nv]})
            want = nc.restate(idxs, steps)
            assert got == want, (name, [(i, x, y) for i, (x, y) in enumerate(zip(got, want)) if x != y][:3])
            pins[name] = {"steps": [list(x) for x in steps], "results": got}
            print(name, len(steps))
    json.dump(pins, open(nc.PINS, "w"), indent=1)


if __name__ == "__main__":
    main()
