#!/usr/bin/env python3
"""tools/make_library_golden.py <reference checkout> — tests/golden/library_pins.json, generated HERE by the UNMODIFIED reference.

tools/ref_library_harness.cpp compiles espflix.cpp as it is; its own play_pause(), skip(), fast_forward(), rewind(), save_pos(),
get_index() and idx_hdr::pts2offset run every case of tests/library_cases.py's pinned scripts (library_cases.pinned_cases()):
per command the file and byte offset Streamer::get() was asked for, the video.idx byte get_index() read, _speed and pos. Every
result is checked against the restatement before it is written."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import library_cases as lc  # noqa: E402


def build(ref, tmp):
    lib = os.path.join(tmp, "libefref_library.so")
    subprocess.run(["g++", "-std=c++14", "-O2", "-w", "-fpermissive", "-fPIC", "-shared", "-I" + os.path.join(ref, "src"), "-o", lib,
                    os.path.join(ROOT, "tools", "ref_library_harness.cpp")], check=True)
    L = ctypes.CDLL(lib)
    VP, I = ctypes.c_void_p, ctypes.c_int
    L.efref_load.argtypes = [VP, ctypes.c_uint32]
    L.efref_command.argtypes = [I, ctypes.c_int64, ctypes.c_int64]
    L.efref_result.argtypes = [VP, VP, VP, VP, VP]
    return L


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: tools/make_library_golden.py <reference checkout>")
    ref = os.path.abspath(sys.argv[1])
    pins = {}
    with tempfile.TemporaryDirectory() as tmp:
        L = build(ref, tmp)
        f, o, a, s, p = ctypes.c_int(), ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_int(), ctypes.c_int64()
        for name, (idx, steps) in sorted(lc.pinned_cases().items()):
            im = np.frombuffer(idx, dtype=np.uint8).copy()
            L.efref_load(im.ctypes.data, im.size)
            got = []
            for cmd, arg, pts in steps:
                L.efref_command(cmd, arg, pts)
                L.efref_result(ctypes.byref(f), ctypes.byref(o), ctypes.byref(a), ctypes.byref(s), ctypes.byref(p))
                got.append({"file": f.value, "offset": o.value if f.value >= 0 else 0, "idx_at": a.value, "speed": s.value, "pos": p.value})
            want = lc.restate(idx, steps)
            assert got == want, (name, [(i, x, y) for i, (x, y) in enumerate(zip(got, want)) if x != y][:3])
            pins[name] = {"steps": [list(x) for x in steps], "results": got}
            print(name, len(steps))
    json.dump(pins, open(lc.PINS, "w"), indent=1)


if __name__ == "__main__":
    main()
