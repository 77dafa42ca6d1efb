#!/usr/bin/env python3
"""tools/make_keys_golden.py <reference checkout> — tests/golden/keys_pins.json, generated HERE by the UNMODIFIED reference.

tools/ref_keys_harness.cpp compiles espflix.cpp as it is and runs its own loop() and key_event() over every case of tests/keys_cases.py's
pinned scripts (keys_cases.pinned_cases()): per step the file and byte offset Streamer::get() was asked for, the mode flush_picture() was
given, the NVS writes, _nav, _speed, _state, _video_composite_blend, _last_seconds, pos and the saved position of every title. Every
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
from tests import keys_cases as kc  # noqa: E402


def build(ref, tmp):
    lib = os.path.join(tmp, "libefref_keys.so")
    subprocess.run(["g++", "-std=c++14", "-O2", "-w", "-fpermissive", "-fPIC", "-shared", "-I" + os.path.join(ref, "src"), "-o", lib,
                    os.path.join(ROOT, "tools", "ref_keys_harness.cpp")], check=True)
    L = ctypes.CDLL(lib)
    VP, I = ctypes.c_void_p, ctypes.c_int
    L.efref_keys_run.argtypes = [I, VP, VP, I, VP, VP, VP, VP]
    L.efref_keys_sentinel.restype = I
    return L


def run(L, idxs, steps):
    blob = np.frombuffer(b"".join(idxs), dtype=np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(i) for i in idxs])]).astype(np.uint64)
    nec = np.array([s[0] for s in steps], np.int32)
    ended = np.array([s[1] for s in steps], np.int32)
    pts = np.array([s[2] for s in steps], np.int64)
    out = np.zeros((len(steps), 10 + len(idxs)), np.int64)
    L.efref_keys_run(len(idxs), blob.ctypes.data, off.ctypes.data, len(steps), nec.ctypes.data, ended.ctypes.data, pts.ctypes.data,
                     out.ctypes.data)
    return [[int(x) for x in row] for row in out]


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: tools/make_keys_golden.py <reference checkout>")
    ref = os.path.abspath(sys.argv[1])
    pins = {}
    with tempfile.TemporaryDirectory() as tmp:
        L = build(ref, tmp)
        sentinel = L.efref_keys_sentinel()
        for name, (idxs, steps) in sorted(kc.pinned_cases().items()):
            got = run(L, idxs, steps)
            want = kc.restate(idxs, steps, sentinel)
            bad = [(i, s, x, y) for i, (s, x, y) in enumerate(zip(steps, got, want)) if x != y]
            assert not bad, (name, bad[:3])
            pins[name] = {"steps": [list(s) for s in steps], "results": got}
    json.dump({"sentinel": sentinel, "cases": pins}, open(kc.PINS, "w"), indent=None, separators=(",", ":"))
    print(len(pins), "cases")


if __name__ == "__main__":
    main()
