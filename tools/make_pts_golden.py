#!/usr/bin/env python3
"""tools/make_pts_golden.py — pins the pts the UNMODIFIED reference decoder pushes with every picture.

Compiles the reference's src/player.cpp and src/streamer.cpp with oracle/ref_decode_harness.cpp (whose push_video stub
records the pts of every push) into a shared library in a temporary directory, runs it on splash.ts, vmedia.ts and every
in-domain program of tests/pts_cases.py (one process per program: the reference keeps its decoder state in globals and its
decoder thread never returns), and writes tests/golden/pts_pins.json. Each program's pushes are also checked against the
restatement in tests/pts_cases.py before anything is written.

  EF_REFERENCE=<checkout of the reference> python tools/make_pts_golden.py
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

_RUN_ONE = r"""
import ctypes, os, sys
import numpy as np
lib = ctypes.CDLL(sys.argv[1])
ts = np.fromfile(sys.argv[2], dtype=np.uint8)
pts = np.zeros(4096, dtype=np.int64)
lib.efref_decode_ts.restype = ctypes.c_long
lib.efref_decode_ts.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
frames = np.zeros((4096, 352 * 192 * 3 // 2), dtype=np.uint8)
n = lib.efref_decode_ts(ts.ctypes.data, ts.size, 1, frames.ctypes.data, 4096, pts.ctypes.data)
pts[:min(n, 4096)].tofile(sys.argv[3])
sys.stdout.flush()
os._exit(0)                 # the parked decoder thread would block a normal exit
"""


def build_ref(ref, d):
    src = os.path.join(ref, "src")
    flags = ["-std=c++14", "-O2", "-w", "-fpermissive", "-fPIC", "-I" + src]
    objs = []
    for name, extra in (("player.cpp", []), ("streamer.cpp", ["-fno-builtin-putchar", "-include", os.path.join(ROOT, "oracle", "ref_quiet_shim.h")])):
        o = os.path.join(d, name + ".o")
        subprocess.run(["g++"] + flags + extra + ["-c", os.path.join(src, name), "-o", o], check=True)
        objs.append(o)
    o = os.path.join(d, "harness.o")
    subprocess.run(["g++"] + flags + ["-c", os.path.join(ROOT, "oracle", "ref_decode_harness.cpp"), "-o", o], check=True)
    lib = os.path.join(d, "libefref_pts.so")
    subprocess.run(["g++", "-shared", "-o", lib] + objs + [o, "-lpthread"], check=True)
    return lib


def ref_pts(lib, ts, d):
    import numpy as np
    tin, tout = os.path.join(d, "in.ts"), os.path.join(d, "pts.bin")
    open(tin, "wb").write(bytes(ts))
    subprocess.run([sys.executable, "-c", _RUN_ONE, lib, tin, tout], check=True, timeout=300)
    return [int(v) for v in np.fromfile(tout, dtype=np.int64)]


def main():
    ref = os.environ.get("EF_REFERENCE")
    if not ref or not os.path.isdir(os.path.join(ref, "src")):
        raise SystemExit("make_pts_golden.py needs EF_REFERENCE=<checkout of the reference>")
    import __graft_entry__
    __graft_entry__.build()
    from tests import pts_cases
    progs = [(n, open(os.path.join(pts_cases.GOLDEN, n + ".ts"), "rb").read()) for n in pts_cases.FIXTURES]
    progs += [(n, ts) for n, ts in pts_cases.cases() if pts_cases.in_domain(ts)]
    pins = {"rule": "pts(picture) = PTS of the last valid video PES start whose first payload byte lies at ES offset <= code byte + 2; -1 if none",
            "programs": {}}
    with tempfile.TemporaryDirectory() as d:
        lib = build_ref(ref, d)
        for name, ts in progs:
            got = ref_pts(lib, ts, d)
            want = pts_cases.picture_pts(ts)
            if got != want:
                bad = [k for k in range(min(len(got), len(want))) if got[k] != want[k]]
                raise SystemExit("%s: the reference pushed %d pictures, the restatement has %d; first differences at %s" % (name, len(got), len(want), bad[:8]))
            pins["programs"][name] = {"pictures": len(got), "pts": got}
            print("%-24s %4d pictures, %d distinct pts" % (name, len(got), len(set(got))))
    path = os.path.join(ROOT, "tests", "golden", "pts_pins.json")
    with open(path, "w") as f:
        json.dump(pins, f, indent=None, separators=(",", ":"))
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
