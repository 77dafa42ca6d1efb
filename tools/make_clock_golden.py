#!/usr/bin/env python3
"""tools/make_clock_golden.py <reference checkout> — golden vectors of the overlay clock, generated HERE by the UNMODIFIED reference.

1. tests/golden/font8.bin: the reference's glyph atlas, extracted from src/font.h (_font8: 16 x 1024 bytes, then _font8_rights as
   little-endian int16). A data fixture: the numbers only.
2. tests/golden/clock_pins.json: tools/ref_clock_harness.cpp compiles espflix.cpp as it is and calls its own update_progress()
   (get_pts() stubbed to the case's value) over every case of tests/clock_cases.py, and show_time() directly over a list of
   (seconds, icon). Every result is checked against the restatement before it is written."""
import ctypes
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import clock_cases as cc  # noqa: E402

SHOW_TIME = [(0, cc.PLAY), (9, cc.PAUSE), (59, cc.FFWD), (60, cc.RWND), (3599, cc.STOP), (3600, cc.PLAY), (3723, cc.PLAY), (36000 + 671, cc.PLAY),
             (359999, cc.PLAY), (360000, cc.PLAY), (3599999, cc.RWND), (-1, cc.PLAY), (-61, cc.PAUSE), (-3725, cc.RWND), (-360000, cc.FFWD),
             (-7322, cc.PLAY), (2 ** 31 - 1 - (2 ** 31 - 1) % 3600 + 3599 - 3600, cc.PLAY)]


def extract_font(ref):
    text = open(os.path.join(ref, "src", "font.h")).read()
    rights = [int(v) for v in re.search(r"_font8_rights\[\]\s*=\s*\{([^}]*)\}", text).group(1).split(",") if v.strip()]
    atlas = [int(v, 0) for v in re.search(r"_font8\[1024\*16\]\s*=\s*\{([^}]*)\}", text).group(1).split(",") if v.strip()]
    assert len(atlas) == 16 * 1024 and len(rights) >= 35, (len(atlas), len(rights))
    with open(cc.FONT, "wb") as f:
        f.write(np.array(atlas, dtype=np.uint8).tobytes() + np.array(rights, dtype="<i2").tobytes())


def build(ref, tmp):
    lib = os.path.join(tmp, "libefref_clock.so")
    subprocess.run(["g++", "-std=c++14", "-O2", "-w", "-fpermissive", "-fPIC", "-shared", "-I" + os.path.join(ref, "src"), "-o", lib,
                    os.path.join(ROOT, "tools", "ref_clock_harness.cpp")], check=True)
    L = ctypes.CDLL(lib)
    VP, I = ctypes.c_void_p, ctypes.c_int
    L.efref_update_progress.argtypes = [VP, I, I, I, ctypes.c_int64, VP, VP, VP]
    L.efref_show_time.argtypes = [I, I, VP]
    L.efref_set_last_seconds.argtypes = [ctypes.c_int64]
    return L


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: tools/make_clock_golden.py <reference checkout>")
    ref = os.path.abspath(sys.argv[1])
    extract_font(ref)
    atlas, rights = cc.font()
    pins = {"update_progress": {}, "show_time": []}
    with tempfile.TemporaryDirectory() as tmp:
        L = build(ref, tmp)
        bm, prog, last = np.zeros(1280, np.uint8), ctypes.c_int(), ctypes.c_int64()
        for name, steps in sorted(cc.cases().items()):
            L.efref_show_time(0, 0, bm.ctypes.data)                     # a fresh player: erased bitmap, _last_seconds 0
            L.efref_set_last_seconds(0)
            got = []
            for hdr, speed, paused, zero, pts in steps:
                h = np.frombuffer(hdr, dtype=np.uint8).copy()
                L.efref_update_progress(h.ctypes.data, speed, int(paused), int(zero), pts, bm.ctypes.data, ctypes.byref(prog), ctypes.byref(last))
                got.append((hashlib.sha256(bm.tobytes()).hexdigest(), prog.value, last.value))
            want = cc.restate(steps, atlas, rights)
            assert got == want, (name, got, want)
            pins["update_progress"][name] = [{"sha256": s, "progress": p, "last_seconds": ls} for s, p, ls in got]
            print(name, [(p, ls) for _, p, ls in got])
        for s, icon in SHOW_TIME:
            L.efref_show_time(s, icon, bm.ctypes.data)
            text = cc.time_text(s, icon)
            assert np.array_equal(bm, cc.render(text, atlas, rights)), (s, icon)
            pins["show_time"].append({"seconds": s, "icon": icon, "width": cc.text_width(text, rights), "sha256": hashlib.sha256(bm.tobytes()).hexdigest()})
            print(s, repr(text), cc.text_width(text, rights))
    json.dump(pins, open(cc.PINS, "w"), indent=1)


if __name__ == "__main__":
    main()
