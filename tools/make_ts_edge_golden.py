#!/usr/bin/env python3
"""tools/make_ts_edge_golden.py — writes tests/golden/ts_edge_pins.json: for every in-domain program of tests/ts_edge_cases.py, what
the UNMODIFIED reference makes of it:

  - the decoder (src/player.cpp + streamer.cpp with oracle/ref_decode_harness.cpp, built into a temporary directory as
    tools/make_pts_golden.py does): the number of pictures pushed, the pts of every push, and the SHA-256 of the pushed frames;
  - the audio chain (oracle/_ref/efref_audio): the SHA-256 of the bytes handed to push_audio(), of the PCM and of the PDM words;
  - for the main titles, the indexer (oracle/_ref/libefref_idx.so): make_index()'s table and first / last pts, and the SHA-256 of
    the video.idx merge_index() writes for the title as its own main, fast-forward and rewind file.

Every pin is first checked against the restatements (tests/pts_cases.py, the C oracle's decode, audio demux and index).

  EF_REFERENCE=<checkout of the reference> python tools/make_ts_edge_golden.py     (after `make -C oracle ref REF=...`)
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from tests import pts_cases, ts_edge_cases as te  # noqa: E402
from tests.oracle_lib import ROOT as _R, Oracle, RefIndexer, have_ref_index  # noqa: E402
from tools.make_pts_golden import build_ref  # noqa: E402

REF_AUDIO = os.path.join(_R, "oracle", "_ref", "efref_audio")

_RUN_ONE = r"""
import ctypes, os, sys
import numpy as np
lib = ctypes.CDLL(sys.argv[1])
ts = np.fromfile(sys.argv[2], dtype=np.uint8)
pts = np.zeros(4096, dtype=np.int64)
lib.efref_decode_ts.restype = ctypes.c_long
lib.efref_decode_ts.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
frames = np.zeros((512, 352 * 192 * 3 // 2), dtype=np.uint8)
n = lib.efref_decode_ts(ts.ctypes.data, ts.size, 1, frames.ctypes.data, 512, pts.ctypes.data)
pts[:min(n, 512)].tofile(sys.argv[3])
frames[:min(n, 512)].tofile(sys.argv[4])
sys.stdout.flush()
os._exit(0)                 # the parked decoder thread would block a normal exit
"""


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def ref_decode(lib, ts, d):
    tin, tp, tf = (os.path.join(d, x) for x in ("in.ts", "pts.bin", "frames.bin"))
    open(tin, "wb").write(bytes(ts))
    subprocess.run([sys.executable, "-c", _RUN_ONE, lib, tin, tp, tf], check=True, timeout=600)
    return [int(v) for v in np.fromfile(tp, dtype=np.int64)], np.fromfile(tf, dtype=np.uint8)


def ref_audio(ts, d):
    tin, tout = os.path.join(d, "a.ts"), os.path.join(d, "a.bin")
    open(tin, "wb").write(bytes(ts))
    subprocess.run([REF_AUDIO, tin, tout], check=True, timeout=600, capture_output=True)
    raw = open(tout, "rb").read()
    n_es, n_pcm = np.frombuffer(raw[:16], dtype=np.uint64)
    es = raw[16:16 + int(n_es)]
    pcm = raw[16 + int(n_es):16 + int(n_es) + 2 * int(n_pcm)]
    pdm = raw[16 + int(n_es) + 2 * int(n_pcm):]
    return es, pcm, pdm


def restated_audio(oracle, ts):
    es = oracle.demux_audio_ts(ts)
    pcm = oracle.sbc_decode(es)
    assert not isinstance(pcm, int), pcm
    return bytes(es), pcm.tobytes(), oracle.pdm(pcm).tobytes()


def main():
    ref = os.environ.get("EF_REFERENCE")
    if not ref or not os.path.isdir(os.path.join(ref, "src")):
        raise SystemExit("make_ts_edge_golden.py needs EF_REFERENCE=<checkout of the reference>")
    if not (have_ref_index() and os.path.exists(REF_AUDIO)):
        raise SystemExit("oracle/_ref is not built: make -C oracle ref REF=<checkout of the reference>")
    oracle, rix = Oracle(), RefIndexer()
    pins = {}
    with tempfile.TemporaryDirectory() as d:
        lib = build_ref(ref, d)
        for name, (ts, roles) in te.programs().items():
            if not te.in_domain(name):
                continue
            pts, frames = ref_decode(lib, ts, d)
            want = pts_cases.picture_pts(ts)
            if pts != want:
                raise SystemExit("%s: the reference pushed %d pts, the restatement has %d" % (name, len(pts), len(want)))
            mine = oracle.decode_ts(ts, max_frames=512)
            if mine.tobytes() != frames.tobytes():
                raise SystemExit("%s: the oracle's frames differ from the reference's" % name)
            a = ref_audio(ts, d)
            if restated_audio(oracle, ts) != a:
                raise SystemExit("%s: the oracle's audio differs from the reference's" % name)
            p = {"pictures": len(pts), "pts": pts, "frames_sha256": sha(frames), "audio_es_bytes": len(a[0]), "audio_es_sha256": sha(a[0]),
                 "pcm_samples": len(a[1]) // 2, "pcm_sha256": sha(a[1]), "pdm_sha256": sha(a[2])}
            if "main" in roles:
                assert te.index_in_domain(ts), name
                ix = rix.make_index(ts)
                mo = oracle.make_index(ts)
                if any(not np.array_equal(ix[k], mo[k]) for k in ("seq_pts", "seq_pos")) or (ix["first_pts"], ix["last_pts"]) != (mo["first_pts"], mo["last_pts"]):
                    raise SystemExit("%s: the oracle's index differs from the reference's" % name)
                idx = rix.build_idx([ts, ts, ts])
                if oracle.build_idx([ts, ts, ts]) != idx:
                    raise SystemExit("%s: the oracle's video.idx differs from the reference's" % name)
                p.update({"first_pts": ix["first_pts"], "last_pts": ix["last_pts"], "seq_pts": [int(v) for v in ix["seq_pts"]],
                          "seq_pos": [int(v) for v in ix["seq_pos"]], "video_idx_bytes": len(idx), "video_idx_sha256": sha(idx)})
            pins[name] = p
            print("%-20s %4d pictures, %7d audio bytes, %7d PCM samples%s" % (name, len(pts), len(a[0]), len(a[1]) // 2,
                                                                             ", %d sequence entries" % len(p["seq_pts"]) if "main" in roles else ""))
    path = os.path.join(ROOT, "tests", "golden", "ts_edge_pins.json")
    with open(path, "w") as f:
        json.dump(pins, f, indent=None, separators=(",", ":"), sort_keys=True)
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
