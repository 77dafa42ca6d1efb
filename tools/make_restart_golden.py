#!/usr/bin/env python3
"""tools/make_restart_golden.py <reference checkout> — golden vectors of the per-stream restart, generated HERE by the UNMODIFIED
reference. Builds the reference with the oracle's recipe (make -C oracle ref), then in a temporary directory:
  * tools/ref_restart_harness.cpp as a CLI over the reference's decoder thread (player.cpp with the audio harness's hooks): every
    case of tests/restart_cases.decoder_cases() played program after program with MpegDecoder::reset() + video_reset() between
    them -> the pts of every push_video, get_pts() after every program, PCM and PDM;
  * tools/ref_overlay_harness.cpp with its video_reset() routed to video_reset() or video_pause(0) -> the paced field stream of
    every case of tests/restart_cases.paced_cases(), frame stores carried over.
Every case is checked against the restatement in tests/restart_cases.py before tests/golden/restart_pins.json is written."""
import hashlib
import importlib.util
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import restart_cases as rc  # noqa: E402
from tests.oracle_lib import Oracle  # noqa: E402

FLAGS = ["-std=c++14", "-O2", "-w", "-fpermissive", "-fPIC"]


def build(ref, tmp):
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "ref", "REF=" + os.path.abspath(ref)], check=True, capture_output=True)
    obj = lambda o: os.path.join(ROOT, "oracle", "_ref", o + ".o")            # noqa: E731
    inc = ["-I" + os.path.join(ref, "src"), "-I" + os.path.join(ROOT, "oracle")]
    harness = os.path.join(ROOT, "tools", "ref_restart_harness.cpp")
    cli = os.path.join(tmp, "efref_restart")
    subprocess.run(["g++"] + FLAGS + inc + ["-DEFREF_RESTART_DECODER", "-o", cli, harness]
                   + [obj(o) for o in ("player_aud", "streamer", "sbc_decoder", "video")] + ["-lpthread", "-lm"], check=True)
    ovl, hook = os.path.join(tmp, "ovl.o"), os.path.join(tmp, "hook.o")
    subprocess.run(["g++"] + FLAGS + inc + ["-Dvideo_reset=efref_restart_hook", "-c", "-o", ovl, os.path.join(ROOT, "tools", "ref_overlay_harness.cpp")], check=True)
    subprocess.run(["g++"] + FLAGS + inc + ["-DEFREF_RESTART_PACED", "-c", "-o", hook, harness], check=True)
    lib = os.path.join(tmp, "libefref_restart.so")
    subprocess.run(["g++", "-shared", "-Wl,-Bsymbolic", "-o", lib, ovl, hook]
                   + [obj(o) for o in ("video", "player", "streamer", "sbc_decoder", "ref_video_harness")] + ["-lpthread", "-lm"], check=True)
    return cli, lib


def run_decoder(cli, programs, tmp):
    paths = []
    for i, ts in enumerate(programs):
        p = os.path.join(tmp, "prog%d.ts" % i)
        open(p, "wb").write(bytes(ts))
        paths.append(p)
    out = os.path.join(tmp, "out.bin")
    subprocess.run([cli, out] + paths, check=True, timeout=300)
    b = open(out, "rb").read()
    n_prog, n_push, n_pcm = np.frombuffer(b[:24], dtype=np.int64)
    o = 24
    ends = np.frombuffer(b[o:o + 24 * n_prog], dtype=np.int64).reshape(-1, 3)
    o += 24 * n_prog
    pushes = np.frombuffer(b[o:o + 8 * n_push], dtype=np.int64)
    o += 8 * n_push
    pcm = np.frombuffer(b[o:o + 2 * n_pcm], dtype=np.int16)
    o += 2 * n_pcm
    pdm = np.frombuffer(b[o:o + 4 * n_pcm], dtype=np.uint16)
    return ends, pushes, pcm, pdm


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: tools/make_restart_golden.py <reference checkout>")
    o = Oracle()
    spec = importlib.util.spec_from_file_location("mog", os.path.join(ROOT, "tools", "make_overlay_golden.py"))
    mog = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mog)
    pins = {"decoder": {}, "paced": {}}
    with tempfile.TemporaryDirectory() as tmp:
        cli, lib = build(sys.argv[1], tmp)
        for name, progs in sorted(rc.decoder_cases().items()):
            ends, pushes, pcm, pdm = run_decoder(cli, progs, tmp)
            want = rc.decoder_restate(progs)
            pcms, want_pdm = rc.audio_restate(o, progs)
            assert pushes.tolist() == want["pushes"], (name, pushes.tolist(), want["pushes"])
            assert ends[:, 2].tolist() == want["last"], (name, ends[:, 2].tolist(), want["last"])
            cuts = [0] + ends[:, 1].tolist()
            ref_pcms = [pcm[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
            assert [p.size for p in ref_pcms] == [p.size for p in pcms], (name, [p.size for p in ref_pcms], [p.size for p in pcms])
            assert all(np.array_equal(a, b) for a, b in zip(ref_pcms, pcms)), name
            assert np.array_equal(pdm, want_pdm), name
            pins["decoder"][name] = {"pushes": pushes.tolist(), "pictures": [len(p) for p in want["pic_pts"]], "get_pts": ends[:, 2].tolist(),
                                     "pcm_samples": [int(p.size) for p in ref_pcms], "pcm_sha256": [sha(p) for p in ref_pcms],
                                     "pdm_sha256": sha(pdm)}
            print(name, "pushes", len(pushes), "pcm", [p.size for p in ref_pcms])
        import ctypes
        L = ctypes.CDLL(lib)
        VP, I = ctypes.c_void_p, ctypes.c_int
        L.efref_paced_overlay.restype = ctypes.c_long
        L.efref_paced_overlay.argtypes = [VP, I, VP, VP, VP, I, I, I, VP, VP, VP, VP, I, VP, VP, VP, VP]
        L.efref_geometry.argtypes = [VP]
        for name, case in sorted(rc.paced_cases().items()):
            frames = [o.decode_ts(oc_ts) for oc_ts in (mog.oc.segment_ts(seed, pts) for seed, pts in case["segments"])]
            L.efref_restart_op(case["op"])
            n, ff, fl, stream, blend = mog.run(L, case, frames)
            fields, flips, whole = rc.paced_restate(case, frames, o)
            assert fields == n and flips == ff, (name, fields, n, flips, ff)
            assert sha(stream) == whole, name
            pins["paced"][name] = {"fields": n, "flip_field": ff, "flip_line": fl, "stream_sha256": whole}
            print(name, n, "fields")
    with open(os.path.join(ROOT, "tests", "golden", "restart_pins.json"), "w") as f:
        json.dump(pins, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
