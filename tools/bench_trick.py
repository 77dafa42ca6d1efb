"""tools/bench_trick.py — ef_trick_build on a catalogue of synthetic mains: video_fwd.ts and video_rwd.ts of about an hour of 24 fps
material in one call.

The catalogue: efsynth programs (GOPs of 12, the benchmark's quantiser and grain) and restart_cases programs that carry SBC audio on
PID 0x101, a few distinct seeds each, replicated to --minutes of main. Reports, with the card's name and power limit read in the
same run: the build's wall time (host clock around the call, which includes the host's segment plan and the copies) per hour of
main; the device time of the decode (upload, K0, K1a, K1b), the gather, the encode (FDCT, quantiser, VLC, assembly) and the mux from
CUDA events (ef_trick_stage_ms); encoded pictures per second of the encode phase; input and output bytes. One JSON line.

    python tools/bench_trick.py [--minutes 60] [--qscale 8] [--repeats 2]"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def catalogue(minutes, main_pictures=720):
    """[(ts, pictures)]: 4 efsynth seeds and 2 audio-carrying programs, 30 s each, replicated"""
    from espflix_b200 import synth
    from tests import restart_cases
    with ThreadPoolExecutor(4) as ex:            # efsynth runs outside the GIL
        gen = list(ex.map(lambda k: synth.generate(synth.SEED0 + 900 + k, n_pictures=main_pictures, gop=12), range(4)))
    distinct = [bytes(synth.wrap_ts(es, off)) for es, off in gen]
    for k in range(2):        # one sequence header per 24-picture program, audio interleaved
        per = 24
        distinct.append(b"".join(restart_cases.program(950 + 10 * k + j, per, 90000 + j * per * 3003, audio=dict(seed=60 + k, frames=40, cut=0))
                                 for j in range(main_pictures // per)))
    n = max(1, round(minutes * 60 * 24 / main_pictures))
    return [distinct[i % len(distinct)] for i in range(n)], n * main_pictures


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--qscale", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    from espflix_b200 import capi
    capi.load_library()
    t0 = time.time()
    mains, pictures = catalogue(a.minutes)
    gen_s = time.time() - t0
    in_bytes = sum(len(m) for m in mains)
    capi.trick_build(mains[:2], qscale=a.qscale)                  # warm-up: module load, first allocations
    runs = []
    for _ in range(a.repeats):
        t = time.perf_counter()
        out = capi.trick_build(mains, qscale=a.qscale)
        wall = time.perf_counter() - t
        runs.append((wall, capi.trick_stage_ms()))
    wall, (dec, gat, enc, mux) = min(runs, key=lambda r: r[0])
    hours = pictures / 24 / 3600
    fwd_pics = len(range(0, 720, 15)) * len(mains)
    res = {
        "metric": "trick streams built per hour of 24 fps main", "card": card(), "qscale": a.qscale,
        "mains": len(mains), "main_pictures": pictures, "main_hours": round(hours, 3), "main_bytes": in_bytes,
        "wall_s": round(wall, 3), "wall_s_per_hour_of_main": round(wall / hours, 3),
        "device_ms": {"decode": round(dec, 2), "gather": round(gat, 2), "encode": round(enc, 2), "mux": round(mux, 2)},
        "fwd_pictures": fwd_pics, "encode_pictures_per_s": round(fwd_pics / (enc / 1e3), 1) if enc else None,
        "fwd_bytes": sum(len(f) for f, _ in out), "rwd_bytes": sum(len(r) for _, r in out),
        "repeats_wall_s": [round(r[0], 3) for r in runs], "catalogue_generation_s": round(gen_s, 1),
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
