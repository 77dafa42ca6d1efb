#!/usr/bin/env python3
"""tools/bench_library.py — TS submits from host memory against submits gathered on the device from titles held in HBM (ef_library_*).

Workload: tools/bench_carry.py's packet_cuts arm (4,096 streams x one GOP of 12 pictures per submit, every submit cut half way into
a picture, distinct seeds replicated). Two carrying, PTS-enabled contexts, timed alternately (--rounds each), every step ending in a
device synchronise:
  (a) "host": ef_submit_ts_host of the step's window from pinned memory (the bytes cross the host link every step);
  (b) "library": every distinct GOP repeated into one title (main file only, a one-sample video.idx), added once with
      ef_library_add; every stream PLAY_AT 0 of its title, then ef_library_submit with each stream's GOP packet count as its budget
      (the same bytes per stream and step as (a)).
Per step: submit -> ef_index -> ef_decode_all(12) -> ef_read_latest_i420_async -> synchronise. Reported: ms per step of both arms
(median and all rounds), the host time of the submit call alone, the device time per step of the library kernels and the staging
copy (torch.profiler, two untimed steps) and the card's name and power limit. Writes nothing into the tree.

  python tools/bench_library.py [--streams 4096] [--steps 12] [--warmup 3] [--rounds 3] [--max-carry 32768]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.dont_write_bytecode = True                            # the tree may be read-only
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-carry", type=int, default=32768)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import capi, synth
    from tests import library_cases as lc

    if not torch.cuda.is_available():
        raise SystemExit("bench_library.py: no CUDA device; the product has no CPU path")
    torch.cuda.set_device(args.device)
    streams, P = args.streams, bench.PICTURES
    gen, _ = bench.make_streams(streams)
    d = len(gen)
    gop = [np.frombuffer(bytes(synth.wrap_ts(*g)), dtype=np.uint8) for g in gen]
    npk = [g.size // 188 for g in gop]
    half = [n // 2 for n in npk]
    first = [g[:188 * h] for g, h in zip(gop, half)]
    window = [np.concatenate([g[188 * h:], g[:188 * h]]) for g, h in zip(gop, half)]
    total_steps = 2 + args.rounds * (args.warmup + args.steps) + 2 + 1

    def pin(parts):
        off = np.zeros(streams + 1, dtype=np.uint64)
        off[1:] = np.cumsum([parts[i % d].size for i in range(streams)])
        t = torch.empty(max(int(off[-1]), 1), dtype=torch.uint8, pin_memory=True)
        v = t.numpy()
        for i in range(streams):
            v[int(off[i]):int(off[i + 1])] = parts[i % d]
        return t, off

    first_in, window_in = pin(first), pin(window)
    pinned_out = [torch.empty((streams, bench.FRAME_BYTES), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    st = 0
    cap = int(window_in[1][-1]) + 4096
    ctxs = {}
    for leg in ("host", "library"):
        c = espflix_b200.Context(n_streams=streams, max_pictures=P + 1, max_slices_per_picture=12, es_capacity=cap, device=args.device, fields=False)
        c.enable_pts()
        c.enable_carry(args.max_carry)
        ctxs[leg] = c
    lib = ctxs["library"]
    idx = lc.image((0, 1, 1, 1, 1), (0, 1, 1, 1, 0), (0, 1, 1, 1, 0), [0])   # one sample: packet 0
    for g in gop:
        lib.library_add(idx, np.tile(g, total_steps).tobytes())
    for s in range(streams):
        lib.library_command(capi.LIB_PLAY_AT, s, 1, s % d, 0)
    budget_first = np.array([half[s % d] for s in range(streams)], dtype=np.uint32)
    budget = np.array([npk[s % d] for s in range(streams)], dtype=np.uint32)
    submit_ms = {"host": [], "library": []}

    def submit(leg, first_step=False):
        c = ctxs[leg]
        t0 = time.perf_counter()
        if leg == "host":
            t, off = first_in if first_step else window_in
            c.submit_ts(t.data_ptr(), off, st, device=False)
        else:
            c.library_submit(per_stream=budget_first if first_step else budget, stream=st)
        submit_ms[leg].append(1000.0 * (time.perf_counter() - t0))

    def step(leg, k, first_step=False):
        c = ctxs[leg]
        submit(leg, first_step)
        c.index(st)
        c.decode_all(P, st)
        c.read_latest_i420_async(0, streams, pinned_out[k & 1].data_ptr(), st)
        c.sync(st)
        torch.cuda.synchronize()

    for leg in ctxs:
        step(leg, 0, first_step=True)
        step(leg, 1)
        info = ctxs[leg].index_info()
        if info["total_pictures"] != streams * P or info["max_pictures"] != P:
            raise SystemExit("bench_library.py: arm %s does not complete 12 pictures per stream and submit: %s" % (leg, info))
    a = ctxs["host"].read_latest_i420()
    b = ctxs["library"].read_latest_i420()
    if not np.array_equal(a, b):
        raise SystemExit("bench_library.py: the two arms decoded different pictures")
    for leg in submit_ms:
        submit_ms[leg].clear()

    def timed(leg):
        for k in range(args.warmup):
            step(leg, k)
        w0 = time.perf_counter()
        for k in range(args.steps):
            step(leg, k)
        return 1000.0 * (time.perf_counter() - w0) / args.steps

    ms = {leg: [] for leg in ctxs}
    for _ in range(args.rounds):
        for leg in ctxs:
            ms[leg].append(round(timed(leg), 4))
    res = {leg: {"ms_per_step_median": float(np.median(v)), "ms_per_step_rounds": v,
                 "submit_call_host_ms_median": round(float(np.median(submit_ms[leg])), 4)} for leg, v in ms.items()}

    from torch.profiler import ProfilerActivity, profile       # device time per kernel / copy, two untimed steps per arm
    kern = {}
    for leg in ctxs:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(2):
                step(leg, k)
        kern[leg] = {}
        for e in prof.key_averages():
            if any(x in e.key for x in ("library", "Memcpy")):
                kern[leg][e.key.split("(")[0]] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 2, 2)
    for ctx in ctxs.values():
        ctx.close()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams, one GOP of 12 pictures per submit cut half way into a picture, %d distinct seeds replicated" % (streams, d),
        "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "card": card, "max_carry": args.max_carry,
        "ts_bytes_per_step": int(window_in[1][-1]), "arms": res, "device_us_per_step": kern,
    }), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
