#!/usr/bin/env python3
"""tools/bench_pts.py — the cost of per-picture presentation timestamps (ef_pts_enable) at batch scale.

Workload: bench.py's config 4 (4,096 streams x one GOP of 12 pictures, 64 distinct seeds replicated) as transport streams
(espflix_b200.synth.wrap_ts: one video PES with a PTS per picture). Per step, on both of two contexts over the same pinned
input: ef_submit_ts_host -> ef_index -> ef_decode_all(12) -> ef_read_latest_i420_async. One context never enables PTS; the
other calls ef_pts_enable, so every submit also runs the packet pass and every ef_index the resolve pass. The two legs are
timed alternately (--rounds each). Reported: ms per step of both legs (median and all rounds), the device time of the two
PTS kernels (torch.profiler, two untimed steps), and the card's name and power limit. After the timed steps the pts of the
first distinct streams are checked against the restatement in tests/pts_cases.py (--no-verify skips it). Writes nothing into
the tree.

  python tools/bench_pts.py [--streams 4096] [--steps 20] [--warmup 3] [--rounds 3] [--no-verify]
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--no-verify", action="store_true")
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_pts.py: no CUDA device; the product has no CPU path")
    torch.cuda.set_device(args.device)
    streams, P = args.streams, bench.PICTURES
    gen, _ = bench.make_streams(streams)
    d = len(gen)
    ts = [synth.wrap_ts(*g) for g in gen]
    off = np.zeros(streams + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(ts[i % d]) for i in range(streams)])
    pinned_ts = torch.empty(int(off[-1]), dtype=torch.uint8, pin_memory=True)
    view = pinned_ts.numpy()
    for i in range(streams):
        view[int(off[i]):int(off[i + 1])] = ts[i % d]
    pinned_out = [torch.empty((streams, bench.FRAME_BYTES), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    st = 0

    ctxs = {}
    for leg in ("e2e_ts", "e2e_ts_pts"):
        ctx = espflix_b200.Context(n_streams=streams, max_pictures=P, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096,
                                   device=args.device, fields=False)
        if leg == "e2e_ts_pts":
            ctx.enable_pts()
        ctxs[leg] = ctx

    def step(ctx, k):
        ctx.submit_ts(pinned_ts.data_ptr(), off, st, device=False)
        ctx.index(st)
        ctx.decode_all(P, st)
        ctx.read_latest_i420_async(0, streams, pinned_out[k & 1].data_ptr(), st)

    def timed(ctx):
        for k in range(args.warmup):
            step(ctx, k)
        ctx.sync(st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        w0 = time.perf_counter()
        for k in range(args.steps):
            step(ctx, k)
        e1.record()
        ctx.sync(st)
        torch.cuda.synchronize()
        return max(e0.elapsed_time(e1), 1000.0 * (time.perf_counter() - w0)) / args.steps

    ms = {leg: [] for leg in ctxs}
    for _ in range(args.rounds):
        for leg, ctx in ctxs.items():
            ms[leg].append(round(timed(ctx), 4))
    res = {leg: {"ms_per_step_median": float(np.median(v)), "ms_per_step_rounds": v,
                 "video_frames_per_s": streams * P / (float(np.median(v)) / 1000.0)} for leg, v in ms.items()}

    ctx = ctxs["e2e_ts_pts"]
    if not args.no_verify:
        from tests import pts_cases
        pic, last = ctx.picture_pts()
        for i in range(min(4, d)):
            want = pts_cases.picture_pts(ts[i])
            if [int(v) for v in pic[i]] != want or int(last[i]) != want[-1]:
                raise SystemExit("bench_pts.py: stream %d: pts differ from the restatement" % i)
        res["verify"] = "ok: the pts of %d distinct streams equal the restatement" % min(4, d)

    from torch.profiler import ProfilerActivity, profile       # device time per kernel, two untimed steps
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(2):
            step(ctx, k)
        ctx.sync(st)
    kern = {}
    for e in prof.key_averages():
        if "pts_" in e.key:
            kern[e.key.split("(")[0]] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 2, 2)
    for c in ctxs.values():
        c.close()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams x 12 pictures (one video PES with PTS per picture), %d distinct seeds replicated" % (streams, d),
        "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "card": card,
        "packets_per_step": int(off[-1]) // 188,
        "legs": res,
        "pts_kernel_us_per_step": kern,
    }), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
