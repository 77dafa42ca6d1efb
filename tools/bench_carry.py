#!/usr/bin/env python3
"""tools/bench_carry.py — the cost of TS submits cut at any packet boundary (ef_carry_enable) at batch scale.

Workload: bench.py's content (4,096 streams x one GOP of 12 pictures, distinct seeds replicated) as transport streams
(espflix_b200.synth.wrap_ts: one video PES with a PTS per picture), each stream's GOP repeated for as many GOPs as there are
steps. Two arms over the same streams, timed alternately (--rounds each), every step ending in a device synchronise:
  (a) "picture_cuts": a non-carrying context, one whole GOP per submit (cut at picture boundaries, as today);
  (b) "packet_cuts": a carrying context, every stream cut at a fixed packet count = the packets of its GOP, the first cut half
      way into it, so every submit ends inside a picture and each stream holds part of one between submits (the same bytes,
      and in the steady state the same 12 complete pictures, per submit).
Per step: ef_submit_ts_host -> ef_index -> ef_decode_all(12) -> ef_read_latest_i420_async -> synchronise. Reported: ms per step
of both arms (median and all rounds), the device time per step of the kernels the carrying arm adds or changes (torch.profiler,
two untimed steps), the bytes held per submit, and the card's name and power limit. Writes nothing into the tree.

  python tools/bench_carry.py [--streams 4096] [--steps 12] [--warmup 3] [--rounds 3] [--max-carry 32768]
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
    from espflix_b200 import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_carry.py: no CUDA device; the product has no CPU path")
    torch.cuda.set_device(args.device)
    streams, P = args.streams, bench.PICTURES
    gen, _ = bench.make_streams(streams)
    d = len(gen)
    gop = [np.frombuffer(bytes(synth.wrap_ts(*g)), dtype=np.uint8) for g in gen]
    for g in gop:
        assert g.size % 188 == 0
    npk = [g.size // 188 for g in gop]
    # (b): a stream's steady-state submit is the second half of its GOP followed by the first half of the next copy; the GOP
    # repeats, so every step's window holds the same payload bytes (only the PTS fields differ, which this workload does not read)
    half = [n // 2 for n in npk]
    first = [g[:188 * h] for g, h in zip(gop, half)]
    window = [np.concatenate([g[188 * h:], g[:188 * h]]) for g, h in zip(gop, half)]

    def pin(parts):
        off = np.zeros(streams + 1, dtype=np.uint64)
        off[1:] = np.cumsum([parts[i % d].size for i in range(streams)])
        t = torch.empty(max(int(off[-1]), 1), dtype=torch.uint8, pin_memory=True)
        v = t.numpy()
        for i in range(streams):
            v[int(off[i]):int(off[i + 1])] = parts[i % d]
        return t, off

    whole_in, first_in, window_in = pin(gop), pin(first), pin(window)
    pinned_out = [torch.empty((streams, bench.FRAME_BYTES), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    st = 0
    cap = int(whole_in[1][-1]) + 4096
    ctxs = {
        "picture_cuts": espflix_b200.Context(n_streams=streams, max_pictures=P + 1, max_slices_per_picture=12, es_capacity=cap,
                                             device=args.device, fields=False),
        "packet_cuts": espflix_b200.Context(n_streams=streams, max_pictures=P + 1, max_slices_per_picture=12, es_capacity=cap,
                                            device=args.device, fields=False),
    }
    ctxs["packet_cuts"].enable_carry(args.max_carry)
    inputs = {"picture_cuts": whole_in, "packet_cuts": window_in}

    def step(leg, k):
        ctx = ctxs[leg]
        t, off = inputs[leg]
        ctx.submit_ts(t.data_ptr(), off, st, device=False)
        ctx.index(st)
        ctx.decode_all(P, st)
        ctx.read_latest_i420_async(0, streams, pinned_out[k & 1].data_ptr(), st)
        ctx.sync(st)
        torch.cuda.synchronize()

    # the carrying context starts with the first half GOP; afterwards every submit completes 12 pictures per stream
    c = ctxs["packet_cuts"]
    c.submit_ts(first_in[0].data_ptr(), first_in[1], st, device=False)
    c.index(st)
    c.decode_all(P, st)
    step("packet_cuts", 0)
    info = c.index_info()
    held, flags = c.carry_info()
    if info["total_pictures"] != streams * P or info["max_pictures"] != P or flags.any():
        raise SystemExit("bench_carry.py: the carrying arm does not complete 12 pictures per stream and submit: %s" % info)

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
    res = {leg: {"ms_per_step_median": float(np.median(v)), "ms_per_step_rounds": v} for leg, v in ms.items()}
    held, _ = c.carry_info()

    from torch.profiler import ProfilerActivity, profile       # device time per kernel, two untimed steps per arm
    kern = {}
    for leg in ctxs:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(2):
                step(leg, k)
        kern[leg] = {}
        for e in prof.key_averages():
            if any(x in e.key for x in ("carry", "scan_kernel", "ts_")):
                kern[leg][e.key.split("(")[0]] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 2, 2)
    for ctx in ctxs.values():
        ctx.close()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams, one GOP of 12 pictures per submit, %d distinct seeds replicated" % (streams, d),
        "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "card": card, "max_carry": args.max_carry,
        "ts_bytes_per_step": {"picture_cuts": int(whole_in[1][-1]), "packet_cuts": int(window_in[1][-1])},
        "held_bytes_per_submit": {"total": int(held.sum()), "mean": float(held.mean()), "max": int(held.max())},
        "arms": res,
        "kernel_us_per_step": kern,
    }), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
