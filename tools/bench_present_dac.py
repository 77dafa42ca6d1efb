#!/usr/bin/env python3
"""tools/bench_present_dac.py — paced presentation in the two field formats (ef_present_format): EF_FIELD_U16, the reference's
uint16 DMA line buffer, against EF_FIELD_DAC8, the bytes the video DAC plays (half the bytes per field).

Workload: tools/bench_present.py's (4,096 TS streams x 12 pictures per step, pts step 3003, ef_reset between steps), on one U16
and one DAC8 context per standard, alternated step by step. Reported per standard and format:
  * ms per step: host clock around the synchronous present calls of a step (each ends in a stream synchronise), mean and range;
  * the paced K2's device time per step and its output bytes/s, from a separate torch.profiler run of two steps;
  * ms per step when every call's fields are also copied to pinned host memory (through one reused 1 GiB pinned buffer,
    stream-ordered behind the call): what a consumer that takes the fields off the card pays end to end;
and a check that one step of the DAC8 context is, call by call, the conversion of the U16 context's fields
(tests/dac_cases.py). The card's name and power limit go with the numbers. Writes nothing into the tree.

  python tools/bench_present_dac.py [--streams 4096] [--steps 10] [--warmup 2] [--copy-steps 4]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

sys.dont_write_bytecode = True                            # the tree may be read-only
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

STAGE = 1 << 30                                           # bytes of the pinned staging buffer of the copy arm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--copy-steps", type=int, default=4)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import capi, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_present_dac.py: no CUDA device; the product has no CPU path")
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
    stage = torch.empty(STAGE, dtype=torch.uint8, pin_memory=True)
    formats = {"u16": capi.EF_FIELD_U16, "dac8": capi.EF_FIELD_DAC8}
    results = {}
    for ntsc in (1, 0):
        arms = {}
        for name, fmt in formats.items():
            ctx = espflix_b200.Context(n_streams=streams, max_pictures=P, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096,
                                       device=args.device, fields=False)
            ctx.enable_pts()
            ctx.video_init(ntsc)
            if fmt != capi.EF_FIELD_U16:
                ctx.present_format(fmt)
            ctx.enable_present(1)                          # frame counter 1, as bench_present.py
            w, nl = ctx.geometry()
            cap = 3 * streams
            out = torch.empty(cap * w * nl, dtype=torch.uint16 if fmt == capi.EF_FIELD_U16 else torch.uint8, device="cuda")
            nbytes = 2 if fmt == capi.EF_FIELD_U16 else 1
            arms[name] = {"ctx": ctx, "out": out, "bytes": out.view(torch.int16).view(torch.uint8) if nbytes == 2 else out,
                          "field_bytes": w * nl * nbytes, "ms": [], "copy_ms": []}

        def start(a):
            ctx = a["ctx"]
            ctx.reset()
            ctx.submit_ts(pinned_ts.data_ptr(), off, 0, device=False)
            ctx.index(0)

        def step(a, copy=False):
            start(a)
            n = 0
            for p in range(P):
                info = a["ctx"].present_picture(p, None, a["out"], 0)
                k = int(info["n_fields"].sum())
                n += k
                if copy:
                    src = a["bytes"][:k * a["field_bytes"]]
                    for b in range(0, src.numel(), STAGE):
                        c = src[b:b + STAGE]
                        stage[:c.numel()].copy_(c, non_blocking=True)
            return n

        for _ in range(args.warmup):
            for a in arms.values():
                step(a)
        torch.cuda.synchronize()
        fields = {}
        for _ in range(args.steps):                        # U16 and DAC8 steps alternate
            for name, a in arms.items():
                t0 = time.perf_counter()
                fields[name] = step(a)
                torch.cuda.synchronize()
                a["ms"].append(1000.0 * (time.perf_counter() - t0))
        for _ in range(args.copy_steps):
            for name, a in arms.items():
                t0 = time.perf_counter()
                step(a, copy=True)
                torch.cuda.synchronize()
                a["copy_ms"].append(1000.0 * (time.perf_counter() - t0))
        assert fields["u16"] == fields["dac8"]

        from torch.profiler import ProfilerActivity, profile   # the paced K2's device time, two untimed steps per format
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            pf = {name: step(a) + step(a) for name, a in arms.items()}
            torch.cuda.synchronize()
        k2 = {"u16": 0.0, "dac8": 0.0}
        for e in prof.key_averages():
            m = re.search(r"ef_composite_kernel<([^>]*)>", e.key)
            if not m:
                continue
            targs = [x.strip() for x in m.group(1).split(",")]
            if len(targs) >= 2 and targs[1] == "true":   # paced
                k2["dac8" if len(targs) == 5 and targs[4] == "true" else "u16"] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))

        u, dc = arms["u16"], arms["dac8"]                  # one more step of both in lockstep: DAC8 = the conversion of U16, call by call
        start(u)
        start(dc)
        for p in range(P):
            iu = u["ctx"].present_picture(p, None, u["out"], 0)
            idd = dc["ctx"].present_picture(p, None, dc["out"], 0)
            if not (iu == idd).all():
                raise SystemExit("bench_present_dac.py: picture %d: the info rows of the two formats differ" % p)
            k = int(iu["n_fields"].sum()) * dc["field_bytes"]
            conv = u["bytes"][:2 * k].view(-1, 4)[:, [3, 1]].reshape(-1)
            if not torch.equal(conv, dc["out"][:k]):
                raise SystemExit("bench_present_dac.py: picture %d: the DAC8 fields are not the conversion of the U16 fields" % p)
            del conv

        res = {"fields_per_step": fields["u16"]}
        for name, a in arms.items():
            ms = np.array(a["ms"])
            res[name] = {"ms_per_step": round(float(ms.mean()), 3), "ms_range": [round(float(ms.min()), 3), round(float(ms.max()), 3)],
                         "field_bytes": a["field_bytes"], "GB_per_step": round(fields[name] * a["field_bytes"] / 1e9, 2),
                         "paced_k2_ms_per_step": round(k2[name] / 2e3, 3),
                         "paced_k2_GBps": round(pf[name] * a["field_bytes"] / (k2[name] * 1e3), 1) if k2[name] else None,
                         "ms_per_step_with_host_copy": round(float(np.mean(a["copy_ms"])), 3) if a["copy_ms"] else None}
        res["dac8_over_u16"] = {"step": round(res["dac8"]["ms_per_step"] / res["u16"]["ms_per_step"], 3),
                                "paced_k2": round(res["dac8"]["paced_k2_ms_per_step"] / res["u16"]["paced_k2_ms_per_step"], 3),
                                "with_host_copy": round(res["dac8"]["ms_per_step_with_host_copy"] / res["u16"]["ms_per_step_with_host_copy"], 3)
                                if args.copy_steps else None}
        res["verify"] = "ok: one step of DAC8 fields equals the conversion of the U16 fields, call by call"
        results["ntsc" if ntsc else "pal"] = res
        for a in arms.values():
            a["ctx"].close()
        del arms
        torch.cuda.empty_cache()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams x 12 pictures per step (pts step 3003), %d distinct seeds replicated, U16 and DAC8 steps alternated" % (streams, d),
        "steps": args.steps, "warmup": args.warmup, "copy_steps": args.copy_steps, "card": card, "standards": results}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
