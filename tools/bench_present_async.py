#!/usr/bin/env python3
"""tools/bench_present_async.py — paced presentation enqueued without waiting (ef_present_*_async) against the synchronous calls.

Workload: tools/bench_present.py's (4,096 TS streams x 12 pictures per step, pts step 3003, ef_reset between steps), NTSC and
PAL, one context each. Two arms run alternately, step by step, on the same context:
  sync   ef_present_picture(0..11), each into one buffer that holds the largest call (today's loop)
  async  ef_present_picture_async(0..11) into consecutive slices of one buffer, each slice sized from the same call of the
         previous step plus a margin of 64 fields, then one ef_present_wait
Reported per standard and arm: ms per step (host clock, with a device synchronise inside it), the host time spent enqueueing
the present calls, and the device time per step of every kernel of the async arm (torch.profiler over two more steps: schedule,
size kernel, K1a, K1b, descriptors, paced K2 including its idle CTAs). The card's name and power limit. Every async step is
checked to fit (ef_present_wait == EF_OK with all 12 calls presented). Writes nothing into the tree.

  python tools/bench_present_async.py [--streams 4096] [--steps 10] [--warmup 2]
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

MARGIN = 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import capi, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_present_async.py: no CUDA device; the product has no CPU path")
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
    st = 0
    results = {}
    for ntsc in (1, 0):
        ctx = espflix_b200.Context(n_streams=streams, max_pictures=P, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096,
                                   device=args.device, fields=False)
        ctx.enable_pts()
        ctx.video_init(ntsc)
        ctx.enable_present(1)
        w, nl = ctx.geometry()
        need = [0] * P                                 # fields of every call, from the previous step
        out = [torch.empty(3 * streams * w * nl, dtype=torch.uint16, device="cuda")]
        infos = [torch.zeros((streams, 8), dtype=torch.int32, device="cuda") for _ in range(P)]

        def begin():
            ctx.reset()
            ctx.submit_ts(pinned_ts.data_ptr(), off, st, device=False)
            ctx.index(st)

        def sync_step():
            begin()
            h0 = time.perf_counter()
            for p in range(P):
                need[p] = int(ctx.present_picture(p, None, out[0], st)["n_fields"].sum())
            return time.perf_counter() - h0

        def async_step():
            begin()
            h0 = time.perf_counter()
            a = 0
            for p in range(P):
                cap = need[p] + MARGIN
                ctx.present_picture_async(p, big[a * w * nl:(a + cap) * w * nl], infos[p], stream=st)
                a += cap
            h = time.perf_counter() - h0
            rc, k = ctx.present_wait()
            if rc != capi.EF_OK or k != P:
                raise SystemExit("bench_present_async.py: a call did not fit (rc %d, %d presented)" % (rc, k))
            for p in range(P):
                need[p] = int(ctx.present_info(infos[p])["n_fields"].sum())
            return h

        sync_step()                                    # the first step sizes the buffers of both arms
        out[0] = torch.empty((max(need) + MARGIN) * w * nl, dtype=torch.uint16, device="cuda")
        torch.cuda.empty_cache()
        big = torch.empty((sum(need) + P * MARGIN) * w * nl, dtype=torch.uint16, device="cuda")
        arms = {"sync": sync_step, "async": async_step}
        for _ in range(args.warmup):
            for f in arms.values():
                f()
        torch.cuda.synchronize()
        wall = {k: 0.0 for k in arms}
        host = {k: 0.0 for k in arms}
        for _ in range(args.steps):
            for k, f in arms.items():
                w0 = time.perf_counter()
                host[k] += f()
                torch.cuda.synchronize()
                wall[k] += time.perf_counter() - w0
        res = {k: {"ms_per_step_with_reset": round(1000.0 * wall[k] / args.steps, 3), "host_ms_enqueue_present": round(1000.0 * host[k] / args.steps, 3)}
               for k in arms}
        res["fields_per_step"] = sum(need)

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            async_step()
            async_step()
            torch.cuda.synchronize()
        names = (("ef_pace_size_kernel", "size"), ("ef_pace_kernel", "schedule"), ("ef_pace_fill_kernel", "descriptors"), ("ef_parse_kernel", "k1a"),
                 ("ef_recon_kernel", "k1b"), ("ef_composite_kernel", "paced_k2"))
        kern = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            for pat, short in names:
                if pat in e.key:
                    kern[short] = kern.get(short, 0.0) + t
                    break
        res["async_kernel_us_per_step"] = {k: round(v / 2, 1) for k, v in kern.items()}
        res["async_idle_k2_ctas_per_step"] = P * MARGIN * ((nl + 15) // 16)
        results["ntsc" if ntsc else "pal"] = res
        del out, big
        ctx.close()
        torch.cuda.empty_cache()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams x 12 pictures per step (pts step 3003), %d distinct seeds replicated, ef_reset between steps" % (streams, d),
        "steps": args.steps, "warmup": args.warmup, "margin_fields": MARGIN, "card": card, "standards": results}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
