#!/usr/bin/env python3
"""tools/bench_present_clock.py — the overlay clock on the device (ef_present_clock) against the host-driven equivalent.

Workload: tools/bench_present_async.py's (4,096 TS streams x 12 pictures per step, pts step 3003, ef_reset between steps), NTSC and
PAL, with the overlay shown and a clock on every stream (a one-hour title, speed 0). Two arms, one context each, run alternately
step by step:
  device  ef_present_picture_async(0..11) with the clock on: update_progress() runs on the device, then one ef_present_wait
  host    before every push: ef_picture_pts, update_progress() on the host (tests/clock_cases.py, each text rendered once) and
          ef_present_overlay of the bitmaps and progress; then the same ef_present_picture_async call and its ef_present_wait
          (the next ef_present_overlay would wait for it anyway)
Reported per standard and arm: ms per step (host clock, with a device synchronise inside it) and the host time of the present
calls (the host arm's includes its read-back, render and staging); for the device arm the device time per step of the clock
kernel and its commit (torch.profiler over two more steps). The card's name and power limit. Writes nothing into the tree.

  python tools/bench_present_clock.py [--streams 4096] [--steps 5] [--warmup 1]
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
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import capi, synth
    from tests import clock_cases as cc

    if not torch.cuda.is_available():
        raise SystemExit("bench_present_clock.py: no CUDA device; the product has no CPU path")
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
    atlas, rights = cc.font()
    hdr = cc.header((0, 90000 * 3600), (0, 90000 * 360), (0, 90000 * 360))
    st = 0
    results = {}
    for ntsc in (1, 0):
        ctxs = {}
        for arm in ("device", "host"):
            c = espflix_b200.Context(n_streams=streams, max_pictures=P, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096,
                                     device=args.device, fields=False)
            c.enable_pts()
            c.video_init(ntsc)
            c.enable_present(1)
            c.present_overlay(None, -1, None, set=np.full(streams, 2, np.uint8))
            if arm == "device":
                c.present_font(atlas, rights)
                c.present_clock(np.frombuffer(hdr, dtype=np.uint8), 0, 1)
            ctxs[arm] = c
        clocks = [cc.Clock() for _ in range(streams)]
        for k in clocks:
            k.set(hdr, 0, 1)
        w, nl = ctxs["device"].geometry()
        need = [0] * P
        infos = [torch.zeros((streams, 8), dtype=torch.int32, device="cuda") for _ in range(P)]
        bm, pr, setb = np.zeros((streams, 1280), np.uint8), np.zeros(streams, np.int32), np.zeros(streams, np.uint8)

        def begin(c):
            c.reset()
            c.submit_ts(pinned_ts.data_ptr(), off, st, device=False)
            c.index(st)

        def host_clock(c, p):
            pic, last = c.picture_pts(n_pictures=p + 1)
            for s, k in enumerate(clocks):
                r = k.step(int(pic[s, p]) if p < counts[s] else int(last[s]))
                k.commit(r)
                setb[s] = 5 if r[0] is not None else 4
                pr[s] = r[1]
                if r[0] is not None:
                    bm[s] = r[0]
            c.present_overlay(bm, None, pr, setb)

        def check(rc, k, want):
            if rc != capi.EF_OK or k != want:
                raise SystemExit("bench_present_clock.py: a call did not fit (rc %d, %d presented)" % (rc, k))

        def step(arm):
            c = ctxs[arm]
            begin(c)
            h0 = time.perf_counter()
            a = 0
            for p in range(P):
                if arm == "host":
                    host_clock(c, p)
                cap = need[p] + MARGIN
                c.present_picture_async(p, big[a * w * nl:(a + cap) * w * nl], infos[p], stream=st)
                a += cap
                if arm == "host":                           # what the next ef_present_overlay does first anyway
                    check(*c.present_wait(), 1)
            h = time.perf_counter() - h0
            if arm == "device":
                check(*c.present_wait(), P)
            for p in range(P):
                need[p] = int(c.present_info(infos[p])["n_fields"].sum())
            return h

        c = ctxs["device"]                                  # size the buffer from one step's calls
        begin(c)
        counts = [c.stream_info(s)[0] for s in range(streams)]
        tmp = torch.empty(3 * streams * w * nl, dtype=torch.uint16, device="cuda")
        for p in range(P):
            need[p] = int(c.present_picture(p, None, tmp, st)["n_fields"].sum())
        del tmp
        big = torch.empty((sum(need) + P * MARGIN) * w * nl, dtype=torch.uint16, device="cuda")
        for _ in range(args.warmup):
            for arm in ctxs:
                step(arm)
        torch.cuda.synchronize()
        wall = {k: 0.0 for k in ctxs}
        host = {k: 0.0 for k in ctxs}
        for _ in range(args.steps):
            for arm in ctxs:
                w0 = time.perf_counter()
                host[arm] += step(arm)
                torch.cuda.synchronize()
                wall[arm] += time.perf_counter() - w0
        res = {k: {"ms_per_step_with_reset": round(1000.0 * wall[k] / args.steps, 3), "host_ms_present_calls": round(1000.0 * host[k] / args.steps, 3)}
               for k in ctxs}
        res["fields_per_step"] = sum(need)

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step("device")
            step("device")
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            for pat, short in (("ef_clock_commit_kernel", "clock_commit"), ("ef_clock_kernel", "clock")):
                if pat in e.key:
                    kern[short] = kern.get(short, 0.0) + t
                    break
        res["device_clock_kernel_us_per_step"] = {k: round(v / 2, 1) for k, v in kern.items()}
        results["ntsc" if ntsc else "pal"] = res
        del big
        for c in ctxs.values():
            c.close()
        torch.cuda.empty_cache()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams x 12 pictures per step (pts step 3003), %d distinct seeds replicated, ef_reset between steps, "
                    "a clock on every stream" % (streams, d),
        "steps": args.steps, "warmup": args.warmup, "margin_fields": MARGIN, "card": card, "standards": results}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
