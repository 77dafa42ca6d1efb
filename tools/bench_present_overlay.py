#!/usr/bin/env python3
"""tools/bench_present_overlay.py — the cost of the paced overlay (ef_present_overlay) at batch scale.

Workload: tools/bench_present.py's (4,096 TS streams x one GOP of 12 pictures per step, ef_reset at the start of every step,
ef_present_picture(0..11) into one device buffer), on two contexts per standard: one that never stages an overlay and one
that stages, at the start of every step, a distinct bitmap, a fading blend (60, so every field of the step draws the
overlay) and a progress value on every stream, as a player does when a title starts (show_progress()). Steps alternate
between the two contexts in the same run. Reported per standard and context: ms per step (host clock around synchronous
calls, the staging call included), and in a separate profiled run of two steps each the device time per step of the paced
K2 and of the schedule and descriptor kernels; the card's name and power limit. The last step's fields of --verify streams
of the overlay context are checked against the restatement (tests/overlay_cases.py rendered by the C checker). Writes
nothing into the tree.

  python tools/bench_present_overlay.py [--streams 4096] [--steps 10] [--warmup 2] [--verify 2]
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
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--verify", type=int, default=2, help="streams of the last overlay step checked against the restatement (0: none)")
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import synth
    from tests import overlay_cases as oc

    if not torch.cuda.is_available():
        raise SystemExit("bench_present_overlay.py: no CUDA device; the product has no CPU path")
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
    bitmaps = np.stack([oc.bitmap(s) for s in range(streams)])
    blend = np.full(streams, 60, dtype=np.int32)
    progress = (np.arange(streams, dtype=np.int32) * 7) % 241
    st = 0
    results = {}
    for ntsc in (1, 0):
        std = "ntsc" if ntsc else "pal"
        ctxs = {}
        for name in ("off", "on"):
            c = espflix_b200.Context(n_streams=streams, max_pictures=P, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096,
                                     device=args.device, fields=False)
            c.enable_pts()
            c.video_init(ntsc)
            c.enable_present(1)
            ctxs[name] = c
        w, nl = ctxs["off"].geometry()
        out = torch.empty(3 * streams * w * nl, dtype=torch.uint16, device="cuda")
        keep = {}

        def step(name, keep_fields=False):
            c = ctxs[name]
            c.reset()                                      # keeps the overlay, as video_reset() does
            if name == "on":
                c.present_overlay(bitmaps, blend, progress)
            c.submit_ts(pinned_ts.data_ptr(), off, st, device=False)
            c.index(st)
            n = 0
            for p in range(P):
                info = c.present_picture(p, None, out, st)
                n += int(info["n_fields"].sum())
                if keep_fields:
                    for s in range(args.verify):
                        a, k = int(info[s]["first"]), int(info[s]["n_fields"])
                        keep.setdefault(s, []).append(out[a * w * nl:(a + k) * w * nl].view(torch.int16).cpu().numpy().view(np.uint16).reshape(k, w * nl))
            return n

        for _ in range(args.warmup):
            for name in ctxs:
                step(name)
        ms = {name: 0.0 for name in ctxs}
        fields = {name: 0 for name in ctxs}
        for _ in range(args.steps):                        # alternate the two contexts step by step
            for name in ctxs:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fields[name] += step(name)
                torch.cuda.synchronize()
                ms[name] += 1000.0 * (time.perf_counter() - t0)
        res = {name: {"ms_per_step": round(ms[name] / args.steps, 3), "fields_per_step": fields[name] / args.steps} for name in ctxs}

        from torch.profiler import ProfilerActivity, profile
        for name in ctxs:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                step(name) + step(name)
                torch.cuda.synchronize()
            kern = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
                key = ("schedule" if "ef_pace_kernel" in e.key else "descriptors" if "ef_pace_fill_kernel" in e.key
                       else "staging" if "ef_overlay_stage_kernel" in e.key else "paced_k2" if "ef_composite_kernel" in e.key else None)
                if key:
                    kern[key] = kern.get(key, 0.0) + t
            res[name]["kernel_us_per_step"] = {k: round(v / 2, 1) for k, v in sorted(kern.items())}
        res["paced_k2_on_over_off"] = round(res["on"]["kernel_us_per_step"]["paced_k2"] / res["off"]["kernel_us_per_step"]["paced_k2"], 4)
        res["step_on_over_off"] = round(res["on"]["ms_per_step"] / res["off"]["ms_per_step"], 4)

        if args.verify:                                    # the overlay context's last step against the restatement
            from tests.oracle_lib import Oracle
            o = Oracle()
            runs = args.warmup + args.steps + 2
            step("on", keep_fields=True)
            pts = 129003 + 3003 * np.arange(P)
            for s in range(args.verify):
                dsp = oc.OverlayDisplay(ntsc, 1)
                for _ in range(runs):                      # the steps before: positions and the blend latched at every step's start
                    dsp.reset()
                    dsp.stage(bitmaps[s], int(blend[s]), int(progress[s]))
                    for p in pts:
                        dsp.push(int(p))
                dsp.reset()
                dsp.stage(bitmaps[s], int(blend[s]), int(progress[s]))
                n0 = len(dsp.emitted)
                frames = o.decode_ts(ts[s % d])
                fl = [(f, k) for k, p in enumerate(pts) for f in dsp.push(int(p))[0]]
                ovs = dsp.overlays()[n0:]
                got = np.concatenate(keep[s]) if keep[s] else np.zeros((0, w * nl), np.uint16)
                r = oc.OverlayRenderer(o, ntsc)            # ef_reset zero-filled both stores
                want, k_done = [], -1
                for (f, k), ov in zip(fl, ovs):
                    while k_done < k:                      # push k's fields are drawn once picture k is decoded
                        k_done += 1
                        r.decoded(k_done, frames[k_done])
                    want.append(r.field(f, ov))
                if len(want) != got.shape[0] or any(not np.array_equal(a, b) for a, b in zip(want, got)):
                    raise SystemExit("bench_present_overlay.py: stream %d: fields differ from the restatement" % s)
            res["verify"] = "ok: the last overlay step's fields of %d streams equal the restatement" % args.verify
        results[std] = res
        del out
        for c in ctxs.values():
            c.close()
        torch.cuda.empty_cache()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams x 12 pictures per step (pts step 3003), %d distinct seeds replicated; overlay off / on alternated" % (streams, d),
        "steps": args.steps, "warmup": args.warmup, "card": card, "standards": results}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
