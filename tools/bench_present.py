#!/usr/bin/env python3
"""tools/bench_present.py — paced presentation (ef_present_*) at batch scale.

Workload: bench.py's config 4 (4,096 streams x one GOP of 12 pictures, 64 distinct seeds replicated) as transport streams
(espflix_b200.synth.wrap_ts: pts 129003 + 3003 k). Per step: ef_submit_ts_host -> ef_index -> ef_present_picture(0..11)
into one device buffer that holds the fields of one picture index (3 per stream). Every step is a new 12-picture clip per
stream, so a step starts with ef_reset, video_reset() as a player does between files: the same pts again without it would
put every display's next flip 2^32 fields ahead (push_video's unsigned arithmetic), which ef_present_picture reports as
EF_ENOMEM. Both standards, one context each.
Reported per standard: ms per step (host clock around synchronous calls), fields/s, the device time per step of the
schedule, descriptor and paced K2 kernels (torch.profiler, two untimed steps), and the paced K2's output bytes/s against
ef_composite_field's on the same context in the same profiled run; the card's name and power limit. An extra step at the
end is checked, for --verify streams, against the restatement in tests/present_cases.py rendered by the C checker. Writes
nothing into the tree.

  python tools/bench_present.py [--streams 4096] [--steps 10] [--warmup 2] [--verify 3]
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
    ap.add_argument("--verify", type=int, default=3, help="streams of the extra step checked against the restatement (0: none)")
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_present.py: no CUDA device; the product has no CPU path")
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
                                   device=args.device, fields=True)
        ctx.enable_pts()
        ctx.video_init(ntsc)
        ctx.enable_present(1)                              # frame counter 1: not the _frame_counter_origin == 0 quirk
        w, nl = ctx.geometry()
        cap = 3 * streams
        out = torch.empty(cap * w * nl, dtype=torch.uint16, device="cuda")
        keep = {}

        def step(keep_fields=False):
            ctx.reset()
            ctx.submit_ts(pinned_ts.data_ptr(), off, st, device=False)
            ctx.index(st)
            n = 0
            for p in range(P):
                info = ctx.present_picture(p, None, out, st)
                n += int(info["n_fields"].sum())
                if keep_fields:
                    for s in range(args.verify):
                        a, k = int(info[s]["first"]), int(info[s]["n_fields"])
                        keep.setdefault(s, []).append(out[a * w * nl:(a + k) * w * nl].view(torch.int16).cpu().numpy().view(np.uint16).reshape(k, w * nl))
            return n

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        fields = sum(step() for _ in range(args.steps))
        torch.cuda.synchronize()
        ms = 1000.0 * (time.perf_counter() - w0) / args.steps
        res = {"ms_per_step_with_reset": round(ms, 3), "fields_per_step": fields / args.steps, "fields_per_s": round(fields / (ms * args.steps / 1000.0)),
               "field_bytes": w * nl * 2}

        from torch.profiler import ProfilerActivity, profile   # device time per kernel, two untimed steps + 4 plain K2 launches
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            pf = step() + step()
            for k in range(4):
                ctx.composite_field(-1, k, st)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            if "ef_pace_kernel" in e.key:
                kern["schedule"] = kern.get("schedule", 0.0) + t
            elif "ef_pace_fill_kernel" in e.key:
                kern["descriptors"] = kern.get("descriptors", 0.0) + t
            elif "ef_composite_kernel" in e.key and ("true, true" in e.key or "false, true" in e.key):
                kern["paced_k2"] = kern.get("paced_k2", 0.0) + t
            elif "ef_composite_kernel" in e.key:
                kern["composite_field"] = kern.get("composite_field", 0.0) + t
        fb = w * nl * 2
        res["kernel_us_per_step"] = {k: round(kern.get(k, 0.0) / 2, 1) for k in ("schedule", "descriptors", "paced_k2")}
        res["paced_k2_GBps"] = round(pf * fb / (kern["paced_k2"] * 1e3), 1)
        res["composite_field_GBps"] = round(4 * streams * fb / (kern["composite_field"] * 1e3), 1)
        res["paced_over_plain"] = round(res["paced_k2_GBps"] / res["composite_field_GBps"], 3)

        if args.verify:                                    # the extra step against the restatement
            from tests import present_cases as pc
            from tests.oracle_lib import Oracle
            o = Oracle()
            disp = [pc.Display(ntsc, 1) for _ in range(args.verify)]
            pts = 129003 + 3003 * np.arange(P)
            for _ in range(args.warmup + args.steps + 2):
                for dsp in disp:
                    dsp.reset()
                    for p in pts:
                        dsp.push(int(p))
            for dsp in disp:
                dsp.reset()
            step(keep_fields=True)
            for s in range(args.verify):
                frames = o.decode_ts(ts[s % d])
                r = pc.Renderer(o, ntsc)                      # ef_reset zero-filled both stores
                got = np.concatenate(keep[s]) if keep[s] else np.zeros((0, w * nl), np.uint16)
                want = []
                for k, p in enumerate(pts):
                    r.decoded(k, frames[k])
                    want += [r.field(f) for f in disp[s].push(int(p))[0]]
                if len(want) != got.shape[0] or any(not np.array_equal(a, b) for a, b in zip(want, got)):
                    raise SystemExit("bench_present.py: stream %d: fields differ from the restatement" % s)
            res["verify"] = "ok: the last step's fields of %d streams equal the restatement" % args.verify
        results["ntsc" if ntsc else "pal"] = res
        del out
        ctx.close()
        torch.cuda.empty_cache()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams x 12 pictures per step (pts step 3003), %d distinct seeds replicated" % (streams, d),
        "steps": args.steps, "warmup": args.warmup, "card": card, "standards": results}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
