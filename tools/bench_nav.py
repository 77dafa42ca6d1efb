#!/usr/bin/env python3
"""tools/bench_nav.py — browsing posters: 4,096 streams stepping one poster right per step, the library against a host-fed twin.

Workload: --titles titles, each a short synthetic main and a poster.ts made by capi.encode_poster; --streams streams, stream s
starting on title s mod titles. Two presenting (NTSC, EF_FIELD_DAC8), carrying, PTS-enabled contexts, timed alternately (--rounds each):
  (a) "library": ef_library_command(EF_LIB_NAV_STEP, +1) over every stream (a stream at the end of the row wraps with EF_LIB_NAV to
      title 0 next step), ef_library_submit of the whole posters, ef_index, ef_present_picture_async of the poster (its mode pushed
      on the device) and ef_present_idle_async of the 17-field scroll;
  (b) "host": the same posters' bytes from pinned host memory (ef_submit_ts_host), ef_restart_streams op 1, ef_end_streams,
      ef_present_overlay of the hidden progress, and the modes passed to ef_present_picture_async by the host.
Each step ends in ef_present_wait and a device synchronise. Reported: ms per step of both arms (median and all rounds) and the card's
name and power limit. Writes nothing into the tree.

  python tools/bench_nav.py [--streams 4096] [--titles 64] [--steps 8] [--warmup 2] [--rounds 3]
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
    ap.add_argument("--titles", type=int, default=64)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    import espflix_b200
    from espflix_b200 import capi
    from tests import restart_cases

    if not torch.cuda.is_available():
        raise SystemExit("bench_nav.py: no CUDA device; the product has no CPU path")
    torch.cuda.set_device(args.device)
    n, T = args.streams, args.titles
    rng = np.random.default_rng(7)
    posters, titles = [], []
    for t in range(T):
        y = np.clip(np.add.outer(np.arange(192) * rng.uniform(0.1, 0.6), np.arange(352) * rng.uniform(0.1, 0.4)) + 20 + t, 0, 235)
        pic = np.concatenate([y.astype(np.uint8).reshape(-1), np.full(2 * 96 * 176, 100 + t, np.uint8)])
        posters.append(capi.encode_poster(pic, device=args.device))
        main = restart_cases.program(1000 + t, 4, 90000)
        titles.append((capi.build_video_idx(main, main, main, device=args.device), main))
    most = max(len(p) for p in posters) // 188
    cap = n * most * 188 + (1 << 20)

    def context():
        ctx = espflix_b200.Context(n_streams=n, max_pictures=2, max_slices_per_picture=12, es_capacity=cap, fields=False, device=args.device)
        ctx.enable_pts()
        ctx.enable_carry(1 << 17)
        ctx.video_init(1)
        ctx.present_format(capi.EF_FIELD_DAC8)              # half the bytes of a U16 field: 4,096 x 18 fields fit in HBM
        ctx.enable_present()
        ctx.present_overlay(np.zeros((n, 1280), np.uint8), np.full(n, 180, np.int32), np.zeros(n, np.int32))
        return ctx

    lib, host = context(), context()
    for k, (idx, main) in enumerate(titles):
        lib.library_add(idx, main)
        lib.library_add_poster(k, posters[k])
    title = np.arange(n) % T
    for s in range(n):                                    # every stream on its first poster
        lib.library_command(capi.LIB_NAV, s, 1, int(title[s]), 0)
    w, nl = lib.geometry()
    out = torch.empty(n * 24 * w * nl, dtype=torch.uint8, device="cuda")
    info = torch.zeros((n, 8), dtype=torch.int32, device="cuda")
    ones, zeros = np.ones(n, np.uint8), np.zeros(n, np.int32)

    def present(ctx, modes):
        ctx.index()
        ctx.present_picture_async(0, out, info, modes=modes)
        ctx.present_idle_async(17, out, info)
        assert ctx.present_wait() == (capi.EF_OK, 2)

    def step_lib(k):
        at_end = np.nonzero(title == T - 1)[0]
        lib.library_command(capi.LIB_NAV_STEP, 0, n, 0, 1)        # the ones at the end of the row stay (nav()'s early return)
        for s in at_end:
            lib.library_command(capi.LIB_NAV, int(s), 1, 0, 0)
        title[:] = (title + 1) % T
        lib.library_submit(most)
        present(lib, None)
        torch.cuda.synchronize()

    htitle = np.arange(n) % T
    blobs = [host.pack([posters[(int(t) + k) % T] for t in htitle]) for k in range(T)]

    def step_host(k):
        blob, off = blobs[(k + 1) % T]
        host.restart_streams(ones)
        host.present_overlay(blend=zeros, set=np.full(n, 2, np.uint8))
        host.submit_ts(blob, off)
        host.end_streams(ones)
        present(host, np.full(n, 2, np.uint8))
        torch.cuda.synchronize()

    res = {"library": [], "host": []}
    for r in range(args.rounds):
        for name, fn in (("library", step_lib), ("host", step_host)):
            for k in range(args.warmup):
                fn(k)
            t0 = time.perf_counter()
            for k in range(args.steps):
                fn(args.warmup + k)
            res[name].append((time.perf_counter() - t0) * 1e3 / args.steps)
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"streams": n, "titles": T, "poster_packets_max": most, "card": card,
                      "ms_per_step": {k: {"median": float(np.median(v)), "rounds": v} for k, v in res.items()}}))
    lib.close()
    host.close()


if __name__ == "__main__":
    main()
