#!/usr/bin/env python3
"""tools/phase_k1b.py — where a warp of K1b (ef_recon_kernel) spends its time, phase by phase, on the benchmark's batch.

Builds the measurement variant of the library (-DEF_K1B_PHASE_CLOCKS: lane 0 of every warp sums clock64() ticks per phase of
an iteration; espflix_b200/libespflix_b200.phase.so, never the product and never timed against it), decodes bench.py's
4,096 resident streams x 12 pictures `--steps` times and prints each phase's share of a warp's iteration, the ticks per
iteration, and the card's name and power limit. The ticks are wall time of one warp among those resident on its SM: a
phase's share says where a warp waits or works, not how many instructions it issues.
`--build-only` compiles the variant and stops (no GPU needed)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PHASES = ["record decode, list loads and tile copy issued, skip copy", "list expansion (waits for the list loads)", "column passes",
          "wait for the reference tiles", "row IDCT", "prediction", "combine + store"]
PICTURES = 12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--build-only", action="store_true")
    args = ap.parse_args()
    from espflix_b200 import build
    lib = os.path.join(build.PKG, "libespflix_b200.phase.so")
    if args.build_only or not os.path.exists(lib):
        lib = build.build_variant("phase", "-DEF_K1B_PHASE_CLOCKS")
    if args.build_only:
        print(lib)
        return 0

    os.environ["EF_LIB"] = lib
    import numpy as np
    import torch
    import bench
    from espflix_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("phase_k1b.py: no CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    _, stream_list = bench.make_streams(args.streams)
    ctx = capi.Context(n_streams=args.streams, max_pictures=PICTURES, max_slices_per_picture=12,
                       es_capacity=sum(len(s) for s in stream_list) + 4096, fields=False)
    read = ctx.lib.ef_k1b_phase_clocks
    read.restype, read.argtypes = ctypes.c_int, [ctypes.c_void_p]
    blob, off = ctx.pack(stream_list)
    ctx.submit_es(blob, off)
    ticks = np.zeros(len(PHASES) + 1, dtype=np.uint64)
    for k in range(2 + args.steps):
        if k == 2:                       # two warm-up steps, then clear the sums
            assert read(ticks.ctypes.data) == 0
        ctx.index(0)
        ctx.decode_all(PICTURES, 0)
    assert read(ticks.ctypes.data) == 0
    ctx.close()
    total, iters = float(ticks[:-1].sum()), int(ticks[-1])
    print("card: %s; %d streams x %d pictures x %d steps; %d warp iterations, %.0f ticks each" % (card, args.streams, PICTURES, args.steps, iters, total / iters))
    for name, t in zip(PHASES, ticks[:-1]):
        print("  %5.1f %%  %7.0f ticks  %s" % (100.0 * float(t) / total, float(t) / iters, name))
    print(json.dumps({"card": card, "iterations": iters, "ticks_per_iteration": total / iters,
                      "share": {n: float(t) / total for n, t in zip(PHASES, ticks[:-1])}}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
