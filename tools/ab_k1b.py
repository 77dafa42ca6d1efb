#!/usr/bin/env python3
"""tools/ab_k1b.py — two builds of the CUDA library timed against each other on the benchmark's step, alternated in one
process on one card.

  tools/ab_k1b.py --build-a REV      compile REV's espflix_b200/csrc (git archive) into espflix_b200/libespflix_b200.a_<REV>.so
                                     (needs git and nvcc, no GPU)
  tools/ab_k1b.py --a LIB [--b LIB ...]  time arm A against one or more B arms (default B: the product library)

Each arm gets its own context with bench.py's 4,096 resident streams (64 distinct seeds). After a warm-up of both, the
arms alternate A B A B ...: `--pairs` rounds of `--steps` steps (ef_index + ef_decode_all(12)) between two CUDA events,
then three profiled steps for the library's own stage split (K1a, 12 x K1b). Prints per arm the median and the range over
the rounds, the card's name and power limit read in the same run, and whether the two arms decoded the same pictures.
One JSON line at the end."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PICTURES = 12


def build_rev(rev):
    from espflix_b200 import build
    out = os.path.join(build.PKG, "libespflix_b200.a_%s.so" % rev.replace("/", "_"))
    with tempfile.TemporaryDirectory() as tmp:
        tar = subprocess.run(["git", "-C", ROOT, "archive", rev, "espflix_b200/csrc", "include"], capture_output=True, check=True).stdout
        subprocess.run(["tar", "-x", "-C", tmp], input=tar, check=True)
        csrc = os.path.join(tmp, "espflix_b200", "csrc")
        build._run([build.nvcc_path()] + list(build.NVCC_FLAGS) + ["-o", out] + [os.path.join(csrc, s) for s in build.CUDA_SOURCES], cwd=csrc)
    print(out)


def open_arm(path, streams, stream_list, capacity):
    """a context of the library at `path` (the binding keeps one library per context)"""
    from espflix_b200 import capi
    os.environ["EF_LIB"] = os.path.abspath(path)
    capi._lib = None
    ctx = capi.Context(n_streams=streams, max_pictures=PICTURES, max_slices_per_picture=12, es_capacity=capacity, fields=False)
    blob, off = ctx.pack(stream_list)
    ctx.submit_es(blob, off)
    return ctx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-a", metavar="REV")
    ap.add_argument("--a")
    ap.add_argument("--b", nargs="+", default=[os.path.join(ROOT, "espflix_b200", "libespflix_b200.so")])
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--pairs", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if args.build_a:
        return build_rev(args.build_a)
    if not args.a:
        ap.error("--a LIB is required")

    import numpy as np
    import torch
    import bench
    if not torch.cuda.is_available():
        raise SystemExit("ab_k1b.py: no CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    _, stream_list = bench.make_streams(args.streams)
    capacity = sum(len(s) for s in stream_list) + 4096
    names = ["a"] + ["b%d" % i if len(args.b) > 1 else "b" for i in range(len(args.b))]
    arms = {k: open_arm(p, args.streams, stream_list, capacity) for k, p in zip(names, [args.a] + args.b)}

    def step(ctx):
        ctx.index(0)
        ctx.decode_all(PICTURES, 0)

    for ctx in arms.values():
        for _ in range(3):
            step(ctx)
    torch.cuda.synchronize()
    want = arms["a"].read_latest_i420()
    same = all(bool(np.array_equal(want, arms[k].read_latest_i420())) for k in names[1:])
    del want

    rounds = {k: {"step": [], "k1a": [], "k1b": []} for k in arms}
    for _ in range(args.pairs):
        for k, ctx in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.steps):
                step(ctx)
            e1.record()
            torch.cuda.synchronize()
            rounds[k]["step"].append(e0.elapsed_time(e1) / args.steps)
            ctx.set_profiling(True)
            st = np.zeros(3)
            for _ in range(3):
                step(ctx)
                st += np.array(ctx.stage_ms())
            ctx.set_profiling(False)
            rounds[k]["k1a"].append(float(st[1]) / 3)
            rounds[k]["k1b"].append(float(st[2]) / 3)

    out = {"card": card, "streams": args.streams, "pairs": args.pairs, "steps": args.steps, "same_pictures": same,
           "libs": {k: os.path.basename(p) for k, p in zip(names, [args.a] + args.b)}}
    print("card: %s; %d streams x %d pictures; %d alternated rounds of %d steps; same pictures: %s" % (card, args.streams, PICTURES, args.pairs, args.steps, same))
    for what, label in (("step", "step ms"), ("k1a", "K1a ms"), ("k1b", "12 x K1b ms")):
        for k in arms:
            v = rounds[k][what]
            out["%s_%s" % (k, what)] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
            print("  %-12s %s  median %.3f  range %.3f - %.3f" % (label, k.upper(), statistics.median(v), min(v), max(v)))
        a = out["a_" + what]
        for k in names[1:]:
            b = out["%s_%s" % (k, what)]
            out["%s_%s_over_a" % (what, k)] = b["median"] / a["median"]
            out["%s_%s_ranges_overlap" % (what, k)] = not (b["max"] < a["min"] or a["max"] < b["min"])
    fps = {k: args.streams * PICTURES / (out[k + "_step"]["median"] / 1000.0) for k in arms}
    out["frames_per_s"] = fps
    print("  frames/s     " + "  ".join("%s %.0f (x%.4f)" % (k.upper(), fps[k], fps[k] / fps["a"]) for k in names))
    print(json.dumps(out))
    for ctx in arms.values():
        ctx.close()
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
