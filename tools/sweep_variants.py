#!/usr/bin/env python3
"""tools/sweep_variants.py — tuning sweeps over compile-time knobs of the CUDA library.

  here (no GPU):   python tools/sweep_variants.py build  tag1="-DEF_K1A_HDR_BATCH=8" tag2="..."
                   cross-compiles espflix_b200/libespflix_b200.<tag>.so for every tag (they travel to the GPU box)
  under gpurun:    python tools/sweep_variants.py run [--check] [--bench-args "..."] tag1 tag2 ...
                   per tag: optional quick parity check (a subset of tests/test_decode_gpu.py, then tests/test_syntax_gpu.py),
                   then bench.py --no-cpu; one line per tag in gpurun_out/sweep_variants.txt
The product library (tag "base" = libespflix_b200.so) is never replaced by a variant."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def lib_name(tag):
    return "libespflix_b200.so" if tag == "base" else "libespflix_b200.%s.so" % tag


def main():
    mode = sys.argv[1]
    args = sys.argv[2:]
    if mode == "build":
        from espflix_b200 import build
        for a in args:
            tag, defs = a.split("=", 1)
            build.build_variant(tag, defs)
            print("built", tag, defs)
        return 0
    check = "--check" in args
    bench_args = "--steps 10 --warmup 3 --no-cpu"
    if "--bench-args" in args:
        i = args.index("--bench-args")
        bench_args = args[i + 1]
        del args[i:i + 2]
    tags = [a for a in args if not a.startswith("--")]
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    out = open(os.path.join(ROOT, "gpurun_out", "sweep_variants.txt"), "a")
    for tag in tags:
        env = dict(os.environ, EF_LIB=lib_name(tag))
        status = ""
        if check:
            r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_decode_gpu.py", "-x", "-q", "-m", "gpu", "-k",
                                "coverage or mixed or outside or multi_picture"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
            if r.returncode == 0:       # the syntax-level streams reach the header and K1b paths the coverage streams do not
                r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_syntax_gpu.py", "-x", "-q", "-m", "gpu"],
                                   cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
            status = "parity " + ("ok" if r.returncode == 0 else "FAILED " + r.stdout[-400:].replace("\n", " | "))
        r = subprocess.run([sys.executable, "bench.py"] + bench_args.split(), cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
        try:
            d = json.loads(r.stdout.strip().splitlines()[-1])
            extra = d.get("stages_ms", {})
            line = "%-28s value %9.0f  ms/step %6.3f  k1 %6.3f  e2e %9.0f  ntsc %.3f pal %.3f  %s %s" % (
                tag, d["value"], d["ms_per_step"], d["roofline"]["k1_ms_per_step"], d["e2e"]["value"],
                d["composite"]["ntsc"]["frac"], d["composite"]["pal"]["frac"], json.dumps(extra), status)
        except Exception as e:      # noqa: BLE001
            line = "%-28s FAILED %s %s %s" % (tag, e, r.stderr[-300:].replace("\n", " | "), status)
        print(line, flush=True)
        out.write(line + "\n")
        out.flush()
    return 0


if __name__ == "__main__":
    sys.exit(main())
