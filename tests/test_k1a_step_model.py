"""CPU model test of K1a's coefficient step: tests/k1a_step_model.cpp compiles the SAME header the kernel uses
(espflix_b200/csrc/ef_coef_step.cuh: one symbol per step through the clz-indexed table, the end-of-block fold, list-entry
packing) for the host and holds it to a symbol-by-symbol restatement of block() (player.cpp:1068-1121) over ~400,000
encoded, random and exhaustive prefix blocks. Runs without a GPU."""
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_one_symbol_step_matches_the_symbol_by_symbol_parser(tmp_path):
    exe = str(tmp_path / "k1a_step_model")
    cuda_inc = "/usr/local/cuda/include"
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", cuda_inc, "-x", "c++", os.path.join(ROOT, "tests", "k1a_step_model.cpp"),
                    os.path.join(ROOT, "espflix_b200", "csrc", "ef_tables.cpp"), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["bad"] == 0 and out["blocks"] > 400000 and out["coefficients"] > 2000000
