"""tools/bench_encode_rate.py — ef_encode_build_rate throughput against ef_encode_build in the same run: a title of `--minutes` at 24 fps
(GOP 12) of bench_encode.py's seeded synthetic clips, encoded from pinned host memory at ENCODE_RATE_DEFAULTS (1.5 Mbit/s, 250,000
bits, q 3..31) and at the fixed q8 / q8. Prints one JSON line: wall time and pictures/s of both, the ef_encode_stage_ms split (the
census and the choice count in "code"), the largest bucket draw and the fallback count, the quantiser histogram, ES and TS kbit/s per
GOP, with the card's name and power limit read in the same run.

  python tools/bench_encode_rate.py [--minutes 60] [--clips 16] [--repeats 2]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gop_kbit(pk, n):
    """TS kbit/s of every GOP of 12 pictures (0.5 s at 24 fps): packets from one GOP's sequence header to the next"""
    seq = ((pk[:, 1] & 0x40) != 0) & ((pk[:, 3] & 0x20) == 0) & (pk[:, 18] == 0) & (pk[:, 19] == 0) & (pk[:, 20] == 1) & (pk[:, 21] == 0xB3)
    starts = list(np.nonzero(seq)[0]) + [pk.shape[0]]
    assert len(starts) == n // 12 + 1
    return np.diff(starts) * 188 * 8 / 1000 / 0.5


def stats(v):
    return dict(min=round(float(v.min()), 1), mean=round(float(v.mean()), 1), max=round(float(v.max()), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    import torch
    from espflix_b200 import capi
    from tests import encode_cases as ec

    n = int(round(a.minutes * 60 * 24))
    n -= n % 12
    clips = [ec.translated(100 + c, 12, ((c % 5) - 2, (c % 3) - 1)) for c in range(a.clips)]
    buf = torch.empty((n, ec.PICTURE_BYTES), dtype=torch.uint8, pin_memory=True)
    view = buf.numpy()
    for g in range(n // 12):
        view[g * 12:(g + 1) * 12] = clips[g % a.clips]
    lib = capi.load_library()
    par = capi.EncodeParams(**capi.ENCODE_DEFAULTS)
    rp = capi.RateParams(**capi.ENCODE_RATE_DEFAULTS)
    off = np.array([0, n], np.uint64)
    to = np.zeros(2, np.uint64)
    cap = n * 20000
    out = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
    q = np.zeros(n, np.uint8)
    nb = np.zeros(n, np.uint32)
    result = {}
    for mode in ("rate", "fixed"):
        runs = []
        for r in range(a.repeats):
            t0 = time.perf_counter()
            if mode == "rate":
                rc = lib.ef_encode_build_rate(0, view.ctypes.data, off.ctypes.data, 1, ctypes.byref(par), ctypes.byref(rp), out.data_ptr(), cap,
                                              to.ctypes.data, q.ctypes.data, nb.ctypes.data)
            else:
                rc = lib.ef_encode_build(0, view.ctypes.data, off.ctypes.data, 1, ctypes.byref(par), out.data_ptr(), cap, to.ctypes.data)
            wall = time.perf_counter() - t0
            if rc != 0:
                raise SystemExit("%s: %d %s" % (mode, rc, lib.ef_last_error().decode() if lib.ef_last_error() else ""))
            runs.append(dict(wall_s=round(wall, 3), pictures_per_s=round(n / wall, 1), stage_ms=[round(x, 2) for x in capi.encode_stage_ms()]))
        pk = out[:int(to[1])].numpy().reshape(-1, 188)
        result[mode] = dict(runs=runs, ts_bytes=int(to[1]), gop_ts_kbit_s=stats(gop_kbit(pk, n)))
    # the bucket of every GOP from the rate encode's picture sizes, in 1/90000 bit
    U, B = 90000, capi.ENCODE_RATE_DEFAULTS["vbv_bits"]
    r = capi.ENCODE_RATE_DEFAULTS["bit_rate"] * capi.ENCODE_DEFAULTS["pts_step"]
    s = nb.astype(np.int64).reshape(-1, 12) * 8 * U
    f = np.full(s.shape[0], B * U, np.int64)
    draw = np.zeros(s.shape[0], np.int64)
    for j in range(12):
        draw = np.maximum(draw, B * U - (f - s[:, j]))
        assert (s[:, j] <= f).all()
        f = np.minimum(B * U, f - s[:, j] + r)
    result["rate"].update(max_bucket_draw_bits=int(draw.max() // U), vbv_bits=B, fallbacks=int((q == 0).sum()),
                          q_histogram={int(k): int(v) for k, v in zip(*np.unique(q, return_counts=True))},
                          gop_es_kbit_s=stats(nb.astype(np.int64).reshape(-1, 12).sum(axis=1) * 8 / 1000 / 0.5))
    rw = min(x["wall_s"] for x in result["rate"]["runs"])
    fw = min(x["wall_s"] for x in result["fixed"]["runs"])
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(pictures=n, gops=n // 12, rate_params=capi.ENCODE_RATE_DEFAULTS, stage_names=["upload", "search", "code", "recon", "mux"],
                          rate=result["rate"], fixed_q8=result["fixed"], rate_over_fixed_wall=round(rw / fw, 2), reference_kbit_s=1500,
                          card=card)))


if __name__ == "__main__":
    main()
