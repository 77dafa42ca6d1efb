"""tools/bench_encode.py — ef_encode_build throughput: a title of `--minutes` at 24 fps (GOP 12) encoded in one call from pinned host
memory, from distinct seeded synthetic clips repeated. Prints one JSON line: wall time, pictures/s, the ef_encode_stage_ms split, the
bytes per picture and the bitrate per GOP against the reference's 1,500 kbit/s, with the card's name and power limit read in the same
run.

  python tools/bench_encode.py [--minutes 60] [--clips 16] [--repeats 2]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    import ctypes
    par = capi.EncodeParams(**capi.ENCODE_DEFAULTS)
    off = np.array([0, n], np.uint64)
    to = np.zeros(2, np.uint64)
    cap = n * 20000
    out = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
    runs = []
    for r in range(a.repeats):
        t0 = time.perf_counter()
        rc = lib.ef_encode_build(0, view.ctypes.data, off.ctypes.data, 1, ctypes.byref(par), out.data_ptr(), cap, to.ctypes.data)
        wall = time.perf_counter() - t0
        if rc != 0:
            raise SystemExit("ef_encode_build: %d %s" % (rc, lib.ef_last_error().decode() if lib.ef_last_error() else ""))
        runs.append(dict(wall_s=round(wall, 3), pictures_per_s=round(n / wall, 1), stage_ms=[round(x, 2) for x in capi.encode_stage_ms()]))
    pk = out[:int(to[1])].numpy().reshape(-1, 188)
    # GOP starts: PES-starting packets without adaptation field whose ES opens with a sequence header (an I picture fills its first packet)
    seq = ((pk[:, 1] & 0x40) != 0) & ((pk[:, 3] & 0x20) == 0) & (pk[:, 18] == 0) & (pk[:, 19] == 0) & (pk[:, 20] == 1) & (pk[:, 21] == 0xB3)
    starts = list(np.nonzero(seq)[0]) + [pk.shape[0]]
    assert len(starts) == n // 12 + 1
    gop_kbit = np.diff(starts) * 188 * 8 / 1000 / 0.5          # a GOP of 12 lasts 0.5 s at 24 fps; TS bytes, headers included
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(pictures=n, gops=n // 12, runs=runs, stage_names=["upload", "search", "code", "recon", "mux"],
                          ts_bytes=int(to[1]), ts_bytes_per_picture=round(int(to[1]) / n, 1), gop_kbit_s=dict(min=round(float(gop_kbit.min()), 1),
                          mean=round(float(gop_kbit.mean()), 1), max=round(float(gop_kbit.max()), 1)), reference_kbit_s=1500, card=card)))


if __name__ == "__main__":
    main()
