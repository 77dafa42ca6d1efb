"""tools/bench_encode_audio.py — ef_sbc_encode and ef_mux_audio throughput, with the card's name and power limit read in the same run.

Encode: `--titles` titles of `--minutes` of seeded synthetic 48 kHz mono PCM each at the defaults (bit pool 28, 64-byte frames),
from pinned host memory into pinned host memory, in calls of at most `--per-call` titles (the host holds 345.6 MB of PCM and 24 MB
of SBC per title-hour of one call). Each call is repeated until at least `--seconds` of wall time have passed; one JSON line per
title count gives the mean wall time of the whole set of calls, frames/s, the ef_audio_encode_stage_ms split summed over the calls
and the share of the stage time spent on the host link (upload + download).
Mux: one title of `--minutes` at 24 fps (a video PES of 15 packets per picture, the size ef_encode_build gives synthetic clips)
with its SBC, through capi.mux_audio (the sizing call, then the writing call): wall time and ef_audio_encode_stage_ms's mux stage.

  python tools/bench_encode_audio.py [--minutes 60] [--titles 1 64 256] [--per-call 64] [--seconds 2]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--titles", type=int, nargs="+", default=[1, 64, 256])
    ap.add_argument("--per-call", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=2.0)
    a = ap.parse_args()
    import torch
    from espflix_b200 import capi

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lib = capi.load_library()
    par = capi.AudioParams(**capi.AUDIO_ENCODE_DEFAULTS)
    n = int(a.minutes * 60 * 48000)
    seed = np.random.default_rng(2026).normal(0, 4000, 48000 * 10).clip(-32768, 32767).astype(np.int16)   # 10 s, repeated
    per = min(max(a.titles), a.per_call)
    pcm = torch.empty(per * n, dtype=torch.int16, pin_memory=True)
    view = pcm.numpy()
    for o in range(0, view.size, seed.size):
        view[o:o + seed.size] = seed[:view.size - o]
    fpt = (n + 127) // 128
    out = torch.empty(per * fpt * 64, dtype=torch.uint8, pin_memory=True)
    so = np.zeros(per + 1, np.uint64)

    def call(titles):
        off = np.arange(titles + 1, dtype=np.uint64) * n
        rc = lib.ef_sbc_encode(0, pcm.data_ptr(), off.ctypes.data, titles, ctypes.byref(par), out.data_ptr(), out.numel(), so.ctypes.data)
        assert rc == 0, lib.ef_last_error()
        return capi.audio_encode_stage_ms()

    call(1)                                                         # loads the module: not counted
    for titles in a.titles:
        calls = [per] * (titles // per) + ([titles % per] if titles % per else [])
        walls, ms = [], np.zeros(3)
        t_all = time.perf_counter()
        while not walls or time.perf_counter() - t_all < a.seconds:
            t = time.perf_counter()
            stage = np.zeros(3)
            for c in calls:
                stage += call(c)[:3]
            walls.append(time.perf_counter() - t)
            ms = stage
        wall = float(np.mean(walls))
        link = ms[0] + ms[2]
        print(json.dumps({"gpu": gpu, "what": "encode", "titles": titles, "calls": len(calls), "minutes": a.minutes, "frames": titles * fpt,
                          "repeats": len(walls), "wall_s_mean": round(wall, 4), "wall_s_min": round(min(walls), 4),
                          "wall_s_max": round(max(walls), 4), "frames_per_s": round(titles * fpt / wall),
                          "stage_ms_last": {"upload": round(ms[0], 2), "encode": round(ms[1], 2), "download": round(ms[2], 2)},
                          "host_link_share": round(link / max(ms.sum(), 1e-9), 3)}))

    # mux: one title's video.ts of n_pic pictures (PES of 15 packets) and its SBC
    n_pic = int(a.minutes * 60 * 24)
    pk = np.zeros((n_pic * 15, 188), np.uint8)
    pk[:, 0], pk[:, 1], pk[:, 3] = 0x47, 0x01, 0x10 | (np.arange(pk.shape[0]) & 15)
    st = pk[::15]
    st[:, 1] = 0x41
    st[:, 4:13] = [0, 0, 1, 0xE0, 0, 0, 0x80, 0x80, 5]
    pts = np.arange(n_pic, dtype=np.int64) * 3750
    st[:, 13] = 0x21 | ((pts >> 29) & 0x0E)
    st[:, 14] = (pts >> 22) & 0xFF
    st[:, 15] = 0x01 | ((pts >> 14) & 0xFE)
    st[:, 16] = (pts >> 7) & 0xFF
    st[:, 17] = 0x01 | ((pts << 1) & 0xFE)
    video = pk.tobytes()
    sbc = out.numpy()[:fpt * 64].tobytes()
    walls = []
    for _ in range(2):
        t = time.perf_counter()
        muxed = capi.mux_audio([video], [sbc])[0]
        walls.append(time.perf_counter() - t)
    pes = [min(8, fpt - f) for f in range(0, fpt, 8)]
    assert len(muxed) == len(video) + 188 * sum((14 + 64 * k + 183) // 184 for k in pes)
    print(json.dumps({"gpu": gpu, "what": "mux", "minutes": a.minutes, "video_pes": n_pic, "audio_pes": len(pes),
                      "wall_s": [round(w, 3) for w in walls], "mux_ms_writing_call": round(capi.audio_encode_stage_ms()[3], 1),
                      "out_mb": round(len(muxed) / 1e6, 1)}))


if __name__ == "__main__":
    main()
