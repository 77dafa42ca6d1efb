#!/usr/bin/env python3
"""tools/bench_restart.py — per-stream restarts (ef_restart_streams) at batch scale, against ef_reset of the whole batch.

Workload: 4,096 TS streams x 12 pictures per step (bench.py's video ES, 64 titles replicated) with SBC audio on PID 0x102
(150 frames of 64 bytes per GOP, as tools/bench_audio.py muxes it), PTS and audio enabled. Every step is the next GOP of
each stream's program: video pts and audio PES pts continue from step to step and the audio bytes are the program's next
150 frames. Per step: ef_submit_ts_host -> ef_index -> ef_decode_all -> ef_decode_audio.
Arm "restart": from step 1 on, before each step a rotating twelfth of the streams (group k % 12) switches to a new title
(op 1, then that title's first GOP); the others go on. Arm "reset": the same input, with ef_reset of every stream before
every step, today's only way to restart any of them. Both arms run in one process on one context each, steps alternating.
Reported: ms per step of each arm (host clock around synchronous calls), the restart call's and ef_reset's host time, the
device time of the restart kernels and of ef_reset's memsets (torch.profiler over extra steps), and the card's name and power
limit. --verify streams of the restart arm (half of them in the group restarted last, half untouched the longest) are
checked over every step run: get_pts() -1 right after their restart, the pts of every picture, and their whole PCM and PDM
against the restatement in tests/restart_cases.py. Writes nothing into the tree.

  python tools/bench_restart.py [--streams 4096] [--steps 12] [--warmup 2] [--verify 4]
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

AUDIO_FRAMES = 150                                        # per GOP, 64 bytes each
GOPS = 12                                                 # a stream restarts every 12 steps: GOP index 0..11


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--verify", type=int, default=4)
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from tests import audio_cases, pts_cases, restart_cases
    from tests.oracle_lib import Oracle

    if not torch.cuda.is_available():
        raise SystemExit("bench_restart.py: no CUDA device; the product has no CPU path")
    torch.cuda.set_device(args.device)
    streams, P = args.streams, bench.PICTURES
    gen, _ = bench.make_streams(streams)
    T = len(gen)
    base = [1000000 + 777777 * t for t in range(T)]
    sbc = [audio_cases.sbc_stream(7000 + t, AUDIO_FRAMES * GOPS, bitpool=28) for t in range(T)]
    chunk = AUDIO_FRAMES * 64

    def gop_ts(t, g):
        es = bytes(gen[t][0])
        codes = pts_cases.picture_codes(es)
        pts = [base[t] + 3003 * (P * g + p) for p in range(len(codes))]
        video = pts_cases.wrap(es, [0] + [c - 3 for c in codes[1:]], ["pts"] * len(codes), pts, seed=t)
        audio = audio_cases.mux_audio_ts(sbc[t][g * chunk:(g + 1) * chunk], pid=0x102, first_pts=base[t] + 3003 * P * g)
        return np.concatenate([np.frombuffer(video, dtype=np.uint8), audio])

    table = {(t, g): gop_ts(t, g) for t in range(T) for g in range(GOPS)}
    cap = max(sum(len(table[(i + j) % T, 0]) for i in range(streams)) for j in range(1)) + streams * 4096
    pinned = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
    title = np.arange(streams) % T
    start = np.zeros(streams, dtype=np.int64)             # step at which the stream's current program started
    group = (streams + 11) // 12

    def plan(k):
        """ops and input of step k (advances the programs)"""
        ops = np.zeros(streams, dtype=np.uint8)
        if k:
            g = k % 12
            ops[g * group:(g + 1) * group] = 1
            title[ops == 1] = (title[ops == 1] + 1 + k) % T
            start[ops == 1] = k
        off = np.zeros(streams + 1, dtype=np.uint64)
        parts = [table[int(title[i]), int(k - start[i])] for i in range(streams)]
        off[1:] = np.cumsum([len(p) for p in parts])
        assert int(off[-1]) <= cap
        pinned.numpy()[:int(off[-1])] = np.concatenate(parts)
        return ops, off

    ctxs = {}
    for arm in ("restart", "reset"):
        c = espflix_b200.Context(n_streams=streams, max_pictures=P, max_slices_per_picture=12, es_capacity=cap, device=args.device, fields=False)
        c.enable_pts()
        c.enable_audio()
        ctxs[arm] = c
    times = {"restart": [], "reset": [], "restart_call": [], "reset_call": []}
    n_pcm = streams * AUDIO_FRAMES * 2 * 128
    pcm_out, pdm_out = np.zeros(n_pcm, np.int16), np.zeros(2 * n_pcm, np.uint16)
    last_group = None
    track = {}                                             # stream -> dict(history, pcm, pdm, pts_ok)
    bad = []

    def step(arm, k, ops, off, record):
        c = ctxs[arm]
        t0 = time.perf_counter()
        a = time.perf_counter()
        if arm == "restart":
            c.restart_streams(ops)
        else:
            c.reset()
        t_call = time.perf_counter() - a
        c.submit_ts(pinned.numpy(), off)
        c.index()
        c.decode_all(P)
        res = c.decode_audio(pcm_out=pcm_out, pdm_out=pdm_out)
        c.sync()
        t = time.perf_counter() - t0
        if record:
            times[arm].append(t)
            times[arm + "_call"].append(t_call)
        return res

    o = Oracle()
    total = args.warmup + args.steps + 2
    lg = (total - 1) % 12                                  # the group the last step restarts
    half = max(args.verify, 2) // 2
    vstreams = [lg * group + j for j in range(half)] + [((lg + 1) % 12) * group + j for j in range(half)]   # restarted last / longest ago
    for s in vstreams:
        track[s] = dict(runs=[[]], pcm=[], pdm=[])
    from torch.profiler import ProfilerActivity, profile
    dev = {}
    for k in range(total):
        ops, off = plan(k)
        profiled = k >= args.warmup + args.steps
        for arm in ("restart", "reset"):
            if profiled:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    res = step(arm, k, ops, off, False)
                for e in prof.key_averages():
                    if (arm == "restart" and ("restart" in e.key or "audio_end" in e.key)) or (arm == "reset" and "Memset" in e.key):
                        name = "ef_restart_kernel" if "restart" in e.key else "ef_audio_end_kernel" if "audio_end" in e.key else e.key
                        dev.setdefault(arm, {}).setdefault(name, []).append(e.device_time_total)
            else:
                res = step(arm, k, ops, off, k >= args.warmup)
            if arm == "restart":
                if ops.any():
                    last_group = k % 12
                pic, last = ctxs[arm].picture_pts()
                for s in vstreams:
                    tr = track[s]
                    g = k - int(start[s])
                    if ops[s] and k:
                        tr["runs"].append([])
                    tr["runs"][-1].append(bytes(sbc[int(title[s])][g * chunk:(g + 1) * chunk]))
                    t_ = int(title[s])
                    want = [base[t_] + 3003 * (P * g + p) for p in range(P)]
                    if pic[s].tolist() != want or int(last[s]) != want[-1]:
                        bad.append(("pts", s, k))
                    tr["pcm"].append(res[s]["pcm"])
                    tr["pdm"].append(res[s]["pdm"])
    # get_pts() of a restarted stream reads -1 until its next picture
    c = ctxs["restart"]
    ops = np.zeros(streams, dtype=np.uint8)
    ops[vstreams[0]] = 1
    c.restart_streams(ops)
    if int(c.picture_pts(first=vstreams[0], count=1, n_pictures=0)[1][0]) != -1:
        bad.append(("get_pts", vstreams[0], total))
    for s in vstreams:
        tr = track[s]
        runs = [b"".join(r) for r in tr["runs"]]
        want_pcm, want_pdm = restart_cases.audio_restate_runs(o, runs, 64)
        if not np.array_equal(np.concatenate(tr["pcm"]), np.concatenate(want_pcm)) or not np.array_equal(np.concatenate(tr["pdm"]), want_pdm):
            bad.append(("audio", s, len(runs)))
    restarted_last = [s for s in vstreams if last_group is not None and last_group * group <= s < (last_group + 1) * group]

    def smi(q):
        try:
            return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", str(args.device)], capture_output=True,
                                  text=True, timeout=30).stdout.strip()
        except Exception:
            return "?"

    ms = lambda v: round(1000 * float(np.median(v)), 3)       # noqa: E731
    print(json.dumps({
        "card": torch.cuda.get_device_name(args.device), "power_limit": smi("power.limit"), "streams": streams, "pictures": P,
        "audio_frames_per_step": AUDIO_FRAMES, "steps": args.steps,
        "step_ms_restart_twelfth": ms(times["restart"]), "step_ms_reset_all": ms(times["reset"]),
        "restart_call_host_ms": ms(times["restart_call"]), "reset_call_host_ms": ms(times["reset_call"]),
        "device_us_per_step": {arm: {k: round(float(np.mean(v)), 2) for k, v in d.items()} for arm, d in dev.items()},
        "verified_streams": vstreams, "verified_restarted_in_last_group": restarted_last,
        "restarts_per_verified_stream": {s: len(track[s]["runs"]) - 1 for s in vstreams}, "verify_failures": bad}))
    for c in ctxs.values():
        c.close()
    if bad:
        raise SystemExit("bench_restart.py: verification failed")


if __name__ == "__main__":
    main()
