#!/usr/bin/env python3
"""tools/bench_keys.py — the remote at scale: 4,096 streams, each pressed a seeded key every step, through submit, index and the async
present chain; one ef_library_keys against what a caller has to do without it.

Workload: --titles titles, each a short synthetic main (also used as its fwd and rwd file) and a poster.ts made by capi.encode_poster;
--streams streams, stream s starting on the poster of title s mod titles. Every step each stream gets a seeded key (no key, an unknown
code or one of the seven, so posters are browsed, titles play, pause, skip, trick-play and end). Two presenting (NTSC, EF_FIELD_DAC8),
carrying, PTS-enabled contexts with overlays and clocks on, timed alternately (--rounds each):
  (a) "keys": ef_library_keys with the step's keys;
  (b) "commands": ef_library_info, then per stream the command its key runs as on the state read back (MENU first on an ended title),
      one ef_library_command per run of equal commands over neighbouring streams, then ef_present_overlay of the blends and
      ef_present_clock of the clock states loop() leaves.
Then, in both: ef_library_submit of --packets per stream, ef_index, ef_present_picture_async of every picture index,
ef_present_idle_async of 2 fields, ef_present_wait and a device synchronise. Both arms run the same keys from the same state, so
they do the same work after the keys. Reported: ms per step of both arms (median and all rounds) and the card's name and power
limit. Writes nothing into the tree.

  python tools/bench_keys.py [--streams 4096] [--titles 64] [--steps 6] [--warmup 2] [--rounds 3]
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


def command_of(state, speed, key, capi):
    """what a caller without ef_library_keys must work out from the state it read back: (command, arg, blend or None, zero the
    clock's seconds) for the key on that state (the DONE branch handled before)"""
    play, side, vert = key in (capi.KEY_PLAY, capi.KEY_SELECT), key in (capi.KEY_RIGHT, capi.KEY_LEFT), key in (capi.KEY_UP, capi.KEY_DOWN)
    sign = 1 if key in (capi.KEY_RIGHT, capi.KEY_UP) else -1
    if state == capi.LIB_POSTER:
        return (capi.LIB_PLAY, 0, 180, True) if play else (capi.LIB_NAV_STEP, sign, 0, False) if side else (None, 0, None, False)
    if state == capi.LIB_PLAYING:
        if key == capi.KEY_MENU:
            return (capi.LIB_MENU, 0, 180, True) if speed else (capi.LIB_MENU, 0, 0, False)
        if speed and (play or side or vert):
            return capi.LIB_PLAY, 0, 180, True
        if play:
            return capi.LIB_PAUSE, 0, 180, True
        if side:
            return (capi.LIB_FAST_FORWARD if sign > 0 else capi.LIB_REWIND), 0, -1, False
        if vert:
            return capi.LIB_SKIP, 30 * sign, 180, False
    if state == capi.LIB_PAUSED:
        if key == capi.KEY_MENU:
            return capi.LIB_MENU, 0, 0, False
        if play:
            return capi.LIB_RESUME, 0, 180, True
        if side:
            return (capi.LIB_FAST_FORWARD if sign > 0 else capi.LIB_REWIND), 0, -1, False
    if state == capi.LIB_STOPPED and key == capi.KEY_MENU:
        return capi.LIB_MENU, 0, 0, False
    return None, 0, None, play and state in (capi.LIB_PAUSED, capi.LIB_STOPPED)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--titles", type=int, default=64)
    ap.add_argument("--packets", type=int, default=8)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    import espflix_b200
    from espflix_b200 import capi
    from tests import clock_cases, restart_cases

    if not torch.cuda.is_available():
        raise SystemExit("bench_keys.py: no CUDA device; the product has no CPU path")
    torch.cuda.set_device(args.device)
    n, T = args.streams, args.titles
    rng = np.random.default_rng(7)
    titles = []
    for t in range(T):
        y = np.clip(np.add.outer(np.arange(192) * rng.uniform(0.1, 0.6), np.arange(352) * rng.uniform(0.1, 0.4)) + 20 + t, 0, 235)
        pic = np.concatenate([y.astype(np.uint8).reshape(-1), np.full(2 * 96 * 176, 100 + t, np.uint8)])
        main = restart_cases.program(1000 + t, 4, 90000)
        titles.append((capi.build_video_idx(main, main, main, device=args.device), main, capi.encode_poster(pic, device=args.device)))
    most = max(args.packets, max(len(p) for _, _, p in titles) // 188)
    hdrs = np.stack([np.frombuffer(idx[:104], np.uint8) for idx, _, _ in titles])

    def context():
        ctx = espflix_b200.Context(n_streams=n, max_pictures=8, max_slices_per_picture=12, es_capacity=n * most * 188 + (1 << 20),
                                   fields=False, device=args.device)
        ctx.enable_pts()
        ctx.enable_carry(1 << 17)
        ctx.video_init(1)
        ctx.present_format(capi.EF_FIELD_DAC8)
        ctx.enable_present()
        ctx.present_overlay(np.zeros((n, 1280), np.uint8), np.full(n, 180, np.int32), np.zeros(n, np.int32))
        ctx.present_font(*clock_cases.font())
        for k, (idx, main, poster) in enumerate(titles):
            ctx.library_add(idx, main, main, main)
            ctx.library_add_poster(k, poster)
        for s in range(n):
            ctx.library_command(capi.LIB_NAV, s, 1, s % T, 0)
        ctx.present_clock(hdrs[np.arange(n) % T], 0, 1)
        return ctx

    arms = {"keys": context(), "commands": context()}
    w, nl = arms["keys"].geometry()
    out = torch.empty(n * 16 * w * nl, dtype=torch.uint8, device="cuda")
    info = torch.zeros((n, 8), dtype=torch.int32, device="cuda")
    choices = np.array([0, 0, 0, 99] + [capi.KEY_MENU, capi.KEY_PLAY, capi.KEY_SELECT, capi.KEY_RIGHT, capi.KEY_LEFT, capi.KEY_DOWN, capi.KEY_UP] * 2,
                       np.uint8)
    total = args.rounds * (args.warmup + args.steps)
    scripts = np.random.default_rng(4096).choice(choices, (total, n)).astype(np.uint8)

    def keys_arm(ctx, keys):
        ctx.library_keys(keys)

    def commands_arm(ctx, keys):
        st = ctx.library_info()
        ended = np.nonzero(st["state"] == capi.LIB_ENDED)[0]
        for s in ended:                                       # the DONE branch: back to the poster
            ctx.library_command(capi.LIB_MENU, int(s), 1, 0, 0)
        if len(ended):
            st = ctx.library_info()
        plan = [command_of(int(st["state"][s]), int(st["speed"][s]), int(keys[s]), capi) for s in range(n)]
        blend, setb, zero = np.zeros(n, np.int32), np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        blend[ended], setb[ended] = 0, 2
        s = 0
        while s < n:
            cmd, arg, b, z = plan[s]
            e = s + 1
            while e < n and plan[e][:2] == (cmd, arg):
                e += 1
            if cmd is not None:                               # a step outside the row leaves that stream alone
                ctx.library_command(cmd, s, e - s, 0, arg)
            s = e
        for s, (cmd, arg, b, z) in enumerate(plan):
            if b is not None and cmd is not None:
                blend[s], setb[s] = b, 2
            zero[s] = z
        ctx.present_overlay(blend=blend, set=setb)
        st = ctx.library_info()
        flags = (1 | 2 * (st["state"] == capi.LIB_PAUSED) | 4 * zero).astype(np.uint8)
        ctx.present_clock(hdrs[st["title"]], st["speed"].astype(np.int8), flags)

    def step(name, k):
        ctx = arms[name]
        (keys_arm if name == "keys" else commands_arm)(ctx, scripts[k])
        ctx.library_submit(args.packets)
        ctx.index()
        m = ctx.index_info()["max_pictures"]
        for p in range(m):
            ctx.present_picture_async(p, out, info)
        ctx.present_idle_async(2, out, info)
        assert ctx.present_wait() == (capi.EF_OK, m + 1)
        torch.cuda.synchronize()

    res = {"keys": [], "commands": []}
    k = {"keys": 0, "commands": 0}
    for r in range(args.rounds):
        for name in ("keys", "commands"):
            for _ in range(args.warmup):
                step(name, k[name])
                k[name] += 1
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step(name, k[name])
                k[name] += 1
            res[name].append((time.perf_counter() - t0) * 1e3 / args.steps)
    same = bool((arms["keys"].library_info() == arms["commands"].library_info()).all())
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"streams": n, "titles": T, "packets": args.packets, "card": card, "same_state": same,
                      "ms_per_step": {k: {"median": float(np.median(v)), "rounds": v} for k, v in res.items()}}))
    for ctx in arms.values():
        ctx.close()


if __name__ == "__main__":
    main()
