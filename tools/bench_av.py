#!/usr/bin/env python3
"""tools/bench_av.py — paced presentation and audio of the same submits, one after the other or side by side.

Workload: tools/bench_audio.py's (bench.py's config 4, 4,096 streams x one GOP of 12 pictures, 64 distinct seeds replicated,
each stream's TS followed by 150 SBC frames of 64 B on PID 0x102) on a presenting context (PTS, audio, present), NTSC and
PAL, one context each. Every step is a new clip per stream, so it starts with ef_reset as in tools/bench_present.py, then
ef_submit_ts_host -> ef_index, and then one of three arms, alternated step by step in one run:

  serial     ef_present_picture(0..11), then ef_decode_audio with PCM and PDM to pinned host memory
  async      ef_decode_audio_async on a second non-blocking stream, then ef_present_picture(0..11), then ef_audio_wait
  async_d2h  as async, plus PCM and PDM copied to pinned host memory on the audio stream

Reported per standard: ms per step of each arm (host clock; every arm ends in a wait), the host time of the
ef_decode_audio_async call itself, the device time per step of the audio and presentation kernels (torch.profiler, two
untimed async steps in a run of their own), and the card's name and power limit read in the same command. After the timed
steps an extra async step is checked against the restatement: the fields and the PCM and PDM of --verify streams. Writes
nothing into the tree.

  python tools/bench_av.py [--streams 4096] [--steps 6] [--warmup 1] [--verify 2]
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

AUDIO_FRAMES = 150
ARMS = ("serial", "async", "async_d2h")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=6, help="timed steps per arm")
    ap.add_argument("--warmup", type=int, default=1, help="untimed steps per arm")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--verify", type=int, default=2, help="streams of the extra step checked against the restatement (0: none)")
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import capi, synth
    from tests import audio_cases

    if not torch.cuda.is_available():
        raise SystemExit("bench_av.py: no CUDA device; the product has no CPU path")
    torch.cuda.set_device(args.device)
    streams, P = args.streams, bench.PICTURES
    gen, _ = bench.make_streams(streams)
    d = len(gen)
    audio_es = [audio_cases.sbc_stream(7000 + i, AUDIO_FRAMES, bitpool=28) for i in range(d)]
    tsa = [np.concatenate([synth.wrap_ts(*gen[i]), audio_cases.mux_audio_ts(audio_es[i], pid=0x102)]) for i in range(d)]
    off = np.zeros(streams + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(tsa[i % d]) for i in range(streams)])
    pinned_ts = torch.empty(int(off[-1]), dtype=torch.uint8, pin_memory=True)
    view = pinned_ts.numpy()
    for i in range(streams):
        view[int(off[i]):int(off[i + 1])] = tsa[i % d]
    n_pcm = streams * AUDIO_FRAMES * 128
    pinned_pcm = torch.empty(n_pcm, dtype=torch.int16, pin_memory=True)
    pinned_pdm = torch.empty(2 * n_pcm, dtype=torch.int16, pin_memory=True)        # uint16 words
    dev_pcm = torch.empty(n_pcm, dtype=torch.int16, device="cuda")
    dev_pdm = torch.empty(2 * n_pcm, dtype=torch.int16, device="cuda")
    dev_info = torch.zeros((streams, 4), dtype=torch.int32, device="cuda")
    info = np.zeros(streams, dtype=capi._AUDIO_INFO)
    astream = torch.cuda.Stream()                         # non-blocking (torch's pool streams are)
    st = 0
    results = {}
    for ntsc in (1, 0):
        ctx = espflix_b200.Context(n_streams=streams, max_pictures=P, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096,
                                   device=args.device, fields=False)
        ctx.enable_pts()
        ctx.video_init(ntsc)
        ctx.enable_present(1)
        ctx.enable_audio()
        w, nl = ctx.geometry()
        out = torch.empty(3 * streams * w * nl, dtype=torch.uint16, device="cuda")
        call_ms, keep = [], {}

        def present(keep_fields=False):
            for p in range(P):
                pi = ctx.present_picture(p, None, out, st)
                if keep_fields:
                    for s in range(args.verify):
                        a, k = int(pi[s]["first"]), int(pi[s]["n_fields"])
                        keep.setdefault(s, []).append(out[a * w * nl:(a + k) * w * nl].view(torch.int16).cpu().numpy().view(np.uint16).reshape(k, w * nl))

        def step(arm, keep_fields=False):
            ctx.reset()
            ctx.submit_ts(pinned_ts.data_ptr(), off, st, device=False)
            ctx.index(st)
            if arm == "serial":
                present(keep_fields)
                ctx._check(ctx.lib.ef_decode_audio(ctx._h, None, info.ctypes.data, pinned_pcm.data_ptr(), n_pcm, pinned_pdm.data_ptr(), astream.cuda_stream))
                return
            t0 = time.perf_counter()
            ctx.decode_audio_async(dev_pcm, dev_pdm.view(torch.uint16), info=dev_info, stream=astream)
            call_ms.append(1000.0 * (time.perf_counter() - t0))
            if arm == "async_d2h":
                with torch.cuda.stream(astream):
                    pinned_pcm.copy_(dev_pcm, non_blocking=True)
                    pinned_pdm.copy_(dev_pdm, non_blocking=True)
            present(keep_fields)
            if ctx.audio_wait() != capi.EF_OK:
                raise SystemExit("bench_av.py: the async call did not fit")
            if arm == "async_d2h":
                astream.synchronize()

        n_done = 0
        for _ in range(args.warmup):
            for arm in ARMS:
                step(arm)
                n_done += 1
        call_ms.clear()
        ms = {a: [] for a in ARMS}
        torch.cuda.synchronize()
        for _ in range(args.steps):
            for arm in ARMS:
                t0 = time.perf_counter()
                step(arm)
                torch.cuda.synchronize()
                ms[arm].append(1000.0 * (time.perf_counter() - t0))
                n_done += 1
        res = {a: {"ms_per_step": round(float(np.mean(v)), 2), "min": round(float(np.min(v)), 2), "max": round(float(np.max(v)), 2)} for a, v in ms.items()}
        res["async_call_host_ms"] = {"mean": round(float(np.mean(call_ms)), 3), "max": round(float(np.max(call_ms)), 3)}
        res["async_gain_ms"] = round(res["serial"]["ms_per_step"] - res["async"]["ms_per_step"], 2)

        from torch.profiler import ProfilerActivity, profile   # device time per kernel, two untimed async steps
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(2):
                step("async")
                n_done += 1
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            name = e.key.split("(")[0].split("<")[0].replace("void ", "")
            if any(t in name for t in ("sbc_", "pdm", "audio", "pace", "composite", "parse", "recon")):
                kern[name] = kern.get(name, 0.0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0 / 2
        res["kernel_ms_per_step"] = {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
        audio_k = [k for k in kern if any(t in k for t in ("sbc_", "pdm", "audio"))]
        res["audio_kernel_ms_per_step"] = round(sum(kern[k] for k in audio_k), 3)

        if args.verify:                                    # the extra step against the restatement
            from tests import present_cases as pc
            from tests.oracle_lib import Oracle
            o = Oracle()
            disp = [pc.Display(ntsc, 1) for _ in range(args.verify)]
            pts = 129003 + 3003 * np.arange(P)
            for _ in range(n_done):
                for dsp in disp:
                    dsp.reset()
                    for p in pts:
                        dsp.push(int(p))
            for dsp in disp:
                dsp.reset()
            step("async_d2h", keep_fields=True)
            rows = ctx.audio_info(dev_info)
            got_pcm, got_pdm = pinned_pcm.numpy(), pinned_pdm.numpy().view(np.uint16)
            for s in range(args.verify):
                frames = o.decode_ts(tsa[s % d])
                r = pc.Renderer(o, ntsc)
                got = np.concatenate(keep[s]) if keep[s] else np.zeros((0, w * nl), np.uint16)
                want = []
                for k, p in enumerate(pts):
                    r.decoded(k, frames[k])
                    want += [r.field(f) for f in disp[s].push(int(p))[0]]
                if len(want) != got.shape[0] or any(not np.array_equal(a, b) for a, b in zip(want, got)):
                    raise SystemExit("bench_av.py: stream %d: fields differ from the restatement" % s)
                pcm = o.sbc_decode(audio_es[s % d])
                a = int(rows[s]["pcm_offset"])
                if int(rows[s]["n_frames"]) != AUDIO_FRAMES or not (np.array_equal(got_pcm[a:a + pcm.size], pcm)
                                                                   and np.array_equal(got_pdm[2 * a:2 * a + 2 * pcm.size], o.pdm(pcm))):
                    raise SystemExit("bench_av.py: stream %d: audio differs from the restatement" % s)
            res["verify"] = "ok: fields, PCM and PDM of %d streams of an extra async step equal the restatement" % args.verify
        results["ntsc" if ntsc else "pal"] = res
        del out
        ctx.close()
        torch.cuda.empty_cache()
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d TS streams x (12 pictures + %d SBC frames of 64 B) per step, ef_reset between steps, %d distinct seeds replicated"
                    % (streams, AUDIO_FRAMES, d),
        "steps_per_arm": args.steps, "warmup_per_arm": args.warmup, "card": card, "standards": results}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
