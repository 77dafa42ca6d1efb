#!/usr/bin/env python3
"""tools/bench_audio.py — the audio of a transport-stream program at batch scale, through the decoder context.

Workload: bench.py's config 4 (4,096 streams x one GOP of 12 pictures, 64 distinct seeds replicated), each stream's TS
followed by the sound of its 12 pictures (12 at 29.97 Hz = 0.4 s): 150 SBC frames of 128 samples, 64 B each (bitpool
28), muxed on PID 0x102 by tests/audio_cases.py. Two legs over the same pinned input, one JSON line:

  e2e_ts        per step: ef_submit_ts_host -> ef_index -> ef_decode_all(12) -> ef_read_latest_i420_async; audio not enabled
  e2e_ts_audio  the same step on a context with ef_audio_enable, plus ef_decode_audio with PCM and PDM of every stream to
                pinned host memory, on a CUDA stream of its own beside the video kernels

Reported: ms per step of both legs, the events around the synchronous ef_decode_audio, the device time of every audio
kernel (torch.profiler, two untimed steps), audio frames/s, the bytes copied back, and the card's name and power limit.
After the timed steps the last step's PCM and PDM of the first distinct streams are checked against the restatement on
all the audio fed so far (--no-verify skips it). Writes nothing into the tree.

  python tools/bench_audio.py [--streams 4096] [--steps 10] [--warmup 2] [--no-verify]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--no-verify", action="store_true")
    args = ap.parse_args()

    import torch
    import bench
    import espflix_b200
    from espflix_b200 import synth
    from tests import audio_cases

    if not torch.cuda.is_available():
        raise SystemExit("bench_audio.py: no CUDA device; the product has no CPU path")
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
    pinned_out = [torch.empty((streams, bench.FRAME_BYTES), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    n_pcm = streams * AUDIO_FRAMES * 128
    pinned_pcm = torch.empty(n_pcm, dtype=torch.int16, pin_memory=True)
    pinned_pdm = torch.empty(2 * n_pcm, dtype=torch.int16, pin_memory=True)         # uint16 words
    info = np.zeros(streams, dtype=espflix_b200.capi._AUDIO_INFO)
    astream = torch.cuda.Stream()
    st = 0

    def run_leg(audio):
        ctx = espflix_b200.Context(n_streams=streams, max_pictures=P, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096,
                                   device=args.device, fields=False)
        if audio:
            ctx.enable_audio()
        calls = []

        def step(k, events=None):
            ctx.submit_ts(pinned_ts.data_ptr(), off, st, device=False)
            ctx.index(st)
            ctx.decode_all(P, st)
            ctx.read_latest_i420_async(0, streams, pinned_out[k & 1].data_ptr(), st)
            if audio:
                if events is not None:
                    events[0].record(astream)
                ctx._check(ctx.lib.ef_decode_audio(ctx._h, None, info.ctypes.data, pinned_pcm.data_ptr(), n_pcm, pinned_pdm.data_ptr(), astream.cuda_stream))
                if events is not None:
                    events[1].record(astream)
                    calls.append(events)

        for k in range(args.warmup):
            step(k)
        ctx.sync(st)
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in range(args.steps)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        w0 = time.perf_counter()
        for k in range(args.steps):
            step(k, ev[k])
        e1.record()
        ctx.sync(st)
        torch.cuda.synchronize()
        ms = max(e0.elapsed_time(e1), 1000.0 * (time.perf_counter() - w0)) / args.steps
        res = {"ms_per_step": ms, "video_frames_per_s": streams * P / (ms / 1000.0)}
        if not audio:
            ctx.close()
            return res
        res["audio_call_ms_per_step"] = float(np.mean([a.elapsed_time(b) for a, b in calls]))
        res["audio_frames_per_s"] = streams * AUDIO_FRAMES / (ms / 1000.0)
        if not bool((info["n_frames"] == AUDIO_FRAMES).all()):
            raise SystemExit("bench_audio.py: a stream did not decode %d frames in the last step" % AUDIO_FRAMES)
        if not args.no_verify:
            from tests.oracle_lib import Oracle
            oracle = Oracle()
            fed = args.warmup + args.steps
            got_pcm, got_pdm = pinned_pcm.numpy(), pinned_pdm.numpy().view(np.uint16)
            for i in range(min(2, d)):
                whole = oracle.sbc_decode(np.tile(audio_es[i], fed))
                want, want_pdm = whole[-AUDIO_FRAMES * 128:], oracle.pdm(whole)[-2 * AUDIO_FRAMES * 128:]
                a = int(info[i]["pcm_offset"])
                if not (np.array_equal(got_pcm[a:a + want.size], want) and np.array_equal(got_pdm[2 * a:2 * a + want_pdm.size], want_pdm)):
                    raise SystemExit("bench_audio.py: stream %d: the last step's audio differs from the restatement" % i)
            res["verify"] = "ok: the last step's PCM and PDM of %d distinct streams equal the restatement on all %d steps of audio fed" % (min(2, d), fed)
        from torch.profiler import ProfilerActivity, profile       # device time per kernel, two untimed steps
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(2):
                step(k)
            ctx.sync(st)
        kern = {}
        for e in prof.key_averages():
            if any(t in e.key for t in ("sbc_", "pdm", "audio")):
                kern[e.key.split("(")[0]] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0 / 2, 4)
        res["audio_kernel_ms_per_step"] = kern
        res["audio_kernel_ms_total"] = round(sum(kern.values()), 4)
        ctx.close()
        return res

    video = run_leg(False)
    audio = run_leg(True)
    card = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "workload": "%d streams x (12 pictures + %d SBC frames of 64 B on PID 0x102), %d distinct seeds replicated" % (streams, AUDIO_FRAMES, d),
        "steps": args.steps, "warmup": args.warmup, "card": card,
        "e2e_ts": video, "e2e_ts_audio": audio,
        "h2d_bytes_per_step": int(off[-1]),
        "d2h_bytes_per_step": {"pictures": streams * bench.FRAME_BYTES, "pcm": n_pcm * 2, "pdm": n_pcm * 4},
    }), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
