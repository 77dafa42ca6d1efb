"""The transport-stream parsers at the edges of the packet and PES header, on the GPU: every directed program of
tests/ts_edge_cases.py in one batch, among the 4,096 streams of the benchmark-sized filler batch, whole and cut at every packet
boundary on a carrying context, through the audio demux and the trick index, and played from the library. Inside the reference's domain the pictures, pts, audio and index equal what the unmodified reference
made (tests/golden/ts_edge_pins.json); outside it the ES and pts equal the device's rule restated (ts_edge_cases.device_demux)."""
import hashlib
import json
import os

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import pts_cases, ts_edge_cases as te
from tests.carry_cases import packets
from tests.harness import submits
from tests.oracle_lib import Oracle

pytestmark = pytest.mark.gpu
MAX_CARRY = 65536


@pytest.fixture(scope="module")
def pins():
    return json.load(open(os.path.join(pts_cases.GOLDEN, "ts_edge_pins.json")))


@pytest.fixture(scope="module")
def progs():
    return te.programs()


@pytest.fixture(scope="module")
def want(pins, progs):
    """per program: (sha256 of its frames, pts of every picture); outside the domain from the device's rule and the C oracle's
    decode of the ES that rule takes"""
    oracle = Oracle()
    out = {}
    for name, (ts, _) in progs.items():
        if name in pins:
            out[name] = (pins[name]["frames_sha256"], pins[name]["pts"])
        else:
            es, _ = te.device_demux(ts)
            f = oracle.decode_es(es, max_frames=512)
            out[name] = (hashlib.sha256(f.tobytes()).hexdigest(), te.device_picture_pts(ts))
            assert f.shape[0] == len(out[name][1]), name
    return out


def _sha(b):
    return hashlib.sha256(np.ascontiguousarray(b).tobytes()).hexdigest()


def _context(n, carry=False, audio=True, es_capacity=1 << 24):
    ctx = espflix_b200.Context(n_streams=n, max_pictures=110, max_slices_per_picture=12, es_capacity=es_capacity, fields=False)
    ctx.enable_pts()
    if carry:
        ctx.enable_carry(MAX_CARRY)
    if audio:
        ctx.enable_audio()
    return ctx


def _drive(ctx, chunks, carry=False, audio=True):
    """chunks[k][s]: the TS of stream s in submit k -> per stream: frames (as one hash), pts, PCM, PDM"""
    n = len(chunks[0])
    frames = [hashlib.sha256() for _ in range(n)]
    pts, pcm, pdm = [[] for _ in range(n)], [[] for _ in range(n)], [[] for _ in range(n)]
    for k, chunk in enumerate(chunks):
        ctx.submit_ts(*ctx.pack(chunk))
        if carry and k == len(chunks) - 1:
            ctx.end_streams(np.ones(n, np.uint8))
        ctx.index()
        ctx.index_info()
        counts = [ctx.stream_info(s)[0] for s in range(n)]
        for p in range(max(counts)):
            ctx.decode_picture(p)
            for s in range(n):
                if p < counts[s]:
                    frames[s].update(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1).tobytes())
        pic, _ = ctx.picture_pts()
        for s in range(n):
            pts[s] += [int(v) for v in pic[s, :counts[s]]]
        if audio:
            r = ctx.decode_audio(end=[k == len(chunks) - 1] * n)
            for s in range(n):
                pcm[s].append(r[s]["pcm"])
                pdm[s].append(r[s]["pdm"])
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int16)
    return [f.hexdigest() for f in frames], pts, [cat(x) for x in pcm], [cat(x) for x in pdm]


def _check(names, got, pins, want, audio=True):
    frames, pts, pcm, pdm = got
    for s, name in enumerate(names):
        assert pts[s] == want[name][1], name
        assert frames[s] == want[name][0], name
        if audio and name in pins:
            assert pcm[s].size == pins[name]["pcm_samples"] and _sha(pcm[s]) == pins[name]["pcm_sha256"], name
            assert _sha(pdm[s]) == pins[name]["pdm_sha256"], name


def test_every_program_in_one_batch(pins, progs, want):
    """every program whole, in one batch, and again as four copies of the batch: pictures, pts, decode_audio, and
    decode_audio_async on the same submit"""
    import torch
    names = list(progs)
    ctx = _context(len(names))
    _check(names, _drive(ctx, [[progs[n][0] for n in names]]), pins, want)
    ctx.close()

    big = names * 4
    blob, off = espflix_b200.Context.pack([progs[n][0] for n in big])
    ctx = _context(len(big), es_capacity=int(off[-1]) + 4096)
    ctx.submit_ts(blob, off)
    ctx.index()
    ctx.index_info()
    pic, _ = ctx.picture_pts()
    for s, name in enumerate(big):
        n = ctx.stream_info(s)[0]
        assert [int(v) for v in pic[s, :n]] == want[name][1], (s, name)
    cap = sum(2 * len(te.device_audio_demux(progs[n][0])) + 256 for n in big)       # 128 samples per frame of at least 64 bytes
    pcm_t = torch.zeros(cap, dtype=torch.int16, device="cuda")
    pdm_t = torch.zeros(2 * cap, dtype=torch.uint16, device="cuda")
    info = ctx.decode_audio_async(pcm_t, pdm_t, end=True)
    assert ctx.audio_wait() == capi.EF_OK
    rows = ctx.audio_info(info)
    host_pcm = pcm_t.cpu().numpy()
    host_pdm = pdm_t.view(torch.int16).cpu().numpy().view(np.uint16)
    for s, name in enumerate(big):
        if name not in pins:
            continue
        a, k = int(rows[s]["pcm_offset"]), int(rows[s]["n_frames"]) * 128
        assert k == pins[name]["pcm_samples"] and _sha(host_pcm[a:a + k]) == pins[name]["pcm_sha256"], (s, name)
        assert _sha(host_pdm[2 * a:2 * (a + k)]) == pins[name]["pdm_sha256"], (s, name)
    ctx.close()


def test_cut_at_every_packet_with_carry(pins, progs, want):
    """every program cut before every packet (one packet per submit) on a carrying context: the submits' pictures, pts and audio
    concatenated equal the whole program's"""
    names = list(progs)
    per_stream = [packets(progs[n][0]) for n in names]
    ctx = _context(len(names), carry=True)
    _check(names, _drive(ctx, submits(per_stream), carry=True), pins, want)
    ctx.close()


def test_audio_demux_of_every_program(progs):
    """ef_audio_demux_ts: the bytes push_audio() receives, as the device's rule restated (inside the domain the reference's)"""
    names = list(progs)
    got = espflix_b200.audio_demux_ts([progs[n][0] for n in names])
    for name, g in zip(names, got):
        assert g.tobytes() == te.device_audio_demux(progs[name][0]), name


def test_among_benchmark_sized_filler(pins, progs, want):
    """the directed programs at tile edges of a 4,096-stream batch (the benchmark's stream count) whose other streams are the
    batch-scale filler (tests/scale_cases.py): their pictures, pts and audio as pinned, and every filler stream's pts"""
    from tests import scale_cases
    batch = scale_cases.batch()
    N = scale_cases.N
    names = list(progs)
    at = dict(zip([0, 1023, 1024, 1025, 2047, 2048, 3071, 3072, 3073, 4094, 4095][:len(names)], names))
    assert len(at) == len(names)
    streams = [progs[at[s]][0] if s in at else batch.ts(s) for s in range(N)]
    blob, off = espflix_b200.Context.pack(streams)
    ctx = espflix_b200.Context(n_streams=N, max_pictures=110, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096, fields=False)
    ctx.enable_pts()
    ctx.enable_audio()
    ctx.submit_ts(blob, off)
    ctx.index()
    ctx.index_info()
    counts = [ctx.stream_info(s)[0] for s in range(N)]
    pic, _ = ctx.picture_pts()
    for s in range(N):
        w = want[at[s]][1] if s in at else batch.pts[s % scale_cases.D]
        assert [int(v) for v in pic[s, :counts[s]]] == w, (s, at.get(s))
    frames = {s: hashlib.sha256() for s in at}
    for p in range(max(counts)):
        ctx.decode_picture(p)
        for s in at:
            if p < counts[s]:
                frames[s].update(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1).tobytes())
    for s, name in at.items():
        assert frames[s].hexdigest() == want[name][0], (s, name)
    r = ctx.decode_audio(end=True)
    for s, name in at.items():
        if name in pins:
            assert r[s]["pcm"].size == pins[name]["pcm_samples"] and _sha(r[s]["pcm"]) == pins[name]["pcm_sha256"], (s, name)
            assert _sha(r[s]["pdm"]) == pins[name]["pdm_sha256"], (s, name)
    ctx.close()


def test_trick_index_of_the_main_titles(pins, progs):
    names = [n for n, (_, roles) in progs.items() if "main" in roles]
    got = espflix_b200.tsidx_scan([progs[n][0] for n in names])
    for name, g in zip(names, got):
        p = pins[name]
        assert [int(v) for v in g["seq_pts"]] == p["seq_pts"] and [int(v) for v in g["seq_pos"]] == p["seq_pos"], name
        assert (g["first_pts"], g["last_pts"]) == (p["first_pts"], p["last_pts"]), name
        ts = progs[name][0]
        idx = espflix_b200.build_video_idx(ts, ts, ts)
        assert len(idx) == p["video_idx_bytes"] and hashlib.sha256(idx).hexdigest() == p["video_idx_sha256"], name


def test_library_plays_the_main_titles(pins, progs, want):
    """each main title added with its video.idx and played from PLAY_AT 0 to its end in seeded budgets: every picture and pts"""
    names = [n for n, (_, roles) in progs.items() if "main" in roles]
    for j, name in enumerate(names):
        ts = progs[name][0]
        ctx = _context(1, carry=True, audio=False)
        t = ctx.library_add(espflix_b200.build_video_idx(ts, ts, ts), ts)
        ctx.library_command(capi.LIB_PLAY_AT, 0, 1, t, 0)
        rng = np.random.default_rng(50 + j)
        frames, pts = hashlib.sha256(), []
        while ctx.library_info()[0]["state"] == capi.LIB_PLAYING:
            ctx.library_submit(int(rng.integers(1, 300)))
            ctx.index()
            n = ctx.stream_info(0)[0]
            for p in range(n):
                ctx.decode_picture(p)
                frames.update(ctx.read_frame_i420(0, (ctx.stream_info(0)[1] + p + 1) & 1).tobytes())
            pts += [int(v) for v in ctx.picture_pts()[0][0, :n]]
        assert ctx.library_info()[0]["state"] == capi.LIB_ENDED
        ctx.close()
        assert pts == want[name][1], name
        assert frames.hexdigest() == want[name][0], name
