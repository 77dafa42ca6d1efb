"""ef_decode_audio_async: the context's audio decode into device memory, returning before the decode is done. Two contexts
get the same submits; one calls ef_decode_audio, the other the asynchronous call. info, PCM and PDM must be equal after every
call, on the reference fixtures, the synthetic batches, streams that end or restart, the benchmark-sized batch and beside
paced presentation; a call that does not fit must leave everything as it was."""
import os

import numpy as np
import pytest
import torch

import espflix_b200
from espflix_b200 import capi
from tests import audio_cases, restart_cases as rc
from tests.carry_cases import cut, packets
from tests.harness import audio_results, present_call, presenting_context, same_audio, submits

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SENTINEL = 0x5A5A


def decode_async(ctx, end=None, stream=0):
    """an asynchronous sizing call (one sample of room), then, when it did not fit, the call into buffers of exactly its size"""
    pcm = torch.full((1,), SENTINEL, dtype=torch.int16, device="cuda")
    pdm = torch.full((2,), SENTINEL, dtype=torch.int16, device="cuda").view(torch.uint16)
    info = ctx.decode_audio_async(pcm, pdm, end=end, stream=stream)
    if ctx.audio_wait() == capi.EF_ENOMEM:
        need = int(ctx.audio_info(info)["n_frames"].sum()) * 128
        pcm = torch.empty(need, dtype=torch.int16, device="cuda")
        pdm = torch.empty(2 * need, dtype=torch.int16, device="cuda").view(torch.uint16)
        info = ctx.decode_audio_async(pcm, pdm, end=end, stream=stream)
        assert ctx.audio_wait() == capi.EF_OK
    return audio_results(info, pcm, pdm)


def _pair(chunks, ends=None, queue_ahead=False, ops=None, mode="async", **kw):
    """chunks[k][s] through a synchronous and an asynchronous context side by side; ops[k]: restart ops after call k.
    mode "alternate": the second context calls ef_decode_audio_async on even submits and ef_decode_audio on odd ones."""
    n, K = len(chunks[0]), len(chunks)
    ends = ends if ends is not None else [[k == K - 1] * n for k in range(K)]
    kw = dict(dict(max_pictures=2, es_capacity=1 << 22, fields=False), **kw)
    ctxs = [espflix_b200.Context(n_streams=n, **kw) for _ in range(2)]
    for c in ctxs:
        c.enable_audio()
    packed = [ctxs[0].pack(c) for c in chunks]
    for c in ctxs:
        c.submit_ts(*packed[0])
    got = []
    for k in range(K):
        end = np.array(ends[k], dtype=np.uint8)
        res = []
        for i, c in enumerate(ctxs):
            c.index()
            if queue_ahead and k + 1 < K:
                c.submit_ts(*packed[k + 1])
            if i == 0 or (mode == "alternate" and k % 2):
                res.append(c.decode_audio(end=end))
            else:
                res.append(decode_async(c, end=end))
            if ops is not None and ops[k] is not None:
                c.restart_streams(ops[k])
            if not queue_ahead and k + 1 < K:
                c.submit_ts(*packed[k + 1])
        same_audio(res[0], res[1], "submit %d" % k)
        got.append(res[1])
    for c in ctxs:
        c.close()
    return got


def test_reference_fixtures_cut_at_video_pes_starts():
    ts = [open(os.path.join(G, n + ".ts"), "rb").read() for n in ("splash", "vmedia")]
    per_stream = []
    for i, t in enumerate(ts):
        pk = packets(t)
        starts = [k for k, q in enumerate(pk) if ((int(q[1]) << 8 | int(q[2])) & 0x1FFF) == 0x100 and q[1] & 0x40]
        per_stream.append(cut(t, starts[7 + 3 * i::9 + 2 * i]))
    got = _pair(submits(per_stream), max_pictures=13, max_slices_per_picture=8, es_capacity=1 << 21)
    whole = espflix_b200.audio_decode(espflix_b200.audio_demux_ts(ts))
    for s in range(2):
        assert np.array_equal(np.concatenate([g[s]["pcm"] for g in got]), whole[s]["pcm"])
        assert np.array_equal(np.concatenate([g[s]["pdm"] for g in got]).astype(np.uint16), whole[s]["pdm"])


@pytest.mark.parametrize("mode", ["async", "alternate"])
def test_cut_anywhere_batch_with_rejected_frames(mode):
    streams = audio_cases.synthetic_batch() + [audio_cases.overrun_stream(31), audio_cases.overrun_stream(32)]
    K = 7
    ts = [audio_cases.mux_audio_ts(es, pid=0x101 if i % 2 else 0x102, pes_bytes=[61, 188, 333, 1024, 2000][i % 5]) for i, es in enumerate(streams)]
    chunks = []
    for i, t in enumerate(ts):
        r = np.random.RandomState(1900 + i)
        chunks.append(cut(t, sorted(r.randint(0, t.size // 188 + 1, size=K - 1).tolist())))
    got = _pair(submits(chunks), mode=mode)
    whole = espflix_b200.audio_decode(streams)
    for s in range(len(streams)):
        assert np.array_equal(np.concatenate([g[s]["pcm"] for g in got]).astype(np.int16), whole[s]["pcm"]), s


@pytest.mark.parametrize("queue_ahead", [False, True])
def test_streams_ending_at_different_submits(queue_ahead):
    a = audio_cases.sbc_stream(11, 30, bitpool=31, consistent=False, bad_frames=(7,))
    b = audio_cases.sbc_stream(12, 25, bitpool=12, allocation=1, frequency=0)
    c = audio_cases.sbc_stream(13, 20, bitpool=60, loud=True)
    ta, tb, tc = (audio_cases.mux_audio_ts(x, pes_bytes=400) for x in (a, b, c))
    tb_tail = b"".join(packets(tb)[1:])
    pa, pb, pc = (cut(t, [len(t) // 188 // 3, 2 * len(t) // 188 // 3]) for t in (ta, tb_tail, tc))
    empty = np.zeros(0, dtype=np.uint8)
    chunks = [[pa[0], pc[0], b"".join(packets(tc)[:5])], [pa[1], empty, b"".join(packets(tc)[5:])], [pa[2], pc[1], empty],
              [pb[0], empty, empty], [pb[1], pc[2], empty], [pb[2], empty, empty]]
    ends = [[0, 0, 0], [0, 0, 1], [1, 0, 0], [0, 0, 0], [0, 0, 0], [1, 1, 1]]
    _pair(chunks, ends, queue_ahead=queue_ahead)


def test_restart_between_calls():
    dec = rc.decoder_cases()
    names = sorted(dec)
    K = max(len(p) for p in dec.values())
    progs = [dec[nm] + [b""] * (K - len(dec[nm])) for nm in names]
    chunks = [[np.frombuffer(p[k], dtype=np.uint8) for p in progs] for k in range(K)]
    ops = [np.array([1 if k + 1 < len(dec[nm]) else 0 for nm in names], dtype=np.uint8) if k + 1 < K else None for k in range(K)]
    _pair(chunks, ops=ops, max_pictures=12, es_capacity=len(names) * 12 * 40000)


def _two_contexts(n, chunk):
    ctxs = [espflix_b200.Context(n_streams=n, max_pictures=2, es_capacity=1 << 21, fields=False) for _ in range(2)]
    for c in ctxs:
        c.enable_audio()
        c.submit_ts(*c.pack(chunk))
        c.index()
    return ctxs


def _streams(n, frames=40):
    return [audio_cases.mux_audio_ts(audio_cases.sbc_stream(300 + s, frames + 3 * s, bitpool=[12, 31, 60][s % 3])) for s in range(n)]


def test_returns_before_the_decode_is_done():
    ts = _streams(4)
    ref, ctx = _two_contexts(4, ts)
    want = ref.decode_audio()
    need = sum(r["n_frames"] for r in want) * 128
    pcm = torch.empty(need, dtype=torch.int16, device="cuda")
    pdm = torch.empty(2 * need, dtype=torch.int16, device="cuda").view(torch.uint16)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(2_000_000_000)               # about a second of device time ahead of the call on its stream
    info = ctx.decode_audio_async(pcm, pdm, stream=side)
    assert not side.query()
    assert ctx.audio_wait() == capi.EF_OK
    same_audio(want, audio_results(info, pcm, pdm), "behind a busy stream")
    ref.close()
    ctx.close()


def test_overflow_changes_nothing_and_a_retry_fits():
    ts = _streams(3)
    halves = [cut(t, [t.size // 188 // 2]) for t in ts]
    ref, ctx = _two_contexts(3, [h[0] for h in halves])
    for c in (ref, ctx):
        c.submit_ts(*c.pack([h[1] for h in halves]))    # queued: the failed call must not touch its demux gate either
    end = np.array([1, 0, 1], dtype=np.uint8)
    want = ref.decode_audio(end=end)
    need = sum(r["n_frames"] for r in want) * 128
    pcm = torch.full((need - 1,), SENTINEL, dtype=torch.int16, device="cuda")
    pdm = torch.full((2 * (need - 1),), SENTINEL, dtype=torch.int16, device="cuda").view(torch.uint16)
    info = ctx.decode_audio_async(pcm, pdm, end=end)
    assert ctx.audio_wait() == capi.EF_ENOMEM
    rows = ctx.audio_info(info)
    assert [int(x) for x in rows["n_frames"]] == [r["n_frames"] for r in want]
    assert [int(x) for x in rows["frame_size"]] == [r["frame_size"] for r in want]
    assert bool((pcm == SENTINEL).all()) and bool((pdm.view(torch.int16) == SENTINEL).all())
    with pytest.raises(espflix_b200.EspflixError) as e:
        ctx.index()
    assert e.value.code == capi.EF_ESTATE
    same_audio(want, decode_async(ctx, end=end), "retry")
    for c in (ref, ctx):                                 # the calls after it: the state really was untouched
        c.index()
    same_audio(ref.decode_audio(end=True), decode_async(ctx, end=True), "after the retry")
    ref.close()
    ctx.close()


def test_runs_beside_paced_presentation():
    """audio on one stream, present_picture(0..11) on another: the fields equal a run without audio, the audio the sync path"""
    n, K = 4, 3
    progs = [[rc.program(700 + 10 * s + k, 12, 300000 + 36036 * k, audio=dict(seed=90 + 7 * s + k, frames=60, cut=0)) for k in range(K)] for s in range(n)]
    runs = []
    for audio in (False, True):
        ctx = presenting_context(n, 1, [0, 3, 1000, 7], max_pictures=12)
        ref = espflix_b200.Context(n_streams=n, max_pictures=12, es_capacity=n * 12 * 40000, fields=False)
        if audio:
            ctx.enable_audio()
            ref.enable_audio()
        ast, pst = torch.cuda.Stream(), torch.cuda.Stream()
        fields, sound = [], []
        for k in range(K):
            for c in (ctx, ref):
                c.submit_ts(*c.pack([np.frombuffer(p[k], dtype=np.uint8) for p in progs]))
                c.index()
            if audio:
                want = ref.decode_audio()
                need = sum(r["n_frames"] for r in want) * 128
                pcm = torch.empty(need, dtype=torch.int16, device="cuda")
                pdm = torch.empty(2 * need, dtype=torch.int16, device="cuda").view(torch.uint16)
                info = ctx.decode_audio_async(pcm, pdm, stream=ast)
            for p in range(12):
                fields.append(present_call(ctx, lambda out: ctx.present_picture(p, out=out, stream=pst.cuda_stream)))
            if audio:
                assert ctx.audio_wait() == capi.EF_OK
                same_audio(want, audio_results(info, pcm, pdm), "submit %d" % k)
                sound.append(want)
        runs.append(fields)
        ctx.close()
        ref.close()
    for (ia, fa), (ib, fb) in zip(*runs):
        assert (ia == ib).all() and np.array_equal(fa, fb)


def test_batch_scale():
    """the 4,096 streams of tests/scale_cases.py over three submits: more than one tile of the sizing scan, period 335"""
    from tests import scale_cases
    b = scale_cases.batch()
    assert scale_cases.period_is_coprime_to_tiles() and b.n > 1024
    first, second = [], []
    for k in range(b.n):
        first_k, second_k = cut(b.ts(k), [b.cut(k)[0]])
        first.append(first_k)
        second.append(second_k)
    empty = [np.zeros(0, dtype=np.uint8)] * b.n
    cap = sum(len(b.ts(k)) for k in range(b.n)) + (1 << 20)
    got = _pair([first, second, empty], ends=[[0] * b.n, [k % 3 == 0 for k in range(b.n)], [1] * b.n], max_pictures=12, es_capacity=cap)
    for k in range(b.n):                                 # replicas of one distinct stream carry the same audio
        d = b.distinct(k)
        assert np.array_equal(np.concatenate([g[k]["pcm"] for g in got]), np.concatenate([g[d]["pcm"] for g in got])), k


def test_errors():
    ctx = espflix_b200.Context(n_streams=2, max_pictures=2, es_capacity=1 << 20, fields=False)
    pcm = torch.empty(256, dtype=torch.int16, device="cuda")
    info = torch.zeros((2, 4), dtype=torch.int32, device="cuda")
    rc_ = ctx.lib.ef_decode_audio_async(ctx._h, None, info.data_ptr(), pcm.data_ptr(), 256, None, 0)
    assert rc_ == capi.EF_ESTATE
    ctx.enable_audio()
    ctx.submit_ts(*ctx.pack(_streams(2, 4)))
    ctx.index()
    assert ctx.lib.ef_decode_audio_async(ctx._h, None, info.data_ptr(), None, 256, None, 0) == capi.EF_EINVAL
    host = np.zeros(256, dtype=np.int16)
    pinned = torch.empty(256, dtype=torch.int16, pin_memory=True)
    for p in (host.ctypes.data, pinned.data_ptr()):
        assert ctx.lib.ef_decode_audio_async(ctx._h, None, info.data_ptr(), p, 256, None, 0) == capi.EF_EINVAL
    assert ctx.lib.ef_decode_audio_async(ctx._h, None, host.ctypes.data, pcm.data_ptr(), 256, None, 0) == capi.EF_EINVAL
    assert ctx.audio_wait() == capi.EF_OK                # nothing outstanding
    ctx.close()
