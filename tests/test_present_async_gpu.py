"""ef_present_picture_async / ef_present_idle_async / ef_present_wait: paced presentation enqueued without waiting for the device.
A synchronous context and an asynchronous one get the same submits and the same present calls; the fields and info[] of every
call must be equal, on the pinned reference cases (whose field streams must still hash to the pins), the irregular programs
whole and cut, with sync and async calls alternating, behind a busy stream, through a call that does not fit and its retry,
around the calls that resolve a chain, beside the asynchronous audio decode, and at the benchmark's batch size."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import espflix_b200
from espflix_b200 import capi
from tests import carry_cases, present_cases as pc, pts_cases, scale_cases
from tests.harness import audio_results, error_code, host_fields, present_call, presenting_context, same_audio, submits

pytestmark = pytest.mark.gpu
PINS = json.load(open(os.path.join(pts_cases.GOLDEN, "pacing_pins.json")))
SENTINEL = 0x5A5A
INFO_FIELDS = ("first", "n_fields", "frame_counter", "flip_field", "flip_line", "flags")


# ---- one program through a synchronous and an asynchronous context -------------------------------------------------------
def build(ctx, submits, mode_of=None, idle_after=None):
    """runs `submits` (lists of per-stream TS chunks) synchronously on ctx -> (steps, records). A step is ("submit", chunk),
    ("pic", p, modes) or ("idle", n_fields); idle_after(k) -> n_fields after submit k (None: no idle run)."""
    n = ctx.n_streams
    steps, recs, seen = [], {}, [0] * n
    for k, chunk in enumerate(submits):
        steps.append(("submit", chunk))
        ctx.submit_ts(*ctx.pack(chunk))
        ctx.index()
        npics = ctx.index_info()["max_pictures"]
        counts = [ctx.stream_info(s)[0] for s in range(n)]
        for p in range(npics):
            modes = np.array([mode_of(s, seen[s] + p) if mode_of and p < counts[s] else 0 for s in range(n)], dtype=np.uint8)
            steps.append(("pic", p, modes))
            recs[len(steps) - 1] = present_call(ctx, lambda o: ctx.present_picture(p, modes, o))
        seen = [a + b for a, b in zip(seen, counts)]
        nf = idle_after(k) if idle_after else None
        if nf is not None:
            nf = np.ascontiguousarray(np.broadcast_to(nf, (n,)), dtype=np.uint32)
            steps.append(("idle", nf))
            recs[len(steps) - 1] = present_call(ctx, lambda o: ctx.present_idle(nf, o))
    return steps, recs


def totals(recs):
    return {i: int(info["n_fields"].sum()) for i, (info, _) in recs.items()}


def replay(ctx, steps, how=lambda i: "async", caps=None, stream=0, between=None):
    """the steps on ctx: a present step synchronously or asynchronously as how(i) says, the async ones into their own
    sentinel-filled buffer of caps[i] fields, one ef_present_wait at the end -> (records, rc, n_presented, buffers).
    between(i, ctx): called before step i."""
    w, nl = ctx.geometry()
    recs, pend, bufs = {}, [], {}
    for i, st in enumerate(steps):
        if how(i) == "skip":
            continue
        if between:
            between(i, ctx)
        if st[0] == "submit":
            ctx.submit_ts(*ctx.pack(st[1]))
            ctx.index()
        elif how(i) == "sync":
            if st[0] == "pic":
                recs[i] = present_call(ctx, lambda o: ctx.present_picture(st[1], st[2], o))
            else:
                recs[i] = present_call(ctx, lambda o: ctx.present_idle(st[1], o))
        else:
            out = torch.full((max(caps[i] * w * nl, 8),), SENTINEL, dtype=torch.int16, device="cuda").view(torch.uint16)
            if st[0] == "pic":
                info = ctx.present_picture_async(st[1], out, modes=st[2], stream=stream)
            else:
                info = ctx.present_idle_async(st[1], out, stream=stream)
            pend.append((i, out, info))
            bufs[i] = out
    rc, k = ctx.present_wait()
    for i, out, info in pend:
        inf = ctx.present_info(info)
        total = min(int(inf["n_fields"].sum()), out.numel() // (w * nl))     # a call that did not fit reports more
        recs[i] = (inf, host_fields(out[:total * w * nl].view(total, w * nl)))
    return recs, rc, k, bufs


def same(a, b, keys=None, what=""):
    for i in (sorted(a) if keys is None else keys):
        (ia, ha), (ib, hb) = a[i], b[i]
        for f in INFO_FIELDS:
            assert np.array_equal(ia[f], ib[f]), "%s step %d: info %s" % (what, i, f)
        assert ha.shape == hb.shape and np.array_equal(ha, hb), "%s step %d: fields" % (what, i)


def stream_hashes(recs, n):
    h = [hashlib.sha256() for _ in range(n)]
    for i in sorted(recs):
        info, host = recs[i]
        for s in range(n):
            a, k = int(info[s]["first"]), int(info[s]["n_fields"])
            for j in range(k):
                h[s].update(host[a + j].tobytes())
    return [x.hexdigest() for x in h]


def _pair_contexts(n, ntsc, fc0, **kw):
    return presenting_context(n, ntsc, fc0=fc0, **kw), presenting_context(n, ntsc, fc0=fc0, **kw)


# ---- the pinned cases as one chain -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ntsc", [1, 0])
def test_pinned_cases_as_one_chain(ntsc):
    names = [n for n in sorted(PINS) if PINS[n]["ntsc"] == ntsc]
    ts = [pc.synth_ts(PINS[n]["seed"], PINS[n]["pictures"]) for n in names] + [pc.synth_ts(60 + ntsc, 7), pc.synth_ts(62 + ntsc, 12)]
    fc0 = [PINS[n]["frame_counter0"] for n in names] + [3, 100]
    modes = {i: PINS[n]["modes"] for i, n in enumerate(names)}
    ref, ctx = _pair_contexts(len(ts), ntsc, fc0)
    chunk = [np.frombuffer(bytes(t), dtype=np.uint8) for t in ts]
    mode_of = lambda s, g: modes[s][g] if s in modes else (2 if g == 4 else 0)      # noqa: E731
    steps, want = build(ref, [chunk], mode_of)
    # the tail as in test_pinned_streams_hash_to_the_reference: up to the pinned field count
    emitted = [sum(int(want[i][0][s]["n_fields"]) for i in want) for s in range(len(ts))]
    tails = [((PINS[n]["flip_field"][-1] + 1 + PINS[n]["tail_fields"] - PINS[n]["frame_counter0"]) & 0xFFFFFFFF) - emitted[i] for i, n in enumerate(names)]
    nf = np.array(tails + [5, 0], dtype=np.uint32)
    steps.append(("idle", nf))
    want[len(steps) - 1] = present_call(ref, lambda o: ref.present_idle(nf, o))
    got, rc, k, _ = replay(ctx, steps, caps=totals(want))
    assert rc == capi.EF_OK and k == len(steps) - 1
    same(got, want, what="pinned")
    hashes = stream_hashes(got, len(ts))
    for i, n in enumerate(names):
        assert hashes[i] == PINS[n]["stream_sha256"], n
    a, b = ref.picture_pts(), ctx.picture_pts()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    ref.close()
    ctx.close()


# ---- irregular programs, whole and cut, sync and async alternating -----------------------------------------------------------
@pytest.fixture(scope="module")
def irregular():
    return pc.irregular_programs()


def _chunks(progs, cuts_seed):
    if cuts_seed is None:
        return [[np.frombuffer(bytes(p[1]), dtype=np.uint8) for p in progs]]
    rng = np.random.RandomState(cuts_seed)
    K = int(rng.randint(2, 5))
    per = []
    for p in progs:
        cand = pts_cases.cut_points(p[1])
        per.append(carry_cases.cut(p[1], sorted(rng.choice(cand, size=K - 1, replace=True).tolist()) if cand else []))
    return submits(per, n=K)


@pytest.mark.parametrize("ntsc", [1, 0])
@pytest.mark.parametrize("cuts_seed", [None, 11])
def test_irregular_programs_mixed(irregular, ntsc, cuts_seed):
    progs = [p for p in irregular if p[3] == ntsc]
    fc0 = [p[4] for p in progs]
    chunks = _chunks(progs, cuts_seed)
    rng = np.random.RandomState(5 + ntsc)
    idles = [rng.randint(0, 3, size=len(progs)) for _ in chunks[:-1]] + [np.array([p[6] + 1 for p in progs])]
    mode_of = lambda s, g: progs[s][5][g]                                           # noqa: E731
    ref = presenting_context(len(progs), ntsc, fc0=fc0)
    steps, want = build(ref, chunks, mode_of, lambda k: idles[k])
    ref.close()
    caps = totals(want)
    for how in (lambda i: "async", lambda i: "async" if (i // 2) % 2 == 0 else "sync", lambda i: "sync" if i % 3 == 0 else "async"):
        ctx = presenting_context(len(progs), ntsc, fc0=fc0)
        got, rc, _, _ = replay(ctx, steps, how, caps)
        assert rc == capi.EF_OK
        same(got, want, what="irregular")
        ctx.close()


# ---- behind a busy stream --------------------------------------------------------------------------------------------------
def test_call_behind_a_busy_stream_returns_before_it_runs():
    ts = [pc.synth_ts(70 + i, n) for i, n in enumerate((5, 3))]
    chunk = [np.frombuffer(bytes(t), dtype=np.uint8) for t in ts]
    ref, ctx = _pair_contexts(2, 1, [1, 2])
    steps, want = build(ref, [chunk])
    cap = max(totals(want).values()) + 2
    caps = {i: cap for i in want}
    side = torch.cuda.Stream()
    w, nl = ctx.geometry()

    def busy(i, c):
        if i == 2:                                      # picture 0 is in (it grew the descriptor arrays), picture 1 is next
            assert c.present_wait() == (capi.EF_OK, 1)
            torch.cuda.synchronize()
            with torch.cuda.stream(side):
                torch.cuda._sleep(2_000_000_000)        # about a second of device time ahead of the call on its stream
    calls = []
    orig = ctx.present_picture_async

    def watched(*a, **kw):
        info = orig(*a, **kw)
        calls.append(side.query())
        return info
    ctx.present_picture_async = watched
    got, rc, _, _ = replay(ctx, steps, caps=caps, stream=side, between=busy)
    assert rc == capi.EF_OK and calls[1] is False
    same(got, want, what="busy")
    ref.close()
    ctx.close()


# ---- a call that does not fit, and its retry ----------------------------------------------------------------------------------
@pytest.mark.parametrize("j", [3, 4])                  # rec_pics 3: picture 3 starts a K1a range, picture 4 is inside one
def test_short_call_and_retry(j, monkeypatch):
    monkeypatch.setenv("EF_REC_PICS", "3")
    ts = [pc.synth_ts(120 + i, n) for i, n in enumerate((7, 6, 7))]
    chunk = [np.frombuffer(bytes(t), dtype=np.uint8) for t in ts]
    ref, ctx = _pair_contexts(3, 0, [5, 6, 7], max_pictures=8)
    steps, want = build(ref, [chunk], lambda s, g: 3 if (s, g) == (1, 2) else 0, lambda k: [2, 3, 4])
    caps = totals(want)
    bad = j + 1                                         # step 0 is the submit: picture p is step p + 1
    assert caps[bad] > 0
    short = dict(caps)
    short[bad] -= 1
    got, rc, k, bufs = replay(ctx, steps, caps=short)
    assert rc == capi.EF_ENOMEM and k == j
    same(got, want, keys=range(1, bad), what="before the short call")
    info = got[bad][0]
    assert np.array_equal(info["n_fields"], want[bad][0]["n_fields"]) and np.array_equal(info["first"], want[bad][0]["first"])
    assert (info["flags"] & 2).all()
    for i in range(bad + 1, len(steps)):
        assert (got[i][0]["flags"] & 2).all() and (got[i][0]["n_fields"] == 0).all()
    for i in range(bad, len(steps)):
        assert bool((bufs[i].view(torch.int16) == SENTINEL).all()), "step %d wrote dst" % i
    with pytest.raises(espflix_b200.EspflixError) as e:             # the next index rolled back to the short call
        ctx.present_picture_async(j + 1, bufs[bad])
    assert e.value.code == capi.EF_ESTATE
    retry, rc, k, _ = replay(ctx, [("submit-done",)] * bad + steps[bad:], how=lambda i: "async" if i >= bad else "skip", caps=caps)
    assert rc == capi.EF_OK and k == len(steps) - bad
    same(retry, want, keys=range(bad, len(steps)), what="retry")
    a, b = ref.picture_pts(), ctx.picture_pts()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    ref.close()
    ctx.close()


# ---- the calls that resolve a chain ------------------------------------------------------------------------------------------
def test_calls_that_resolve_a_chain():
    """overlay changes staged between async calls, ef_restart_streams, ef_index and ef_reset after a chain nobody waited for,
    and synchronous calls in the middle of one: the same fields and info as the all-synchronous run"""
    n = 3
    subs = [[np.frombuffer(bytes(pc.synth_ts(140 + 3 * k + s, 4 + s)), dtype=np.uint8) for s in range(n)] for k in range(4)]
    c0 = presenting_context(n, 1, fc0=[0, 5, 9])
    steps, _ = build(c0, subs, idle_after=lambda k: [1, 0, 2])
    c0.close()
    starts = [i for i, st in enumerate(steps) if st[0] == "submit"]
    bm = np.random.RandomState(3).randint(0, 256, size=(n, 1280)).astype(np.uint8)

    def hooks(i, c):
        if i == starts[0] + 2:
            c.present_overlay(bm, blend=[20, -1, 5], progress=[50, 100, 0])
        if i == starts[1] + 3:
            c.present_overlay(blend=[0, 31, 2], set=[2, 2, 2])
        if i == starts[2]:
            c.restart_streams([1, 2, 0])
        if i == starts[3]:
            c.reset()
    ref = presenting_context(n, 1, fc0=[0, 5, 9])
    want, rc, _, _ = replay(ref, steps, lambda i: "sync", between=hooks)
    ref.close()
    caps = totals(want)
    for how in (lambda i: "async", lambda i: "sync" if i in (starts[1] + 2, starts[2] + 1) else "async"):
        ctx = presenting_context(n, 1, fc0=[0, 5, 9])
        got, rc, _, _ = replay(ctx, steps, how, caps, between=hooks)
        assert rc == capi.EF_OK
        same(got, want, what="resolving calls")
        ctx.close()


# ---- beside the asynchronous audio decode ------------------------------------------------------------------------------------
def test_beside_async_audio():
    """ef_decode_audio_async on one stream, a submit's presentation as one async chain on another: the fields equal a run
    without audio, the audio the synchronous decode"""
    from tests import restart_cases as rc
    n, K = 4, 2
    progs = [[rc.program(700 + 10 * s + k, 12, 300000 + 36036 * k, audio=dict(seed=90 + 7 * s + k, frames=60, cut=0)) for k in range(K)] for s in range(n)]
    subs = [[np.frombuffer(p[k], dtype=np.uint8) for p in progs] for k in range(K)]
    plain = presenting_context(n, 1, fc0=[0, 3, 1000, 7], max_pictures=12)
    steps, want = build(plain, subs)
    plain.close()
    caps = totals(want)
    ctx = presenting_context(n, 1, fc0=[0, 3, 1000, 7], max_pictures=12)
    ref = espflix_b200.Context(n_streams=n, max_pictures=12, es_capacity=n * 12 * 40000, fields=False)
    ctx.enable_audio()
    ref.enable_audio()
    ast, pst = torch.cuda.Stream(), torch.cuda.Stream()
    heard = []

    def check(c, i):
        if heard:                                       # the previous submit's audio, decoded beside its presentation
            want_a, info, pcm, pdm = heard.pop()
            assert c.audio_wait() == capi.EF_OK
            same_audio(want_a, audio_results(info, pcm, pdm), "step %d" % i)

    def audio(i, c):
        if steps[i][0] == "submit":
            check(c, i)
        if steps[i][0] == "pic" and steps[i][1] == 0:
            ref.submit_ts(*ref.pack(subs[len([s for s in steps[:i] if s[0] == "submit"]) - 1]))
            ref.index()
            want_a = ref.decode_audio()
            need = sum(r["n_frames"] for r in want_a) * 128
            pcm = torch.empty(need, dtype=torch.int16, device="cuda")
            pdm = torch.empty(2 * need, dtype=torch.int16, device="cuda").view(torch.uint16)
            heard.append((want_a, c.decode_audio_async(pcm, pdm, stream=ast), pcm, pdm))
    got, rcode, _, _ = replay(ctx, steps, caps=caps, stream=pst.cuda_stream, between=audio)
    check(ctx, len(steps))
    assert rcode == capi.EF_OK
    same(got, want, what="beside audio")
    ctx.close()
    ref.close()


# ---- API rules and launch counts ---------------------------------------------------------------------------------------------
def test_api_rules_and_launch_counts():
    ts = [pc.synth_ts(70 + i, n) for i, n in enumerate((5, 3))]
    blob, off = espflix_b200.Context.pack(ts)
    ctx = espflix_b200.Context(n_streams=2, max_pictures=5, fields=False)
    out = torch.zeros(4 * 1136 * 312, dtype=torch.uint16, device="cuda")
    assert error_code(lambda: ctx.present_idle_async([1, 1], out)) == capi.EF_ESTATE                   # before ef_present_enable
    ctx.enable_pts()
    ctx.video_init(0)
    ctx.enable_present([10, 20])
    assert error_code(lambda: ctx.present_picture_async(0, out)) == capi.EF_ESTATE                    # no ef_index since enabling
    ctx.submit_ts(blob, off)
    ctx.index()
    w, nl = ctx.geometry()
    info = torch.zeros((2, 8), dtype=torch.int32, device="cuda")
    nf = np.ones(2, dtype=np.uint32)
    lib, h = ctx.lib, ctx._h
    host = np.zeros(4 * w * nl, dtype=np.uint16)
    host_info = np.zeros(2, dtype=capi.PRESENT_INFO)
    for dst, inf in ((None, info.data_ptr()), (out.data_ptr(), None), (host.ctypes.data, info.data_ptr()), (out.data_ptr(), host_info.ctypes.data),
                     (out.data_ptr() + 2, info.data_ptr())):
        assert lib.ef_present_idle_async(h, nf.ctypes.data, dst, 3, inf, None) == capi.EF_EINVAL
        assert lib.ef_present_picture_async(h, 0, None, dst, 3, inf, None) == capi.EF_EINVAL
    assert lib.ef_present_idle_async(h, None, out.data_ptr(), 3, info.data_ptr(), None) == capi.EF_EINVAL
    with pytest.raises(TypeError):
        ctx.present_idle_async(nf, out.cpu())
    assert error_code(lambda: ctx.present_picture_async(1, out)) == capi.EF_ESTATE                    # out of order
    assert error_code(lambda: ctx.present_picture_async(0, out, modes=[4, 0])) == capi.EF_EINVAL
    assert ctx.present_wait() == (capi.EF_OK, 0)                                                  # nothing enqueued
    cap = 65535 + 3                                                                               # two K2 launches per call
    big = torch.empty(cap * w * nl, dtype=torch.uint16, device="cuda")
    n0 = ctx.launch_count()
    ctx.present_picture_async(0, big)
    # schedule + size + K1a (picture 0 starts the range) + K1b + descriptors + ceil(dst_fields / 65,535) K2
    assert ctx.launch_count() - n0 == 1 + 1 + 1 + 1 + 1 + 2
    n0 = ctx.launch_count()
    ctx.present_picture_async(1, big[:8 * w * nl])
    assert ctx.launch_count() - n0 == 1 + 1 + 0 + 1 + 1 + 1
    n0 = ctx.launch_count()
    ctx.present_idle_async(nf, big[:8])                                                           # dst_fields 0: no K2
    assert ctx.launch_count() - n0 == 1 + 1 + 1
    assert ctx.present_wait() == (capi.EF_ENOMEM, 2)                                              # the idle call had no room
    # a short picture call inside the range, then its retry: K1a again at the retried index
    need = int(ctx.present_picture(2)["n_fields"].sum())
    assert need > 0
    ctx.present_picture_async(2, big[:(need - 1) * w * nl])
    assert ctx.present_wait() == (capi.EF_ENOMEM, 0)
    n0 = ctx.launch_count()
    ctx.present_picture_async(2, big[:need * w * nl])
    assert ctx.launch_count() - n0 == 1 + 1 + 1 + 1 + 1 + 1
    assert ctx.present_wait() == (capi.EF_OK, 1)
    assert error_code(lambda: ctx.submit_ts(blob, off) or ctx.index()) == capi.EF_ESTATE               # pictures 3, 4 unpresented
    ctx.present_picture_async(3, big[:8 * w * nl])
    ctx.present_picture_async(4, big[:8 * w * nl])
    ctx.submit_ts(blob, off)
    ctx.index()                                                                                   # resolves the chain
    assert ctx.present_wait() == (capi.EF_OK, 2)
    ctx.close()


# ---- the benchmark's batch size --------------------------------------------------------------------------------------------
def _digests(rows, k, weights):
    """one int64 digest per field row of the first k rows, on the device, on the current stream"""
    out = []
    for a in range(0, k, 256):
        out.append((rows[a:min(k, a + 256)].to(torch.int64) * weights).sum(dim=1))
    return torch.cat(out) if out else torch.zeros(0, dtype=torch.int64, device="cuda")


@pytest.mark.parametrize("n", [4096, 3001])
def test_batch_step_as_one_chain(n):
    """a full step of the benchmark-sized batch (12 pictures and an idle tail) as one async chain into one reused buffer,
    against the synchronous run: info of every call, and a digest of every stream's every field"""
    b = scale_cases.batch()
    blob, off = espflix_b200.Context.pack(b.all_ts()[:n])
    fc0 = [b.fc0(s) for s in range(n)]

    def make():
        ctx = espflix_b200.Context(n_streams=n, max_pictures=12, max_slices_per_picture=12, es_capacity=int(off[-1]) + 4096, fields=False)
        ctx.enable_pts()
        ctx.video_init(1)
        ctx.enable_present(fc0)
        ctx.submit_ts(blob, off)
        ctx.index()
        return ctx
    calls = [("pic", p, np.array([b.modes(s)[p] for s in range(n)], dtype=np.uint8)) for p in range(12)]
    calls.append(("idle", np.array([scale_cases.idle_fields(s % scale_cases.D) for s in range(n)], dtype=np.uint32)))
    ctx = make()
    w, nl = ctx.geometry()
    weights = torch.randint(1, 1 << 20, (w * nl,), dtype=torch.int64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    want = []
    for c in calls:
        fn = (lambda o: ctx.present_picture(c[1], c[2], o)) if c[0] == "pic" else (lambda o: ctx.present_idle(c[1], o))
        info = fn(None)
        total = int(info["n_fields"].sum())
        out = torch.empty(max(total, 1) * w * nl, dtype=torch.uint16, device="cuda")
        assert (fn(out) == info).all()
        want.append((info, _digests(out.view(torch.int16).view(-1, w * nl), total, weights).cpu().numpy()))
        del out
    ctx.close()
    torch.cuda.empty_cache()
    ctx = make()
    cap = max(int(i["n_fields"].sum()) for i, _ in want) + 64                 # the largest call plus a margin
    buf = torch.full((cap * w * nl,), SENTINEL, dtype=torch.int16, device="cuda")
    rows = buf.view(-1, w * nl)
    got = []
    for c, (wi, _) in zip(calls, want):
        if c[0] == "pic":
            info = ctx.present_picture_async(c[1], buf.view(torch.uint16), modes=c[2], stream=torch.cuda.current_stream())
        else:
            info = ctx.present_idle_async(c[1], buf.view(torch.uint16), stream=torch.cuda.current_stream())
        got.append((info, _digests(rows, int(wi["n_fields"].sum()), weights)))   # stream-ordered behind the call
    assert ctx.present_wait() == (capi.EF_OK, len(calls))
    for k, ((wi, wd), (gi, gd)) in enumerate(zip(want, got)):
        gi = ctx.present_info(gi)
        for f in INFO_FIELDS:
            assert np.array_equal(gi[f], wi[f]), "call %d: info %s" % (k, f)
        gd = gd.cpu().numpy()
        bad = np.nonzero(gd != wd)[0]
        assert bad.size == 0, "call %d: field %d differs" % (k, bad[0])
    ctx.close()
    del buf, rows
    torch.cuda.empty_cache()
