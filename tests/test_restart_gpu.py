"""ef_restart_streams through the decoder context: restarted streams must give what the unmodified reference gave on the same
programs (tests/golden/restart_pins.json) and the restatement in tests/restart_cases.py - pts of every picture, get_pts(), PCM,
PDM and paced fields with the overlay on - while every other stream stays bit-identical to the same context run without any
restart call."""
import hashlib
import json
import os

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import overlay_cases as oc, restart_cases as rc
from tests.harness import present_call, presenting_context, sha, stage_overlay

pytestmark = pytest.mark.gpu
PINS = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "restart_pins.json")))
DEC = rc.decoder_cases()
NAMES = sorted(DEC)
FILLERS = 3


def _filler_programs(i, k):
    """k back-to-back GOPs of one program for an untouched stream: pts and audio continue from submit to submit"""
    return [rc.program(400 + 10 * i + j, 6, 500000 + 18018 * j, audio=dict(seed=60 + 7 * i + j, frames=36, cut=0)) for j in range(k)]


def _decoder_run(restart, queued=False):
    """the decoder cases on streams 0..3 and FILLERS untouched streams after them, one submit per program. restart: call
    ef_restart_streams (op 1 on the cases' streams that start a new program, 0 elsewhere). queued: the next submit is made
    before the restart call. -> per stream (pic_pts per submit, last_pts per submit, pcm per submit, whole pdm)"""
    K = max(len(p) for p in DEC.values())
    progs = [DEC[n] + [b""] * (K - len(DEC[n])) for n in NAMES] + [_filler_programs(i, K) for i in range(FILLERS)]
    n = len(progs)
    ctx = espflix_b200.Context(n_streams=n, max_pictures=12, es_capacity=n * 12 * 40000, fields=False)
    ctx.enable_pts()
    ctx.enable_audio()
    out = [dict(pic=[], last=[], pcm=[], pdm=[]) for _ in range(n)]
    ctx.submit_ts(*ctx.pack([p[0] for p in progs]))
    for k in range(K):
        ctx.index()
        pic, last = ctx.picture_pts()
        end = np.array([k == K - 1] * n, dtype=np.uint8)
        res = ctx.decode_audio(end=end)
        for s in range(n):
            out[s]["pic"].append([int(v) for v in pic[s]])
            out[s]["last"].append(int(last[s]))
            out[s]["pcm"].append(res[s]["pcm"])
            out[s]["pdm"].append(res[s]["pdm"])
        if k + 1 == K:
            break
        ops = np.array([1 if k + 1 < len(DEC[nm]) else 0 for nm in NAMES] + [0] * FILLERS, dtype=np.uint8)
        if queued:
            ctx.submit_ts(*ctx.pack([p[k + 1] for p in progs]))
        if restart:
            before = ctx.launch_count()
            ctx.restart_streams(ops)
            assert ctx.launch_count() - before == 2           # the restart kernel and the demux-gate kernel
        if not queued:
            ctx.submit_ts(*ctx.pack([p[k + 1] for p in progs]))
    ctx.close()
    return out


@pytest.fixture(scope="module")
def plain():
    return _decoder_run(False)


@pytest.mark.parametrize("queued", [False, True])
def test_mixed_batch_decoder(queued, plain):
    got = _decoder_run(True, queued)
    for s, name in enumerate(NAMES):
        pin, progs = PINS["decoder"][name], DEC[name]
        P = len(progs)
        want = rc.decoder_restate(progs)
        for p in range(P):
            npics = pin["pictures"][p]
            pic = got[s]["pic"][p][:npics]
            assert pic == want["pic_pts"][p], (name, p, pic, want["pic_pts"][p])
            assert got[s]["last"][p] == pin["get_pts"][p], (name, p)
            assert got[s]["pcm"][p].size == pin["pcm_samples"][p] and sha(got[s]["pcm"][p]) == pin["pcm_sha256"][p], (name, p)
        assert sha(np.concatenate(got[s]["pdm"][:P])) == pin["pdm_sha256"], name
        # the reference's pushes: every program's pictures but its last, all of the last program's
        pushes = [v for p in range(P) for v in (want["pic_pts"][p] if p == P - 1 else want["pic_pts"][p][:-1])]
        assert pushes == pin["pushes"]
    for s in range(len(NAMES), len(NAMES) + FILLERS):       # untouched streams: bit-identical to the run without restarts
        assert got[s]["pic"] == plain[s]["pic"] and got[s]["last"] == plain[s]["last"]
        for a, b in zip(got[s]["pcm"], plain[s]["pcm"]):
            assert np.array_equal(a, b)
        for a, b in zip(got[s]["pdm"], plain[s]["pdm"]):
            assert np.array_equal(a, b)


PACED = dict(rc.paced_cases(), **rc.idle_resume_cases())
CASE_AT = 2                                                     # the case's stream; streams 0, 1 and 3 are untouched fillers


def _paced_run(case, restart):
    """the case on stream CASE_AT of a 4-stream context, fillers with their own programs (pts continuing over the segments)
    around it. restart: ef_restart_streams(op) on the case's stream alone (first = CASE_AT) before every later segment.
    -> (per stream SHA-256 of its field stream, the case's flip fields, the case's fields)"""
    n = 4
    ctx = presenting_context(n, case["ntsc"], case["fc0"])
    disps = [oc.OverlayDisplay(case["ntsc"], case["fc0"]) for _ in range(n)]
    whole = [hashlib.sha256() for _ in range(n)]
    flips, emitted, k, base = [], [0] * n, 0, 0

    def take(info, host):
        for s in range(n):
            a, m = int(info[s]["first"]), int(info[s]["n_fields"])
            whole[s].update(host[a:a + m].tobytes())
            emitted[s] += m

    for si, (seed, pts) in enumerate(case["segments"]):
        if si and case.get("idle_before") and case["idle_before"][si]:
            nf = np.zeros(n, np.uint32)
            nf[CASE_AT] = case["idle_before"][si]
            take(*present_call(ctx, lambda o: ctx.present_idle(nf, o)))
        if si and restart:
            ctx.restart_streams([case["op"]], first=CASE_AT)
        ts = [oc.segment_ts(600 + 10 * s + si, [200000 + 50000 * s + 3003 * (base + j) for j in range(len(pts))]) for s in range(n)]
        ts[CASE_AT] = oc.segment_ts(seed, pts) if restart else b""      # without the restart the case's pts would run backwards
        base += len(pts)
        ctx.submit_ts(*ctx.pack(ts))
        ctx.index()
        for j in range(len(pts)):
            cmds = [None] * n
            cmds[CASE_AT] = case["cmds"][k] if restart else None
            stage_overlay(ctx, disps, cmds)
            modes = np.zeros(n, np.uint8)
            modes[CASE_AT] = case["modes"][k] if restart else 0
            info, host = present_call(ctx, lambda o: ctx.present_picture(j, modes=modes, out=o))
            take(info, host)
            flips.append(int(info[CASE_AT]["flip_field"]))
            k += 1
    return ctx, whole, flips, emitted, take


@pytest.mark.parametrize("name", sorted(PACED))
def test_paced_mixed_batch_with_overlay(name, oracle_frames):
    """the restarted stream equals the pins (and, for the idle-run resumes, the restatement); its neighbours' fields are
    bit-identical to the same context run without the restart call"""
    case = PACED[name]
    want_fields, want_flips, want_sha = rc.paced_restate(case, oracle_frames(case), oracle_frames.oracle)
    if name in PINS["paced"]:
        pin = PINS["paced"][name]
        assert (want_fields, want_flips, want_sha) == (pin["fields"], pin["flip_field"], pin["stream_sha256"])
    runs = []
    for restart in (True, False):
        ctx, whole, flips, emitted, take = _paced_run(case, restart)
        nf = np.full(4, 5, np.uint32)
        nf[CASE_AT] = want_fields - emitted[CASE_AT] if restart else 5
        take(*present_call(ctx, lambda o: ctx.present_idle(nf, o)))
        ctx.close()
        runs.append(([h.hexdigest() for h in whole], flips))
    (got, flips), (plain, _) = runs
    assert flips == want_flips
    assert got[CASE_AT] == want_sha
    assert [got[s] for s in range(4) if s != CASE_AT] == [plain[s] for s in range(4) if s != CASE_AT]


@pytest.fixture(scope="module")
def oracle_frames():
    from tests.oracle_lib import Oracle
    o = Oracle()

    def frames(case):
        return [o.decode_ts(oc.segment_ts(seed, pts)) for seed, pts in case["segments"]]
    frames.oracle = o
    return frames


def test_errors_and_launches():
    ts = rc.program(501, 4, 90000, audio=dict(seed=5, frames=20))
    ctx = espflix_b200.Context(n_streams=2, max_pictures=8, es_capacity=2 * 8 * 40000, fields=False)
    for bad in ((-1, 1), (2, 1), (1, 2)):
        with pytest.raises(capi.EspflixError) as e:
            ctx.restart_streams(np.zeros(bad[1], np.uint8), first=bad[0])
        assert e.value.code == capi.EF_EINVAL
    with pytest.raises(capi.EspflixError) as e:
        ctx.restart_streams([3, 0])
    assert e.value.code == capi.EF_EINVAL
    before = ctx.launch_count()
    ctx.restart_streams([1, 2])                                 # nothing enabled: the kernel only
    assert ctx.launch_count() - before == 1
    ctx.restart_streams([])
    assert ctx.launch_count() - before == 1
    ctx.enable_pts()
    ctx.enable_audio()
    ctx.submit_ts(*ctx.pack([ts, ts]))
    ctx.index()
    with pytest.raises(capi.EspflixError) as e:                 # the current submit's audio is unconsumed
        ctx.restart_streams([1, 0])
    assert e.value.code == capi.EF_ESTATE
    ctx.decode_audio()
    before = ctx.launch_count()
    ctx.restart_streams([2, 0])                                 # no op 1: no demux-gate kernel
    assert ctx.launch_count() - before == 1
    ctx.close()
    ctx = presenting_context(2, 1, 0)
    ctx.submit_ts(*ctx.pack([ts, ts]))
    ctx.index()
    present_call(ctx, lambda o: ctx.present_picture(0, out=o))
    with pytest.raises(capi.EspflixError) as e:                 # pictures 1.. of the current submit are unpresented
        ctx.restart_streams([1, 1])
    assert e.value.code == capi.EF_ESTATE
    for p in range(1, 4):
        present_call(ctx, lambda o: ctx.present_picture(p, out=o))
    ctx.restart_streams([1, 1])
    ctx.close()


def test_scale_staggered_restarts():
    """tests/scale_cases.py's 4,096-stream batch over three submits of the same programs. Before submits 1 and 2, streams with
    one SBC frame size throughout (d % 3 != 0) restart into the start of their program, staggered (s % 4 == 1: before submit 1,
    2: before submit 2, 3: both), through two calls on sub-ranges ([0, 1000) and [1000, 4096): several CTAs, first > 0).
    Every stream is checked: get_pts() between the restart and the next submit, the pts of every picture, the latest picture,
    and PCM and PDM against the restatement (a single run: the whole-stream checker on the three copies)."""
    from tests import scale_cases
    from tests.oracle_lib import Oracle
    o = Oracle()
    b = scale_cases.batch()
    N, D, K = scale_cases.N, scale_cases.D, 3
    pattern = lambda s: (s % 4) if (s % D) % 3 else 0                  # noqa: E731
    restarted = lambda s, j: pattern(s) in (j, 3)                       # noqa: E731
    blob, off = espflix_b200.Context.pack(b.all_ts())
    ctx = espflix_b200.Context(n_streams=N, max_pictures=12, es_capacity=int(off[-1]) + 4096, fields=False)
    ctx.enable_pts()
    ctx.enable_audio()
    pcm, pdm, fsz = [[] for _ in range(N)], [[] for _ in range(N)], [0] * N
    want_pts = np.array([b.pts[s % D] for s in range(N)], dtype=np.int64)
    for j in range(K):
        if j:
            ops = np.array([1 if restarted(s, j) else 0 for s in range(N)], dtype=np.uint8)
            before = ctx.launch_count()
            ctx.restart_streams(ops[:1000])
            ctx.restart_streams(ops[1000:], first=1000)
            assert ctx.launch_count() - before == 4
            _, last = ctx.picture_pts(n_pictures=0)
            want = np.where(ops == 1, -1, want_pts[:, -1])
            bad = np.nonzero(last != want)[0]
            assert bad.size == 0, "submit %d: get_pts of stream %d after the restart" % (j, bad[0])
        ctx.submit_ts(blob, off)
        ctx.index()
        ctx.decode_all(12)
        pic, last = ctx.picture_pts()
        bad = np.nonzero((pic != want_pts).any(axis=1) | (last != want_pts[:, -1]))[0]
        assert bad.size == 0, "submit %d: pts of stream %d" % (j, bad[0])
        res = ctx.decode_audio(end=[j == K - 1] * N)
        for s in range(N):
            pcm[s].append(res[s]["pcm"])
            pdm[s].append(res[s]["pdm"])
            if j == 0:
                fsz[s] = res[s]["frame_size"]
    latest = ctx.read_latest_i420()
    ctx.close()
    frames, audio, want = {}, {}, {}
    for s in range(N):
        d, pt = s % D, pattern(s)
        if d not in frames:
            frames[d] = o.decode_ts(b.ts(d))[-1]
            audio[d] = bytes(o.demux_audio_ts(b.ts(d)))
        assert np.array_equal(latest[s], frames[d]), "latest picture of stream %d" % s
        if (d, pt) not in want:
            if pt == 0:
                p = o.sbc_decode(audio[d] * K)
                want[d, pt] = ([p], o.pdm(p))
            else:
                cuts = [j for j in (1, 2) if pt in (j, 3)]
                edges = [0] + cuts + [K]
                runs = [audio[d] * (e1 - e0) for e0, e1 in zip(edges[:-1], edges[1:])]
                want[d, pt] = rc.audio_restate_runs(o, runs, fsz[s])
        wp, wd = want[d, pt]
        assert np.array_equal(np.concatenate(pcm[s]), np.concatenate(wp)), "PCM of stream %d (pattern %d)" % (s, pt)
        assert np.array_equal(np.concatenate(pdm[s]), wd), "PDM of stream %d (pattern %d)" % (s, pt)
