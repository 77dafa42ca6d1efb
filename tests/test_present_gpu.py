"""Paced presentation through the decoder context (ef_present_enable / ef_present_picture / ef_present_idle): every stream's
composite fields, concatenated over the calls, must hash to the field stream the unmodified reference emitted
(tests/golden/pacing_pins.json) and equal, field by field, K2's rendering of the restatement in tests/present_cases.py."""
import json
import os

import numpy as np
import pytest
import torch

import espflix_b200
from espflix_b200 import capi, synth
from tests import carry_cases, overlay_cases as oc, present_cases as pc, pts_cases
from tests.harness import Paced, error_code, present_call, presenting_context, sha, submits
from tests.oracle_lib import Oracle

pytestmark = pytest.mark.gpu
G = pts_cases.GOLDEN
PINS = json.load(open(os.path.join(G, "pacing_pins.json")))
IRREGULAR = json.load(open(os.path.join(G, "ref_pins.json")))["pacing_irregular"]


def _driver(ctx, ntsc, frames, fc0, oracle):
    """the paced driver over present_cases' displays and renderers"""
    return Paced(ctx, [pc.Display(ntsc, int(f)) for f in fc0], [pc.Renderer(oracle, ntsc) for _ in frames], frames)


@pytest.mark.parametrize("ntsc", [1, 0])
def test_pinned_streams_hash_to_the_reference(ntsc):
    """the pinned cases of one standard in one context, with filler streams of other lengths: pts, flips and the whole
    field stream of each pinned case as the reference emitted it"""
    o = Oracle()
    names = [n for n in sorted(PINS) if PINS[n]["ntsc"] == ntsc]
    ts = [pc.synth_ts(PINS[n]["seed"], PINS[n]["pictures"]) for n in names] + [pc.synth_ts(60 + ntsc, 7), pc.synth_ts(62 + ntsc, 12)]
    fc0 = [PINS[n]["frame_counter0"] for n in names] + [3, 100]
    frames = [o.decode_ts(t) for t in ts]
    ctx = presenting_context(len(ts), ntsc, fc0=fc0)
    r = _driver(ctx, ntsc, frames, fc0, o)
    modes = {i: PINS[n]["modes"] for i, n in enumerate(names)}
    r.submit([np.frombuffer(bytes(t), dtype=np.uint8) for t in ts], lambda s, g: modes[s][g] if s in modes else (2 if g == 4 else 0))
    tails = [((PINS[n]["flip_field"][-1] + 1 + PINS[n]["tail_fields"] - PINS[n]["frame_counter0"]) & pc.M32) - len(r.dev[i]) for i, n in enumerate(names)]
    r.idle(tails + [5, 0])
    for i, n in enumerate(names):
        p = PINS[n]
        assert r.pts[i] == [129003 + 3003 * k for k in range(p["pictures"])]
        assert [a for a, _ in r.flips[i]] == p["flip_field"] and [b for _, b in r.flips[i]] == p["flip_line"], n
        assert len(r.dev[i]) == p["fields"]
        assert r.stream_hash[i].hexdigest() == p["stream_sha256"], n
    r.check()
    ctx.close()


@pytest.fixture(scope="module")
def irregular():
    o = Oracle()
    return [(c, ts, pts, ntsc, fc0, modes, tail, o.decode_ts(ts)) for c, ts, pts, ntsc, fc0, modes, tail in pc.irregular_programs()]


def _run_irregular(progs, ntsc, cuts_seed=None, idle_between=False):
    progs = [p for p in progs if p[3] == ntsc]
    o = Oracle()
    fc0 = [p[4] for p in progs]
    ctx = presenting_context(len(progs), ntsc, fc0=fc0)
    r = _driver(ctx, ntsc, [p[7] for p in progs], fc0, o)
    mode_of = lambda s, g: progs[s][5][g]                                         # noqa: E731
    if cuts_seed is None:
        chunks = [[np.frombuffer(bytes(p[1]), dtype=np.uint8) for p in progs]]
    else:
        rng = np.random.RandomState(cuts_seed)
        K = int(rng.randint(2, 5))
        per = []
        for p in progs:
            cand = pts_cases.cut_points(p[1])
            per.append(carry_cases.cut(p[1], sorted(rng.choice(cand, size=K - 1, replace=True).tolist()) if cand else []))
        chunks = submits(per, n=K)
    rng = np.random.RandomState(99)
    for k, c in enumerate(chunks):
        r.submit(c, mode_of)
        if idle_between and k + 1 < len(chunks):
            r.idle(rng.randint(0, 3, size=len(progs)))
    r.idle([p[6] + 1 for p in progs])
    return r, progs, ctx


@pytest.mark.parametrize("ntsc", [1, 0])
def test_irregular_schedules_as_ts_programs(irregular, ntsc):
    r, progs, ctx = _run_irregular(irregular, ntsc)
    for s, p in enumerate(progs):
        want = IRREGULAR[p[0]]
        assert r.pts[s] == p[2]
        assert [a for a, _ in r.flips[s]] == want["flip_field"] and [b for _, b in r.flips[s]] == want["flip_line"], p[0]
    r.check()
    ctx.close()


@pytest.mark.parametrize("ntsc", [1, 0])
def test_cut_submits_equal_the_uncut_run(irregular, ntsc):
    whole, progs, ctx = _run_irregular(irregular, ntsc)
    ctx.close()
    for seed in (5, 6):
        cut, _, ctx = _run_irregular(irregular, ntsc, cuts_seed=seed + ntsc)
        assert cut.dev == whole.dev and cut.flips == whole.flips
        ctx.close()
    mixed, _, ctx = _run_irregular(irregular, ntsc, cuts_seed=7 + ntsc, idle_between=True)   # idle runs between submits
    mixed.check()
    assert [a for a, _ in mixed.flips[0]] != [] and mixed.pts == whole.pts
    ctx.close()


def test_fixtures_step_by_step():
    """splash.ts and vmedia.ts presented one picture index at a time: the pictures still as decode_pins.json, the fields
    as the restatement renders them"""
    dpins = json.load(open(os.path.join(G, "decode_pins.json")))
    o = Oracle()
    names = list(pts_cases.FIXTURES)
    ts = [open(os.path.join(G, n + ".ts"), "rb").read() for n in names]
    frames = [o.decode_ts(t) for t in ts]
    for ntsc in (1, 0):
        ctx = presenting_context(2, ntsc, max_pictures=100, fc0=[1, 2])
        r = _driver(ctx, ntsc, frames, [1, 2], o)
        got = [[], []]
        orig = r.ctx.present_picture

        def present_and_read(pic, modes=None, out=None, stream=0):
            info = orig(pic, modes, out, stream)
            if out is not None:
                for s in range(2):
                    if pic < ctx.stream_info(s)[0]:
                        got[s].append(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + pic + 1) & 1))
            return info
        r.ctx.present_picture = present_and_read
        r.submit([np.frombuffer(t, dtype=np.uint8) for t in ts], lambda s, g: 1 if g == len(frames[s]) - 1 else 0)
        r.idle(3)
        for s, n in enumerate(names):
            assert len(got[s]) == dpins[n]["frames"]
            for k, f in enumerate(got[s]):
                assert sha(f) == dpins[n]["frame_sha256"][k], "%s picture %d" % (n, k)
        r.check()
        ctx.close()


def test_api_rules_and_launch_counts():
    o = Oracle()
    ts = [pc.synth_ts(70 + i, n) for i, n in enumerate((5, 3))]
    frames = [o.decode_ts(t) for t in ts]
    blob, off = espflix_b200.Context.pack(ts)

    ctx = espflix_b200.Context(n_streams=2, max_pictures=5, fields=False)
    assert error_code(lambda: ctx.enable_present()) == capi.EF_ESTATE                  # needs PTS first
    ctx.enable_pts()
    ctx.video_init(0)
    ctx.enable_present([10, 20])
    assert error_code(lambda: ctx.enable_present()) == capi.EF_ESTATE
    assert error_code(lambda: ctx.video_init(1)) == capi.EF_ESTATE                      # the standard is fixed
    ctx.video_init(0)
    assert error_code(lambda: ctx.present_picture(0)) == capi.EF_ESTATE                # no ef_index since enabling
    ctx.submit_ts(blob, off)
    ctx.index()
    assert error_code(lambda: ctx.decode_picture(0)) == capi.EF_ESTATE
    assert error_code(lambda: ctx.decode_all(5)) == capi.EF_ESTATE
    out_host = np.zeros((5, 2, 101376), dtype=np.uint8)
    assert error_code(lambda: ctx.decode_all_to_host(5, out_host)) == capi.EF_ESTATE
    assert error_code(lambda: ctx.present_picture(1)) == capi.EF_ESTATE                # out of order
    assert error_code(lambda: ctx.present_picture(0, [4, 0])) == capi.EF_EINVAL
    w, nl = ctx.geometry()
    # a sizing call changes nothing; too small a buffer is EF_ENOMEM and changes nothing either
    n0 = ctx.launch_count()
    i1 = ctx.present_picture(0)
    i2 = ctx.present_picture(0)
    assert (i1 == i2).all() and ctx.launch_count() == n0 + 2
    assert error_code(lambda: ctx.present_picture(1)) == capi.EF_ESTATE                # sizing did not advance it
    r = _driver(ctx, 0, frames, [10, 20], o)
    fields = [[], []]
    for p in range(5):
        info = ctx.present_picture(p)
        total = int(info["n_fields"].sum())
        if total:
            small = torch.empty(total * w * nl - 8, dtype=torch.uint16, device="cuda")   # room for total - 1 fields
            assert error_code(lambda: ctx.present_picture(p, None, small)) == capi.EF_ENOMEM
        if p == 2:
            assert error_code(lambda: ctx.submit_ts(blob, off) or ctx.index()) == capi.EF_ESTATE   # pictures 3, 4 unpresented
        n0 = ctx.launch_count()
        want = []
        for s in range(2):
            if p < len(frames[s]):
                r.rend[s].decoded(p, frames[s][p])
                want.append(r.disp[s].push(129003 + 3003 * p)[0])
            else:
                want.append([])
        got, host = present_call(ctx, lambda o_: ctx.present_picture(p, None, o_))
        # sizing (1) + schedule (1) + K1a at picture 0 + K1b (1) + descriptors (1) + one K2 per 65,535 fields
        assert ctx.launch_count() - n0 == 1 + 1 + (p == 0) + 1 + 1 + (1 if total else 0)
        r.collect(got, host, want)
    assert error_code(lambda: ctx.present_picture(5)) == capi.EF_ESTATE
    r.idle(2)
    r.check()
    # ef_reset mid-run is video_reset(): new origin, position / store / scroll kept; the frame stores are zero-filled
    ctx.reset()
    for s in range(2):
        r.disp[s].reset()
        r.rend[s].reset()
    r.seen = [0, 0]
    late = [oc.segment_ts(80 + i, [9000000 + 3003 * k for k in range(3)]) for i in range(2)]
    r.frames = [o.decode_ts(t) for t in late]
    r.submit([np.frombuffer(t, dtype=np.uint8) for t in late])
    r.idle(1)
    r.check()
    ctx.close()

    # a picture without pts (an ES submit carries no PES) is not pushed: flag 1
    ctx = presenting_context(1, 1, max_pictures=4)
    es, _ = synth.generate(synth.SEED0 + 90, n_pictures=2)
    ctx.submit_es(*ctx.pack([es]))
    ctx.index()
    info, _ = present_call(ctx, lambda o_: ctx.present_picture(0, None, o_))
    assert int(info[0]["flags"]) == 1 and int(info[0]["flip_line"]) == -1 and int(info[0]["n_fields"]) == 0
    ctx.close()

    # a context that never presents launches what it launched before
    ctx = espflix_b200.Context(n_streams=2, max_pictures=5)
    ctx.enable_pts()
    ctx.submit_ts(blob, off)
    n0 = ctx.launch_count()
    ctx.index()
    ctx.decode_all(5)
    ctx.composite_field(-1, 1)
    assert ctx.launch_count() - n0 == 4 + 1 + 5 + 1
    ctx.close()
