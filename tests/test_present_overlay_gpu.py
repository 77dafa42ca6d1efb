"""The overlay of paced presentation through the decoder context (ef_present_overlay): every stream's fields, concatenated over
the calls, must hash to the field stream the unmodified reference emitted (tests/golden/overlay_pins.json) and equal, field by
field, the C checker's rendering of the restatement in tests/overlay_cases.py."""
import json
import os

import numpy as np
import pytest
import torch

import espflix_b200
from espflix_b200 import capi
from tests import carry_cases, overlay_cases as oc
from tests import present_cases as pc
from tests import pts_cases, scale_cases
from tests.harness import Paced, error_code, host_fields, present_call, presenting_context, stage_overlay, submits
from tests.oracle_lib import Oracle

pytestmark = pytest.mark.gpu
PINS = json.load(open(os.path.join(pts_cases.GOLDEN, "overlay_pins.json")))
CASES = oc.cases()


class Drive(Paced):
    """the paced driver over an overlay context, cases (tests/overlay_cases.py's dicts, one per stream) and the overlay
    restatement: every segment after the first follows ef_reset, overlay changes are staged before the pushes and idle runs
    of the tail. cut_seed: every segment goes in as 2-4 TS submits with idle runs (and overlay changes) between them."""

    def __init__(self, ctx, cases, oracle, cut_seed=None):
        ntsc = cases[0]["ntsc"]
        super().__init__(ctx, [oc.OverlayDisplay(ntsc, c["fc0"]) for c in cases], [oc.OverlayRenderer(oracle, ntsc) for _ in cases], None)
        self.cases, self.o = cases, oracle
        self.rng = np.random.default_rng(cut_seed)
        self.cut = cut_seed is not None

    def render(self, s, fields):
        ovs = self.disp[s].overlays()[len(self.disp[s].emitted) - len(fields):]
        return [self.rend[s].field(f, ov) for f, ov in zip(fields, ovs)]

    def _random_cmd(self):
        r = self.rng
        if r.random() < 0.4:
            return None
        return oc._cmd(int(r.integers(1, 1000)) if r.random() < 0.5 else None, int(r.integers(-1, 60)) if r.random() < 0.6 else None,
                       int(r.integers(-10, 260)) if r.random() < 0.5 else None)

    def run(self):
        n = len(self.cases)
        for si in range(max(len(c["segments"]) for c in self.cases)):
            segs = [c["segments"][si] if si < len(c["segments"]) else None for c in self.cases]
            base = [len(x) for x in self.pts]                # pushes before this segment
            pre = [False] * n
            if si:                                          # the first push's changes are staged before the reset: they survive it
                pre = [sg is not None for sg in segs]
                stage_overlay(self.ctx, self.disp, [self.cases[s]["cmds"][base[s]] if pre[s] else None for s in range(n)])
                self.ctx.reset()
                for s in range(n):
                    self.disp[s].reset()
                    self.rend[s].reset()
            ts = [oc.segment_ts(*sg) if sg else b"" for sg in segs]
            self.frames = [self.o.decode_ts(t) if sg else [] for t, sg in zip(ts, segs)]
            self.seen = [0] * n
            chunks = [ts]
            if self.cut:
                K = int(self.rng.integers(2, 5))
                per = []
                for t in ts:
                    cand = pts_cases.cut_points(t) if len(t) else []
                    per.append(carry_cases.cut(t, sorted(self.rng.choice(cand, size=K - 1, replace=True).tolist()) if cand else []))
                chunks = submits(per, n=K)

            def stage_pushes(p, pushes):
                stage_overlay(self.ctx, self.disp, [self.cases[s]["cmds"][len(self.pts[s])] if pushes[s] and not pre[s] else None for s in range(n)])
                pre[:] = [a and not b for a, b in zip(pre, pushes)]
            for ci, chunk in enumerate(chunks):
                self.submit(chunk, lambda s, g: self.cases[s]["modes"][base[s] + g], before_call=stage_pushes)
                if self.cut and ci + 1 < len(chunks):
                    nf = self.rng.integers(0, 3, size=n).astype(np.uint32)
                    cmds = [self._random_cmd() for _ in range(n)]
                    self.idle(nf, lambda: stage_overlay(self.ctx, self.disp, cmds))
            for s in range(n):
                assert self.pts[s][base[s]:] == (list(segs[s][1]) if segs[s] else []), s
        last = [f[-1][0] for f in self.flips]
        total = [(last[s] + 1 + c["tail_fields"] - c["fc0"]) & pc.M32 for s, c in enumerate(self.cases)]
        while any(len(d.emitted) < t for d, t in zip(self.disp, total)):
            need = [len(d.emitted) < t for d, t in zip(self.disp, total)]
            cmds = [self.cases[s]["tail_cmds"].get((d.F + (0 if d.L == 0 else 1) - last[s] - 1) & pc.M32) if need[s] else None
                    for s, d in enumerate(self.disp)]
            self.idle(np.array(need, dtype=np.uint32), lambda: stage_overlay(self.ctx, self.disp, cmds))
        return self


def _filler(ntsc, seed, overlay):
    rng = np.random.default_rng(seed)
    n = 7
    cmds = [oc._cmd(int(rng.integers(1, 999)), int(rng.integers(-1, 40)), int(rng.integers(0, 241))) if overlay and rng.random() < 0.7 else None
            for _ in range(n)]
    return dict(ntsc=ntsc, fc0=100 + seed, segments=[(60 + seed, [129003 + 3003 * k for k in range(n)])], modes=[0] * (n - 1) + [2],
                tail_fields=18, cmds=cmds, tail_cmds={2: oc._cmd(None, 30, None)} if overlay else {})


@pytest.mark.parametrize("ntsc", [1, 0])
def test_pinned_cases_among_filler_streams(ntsc):
    """the pinned cases of one standard, with filler streams that carry other overlays or none: the whole field stream of each
    pinned case as the reference emitted it, every field of every stream as the restatement renders it. The reset case runs
    in a context of its own, since ef_reset acts on every stream"""
    o = Oracle()
    names = [n for n in sorted(CASES) if CASES[n]["ntsc"] == ntsc]
    for group in ([n for n in names if len(CASES[n]["segments"]) == 1], [n for n in names if len(CASES[n]["segments"]) > 1]):
        cases = [CASES[n] for n in group] + [_filler(ntsc, 1, True), _filler(ntsc, 2, False)]
        ctx = presenting_context(len(cases), ntsc, [c["fc0"] for c in cases])
        d = Drive(ctx, cases, o).run()
        for i, n in enumerate(group):
            assert len(d.dev[i]) == PINS[n]["fields"], n
            assert d.stream_hash[i].hexdigest() == PINS[n]["stream_sha256"], n
        d.check()
        ctx.close()


def _irregular_cases(ntsc, seed):
    rng = np.random.default_rng(seed)
    out = []
    for case, (pts, nt, fc0, modes, tail) in enumerate(pc.irregular_cases()):
        if nt != ntsc:
            continue
        cmd = lambda: (oc._cmd(int(rng.integers(1, 999)) if rng.random() < 0.5 else None, int(rng.integers(-1, 50)) if rng.random() < 0.6 else None,  # noqa: E731
                               int(rng.integers(-20, 300)) if rng.random() < 0.5 else None) if rng.random() < 0.7 else None)
        out.append(dict(ntsc=ntsc, fc0=fc0, segments=[(200 + case, [int(v) for v in pts])], modes=[int(m) for m in modes], tail_fields=tail + 1,
                        cmds=[cmd() for _ in pts], tail_cmds={t: cmd() for t in range(tail + 1) if rng.random() < 0.3}))
    return out


@pytest.mark.parametrize("ntsc", [1, 0])
def test_irregular_schedules_with_overlay_commands(ntsc):
    """the 24 irregular schedules as TS programs with seeded overlay changes between calls, whole and cut into 2-4 submits with
    idle runs between them"""
    o = Oracle()
    cases = _irregular_cases(ntsc, 40 + ntsc)
    fc0 = [c["fc0"] for c in cases]
    ctx = presenting_context(len(cases), ntsc, fc0)
    Drive(ctx, cases, o).run().check()
    ctx.close()
    for seed in (3, 4):
        ctx = presenting_context(len(cases), ntsc, fc0)
        Drive(ctx, cases, o, cut_seed=seed + 10 * ntsc).run().check()
        ctx.close()


# ---- the benchmark's batch size -------------------------------------------------------------------------------------------
def _batch_cmd(s, p):
    """stream s's change before picture p: a distinct bitmap, blend and progress on every stream, changed as the title plays"""
    if p == 0:
        return oc._cmd(5000 + s, 20 + s % 170, s % 300 - 30)
    if p == 5 and s % 2:
        return oc._cmd(9000 + s, None, (s * 7) % 260)
    if p == 9 and s % 3 == 0:
        return oc._cmd(None, -1 if s % 9 == 0 else 1 + s % 40, None)
    return oc._cmd(None, None, 10 * p + s % 11) if p % 3 == 1 else None


def test_batch_scale_overlay_on_every_stream(oracle):
    """4,096 TS streams x 12 pictures (tests/scale_cases.py), every stream with its own overlay, beside a context that never
    stages one: on every stream, the 16 overlay lines of every field equal the restatement (tests/overlay_cases.py's
    overlay_band) and every other line equals the overlay-free run; the present info and the launches of every call are
    the same; a seeded sample of streams is checked whole against the C checker"""
    from tests.scale_cases import D, N, PICTURES
    b = scale_cases.batch()
    blob, off = espflix_b200.Context.pack(b.all_ts())
    sample = sorted(np.random.default_rng(17).choice(N, size=6, replace=False).tolist())
    for ntsc in (1, 0):
        ctxs = []
        for _ in range(2):
            c = presenting_context(N, ntsc, [b.fc0(s) for s in range(N)], max_pictures=PICTURES, es_capacity=int(off[-1]) + 4096)
            c.submit_ts(blob, off)
            c.index()
            ctxs.append(c)
        plain, ovl = ctxs
        w, nl = plain.geometry()
        _, top, bottom, _ = pc.geometry(ntsc)
        band = slice((bottom + 2) * w, (bottom + 18) * w)
        disp = [oc.OverlayDisplay(ntsc, b.fc0(s)) for s in range(N)]
        rend = {s: oc.OverlayRenderer(oracle, ntsc) for s in sample}
        frames = {s: oracle.decode_es(b.es[s % D]) for s in sample}
        bitmaps = torch.as_tensor(np.stack([oc.bitmap(5000 + s) for s in range(N)] + [oc.bitmap(9000 + s) for s in range(N)]), device="cuda")
        template = torch.as_tensor(oracle.field_ex(np.zeros(101376, np.uint8), np.zeros(101376, np.uint8), ntsc, 0).astype(np.int32)[band].reshape(16, w),
                                   device="cuda")

        def call(fn, want):
            outs, infos, launches = [], [], []
            for c in (plain, ovl):
                i0 = fn(c, None)
                total = int(i0["n_fields"].sum())
                out = torch.empty(max(total, 1) * w * nl, dtype=torch.uint16, device="cuda")
                n0 = c.launch_count()
                infos.append(fn(c, out))
                launches.append(c.launch_count() - n0)
                outs.append(out[:total * w * nl].view(torch.int16).view(total, w * nl))
            assert (infos[0] == infos[1]).all() and launches[0] == launches[1]
            info, (A, B) = infos[1], outs
            assert bool((A[:, :band.start] == B[:, :band.start]).all()) and bool((A[:, band.stop:] == B[:, band.stop:]).all())
            bl, pr, slot = [], [], []
            for s in range(N):
                k = int(info[s]["n_fields"])
                assert k == len(want[s])
                for blend, progress, bm in disp[s].overlays()[len(disp[s].emitted) - k:]:
                    bl.append(blend)
                    pr.append(progress)
                    slot.append(s if not bm.any() or np.array_equal(bm, oc.bitmap(5000 + s)) else N + s)
            for f0 in range(0, len(bl), 4096):
                sl = slice(f0, min(f0 + 4096, len(bl)))
                idx = torch.as_tensor(np.array(slot[sl]), device="cuda")
                want_band = oc.overlay_band(template, bitmaps[idx], torch.as_tensor(np.array(bl[sl]), device="cuda"),
                                            torch.as_tensor(np.array(pr[sl]), device="cuda"), ntsc)
                got = B[sl, band].view(-1, 16, w).to(torch.int32) & 0xFFFF
                bad = (got != want_band).flatten(1).any(1)
                assert not bool(bad.any()), "overlay lines of field %d differ" % (f0 + int(torch.nonzero(bad)[0, 0]))
            for s in sample:
                a, k = int(info[s]["first"]), int(info[s]["n_fields"])
                host = B[a:a + k].cpu().numpy().view(np.uint16)
                ovs = disp[s].overlays()[len(disp[s].emitted) - k:]
                for j in range(k):
                    assert np.array_equal(host[j], rend[s].field(want[s][j], ovs[j])), "stream %d field %d" % (s, j)
            del outs, A, B
            torch.cuda.empty_cache()

        for p in range(PICTURES):
            cmds = [_batch_cmd(s, p) for s in range(N)]
            stage_overlay(ovl, disp, cmds)
            modes = [b.modes(s)[p] for s in range(N)]
            want = []
            for s in range(N):
                if s in rend:
                    rend[s].decoded(p, frames[s][p])
                want.append(disp[s].push(b.pts[s % D][p], modes[s])[0])
            call(lambda c, o: c.present_picture(p, modes, o), want)
        nf = [scale_cases.idle_fields(s % D) for s in range(N)]
        call(lambda c, o: c.present_idle(nf, o), [disp[s].idle(nf[s]) for s in range(N)])
        for c in ctxs:
            c.close()
        torch.cuda.empty_cache()


# ---- unchanged behaviour, sizing, errors -----------------------------------------------------------------------------------
def _two_streams(ntsc):
    return [dict(ntsc=ntsc, fc0=f, segments=[(70 + i, [129003 + 3003 * k for k in range(5)])], modes=[0] * 5, tail_fields=3, cmds=[None] * 5,
                 tail_cmds={}) for i, f in enumerate((10, 20))]


def _fields(ctx, cases, sizing=True, stage=None, enomem=False):
    """present the cases' single segment picture by picture, then 3 idle fields: (every call's fields, launches per call)"""
    ts = [oc.segment_ts(*c["segments"][0]) for c in cases]
    ctx.submit_ts(*ctx.pack(ts))
    ctx.index()
    w, nl = ctx.geometry()
    got, launches = [], []
    for p in range(6):
        if stage:
            stage(ctx, p)
        fn = (lambda o_: ctx.present_picture(p, None, o_)) if p < 5 else (lambda o_: ctx.present_idle([3, 3], o_))
        if enomem:
            total = int(fn(None)["n_fields"].sum())
            if total:
                small = torch.empty(total * w * nl - 8, dtype=torch.uint16, device="cuda")
                with pytest.raises(espflix_b200.EspflixError) as e:
                    fn(small)
                assert e.value.code == capi.EF_ENOMEM
        n0 = ctx.launch_count()
        if sizing:
            info, host = present_call(ctx, fn)
        else:
            out = torch.empty(64 * w * nl, dtype=torch.uint16, device="cuda")
            info = fn(out)
            host = host_fields(out[:int(info["n_fields"].sum()) * w * nl].view(-1, w * nl))
        launches.append(ctx.launch_count() - n0 - (1 if sizing else 0))
        got.append(host.copy())
    return got, launches


def _stager(ctx, p):
    rng = np.random.default_rng(p)
    ctx.present_overlay(rng.integers(0, 256, size=(2, 1280)), [[40, -1, 3, 0, 17, 5][p], 31], [p * 40, 240 - p], [7, 7 if p % 2 else 2])


def test_never_staging_and_staging_change_only_what_they_should():
    for ntsc in (1, 0):
        cases = _two_streams(ntsc)
        fc0 = [c["fc0"] for c in cases]
        plain, lp = _fields(presenting_context(2, ntsc, fc0), cases)
        off, lo = _fields(presenting_context(2, ntsc, fc0), cases, stage=lambda c, p: c.present_overlay(oc.bitmap(p), 0, p, None))   # blend 0: nothing drawn
        on, ln = _fields(presenting_context(2, ntsc, fc0), cases, stage=_stager)
        assert lp == lo == ln
        assert all(np.array_equal(a, b) for a, b in zip(plain, off))
        assert any(not np.array_equal(a, b) for a, b in zip(plain, on))
        # the same fields without sizing calls, and with an EF_ENOMEM call before every real one
        bare, _ = _fields(presenting_context(2, ntsc, fc0), cases, sizing=False, stage=_stager)
        nomem, _ = _fields(presenting_context(2, ntsc, fc0), cases, stage=_stager, enomem=True)
        assert all(np.array_equal(a, b) and np.array_equal(a, c) for a, b, c in zip(on, bare, nomem))


def test_reset_keeps_latched_and_staged_overlays():
    o = Oracle()
    for ntsc in (1, 0):
        cases = _two_streams(ntsc)
        for c in cases:
            c["cmds"] = [oc._cmd(3, 50, 77), None, None, None, oc._cmd(4, -1, 200)]
        cases = [dict(c, segments=c["segments"] + [(80 + i, [900000 + 3003 * k for k in range(3)])], modes=[0] * 8,
                      cmds=c["cmds"] + [oc._cmd(5, 9, None), None, None]) for i, c in enumerate(cases)]
        ctx = presenting_context(2, ntsc, [c["fc0"] for c in cases])
        d = Drive(ctx, cases, o).run()
        d.check()
        ctx.close()


def test_error_codes():
    ctx = espflix_b200.Context(n_streams=3, max_pictures=4, fields=False)
    assert error_code(lambda: ctx.present_overlay(None, 5, 0)) == capi.EF_ESTATE          # before ef_present_enable
    ctx.enable_pts()
    ctx.enable_present()
    assert error_code(lambda: ctx.present_overlay(None, 5, 0, first=-1, count=1)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.present_overlay(None, 5, 0, first=2, count=2)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.present_overlay(None, -2, 0)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.present_overlay(None, [0, -1, -3], 0, first=0, count=3)) == capi.EF_EINVAL
    ctx.present_overlay(None, [0, -1, -3], 0, set=[2, 2, 4])                        # the blend of stream 2 is not set
    ctx.present_overlay(np.zeros((1, 1280), np.uint8), -1, (1 << 31) - 1, first=2, count=1)
    ctx.present_overlay(None, None, None, first=3, count=0)
    ctx.close()
