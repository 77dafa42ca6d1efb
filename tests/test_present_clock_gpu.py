"""The overlay clock of paced presentation (ef_present_font / ef_present_clock) against the host-driven equivalent: context A runs
update_progress() on the device; context B gets the same input, and before every call the host stages through
ef_present_overlay the bitmap and progress that the restatement (tests/clock_cases.py) computes from ef_picture_pts. Every paced
field and every info row of A must equal B's."""
import numpy as np
import pytest
import torch

import espflix_b200
from espflix_b200 import capi
from tests import carry_cases, clock_cases as cc
from tests import overlay_cases as oc
from tests import pts_cases, scale_cases
from tests.harness import error_code, overlay_arrays, present_call, presenting_context, submits
from tests.present_cases import irregular_cases

pytestmark = pytest.mark.gpu
ATLAS, RIGHTS = cc.font()


def _ctx(n, ntsc, fc0, font=True, **kw):
    return presenting_context(n, ntsc, fc0, font=(ATLAS, RIGHTS) if font else None, **kw)


def _header(rng, base):
    v0 = base - int(rng.integers(0, 90000 * 5))
    span = int(rng.integers(90000 * 4, 90000 * 7200))
    f0, r0 = base - int(rng.integers(-90000, 90000)), base - int(rng.integers(-90000, 90000))
    return cc.header((v0, v0 + span), (f0, f0 + int(rng.integers(1, 90000 * 600))), (r0, r0 + int(rng.integers(1, 90000 * 600))))


class Pair:
    """A (the clock on the device) and B (the host's staging of the restatement), driven alike"""

    def __init__(self, n, ntsc, fc0, **kw):
        self.n = n
        self.a = _ctx(n, ntsc, fc0, **kw)
        self.b = _ctx(n, ntsc, fc0, font=False, **kw)
        self.b.present_overlay(None, None, None, count=0)
        self.clocks = [cc.Clock() for _ in range(n)]
        self.w, self.nl = self.a.geometry()
        self.counts, self.pic_pts, self.last = [0] * n, None, None
        self.calls = self.shorted = self.draws = 0

    def close(self):
        self.a.close()
        self.b.close()

    def clock(self, hdrs, speed, flags, first=0):
        k = len(hdrs)
        self.a.present_clock(np.stack([np.frombuffer(h, dtype=np.uint8) for h in hdrs]), speed, flags, first=first, count=k)
        for i in range(k):
            self.clocks[first + i].set(hdrs[i], np.broadcast_to(speed, (k,))[i], np.broadcast_to(flags, (k,))[i])

    def overlay(self, *a, **kw):
        self.a.present_overlay(*a, **kw)
        self.b.present_overlay(*a, **kw)

    def both(self, fn):
        fn(self.a)
        fn(self.b)

    def submit(self, chunks):
        for c in (self.a, self.b):
            c.submit_ts(*c.pack(chunks))
            c.index()
        self.counts = [self.b.stream_info(s)[0] for s in range(self.n)]
        self.pic_pts, self.last = self.b.picture_pts()

    def _steps(self, pic):
        out = []
        for s, k in enumerate(self.clocks):
            pts = int(self.pic_pts[s, pic]) if 0 <= pic < self.counts[s] else int(self.last[s])
            out.append(k.step(pts))
        return out

    def _commit(self, steps):
        for k, r in zip(self.clocks, steps):
            k.commit(r)
            self.draws += r is not None and r[0] is not None

    def _stage_b(self, steps):
        bm, pr, st = np.zeros((self.n, 1280), np.uint8), np.zeros(self.n, np.int32), np.zeros(self.n, np.uint8)
        for s, r in enumerate(steps):
            if r is not None:
                st[s] = 4 | (1 if r[0] is not None else 0)
                pr[s] = r[1]
                if r[0] is not None:
                    bm[s] = r[0]
        if st.any():
            self.b.present_overlay(bm, None, pr, st)

    def _b_call(self, pic, arg):
        return present_call(self.b, _fn(self.b, pic, arg), device=True)

    def _same(self, info_a, out_a, info_b, out_b):
        assert (info_a == info_b).all(), "info rows differ (call %d)" % self.calls
        total = out_b.shape[0]
        got = out_a[:total * self.w * self.nl].view(total, self.w * self.nl)
        if not torch.equal(got, out_b):
            bad = torch.nonzero((got != out_b).any(1))[:8, 0].tolist()
            raise AssertionError("call %d: fields %s differ" % (self.calls, bad))
        return info_a, got

    def sync(self, pic, arg, sizing=True, enomem=False):
        """one synchronous call on both, A after an optional EF_ENOMEM call and a sizing call -> A's (info, fields)"""
        steps = self._steps(pic)
        fn = _fn(self.a, pic, arg)
        total = int(fn(None)["n_fields"].sum())
        if enomem and total:
            small = torch.empty((total - 1) * self.w * self.nl + 8, dtype=torch.uint16, device="cuda")
            with pytest.raises(espflix_b200.EspflixError) as e:
                fn(small)
            assert e.value.code == capi.EF_ENOMEM
        if sizing:
            fn(None)
        out = torch.empty(max(total, 1) * self.w * self.nl, dtype=torch.uint16, device="cuda")
        info_a = fn(out)
        self._stage_b(steps)
        info_b, out_b = self._b_call(pic, arg)
        r = self._same(info_a, out, info_b, out_b)
        self._commit(steps)
        self.calls += 1
        return r

    def chain(self, calls, short=None):
        """calls [(pic, arg)] as one async chain on A; call `short` (when it has fields) gets a buffer one field short, so that it
        and the calls after it take no effect. B runs the calls that take effect synchronously, after staging. -> (the calls that
        did not take effect, A's (info, fields) of the last call that did)"""
        want, done = [], len(calls)
        for i, (pic, arg) in enumerate(calls):
            if i == short:
                short_cap = int(_fn(self.b, pic, arg)(None)["n_fields"].sum()) - 1
                if short_cap >= 1:                              # a buffer of no fields is no device memory
                    done = i
                    break
            steps = self._steps(pic)
            self._stage_b(steps)
            want.append(self._b_call(pic, arg))
            self._commit(steps)
        outs = []
        st = torch.cuda.current_stream()
        for i, (pic, arg) in enumerate(calls):
            cap = max(want[i][1].shape[0], 1) if i < done else short_cap if i == done else 64
            base = torch.empty(max(cap, 1) * self.w * self.nl, dtype=torch.uint16, device="cuda")
            out = base[:cap * self.w * self.nl]
            info = torch.zeros((self.n, 8), dtype=torch.int32, device="cuda")
            if pic >= 0:
                self.a.present_picture_async(pic, out, info, modes=arg, stream=st)
            else:
                self.a.present_idle_async(arg, out, info, stream=st)
            outs.append((out, info))
        rc, k = self.a.present_wait()
        assert (rc, k) == ((capi.EF_OK, len(calls)) if done == len(calls) else (capi.EF_ENOMEM, done))
        last = None
        for i in range(done):
            last = self._same(self.a.present_info(outs[i][1]), outs[i][0], *want[i])
            self.calls += 1
        self.shorted += done < len(calls)
        return calls[done:], last


def _fn(ctx, pic, arg):
    if pic >= 0:
        return lambda o: ctx.present_picture(pic, arg, o)
    return lambda o: ctx.present_idle(arg, o)


def _programs(ntsc, seed):
    """the irregular schedules of one standard as TS programs, plus a header, speed and flags per stream"""
    rng = np.random.default_rng(seed)
    progs = []
    for case, (pts, nt, fc0, modes, tail) in enumerate(irregular_cases()):
        if nt == ntsc:
            progs.append(dict(ts=oc.segment_ts(300 + case, [int(v) for v in pts]), modes=[int(m) for m in modes], fc0=fc0, tail=tail + 1,
                              hdr=_header(rng, int(pts[0]))))
    return progs, rng


def _chunks(progs, rng, cut):
    if not cut:
        return [[p["ts"] for p in progs]]
    K = int(rng.integers(2, 4))
    per = []
    for p in progs:
        cand = pts_cases.cut_points(p["ts"])
        per.append(carry_cases.cut(p["ts"], sorted(rng.choice(cand, size=K - 1, replace=True).tolist()) if cand else []))
    return submits(per, n=K)


def _run(ntsc, seed, cut, async_p):
    progs, rng = _programs(ntsc, seed)
    n = len(progs)
    pair = Pair(n, ntsc, [p["fc0"] for p in progs])
    on = (rng.random(n) < 0.8).astype(np.uint8)
    pair.clock([p["hdr"] for p in progs], rng.integers(-1, 2, size=n), on | (rng.integers(0, 2, size=n) << 1).astype(np.uint8))
    pair.overlay(None, rng.integers(-1, 60, size=n).astype(np.int32), None, set=np.full(n, 2, np.uint8))
    k = [0] * n
    for ci, chunk in enumerate(_chunks(progs, rng, cut)):
        pair.submit(chunk)
        calls = []
        for p in range(max(pair.counts)):
            modes = np.array([progs[s]["modes"][k[s] + p] if p < pair.counts[s] else 0 for s in range(n)], np.uint8)
            calls.append((p, modes))
            if rng.random() < 0.25:
                calls.append((-1, rng.integers(0, 3, size=n).astype(np.uint32)))
        k = [a + b for a, b in zip(k, pair.counts)]
        i = 0
        while i < len(calls):
            r = rng.random()
            if r < 0.2:                                         # host changes between calls: blend, sometimes a bitmap and progress
                m = rng.random(n) < 0.5
                pair.overlay(rng.integers(0, 256, size=(n, 1280)).astype(np.uint8), rng.integers(-1, 50, size=n).astype(np.int32),
                             rng.integers(-5, 250, size=n).astype(np.int32), set=np.where(m, 7, 2).astype(np.uint8))
            if r > 0.9:                                          # pause with _last_seconds zeroed, or a new header and speed
                s = int(rng.integers(0, n))
                pair.clock([progs[s]["hdr"] if rng.random() < 0.5 else _header(rng, int(pair.last[s]) if pair.last[s] >= 0 else 0)],
                           int(rng.integers(-1, 2)), int(1 | (rng.integers(0, 2) << 1) | (rng.integers(0, 2) << 2)), first=s)
            if rng.random() < async_p:
                j = min(len(calls), i + int(rng.integers(1, 5)))
                short = 1 + int(rng.integers(0, j - i - 1)) if j - i >= 2 and rng.random() < 0.5 else None
                rest, _ = pair.chain(calls[i:j], short)
                for pic, arg in rest:                           # the retry, synchronously
                    pair.sync(pic, arg)
                i = j
            else:
                pair.sync(*calls[i], sizing=rng.random() < 0.7, enomem=rng.random() < 0.2)
                i += 1
        if ci == 0 and cut:                                     # restarts between submits: op 1 on some streams, op 2 on others
            ops = rng.integers(0, 3, size=n).astype(np.uint8)
            pair.both(lambda c: c.restart_streams(ops))
    pair.sync(-1, np.array([p["tail"] for p in progs], np.uint32))
    pair.both(lambda c: c.reset())
    pair.clock([p["hdr"] for p in progs], 0, 1 | 4)
    pair.submit([oc.segment_ts(700 + s, [900000 + 3003 * 7 * j for j in range(3 + s % 3)]) for s in range(n)])
    calls = [(p, None) for p in range(max(pair.counts))] + [(-1, np.full(n, 2, np.uint32)), (-1, np.full(n, 1, np.uint32))]
    rest, _ = pair.chain(calls, short=1)
    for pic, arg in rest:                                       # the retry, as a chain
        pair.chain([(pic, arg)])
    assert pair.shorted >= 1 and pair.draws >= n
    pair.close()


@pytest.mark.parametrize("ntsc", [1, 0])
def test_irregular_schedules_whole(ntsc):
    _run(ntsc, 10 + ntsc, cut=False, async_p=0.0)


@pytest.mark.parametrize("ntsc", [1, 0])
def test_irregular_schedules_cut_sync_async_mixed(ntsc):
    for seed in (20, 21):
        _run(ntsc, seed + 2 * ntsc, cut=True, async_p=0.5)


@pytest.mark.parametrize("ntsc", [1, 0])
def test_pinned_overlay_cases_with_host_changes(ntsc):
    """the pinned overlay cases' programs with their own overlay changes staged by the host between calls, the clock on every
    stream, and ef_reset before a later segment"""
    cases = [c for _, c in sorted(oc.cases().items()) if c["ntsc"] == ntsc]
    n = len(cases)
    rng = np.random.default_rng(5 + ntsc)
    pair = Pair(n, ntsc, [c["fc0"] for c in cases])
    pair.clock([_header(rng, c["segments"][0][1][0]) for c in cases], [0, 1, -1, 0, 1][:n], [1, 1, 1, 3, 1][:n])
    k = [0] * n
    for si in range(max(len(c["segments"]) for c in cases)):
        if si:
            pair.both(lambda c: c.reset())
        segs = [c["segments"][si] if si < len(c["segments"]) else None for c in cases]
        pair.submit([oc.segment_ts(*sg) if sg else b"" for sg in segs])
        for p in range(max(pair.counts)):
            pair.overlay(*overlay_arrays([c["cmds"][k[s] + p] if p < pair.counts[s] else None for s, c in enumerate(cases)]))
            modes = np.array([c["modes"][k[s] + p] if p < pair.counts[s] else 0 for s, c in enumerate(cases)], np.uint8)
            pair.sync(p, modes)
        k = [a + b for a, b in zip(k, pair.counts)]
    for t in range(12):
        if t in (2, 7):
            pair.overlay(None, [9, -1, 0, 31, 4][:n], None, set=np.full(n, 2, np.uint8))
        pair.sync(-1, np.full(n, 1 + t % 3, np.uint32))
    pair.close()


# ---- the benchmark's batch size ------------------------------------------------------------------------------------------------
def test_batch_scale_clock_on_a_subset():
    """4,096 TS streams x 12 pictures (tests/scale_cases.py): clocks on a seeded subset, off on the rest. Every stream of A equals
    B, and the streams whose clock is off equal a context that never set a clock"""
    from tests.scale_cases import N, PICTURES
    b = scale_cases.batch()
    blob, off = espflix_b200.Context.pack(b.all_ts())
    rng = np.random.default_rng(31)
    on = rng.random(N) < 0.6
    hdrs = [_header(rng, b.pts[s % scale_cases.D][0]) for s in range(N)]
    for ntsc in (1, 0):
        fc0 = [b.fc0(s) for s in range(N)]
        pair = Pair(N, ntsc, fc0, max_pictures=PICTURES, es_capacity=int(off[-1]) + 4096)
        plain = _ctx(N, ntsc, fc0, font=False, max_pictures=PICTURES, es_capacity=int(off[-1]) + 4096)
        pair.clock(hdrs, rng.integers(-1, 2, size=N), np.where(on, 1 | (rng.integers(0, 2, size=N) << 1), 0).astype(np.uint8))
        pair.overlay(None, np.where(on, 180, 0).astype(np.int32), None, set=np.full(N, 2, np.uint8))
        pair.submit(b.all_ts())
        plain.submit_ts(blob, off)
        plain.index()
        off_streams = torch.as_tensor(np.nonzero(~on)[0], device="cuda")
        calls = [(p, np.array([b.modes(s)[p] for s in range(N)], np.uint8)) for p in range(PICTURES)]
        calls.append((-1, np.array([scale_cases.idle_fields(s % scale_cases.D) for s in range(N)], np.uint32)))
        for i, (pic, arg) in enumerate(calls):
            if i % 4 == 3:
                _, (info_a, out_a) = pair.chain([(pic, arg)])
            else:
                info_a, out_a = pair.sync(pic, arg, sizing=False)
            info_p, out_p = present_call(plain, _fn(plain, pic, arg), device=True)
            assert (info_a == info_p).all()
            first = torch.as_tensor(info_p["first"].astype(np.int64), device="cuda")
            nf = torch.as_tensor(info_p["n_fields"].astype(np.int64), device="cuda")
            sel = torch.repeat_interleave(first[off_streams], nf[off_streams]) + (
                torch.arange(int(nf[off_streams].sum()), device="cuda") - torch.repeat_interleave(torch.cumsum(nf[off_streams], 0) - nf[off_streams], nf[off_streams]))
            assert torch.equal(out_a.view(torch.int16)[sel], out_p.view(torch.int16)[sel]), "call %d: a stream whose clock is off differs from the clock-free context" % i
            del info_a, out_a, info_p, out_p, sel
        assert int(on.sum()) and int((~on).sum())
        pair.close()
        plain.close()
        torch.cuda.empty_cache()


# ---- launches and errors -------------------------------------------------------------------------------------------------------
def test_launch_counts():
    """a context that loads a font but never sets a clock launches what an overlay context launches; a clock context adds the
    clock kernel to every call (sizing calls too) and its commit to every call that takes effect"""
    progs = [oc.segment_ts(90 + s, [129003 + 9009 * k for k in range(4)]) for s in range(3)]
    ctxs = [_ctx(3, 1, 1, font=False), _ctx(3, 1, 1), _ctx(3, 1, 1)]
    for c in ctxs:
        c.present_overlay(None, 40, None, set=[2, 2, 2])
    ctxs[2].present_clock(np.frombuffer(cc.H_MAIN, dtype=np.uint8), 0, [1, 0, 3])
    w, nl = ctxs[0].geometry()
    for c in ctxs:
        c.submit_ts(*c.pack(progs))
        c.index()
    for p in range(4):
        d = []
        for c in ctxs:
            n0 = c.launch_count()
            total = int(c.present_picture(p, None, None)["n_fields"].sum())
            n1 = c.launch_count()
            if p == 1:
                assert total > 1
                small = torch.empty(max(total - 1, 0) * w * nl + 8, dtype=torch.uint16, device="cuda")
                with pytest.raises(espflix_b200.EspflixError):
                    c.present_picture(p, None, small)
            n2 = c.launch_count()
            out = torch.empty(max(total, 1) * w * nl, dtype=torch.uint16, device="cuda")
            if p == 3:
                c.present_picture_async(p, out)
                assert c.present_wait() == (capi.EF_OK, 1)
            else:
                c.present_picture(p, None, out)
            d.append((n1 - n0, n2 - n1, c.launch_count() - n2))
        assert d[0] == d[1], d
        assert d[2] == (d[0][0] + 1, d[0][1] + (1 if p == 1 else 0), d[0][2] + 2), d
    for c in ctxs:
        c.close()


def test_error_codes():
    ctx = espflix_b200.Context(n_streams=3, max_pictures=4, fields=False)
    h = np.frombuffer(cc.H_MAIN, dtype=np.uint8)
    assert error_code(lambda: ctx.present_clock(h, 0, 1)) == capi.EF_ESTATE                # before ef_present_enable
    ctx.enable_pts()
    ctx.enable_present()
    assert error_code(lambda: ctx.present_clock(h, 0, 1)) == capi.EF_ESTATE                # before ef_present_font
    assert error_code(lambda: ctx.present_font(ATLAS, RIGHTS[:34])) == capi.EF_EINVAL      # does not reach ':'
    bad = RIGHTS.copy()
    bad[5] = bad[4]
    assert error_code(lambda: ctx.present_font(ATLAS, bad)) == capi.EF_EINVAL              # not increasing
    bad = RIGHTS.copy()
    bad[-1] = 1025
    assert error_code(lambda: ctx.present_font(ATLAS, bad)) == capi.EF_EINVAL              # past the atlas
    with pytest.raises(ValueError):
        ctx.present_font(ATLAS[:, :512], RIGHTS)
    ctx.present_font(ATLAS, RIGHTS)
    assert error_code(lambda: ctx.present_clock(h, 0, 1, first=-1, count=1)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.present_clock(h, 0, 1, first=2, count=2)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.present_clock(h, 2, 1)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.present_clock(h, -2, 0)) == capi.EF_EINVAL               # checked on streams that stay off too
    zero_last = cc.header((5, 0), (0, 10), (0, 10))
    flat_fwd = cc.header((5, 100), (7, 7), (0, 10))
    flat_rwd = cc.header((5, 100), (0, 10), (-3, -3))
    for hdr, speed in ((zero_last, 0), (flat_fwd, 1), (flat_rwd, -1)):
        a = np.frombuffer(hdr, dtype=np.uint8)
        assert error_code(lambda: ctx.present_clock(a, speed, 1)) == capi.EF_EINVAL
        ctx.present_clock(a, speed, 0)                                                # off: the header is not read
    ctx.present_clock(np.frombuffer(flat_fwd, dtype=np.uint8), -1, 1)                 # the flat record is not the one used
    ctx.present_clock(np.frombuffer(flat_rwd, dtype=np.uint8), 1, 1)
    ctx.present_clock(h, 0, 7, first=3, count=0)
    ctx.close()
