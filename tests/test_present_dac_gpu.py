"""EF_FIELD_DAC8 (ef_present_format) on the GPU: a U16 context and a DAC8 context get the same submits and the same calls in
lockstep. Every DAC8 field must equal tests/dac_cases.py's conversion of its twin's field, and every info row, every return
code and every call's launch count must be identical. The U16 side is held to the reference's pins by the other presentation
tests. Each case runs in both standards, synchronously and asynchronously, with and without the overlay: all eight DAC8
instantiations of the paced K2."""
import json
import os

import numpy as np
import pytest
import torch

import espflix_b200
from espflix_b200 import capi
from tests import clock_cases as cc, dac_cases, present_cases as pc, pts_cases, scale_cases
from tests.harness import error_code, host_fields

pytestmark = pytest.mark.gpu
PINS = json.load(open(os.path.join(pts_cases.GOLDEN, "pacing_pins.json")))
INFO_FIELDS = ("first", "n_fields", "frame_counter", "flip_field", "flip_line", "flags")
SENTINEL = 0x5A
ATLAS, RIGHTS = cc.font()


def dac8_on_device(u16):
    """dac_cases.dac8 of a CUDA uint16 tensor, on the device: a pair of samples is the bytes lo0 hi0 lo1 hi1, and plays hi1 hi0"""
    return u16.view(torch.int16).view(torch.uint8).view(-1, 4)[:, [3, 1]].reshape(-1)


def make(n, ntsc, fc0, fmt, font=False, max_pictures=13, es_capacity=None):
    """a presenting context; the U16 twin never calls ef_present_format"""
    ctx = espflix_b200.Context(n_streams=n, max_pictures=max_pictures, max_slices_per_picture=12,
                               es_capacity=es_capacity or n * max_pictures * 40000, fields=False)
    ctx.enable_pts()
    ctx.video_init(ntsc)
    if fmt != capi.EF_FIELD_U16:
        ctx.present_format(fmt)
    ctx.enable_present(fc0)
    if font:
        ctx.present_font(ATLAS, RIGHTS)
    return ctx


def same_info(a, b, what):
    for f in INFO_FIELDS:
        assert np.array_equal(a[f], b[f]), "%s: info %s" % (what, f)


class Twins:
    """a U16 and a DAC8 context driven through the same calls"""

    def __init__(self, n, ntsc, fc0, device=False, **kw):
        self.u = make(n, ntsc, fc0, capi.EF_FIELD_U16, **kw)
        self.d = make(n, ntsc, fc0, capi.EF_FIELD_DAC8, **kw)
        w, nl = self.u.geometry()
        self.S = w * nl                                  # samples of a field: DAC8 bytes
        assert self.S == dac_cases.FIELD_BYTES[ntsc]
        self.device = device                             # compare on the device (batch scale) instead of on the host
        self.fields = 0

    def close(self):
        self.u.close()
        self.d.close()

    def both(self, fn):
        fn(self.u)
        fn(self.d)

    def submit(self, chunk):
        for c in (self.u, self.d):
            c.submit_ts(*c.pack(chunk))
            c.index()
        return self.u.index_info()["max_pictures"], [self.u.stream_info(s)[0] for s in range(self.u.n_streams)]

    @staticmethod
    def _counted(c, fn):
        n0 = c.launch_count()
        r = fn()
        return r, c.launch_count() - n0

    def same_fields(self, bu, bd, k, what):
        """the first k fields of the U16 buffer bu, converted, equal those of the DAC8 buffer bd"""
        if not k:
            return
        n = k * self.S
        if self.device:
            assert torch.equal(dac8_on_device(bu[:n]), bd[:n]), what
        else:
            want = dac_cases.dac8(host_fields(bu[:n].view(k, self.S)))
            got = bd[:n].view(k, self.S).cpu().numpy()
            bad = np.nonzero((want != got).any(axis=1))[0]
            assert bad.size == 0, "%s: fields %s differ from the conversion of the U16 twin's" % (what, bad[:8].tolist())
        self.fields += k

    def sync(self, fn, what, enomem=False):
        """fn(ctx, out): one synchronous present call on both - the sizing call, with enomem a call one field short (EF_ENOMEM),
        then the call into buffers of exactly that size -> info"""
        (iu, lu), (idd, ld) = self._counted(self.u, lambda: fn(self.u, None)), self._counted(self.d, lambda: fn(self.d, None))
        same_info(iu, idd, what + " sizing")
        assert lu == ld, (what, lu, ld)
        total = int(iu["n_fields"].sum())
        if enomem and total:
            short = {self.u: torch.empty((total - 1) * self.S + 8, dtype=torch.uint16, device="cuda"),
                     self.d: torch.empty((total - 1) * self.S + 8, dtype=torch.uint8, device="cuda")}
            got = [self._counted(c, lambda: error_code(lambda: fn(c, short[c]))) for c in (self.u, self.d)]
            assert got[0] == got[1] and got[0][0] == capi.EF_ENOMEM, (what, got)
        bu = torch.empty(max(total, 1) * self.S, dtype=torch.uint16, device="cuda")
        bd = torch.empty(max(total, 1) * self.S, dtype=torch.uint8, device="cuda")
        (gu, lu), (gd, ld) = self._counted(self.u, lambda: fn(self.u, bu)), self._counted(self.d, lambda: fn(self.d, bd))
        assert (gu == iu).all() and (gd == idd).all(), what      # the sizing call reported what the call did
        assert lu == ld, (what, lu, ld)
        self.same_fields(bu, bd, total, what)
        return gu

    def chain(self, calls, caps, what):
        """calls[i](ctx, out): asynchronous present calls, each into its own sentinel-filled buffer of caps[i] fields, then one
        ef_present_wait on each twin -> (rc, calls that took effect, info rows)"""
        bufs, infos = {self.u: [], self.d: []}, {self.u: [], self.d: []}
        for i, (fn, cap) in enumerate(zip(calls, caps)):
            n = max(cap * self.S, 8)
            bu = torch.full((n,), SENTINEL * 0x101, dtype=torch.int16, device="cuda").view(torch.uint16)
            bd = torch.full((n,), SENTINEL, dtype=torch.uint8, device="cuda")
            launches = []
            for c, b in ((self.u, bu), (self.d, bd)):
                info, k = self._counted(c, lambda: fn(c, b))
                bufs[c].append(b)
                infos[c].append(info)
                launches.append(k)
            assert launches[0] == launches[1], (what, i, launches)
        (ru, ku), (rd, kd) = self.u.present_wait(), self.d.present_wait()
        assert (ru, ku) == (rd, kd), what
        rows = []
        for i, cap in enumerate(caps):
            iu, idd = self.u.present_info(infos[self.u][i]), self.d.present_info(infos[self.d][i])
            same_info(iu, idd, "%s call %d" % (what, i))
            bu, bd = bufs[self.u][i], bufs[self.d][i]
            if i < ku:
                self.same_fields(bu, bd, cap, "%s call %d" % (what, i))                  # slots past the call's fields: both untouched
            else:
                assert bool((bu.view(torch.int16) == SENTINEL * 0x101).all()) and bool((bd == SENTINEL).all()), "%s call %d wrote dst" % (what, i)
            rows.append(iu)
        return ru, ku, rows


def picture(p, modes=None):
    return lambda c, o: c.present_picture(p, modes, o)


def idle(nf):
    return lambda c, o: c.present_idle(nf, o)


def picture_async(p, modes=None):
    return lambda c, o: c.present_picture_async(p, o, modes=modes)


def idle_async(nf):
    return lambda c, o: c.present_idle_async(nf, o)


# ---- the pinned schedules, idle tails, poster scroll, sizing calls and EF_ENOMEM ----------------------------------------------
@pytest.mark.parametrize("ntsc", [1, 0])
def test_pinned_schedules(ntsc):
    """present_cases' pinned schedules of one standard with two filler streams, one scrolling a poster left (mode 2) and one
    right (mode 3), then the idle tails; every third call is first tried one field short"""
    names = [n for n in sorted(PINS) if PINS[n]["ntsc"] == ntsc]
    ts = [pc.synth_ts(PINS[n]["seed"], PINS[n]["pictures"]) for n in names] + [pc.synth_ts(60 + ntsc, 7), pc.synth_ts(62 + ntsc, 12)]
    fc0 = [PINS[n]["frame_counter0"] for n in names] + [3, 100]
    t = Twins(len(ts), ntsc, fc0)
    npics, counts = t.submit([np.frombuffer(bytes(x), dtype=np.uint8) for x in ts])
    k = len(names)
    emitted = [0] * len(ts)
    for p in range(npics):
        modes = np.array([PINS[names[s]]["modes"][p] if s < k and p < counts[s] else 0 for s in range(len(ts))], dtype=np.uint8)
        modes[k] = 2 if p == 4 else 0
        modes[k + 1] = 3 if p == 6 else 0
        info = t.sync(picture(p, modes), "picture %d" % p, enomem=p % 3 == 1)
        emitted = [a + int(b) for a, b in zip(emitted, info["n_fields"])]
    tails = [((PINS[n]["flip_field"][-1] + 1 + PINS[n]["tail_fields"] - PINS[n]["frame_counter0"]) & pc.M32) - emitted[i] for i, n in enumerate(names)]
    t.sync(idle(np.array(tails + [5, 0], dtype=np.uint32)), "idle tail", enomem=True)
    t.sync(idle(np.array([1] * len(ts), dtype=np.uint32)), "idle")
    assert t.fields > 0
    t.close()


# ---- overlay with fade and progress, the clock, ef_reset ---------------------------------------------------------------------
@pytest.mark.parametrize("ntsc", [1, 0])
def test_overlay_clock_and_reset(ntsc):
    """overlay bitmaps with a fading, a full-strength and a short blend and their progress bars, a clock on two streams, changes
    staged between calls; the first submit synchronous, then ef_reset (which keeps the format) and a second submit as one async
    chain"""
    n = 3
    rng = np.random.RandomState(40 + ntsc)
    t = Twins(n, ntsc, [0, 5, 9], font=True)
    bm = rng.randint(0, 256, size=(n, 1280)).astype(np.uint8)
    t.both(lambda c: c.present_overlay(bm, blend=[20, -1, 5], progress=[50, 240, 0]))
    t.both(lambda c: c.present_clock(np.frombuffer(cc.H_MAIN, dtype=np.uint8), 0, [0, 1, 3]))
    subs = [[np.frombuffer(bytes(pc.synth_ts(150 + 3 * k + s, 5 + s)), dtype=np.uint8) for s in range(n)] for k in range(2)]
    npics, _ = t.submit(subs[0])
    for p in range(npics):
        if p == 2:
            t.both(lambda c: c.present_overlay(blend=[31, 0, 12], progress=[10, 120, 239], set=[6, 2, 6]))
        t.sync(picture(p), "submit 0 picture %d" % p, enomem=p == 3)
    t.sync(idle(np.array([2, 1, 3], dtype=np.uint32)), "submit 0 idle")
    t.both(lambda c: c.reset())
    npics, _ = t.submit(subs[1])
    t.both(lambda c: c.present_overlay(bm[::-1].copy(), blend=[25, 8, -1], progress=[200, 0, 90]))
    calls = [picture_async(p) for p in range(npics)] + [idle_async(np.array([4, 2, 1], dtype=np.uint32))]
    ref = make(n, ntsc, [0, 5, 9], capi.EF_FIELD_U16, font=True)                     # the chain's capacities, from a third run
    caps = _caps(ref, subs, lambda c: (c.present_overlay(bm, blend=[20, -1, 5], progress=[50, 240, 0]),
                                       c.present_clock(np.frombuffer(cc.H_MAIN, dtype=np.uint8), 0, [0, 1, 3])),
                 {(0, 2): lambda c: c.present_overlay(blend=[31, 0, 12], progress=[10, 120, 239], set=[6, 2, 6]),
                  (1, 0): lambda c: c.present_overlay(bm[::-1].copy(), blend=[25, 8, -1], progress=[200, 0, 90])},
                 [np.array([2, 1, 3], dtype=np.uint32), np.array([4, 2, 1], dtype=np.uint32)])[1]
    ref.close()
    rc, k, _ = t.chain(calls, [c + 1 for c in caps], "submit 1")
    assert rc == capi.EF_OK and k == len(calls)
    t.close()


def _caps(ctx, subs, setup, hooks, idles, modes=None):
    """the fields of every call of every submit on a synchronous U16 context -> per submit, a list with one entry per call.
    hooks[(submit, picture)](ctx) runs before that call, modes[(submit, picture)] are its modes; every submit ends with an idle
    call of idles[submit]; ef_reset between submits"""
    setup(ctx)
    out = []
    for k, chunk in enumerate(subs):
        if k:
            ctx.reset()
        ctx.submit_ts(*ctx.pack(chunk))
        ctx.index()
        w, nl = ctx.geometry()
        caps = []
        for p in range(ctx.index_info()["max_pictures"]):
            if (k, p) in hooks:
                hooks[(k, p)](ctx)
            md = (modes or {}).get((k, p))
            total = int(ctx.present_picture(p, md)["n_fields"].sum())
            ctx.present_picture(p, md, torch.empty(max(total, 1) * w * nl, dtype=torch.uint16, device="cuda"))
            caps.append(total)
        total = int(ctx.present_idle(idles[k])["n_fields"].sum())
        ctx.present_idle(idles[k], torch.empty(max(total, 1) * w * nl, dtype=torch.uint16, device="cuda"))
        caps.append(total)
        out.append(caps)
    return out


# ---- an async chain with a call one field short, its retry, and the calls behind it ------------------------------------------
@pytest.mark.parametrize("ntsc", [1, 0])
@pytest.mark.parametrize("overlay", [False, True])
def test_short_call_in_a_chain_and_retry(ntsc, overlay):
    n = 3
    ts = [pc.synth_ts(120 + i, m) for i, m in enumerate((7, 6, 7))]
    chunk = [np.frombuffer(bytes(x), dtype=np.uint8) for x in ts]
    modes = np.array([0, 3, 2], dtype=np.uint8)
    nf = np.array([2, 3, 4], dtype=np.uint32)
    bm = np.random.RandomState(7).randint(0, 256, size=(n, 1280)).astype(np.uint8)

    def setup(c):
        if overlay:
            c.present_overlay(bm, blend=[30, -1, 3], progress=[100, 7, 240])
    ref = make(n, ntsc, [5, 6, 7], capi.EF_FIELD_U16, max_pictures=8)
    caps = _caps(ref, [chunk], setup, {}, [nf], {(0, 2): modes})[0]
    ref.close()
    t = Twins(n, ntsc, [5, 6, 7], max_pictures=8)
    t.both(setup)
    npics, _ = t.submit(chunk)
    assert npics == 7 and len(caps) == 8
    calls = [picture_async(p, modes if p == 2 else None) for p in range(npics)] + [idle_async(nf)]
    bad = 4
    assert caps[bad] > 0
    short = list(caps)
    short[bad] -= 1
    rc, k, rows = t.chain(calls, short, "short chain")
    assert rc == capi.EF_ENOMEM and k == bad
    assert (rows[bad]["flags"] & 2).all() and int(rows[bad]["n_fields"].sum()) == caps[bad]
    for r in rows[bad + 1:]:
        assert (r["flags"] & 2).all() and (r["n_fields"] == 0).all()
    rc, k, rows = t.chain(calls[bad:], caps[bad:], "retry")
    assert rc == capi.EF_OK and k == len(calls) - bad
    t.close()


# ---- errors ------------------------------------------------------------------------------------------------------------------
def test_format_rules():
    ctx = espflix_b200.Context(n_streams=2, max_pictures=5, fields=False)
    assert ctx.lib.ef_present_format(None, capi.EF_FIELD_DAC8) == capi.EF_EINVAL
    for bad in (2, -1, 256):
        assert error_code(lambda: ctx.present_format(bad)) == capi.EF_EINVAL
    ctx.present_format(capi.EF_FIELD_DAC8)                                          # before ef_pts_enable / ef_video_init too
    ctx.present_format(capi.EF_FIELD_U16)
    ctx.present_format(capi.EF_FIELD_DAC8)
    ctx.enable_pts()
    ctx.video_init(1)
    ctx.enable_present([1, 2])
    for fmt in (capi.EF_FIELD_DAC8, capi.EF_FIELD_U16):
        assert error_code(lambda: ctx.present_format(fmt)) == capi.EF_ESTATE
    assert error_code(lambda: ctx.present_format(9)) == capi.EF_EINVAL
    ctx.reset()
    assert error_code(lambda: ctx.present_format(capi.EF_FIELD_U16)) == capi.EF_ESTATE
    ts = [pc.synth_ts(70 + i, m) for i, m in enumerate((3, 2))]
    ctx.submit_ts(*ctx.pack(ts))
    ctx.index()
    w, nl = ctx.geometry()
    wide = torch.zeros(4 * w * nl, dtype=torch.uint16, device="cuda")
    nf = np.ones(2, dtype=np.uint32)
    with pytest.raises(TypeError):
        ctx.present_picture(0, None, wide)
    with pytest.raises(TypeError):
        ctx.present_idle(nf, wide)
    with pytest.raises(TypeError):
        ctx.present_picture_async(0, wide)
    with pytest.raises(TypeError):
        ctx.present_idle_async(nf, wide)
    with pytest.raises(TypeError):
        ctx.present_picture(0, None, torch.zeros(4 * w * nl, dtype=torch.uint8))   # host memory
    assert ctx.present_wait() == (capi.EF_OK, 0)                                    # nothing was enqueued
    out = torch.zeros(4 * w * nl, dtype=torch.uint8, device="cuda")
    ctx.present_picture(0, None, out)                                               # picture 0 was not consumed by the rejections
    ctx.close()


# ---- the benchmark's batch size ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ntsc", [1, 0])
def test_batch_step(ntsc):
    """a full step of the 4,096-stream batch (12 pictures and an idle tail), compared call by call on the device"""
    b = scale_cases.batch()
    n = scale_cases.N
    blob, off = espflix_b200.Context.pack(b.all_ts())
    t = Twins(n, ntsc, [b.fc0(s) for s in range(n)], device=True, max_pictures=12, es_capacity=int(off[-1]) + 4096)
    for c in (t.u, t.d):
        c.submit_ts(blob, off)
        c.index()
    for p in range(12):
        t.sync(picture(p, np.array([b.modes(s)[p] for s in range(n)], dtype=np.uint8)), "picture %d" % p)
        torch.cuda.empty_cache()
    t.sync(idle(np.array([scale_cases.idle_fields(s % scale_cases.D) for s in range(n)], dtype=np.uint32)), "idle")
    assert t.fields > 12 * n
    t.close()
    torch.cuda.empty_cache()
