"""The remote (ef_library_keys) on the GPU. A keys-driven context runs seeded per-stream key scripts beside a twin driven by
ef_library_command per stream, with the ef_present_overlay blends and ef_present_clock states tests/keys_cases.py's restatement names:
every paced field, info row, ef_library_info row and saved position must be equal, and every done code must be the restatement's.
Also: keys from a device producer with no host wait before the async present chain, restarts with a submit queued and with audio,
4,096 streams over 64 titles, the error cases and the launches per call."""
import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import clock_cases
from tests import keys_cases as kc
from tests import nav_cases as nc
from tests import restart_cases
from tests.harness import error_code, host_fields, sha

pytestmark = pytest.mark.gpu
MAX_CARRY = 1 << 17
KEY_CHOICES = np.array([0, 0, 99] + list(kc.KEYS) * 2, np.uint8)


def _picture(seed):
    """a smooth seeded 352 x 192 I420 picture (a poster at quantiser 2)"""
    rng = np.random.default_rng(seed)
    y = np.clip(np.add.outer(np.arange(192) * rng.uniform(0.1, 0.6), np.arange(352) * rng.uniform(0.1, 0.4)) + rng.integers(16, 90), 0, 235).astype(np.uint8)
    return np.concatenate([y.reshape(-1), np.full(2 * 96 * 176, int(rng.integers(64, 192)), np.uint8)])


def _title(seed, audio=False):
    """a synthetic title with trick files and a poster: (idx, main, fwd, rwd, poster)"""
    P = 6 * 3003
    au = (lambda j: dict(seed=seed * 10 + j, frames=40)) if audio else (lambda j: None)
    main = b"".join(restart_cases.program(seed * 10 + j, 6, 90000 + j * P, audio=au(j)) for j in range(2))
    fwd = b"".join(restart_cases.program(seed * 10 + 5 + j, 3, 90000 + j * P) for j in range(2))
    rwd = b"".join(restart_cases.program(seed * 10 + 7 + j, 3, 90000 + j * P) for j in range(2))
    return capi.build_video_idx(main, fwd, rwd), main, fwd, rwd, capi.encode_poster(_picture(seed))


@pytest.fixture(scope="module")
def titles():
    return [_title(s) for s in range(1, 4)]


def _context(n, titles, cap, ntsc=None, dac8=False, clock=False, audio=False):
    ctx = espflix_b200.Context(n_streams=n, max_pictures=40, max_slices_per_picture=12, es_capacity=cap, fields=False)
    ctx.enable_pts()
    ctx.enable_carry(MAX_CARRY)
    if audio:
        ctx.enable_audio()
    for k, (idx, m, f, r, p) in enumerate(titles):
        assert ctx.library_add(idx, m, f, r) == k
        ctx.library_add_poster(k, p)
    if ntsc is not None:
        ctx.video_init(ntsc)
        if dac8:
            ctx.present_format(capi.EF_FIELD_DAC8)
        ctx.enable_present()
        bm = np.random.default_rng(n).integers(0, 256, (n, 1280)).astype(np.uint8)
        ctx.present_overlay(bm, np.full(n, 180, np.int32), np.full(n, 100, np.int32))
        if clock:
            ctx.present_font(*clock_cases.font())
    return ctx


def _done_tensor(n):
    import torch
    return torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")


class Twins:
    """the keys-driven context, its command-driven twin and the restatement, driven together"""

    def __init__(self, n, titles, budget_max, ntsc=None, dac8=False, clock=False, audio=False):
        self.n, self.paced, self.dac8, self.clock, self.audio = n, ntsc is not None, dac8, clock, audio
        cap = max(n * budget_max * 188, 1 << 20)
        self.lib, self.twin = (_context(n, titles, cap, ntsc, dac8, clock, audio) for _ in range(2))
        self.titles = [nc.Title(idx, m, f, r, p) for idx, m, f, r, p in titles]
        self.st = [kc.Stream() for _ in range(n)]
        self.nv = nc.new_nv(len(titles), n)
        self.last = np.full(n, -1, np.int64)
        for s in range(n):
            for ctx in (self.lib, self.twin):
                ctx.library_command(nc.NAV, s, 1, s % len(titles))
            self.st[s].command(self.titles, nc.NAV, s % len(titles), nv=self.nv, s=s)
        if clock:
            for ctx in (self.lib, self.twin):
                ctx.present_clock(self._hdrs(), 0, 1)

    def _hdrs(self):
        return np.stack([np.frombuffer(self.titles[st.title].idx[:104], np.uint8) for st in self.st])

    def keys(self, keys):
        """one ef_library_keys on the keys context; the commands, blends and clock states the restatement names on the twin"""
        done = _done_tensor(self.n)
        self.lib.library_keys(keys, done)
        blend, setb, zero = np.zeros(self.n, np.int32), np.zeros(self.n, np.uint8), np.zeros(self.n, np.uint8)
        want = []
        for s, st in enumerate(self.st):
            r = st.key(self.titles, int(keys[s]), int(self.last[s]), nv=self.nv, s=s)
            want.append(r["done"])
            if r["done"] & kc.ENDED_BIT:
                self.twin.library_command(nc.MENU, s)
            cmd, k = r["done"] & 0xF, int(keys[s])
            if cmd != kc.NOTHING:
                sign = 1 if k in (kc.KEY_RIGHT, kc.KEY_UP) else -1
                self.twin.library_command(cmd, s, 1, 0, sign if cmd == nc.NAV_STEP else 30 * sign if cmd == nc.SKIP else 0)
            if r["blend"] is not None:
                blend[s], setb[s] = r["blend"], 2
            zero[s] = r["zero"]
        if self.paced and setb.any():
            self.twin.present_overlay(blend=blend, set=setb)
        if self.clock:
            flags = 1 | np.array([2 * (st.state == nc.PAUSED) for st in self.st], np.uint8) | 4 * zero
            self.twin.present_clock(self._hdrs(), np.array([st.speed for st in self.st], np.int8), flags)
        assert done.cpu().numpy().tolist() == want
        return want

    def submit(self, budgets):
        """a library submit on both; every picture presented (or decoded) on both and compared"""
        for s, st in enumerate(self.st):
            st.submit(self.titles, int(budgets[s]))
        k = [ctx.launch_count() for ctx in (self.lib, self.twin)]
        for ctx in (self.lib, self.twin):
            ctx.library_submit(per_stream=budgets)
            ctx.index()
        assert self.lib.launch_count() - k[0] == self.twin.launch_count() - k[1]
        pic, last = self.lib.picture_pts()
        pic2, last2 = self.twin.picture_pts()
        assert (pic == pic2).all() and (last == last2).all()
        if self.paced:
            for p in range(self.lib.index_info()["max_pictures"]):
                self._present(lambda ctx, o: ctx.present_picture(p, None, o))
            self._present(lambda ctx, o: ctx.present_idle(np.full(self.n, 3, np.uint32), o))
        else:
            m = self.lib.index_info()["max_pictures"]
            for ctx in (self.lib, self.twin):
                ctx.decode_all(m)
            assert sha(self.lib.read_latest_i420()) == sha(self.twin.read_latest_i420())
        if self.audio:
            a, b = self.lib.decode_audio(), self.twin.decode_audio()
            for x, y in zip(a, b):
                assert x["n_frames"] == y["n_frames"] and (x["pcm"] == y["pcm"]).all()
        held, fl = self.lib.carry_info()
        held2, fl2 = self.twin.carry_info()
        assert (held == held2).all() and (fl == fl2).all()
        self.last = np.array(last, np.int64)
        self.check_state()

    def _present(self, f):
        import torch
        w, nl = self.lib.geometry()
        got = []
        for ctx in (self.lib, self.twin):
            total = int(f(ctx, None)["n_fields"].sum())
            out = torch.empty(max(total, 1) * w * nl, dtype=torch.uint8 if self.dac8 else torch.uint16, device="cuda")
            info = f(ctx, out)
            fields = out[:total * w * nl].cpu().numpy() if self.dac8 else host_fields(out[:total * w * nl].view(total, w * nl))
            got.append((info, sha(fields)))
        assert (got[0][0] == got[1][0]).all()
        assert got[0][1] == got[1][1], "the keys context's fields differ from its twin's"

    def check_state(self):
        a, b = self.lib.library_info(), self.twin.library_info()
        assert (a == b).all()
        assert [tuple(int(v) for v in r) for r in a] == [st.status() for st in self.st]
        for t in range(len(self.titles)):
            assert self.lib.library_nv_read(t).tolist() == self.twin.library_nv_read(t).tolist() == self.nv[t]

    def close(self):
        self.lib.close()
        self.twin.close()


@pytest.mark.parametrize("ntsc,dac8", [(1, False), (0, True)])
def test_twins_seeded_keys(titles, ntsc, dac8):
    """eight streams, a different seeded key on every stream at every step, budgets that end titles (the DONE branch)"""
    n = 8
    rng = np.random.default_rng(77 + ntsc)
    tw = Twins(n, titles, 2000, ntsc=ntsc, dac8=dac8, clock=True)
    tw.submit(np.full(n, 60, np.uint32))
    codes = set()
    for k in range(16):
        if k in (6, 12):                                  # PLAY everywhere, then whole files: the titles that play end
            codes.update(tw.keys(np.full(n, kc.KEY_PLAY, np.uint8)))
            tw.submit(np.full(n, 2000, np.uint32))
        codes.update(tw.keys(rng.choice(KEY_CHOICES, n).astype(np.uint8)))
        tw.submit(rng.integers(2, 60, n).astype(np.uint32))
    assert any(c & kc.ENDED_BIT for c in codes) and {nc.PLAY, nc.PAUSE, nc.NAV_STEP, nc.MENU} <= {c & 0xF for c in codes}
    tw.close()


def test_twins_with_audio_and_a_queued_submit():
    """audio and carry on, and keys with a library submit queued behind the current one: audio, held bytes, pictures and states equal
    the command twin's"""
    ts = [_title(s, audio=True) for s in (4, 5)]
    n = 4
    tw = Twins(n, ts, 40, audio=True)
    rng = np.random.default_rng(5)
    tw.submit(np.full(n, 40, np.uint32))
    for k in range(8):
        keys = rng.choice(KEY_CHOICES, n).astype(np.uint8)
        if k % 2:
            tw.keys(keys)
            tw.submit(rng.integers(3, 40, n).astype(np.uint32))
            continue
        budgets = rng.integers(3, 40, n).astype(np.uint32)   # queued first: the keys act between the current submit and it
        for s, st in enumerate(tw.st):
            st.submit(tw.titles, int(budgets[s]))
        for ctx in (tw.lib, tw.twin):
            ctx.library_submit(per_stream=budgets)
        tw.keys(keys)
        for ctx in (tw.lib, tw.twin):
            ctx.index()
            m = ctx.index_info()["max_pictures"]
            ctx.decode_all(m)
        a, b = tw.lib.decode_audio(), tw.twin.decode_audio()
        assert all(x["n_frames"] == y["n_frames"] and (x["pcm"] == y["pcm"]).all() for x, y in zip(a, b))
        assert sha(tw.lib.read_latest_i420()) == sha(tw.twin.read_latest_i420())
        tw.last = np.array(tw.lib.picture_pts()[1], np.int64)
        tw.check_state()
    tw.close()


def _async_run(titles, n, scripts, device_keys):
    """keys, submit, index and the async present chain for every step with no host wait between them; keys from host arrays or
    written by a torch op on the same stream -> (sha of every call's info rows and fields, done codes, library_info)"""
    import torch
    ctx = _context(n, titles, n * 40 * 188, ntsc=1)
    for s in range(n):
        ctx.library_command(nc.NAV, s, 1, s % len(titles))
    st = torch.cuda.Stream()
    w, nl = ctx.geometry()
    table = torch.tensor(scripts, dtype=torch.uint8, device="cuda")
    shas, dones = [], []

    def chain():
        calls = []
        for p in range(ctx.max_pictures):
            out = torch.zeros(n * 16 * w * nl, dtype=torch.uint16, device="cuda")
            try:
                calls.append((ctx.present_picture_async(p, out, stream=st), out))
            except capi.EspflixError as e:
                assert e.code == capi.EF_ESTATE                  # past the submit's pictures
                break
        out = torch.zeros(n * 16 * w * nl, dtype=torch.uint16, device="cuda")
        calls.append((ctx.present_idle_async(np.full(n, 2, np.uint32), out, stream=st), out))
        return calls

    with torch.cuda.stream(st):
        ctx.library_submit(per_stream=np.full(n, 40, np.uint32), stream=st)
        ctx.index(stream=st.cuda_stream)
        calls = chain()
        for k in range(len(scripts)):
            done = torch.empty(n, dtype=torch.uint8, device="cuda")
            if device_keys:
                keys = torch.empty(n, dtype=torch.uint8, device="cuda")
                keys.copy_(table[k])                              # the producer, on the same stream
            else:
                keys = np.array(scripts[k], np.uint8)
            ctx.library_keys(keys, done, stream=st)
            ctx.library_submit(per_stream=np.full(n, 12, np.uint32), stream=st)
            ctx.index(stream=st.cuda_stream)
            calls += chain()
            dones.append(done)
    assert ctx.present_wait()[0] == capi.EF_OK
    st.synchronize()
    for info, out in calls:
        shas.append(sha(info.cpu().numpy()) + sha(out.cpu().numpy()))
    info = ctx.library_info().copy()
    ctx.close()
    return shas, [d.cpu().numpy().tolist() for d in dones], info


def test_device_producer_equals_host_keys(titles):
    n = 6
    rng = np.random.default_rng(11)
    scripts = rng.choice(KEY_CHOICES, (10, n)).astype(np.uint8).tolist()
    a = _async_run(titles, n, scripts, True)
    b = _async_run(titles, n, scripts, False)
    assert a[0] == b[0] and a[1] == b[1] and (a[2] == b[2]).all()


def test_scale_4096_streams_64_titles(titles):
    """4,096 streams over 64 titles (the three payloads, each added many times), mixed keys every step, against the restatement"""
    n, n_titles = 4096, 64
    ts = [titles[t % 3] for t in range(n_titles)]
    ctx = _context(n, ts, n * 6 * 188)
    rt = [nc.Title(idx, m, f, r, p) for idx, m, f, r, p in ts]
    sts = [kc.Stream() for _ in range(n)]
    nv = nc.new_nv(n_titles, n)
    ctx.library_command(nc.NAV, 0, n, 0)
    for s in range(n):
        sts[s].command(rt, nc.NAV, 0, nv=nv, s=s)
    rng = np.random.default_rng(4096)
    last = np.full(n, -1, np.int64)
    import torch
    done = torch.empty(n, dtype=torch.uint8, device="cuda")
    for step in range(10):
        keys = rng.choice(KEY_CHOICES, n).astype(np.uint8)
        if step == 0:
            keys[:] = np.where(rng.random(n) < 0.5, kc.KEY_RIGHT, kc.KEY_PLAY)
        ctx.library_keys(keys, done)
        want = [st.key(rt, int(keys[s]), int(last[s]), nv=nv, s=s)["done"] for s, st in enumerate(sts)]
        assert done.cpu().numpy().tolist() == want
        budgets = rng.integers(1, 6, n).astype(np.uint32)
        for s, st in enumerate(sts):
            st.submit(rt, int(budgets[s]))
        ctx.library_submit(per_stream=budgets)
        ctx.index()
        last = np.array(ctx.picture_pts()[1], np.int64)
        assert [tuple(int(v) for v in r) for r in ctx.library_info()] == [st.status() for st in sts]
    for t in range(n_titles):
        assert ctx.library_nv_read(t).tolist() == nv[t]
    ctx.close()


def test_errors_and_launches(titles):
    import torch
    n = 4
    ctx = espflix_b200.Context(n_streams=n, max_pictures=40, es_capacity=1 << 20, fields=False)
    keys = np.zeros(n, np.uint8)
    assert error_code(lambda: ctx.library_keys(keys)) == capi.EF_ESTATE                     # no title yet
    idx, m, f, r, p = titles[0]
    ctx.library_add(idx, m, f, r)
    assert error_code(lambda: ctx.library_keys(keys)) == capi.EF_ESTATE                     # no PTS, no carry
    ctx.close()
    ctx = _context(n, titles, 1 << 20, ntsc=1)
    assert ctx.lib.ef_library_keys(ctx._h, None, None, None) == capi.EF_EINVAL            # keys NULL
    host_done = np.zeros(n, np.uint8)
    assert ctx.lib.ef_library_keys(ctx._h, keys.ctypes.data, host_done.ctypes.data, None) == capi.EF_EINVAL
    ctx.library_command(nc.NAV, 0, n, 0)
    k = ctx.launch_count()
    ctx.library_keys(keys, _done_tensor(n))
    assert ctx.launch_count() - k == 3                                                     # keys, restart, carry restart
    ctx.library_submit(per_stream=np.full(n, 40, np.uint32))
    ctx.index()
    assert error_code(lambda: ctx.library_keys(keys)) == capi.EF_ESTATE                     # pictures not presented yet
    ctx.close()
    ctx = _context(n, titles, 1 << 20, audio=True)
    ctx.library_command(nc.NAV, 0, n, 0)
    k = ctx.launch_count()
    ctx.library_keys(torch.zeros(n, dtype=torch.uint8, device="cuda"))
    assert ctx.launch_count() - k == 4                                                     # and the audio end
    ctx.library_submit(per_stream=np.full(n, 40, np.uint32))
    ctx.index()
    assert error_code(lambda: ctx.library_keys(keys)) == capi.EF_ESTATE                     # the submit's audio not consumed
    ctx.close()
