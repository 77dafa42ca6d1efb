"""The title library's poster menu (EF_LIB_NAV / EF_LIB_NAV_STEP / EF_LIB_MENU, ef_library_add_poster, ef_library_nv_*) on the GPU.
A library-fed context runs seeded browse-and-play scripts beside a twin fed the same bytes from the host, with ef_restart_streams,
ef_end_streams, ef_present_overlay (the hidden progress) and the poster modes passed to ef_present_picture where tests/nav_cases.py's
restatement puts them: decoded pictures and pts, or every paced field and info row, must be identical, and ef_library_info and every
saved-position table must equal the restatement after every submit."""
import os
import subprocess

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import encode_cases as ec
from tests import nav_cases as nc
from tests import present_cases as pc
from tests import restart_cases
from tests.harness import error_code, host_fields, sha

pytestmark = pytest.mark.gpu
MAX_CARRY = 1 << 17
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "espflix_b200", "host", "ef_indexer_cli")


def _picture(seed):
    """a smooth seeded 352 x 192 I420 picture (a small poster at quantiser 2)"""
    rng = np.random.default_rng(seed)
    y = np.clip(np.add.outer(np.arange(192) * rng.uniform(0.1, 0.6), np.arange(352) * rng.uniform(0.1, 0.4)) + rng.integers(16, 90), 0, 235).astype(np.uint8)
    c = np.full(2 * 96 * 176, int(rng.integers(64, 192)), np.uint8)
    return np.concatenate([y.reshape(-1), c])


def _title(seed, trick=(True, True)):
    """a synthetic title with its poster: main = two programs (pts running on), fwd and rwd two short programs each, indexed with
    ef_tsidx_* -> (idx, main, fwd, rwd)"""
    P = 6 * 3003
    main = b"".join(restart_cases.program(seed * 10 + j, 6, 90000 + j * P) for j in range(2))
    fwd = b"".join(restart_cases.program(seed * 10 + 5 + j, 3, 90000 + j * P) for j in range(2))
    rwd = b"".join(restart_cases.program(seed * 10 + 7 + j, 3, 90000 + j * P) for j in range(2))
    idx = capi.build_video_idx(main, fwd, rwd)
    return idx, main, fwd if trick[1] else None, rwd if trick[0] else None


@pytest.fixture(scope="module")
def titles():
    """four titles, the third without a poster: (idx, main, fwd, rwd, poster)"""
    out = []
    for s in range(1, 5):
        idx, m, f, r = _title(s, trick=[(True, True), (False, True), (True, False), (True, True)][s % 4])
        out.append((idx, m, f, r, None if s == 3 else capi.encode_poster(_picture(s))))
    return out


def _context(n, es_capacity, ntsc=None, dac8=False, max_pictures=40):
    ctx = espflix_b200.Context(n_streams=n, max_pictures=max_pictures, max_slices_per_picture=12, es_capacity=es_capacity, fields=False)
    ctx.enable_pts()
    ctx.enable_carry(MAX_CARRY)
    if ntsc is not None:
        ctx.video_init(ntsc)
        if dac8:
            ctx.present_format(capi.EF_FIELD_DAC8)
        ctx.enable_present()
    return ctx


class Twins:
    """the library-fed context, its host-fed twin and the restatement, driven together. ntsc: presentation on (None: decode and
    compare pictures instead)"""

    def __init__(self, n, titles, budget_max, ntsc=None, dac8=False):
        self.n, self.paced, self.dac8 = n, ntsc is not None, dac8
        cap = max(n * budget_max * 188, 1 << 20)
        self.lib, self.twin = _context(n, cap, ntsc, dac8), _context(n, cap, ntsc, dac8)
        self.titles = [nc.Title(idx, m, f, r, p) for idx, m, f, r, p in titles]
        for k, (idx, m, f, r, p) in enumerate(titles):
            assert self.lib.library_add(idx, m, f, r) == k
            if p is not None:
                self.lib.library_add_poster(k, p)
        self.st = [nc.Stream() for _ in range(n)]
        self.nv = nc.new_nv(len(titles), n)
        self.last = np.full(n, -1, np.int64)
        self.ops = np.zeros(n, np.uint8)
        self.hide = np.zeros(n, np.uint8)
        self.poster_ends = 0                         # submits that ended a poster, over all streams
        if self.paced:
            self.disp = [pc.Display(ntsc) for _ in range(n)]
            self.exact = [True] * n                  # the display restatement holds (no picture outside the domain yet)
            rng = np.random.default_rng(n)
            bm = rng.integers(0, 256, (n, 1280)).astype(np.uint8)
            for ctx in (self.lib, self.twin):        # the progress is showing, so that hiding it shows in the fields
                ctx.present_overlay(bm, np.full(n, 180, np.int32), np.full(n, 100, np.int32))

    def command(self, s, cmd, title=0, arg=0, count=1):
        """one ef_library_command on streams [s, s + count); the twin's restarts and hidden progress wait for the next submit"""
        sts = self.st[s:s + count]
        if any(nc.check_command(self.titles, st, cmd, title, arg) for st in sts):
            before = self.lib.library_info().copy()
            assert error_code(lambda: self.lib.library_command(cmd, s, count, title, arg)) == capi.EF_EINVAL
            assert (self.lib.library_info() == before).all()
            return False
        self.lib.library_command(cmd, s, count, title, arg)
        for k, st in enumerate(sts):
            op, hide = st.command(self.titles, cmd, title, arg, int(self.last[s + k]), nv=self.nv, s=s + k)
            if op:
                self.ops[s + k] = op
                if self.paced:
                    self.disp[s + k].fc_origin = 0
            self.hide[s + k] |= hide
        return True

    def _flush_commands(self):
        if self.ops.any():
            self.twin.restart_streams(self.ops)
        if self.paced and self.hide.any():
            self.twin.present_overlay(blend=np.zeros(self.n, np.int32), set=self.hide * 2)
        self.ops[:] = 0
        self.hide[:] = 0

    def submit(self, budgets, use_async=False, caller_modes=None):
        """one library submit and its twin; presentation on: every picture index presented on both (caller_modes(p): the modes a
        caller passes to both, or None), else every picture decoded. Returns the picture counts."""
        self._flush_commands()
        chunks, ends, smode = [], np.zeros(self.n, np.uint8), np.zeros(self.n, np.uint8)
        for s, st in enumerate(self.st):
            run = st.submit(self.titles, int(budgets[s]))
            if run is None:
                chunks.append(b"")
                continue
            f, a, k, end = run
            chunks.append(self.titles[st.title].files[f][a:a + 188 * k])
            ends[s], smode[s] = end, st.end_mode(run)
        launches = [self.lib.launch_count(), self.twin.launch_count()]
        self.lib.library_submit(per_stream=budgets)
        self.twin.submit_ts(*self.twin.pack(chunks))
        if ends.any():
            self.twin.end_streams(ends)
        d_lib, d_twin = self.lib.launch_count() - launches[0], self.twin.launch_count() - launches[1]
        assert d_lib == d_twin + (2 if int(np.sum(budgets)) else 1)           # the count kernel, and the gather kernel for a bound > 0
        self.poster_ends += int((smode != 0).sum())
        for ctx in (self.lib, self.twin):
            ctx.index()
        counts = [self.lib.stream_info(s)[0] for s in range(self.n)]
        assert counts == [self.twin.stream_info(s)[0] for s in range(self.n)]
        pic, last = self.lib.picture_pts()
        pic2, last2 = self.twin.picture_pts()
        assert (pic == pic2).all() and (last == last2).all()
        if self.paced:
            for p in range(self.lib.index_info()["max_pictures"]):
                caller = np.zeros(self.n, np.uint8) if caller_modes is None else np.asarray(caller_modes(p), np.uint8)
                twin_modes = np.where(caller != 0, caller, np.where(np.array(counts) == p + 1, smode, 0)).astype(np.uint8)
                info = self._present(lambda ctx, o: ctx.present_picture(p, None if caller_modes is None else caller, o),
                                     lambda ctx, o: ctx.present_picture(p, twin_modes, o), use_async,
                                     lambda ctx, o: ctx.present_picture_async(p, o, modes=None if caller_modes is None else caller),
                                     lambda ctx, o: ctx.present_picture_async(p, o, modes=twin_modes))
                for s in range(self.n):
                    if p < counts[s] and self.exact[s]:
                        fields, F, fl = self.disp[s].push(int(pic[s, p]), int(twin_modes[s]))
                        if F is None:
                            self.exact[s] = False
                            continue
                        assert int(info[s]["n_fields"]) == len(fields) and (int(info[s]["flip_field"]), int(info[s]["flip_line"])) == (F, fl)
        else:
            info = self.lib.index_info()
            for ctx in (self.lib, self.twin):
                ctx.decode_all(info["max_pictures"])
            held, flags = self.lib.carry_info()
            held2, flags2 = self.twin.carry_info()
            assert (held == held2).all() and (flags == flags2).all()
            if self.n <= 64:
                assert sha(self.lib.read_latest_i420()) == sha(self.twin.read_latest_i420())
        self.last = np.array(last, np.int64)
        self.check_state()
        return counts

    def idle(self, n_fields, use_async=False):
        """an idle tail of n_fields on both contexts"""
        self._flush_commands()
        info = self._present(lambda ctx, o: ctx.present_idle(n_fields, o), lambda ctx, o: ctx.present_idle(n_fields, o), use_async,
                             lambda ctx, o: ctx.present_idle_async(n_fields, o), lambda ctx, o: ctx.present_idle_async(n_fields, o))
        for s in range(self.n):
            if self.exact[s]:
                assert int(info[s]["n_fields"]) == len(self.disp[s].idle(n_fields))

    def _present(self, f_lib, f_twin, use_async, a_lib, a_twin):
        """one present call on both contexts (synchronous, or asynchronous into a buffer sized by a synchronous sizing call): equal
        info rows, fields and kernel launches -> the info"""
        import torch
        w, nl = self.lib.geometry()
        got = []
        for ctx, f, a in ((self.lib, f_lib, a_lib), (self.twin, f_twin, a_twin)):
            total = int(f(ctx, None)["n_fields"].sum())
            k = ctx.launch_count()
            if self.dac8:
                out = torch.empty(max(total, 1) * w * nl, dtype=torch.uint8, device="cuda")
            else:
                out = torch.empty(max(total, 1) * w * nl, dtype=torch.uint16, device="cuda")
            if use_async:
                info = ctx.present_info(a(ctx, out))
                assert ctx.present_wait() == (capi.EF_OK, 1)
            else:
                info = f(ctx, out)
            fields = out[:total * w * nl].cpu().numpy() if self.dac8 else host_fields(out[:total * w * nl].view(total, w * nl))
            got.append((info, sha(fields), ctx.launch_count() - k))
        assert (got[0][0] == got[1][0]).all()
        assert got[0][1] == got[1][1], "the library context's fields differ from its twin's"
        assert got[0][2] == got[1][2], "a present call launched %d kernels, its twin %d" % (got[0][2], got[1][2])
        return got[0][0]

    def check_state(self):
        got = self.lib.library_info()
        assert [tuple(int(v) for v in r) for r in got] == [st.status() for st in self.st]
        for t in range(len(self.titles)):
            assert self.lib.library_nv_read(t).tolist() == self.nv[t]

    def close(self):
        self.lib.close()
        self.twin.close()


def _trick(tw):
    return lambda t: (tw.titles[t].sizes[0] > 0, tw.titles[t].sizes[2] > 0)


@pytest.mark.parametrize("budget", [1, 8, 37, 100000])
def test_twins_seeded_scripts(titles, budget):
    """four streams over four titles browse posters and play titles: a seeded command on each stream with probability 0.3 before
    every submit, among them the ones the library refuses"""
    n, steps = 4, 30
    rng = np.random.default_rng(2000 + budget)
    tw = Twins(n, titles, budget)
    pick = nc.script(rng, len(titles), trick=_trick(tw))
    for s in range(n):
        tw.command(s, nc.NAV, [0, 1, 3, 1][s])
    for k in range(steps):
        if k:
            for s in range(n):
                if rng.random() < 0.3:
                    tw.command(s, *pick(tw.st[s]))
        tw.submit(np.full(n, budget, np.uint32))
    assert tw.poster_ends > 0 or budget < 37
    tw.close()


def test_batched_steps_and_menus(titles):
    """NAV_STEP and MENU over a whole range in one call: the streams the step takes outside the row, and the streams already on a
    poster, are left alone while the others move (per-stream restart ops from one call)"""
    n = 6
    tw = Twins(n, titles, 400)
    tw.command(0, nc.NAV, 0, count=3)
    tw.command(3, nc.NAV, 3, count=3)
    tw.submit(np.full(n, 400, np.uint32))
    assert tw.command(0, nc.NAV_STEP, arg=2, count=n) is False                    # 0 + 2 = 2 has no poster: the call is refused
    assert tw.command(0, nc.NAV_STEP, arg=-1, count=n) is False                   # 0 - 1 is outside, but 3 - 1 = 2 has no poster
    assert tw.command(0, nc.NAV_STEP, arg=3, count=n)                              # 0 -> 3; 3 + 3 is outside: left alone
    assert [st.title for st in tw.st] == [3] * n
    tw.submit(np.full(n, 400, np.uint32))
    tw.command(0, nc.PLAY, count=2)
    tw.command(2, nc.PLAY, count=1)
    tw.submit(np.full(n, 7, np.uint32))
    tw.command(2, nc.FAST_FORWARD)
    tw.submit(np.full(n, 7, np.uint32))
    tw.command(1, nc.PAUSE)
    assert tw.command(0, nc.MENU, count=n)                                         # PLAYING 0, PAUSED 1, trick 2, POSTER 3..5
    assert [st.state for st in tw.st] == [nc.POSTER, nc.POSTER, nc.PLAYING] + [nc.POSTER] * 3 and tw.st[2].speed == 0
    assert tw.nv[3][0] == tw.st[0].pos and tw.nv[3][2] == tw.st[2].pos and tw.nv[3][1] == 0
    tw.submit(np.full(n, 400, np.uint32))
    tw.close()


@pytest.mark.parametrize("std", ["ntsc", "pal_dac8"])
def test_twins_presenting(titles, std):
    """the library-fed context and its host-fed twin with presentation on, through synchronous and asynchronous present calls: every
    field, info row and launch count equal, every push as present_cases' display restatement schedules it, the scroll run out over
    idle tails of 17 fields; callers' nonzero modes win over the library's"""
    ntsc, dac8 = std == "ntsc", std.endswith("dac8")
    n = 4
    rng = np.random.default_rng(31 if ntsc else 32)
    tw = Twins(n, titles, 3000, ntsc=ntsc, dac8=dac8)
    pick = nc.script(rng, len(titles), trick=_trick(tw))
    tw.command(0, nc.NAV, 0, count=2)
    tw.command(2, nc.NAV, 3, count=2)
    modes_seen = set()
    for k in range(16):
        if k == 1:
            tw.command(0, nc.NAV_STEP, arg=1, count=2)                               # 0 -> 1: the scroll one way (mode 2)
            tw.command(2, nc.NAV_STEP, arg=-2, count=2)                              # 3 -> 1: the other (mode 3)
        elif k:
            for s in range(n):
                if rng.random() < 0.5:
                    tw.command(s, *pick(tw.st[s]))
        for st in tw.st:
            modes_seen.add(st.mode if st.state == nc.POSTER else 0)
        caller = None
        if k % 5 == 4:
            c = np.where(rng.random(n) < 0.5, rng.integers(1, 4, n), 0).astype(np.uint8)
            caller = lambda p: c                                                    # noqa: E731
        tw.submit(rng.integers(20, 3000, n).astype(np.uint32), use_async=k % 2 == 1, caller_modes=caller)
        tw.idle(17, use_async=k % 3 == 2)
    assert {1, 2, 3} <= modes_seen
    assert all(tw.exact)
    tw.close()


def test_scale_4096_streams(titles):
    """4,096 streams over 64 titles (the four titles added many times), each on its own seeded browse-and-play script for four
    steps: every stream equals its twin and the restatement"""
    n = 4096
    rng = np.random.default_rng(4096)
    many = [titles[k % len(titles)] for k in range(64)]
    tw = Twins(n, many, 30)
    pick = nc.script(rng, 64, trick=_trick(tw))
    for s in range(n):
        tw.command(s, nc.NAV, int(rng.integers(64)))
    tw.submit(rng.integers(0, 30, n).astype(np.uint32))
    for _ in range(4):
        for s in range(n):
            tw.command(s, *pick(tw.st[s]))
        tw.submit(rng.integers(0, 30, n).astype(np.uint32))
    tw.close()


def test_errors_and_state(titles):
    """every EF_EINVAL / EF_ESTATE case of the poster calls and commands, each leaving every state unchanged"""
    idx, m, f, r, p = titles[0]
    plain = espflix_b200.Context(n_streams=2, max_pictures=8, es_capacity=1 << 20, fields=False)
    assert error_code(lambda: plain.library_add_poster(0, p)) == capi.EF_ESTATE
    assert error_code(lambda: plain.library_nv_read(0)) == capi.EF_ESTATE
    assert error_code(lambda: plain.library_nv_write(0, [1, 2])) == capi.EF_ESTATE
    plain.close()
    ctx = _context(3, 1 << 20)
    for t in titles:
        ctx.library_add(*t[:4])
    assert error_code(lambda: ctx.library_add_poster(4, p)) == capi.EF_EINVAL                # unknown title
    assert error_code(lambda: ctx.library_add_poster(-1, p)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.library_add_poster(0, p[:-1])) == capi.EF_EINVAL           # not whole packets
    assert error_code(lambda: ctx.library_add_poster(0, b"")) == capi.EF_EINVAL
    assert ctx.library_read(0, 3) == b""
    ctx.library_add_poster(0, p)
    ctx.library_add_poster(3, titles[3][4])
    assert error_code(lambda: ctx.library_add_poster(0, titles[1][4])) == capi.EF_ESTATE     # a second poster
    assert ctx.library_read(0, 3) == p and ctx.library_read(3, 3) == titles[3][4] and ctx.library_read(1, 3) == b""
    assert error_code(lambda: ctx.library_read(0, 4)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.library_nv_read(4)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.library_nv_read(0, 2, 2)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.library_nv_write(0, [1, 2], first=2)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.library_nv_write(-1, [1])) == capi.EF_EINVAL
    ctx.library_nv_write(3, [11, 22, 33])
    assert ctx.library_nv_read(3).tolist() == [11, 22, 33] and ctx.library_nv_read(0).tolist() == [0, 0, 0]

    def refused(cmd, first=0, count=1, title=0, arg=0):
        before = ctx.library_info().copy()
        nv = [ctx.library_nv_read(t).tolist() for t in range(4)]
        assert error_code(lambda: ctx.library_command(cmd, first, count, title, arg)) == capi.EF_EINVAL, (cmd, first, count, title, arg)
        assert (ctx.library_info() == before).all() and [ctx.library_nv_read(t).tolist() for t in range(4)] == nv

    refused(capi.LIB_MENU)                                                                 # IDLE
    refused(capi.LIB_NAV_STEP, arg=1)
    refused(capi.LIB_NAV, title=4)                                                        # unknown title
    refused(capi.LIB_NAV, title=1)                                                        # no poster
    refused(capi.LIB_MENU + 1)
    ctx.library_command(capi.LIB_NAV, 0, 3, 3, 0)
    st = ctx.library_info()
    assert (st["state"] == capi.LIB_POSTER).all() and (st["file"] == capi.LIB_POSTER_FILE).all() and st["pos"].tolist() == [11, 22, 33]
    refused(capi.LIB_NAV_STEP, arg=-1)                                                    # title 2 has no poster
    refused(capi.LIB_NAV_STEP, arg=-2, count=3)                                           # title 1 neither
    refused(capi.LIB_NAV_STEP, arg=2 ** 31)
    refused(capi.LIB_RESUME)
    ctx.library_command(capi.LIB_NAV_STEP, 0, 1, 0, -3)                                   # stream 0 to title 0
    ctx.library_command(capi.LIB_NAV_STEP, 1, 1, 0, 5)                                    # outside the row: nothing
    st = ctx.library_info()
    assert st["title"].tolist() == [0, 3, 3] and st["pos"].tolist() == [0, 22, 33]
    ctx.library_command(capi.LIB_PAUSE, 0, 3)                                            # nothing on a poster
    assert (ctx.library_info() == st).all()
    ctx.library_command(capi.LIB_PLAY, 1, 2)
    refused(capi.LIB_NAV, 1, 1, 0)                                                        # PLAYING
    refused(capi.LIB_NAV_STEP, 1, 1, 0, 1)
    ctx.library_command(capi.LIB_STOP, 2, 1)
    refused(capi.LIB_NAV_STEP, 2, 1, 0, 1)                                                # STOPPED
    ctx.close()


def test_launches_without_posters(titles):
    """a library context whose titles have no poster launches per submit and command what one with posters launches, and no more
    than the count and gather kernels beside a host submit's upload"""
    counts = []
    for with_posters in (False, True):
        ctx = _context(2, 1 << 20)
        for k, t in enumerate(titles):
            ctx.library_add(*t[:4])
            if with_posters and t[4] is not None:
                ctx.library_add_poster(k, t[4])
        k0 = ctx.launch_count()
        ctx.library_command(capi.LIB_PLAY_AT, 0, 2, 0, 90000)
        k1 = ctx.launch_count()
        ctx.library_submit(40)
        k2 = ctx.launch_count()
        ctx.index()
        ctx.library_command(capi.LIB_SKIP, 0, 2, 0, 1)
        counts.append((k1 - k0, k2 - k1, ctx.launch_count() - k2))
        ctx.close()
    assert counts[0] == counts[1]


def test_encode_poster(titles, tmp_path):
    """capi.encode_poster equals the encoder's restatement at gop 1 / q 2, the oracle decodes it to the restated picture, the library
    shows that picture after a NAV, and ef_indexer_cli --poster writes the same file"""
    from tests.oracle_lib import Oracle
    oracle = Oracle()
    pic = _picture(9)
    ts = capi.encode_poster(pic)
    want, es, recon, _ = ec.encode_title(pic[None], oracle, gop=1, qscale_i=2)
    assert ts == want and len(es) == 1
    assert np.array_equal(oracle.decode_es(es[0])[0], recon[0])
    ctx = _context(1, 1 << 20)
    idx, m, f, r, _ = titles[0]
    ctx.library_add(idx, m, f, r)
    ctx.library_add_poster(0, ts)
    ctx.library_command(capi.LIB_NAV, 0, 1, 0, 0)
    ctx.library_submit(1000)
    ctx.index()
    assert ctx.stream_info(0)[0] == 1
    ctx.decode_all(1)
    assert np.array_equal(ctx.read_latest_i420()[0].reshape(-1), recon[0].reshape(-1))
    assert ctx.library_info()[0]["state"] == capi.LIB_POSTER
    ctx.close()
    src, poster = tmp_path / "pictures.i420", tmp_path / "poster.i420"
    src.write_bytes(ec.translated(3, 2, (1, 1)).tobytes())
    poster.write_bytes(pic.tobytes())
    d = tmp_path / "title"
    d.mkdir()
    subprocess.run([CLI, "--encode", str(src), str(d), "--poster", str(poster)], check=True, capture_output=True, timeout=300)
    assert (d / "poster.ts").read_bytes() == ts
    assert (d / "video.ts").read_bytes() == capi.encode_build([ec.translated(3, 2, (1, 1))])[0]
