"""Titles held in device memory (ef_library_*) on the GPU. A library-fed context runs seeded command scripts beside a twin fed the
same bytes through ef_submit_ts_host, with ef_restart_streams / ef_end_streams where tests/library_cases.py's restatement puts
them: picture counts, pictures, pts, audio and carry state must be identical, and ef_library_info must equal the restatement after
every submit. The fixture title played from PLAY_AT 0 to its end gives what decode_pins.json / pts_pins.json pin."""
import json
import os

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import library_cases as lc, pts_cases, restart_cases
from tests.harness import error_code, sha

pytestmark = pytest.mark.gpu
G = pts_cases.GOLDEN
MAX_CARRY = 1 << 17


def _context(n, es_capacity, max_pictures=40, audio=True):
    ctx = espflix_b200.Context(n_streams=n, max_pictures=max_pictures, max_slices_per_picture=12, es_capacity=es_capacity, fields=False)
    ctx.enable_pts()
    ctx.enable_carry(MAX_CARRY)
    if audio:
        ctx.enable_audio()
    return ctx


def _title(seed, n_programs=3, trick=(True, True)):
    """a synthetic title: main = n_programs programs with audio (one sequence header each, pts running on), fwd and rwd two short
    programs each; indexed with ef_tsidx_* -> (idx, main, fwd, rwd)"""
    P = 6 * 3003
    main = b"".join(restart_cases.program(seed * 10 + j, 6, 90000 + j * P, audio=dict(seed=seed * 10 + j, frames=30, cut=0)) for j in range(n_programs))
    fwd = b"".join(restart_cases.program(seed * 10 + 5 + j, 3, 90000 + j * P, audio=None) for j in range(2))
    rwd = b"".join(restart_cases.program(seed * 10 + 7 + j, 3, 90000 + j * P, audio=None) for j in range(2))
    idx = capi.build_video_idx(main, fwd, rwd)
    return idx, main, fwd if trick[1] else None, rwd if trick[0] else None


@pytest.fixture(scope="module")
def titles():
    return [_title(s, trick=[(True, True), (False, True), (True, False)][s % 3]) for s in range(1, 4)]


class Twins:
    """the library-fed context, its twin and the restatement, driven together"""

    def __init__(self, n, titles, budget_max, audio=True):
        self.n, self.audio = n, audio
        cap = max(n * budget_max * 188, 1 << 20)
        self.lib, self.twin = _context(n, cap, audio=audio), _context(n, cap, audio=audio)
        self.titles = [lc.Title(idx, m, f, r) for idx, m, f, r in titles]
        for k, (idx, m, f, r) in enumerate(titles):
            assert self.lib.library_add(idx, m, f, r) == k
        self.st = [lc.Stream() for _ in range(n)]
        self.last = np.full(n, -1, np.int64)

    def command(self, s, cmd, title=0, arg=0):
        st = self.st[s]
        if lc.check_command(self.titles, st, cmd, title, arg):
            assert error_code(lambda: self.lib.library_command(cmd, s, 1, title, arg)) == capi.EF_EINVAL
            return
        self.lib.library_command(cmd, s, 1, title, arg)
        op, _ = st.command(self.titles, cmd, title, arg, int(self.last[s]))
        if op:
            ops = np.zeros(self.n, np.uint8)
            ops[s] = op
            self.twin.restart_streams(ops)

    def submit(self, budgets):
        chunks, ends = [], np.zeros(self.n, np.uint8)
        for s in range(self.n):
            run = self.st[s].submit(self.titles, int(budgets[s]))
            if run is None:
                chunks.append(b"")
                continue
            f, a, k, end = run
            chunks.append(self.titles[self.st[s].title].files[f][a:a + 188 * k])
            ends[s] = end
        self.lib.library_submit(per_stream=budgets)
        self.twin.submit_ts(*self.twin.pack(chunks))
        if ends.any():
            self.twin.end_streams(ends)
        out = []
        for ctx in (self.lib, self.twin):
            ctx.index()
            info = ctx.index_info()
            counts = [ctx.stream_info(s)[0] for s in range(self.n)]
            ctx.decode_all(info["max_pictures"])
            pic, last = ctx.picture_pts()
            held, flags = ctx.carry_info()
            frames = sha(ctx.read_latest_i420())
            aud = ctx.decode_audio() if self.audio else []
            out.append((counts, pic.tolist(), last.tolist(), held.tolist(), flags.tolist(), frames,
                        [(a["n_frames"], sha(a["pcm"]), sha(a["pdm"])) for a in aud]))
        assert out[0] == out[1]
        self.last = np.array(out[0][2], np.int64)
        got = self.lib.library_info()
        want = [st.status() for st in self.st]
        assert [tuple(int(v) for v in r) for r in got] == want
        return out[0]

    def close(self):
        self.lib.close()
        self.twin.close()


@pytest.mark.parametrize("budget", [1, 8, 37, 100000])
def test_twins_seeded_scripts(titles, budget):
    """four streams over three titles, a seeded command on each stream with probability 0.2 before every submit"""
    n, steps = 4, 24
    rng = np.random.default_rng(1000 + budget)
    tw = Twins(n, titles, budget)
    pick = lc.script(rng, len(titles), steps, trick=lambda t: (tw.titles[t].sizes[0] > 0, tw.titles[t].sizes[2] > 0))
    for s in range(n):
        tw.command(s, lc.PLAY_AT, s % len(titles), int(rng.integers(0, 90000 * 4)))
    pictures = 0
    for k in range(steps):
        if k:
            for s in range(n):
                if rng.random() < 0.2:
                    tw.command(s, *pick(tw.st[s]))
        pictures += sum(tw.submit(np.full(n, budget, np.uint32))[0])
    tw.close()
    assert pictures > 0 or budget < 37          # 24 steps of 1 or 8 packets between restarts may complete no picture


def test_fixture_title_against_pins():
    """video.idx of the fixtures with vmedia.ts as main and rwd and splash.ts as fwd, played from PLAY_AT 0 to its end in seeded
    budgets: every picture and pts as decode_pins.json / pts_pins.json pin for vmedia"""
    idx = open(os.path.join(G, "video_idx_fixture.bin"), "rb").read()
    vm = open(os.path.join(G, "vmedia.ts"), "rb").read()
    sp = open(os.path.join(G, "splash.ts"), "rb").read()
    dpins = json.load(open(os.path.join(G, "decode_pins.json")))["vmedia"]["frame_sha256"]
    ppins = json.load(open(os.path.join(G, "pts_pins.json")))["programs"]["vmedia"]["pts"]
    ctx = _context(1, 1 << 20, max_pictures=100, audio=False)
    t = ctx.library_add(idx, vm, sp, vm)
    ctx.library_command(capi.LIB_PLAY_AT, 0, 1, t, 0)
    _, first = lc.get_index(idx, 0, 0)
    assert int(ctx.library_info()[0]["cursor"]) == first * 188
    rng = np.random.default_rng(5)
    frames, pts = [], []
    while ctx.library_info()[0]["state"] == capi.LIB_PLAYING:
        ctx.library_submit(int(rng.integers(1, 300)))
        ctx.index()
        n = ctx.stream_info(0)[0]
        for p in range(n):
            ctx.decode_picture(p)
            frames.append(sha(ctx.read_frame_i420(0, (ctx.stream_info(0)[1] + p + 1) & 1)))
        pts += [int(v) for v in ctx.picture_pts()[0][0, :n]]
    st = ctx.library_info()[0]
    assert st["state"] == capi.LIB_ENDED and st["pos"] == 0 and st["cursor"] == len(vm)
    ctx.close()
    assert frames == dpins
    assert pts == ppins


def test_errors_and_state(titles):
    """every EF_EINVAL / EF_ESTATE / EF_ENOMEM case of the four calls, and ef_reset keeping titles, states and cursors"""
    idx, m, f, r = titles[2]                                                                         # all three files
    plain = espflix_b200.Context(n_streams=2, max_pictures=8, es_capacity=1 << 20, fields=False)
    assert error_code(lambda: plain.library_info()) == capi.EF_ESTATE
    assert error_code(lambda: plain.library_submit(1)) == capi.EF_ESTATE
    plain.library_add(idx, m, f, r)
    assert error_code(lambda: plain.library_command(capi.LIB_PLAY_AT, 0, 1, 0, 0)) == capi.EF_ESTATE   # no pts / carry
    plain.close()
    ctx = _context(2, 40 * 188 * 2)
    bad = bytearray(idx)
    bad[0] ^= 1
    assert error_code(lambda: ctx.library_add(bytes(bad), m)) == capi.EF_EINVAL                      # signature
    bad = bytearray(idx)
    bad[4] = 2
    assert error_code(lambda: ctx.library_add(bytes(bad), m)) == capi.EF_EINVAL                      # len != 3
    assert error_code(lambda: ctx.library_add(idx[:-4], m)) == capi.EF_EINVAL                        # samples past the end
    bad = bytearray(idx)
    bad[24:28] = b"\0\0\0\0"
    assert error_code(lambda: ctx.library_add(bytes(bad), m)) == capi.EF_EINVAL                      # video bin_size 0
    bad = bytearray(idx)
    bad[60:64] = b"\0\0\0\0"
    assert error_code(lambda: ctx.library_add(bytes(bad), m, f)) == capi.EF_EINVAL                   # fwd trick_speed 0
    ctx.library_add(bytes(bad), m, None, r)                                                          # ... fine without fwd
    bad = bytearray(idx)
    bad[80:88] = bad[72:80]
    assert error_code(lambda: ctx.library_add(bytes(bad), m, f, r)) == capi.EF_EINVAL                # rwd last == first
    assert error_code(lambda: ctx.library_add(idx, m[:-1])) == capi.EF_EINVAL                        # not whole packets
    t = ctx.library_add(idx, m, f, None)
    assert error_code(lambda: ctx.library_command(capi.LIB_PLAY_AT, 0, 1, 99, 0)) == capi.EF_EINVAL   # unknown title
    assert error_code(lambda: ctx.library_command(capi.LIB_PLAY, 0, 1)) == capi.EF_EINVAL             # never played
    assert error_code(lambda: ctx.library_command(9, 0, 1)) == capi.EF_EINVAL
    ctx.library_command(capi.LIB_PLAY_AT, 0, 2, t, 90000)
    assert error_code(lambda: ctx.library_command(capi.LIB_REWIND, 0, 1)) == capi.EF_EINVAL           # no rwd file
    assert error_code(lambda: ctx.library_command(capi.LIB_RESUME, 0, 1)) == capi.EF_EINVAL           # not paused
    assert error_code(lambda: ctx.library_command(capi.LIB_SKIP, 0, 1, 0, 2 ** 31)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.library_submit(41)) == capi.EF_ENOMEM                              # 2 x 41 x 188 > capacity
    assert error_code(lambda: ctx.library_submit(0, [80, 1])) == capi.EF_ENOMEM
    before = ctx.library_info().copy()
    ctx.library_submit(5)
    assert error_code(lambda: ctx.library_submit(5)) == capi.EF_ESTATE                               # a submit pending
    assert error_code(lambda: ctx.end_streams(np.ones(2, np.uint8))) == capi.EF_ESTATE
    ctx.index()
    assert error_code(lambda: ctx.library_command(capi.LIB_PAUSE, 0, 1)) == capi.EF_ESTATE            # audio unconsumed
    ctx.decode_audio()
    ctx.library_command(capi.LIB_PAUSE, 0, 1)
    after = ctx.library_info().copy()
    assert (after["cursor"] == before["cursor"] + 5 * 188).all()
    assert after[0]["state"] == capi.LIB_PAUSED and after[1]["state"] == capi.LIB_PLAYING
    ctx.reset()
    assert (ctx.library_info() == after).all()                                                      # ef_reset keeps them
    ctx.library_command(capi.LIB_RESUME, 0, 1)
    assert ctx.library_info()[0]["state"] == capi.LIB_PLAYING
    ctx.close()


def test_paced_command_gate(titles):
    """a command while picture indices of the current submit are unpresented returns EF_ESTATE, as ef_restart_streams does"""
    idx, m, f, r = titles[0]
    ctx = espflix_b200.Context(n_streams=1, max_pictures=40, es_capacity=1 << 20, fields=False)
    ctx.enable_pts()
    ctx.enable_carry(MAX_CARRY)
    ctx.video_init(1)
    ctx.enable_present()
    ctx.library_add(idx, m, f, r)
    ctx.library_command(capi.LIB_PLAY_AT, 0, 1, 0, 0)
    ctx.library_submit(400)
    ctx.index()
    assert ctx.index_info()["max_pictures"] > 0
    assert error_code(lambda: ctx.library_command(capi.LIB_SKIP, 0, 1, 0, 5)) == capi.EF_ESTATE
    ctx.close()


def test_scale_4096_streams(titles):
    """4,096 streams over 64 titles (the three synthetic titles, each added many times) for one step of seeded commands: every
    stream equals its twin and the restatement"""
    n = 4096
    rng = np.random.default_rng(77)
    many = [titles[k % len(titles)] for k in range(64)]
    tw = Twins(n, many, 20, audio=False)
    for s in range(n):
        tw.command(s, lc.PLAY_AT, int(rng.integers(64)), int(rng.integers(0, 90000 * 3)))
    tw.submit(np.full(n, 20, np.uint32))
    for s in range(n):
        if rng.random() < 0.5:
            pick = lc.script(rng, 64, 1, trick=lambda t: (tw.titles[t].sizes[0] > 0, tw.titles[t].sizes[2] > 0))
            tw.command(s, *pick(tw.st[s]))
    tw.submit(rng.integers(0, 30, n).astype(np.uint32))
    tw.close()
