"""ef_library_add_trick on the GPU: a title added with its main only, then given its trick files on the device, against a twin added
from the host with build_video_idx(main, fwd, rwd) and the files trick_build returned. Seeded PLAY / FAST_FORWARD / REWIND / SKIP
scripts with submits give identical pictures, pts and ef_library_info, the idx images and files are equal, a second call is
EF_ESTATE; and ef_indexer_cli writes the same three files for a title directory that holds only video.ts."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import library_cases as lc, restart_cases
from tests.harness import error_code, sha

pytestmark = pytest.mark.gpu
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "espflix_b200", "host", "ef_indexer_cli")


def _mains():
    from espflix_b200 import synth
    P = 8 * 3003
    audio = b"".join(restart_cases.program(300 + j, 8, 90000 + j * P, audio=dict(seed=30 + j, frames=40, cut=0)) for j in range(3))
    es, off = synth.generate(synth.SEED0 + 31, n_pictures=62, gop=12)
    return [audio, bytes(synth.wrap_ts(es, off))]


@pytest.fixture(scope="module")
def mains():
    return _mains()


def _context(n, cap):
    ctx = espflix_b200.Context(n_streams=n, max_pictures=64, max_slices_per_picture=12, es_capacity=cap, fields=False)
    ctx.enable_pts()
    ctx.enable_carry(1 << 17)
    return ctx


def _pair(mains, n, cap):
    built, twin = _context(n, cap), _context(n, cap)
    files = capi.trick_build(mains)
    for k, m in enumerate(mains):
        assert built.library_add(capi.build_video_idx(m, b"", b""), m) == k
        built.library_add_trick(k)
        fwd, rwd = files[k]
        assert twin.library_add(capi.build_video_idx(m, fwd, rwd), m, fwd, rwd) == k
    return built, twin, files


def test_built_title_equals_twin(mains):
    built, twin, files = _pair(mains, 1, 1 << 20)
    for k in range(len(mains)):
        assert built.library_read(k, -1) == twin.library_read(k, -1)                 # the rewritten video.idx
        assert built.library_read(k, 2) == files[k][0] and built.library_read(k, 0) == files[k][1]
        assert built.library_read(k, 1) == mains[k]
        assert error_code(lambda: built.library_add_trick(k)) == capi.EF_ESTATE     # a second call
    assert error_code(lambda: built.library_add_trick(len(mains))) == capi.EF_EINVAL
    assert error_code(lambda: twin.library_add_trick(0)) == capi.EF_ESTATE           # added with its trick files
    built.close()
    twin.close()


def test_errors_leave_the_title_alone(mains):
    from espflix_b200 import synth
    ctx = _context(1, 1 << 20)
    assert error_code(lambda: ctx.library_add_trick(0)) == capi.EF_ESTATE          # no title yet
    es, off = synth.generate(synth.SEED0 + 40, n_pictures=10, gop=12)
    short = bytes(synth.wrap_ts(es, off))
    idx = capi.build_video_idx(short, b"", b"")
    assert ctx.library_add(idx, short) == 0
    assert error_code(lambda: ctx.library_add_trick(0, qscale=0)) == capi.EF_EINVAL
    assert error_code(lambda: ctx.library_add_trick(0)) == capi.EF_EINVAL          # one fwd picture: the reference divides by zero
    assert ctx.library_read(0, -1) == idx and ctx.library_read(0, 2) == b""
    ctx.close()


@pytest.mark.parametrize("budget", [3, 16, 100000])
def test_seeded_scripts(mains, budget):
    n, steps = 4, 30
    rng = np.random.default_rng(77 + budget)
    built, twin, files = _pair(mains, n, max(n * budget * 188, 1 << 20))
    titles = [lc.Title(capi.build_video_idx(m, f, r), m, f, r) for m, (f, r) in zip(mains, files)]
    st = [lc.Stream() for _ in range(n)]
    pick = lc.script(rng, len(titles), steps)
    last = np.full(n, -1, np.int64)

    def command(s, cmd, title=0, arg=0):
        if lc.check_command(titles, st[s], cmd, title, arg):
            for ctx in (built, twin):
                assert error_code(lambda: ctx.library_command(cmd, s, 1, title, arg)) == capi.EF_EINVAL
            return
        for ctx in (built, twin):
            ctx.library_command(cmd, s, 1, title, arg)
        st[s].command(titles, cmd, title, arg, int(last[s]))

    for s in range(n):
        command(s, lc.PLAY_AT, s % len(titles), int(rng.integers(0, 90000 * 2)))
    for k in range(steps):
        for s in range(n):
            if k and rng.random() < 0.3:
                command(s, *pick(st[s]))
        for s in range(n):
            st[s].submit(titles, budget)
        out = []
        for ctx in (built, twin):
            ctx.library_submit(packets=budget)
            ctx.index()
            info = ctx.index_info()
            counts = [ctx.stream_info(s)[0] for s in range(n)]
            ctx.decode_all(info["max_pictures"])
            pic, lp = ctx.picture_pts()
            out.append((counts, pic.tolist(), lp.tolist(), sha(ctx.read_latest_i420()), [tuple(int(v) for v in r) for r in ctx.library_info()]))
        assert out[0] == out[1], "step %d" % k
        assert out[0][4] == [x.status() for x in st]
        last = np.array(out[0][2], np.int64)
    built.close()
    twin.close()


def test_indexer_cli_title_directory(mains):
    m = mains[1]
    (fwd, rwd), = capi.trick_build([m])
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "video.ts"), "wb").write(m)
        subprocess.run([CLI, d], check=True, capture_output=True, timeout=300)
        assert open(os.path.join(d, "video_fwd.ts"), "rb").read() == fwd
        assert open(os.path.join(d, "video_rwd.ts"), "rb").read() == rwd
        assert open(os.path.join(d, "video.idx"), "rb").read() == capi.build_video_idx(m, fwd, rwd)
