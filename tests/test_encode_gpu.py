"""ef_encode_build against the restatement (tests/encode_cases.py): video.ts byte for byte, the reconstruction the device predicted from,
a title through the library, and the argument checks."""
import ctypes

import numpy as np
import pytest

from tests import encode_cases as ec
from tests import trick_cases as tc
from tests.oracle_lib import Oracle

pytestmark = pytest.mark.gpu


def _capi():
    from espflix_b200 import capi
    return capi


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def _check(oracle, titles, **params):
    got = _capi().encode_build(titles, **params)
    assert len(got) == len(titles)
    for t, (pics, ts) in enumerate(zip(titles, got)):
        want = ec.encode_title(pics, oracle, **params)[0]
        assert len(ts) == len(want) and ts == want, "title %d (%d pictures, %s): first difference at byte %s" % (
            t, len(pics), params, next((i for i in range(min(len(ts), len(want))) if ts[i] != want[i]), min(len(ts), len(want))))
    return got


@pytest.mark.parametrize("q", [None, 1, 31])
@pytest.mark.parametrize("name", ["vmedia", "splash"])
def test_fixture_pictures(oracle, name, q):
    pics = ec.fixture_pictures(name, oracle)
    params = {} if q is None else dict(qscale_i=q, qscale_p=q)
    _check(oracle, [pics], **params)


@pytest.mark.parametrize("case", ["static", "integer", "half", "cut", "edge", "beyond"])
def test_synthetic_motion(oracle, case):
    pics = {"static": lambda: ec.translated(1, 6, (0, 0), grain=0.0), "integer": lambda: ec.translated(2, 6, (4, -2)),
            "half": lambda: ec.translated(3, 6, (1, 3)), "cut": lambda: ec.scene_cut(4, 6, 3),
            "edge": lambda: ec.translated(5, 4, (14, -14)), "beyond": lambda: ec.translated(6, 4, (-16, 20))}[case]()
    _check(oracle, [pics])


@pytest.mark.parametrize("q", [1, 8, 31])
def test_noise_and_checkerboards(oracle, q):
    titles = [ec.noise(7, 4), ec.checkerboard(4, cell=1), ec.checkerboard(4, cell=8, phase=1)]
    _check(oracle, titles, qscale_i=q, qscale_p=q)


@pytest.mark.parametrize("search", [0, 3, 15])
def test_search_radius(oracle, search):
    _check(oracle, [ec.translated(8, 4, (6, 4))], search=search)


@pytest.mark.parametrize("gop", [1, 3, 12, 15])
def test_title_lengths_and_gops(oracle, gop):
    src = ec.translated(9, 25, (2, 1))
    titles = [src[:n] for n in (1, 11, 12, 13, 25)]
    _check(oracle, titles, gop=gop, aspect=3, rate=5, pts0=(1 << 33) - 1 - 24 * 3003, pts_step=3003)


def test_batch_boundary(oracle):
    """more GOPs than one batch of the internal decode context: 513 GOPs of 2 pictures (the batch holds 512)"""
    clips = [ec.translated(10 + i, 2, (2 * i, -i)) for i in range(3)]
    order = [(g * 7) % 3 for g in range(513)]
    title = np.concatenate([clips[i] for i in order])
    got = _capi().encode_build([title], gop=2)[0]
    es = [ec.encode_title(c, oracle, gop=2)[1] for c in clips]
    pics = [e for i in order for e in es[i]]
    pts = [3750 * k for k in range(len(pics))]
    assert got == tc.mux(pics, pts)


def test_errors():
    capi = _capi()
    lib = capi.load_library()
    pics = np.zeros((2, ec.PICTURE_BYTES), np.uint8)
    off = np.array([0, 2], np.uint64)
    to = np.zeros(2, np.uint64)
    out = np.zeros(1 << 20, np.uint8)

    def call(n=1, off_=off, ts=out, cap=out.size, **kw):
        p = capi.EncodeParams(**dict(capi.ENCODE_DEFAULTS, **kw))
        return lib.ef_encode_build(0, pics.ctypes.data, off_.ctypes.data, n, ctypes.byref(p), ts.ctypes.data if ts is not None else None, cap,
                                   to.ctypes.data)
    assert call() == capi.EF_OK
    need = int(to[-1])
    assert call(gop=1024) == capi.EF_OK
    for kw in [dict(gop=0), dict(gop=1025), dict(qscale_i=0), dict(qscale_p=32), dict(search=-1), dict(search=16), dict(aspect=0), dict(aspect=15),
               dict(rate=0), dict(rate=9), dict(pts0=-1), dict(pts0=(1 << 33) - 3750)]:
        assert call(**kw) == capi.EF_EINVAL, kw
    assert call(n=0) == capi.EF_EINVAL
    assert call(off_=np.array([0, 0], np.uint64)) == capi.EF_EINVAL
    assert call(pts0=(1 << 33) - 3751) == capi.EF_OK
    out[:] = 0xAA
    to[:] = 0
    assert call(cap=need - 1) == capi.EF_ENOMEM and int(to[-1]) == need and (out == 0xAA).all()
    assert call(ts=None, cap=0) == capi.EF_ENOMEM and int(to[-1]) == need


def test_split_reconstruction_submits(oracle):
    """rounds whose pictures exceed one reconstruction submit (32 MB of ES): 220 GOPs of noise at qscale 1, about 170 KB a picture"""
    clips = [ec.noise(40 + i, 2) for i in range(3)]
    order = [(g * 5) % 3 for g in range(220)]
    title = np.concatenate([clips[i] for i in order])
    got = _capi().encode_build([title], gop=2, qscale_i=1, qscale_p=1)[0]
    es = [ec.encode_title(c, oracle, gop=2, qscale_i=1, qscale_p=1)[1] for c in clips]
    assert sum(len(es[i][1]) for i in order) > 32 << 20
    pics = [e for i in order for e in es[i]]
    assert got == tc.mux(pics, [3750 * k for k in range(len(pics))])


def test_indexer_cli_encode(oracle, tmp_path):
    """ef_indexer_cli --encode: the fixture's pictures -> video.ts (ef_encode_build at the defaults), video_fwd.ts, video_rwd.ts and
    video.idx, the last equal to build_video_idx of the three files"""
    import os
    import subprocess
    capi = _capi()
    cli = os.path.join(ec.ROOT, "espflix_b200", "host", "ef_indexer_cli")
    pics = ec.fixture_pictures("vmedia", oracle)
    src = tmp_path / "pictures.i420"
    src.write_bytes(pics.tobytes())
    d = tmp_path / "title"
    d.mkdir()
    subprocess.run([cli, "--encode", str(src), str(d)], check=True, capture_output=True, timeout=300)
    main = (d / "video.ts").read_bytes()
    assert main == ec.encode_title(pics, oracle)[0]
    fwd, rwd = capi.trick_build([main])[0]
    assert (d / "video_fwd.ts").read_bytes() == fwd and (d / "video_rwd.ts").read_bytes() == rwd
    assert (d / "video.idx").read_bytes() == capi.build_video_idx(main, fwd, rwd)
    d2 = tmp_path / "q"
    d2.mkdir()
    subprocess.run([cli, "--encode", str(src), str(d2), "4", "12"], check=True, capture_output=True, timeout=300)
    assert (d2 / "video.ts").read_bytes() == capi.encode_build([pics], qscale_i=4, qscale_p=12)[0]
    bad = tmp_path / "bad.i420"
    bad.write_bytes(bytes(1000))
    assert subprocess.run([cli, "--encode", str(bad), str(d2)], capture_output=True, timeout=60).returncode == 1


def _play(ctx, packets):
    """one library submit of `packets` packets: (decoded pictures [n, I420], their pts)"""
    ctx.library_submit(packets=packets)
    ctx.index()
    n = ctx.stream_info(0)[0]
    out = np.zeros((ctx.max_pictures, 1, ec.PICTURE_BYTES), np.uint8)
    ctx.decode_all_to_host(ctx.index_info()["max_pictures"], out)
    ctx.sync()
    pts, _ = ctx.picture_pts()
    return out[:n, 0].copy(), pts[0, :n].tolist()


def test_library_round_trip(oracle):
    """an encoded title added to the library and given its trick files on the device: played from the start, skipped to a later
    GOP and fast-forwarded, every decoded picture is the encoder's reconstruction (or, fast-forwarding, the fwd file's picture) with
    the requested pts"""
    import espflix_b200
    from tests import pts_cases
    capi = _capi()
    pics = ec.translated(11, 40, (1, 1))
    ts = capi.encode_build([pics], pts0=900, pts_step=3750)[0]
    rec = ec.encode_title(pics, oracle, pts0=900, pts_step=3750)[2]
    ctx = espflix_b200.Context(n_streams=1, max_pictures=64, max_slices_per_picture=12, es_capacity=len(ts) + (1 << 16), fields=False)
    ctx.enable_pts()
    ctx.enable_carry(1 << 17)
    assert ctx.library_add(capi.build_video_idx(ts, b"", b""), ts) == 0
    ctx.library_add_trick(0)
    ctx.library_command(capi.LIB_PLAY_AT, 0, 1, 0, 900)
    got, pts = _play(ctx, len(ts) // 188)
    assert len(got) >= 39
    assert np.array_equal(got, rec[:len(got)]) and pts == [900 + 3750 * k for k in range(len(got))]
    # skip: PLAY_AT a position inside the third GOP starts at a GOP's first picture at or before it
    ctx.library_command(capi.LIB_PLAY_AT, 0, 1, 0, 900 + 27 * 3750)
    got, pts = _play(ctx, len(ts) // 188)
    k0 = (pts[0] - 900) // 3750
    assert len(got) > 0 and k0 % 12 == 0 and 12 <= k0 <= 27
    assert np.array_equal(got, rec[k0:k0 + len(got)]) and pts == [900 + 3750 * (k0 + k) for k in range(len(got))]
    # fast-forward: the pictures of video_fwd.ts, as the oracle decodes that file
    fwd = ctx.library_read(0, 2)
    want = dict(zip(pts_cases.picture_pts(fwd), oracle.decode_ts(fwd, max_frames=64)))
    ctx.library_command(capi.LIB_FAST_FORWARD, 0, 1)
    seen = 0
    for _ in range(3):
        got, pts = _play(ctx, len(fwd) // 188 + 1)
        for f, p in zip(got, pts):
            assert p in want and np.array_equal(f, want[p])
            seen += 1
    assert seen > 0 and ctx.library_info()[0]["speed"] == 1
    ctx.close()
