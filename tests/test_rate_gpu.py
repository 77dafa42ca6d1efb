"""ef_encode_build_rate against the restatement (tests/rate_cases.py): video.ts byte for byte with every picture's quantiser and
bytes, batches past one decode context, the argument checks, the CLI and a rate-encoded title with audio through the library."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import encode_cases as ec
from tests import rate_cases as rc
from tests.oracle_lib import Oracle

pytestmark = pytest.mark.gpu


def _capi():
    from espflix_b200 import capi
    return capi


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def _check(oracle, titles, **params):
    got = _capi().encode_build_rate(titles, **params)
    assert len(got) == len(titles)
    for t, (pics, (ts, q, nb)) in enumerate(zip(titles, got)):
        want, es, _, chosen, _ = rc.encode_title(pics, oracle, **params)
        assert list(q) == chosen, (t, params)
        assert list(nb) == [len(e) for e in es], (t, params)
        assert len(ts) == len(want) and ts == want, "title %d (%d pictures, %s): first difference at byte %s" % (
            t, len(pics), params, next((i for i in range(min(len(ts), len(want))) if ts[i] != want[i]), min(len(ts), len(want))))
    return got


@pytest.mark.parametrize("params", [{}, dict(bit_rate=300000), dict(bit_rate=800000, vbv_bits=60000, qmin=2, qmax=20)])
def test_fixture_vmedia(oracle, params):
    _check(oracle, [ec.fixture_pictures("vmedia", oracle)], **params)


def test_fixture_splash(oracle):
    _check(oracle, [ec.fixture_pictures("splash", oracle)[:30]], bit_rate=400000, vbv_bits=40000)


@pytest.mark.parametrize("case", ["static", "half", "cut", "noise", "checker1", "checker8"])
@pytest.mark.parametrize("params", [{}, dict(bit_rate=700000, vbv_bits=40000, qmin=1, qmax=31), dict(qmin=5, qmax=5),
                                    dict(bit_rate=2000000, vbv_bits=500000, qmin=8, qmax=24, gop=5)])
def test_synthetic(oracle, case, params):
    pics = {"static": lambda: ec.translated(1, 6, (0, 0), grain=0.0), "half": lambda: ec.translated(3, 6, (1, 3)),
            "cut": lambda: ec.scene_cut(4, 6, 3), "noise": lambda: ec.noise(7, 4), "checker1": lambda: ec.checkerboard(4, cell=1),
            "checker8": lambda: ec.checkerboard(4, cell=8, phase=1)}[case]()
    _check(oracle, [pics], **params)


@pytest.mark.parametrize("gop", [1, 12, 13])
def test_title_lengths_and_gops(oracle, gop):
    """titles of different lengths in one call, short last GOPs, at a bucket tight enough to use the fallbacks of noise"""
    src = np.concatenate([ec.translated(9, 14, (2, 1)), ec.noise(5, 4), ec.translated(12, 8, (-3, 2))])
    titles = [src[:n] for n in (1, 11, 12, 13, 26)]
    _check(oracle, titles, gop=gop, bit_rate=900000, vbv_bits=200000, aspect=3, rate=5, pts0=1000, pts_step=3003)


def test_fallbacks(oracle):
    """a bucket that forces both fallbacks on noise: the file still decodes and holds the bucket"""
    pics = ec.noise(3, 5)
    got = _check(oracle, [pics], bit_rate=1000000, vbv_bits=40000, qmin=30, qmax=31)[0]
    ts, q, nb = got
    assert q[0] == 0 and (q[1:] == 0).any()
    assert rc.bucket_violations(ts, 1000000, 40000, 3750)[0] == []
    assert len(oracle.decode_ts(ts, max_frames=8)) == len(pics)


def test_batch_boundary(oracle):
    """more GOPs than one batch of the internal decode context: 513 GOPs in titles of three lengths, the last GOP of each title ending
    at an empty buffer"""
    clips = [ec.translated(10 + i, n, (2 * i, -i)) for i, n in enumerate((2, 3, 5))]
    order = [(g * 7) % 3 for g in range(300)]
    titles = [clips[i] for i in order]
    assert sum((len(t) + 1) // 2 for t in titles) > 512
    got = _capi().encode_build_rate(titles, gop=2, bit_rate=1000000, vbv_bits=100000)
    want = [rc.encode_title(c, oracle, gop=2, bit_rate=1000000, vbv_bits=100000) for c in clips]
    for (ts, q, nb), i in zip(got, order):
        assert ts == want[i][0] and list(q) == want[i][3] and list(nb) == [len(e) for e in want[i][1]]


def test_errors():
    capi = _capi()
    lib = capi.load_library()
    pics = np.zeros((2, ec.PICTURE_BYTES), np.uint8)
    off = np.array([0, 2], np.uint64)
    to = np.zeros(2, np.uint64)
    out = np.zeros(1 << 20, np.uint8)
    q = np.zeros(2, np.uint8)
    nb = np.zeros(2, np.uint32)

    def call(n=1, off_=off, ts=out, cap=out.size, rp=None, **kw):
        p = capi.EncodeParams(**dict(capi.ENCODE_DEFAULTS, **kw))
        r = capi.RateParams(**dict(capi.ENCODE_RATE_DEFAULTS, **(rp or {})))
        return lib.ef_encode_build_rate(0, pics.ctypes.data, off_.ctypes.data, n, ctypes.byref(p), ctypes.byref(r),
                                        ts.ctypes.data if ts is not None else None, cap, to.ctypes.data, q.ctypes.data, nb.ctypes.data)
    assert call() == capi.EF_OK
    need = int(to[-1])
    assert call(gop=1024) == capi.EF_OK
    assert call(qscale_i=0, qscale_p=99) == capi.EF_OK                  # not read
    for kw in [dict(gop=0), dict(gop=1025), dict(search=-1), dict(search=16), dict(aspect=0), dict(aspect=15), dict(rate=0), dict(rate=9),
               dict(pts0=-1), dict(pts0=(1 << 33) - 3750)]:
        assert call(**kw) == capi.EF_EINVAL, kw
    for r in [dict(bit_rate=399), dict(bit_rate=400 * 0x3FFFE + 1), dict(vbv_bits=0), dict(vbv_bits=1023 * 16384 + 1), dict(qmin=0),
              dict(qmax=32), dict(qmin=9, qmax=8)]:
        assert call(rp=r) == capi.EF_EINVAL, r
    assert call(rp=dict(bit_rate=400 * 0x3FFFE, vbv_bits=1023 * 16384, qmin=31, qmax=31)) == capi.EF_OK
    assert call(n=0) == capi.EF_EINVAL
    assert call(off_=np.array([0, 0], np.uint64)) == capi.EF_EINVAL
    assert lib.ef_encode_build_rate(0, pics.ctypes.data, off.ctypes.data, 1, ctypes.byref(capi.EncodeParams(**capi.ENCODE_DEFAULTS)), None,
                                    out.ctypes.data, out.size, to.ctypes.data, None, None) == capi.EF_EINVAL
    # the guarantee's boundary: the smallest bucket the rule accepts, and one bit less
    for gop in (1, 2, 12, 13):
        for R in (700000, 1500000):
            B = next(b for b in range(1, 1023 * 16384) if rc.check(gop, R, b, 3, 31, 3750) is None) if gop > 1 else None
            if gop == 1:                                        # GOP 1: the I fallback must fit one refill
                assert (rc.check(1, R, 250000, 3, 31, 3750) is None) == (rc.D_MAX * 8 * 90000 <= R * 3750)
                assert call(gop=1, rp=dict(bit_rate=R)) == (capi.EF_OK if rc.check(1, R, 250000, 3, 31, 3750) is None else capi.EF_EINVAL)
                continue
            assert call(gop=gop, rp=dict(bit_rate=R, vbv_bits=B)) == capi.EF_OK, (gop, R, B)
            assert call(gop=gop, rp=dict(bit_rate=R, vbv_bits=B - 1)) == capi.EF_EINVAL, (gop, R, B)
    R1 = -(-rc.D_MAX * 8 * 90000 // 3750)                       # GOP 1's lowest rate at the default pts step
    assert call(gop=1, rp=dict(bit_rate=R1)) == capi.EF_OK and call(gop=1, rp=dict(bit_rate=R1 - 1)) == capi.EF_EINVAL
    out[:] = 0xAA
    to[:] = 0
    assert call(cap=need - 1) == capi.EF_ENOMEM and int(to[-1]) == need and (out == 0xAA).all()
    assert call(ts=None, cap=0) == capi.EF_ENOMEM and int(to[-1]) == need


def test_indexer_cli_rate(oracle, tmp_path):
    """ef_indexer_cli --encode ... --rate bit_rate vbv_bits [--audio pcm]: video.ts equal to capi's, then the trick files and video.idx"""
    capi = _capi()
    cli = os.path.join(ec.ROOT, "espflix_b200", "host", "ef_indexer_cli")
    pics = ec.fixture_pictures("vmedia", oracle)[:30]
    src = tmp_path / "pictures.i420"
    src.write_bytes(pics.tobytes())
    d = tmp_path / "title"
    d.mkdir()
    subprocess.run([cli, "--encode", str(src), str(d), "--rate", "600000", "80000"], check=True, capture_output=True, timeout=300)
    main = (d / "video.ts").read_bytes()
    assert main == capi.encode_build_rate([pics], bit_rate=600000, vbv_bits=80000)[0][0]
    fwd, rwd = capi.trick_build([main])[0]
    assert (d / "video_fwd.ts").read_bytes() == fwd and (d / "video_rwd.ts").read_bytes() == rwd
    assert (d / "video.idx").read_bytes() == capi.build_video_idx(main, fwd, rwd)
    pcm = (np.sin(np.arange(48000 * 2) * 0.05) * 8000).astype(np.int16)
    (tmp_path / "pcm.s16le").write_bytes(pcm.tobytes())
    d2 = tmp_path / "audio"
    d2.mkdir()
    subprocess.run([cli, "--encode", str(src), str(d2), "--rate", "600000", "80000", "--audio", str(tmp_path / "pcm.s16le")], check=True,
                   capture_output=True, timeout=300)
    assert (d2 / "video.ts").read_bytes() == capi.encode_title(pics, pcm, rate=dict(bit_rate=600000, vbv_bits=80000))
    assert subprocess.run([cli, "--encode", str(src), str(d2), "--rate", "100", "80000"], capture_output=True, timeout=60).returncode == 1


def _play(ctx, packets):
    ctx.library_submit(packets=packets)
    ctx.index()
    n = ctx.stream_info(0)[0]
    out = np.zeros((ctx.max_pictures, 1, ec.PICTURE_BYTES), np.uint8)
    ctx.decode_all_to_host(ctx.index_info()["max_pictures"], out)
    ctx.sync()
    pts, _ = ctx.picture_pts()
    return out[:n, 0].copy(), pts[0, :n].tolist()


def test_library_round_trip_with_audio(oracle):
    """a rate-encoded title with audio added to the library and given its trick files on the device: played from the start, skipped
    to a later GOP and fast-forwarded, every decoded picture is the restatement's reconstruction (or the fwd file's picture)"""
    import espflix_b200
    from tests import pts_cases
    capi = _capi()
    pics = ec.translated(11, 40, (1, 1))
    pcm = (np.sin(np.arange(48000 * 2) * 0.03) * 6000).astype(np.int16)
    rate = dict(bit_rate=500000, vbv_bits=60000)
    ts = capi.encode_title(pics, pcm, rate=rate, pts0=900, pts_step=3750)
    video, _, rec, _, _ = rc.encode_title(pics, oracle, pts0=900, pts_step=3750, **rate)
    assert ts != video and pts_cases.demux(ts)[0] == pts_cases.demux(video)[0]
    ctx = espflix_b200.Context(n_streams=1, max_pictures=64, max_slices_per_picture=12, es_capacity=len(ts) + (1 << 16), fields=False)
    ctx.enable_pts()
    ctx.enable_carry(1 << 17)
    assert ctx.library_add(capi.build_video_idx(ts, b"", b""), ts) == 0
    ctx.library_add_trick(0)
    ctx.library_command(capi.LIB_PLAY_AT, 0, 1, 0, 900)
    got, pts = _play(ctx, len(ts) // 188)
    assert len(got) >= 39
    assert np.array_equal(got, rec[:len(got)]) and pts == [900 + 3750 * k for k in range(len(got))]
    ctx.library_command(capi.LIB_PLAY_AT, 0, 1, 0, 900 + 27 * 3750)
    got, pts = _play(ctx, len(ts) // 188)
    k0 = (pts[0] - 900) // 3750
    assert len(got) > 0 and k0 % 12 == 0 and 12 <= k0 <= 27
    assert np.array_equal(got, rec[k0:k0 + len(got)]) and pts == [900 + 3750 * (k0 + k) for k in range(len(got))]
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
