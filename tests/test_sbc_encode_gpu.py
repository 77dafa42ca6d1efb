"""ef_sbc_encode and ef_mux_audio against the restatement (tests/sbc_encode_cases.py): SBC and muxed video.ts byte for byte, the
argument checks, and the encoded audio through the device decoder."""
import numpy as np
import pytest

from tests import encode_cases as ec
from tests import pts_cases
from tests import sbc_encode_cases as se
from tests import trick_cases as tc

pytestmark = pytest.mark.gpu


def _capi():
    from espflix_b200 import capi
    return capi


def _first_diff(a, b):
    return next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), min(len(a), len(b)))


def _check(pcms, **params):
    p = dict(se.DEFAULTS, **params)
    got = _capi().sbc_encode(pcms, **p)
    for k, (x, g) in enumerate(zip(pcms, got)):
        want = se.encode(x, p["frequency"], p["allocation"], p["bitpool"])
        assert g == want, "stream %d (%d samples, %s): first difference at byte %d" % (k, len(x), params, _first_diff(g, want))
    return got


def test_directed_cases_one_call_each():
    for name, x in se.pcm_cases().items():
        _check([x])
    for bp in (128, 2):
        _check(list(se.pcm_cases().values()), bitpool=bp)


def test_parameter_sweep():
    for f, a, b in se.sweep():
        _check([se.sweep_pcm(f)], frequency=f, allocation=a, bitpool=b)


def test_fixture_audio_at_its_own_header(oracle):
    for name, (fq, bp) in (("splash", (3, 28)), ("vmedia", (1, 20))):
        pcm, _ = se.fixture_pcm(name, oracle)
        _check([pcm], frequency=fq, bitpool=bp)


def test_batch_with_empty_titles():
    c = list(se.pcm_cases().values())
    batch = [np.zeros(0, np.int16)] + c[:5] + [np.zeros(0, np.int16)] * 3 + c[5:] + [np.zeros(0, np.int16)]
    got = _check(batch, bitpool=60)
    assert all(g == b"" for x, g in zip(batch, got) if len(x) == 0)


def test_more_than_one_launch():
    """2^18 frames per launch: a call of 600,000 frames over three titles; the frames around every launch and title boundary against
    the restatement of the samples they read (frames are independent: a window starting a frame early gives the same frame)"""
    rng = np.random.default_rng(5)
    lens = [128 * 250000 + 17, 128 * 200000, 128 * 150000 - 3]
    pcms = [rng.integers(-30000, 30000, n).astype(np.int16) for n in lens]
    got = _capi().sbc_encode(pcms)
    fb = se.frame_bytes(28)
    first = np.cumsum([0] + [se.n_frames(n) for n in lens])
    checks = set()
    for g in (1 << 18, 2 << 18):
        checks.update(range(g - 2, g + 2))
    for t in range(3):
        checks.update([int(first[t]), int(first[t]) + 1, int(first[t + 1]) - 1])
    for gf in sorted(checks):
        t = int(np.searchsorted(first, gf, side="right") - 1)
        f = gf - int(first[t])
        assert len(got[t]) == se.n_frames(lens[t]) * fb
        lo = max(f - 1, 0)
        want = se.encode(pcms[t][128 * lo:128 * (f + 1)])[(f - lo) * fb:(f - lo + 1) * fb]
        assert got[t][f * fb:(f + 1) * fb] == want, (t, f)


def test_batch_scale_4096_titles():
    rng = np.random.default_rng(4096)
    pcms = [rng.integers(-25000, 25000, int(n)).astype(np.int16) for n in rng.integers(0, 400, 4096)]
    got = _capi().sbc_encode(pcms)
    for k, (x, g) in enumerate(zip(pcms, got)):
        assert g == se.encode(x), k


def test_sizing_and_errors():
    import ctypes
    capi = _capi()
    lib = capi.load_library()
    x = np.arange(300, dtype=np.int16)
    off = np.array([0, 300], dtype=np.uint64)
    so = np.zeros(2, dtype=np.uint64)
    par = capi.AudioParams(**capi.AUDIO_ENCODE_DEFAULTS)
    assert lib.ef_sbc_encode(0, x.ctypes.data, off.ctypes.data, 1, ctypes.byref(par), None, 0, so.ctypes.data) == capi.EF_ENOMEM
    assert list(so) == [0, 3 * 64]
    buf = np.full(3 * 64, 7, np.uint8)
    assert lib.ef_sbc_encode(0, x.ctypes.data, off.ctypes.data, 1, ctypes.byref(par), buf.ctypes.data, buf.size - 1, so.ctypes.data) == capi.EF_ENOMEM
    assert (buf == 7).all()
    for bad in (dict(frequency=4), dict(frequency=-1), dict(allocation=2), dict(bitpool=1), dict(bitpool=129)):
        q = capi.AudioParams(**dict(capi.AUDIO_ENCODE_DEFAULTS, **bad))
        assert lib.ef_sbc_encode(0, x.ctypes.data, off.ctypes.data, 1, ctypes.byref(q), buf.ctypes.data, buf.size, so.ctypes.data) == capi.EF_EINVAL, bad
    dec = np.array([0, 300, 200], dtype=np.uint64)
    assert lib.ef_sbc_encode(0, x.ctypes.data, dec.ctypes.data, 2, ctypes.byref(par), buf.ctypes.data, buf.size, so.ctypes.data) == capi.EF_EINVAL
    assert lib.ef_sbc_encode(0, x.ctypes.data, off.ctypes.data, 0, ctypes.byref(par), buf.ctypes.data, buf.size, so.ctypes.data) == capi.EF_EINVAL


def test_device_decoder_equals_oracle(oracle):
    c = se.pcm_cases()
    sbcs = _capi().sbc_encode([c["chirp"], c["noise"], c["square"]], bitpool=97)
    for s, d in zip(sbcs, _capi().audio_decode(sbcs, pdm=False)):
        assert np.array_equal(d["pcm"], oracle.sbc_decode(np.frombuffer(s, np.uint8)))


# ---- mux ---------------------------------------------------------------------------------------------------------------------------------
def _stripped(name):
    ts = tc.fixture(name)
    return b"".join(ts[k:k + 188] for k in range(0, len(ts), 188) if (((ts[k + 1] << 8) | ts[k + 2]) & 0x1FFF) not in (0x101, 0x102))


def _videos(oracle):
    pics = ec.translated(2, 26, (2, -1))
    enc = _capi().encode_build([pics])[0]
    fwd, rwd = _capi().trick_build([enc])[0]
    return {"encoded": enc, "fwd": fwd, "rwd": rwd, "splash": _stripped("splash"), "vmedia": _stripped("vmedia")}


def test_mux_equals_restatement(oracle):
    vids = _videos(oracle)
    rng = np.random.default_rng(9)
    names = list(vids)
    for params in (dict(), dict(frames_per_pes=1, pts0=4000), dict(bitpool=20, frequency=1), dict(frames_per_pes=3, bitpool=128)):
        p = dict(se.DEFAULTS, **params)
        fs = se.FS_HZ[p["frequency"]]
        sbcs = []
        for n in names:
            secs = len(pts_cases.picture_pts(vids[n])) / 24.0 + 0.3
            sbcs.append(_capi().sbc_encode([rng.integers(-8000, 8000, int(secs * fs)).astype(np.int16)], **params)[0])
        sbcs[1] = b""                                          # an empty audio stream leaves its video as it is
        got = _capi().mux_audio([vids[n] for n in names], sbcs, **params)
        for n, s, g in zip(names, sbcs, got):
            want = se.mux(vids[n], s, **params)
            assert g == want, (n, params, _first_diff(g, want))
            assert bytes(oracle.demux_audio_ts(np.frombuffer(g, np.uint8))) == s
            assert pts_cases.picture_pts(g) == pts_cases.picture_pts(vids[n])
        assert got[1] == vids[names[1]]


def test_mux_errors():
    import ctypes
    capi = _capi()
    lib = capi.load_library()
    vid = capi.encode_build([ec.translated(2, 3, (2, -1))])[0]
    sbc = capi.sbc_encode([np.zeros(1280, np.int16)])[0]

    def rc(ts, s, **params):
        tb, to = capi.Context.pack([ts])
        sb, so = capi.Context.pack([s])
        oo = np.zeros(2, dtype=np.uint64)
        par = capi.AudioParams(**dict(capi.AUDIO_ENCODE_DEFAULTS, **params))
        out = np.zeros(len(ts) + 188 * 64, np.uint8)
        return lib.ef_mux_audio(0, tb.ctypes.data, to.ctypes.data, sb.ctypes.data, so.ctypes.data, 1, ctypes.byref(par), out.ctypes.data,
                                out.size, oo.ctypes.data)
    assert rc(vid, sbc) == 0
    with_audio = _capi().mux_audio([vid], [sbc])[0]
    assert rc(with_audio, sbc) == capi.EF_EINVAL
    b = bytearray(vid)
    b[4 + 7] &= 0x7F                                             # the first video PES loses its PTS flag
    assert rc(bytes(b), sbc) == capi.EF_EINVAL
    assert rc(vid[:-1], sbc) == capi.EF_EINVAL
    assert rc(vid, sbc[:-1]) == capi.EF_EINVAL
    assert rc(vid, sbc, pts0=(1 << 33) - 100) == capi.EF_EINVAL
    assert rc(vid, sbc, frames_per_pes=(65535 - 8) // 64 + 1) == capi.EF_EINVAL
    assert rc(vid, sbc, frames_per_pes=(65535 - 8) // 64) == 0
    tb, to = capi.Context.pack([vid])
    sb, so = capi.Context.pack([sbc])
    oo = np.zeros(2, dtype=np.uint64)
    par = capi.AudioParams(**capi.AUDIO_ENCODE_DEFAULTS)
    assert lib.ef_mux_audio(0, tb.ctypes.data, to.ctypes.data, sb.ctypes.data, so.ctypes.data, 1, ctypes.byref(par), None, 0, oo.ctypes.data) == capi.EF_ENOMEM
    assert int(oo[1]) == len(se.mux(vid, sbc))


def test_encode_title_plays_through_the_decoder(oracle):
    pics = ec.translated(2, 24, (2, -1))
    pcm = se.sine(48000, 1000, 48000, 8000)
    ts = _capi().encode_title(pics, pcm)
    video = _capi().encode_build([pics])[0]
    sbc = se.encode(pcm)
    assert ts == se.mux(video, sbc)
    assert np.array_equal(oracle.decode_ts(ts, max_frames=30), oracle.decode_ts(video, max_frames=30))
    es = oracle.demux_audio_ts(np.frombuffer(ts, np.uint8))
    assert bytes(es) == sbc
    assert np.array_equal(_capi().audio_decode([sbc], pdm=False)[0]["pcm"], oracle.sbc_decode(es))


# ---- an encoded title with audio through the product -------------------------------------------------------------------------------
def _titles_with_audio(n=2):
    """n encoded titles (pictures, video-only ts, SBC, ts with audio), each with a second of audio more than its pictures last"""
    out = []
    for i in range(n):
        pics = ec.translated(3 + i, 24 + 6 * i, (2 - i, -1))
        video = _capi().encode_build([pics])[0]
        pcm = se.sine(48000 * (1 + len(pics) // 24) + 77 * i, 440 * (i + 1), 48000, 6000 + 1000 * i)
        sbc = _capi().sbc_encode([pcm])[0]
        out.append((pics, video, sbc, _capi().mux_audio([video], [sbc])[0]))
    return out


def test_encoded_title_through_context_whole_and_cut():
    """titles with audio on a context with enable_audio() and enable_pts(): submitted whole and cut at seeded packets with carry,
    their pictures and pts equal the video-only titles', and the concatenated decode_audio() PCM equals audio_decode of the SBC"""
    import espflix_b200
    from tests import carry_cases
    from tests.harness import sha, submits
    from tests.test_carry_gpu import Run, _carrying, _index_and_read, _whole
    titles = _titles_with_audio()
    progs = [t[3] for t in titles]
    video = _whole([t[1] for t in titles])
    want = _capi().audio_decode([t[2] for t in titles], pdm=False)
    # whole
    ctx = espflix_b200.Context(n_streams=len(progs), max_pictures=100, max_slices_per_picture=12, es_capacity=1 << 23, fields=False)
    ctx.enable_pts()
    ctx.enable_audio()
    ctx.submit_ts(*ctx.pack(progs))
    ctx.index()
    counts = [ctx.stream_info(s)[0] for s in range(len(progs))]
    frames = [[] for _ in progs]
    for p in range(max(counts)):
        ctx.decode_picture(p)
        for s in range(len(progs)):
            if p < counts[s]:
                frames[s].append(sha(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1)))
    pic, _ = ctx.picture_pts()
    out = ctx.decode_audio(end=True, pdm=False)
    ctx.close()
    for s in range(len(progs)):
        assert frames[s] == video.frames[s] and [int(v) for v in pic[s, :counts[s]]] == video.pts[s]
        assert np.array_equal(out[s]["pcm"], want[s]["pcm"]) and len(want[s]["pcm"]) > 0
    # cut at seeded packets, carried across submits
    per_stream = [carry_cases.cut(ts, carry_cases.seeded_cuts(ts, 700 + i, 23)) for i, ts in enumerate(progs)]
    ctx = _carrying(len(progs))
    ctx.enable_audio()
    run = Run(len(progs))
    pcm = [[] for _ in progs]
    for k, chunk in enumerate(submits(per_stream)):
        ctx.submit_ts(*ctx.pack(chunk))
        last = np.array([k == len(per_stream[s]) - 1 for s in range(len(progs))], dtype=np.uint8)
        if last.any():
            ctx.end_streams(last)
        _index_and_read(ctx, run, len(progs))
        for s, r in enumerate(ctx.decode_audio(end=last, pdm=False)):
            pcm[s].append(r["pcm"])
    ctx.close()
    for s in range(len(progs)):
        assert run.frames[s] == video.frames[s] and run.pts[s] == video.pts[s]
        assert np.array_equal(np.concatenate(pcm[s]), want[s]["pcm"])


def test_encoded_title_with_audio_in_the_library(oracle):
    """library_add + library_add_trick on a title with audio: the trick files equal those of the video-only title, and PLAY, SKIP and
    FAST_FORWARD resolve through the rebuilt video.idx to the encoder's reconstructions and the fwd file's pictures"""
    import espflix_b200
    from tests.test_encode_gpu import _play
    capi = _capi()
    pics = ec.translated(11, 40, (1, 1))
    ts = capi.encode_title(pics, se.sine(48000 * 3, 660, 48000, 7000), pts0=900)
    video = capi.encode_build([pics], pts0=900)[0]
    rec = ec.encode_title(pics, oracle, pts0=900)[2]
    ctx = espflix_b200.Context(n_streams=1, max_pictures=64, max_slices_per_picture=12, es_capacity=len(ts) + (1 << 16), fields=False)
    ctx.enable_pts()
    ctx.enable_carry(1 << 17)
    assert ctx.library_add(capi.build_video_idx(ts, b"", b""), ts) == 0
    ctx.library_add_trick(0)
    fwd, rwd = capi.trick_build([video])[0]
    assert ctx.library_read(0, 1) == ts and ctx.library_read(0, 2) == fwd and ctx.library_read(0, 0) == rwd
    assert ctx.library_read(0, -1) == capi.build_video_idx(ts, fwd, rwd)
    ctx.library_command(capi.LIB_PLAY_AT, 0, 1, 0, 900)
    got, pts = _play(ctx, len(ts) // 188)
    assert len(got) >= 39
    assert np.array_equal(got, rec[:len(got)]) and pts == [900 + 3750 * k for k in range(len(got))]
    ctx.library_command(capi.LIB_PLAY_AT, 0, 1, 0, 900 + 27 * 3750)
    got, pts = _play(ctx, len(ts) // 188)
    k0 = (pts[0] - 900) // 3750
    assert len(got) > 0 and k0 % 12 == 0 and 12 <= k0 <= 27
    assert np.array_equal(got, rec[k0:k0 + len(got)]) and pts == [900 + 3750 * (k0 + k) for k in range(len(got))]
    want = dict(zip(pts_cases.picture_pts(fwd), oracle.decode_ts(fwd, max_frames=64)))
    ctx.library_command(capi.LIB_FAST_FORWARD, 0, 1)
    seen = 0
    for _ in range(3):
        got, pts = _play(ctx, len(fwd) // 188 + 1)
        for f, p in zip(got, pts):
            assert p in want and np.array_equal(f, want[p])
            seen += 1
    assert seen > 0
    ctx.close()


def test_indexer_cli_encode_with_audio(oracle, tmp_path):
    """ef_indexer_cli --encode pictures title_dir --audio pcm: video.ts is the restated title with audio (whose reference playback
    tests/test_sbc_encode.py pins), the trick files are the video-only title's, video.idx is build_video_idx of the three files"""
    import os
    import subprocess
    from tests import test_sbc_encode as ts_cpu
    capi = _capi()
    cli = os.path.join(ec.ROOT, "espflix_b200", "host", "ef_indexer_cli")
    pics, pcm = ts_cpu.cli_title(oracle)
    src, snd = tmp_path / "pictures.i420", tmp_path / "sound.s16le"
    src.write_bytes(pics.tobytes())
    snd.write_bytes(pcm.astype("<i2").tobytes())
    d = tmp_path / "title"
    d.mkdir()
    subprocess.run([cli, "--encode", str(src), str(d), "--audio", str(snd)], check=True, capture_output=True, timeout=300)
    main = (d / "video.ts").read_bytes()
    assert main == ts_cpu.cli_title_ts(oracle)
    fwd, rwd = capi.trick_build([capi.encode_build([pics])[0]])[0]
    assert (d / "video_fwd.ts").read_bytes() == fwd and (d / "video_rwd.ts").read_bytes() == rwd
    assert (d / "video.idx").read_bytes() == capi.build_video_idx(main, fwd, rwd)
    d2 = tmp_path / "q"
    d2.mkdir()
    subprocess.run([cli, "--encode", str(src), str(d2), "4", "12", "--audio", str(snd)], check=True, capture_output=True, timeout=300)
    assert (d2 / "video.ts").read_bytes() == se.mux(capi.encode_build([pics], qscale_i=4, qscale_p=12)[0], se.encode(pcm))
    odd = tmp_path / "odd.s16le"
    odd.write_bytes(bytes(3))
    assert subprocess.run([cli, "--encode", str(src), str(d2), "--audio", str(odd)], capture_output=True, timeout=60).returncode == 1
