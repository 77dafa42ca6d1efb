"""The TS, PTS, audio, composite and paced-field paths at the benchmark's batch size (tests/scale_cases.py: 4,096 streams,
period 335), every stream checked. The 67 distinct streams are held to the C restatement (tests/oracle_lib.py) and the
Python restatements (tests/pts_cases.py, tests/present_cases.py); every other stream to its distinct original, value for
value. Past 1,024 streams the offsets scan of TS submits and of the audio input runs over several tiles, the composite
kernels pick each stream's latest frame store from thousands of different ones, and one paced K2 call needs more than one
launch: the code the small batches of the other tests never reach."""
import math

import numpy as np
import pytest

import espflix_b200
from tests import present_cases as pc
from tests import pts_cases, scale_cases
from tests.harness import present_call, presenting_context
from tests.scale_cases import D, N, PICTURES

I420 = 101376


def _where(s):
    return "stream %d (distinct %d)" % (s, s % D)


def test_batch_builder():
    """the batch's period is coprime to the scan tile, stream k and k + 1024 differ, and replicas of one distinct stream
    carry the same ES, PES-to-picture relation, audio, modes and frame-counter parity"""
    from tests.oracle_lib import Oracle
    b = scale_cases.batch()
    o = Oracle()
    assert scale_cases.period_is_coprime_to_tiles() and math.gcd(scale_cases.PERIOD, 1024) == 1
    for k in range(N - 1024):
        assert b.ts(k) != b.ts(k + 1024), k
    for d in range(D):
        replicas = {b.ts(k) for k in range(d, N, D)}                 # replicas differ in their packetisation and length
        assert len(replicas) == scale_cases.V and len({len(t) for t in replicas}) > 2, d
        want_pts = pts_cases.picture_pts(b.ts(d))
        assert want_pts == b.pts[d], d
        for v in range(scale_cases.V):
            t = b.var[d, v]
            es, pes = pts_cases.demux(t)
            assert es == b.es[d], (d, v)
            assert pts_cases.picture_pts(t) == want_pts, (d, v)
            assert np.array_equal(o.demux_audio_ts(t), b.audio[d]), (d, v)
            assert b.var_cuts[d, v], (d, v)
            for c, n_before in b.var_cuts[d, v]:
                assert 0 < n_before < PICTURES and len(pts_cases.picture_codes(pts_cases.demux(t[:188 * c])[0])) == n_before
    for k in range(N):
        d = k % D
        assert b.modes(k) == b.modes(d) and b.fc0(k) % 2 == b.fc0(d) % 2


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def batch():
    return scale_cases.batch()


@pytest.fixture(scope="module")
def frames(batch, oracle):
    """the 12 pictures of every distinct stream, by the C restatement"""
    out = []
    for d in range(D):
        f = oracle.decode_es(batch.es[d])
        assert f.shape[0] == PICTURES, d
        out.append(f)
    return out


@pytest.fixture(scope="module")
def packed(batch):
    return espflix_b200.Context.pack(batch.all_ts())


def _split(batch, salt=0):
    """every stream's TS cut in two at a picture-boundary packet chosen with k -> (parts [2][N], pictures in part 0)"""
    a, b, n0 = [], [], []
    for k in range(N):
        c, n = batch.cut(k, salt)
        t = batch.ts(k)
        a.append(t[:188 * c])
        b.append(t[188 * c:])
        n0.append(n)
    return [a, b], n0


def _context(fields, es_capacity, **kw):
    return espflix_b200.Context(n_streams=N, max_pictures=PICTURES, max_slices_per_picture=12, es_capacity=es_capacity, fields=fields, **kw)


def _check_counts(ctx, batch, n_pics, base, es_bytes=None, tag=""):
    info = ctx.index_info()
    assert info["max_pictures"] == max(n_pics), tag
    assert info["total_pictures"] == sum(n_pics), tag
    assert info["total_slices"] == 12 * sum(n_pics), tag
    if es_bytes is not None:
        assert info["es_bytes"] == es_bytes, tag
    for s in range(N):
        assert ctx.stream_info(s) == (n_pics[s], base[s]), "%s: %s" % (tag, _where(s))


def _check_latest(ctx, frames, latest, tag):
    """every stream's latest picture (read_latest_i420) is picture latest[s] of its distinct stream"""
    got = ctx.read_latest_i420(0, N)
    for s in range(N):
        assert np.array_equal(got[s], frames[s % D][latest[s]]), "%s: %s: latest picture %d" % (tag, _where(s), latest[s])


def _check_last_two(ctx, frames, tag):
    """every stream decoded all 12 pictures: 11 in frame store 0, 10 in store 1"""
    _check_latest(ctx, frames, [PICTURES - 1] * N, tag)
    for s in range(N):
        assert np.array_equal(ctx.read_frame_i420(s, 1), frames[s % D][PICTURES - 2]), "%s: %s: picture 10" % (tag, _where(s))


def _check_async_window(ctx, frames, tag):
    """read_latest_i420_async over streams 1000..1099, across the first tile boundary, into pinned memory"""
    import torch
    out = torch.empty((100, I420), dtype=torch.uint8, pin_memory=True)
    ctx.read_latest_i420_async(1000, 100, out.data_ptr())
    ctx.sync()
    got = out.numpy()
    for i in range(100):
        s = 1000 + i
        assert np.array_equal(got[i], frames[s % D][PICTURES - 1]), "%s: async read-back of %s" % (tag, _where(s))


@pytest.mark.gpu
def test_pts_of_every_picture(batch, packed):
    """picture_pts and get_pts of every stream, whole and cut in two"""
    want = np.array([batch.pts[s % D] for s in range(N)], dtype=np.int64)
    for d in range(D):                                             # the restatement, on the distinct streams' own TS
        assert pts_cases.picture_pts(batch.ts(d)) == batch.pts[d], d
    ctx = _context(False, int(packed[1][-1]) + 4096)
    ctx.enable_pts()
    ctx.submit_ts(*packed)
    ctx.index()
    pic, last = ctx.picture_pts()
    for s in np.nonzero((pic != want).any(axis=1))[0][:1]:
        pytest.fail("whole: %s: pts %s, want %s" % (_where(s), pic[s].tolist(), want[s].tolist()))
    bad = np.nonzero(last != want[:, -1])[0]
    assert bad.size == 0, "whole: get_pts of %s" % _where(bad[0])
    ctx.reset()
    parts, n0 = _split(batch, salt=1)
    got = np.full((N, PICTURES), -2, dtype=np.int64)
    for k, part in enumerate(parts):
        ctx.submit_ts(*ctx.pack(part))
        ctx.index()
        pic, last = ctx.picture_pts()
        for s in range(N):
            a, b = (0, n0[s]) if k == 0 else (n0[s], PICTURES)
            assert (pic[s, b - a:] == -1).all(), "cut part %d: %s" % (k, _where(s))
            got[s, a:b] = pic[s, :b - a]
            assert last[s] == want[s, b - 1], "cut part %d: get_pts of %s" % (k, _where(s))
    for s in np.nonzero((got != want).any(axis=1))[0][:1]:
        pytest.fail("cut: %s: pts %s, want %s" % (_where(s), got[s].tolist(), want[s].tolist()))
    ctx.close()


@pytest.mark.gpu
def test_audio_of_every_stream_across_submits(batch, oracle):
    """every stream's TS in 2 or 3 submits cut with k, the stream ended in the last call: PCM and PDM of every stream
    equal the C restatement of its whole audio"""
    want = []
    for d in range(D):
        pcm = oracle.sbc_decode(batch.audio[d])
        assert not isinstance(pcm, int) and pcm.size >= 100 * 128, d
        want.append((pcm, oracle.pdm(pcm)))
    K = 3
    chunks = [[], [], []]
    for k in range(N):
        t = batch.ts(k)
        cuts = sorted({batch.cut(k, 0)[0], batch.cut(k, 2)[0]}) if k % 3 else [batch.cut(k, 1)[0]]
        edges = [0] + cuts + [len(t) // 188]
        for j in range(K):
            chunks[j].append(t[188 * edges[j]:188 * edges[j + 1]] if j + 1 < len(edges) else b"")
    ctx = _context(False, max(sum(len(x) for x in c) for c in chunks) + 4096)
    ctx.enable_audio()
    pcm = [[] for _ in range(N)]
    pdm = [[] for _ in range(N)]
    for j in range(K):
        ctx.submit_ts(*ctx.pack(chunks[j]))
        ctx.index()
        res = ctx.decode_audio(end=[j == K - 1] * N)
        for s in range(N):
            pcm[s].append(res[s]["pcm"])
            pdm[s].append(res[s]["pdm"])
    ctx.close()
    for s in range(N):
        a, b = np.concatenate(pcm[s]), np.concatenate(pdm[s])
        w = want[s % D]
        assert a.size == w[0].size and np.array_equal(a, w[0]), "%s: PCM (%d samples, want %d)" % (_where(s), a.size, w[0].size)
        assert np.array_equal(b, w[1]), "%s: PDM" % _where(s)


# ---- paced presentation --------------------------------------------------------------------------------------------------
def _equal_rows(F, a, b, tag, where):
    """on the device: rows a[i] of F equal rows b[i]; where(i) names a failing pair"""
    import torch
    a = torch.as_tensor(np.asarray(a, dtype=np.int64), device="cuda")
    b = torch.as_tensor(np.asarray(b, dtype=np.int64), device="cuda")
    for i in range(0, a.numel(), 256):
        bad = (F[a[i:i + 256]] != F[b[i:i + 256]]).any(dim=1)
        if bool(bad.any()):
            pytest.fail("%s: %s differs from its original" % (tag, where(i + int(torch.nonzero(bad)[0, 0]))))


class _Paced:
    """drives a presenting context over the batch, and the restatement of the distinct streams alongside it"""

    def __init__(self, ctx, ntsc, batch, frames, oracle, n):
        self.ctx, self.b, self.n = ctx, batch, n
        self.disp = [pc.Display(ntsc, batch.fc0(d)) for d in range(min(n, D))]
        self.rend = [pc.Renderer(oracle, ntsc) for _ in range(min(n, D))]
        self.frames = frames

    def _expect(self, per_d, flips):
        """expected info of every stream from the distinct streams' fields -> numpy arrays"""
        idx = np.arange(self.n) % D
        nf = np.array([len(per_d[d]) for d in range(len(per_d))], dtype=np.int64)[idx]
        first = np.concatenate([[0], np.cumsum(nf)[:-1]])
        fc = np.array([f[0][0] if f else 0 for f in per_d], dtype=np.int64)[idx]
        return nf, first, fc, idx

    def call(self, fn, per_d, flips, tag):
        import torch
        info, fields = present_call(self.ctx, fn, device=True)
        nf, first, fc, idx = self._expect(per_d, flips)
        for name, got, want in (("n_fields", info["n_fields"], nf), ("first", info["first"], first)):
            bad = np.nonzero(got.astype(np.int64) != want)[0]
            assert bad.size == 0, "%s: %s of %s: %d, want %d" % (tag, name, _where(bad[0]), got[bad[0]], want[bad[0]])
        has = nf > 0
        bad = np.nonzero(has & (info["frame_counter"].astype(np.int64) != fc))[0]
        assert bad.size == 0, "%s: first frame counter of %s" % (tag, _where(bad[0]))
        bad = np.nonzero(info["flags"] != 0)[0]
        assert bad.size == 0, "%s: flags of %s" % (tag, _where(bad[0]))
        if flips is not None:
            ff = np.array([f[0] for f in flips], dtype=np.int64)[idx]
            fl = np.array([f[1] for f in flips], dtype=np.int64)[idx]
            bad = np.nonzero((info["flip_field"].astype(np.int64) != ff) | (info["flip_line"].astype(np.int64) != fl))[0]
            assert bad.size == 0, "%s: flip of %s" % (tag, _where(bad[0]))
        F = fields.view(torch.int16)
        nd = min(self.n, D)
        host = F[:int(first[nd - 1] + nf[nd - 1])].cpu().numpy().view(np.uint16)
        for d in range(nd):                                        # the distinct streams against the restatement
            for j, f in enumerate(per_d[d]):
                want = self.rend[d].field(f)
                diff = np.nonzero(host[first[d] + j] != want)[0]
                assert diff.size == 0, "%s: %s, field %d (%s): %d samples differ, first %d" % (tag, _where(d), j, f, diff.size, diff[0])
        a, b, who = [], [], []                                     # every other stream against its original, on the device
        for s in range(nd, self.n):
            d = s % D
            a += range(first[s], first[s] + nf[s])
            b += range(first[d], first[d] + nf[s])
            who += [(s, j) for j in range(nf[s])]
        if a:
            _equal_rows(F, a, b, tag, lambda i: "%s, field %d" % (_where(who[i][0]), who[i][1]))
        del F, fields
        torch.cuda.empty_cache()                                   # the next call's buffer has another size
        return info

    def picture(self, p, tag):
        modes = [self.b.modes(s)[p] for s in range(self.n)]
        per_d, flips = [], []
        for d in range(len(self.disp)):
            self.rend[d].decoded(p, self.frames[d][p])
            f, a, l_ = self.disp[d].push(self.b.pts[d][p], self.b.modes(d)[p])
            per_d.append(f)
            flips.append((a, l_))
        return self.call(lambda o: self.ctx.present_picture(p, modes, o), per_d, flips, "%s picture %d" % (tag, p))

    def idle(self, n_of, tag):
        per_d = [self.disp[d].idle(n_of(d)) for d in range(len(self.disp))]
        return self.call(lambda o: self.ctx.present_idle([n_of(s % D) for s in range(self.n)], o), per_d, None, "%s idle" % tag)


@pytest.mark.gpu
@pytest.mark.parametrize("ntsc", [1, 0])
def test_paced_fields_of_every_stream(batch, frames, packed, oracle, ntsc):
    """every stream presents its 12 pictures with its own frame counter, pts pattern and modes, then idles: every
    stream's present info against the restatement, the distinct streams' fields against its rendering by the C
    restatement, every other stream's fields against its original's"""
    import torch
    ctx = presenting_context(N, ntsc, [batch.fc0(s) for s in range(N)], max_pictures=PICTURES, es_capacity=int(packed[1][-1]) + 4096)
    ctx.submit_ts(*packed)
    ctx.index()
    r = _Paced(ctx, ntsc, batch, frames, oracle, N)
    tag = "ntsc" if ntsc else "pal"
    for p in range(PICTURES):
        r.picture(p, tag)
    r.idle(scale_cases.idle_fields, tag)
    ctx.close()
    torch.cuda.empty_cache()                                       # the field buffers of the calls


@pytest.mark.gpu
def test_paced_k2_split_over_launches(batch, frames, oracle):
    """one present_idle that emits 65,535 + 9 NTSC fields: the paced K2 runs in two launches, the second at field 65,535"""
    import torch
    n_streams, per_stream = 3, 21848
    total = n_streams * per_stream
    assert total >= 65535 + 8
    es_total = sum(len(batch.ts(s)) for s in range(n_streams))
    ctx = presenting_context(n_streams, 1, [batch.fc0(s) for s in range(n_streams)], max_pictures=PICTURES, es_capacity=es_total + 4096)
    ctx.submit_ts(*ctx.pack([batch.ts(s) for s in range(n_streams)]))
    ctx.index()
    r = _Paced(ctx, 1, batch, frames, oracle, n_streams)
    for p in range(PICTURES):
        r.picture(p, "split")
    w, nl = ctx.geometry()
    need = total * w * nl * 2
    free, _ = torch.cuda.mem_get_info()
    if free < need + (2 << 30):
        ctx.close()
        pytest.skip("the field buffer of %d fields needs %.1f GB of device memory and %.1f GB are free" % (total, need / 2**30, free / 2**30))
    want = [r.disp[d].idle(per_stream) for d in range(n_streams)]
    info0 = ctx.present_idle(per_stream)
    assert int(info0["n_fields"].sum()) == total
    out = torch.empty(total * w * nl, dtype=torch.uint16, device="cuda")
    try:
        n0 = ctx.launch_count()
        info = ctx.present_idle(per_stream, out)
        k2 = ctx.launch_count() - n0 - 2                           # schedule + descriptors, then the paced K2 launches
        assert k2 == -(-total // 65535) == 2
        assert (info == info0).all()
        first = [int(x) for x in info["first"]]
        assert first == [per_stream * s for s in range(n_streams)]
        F = out.view(torch.int16).view(-1, w * nl)

        def check_slot(g):
            s, j = g // per_stream, g % per_stream
            got = F[g].cpu().numpy().view(np.uint16)
            wf = r.rend[s].field(want[s][j])
            diff = np.nonzero(got != wf)[0]
            assert diff.size == 0, "slot %d (%s, field %d %s): %d samples differ, first %d" % (g, _where(s), j, want[s][j], diff.size, diff[0])
        for g in range(65528, 65544):                              # across the launch boundary
            check_slot(g)
        for s in range(n_streams):
            # the restatement's fields settle once a poster scroll has run out: from `settled` on, every field equals the
            # field two earlier (same picture, same hscroll, same frame-counter parity). The fields before it are rendered.
            settled = 1 + max([j for j in range(2, per_stream) if want[s][j][1:] != want[s][j - 2][1:]], default=1)
            assert settled < 64, s
            for j in range(settled):
                check_slot(first[s] + j)
            for j0 in range(settled, per_stream, 2048):
                j1 = min(j0 + 2048, per_stream)
                a, b = F[first[s] + j0:first[s] + j1], F[first[s] + j0 - 2:first[s] + j1 - 2]
                bad = (a != b).any(dim=1)
                if bool(bad.any()):
                    j = j0 + int(torch.nonzero(bad)[0, 0])
                    pytest.fail("slot %d (%s, field %d) differs from the field two earlier" % (first[s] + j, _where(s), j))
        del F
    finally:
        del out
        torch.cuda.empty_cache()
        ctx.close()


# ---- the fields context: decode and composite ---------------------------------------------------------------------------
# These tests come last: the module keeps their context until it ends, and the paced tests' field buffers need the room.
@pytest.fixture(scope="module")
def dctx(packed):
    """a fields context over the whole batch"""
    ctx = _context(True, int(packed[1][-1]) + 4096)
    yield ctx
    ctx.close()


@pytest.mark.gpu
def test_ts_submits_decode_every_stream(dctx, batch, frames, packed):
    """the batch as TS from host memory, from a CUDA tensor, and in two submits (the second queued before the first is
    decoded); then the same ES as one ES submit"""
    import torch
    ctx = dctx
    es_total = sum(len(batch.es[s % D]) for s in range(N))
    blob, off = packed
    full, zero = [PICTURES] * N, [0] * N
    # host memory
    ctx.reset()
    ctx.submit_ts(blob, off)
    ctx.index()
    _check_counts(ctx, batch, full, zero, es_total, "TS host")
    ctx.decode_all(PICTURES)
    _check_last_two(ctx, frames, "TS host")
    _check_async_window(ctx, frames, "TS host")
    # device memory: both the bytes and the offsets on the device
    ctx.reset()
    dblob = torch.from_numpy(blob).cuda()
    doff = torch.from_numpy(off.view(np.int64)).cuda()
    torch.cuda.synchronize()
    ctx.submit_ts(dblob.data_ptr(), doff.data_ptr(), device=True)
    ctx.index()
    _check_counts(ctx, batch, full, zero, es_total, "TS device")
    del dblob, doff
    torch.cuda.empty_cache()
    ctx.decode_all(PICTURES)
    _check_last_two(ctx, frames, "TS device")
    _check_async_window(ctx, frames, "TS device")
    # two submits cut at picture-boundary packets; the second is queued while the first one's decode still runs
    ctx.reset()
    parts, n0 = _split(batch)
    n1 = [PICTURES - n for n in n0]
    p0, p1 = ctx.pack(parts[0]), ctx.pack(parts[1])
    ctx.submit_ts(*p0)
    ctx.index()
    _check_counts(ctx, batch, n0, zero, tag="TS cut, part 0")
    ctx.decode_all(max(n0))
    ctx.submit_ts(*p1)
    _check_latest(ctx, frames, [n - 1 for n in n0], "TS cut, part 0")   # frame store (n0 + 1) & 1: differs from stream to stream
    ctx.index()
    _check_counts(ctx, batch, n1, n0, tag="TS cut, part 1")
    ctx.decode_all(max(n1))
    _check_last_two(ctx, frames, "TS cut")
    _check_async_window(ctx, frames, "TS cut")
    # the same ES as one ES submit
    ctx.reset()
    ctx.submit_es(*ctx.pack([batch.es[s % D] for s in range(N)]))
    ctx.index()
    _check_counts(ctx, batch, full, zero, es_total, "ES")
    ctx.decode_all(PICTURES)
    _check_last_two(ctx, frames, "ES")


@pytest.mark.gpu
def test_composite_fields_of_every_stream(dctx, batch, frames, packed, oracle):
    """ef_composite_field over the decoded batch, then a short ES submit of 0, 1 or 2 pictures per stream so that the
    latest frame store differs from stream to stream: every stream's field against the C restatement"""
    ctx = dctx
    ctx.reset()
    ctx.submit_ts(*packed)
    ctx.index()
    ctx.decode_all(PICTURES)
    extra = []
    for s in range(N):
        e = scale_cases.extra_pictures(s % D)
        extra.append(batch.es[s % D][:batch.codes[s % D][e] - 3] if e else b"")
    ctx.submit_es(*ctx.pack(extra))
    ctx.index()
    ctx.decode_all(ctx.index_info()["max_pictures"])
    # (latest, other) picture of every distinct stream: picture k of the run lives in store (k + 1) & 1
    stores = []
    for d in range(D):
        e, f = scale_cases.extra_pictures(d), frames[d]
        stores.append({0: (f[11], f[10]), 1: (f[0], f[11]), 2: (f[1], f[0])}[e])
    assert len({(12 + scale_cases.extra_pictures(s % D)) & 1 for s in range(N)}) == 2
    rng = np.random.default_rng(67)
    bm = rng.integers(0, 256, 1280, dtype=np.uint8)
    configs = [(1, -1, 0, None), (1, -1, 1, None), (0, -1, 1, None), (1, -2, 1, None), (1, -1, 1, (-24, bm, 5, 200))]
    for ntsc, fb, fc, fx in configs:
        tag = "ntsc %d fb %d fc %d%s" % (ntsc, fb, fc, " scroll+overlay" if fx else "")
        ctx.video_init(ntsc)
        if fx:
            ctx.set_scroll(fx[0])
            ctx.set_overlay(fx[1], fx[2], fx[3])
        ctx.composite_field(fb, fc)
        orig = []
        for d in range(D):
            a, b = stores[d]
            w = oracle.field_ex(a, b, ntsc, fc, *(fx if fx else ()))
            if fb == -2:
                w = pc.blank_field(oracle.field_ex(a, b, ntsc, 0), ntsc)
            orig.append(w)
        for s in range(N):
            got = ctx.read_field(s)
            d = np.nonzero(got != orig[s % D])[0]
            assert d.size == 0, "%s: %s: %d samples differ, first %d" % (tag, _where(s), d.size, d[0])
        if fx:
            ctx.set_scroll(0)
            ctx.set_overlay(None, 0, 0)
