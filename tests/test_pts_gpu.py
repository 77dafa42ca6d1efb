"""Presentation timestamps through the decoder context (ef_pts_enable / ef_picture_pts): the pts of every picture of every
TS submit, concatenated over the submits, must equal the pts the unmodified reference pushes with it (tests/golden/
pts_pins.json) and, outside the reference's domain, the restatement in tests/pts_cases.py."""
import json
import os

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import audio_cases, pts_cases
from tests.carry_cases import cut, packets
from tests.harness import sha, submits

pytestmark = pytest.mark.gpu
G = pts_cases.GOLDEN


@pytest.fixture(scope="module")
def pins():
    return json.load(open(os.path.join(G, "pts_pins.json")))["programs"]


@pytest.fixture(scope="module")
def cases():
    return pts_cases.cases()


def _expected(ts, name, pins):
    return pins[name]["pts"] if name in pins else pts_cases.picture_pts(ts)


def _run(ctx, chunks, queue_ahead=False, decode=None):
    """chunks[k][s]: TS bytes of stream s in submit k -> per stream: pts of every picture over all submits, and last_pts
    after every submit. queue_ahead: submit k + 1 is queued before ef_picture_pts of submit k. decode(ctx, counts): called
    after every ef_index."""
    n, K = len(chunks[0]), len(chunks)
    pts, last = [[] for _ in range(n)], [[] for _ in range(n)]
    packed = [ctx.pack(c) for c in chunks]
    ctx.submit_ts(*packed[0])
    for k in range(K):
        ctx.index()
        ctx.index_info()                                # raises on an index overflow
        counts = [ctx.stream_info(s)[0] for s in range(n)]
        if decode:
            decode(ctx, counts)
        if queue_ahead and k + 1 < K:
            ctx.submit_ts(*packed[k + 1])
        pic, lp = ctx.picture_pts()
        for s in range(n):
            assert (pic[s, counts[s]:] == -1).all()
            pts[s] += [int(v) for v in pic[s, :counts[s]]]
            last[s].append(int(lp[s]))
            assert last[s][-1] == (pts[s][-1] if pts[s] else -1)     # get_pts(): the most recent picture over all submits
        if not queue_ahead and k + 1 < K:
            ctx.submit_ts(*packed[k + 1])
    return pts, last


def test_fixtures_whole_and_cut_at_pes_starts(pins):
    """splash.ts and vmedia.ts in one context, whole and cut at video PES starts into uneven submits: pts as pinned, and
    the pictures still as decode_pins.json"""
    names = list(pts_cases.FIXTURES)
    ts = [open(os.path.join(G, n + ".ts"), "rb").read() for n in names]
    dpins = json.load(open(os.path.join(G, "decode_pins.json")))
    ctx = espflix_b200.Context(n_streams=2, max_pictures=100, max_slices_per_picture=12, es_capacity=1 << 21)
    ctx.enable_pts()
    pts, last = _run(ctx, [[np.frombuffer(t, dtype=np.uint8) for t in ts]])
    for s, n in enumerate(names):
        assert pts[s] == pins[n]["pts"], n
        assert last[s] == [pins[n]["pts"][-1]]
    ctx.close()

    sizes = [[5, 12, 1, 9, 7, 12, 3], [11, 2, 12, 8, 6, 4, 10]]
    per_stream = []
    for i, t in enumerate(ts):
        pk = packets(t)
        starts = [k for k, q in enumerate(pk) if ((int(q[1]) << 8 | int(q[2])) & 0x1FFF) == 0x100 and q[1] & 0x40]
        cuts, p, j = [], 0, 0
        while True:
            p += sizes[i][j % len(sizes[i])]
            j += 1
            if p >= len(starts):
                break
            cuts.append(starts[p])
        per_stream.append(cut(t, cuts))
    frames = [[], []]

    def decode(ctx, counts):
        for p in range(max(counts)):
            ctx.decode_picture(p)
            for s in range(2):
                if p < counts[s]:
                    frames[s].append(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1))

    ctx = espflix_b200.Context(n_streams=2, max_pictures=13, max_slices_per_picture=12, es_capacity=1 << 21)
    ctx.enable_pts()
    pts, last = _run(ctx, submits(per_stream), decode=decode)
    for s, n in enumerate(names):
        assert pts[s] == pins[n]["pts"], n
        assert last[s][-1] == pins[n]["pts"][-1]
        assert len(frames[s]) == dpins[n]["frames"]
        for k, f in enumerate(frames[s]):
            assert sha(f) == dpins[n]["frame_sha256"][k], "%s picture %d" % (n, k)
    ctx.close()


def _cut_cases(cases, K, seed):
    """every case cut at seeded picture-boundary packets into K submits (empty submits included)"""
    chunks = []
    for i, (name, ts) in enumerate(cases):
        cand = pts_cases.cut_points(ts)
        r = np.random.RandomState(seed + i)
        cuts = sorted(r.choice(cand, size=K - 1, replace=True).tolist()) if cand else [len(ts) // 188] * (K - 1)
        chunks.append(cut(ts, cuts))
    return submits(chunks)


@pytest.mark.parametrize("queue_ahead", [False, True])
def test_batch_of_cases_whole_and_cut(pins, cases, queue_ahead):
    """every synthetic and re-wrapped program in one batch, whole and cut at seeded picture-boundary packets; with
    queue_ahead the next submit is already queued (its PES list in the other ES buffer) when the pts are read"""
    n = len(cases)
    want = [_expected(ts, name, pins) for name, ts in cases]
    assert len({len(w) for w in want}) >= 6                       # different picture counts in one batch
    ctx = espflix_b200.Context(n_streams=n, max_pictures=100, max_slices_per_picture=12, es_capacity=1 << 23, fields=False)
    ctx.enable_pts()
    pts, last = _run(ctx, [[np.frombuffer(ts, dtype=np.uint8) for _, ts in cases]], queue_ahead=queue_ahead)
    for s, (name, _) in enumerate(cases):
        assert pts[s] == want[s], name
    ctx.reset()                                                    # every stream starts over
    K = 6
    chunks = _cut_cases(cases, K, 7000)
    pts, last = _run(ctx, chunks, queue_ahead=queue_ahead)
    for s, (name, _) in enumerate(cases):
        assert pts[s] == want[s], name
        assert last[s][-1] == want[s][-1], name
    ctx.close()


def _carry(ts, before):
    """the carried value after a TS chunk: its last valid PES PTS, else what came before"""
    v = [p for _, p in pts_cases.demux(ts)[1] if p >= 0]
    return v[-1] if v else before


def test_es_submits_reindex_reset_and_audio(pins, cases):
    byname = dict(cases)
    ts = byname["synth20_shift"]
    cuts = pts_cases.cut_points(ts)
    a, b, c = cut(ts, [cuts[len(cuts) // 3], cuts[2 * len(cuts) // 3]])
    want = pins["synth20_shift"]["pts"]
    ctx = espflix_b200.Context(n_streams=1, max_pictures=24, max_slices_per_picture=12, es_capacity=1 << 20, fields=False)
    ctx.enable_pts()
    # TS, then the middle part as an ES submit (no PES: the carried value), then TS again
    ctx.submit_ts(*ctx.pack([a]))
    ctx.index()
    na = ctx.stream_info(0)[0]
    pa, la = ctx.picture_pts()
    assert list(pa[0, :na]) == want[:na] and la[0] == want[na - 1]
    carried = _carry(a, -1)
    ctx.submit_es(*ctx.pack([pts_cases.demux(b)[0]]))
    ctx.index()
    nb = ctx.stream_info(0)[0]
    pb, lb = ctx.picture_pts()
    assert nb > 0 and list(pb[0, :nb]) == [carried] * nb and lb[0] == carried
    ctx.submit_ts(*ctx.pack([c]))
    ctx.index()
    nc = ctx.stream_info(0)[0]
    pc, lc = ctx.picture_pts()
    alone = pts_cases.picture_pts(c)
    assert list(pc[0, :nc]) == [carried if v < 0 else v for v in alone] and lc[0] == pc[0, nc - 1]
    # indexing the same submit again: as if the same input followed itself
    for rep in (2, 3):
        ctx.index()
        p, l_ = ctx.picture_pts()
        cc = np.concatenate([np.frombuffer(bytes(c), dtype=np.uint8)] * rep)
        w = pts_cases.picture_pts(cc)[-nc:]
        w = [_carry(c, carried) if v < 0 else v for v in w]
        assert list(p[0, :nc]) == w and l_[0] == w[-1]
    # ef_reset: -1 again, PTS stays enabled; a program whose first PES has no PTS reads -1 until its first PTS
    ctx.reset()
    with pytest.raises(espflix_b200.EspflixError) as e:
        ctx.picture_pts()
    assert e.value.code == capi.EF_ESTATE
    ood = byname["ood_first_without_pts"]
    ctx.submit_ts(*ctx.pack([np.frombuffer(ood, dtype=np.uint8)]))
    ctx.index()
    n = ctx.stream_info(0)[0]
    p, l_ = ctx.picture_pts()
    assert list(p[0, :n]) == pts_cases.picture_pts(ood) and p[0, 0] == -1 and l_[0] == p[0, n - 1]
    ctx.close()

    # audio and PTS together: both results as with either alone
    es = [audio_cases.sbc_stream(300 + i, 40, bitpool=28) for i in range(2)]
    progs = [byname["synth12_shift"], byname["synth9_shift"]]
    chunks = []
    for i in range(2):
        video = b"".join(q for q in packets(progs[i]) if ((int(q[1]) << 8 | int(q[2])) & 0x1FFF) == 0x100)   # without the filler audio PES
        vc = pts_cases.cut_points(video)
        v = [np.frombuffer(x, dtype=np.uint8) for x in cut(video, [vc[len(vc) // 2]])]
        au = audio_cases.mux_audio_ts(es[i], pid=0x102)
        h = au.size // 188 // 2
        chunks.append([np.concatenate([v[0], au[:h * 188]]), np.concatenate([v[1], au[h * 188:]])])
    results = {}
    for mode in ("audio", "pts", "both"):
        ctx = espflix_b200.Context(n_streams=2, max_pictures=24, max_slices_per_picture=12, es_capacity=1 << 21, fields=False)
        if mode != "pts":
            ctx.enable_audio()
        if mode != "audio":
            ctx.enable_pts()
        pts, aud = [[], []], [[], []]
        for k in range(2):
            ctx.submit_ts(*ctx.pack([chunks[0][k], chunks[1][k]]))
            ctx.index()
            counts = [ctx.stream_info(s)[0] for s in range(2)]
            if mode != "audio":
                p, _ = ctx.picture_pts()
                for s in range(2):
                    pts[s] += list(p[s, :counts[s]])
            if mode != "pts":
                r = ctx.decode_audio(end=[k == 1] * 2)
                for s in range(2):
                    aud[s].append(r[s]["pcm"])
        results[mode] = (pts, [np.concatenate(x) if x else None for x in aud])
        ctx.close()
    for s in range(2):
        assert results["both"][0][s] == results["pts"][0][s] == pins[["synth12_shift", "synth9_shift"][s]]["pts"]
        assert np.array_equal(results["both"][1][s], results["audio"][1][s])
        assert np.array_equal(results["both"][1][s], espflix_b200.audio_decode([es[s]], pdm=False)[0]["pcm"])


def test_errors_and_launch_counts(cases):
    ts = [np.frombuffer(t, dtype=np.uint8) for _, t in cases[4:7]]
    plain = espflix_b200.Context(n_streams=3, max_pictures=16, es_capacity=1 << 21, fields=False)
    ctx = espflix_b200.Context(n_streams=3, max_pictures=16, es_capacity=1 << 21, fields=False)
    with pytest.raises(espflix_b200.EspflixError) as e:
        ctx.picture_pts()
    assert e.value.code == capi.EF_ESTATE
    ctx.submit_ts(*ctx.pack(ts))
    ctx.index()
    ctx.enable_pts()
    ctx.enable_pts()                                             # idempotent
    with pytest.raises(espflix_b200.EspflixError) as e:           # no ef_index since enabling
        ctx.picture_pts()
    assert e.value.code == capi.EF_ESTATE
    ctx.index()                                                   # the submit made before enabling carries no PES
    p, l_ = ctx.picture_pts()
    assert (p == -1).all() and (l_ == -1).all()
    for first, count, n_pic in ((-1, 1, 4), (0, 0, 4), (2, 2, 4), (0, 4, 4), (0, 3, 17), (0, 3, -1)):
        assert ctx.lib.ef_picture_pts(ctx._h, first, count, n_pic, None, None) == capi.EF_EINVAL, (first, count, n_pic)
    assert ctx.lib.ef_picture_pts(ctx._h, 1, 2, 0, None, None) == capi.EF_OK
    assert ctx.lib.ef_picture_pts(None, 0, 1, 1, None, None) == capi.EF_EINVAL
    assert ctx.lib.ef_pts_enable(None) == capi.EF_EINVAL
    # one window of the result: streams [1, 3), the first 5 pictures
    ctx.submit_ts(*ctx.pack(ts))
    ctx.index()
    full, lfull = ctx.picture_pts()
    win, lwin = ctx.picture_pts(first=1, count=2, n_pictures=5)
    assert np.array_equal(win, full[1:3, :5]) and np.array_equal(lwin, lfull[1:3])

    def delta(c, submit):
        n0 = c.launch_count()
        submit(c)
        c.index()
        c.decode_all(c.index_info()["max_pictures"])
        c.sync()
        return c.launch_count() - n0

    def ts_submit(c):
        c.submit_ts(*c.pack(ts))

    def es_submit(c):
        c.submit_es(*c.pack([pts_cases.demux(t)[0] for t in ts]))

    plain.submit_ts(*plain.pack(ts))
    plain.index()
    mp = plain.index_info()["max_pictures"]
    d_plain = delta(plain, ts_submit)
    assert d_plain == 4 + 3 + 1 + mp                             # TS demux, K0, K1a, one K1b per picture index: as before
    assert delta(ctx, ts_submit) == d_plain + 2                  # + the packet pass + the resolve pass
    assert delta(ctx, es_submit) == delta(plain, es_submit) + 1  # ES submits: the resolve pass only
    plain.close()
    ctx.close()
