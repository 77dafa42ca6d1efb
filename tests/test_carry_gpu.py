"""TS submits cut at any packet boundary (ef_carry_enable / ef_end_streams / ef_carry_info) on the GPU: decoded pictures, pts,
per-submit picture counts and held bytes, against the reference's pins, the whole-program decode of a non-carrying context and
the restatement in tests/carry_cases.py."""
import json
import os

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import carry_cases, present_cases as pc, pts_cases, restart_cases
from tests.harness import Paced, presenting_context, sha, submits

pytestmark = pytest.mark.gpu
G = pts_cases.GOLDEN
MAX_CARRY = 65536


class Run:
    """per stream: sha256 of every decoded picture, its pts, the picture count and held bytes of every submit"""

    def __init__(self, n):
        self.frames = [[] for _ in range(n)]
        self.pts = [[] for _ in range(n)]
        self.counts = [[] for _ in range(n)]
        self.held = [[] for _ in range(n)]


def _index_and_read(ctx, run, n, decode=True, check_info=True):
    ctx.index()
    if check_info:
        ctx.index_info()
    counts = [ctx.stream_info(s)[0] for s in range(n)]
    if decode:
        for p in range(max(counts) if counts else 0):
            ctx.decode_picture(p)
            for s in range(n):
                if p < counts[s]:
                    run.frames[s].append(sha(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1)))
    pic, _ = ctx.picture_pts()
    held, _ = ctx.carry_info()
    for s in range(n):
        run.pts[s] += [int(v) for v in pic[s, :counts[s]]]
        run.counts[s].append(counts[s])
        run.held[s].append(int(held[s]))


def _drive(ctx, per_stream, end_at=None, decode=True, run=None):
    """per_stream[s]: TS chunks of stream s, one per submit (padded with empty submits); stream s ends with submit end_at[s]
    (default: its last chunk)"""
    n = len(per_stream)
    if end_at is None:
        end_at = [len(c) - 1 for c in per_stream]
    run = run or Run(n)
    for k, chunk in enumerate(submits(per_stream)):
        ctx.submit_ts(*ctx.pack(chunk))
        ends = np.array([1 if end_at[s] == k else 0 for s in range(n)], dtype=np.uint8)
        if ends.any():
            ctx.end_streams(ends)
        _index_and_read(ctx, run, n, decode)
    return run


def _carrying(n, max_pictures=100, max_carry=MAX_CARRY, es_capacity=1 << 22):
    ctx = espflix_b200.Context(n_streams=n, max_pictures=max_pictures, max_slices_per_picture=12, es_capacity=es_capacity, fields=False)
    ctx.enable_pts()
    ctx.enable_carry(max_carry)
    return ctx


def _restated(chunks):
    st = carry_cases.Stream()
    for k, c in enumerate(chunks):
        st.feed(c, end=k == len(chunks) - 1)
    return st


def _whole(programs, max_pictures=100):
    """the whole programs on a non-carrying context -> Run"""
    ctx = espflix_b200.Context(n_streams=len(programs), max_pictures=max_pictures, max_slices_per_picture=12, es_capacity=1 << 23, fields=False)
    ctx.enable_pts()
    run = Run(len(programs))
    ctx.submit_ts(*ctx.pack(programs))
    ctx.index()
    ctx.index_info()
    counts = [ctx.stream_info(s)[0] for s in range(len(programs))]
    for p in range(max(counts)):
        ctx.decode_picture(p)
        for s in range(len(programs)):
            if p < counts[s]:
                run.frames[s].append(sha(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1)))
    pic, _ = ctx.picture_pts()
    for s in range(len(programs)):
        run.pts[s] = [int(v) for v in pic[s, :counts[s]]]
    ctx.close()
    return run


@pytest.fixture(scope="module")
def fixtures():
    return [open(os.path.join(G, n + ".ts"), "rb").read() for n in pts_cases.FIXTURES]


@pytest.fixture(scope="module")
def pins():
    return json.load(open(os.path.join(G, "decode_pins.json"))), json.load(open(os.path.join(G, "pts_pins.json")))["programs"]


@pytest.mark.parametrize("every_packet", [False, True])
def test_fixtures_against_pins(fixtures, pins, every_packet):
    """splash.ts and vmedia.ts share one carrying context, cut at seeded packets into submits of 0 to 40 packets (or before
    every packet): every picture and pts as pinned, per-submit counts and held bytes as restated"""
    dpins, ppins = pins
    per_stream = []
    for i, ts in enumerate(fixtures):
        cuts = list(range(1, len(ts) // 188)) if every_packet else carry_cases.seeded_cuts(ts, 77 + i)
        per_stream.append(carry_cases.cut(ts, cuts))
    ctx = _carrying(2)
    run = _drive(ctx, per_stream, decode=not every_packet)
    ctx.close()
    for s, name in enumerate(pts_cases.FIXTURES):
        want = _restated(per_stream[s])
        K = len(per_stream[s])
        assert run.counts[s][:K] == want.counts, name
        assert run.held[s][:K] == want.held_sizes, name
        assert run.pts[s] == ppins[name]["pts"], name
        if not every_packet:
            assert run.frames[s] == dpins[name]["frame_sha256"], name


def test_cases_batch_cut_anywhere():
    """every program of pts_cases.cases(), custom matrices and a headers-only tail in one batch, each cut at its own seeded
    packets: pictures equal the whole-program decode, pts the whole-program pts"""
    progs = [ts for (name, ts) in carry_cases.programs() if name not in pts_cases.FIXTURES]
    whole = _whole(progs)
    per_stream = [carry_cases.cut(ts, carry_cases.seeded_cuts(ts, 300 + i, 12)) for i, ts in enumerate(progs)]
    ctx = _carrying(len(progs))
    run = _drive(ctx, per_stream)
    ctx.close()
    for s, ts in enumerate(progs):
        assert run.frames[s] == whole.frames[s], s
        assert run.pts[s] == whole.pts[s] == pts_cases.picture_pts(ts), s
        want = _restated(per_stream[s])
        assert run.counts[s][:len(want.counts)] == want.counts, s


def test_audio_beside_carry():
    """audio enabled, video and audio cut at the same seeded packets: PCM / PDM equal the whole-stream decode, video the
    whole-program decode"""
    progs = [restart_cases.program(401 + i, 7, 90000 * (i + 1), audio=dict(seed=31 + i, frames=40)) for i in range(3)]
    whole = _whole(progs)
    want_audio = capi.audio_decode(capi.audio_demux_ts(progs))
    per_stream = [carry_cases.cut(ts, carry_cases.seeded_cuts(ts, 500 + i, 9)) for i, ts in enumerate(progs)]
    ctx = _carrying(3)
    ctx.enable_audio()
    run = Run(3)
    pcm, pdm = [[] for _ in progs], [[] for _ in progs]
    for k, chunk in enumerate(submits(per_stream)):
        ctx.submit_ts(*ctx.pack(chunk))
        last = [k == len(per_stream[s]) - 1 for s in range(3)]
        if any(last):
            ctx.end_streams(np.array(last, dtype=np.uint8))
        _index_and_read(ctx, run, 3)
        out = ctx.decode_audio(end=np.array(last, dtype=np.uint8))
        for s in range(3):
            pcm[s].append(out[s]["pcm"])
            pdm[s].append(out[s]["pdm"])
    ctx.close()
    for s in range(3):
        assert run.frames[s] == whole.frames[s]
        assert run.pts[s] == whole.pts[s]
        assert np.array_equal(np.concatenate(pcm[s]), want_audio[s]["pcm"])
        assert np.array_equal(np.concatenate(pdm[s]), want_audio[s]["pdm"])


def _held_cut(ts, least=200, start=None):
    """a packet to cut a program before (from `start`, default half way) so that the first part ends holding more than `least`
    bytes of a picture"""
    pk = len(ts) // 188
    for c in range(pk // 2 if start is None else start, pk):
        st = carry_cases.Stream()
        st.feed(carry_cases.cut(ts, [c])[0])
        if st.held_sizes[-1] > least:
            return c
    raise AssertionError("no cut holds a picture")


@pytest.mark.parametrize("queued", [False, True])
def test_restart_drops_held_bytes(queued):
    """op 1 with a held tail (the next submit already queued, or not) then a new program from its sequence header: that
    program decodes as on a fresh non-carrying context; a neighbour with op 0 keeps its tail"""
    a = restart_cases.program(411, 9, 90000)
    b = restart_cases.program(412, 6, 900000)
    keep = restart_cases.program(413, 8, 45000)
    whole = _whole([b, keep])
    ca, ck = _held_cut(a), _held_cut(keep)
    a1 = carry_cases.cut(a, [ca])[0]
    k1, k2 = carry_cases.cut(keep, [ck])
    ctx = _carrying(2)
    run = Run(2)
    ctx.submit_ts(*ctx.pack([a1, k1]))
    _index_and_read(ctx, run, 2)
    assert run.held[0][-1] > 0 and run.held[1][-1] > 0
    b_parts = carry_cases.cut(b, carry_cases.seeded_cuts(b, 9, 10))
    if queued:
        ctx.submit_ts(*ctx.pack([b_parts[0], k2]))
        ctx.restart_streams([1, 0])
    else:
        ctx.restart_streams([1, 0])
        ctx.submit_ts(*ctx.pack([b_parts[0], k2]))
    assert ctx.carry_info()[0][0] == 0
    n0 = len(run.frames[0])
    ctx.end_streams(np.array([1 if len(b_parts) == 1 else 0, 1], dtype=np.uint8))
    _index_and_read(ctx, run, 2)
    if len(b_parts) > 1:
        _drive(ctx, [b_parts[1:], [b""] * (len(b_parts) - 1)], end_at=[len(b_parts) - 2, -1], run=run)
    ctx.close()
    assert run.frames[0][n0:] == whole.frames[0]
    assert run.pts[0][n0:] == whole.pts[0]
    full_keep = _whole([keep])
    assert run.frames[1] == full_keep.frames[0] and run.pts[1] == full_keep.pts[0]


def test_restart_with_a_whole_program_queued():
    """op 1 drops a held tail longer than the gap between two pictures of the program queued behind it (one PES per picture):
    the queued program's PES starts stay behind the dropped bytes, so its pictures and pts are those of the program decoded
    on its own"""
    a = restart_cases.program(411, 9, 90000)
    b = restart_cases.program(412, 6, 900000)
    es_b, _ = pts_cases.demux(b)
    codes = pts_cases.picture_codes(es_b)
    gap = min(y - x for x, y in zip(codes, codes[1:]))
    a1 = carry_cases.cut(a, [_held_cut(a, least=gap + 188, start=1)])[0]
    whole = _whole([b])
    ctx = _carrying(1)
    run = Run(1)
    ctx.submit_ts(*ctx.pack([a1]))
    _index_and_read(ctx, run, 1)
    assert run.held[0][-1] > gap
    n0 = len(run.frames[0])
    ctx.submit_ts(*ctx.pack([b]))                                  # queued before the restart
    ctx.restart_streams([1])
    ctx.end_streams(np.ones(1, np.uint8))
    _index_and_read(ctx, run, 1)
    ctx.close()
    assert run.frames[0][n0:] == whole.frames[0]
    assert run.pts[0][n0:] == whole.pts[0] == pts_cases.picture_pts(b)


def test_pause_keeps_and_reset_drops():
    """op 2 between submits keeps the held bytes (the program decodes as uncut); ef_reset drops every stream's"""
    a = restart_cases.program(421, 9, 90000)
    whole = _whole([a])
    parts = carry_cases.cut(a, [_held_cut(a)])
    ctx = _carrying(1)
    run = Run(1)
    ctx.submit_ts(*ctx.pack([parts[0]]))
    _index_and_read(ctx, run, 1)
    assert run.held[0][-1] > 0
    ctx.restart_streams([2])
    ctx.submit_ts(*ctx.pack([parts[1]]))
    ctx.end_streams(np.ones(1, np.uint8))
    _index_and_read(ctx, run, 1)
    assert run.frames[0] == whole.frames[0] and run.pts[0] == whole.pts[0]

    ctx.submit_ts(*ctx.pack([parts[0]]))
    _index_and_read(ctx, run, 1)
    assert ctx.carry_info()[0][0] > 0
    ctx.reset()
    assert ctx.carry_info()[0][0] == 0
    b = restart_cases.program(422, 5, 700000)
    run = _drive(ctx, [carry_cases.cut(b, carry_cases.seeded_cuts(b, 5, 15))])
    ctx.close()
    wb = _whole([b])
    assert run.frames[0] == wb.frames[0] and run.pts[0] == wb.pts[0]


def test_streams_end_at_different_submits_then_new_programs():
    progs = [restart_cases.program(431 + i, 5 + i, 30000 * (i + 1)) for i in range(3)]
    nxt = [restart_cases.program(441 + i, 4, 5000000 + i) for i in range(3)]
    parts = [carry_cases.cut(ts, carry_cases.seeded_cuts(ts, 60 + i, 7 + 5 * i)) for i, ts in enumerate(progs)]
    parts2 = [carry_cases.cut(ts, carry_cases.seeded_cuts(ts, 70 + i, 11)) for i, ts in enumerate(nxt)]
    per = [p + q for p, q in zip(parts, parts2)]
    ends = [[len(p) - 1, len(p) + len(q) - 1] for p, q in zip(parts, parts2)]
    ctx = _carrying(3)
    run = Run(3)
    for k, chunk in enumerate(submits(per)):
        ctx.submit_ts(*ctx.pack(chunk))
        e = np.array([1 if k in ends[s] else 0 for s in range(3)], dtype=np.uint8)
        if e.any():
            ctx.end_streams(e)
        _index_and_read(ctx, run, 3)
        for s in range(3):
            if k in ends[s]:
                assert run.held[s][-1] == 0
    ctx.close()
    for s in range(3):
        w1, w2 = _whole([progs[s]]), _whole([nxt[s]])
        assert run.frames[s] == w1.frames[0] + w2.frames[0]
        assert run.pts[s] == w1.pts[0] + w2.pts[0]


def test_capacity_flag_and_neighbours():
    """a stream whose held bytes exceed max_carry gets its flag and EF_ENOMEM; its neighbour stays exact; after op 1 it
    decodes a new program cleanly"""
    big, small = open(os.path.join(G, "vmedia.ts"), "rb").read(), restart_cases.program(451, 8, 90000)
    big_parts = carry_cases.cut(big, list(range(40, len(big) // 188, 40)))
    small_parts = carry_cases.cut(small, list(range(2, len(small) // 188, 2)))
    fresh = restart_cases.program(452, 5, 123000)
    fresh_parts = carry_cases.cut(fresh, carry_cases.seeded_cuts(fresh, 3, 20))
    max_carry = max(_restated(small_parts).held_sizes + _restated(fresh_parts).held_sizes)
    assert max(_restated(big_parts).held_sizes) > max_carry
    ctx = _carrying(2, max_carry=max_carry)
    run = Run(2)
    flagged = False
    for k, chunk in enumerate(submits([big_parts, small_parts])):
        ctx.submit_ts(*ctx.pack(chunk))
        if k == len(small_parts) - 1:
            ctx.end_streams(np.array([0, 1], dtype=np.uint8))
        try:
            _index_and_read(ctx, run, 2)
        except capi.EspflixError as e:
            assert e.code == capi.EF_ENOMEM
            flagged = True
            _index_and_read_after_error(ctx, run)
    assert flagged
    assert ctx.carry_info()[1][0] & 1 and not ctx.carry_info()[1][1] & 1
    ws = _whole([small])
    assert run.frames[1] == ws.frames[0] and run.pts[1] == ws.pts[0]
    ctx.restart_streams([1, 0])
    assert ctx.carry_info()[1][0] == 0
    r2 = _drive(ctx, [fresh_parts, []], end_at=[len(fresh_parts) - 1, -1])
    ctx.close()
    wf = _whole([fresh])
    assert r2.frames[0] == wf.frames[0] and r2.pts[0] == wf.pts[0]


def _index_and_read_after_error(ctx, run):
    """the rest of _index_and_read once ef_index_info has reported the flag (ef_index has run)"""
    counts = [ctx.stream_info(s)[0] for s in range(2)]
    for p in range(max(counts)):
        ctx.decode_picture(p)
        for s in range(2):
            if p < counts[s]:
                run.frames[s].append(sha(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1)))
    pic, _ = ctx.picture_pts()
    held, _ = ctx.carry_info()
    for s in range(2):
        run.pts[s] += [int(v) for v in pic[s, :counts[s]]]
        run.counts[s].append(counts[s])
        run.held[s].append(int(held[s]))


def test_errors_and_launch_counts():
    ts = restart_cases.program(461, 4, 90000)
    plain = espflix_b200.Context(n_streams=2, max_pictures=8, es_capacity=1 << 20, fields=False)
    blob, off = plain.pack([ts, ts])
    n0 = plain.launch_count()
    plain.submit_ts(blob, off)
    plain.index()
    assert plain.launch_count() - n0 == 4 + 3                   # TS compaction, then scan / prefix / fill, as before carry
    with pytest.raises(capi.EspflixError) as e:
        plain.end_streams(np.ones(2, np.uint8))
    assert e.value.code == capi.EF_ESTATE
    with pytest.raises(capi.EspflixError) as e:
        plain.carry_info()
    assert e.value.code == capi.EF_ESTATE
    plain.close()

    ctx = espflix_b200.Context(n_streams=2, max_pictures=8, es_capacity=1 << 20, fields=False)
    ctx.submit_ts(blob, off)
    with pytest.raises(capi.EspflixError) as e:
        ctx.enable_carry(MAX_CARRY)                             # a submit is pending
    assert e.value.code == capi.EF_ESTATE
    ctx.index()
    ctx.enable_carry(MAX_CARRY)
    for call, code in ((lambda: ctx.enable_carry(MAX_CARRY), capi.EF_ESTATE),
                       (lambda: ctx.submit_es(*ctx.pack([b"\x00\x00\x01\xb3", b""])), capi.EF_ESTATE),
                       (lambda: ctx.end_streams(np.ones(2, np.uint8)), capi.EF_ESTATE),
                       (lambda: ctx.carry_info(first=1, count=2), capi.EF_EINVAL)):
        with pytest.raises(capi.EspflixError) as e:
            call()
        assert e.value.code == code
    ctx.submit_ts(blob, off)
    with pytest.raises(capi.EspflixError) as e:
        ctx.end_streams(np.ones(3, np.uint8))
    assert e.value.code == capi.EF_EINVAL
    n0 = ctx.launch_count()
    ctx.index()
    assert ctx.launch_count() - n0 == 3
    with pytest.raises(capi.EspflixError) as e:
        ctx.index()                                             # re-indexing the same input
    assert e.value.code == capi.EF_ESTATE
    ctx.close()


# -- paced presentation of carried submits -------------------------------------------------------------------------------------
def _paced(progs, ntsc, cut_seed=None, use_async=False):
    """progs: [(ts, fc0, modes, tail fields)]; whole on a non-carrying context, or every program cut at its own seeded packets
    on a carrying one and ended with its last submit"""
    from tests.oracle_lib import Oracle
    o = Oracle()
    fc0 = [p[1] for p in progs]
    ctx = presenting_context(len(progs), ntsc, fc0, carry=None if cut_seed is None else MAX_CARRY)
    r = Paced(ctx, [pc.Display(ntsc, f) for f in fc0], [pc.Renderer(o, ntsc) for _ in progs], [o.decode_ts(p[0]) for p in progs])
    mode_of = lambda s, g: progs[s][2][g]                                        # noqa: E731
    if cut_seed is None:
        r.submit([p[0] for p in progs], mode_of, None, use_async)
    else:
        per = [carry_cases.cut(p[0], carry_cases.seeded_cuts(p[0], cut_seed + s, 25)) for s, p in enumerate(progs)]
        last = [len(c) - 1 for c in per]
        for k, chunk in enumerate(submits(per)):
            r.submit(chunk, mode_of, [k == last[s] for s in range(len(progs))], use_async)
    r.idle([p[3] + 1 for p in progs])
    ctx.close()
    return r


@pytest.mark.parametrize("ntsc", [1, 0])
def test_paced_presentation_of_carried_submits(ntsc):
    """the irregular schedules of tests/test_present_gpu.py (modes 1 to 3 included) cut anywhere, through the synchronous and
    the asynchronous present calls: fields, flips and pts equal the run on whole programs, and the restatement"""
    progs = [(ts, fc0, modes, tail) for _, ts, _, n, fc0, modes, tail in pc.irregular_programs() if n == ntsc]
    whole = _paced(progs, ntsc)
    for seed, use_async in ((20 + ntsc, False), (40 + ntsc, True)):
        r = _paced(progs, ntsc, cut_seed=seed, use_async=use_async)
        assert r.pts == whole.pts
        assert r.flips == whole.flips
        assert r.dev == whole.dev
        assert r.fc == whole.fc
        r.check()


# -- the benchmark's batch size --------------------------------------------------------------------------------------------------
def test_scale_batch_cut_anywhere():
    """the 4,096 streams of tests/scale_cases.py, each cut at its own seeded packets into submits of 0 to 40 packets: per-submit
    picture totals as restated, the pts of every picture of every stream, every stream's latest picture half way and its last
    two pictures at the end as decoded from the whole program"""
    from tests import scale_cases
    from tests.oracle_lib import Oracle
    b = scale_cases.batch()
    N, D, P = scale_cases.N, scale_cases.D, scale_cases.PICTURES
    o = Oracle()
    frames = [o.decode_es(b.es[d]) for d in range(D)]
    per = [carry_cases.cut(b.ts(k), carry_cases.seeded_cuts(b.ts(k), 7000 + k)) for k in range(N)]
    want = [_restated(c) for c in per]
    last = [len(c) - 1 for c in per]
    chunks = submits(per)
    K = len(chunks)
    cap = max(sum(len(c) for c in chunk) for chunk in chunks) + 4096
    ctx = espflix_b200.Context(n_streams=N, max_pictures=P, max_slices_per_picture=12, es_capacity=cap, fields=False)
    ctx.enable_pts()
    ctx.enable_carry(MAX_CARRY)
    seen = np.zeros(N, dtype=np.int64)
    pts = [[] for _ in range(N)]
    for k in range(K):
        ctx.submit_ts(*ctx.pack(chunks[k]))
        ends = np.array([1 if last[s] == k else 0 for s in range(N)], dtype=np.uint8)
        if ends.any():
            ctx.end_streams(ends)
        ctx.index()
        info = ctx.index_info()
        counts = np.array([want[s].counts[k] if k < len(want[s].counts) else 0 for s in range(N)])
        assert info["total_pictures"] == int(counts.sum()) and info["max_pictures"] == int(counts.max()), k
        ctx.decode_all(int(counts.max()))
        pic, _ = ctx.picture_pts()
        for s in range(N):
            pts[s] += [int(v) for v in pic[s, :counts[s]]]
        held, flags = ctx.carry_info()
        assert not flags.any()
        assert [int(h) for h in held] == [want[s].held_sizes[k] if k < len(want[s].held_sizes) else 0 for s in range(N)], k
        seen += counts
        if k == K // 2:
            got = ctx.read_latest_i420(0, N)
            for s in range(N):
                if seen[s]:
                    assert np.array_equal(got[s], frames[s % D][seen[s] - 1]), "stream %d after submit %d" % (s, k)
    for s in range(N):
        assert pts[s] == b.pts[s % D], s
        assert ctx.stream_info(s) == (int(counts[s]), P - int(counts[s])), s
    got = ctx.read_latest_i420(0, N)
    for s in range(N):
        assert np.array_equal(got[s], frames[s % D][P - 1]), s
        assert np.array_equal(ctx.read_frame_i420(s, 1), frames[s % D][P - 2]), s          # picture g went to store (g + 1) & 1
    ctx.close()
