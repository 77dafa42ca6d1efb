"""Audio through the decoder context (ef_audio_enable / ef_decode_audio): every stream's TS cut into submits at packet
boundaries, the stream ended in its last submit. Concatenated over the calls, PCM and PDM must equal the whole-stream
call (ef_audio_decode on ef_audio_demux_ts), the restatement and the reference's pins, element for element."""
import hashlib
import json
import os

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi
from tests import audio_cases

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


def _packets(ts):
    ts = np.frombuffer(bytes(ts), dtype=np.uint8)
    return [ts[i:i + 188] for i in range(0, ts.size, 188)]


def _join(pkts):
    return np.concatenate(pkts) if len(pkts) else np.zeros(0, dtype=np.uint8)


def _masked(pcm, ranges):
    p = pcm.copy()
    for a, b in ranges:
        p[a:b] = 0
    return p


def _cut(ts, cuts):
    """TS -> list of chunks at the packet indices `cuts` (sorted, may repeat: empty chunks)"""
    pk = _packets(ts)
    edges = [0] + list(cuts) + [len(pk)]
    return [_join(pk[a:b]) for a, b in zip(edges[:-1], edges[1:])]


def _run(ctx, chunks, ends=None, queue_ahead=False):
    """chunks[k][s]: TS bytes of stream s in submit k. ends[k][s]: the stream ends after submit k's audio (default: in
    the last submit). queue_ahead: submit k + 1 before ef_decode_audio of submit k. Returns per stream the list of calls'
    results."""
    n, K = len(chunks[0]), len(chunks)
    if ends is None:
        ends = [[k == K - 1] * n for k in range(K)]
    out = [[] for _ in range(n)]
    packed = [ctx.pack(c) for c in chunks]
    ctx.submit_ts(*packed[0])
    for k in range(K):
        ctx.index()
        if queue_ahead and k + 1 < K:
            ctx.submit_ts(*packed[k + 1])
        res = ctx.decode_audio(end=np.array(ends[k], dtype=np.uint8))
        for s in range(n):
            out[s].append(res[s])
        if not queue_ahead and k + 1 < K:
            ctx.submit_ts(*packed[k + 1])
    return out


def _cat(calls, key):
    parts = [c[key] for c in calls]
    return np.concatenate(parts) if parts else np.zeros(0)


def _whole(es_list):
    return espflix_b200.audio_decode(es_list)


def _check_equal(calls, whole, oracle=None, es=None, what=""):
    pcm, pdm = _cat(calls, "pcm").astype(np.int16), _cat(calls, "pdm").astype(np.uint16)
    assert sum(c["n_frames"] for c in calls) == max(whole["n_frames"], 0), what
    assert np.array_equal(pcm, whole["pcm"]), "%s: PCM differs at %s" % (what, np.nonzero(pcm[:whole["pcm"].size] != whole["pcm"][:pcm.size])[0][:4])
    assert np.array_equal(pdm, whole["pdm"]), what
    if oracle is not None:
        want = oracle.sbc_decode(es)
        if isinstance(want, int):
            assert pcm.size == 0, what
        else:
            assert np.array_equal(pcm, want) and np.array_equal(pdm, oracle.pdm(want)), what


def test_whole_program_across_submits(oracle):
    """splash.ts and vmedia.ts in one context, cut at video PES starts into uneven submits of <= 12 pictures: video as
    pinned, audio as pinned and equal to the whole-file call"""
    names = ["splash", "vmedia"]
    ts = [open(os.path.join(G, n + ".ts"), "rb").read() for n in names]
    dpins = json.load(open(os.path.join(G, "decode_pins.json")))
    apins = json.load(open(os.path.join(G, "audio_pins.json")))
    sizes = [[5, 12, 1, 9, 7, 12, 3], [11, 2, 12, 8, 6, 4, 10]]
    per_stream = []
    for i, t in enumerate(ts):
        pk = _packets(t)
        starts = [k for k, q in enumerate(pk) if ((int(q[1]) << 8 | int(q[2])) & 0x1FFF) == 0x100 and q[1] & 0x40]
        cuts, p, j = [], 0, 0
        while True:
            p += sizes[i][j % len(sizes[i])]
            j += 1
            if p >= len(starts):
                break
            cuts.append(starts[p])
        per_stream.append(_cut(t, cuts))
    K = max(len(c) for c in per_stream)
    for c in per_stream:                                 # the shorter program ends early; empty chunks after it
        c += [np.zeros(0, dtype=np.uint8)] * (K - len(c))
    lens = [sum(1 for x in c if x.size) for c in per_stream]
    ends = [[k == lens[s] - 1 for s in range(2)] for k in range(K)]
    ctx = espflix_b200.Context(n_streams=2, max_pictures=13, max_slices_per_picture=8, es_capacity=1 << 21)
    ctx.enable_audio()
    frames = [[], []]
    audio = [[], []]
    for k in range(K):
        ctx.submit_ts(*ctx.pack([per_stream[0][k], per_stream[1][k]]))
        ctx.index()
        counts = [ctx.stream_info(s)[0] for s in range(2)]
        for p in range(max(counts)):
            ctx.decode_picture(p)
            for s in range(2):
                if p < counts[s]:
                    frames[s].append(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1))
        res = ctx.decode_audio(end=ends[k])
        for s in range(2):
            audio[s].append(res[s])
    whole = _whole(espflix_b200.audio_demux_ts(ts))
    for s, n in enumerate(names):
        assert len(frames[s]) == dpins[n]["frames"]
        for k, f in enumerate(frames[s]):
            assert hashlib.sha256(f.tobytes()).hexdigest() == dpins[n]["frame_sha256"][k], "%s picture %d" % (n, k)
        _check_equal(audio[s], whole[s], what=n)
        pcm, pdm = _cat(audio[s], "pcm").astype(np.int16), _cat(audio[s], "pdm").astype(np.uint16)
        assert max(c["frame_size"] for c in audio[s]) == apins[n]["frame_size"] and pcm.size == apins[n]["n_frames"] * 128
        assert hashlib.sha256(_masked(pcm, apins[n]["undefined"]).tobytes()).hexdigest() == apins[n]["pcm_sha256_masked"]
        assert hashlib.sha256(pdm[:apins[n]["pdm_defined_words"]].tobytes()).hexdigest() == apins[n]["pdm_sha256_defined"]
    ctx.close()


def _synthetic_batch():
    streams = []
    for i in range(48):
        streams.append(audio_cases.sbc_stream(5000 + i, 3 + i % 11, bitpool=[2, 7, 12, 28, 31, 60, 97, 120][i % 8], allocation=i & 1, frequency=i % 4,
                                              consistent=i % 3 != 0, bad_frames=(2, 5) if i % 5 == 0 else (), loud=i % 7 == 0))
    streams.append(np.zeros(0, dtype=np.uint8))                          # empty
    streams.append(audio_cases.sbc_stream(1, 1)[:40].copy())             # shorter than its frame
    streams.append(np.full(200, 0x55, dtype=np.uint8))                   # no sync byte at all: rejected
    return streams


def _overrun_stream(seed):
    es = audio_cases.sbc_stream(seed, 24, bitpool=28, consistent=False, bad_frames=(3, 4, 11))
    for k in (1, 2, 6, 7, 9, 23):
        es[k * 64 + 2] = 40                              # bit pool 40: 8 + 2 * 40 bytes read
    return es


def test_batch_cut_anywhere(oracle):
    """the 51 synthetic streams of test_batch_of_synthetic_streams (rejected frames, inconsistent scale factors, loud,
    empty, sub-frame, no sync) and two whose frames read into the next frame, muxed with
    varied PES sizes, each cut at its own seeded packet boundaries over 7 submits (empty and single-packet chunks)"""
    streams = _synthetic_batch() + [_overrun_stream(31), _overrun_stream(32)]
    n, K = len(streams), 7
    ts = [audio_cases.mux_audio_ts(es, pid=0x101 if i % 2 else 0x102, pes_bytes=[61, 188, 333, 1024, 2000][i % 5]) for i, es in enumerate(streams)]
    chunks = []
    for i, t in enumerate(ts):
        r = np.random.RandomState(900 + i)
        n_pk = t.size // 188
        cuts = sorted(r.randint(0, n_pk + 1, size=K - 1).tolist())
        if i % 4 == 0 and n_pk > 2:                      # a single-packet chunk followed by an empty one
            a = int(r.randint(0, n_pk - 1))
            cuts = sorted(cuts[:K - 4] + [a, a + 1, a + 1])
        chunks.append(_cut(t, cuts))
    assert all(len(c) == K for c in chunks)
    ctx = espflix_b200.Context(n_streams=n, max_pictures=2, es_capacity=1 << 22, fields=False)
    ctx.enable_audio()
    out = _run(ctx, [[chunks[s][k] for s in range(n)] for k in range(K)])
    whole = _whole(streams)
    for s in range(n):
        _check_equal(out[s], whole[s], oracle, streams[s], "stream %d" % s)
    assert whole[-5]["n_frames"] == 0 and whole[-4]["n_frames"] == 0
    ctx.close()


def _one(oracle, es, pieces_ts, what, whole_es=None, expect=None):
    """one stream whose audio comes in the given TS pieces, one per submit"""
    ctx = espflix_b200.Context(n_streams=1, max_pictures=2, es_capacity=1 << 20, fields=False)
    ctx.enable_audio()
    out = _run(ctx, [[p] for p in pieces_ts])[0]
    whole_es = es if whole_es is None else whole_es
    _check_equal(out, _whole([whole_es])[0], oracle, whole_es, what)
    if expect:
        expect(out)
    ctx.close()
    return out


def test_cuts_placed_on_purpose(oracle):
    # one frame per submit. Frames whose header asks for a larger bit pool than frame 0's read 88 bytes where the frame
    # size is 64: their bit loader runs into the next frame, whose bytes come one submit later (the frame is held back),
    # the last one past the end of the stream. Rejected frames repeat an accepted frame decoded one or two submits earlier.
    es = _overrun_stream(4242)
    fs = 8 + 2 * 28
    pieces = [audio_cases.mux_audio_ts(es[a:a + fs]) for a in range(0, es.size, fs)]

    def held_back(out):
        got = np.cumsum([c["n_frames"] for c in out])
        assert any(got[k] < k + 1 for k in range(len(out) - 1)), "no frame was held back for its overrun bytes"
    _one(oracle, es, pieces, "one frame per submit", expect=held_back)
    # the same cut two bytes into the next frame, and cuts inside the probe's bytes (header, scale factors, frame 0)
    for cuts in ([3, 7, fs - 1, fs + 2, 3 * fs, 4 * fs + 1], [1, 8, 9, 2 * fs - 1]):
        edges = [0] + cuts + [es.size]
        pieces = [audio_cases.mux_audio_ts(es[a:b]) for a, b in zip(edges[:-1], edges[1:])]
        out = _one(oracle, es, pieces, "cuts %s" % cuts)
        assert out[0]["frame_size"] == 0 and out[0]["n_frames"] == 0   # fewer bytes than the probe needs: nothing learned yet
    # a PES without PTS, cut between its start packet and its continuation packets: the gate stays shut across the submit;
    # and cut right after a PES start with PTS: it stays open
    es = audio_cases.sbc_stream(77, 40)
    ts = audio_cases.mux_audio_ts(es, pes_bytes=512, drop_pts_on=(1, 3))
    pk = _packets(ts)
    starts = [k for k, q in enumerate(pk) if q[1] & 0x40]
    pieces = _cut(ts, [starts[1] + 1, starts[2] + 1, starts[3] + 1, starts[3] + 2])
    want_es = oracle.demux_audio_ts(ts)
    assert np.array_equal(espflix_b200.audio_demux_ts([ts])[0], want_es) and want_es.size == es.size - 1024
    _one(oracle, es, pieces, "gate cut", whole_es=want_es)


def test_streams_ending_at_different_submits(oracle):
    """Per-stream end_of_stream: a new program fed into an ended stream decodes as if it were alone, whether its first
    submit is queued before or after the call that ends the old one; ef_reset clears all audio state."""
    a = audio_cases.sbc_stream(11, 30, bitpool=31, consistent=False, bad_frames=(7,))
    b = audio_cases.sbc_stream(12, 25, bitpool=12, allocation=1, frequency=0)
    c = audio_cases.sbc_stream(13, 20, bitpool=60, loud=True)
    ta, tb, tc = (audio_cases.mux_audio_ts(x, pes_bytes=400) for x in (a, b, c))
    tb_tail = _join(_packets(tb)[1:])                    # program b without its first packet: starts with continuation packets
    b_alone = oracle.demux_audio_ts(tb_tail)
    assert b_alone.size < b.size
    pa, pb, pc = (_cut(t, [t.size // 188 // 3, 2 * t.size // 188 // 3]) for t in (ta, tb_tail, tc))
    empty = np.zeros(0, dtype=np.uint8)
    # stream 0: a over submits 0-2, ends at 2, then b (tail) over 3-5; stream 1: c over 0-5 ends at 5; stream 2: c ends at 1
    chunks = [[pa[0], pc[0], _join(_packets(tc)[:5])],
              [pa[1], empty, _join(_packets(tc)[5:])],
              [pa[2], pc[1], empty],
              [pb[0], empty, empty],
              [pb[1], pc[2], empty],
              [pb[2], empty, empty]]
    ends = [[0, 0, 0], [0, 0, 1], [1, 0, 0], [0, 0, 0], [0, 0, 0], [1, 1, 1]]
    for queue_ahead in (False, True):
        ctx = espflix_b200.Context(n_streams=3, max_pictures=2, es_capacity=1 << 20, fields=False)
        ctx.enable_audio()
        out = _run(ctx, chunks, ends, queue_ahead=queue_ahead)
        wa, wb, wc = _whole([a, b_alone, c])
        _check_equal(out[0][:3], wa, oracle, a, "program a")
        _check_equal(out[0][3:], wb, oracle, b_alone, "program b after a (queued ahead: %s)" % queue_ahead)
        _check_equal(out[1], wc, oracle, c, "stream 1")
        _check_equal(out[2][:2], wc, oracle, c, "stream 2")
        assert all(r["n_frames"] == 0 for r in out[2][2:])
        # ef_reset in the middle of a program: the next program starts from nothing, audio stays enabled
        ctx.reset()
        ctx.submit_ts(*ctx.pack([pa[0], pa[0], pa[0]]))
        ctx.index()
        ctx.decode_audio()
        ctx.reset()
        out = _run(ctx, [[pc[0], pb[0], pa[0]], [pc[1], pb[1], pa[1]], [pc[2], pb[2], pa[2]]])
        for s, (w, e) in enumerate(zip(_whole([c, b_alone, a]), [c, b_alone, a])):
            _check_equal(out[s], w, oracle, e, "after reset, stream %d" % s)
        ctx.close()


def test_sizing_and_errors(oracle):
    es = [audio_cases.sbc_stream(21, 30), audio_cases.sbc_stream(22, 17, bitpool=60, consistent=False)]
    ts = [audio_cases.mux_audio_ts(e) for e in es]
    halves = [_cut(t, [t.size // 188 // 2]) for t in ts]
    ctx = espflix_b200.Context(n_streams=2, max_pictures=2, es_capacity=1 << 20, fields=False)
    with pytest.raises(espflix_b200.EspflixError) as e:
        ctx.decode_audio()
    assert e.value.code == capi.EF_ESTATE
    ctx.enable_audio()
    ctx.enable_audio()                                   # idempotent
    ctx.submit_ts(*ctx.pack([halves[0][0], halves[1][0]]))
    ctx.index()
    info = np.zeros(2, dtype=capi._AUDIO_INFO)
    for _ in range(2):                                   # sizing calls change nothing
        ctx._check(ctx.lib.ef_decode_audio(ctx._h, None, info.ctypes.data, None, 0, None, 0))
    need = int(info["n_frames"].sum()) * 128
    assert need > 0
    small = np.zeros(need - 1, dtype=np.int16)
    rc = ctx.lib.ef_decode_audio(ctx._h, None, info.ctypes.data, small.ctypes.data, small.size, None, 0)
    assert rc == capi.EF_ENOMEM                          # state untouched
    first = ctx.decode_audio()
    assert [r["n_frames"] for r in first] == [int(x) for x in info["n_frames"]]
    ctx.index()                                          # the same front buffer again: no new audio
    again = ctx.decode_audio()
    assert all(r["n_frames"] == 0 for r in again)
    ctx.submit_ts(*ctx.pack([halves[0][1], halves[1][1]]))
    ctx.index()
    ctx.submit_ts(*ctx.pack([halves[0][1], halves[1][1]]))
    with pytest.raises(espflix_b200.EspflixError) as e:   # the current submit's audio has not been consumed
        ctx.index()
    assert e.value.code == capi.EF_ESTATE
    last = ctx.decode_audio(end=True)
    whole = _whole(es)
    for s in range(2):
        _check_equal([first[s], again[s], last[s]], whole[s], oracle, es[s], "stream %d" % s)
    # ES submits carry no audio
    ctx.submit_es(*ctx.pack([es[0], es[1]]))
    ctx.index()
    assert all(r["n_frames"] == 0 and r["frame_size"] == 0 for r in ctx.decode_audio())
    ctx.close()


def test_audio_disabled_context_launches_what_it_did():
    """without ef_audio_enable a TS submit launches exactly the video demux kernels"""
    ctx = espflix_b200.Context(n_streams=2, max_pictures=2, es_capacity=1 << 20, fields=False)
    ts = audio_cases.mux_audio_ts(audio_cases.sbc_stream(5, 10))
    n0 = ctx.launch_count()
    ctx.submit_ts(*ctx.pack([ts, ts]))
    assert ctx.launch_count() - n0 == 4
    ctx.index()
    ctx.enable_audio()
    n0 = ctx.launch_count()
    ctx.submit_ts(*ctx.pack([ts, ts]))
    assert ctx.launch_count() - n0 == 4 + 4
    ctx.close()
