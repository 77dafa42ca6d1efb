"""Parity of the CUDA decode path (through the C-ABI) against the oracle and the committed pins.
Bit-exact: the whole path is integer (the IDCT used is the reference's integer AAN transform)."""
import hashlib
import json
import os

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import synth
from tests.synth_cases import COVERAGE, UNPINNED, make

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


def _first_diff(a, b):
    d = np.nonzero(a != b)[0]
    return "no diff" if d.size == 0 else "%d bytes differ, first at %d (got %d want %d)" % (d.size, d[0], a[d[0]], b[d[0]])


@pytest.mark.parametrize("name", ["splash", "vmedia"])
def test_reference_fixture_es_path(oracle, name):
    """config 2: the reference's own embedded streams, every picture byte-exact vs the pins."""
    pins = json.load(open(os.path.join(G, "decode_pins.json")))[name]
    es = oracle.demux_ts(open(os.path.join(G, name + ".ts"), "rb").read())
    ctx = espflix_b200.Context(n_streams=1, max_pictures=128, max_slices_per_picture=8, es_capacity=1 << 20)
    frames = ctx.decode_sequence([es])[0]
    assert len(frames) == pins["frames"]
    for k, f in enumerate(frames):
        assert hashlib.sha256(f.tobytes()).hexdigest() == pins["frame_sha256"][k], "picture %d" % k
    assert hashlib.sha256(np.concatenate(frames).tobytes()).hexdigest() == pins["i420_sha256"]
    ctx.close()


@pytest.mark.parametrize("name", ["splash", "vmedia"])
def test_reference_fixture_ts_path(oracle, name):
    """next-row f1: the reference's wire format (188-byte TS, PID 0x100) demuxed on the device."""
    pins = json.load(open(os.path.join(G, "decode_pins.json")))[name]
    ts = open(os.path.join(G, name + ".ts"), "rb").read()
    ctx = espflix_b200.Context(n_streams=1, max_pictures=128, max_slices_per_picture=8, es_capacity=1 << 20)
    frames = ctx.decode_sequence([ts], ts=True)[0]
    assert len(frames) == pins["frames"]
    assert hashlib.sha256(np.concatenate(frames).tobytes()).hexdigest() == pins["i420_sha256"]
    ctx.close()


@pytest.mark.parametrize("idx", range(len(COVERAGE)), ids=[c[0] for c in COVERAGE])
def test_synthetic_coverage(oracle, idx):
    name, kw = COVERAGE[idx]
    es, _ = make(idx, kw)
    want = oracle.decode_es(es)
    ctx = espflix_b200.Context(n_streams=1, max_pictures=kw["n_pictures"], es_capacity=1 << 21)
    frames = ctx.decode_sequence([es])[0]
    assert len(frames) == want.shape[0] == kw["n_pictures"]
    for k in range(len(frames)):
        assert np.array_equal(frames[k], want[k]), "%s picture %d: %s" % (name, k, _first_diff(frames[k], want[k]))
    ctx.close()


@pytest.mark.parametrize("idx", range(len(UNPINNED)), ids=[c[0] for c in UNPINNED])
def test_outside_reference_domain_matches_oracle(oracle, idx):
    name, kw = UNPINNED[idx]
    es, _ = synth.generate(synth.SEED0 + 2000 + idx, **kw)
    want = oracle.decode_es(es)
    ctx = espflix_b200.Context(n_streams=1, max_pictures=kw["n_pictures"], es_capacity=1 << 22)
    frames = ctx.decode_sequence([es])[0]
    for k in range(len(frames)):
        assert np.array_equal(frames[k], want[k]), "%s picture %d: %s" % (name, k, _first_diff(frames[k], want[k]))
    ctx.close()


def test_batch_of_mixed_streams(oracle):
    """Many streams of different structure in one context: lanes of one warp parse slices of
    different streams, picture types and slice layouts at the same time."""
    streams = [make(i, kw)[0] for i, (_, kw) in enumerate(COVERAGE) if kw["n_pictures"] == 12]
    streams += [synth.generate(synth.SEED0 + 50 + i)[0] for i in range(37)]
    streams.append(np.zeros(0, dtype=np.uint8))                         # empty stream
    streams.append(streams[0][: streams[0].size // 2].copy())           # ragged: truncated mid-picture
    n = len(streams)
    ctx = espflix_b200.Context(n_streams=n, max_pictures=12, es_capacity=1 << 23)
    blob, off = ctx.pack(streams)
    ctx.submit_es(blob, off)
    ctx.index()
    info = ctx.index_info()
    assert info["max_pictures"] == 12
    ctx.decode_all(12)
    got = ctx.read_latest_i420()
    for i in range(n - 2):
        want = oracle.decode_es(streams[i])
        assert np.array_equal(got[i], want[-1]), "stream %d: %s" % (i, _first_diff(got[i], want[-1]))
    assert ctx.stream_info(n - 2)[0] == 0
    assert (got[n - 2] == 0).all()                                      # never-written frame store stays zero (Frame::init)
    ctx.close()


def test_chunked_submits_carry_state(oracle):
    """Submits cut at GOP boundaries: ping-pong phase and sequence state persist across submits."""
    es, off = synth.generate(synth.SEED0 + 77, n_pictures=36, gop=12, flags=synth.MATRICES)
    want = oracle.decode_es(es)
    ctx = espflix_b200.Context(n_streams=1, max_pictures=13, es_capacity=1 << 22)
    got = []
    for a, b in ((0, 12), (12, 25), (25, 36)):                          # uneven cuts, second one mid-GOP
        got += ctx.decode_sequence([es[off[a]:off[b]]])[0]
    assert len(got) == 36
    for k in range(36):
        assert np.array_equal(got[k], want[k]), "picture %d: %s" % (k, _first_diff(got[k], want[k]))
    ctx.close()


def test_replicated_batch_properties():
    """config 4 shape at reduced width: D distinct streams replicated R times must give R identical
    copies (size-independent property: no cross-stream interference in the warp-shared kernel)."""
    D, R = 16, 24
    distinct = [synth.generate(synth.SEED0 + i)[0] for i in range(D)]
    streams = [distinct[i % D] for i in range(D * R)]
    ctx = espflix_b200.Context(n_streams=D * R, max_pictures=12, es_capacity=1 << 26, fields=False)
    blob, off = ctx.pack(streams)
    ctx.submit_es(blob, off)
    ctx.index()
    info = ctx.index_info()
    assert info["total_pictures"] == D * R * 12 and info["total_slices"] == D * R * 12 * 12
    ctx.decode_all(12)
    got = ctx.read_latest_i420()
    for i in range(D, D * R):
        assert np.array_equal(got[i], got[i % D]), i
    # decoding the same submit again (next GOP period) is idempotent: I pictures refresh everything
    ctx.index()
    ctx.decode_all(12)
    assert np.array_equal(ctx.read_latest_i420(), got)
    ctx.close()


def test_error_paths():
    ctx = espflix_b200.Context(n_streams=2, max_pictures=2, es_capacity=4096)
    with pytest.raises(espflix_b200.EspflixError):
        ctx.index()                                                     # index before submit
    blob = np.zeros(8192, dtype=np.uint8)
    with pytest.raises(espflix_b200.EspflixError):
        ctx.submit_es(blob, np.array([0, 4096, 8192], dtype=np.uint64))  # exceeds es_capacity
    es, _ = synth.generate(synth.SEED0, n_pictures=4, gop=4, noise=0)
    small = espflix_b200.Context(n_streams=1, max_pictures=2, es_capacity=1 << 20)
    b, o = small.pack([es])
    small.submit_es(b, o)
    small.index()
    with pytest.raises(espflix_b200.EspflixError):
        small.index_info()                                              # 4 pictures > max_pictures 2
    small.close()
    ctx.close()


def test_pipelined_submits_and_async_readback(oracle):
    """Submit batch k+1 while batch k is still in flight, read back asynchronously: results must equal
    the plain synchronous sequence (double-buffered ES upload and read-back staging in the C-ABI)."""
    batches = [[synth.generate(synth.SEED0 + 300 + 7 * b + i, n_pictures=6, gop=6)[0] for i in range(5)] for b in range(4)]
    ctx = espflix_b200.Context(n_streams=5, max_pictures=6, es_capacity=1 << 21, fields=False)
    outs = [np.zeros((5, 101376), dtype=np.uint8) for _ in batches]
    packed = [ctx.pack(b) for b in batches]
    for k, (blob, off) in enumerate(packed):
        ctx.submit_es(blob, off)
        ctx.index()
        ctx.decode_all(6)
        ctx.read_latest_i420_async(0, 5, outs[k])
    ctx.sync()
    for k, b in enumerate(batches):
        for i, es in enumerate(b):
            assert np.array_equal(outs[k][i], oracle.decode_es(es)[-1]), (k, i)
    ctx.close()


def test_growing_readback_frees_replaced_staging():
    """Read-backs whose stream count grows call after call: each staging buffer that grows frees the one it replaces, so the
    context holds two buffers of the largest count (2 x 52 MB here), not every earlier one (about 13 GB)."""
    import torch
    n = 512
    es, _ = synth.generate(synth.SEED0, n_pictures=2, gop=2)
    ctx = espflix_b200.Context(n_streams=n, max_pictures=2, es_capacity=n * len(es) + 4096, fields=False)
    ctx.submit_es(*ctx.pack([es] * n))
    ctx.index()
    out = torch.empty(n * 101376, dtype=torch.uint8, pin_memory=True)
    ctx.sync()
    free0, _ = torch.cuda.mem_get_info()
    for k in range(1, n + 1):
        ctx.read_latest_i420_async(0, k, out.data_ptr())
    ctx.sync()
    free1, _ = torch.cuda.mem_get_info()
    ctx.close()
    assert free0 - free1 < 2 << 30, "%.1f GB of device memory held after the read-backs" % ((free0 - free1) / 2**30)


@pytest.mark.parametrize("rec_pics", [None, "1", "5"])
def test_decode_all_multi_picture_parse(oracle, monkeypatch, rec_pics):
    """ef_decode_all parses every slice of up to rec_pics picture indices in ONE K1a launch and rebuilds
    them picture by picture; whatever the chunking, the two frame stores of every stream must end up
    holding its last two pictures. Also: decoding the same index twice gives the same frames."""
    if rec_pics is None:
        monkeypatch.delenv("EF_REC_PICS", raising=False)
    else:
        monkeypatch.setenv("EF_REC_PICS", rec_pics)
    streams = [make(i, kw)[0] for i, (_, kw) in enumerate(COVERAGE) if kw["n_pictures"] == 12][:6]
    streams += [synth.generate(synth.SEED0 + 900 + i)[0] for i in range(11)]
    streams.append(synth.generate(synth.SEED0 + 950, n_pictures=7)[0])      # a shorter stream in the same batch
    want = [oracle.decode_es(s) for s in streams]
    ctx = espflix_b200.Context(n_streams=len(streams), max_pictures=12, es_capacity=sum(len(s) for s in streams) + 4096)
    blob, off = ctx.pack(streams)
    ctx.submit_es(blob, off)
    for _ in range(2):
        ctx.index()
        ctx.decode_all(12)
        for i, w in enumerate(want):
            n = w.shape[0]
            got_last = ctx.read_frame_i420(i, -1)
            assert np.array_equal(got_last, w[n - 1]), "stream %d last picture: %s" % (i, _first_diff(got_last, w[n - 1]))
            base = ctx.stream_info(i)[1]
            got_prev = ctx.read_frame_i420(i, (base + n) & 1 ^ 1)
            assert np.array_equal(got_prev, w[n - 2]), "stream %d previous picture" % i
        ctx.reset()
        ctx.submit_es(blob, off)
    ctx.close()


def test_full_baseline_batch_is_bit_exact(oracle):
    """The benchmarked configuration itself (BASELINE config 4 = bench.py's workload: 4,096 streams x 12
    pictures, 64 distinct seeds replicated 64 times, one ef_decode_all): every distinct stream's last two
    pictures equal the oracle's, and every replica equals its original (no cross-stream interference at the
    size the throughput number is quoted on)."""
    import bench
    gen, streams = bench.make_streams(bench.STREAMS_PER_GPU, 0)
    d = len(gen)
    ctx = espflix_b200.Context(n_streams=len(streams), max_pictures=bench.PICTURES, max_slices_per_picture=12,
                               es_capacity=sum(len(s) for s in streams) + 4096, fields=False)
    blob, off = ctx.pack(streams)
    ctx.submit_es(blob, off)
    ctx.index()
    info = ctx.index_info()
    assert info["total_pictures"] == len(streams) * bench.PICTURES and info["total_slices"] == len(streams) * bench.PICTURES * 12
    ctx.decode_all(bench.PICTURES)
    got = ctx.read_latest_i420()
    for i in range(d):
        want = oracle.decode_es(gen[i][0])
        assert want.shape[0] == bench.PICTURES
        assert np.array_equal(got[i], want[-1]), "stream %d last picture: %s" % (i, _first_diff(got[i], want[-1]))
        base = ctx.stream_info(i)[1]
        prev = ctx.read_frame_i420(i, ((base + bench.PICTURES) & 1) ^ 1)
        assert np.array_equal(prev, want[-2]), "stream %d previous picture" % i
    g = got.reshape(len(streams) // d, d, -1)
    assert np.array_equal(g, np.broadcast_to(g[0], g.shape)), "a replica differs from its original"
    ctx.close()


def _start_codes(es):
    e = np.asarray(es)
    hits = np.nonzero((e[:-3] == 0) & (e[1:-2] == 0) & (e[2:-1] == 1))[0]
    return [(int(p), int(e[p + 3])) for p in hits]


def test_truncated_slice_does_not_disturb_its_neighbours(oracle):
    """Damaged input (a lost TS packet, a cut file): a slice that ends in the middle of a block is followed at once
    by the next stream's start code and payload, i.e. by non-zero bytes in coefficient context. The parser has
    to derail on the 23 zero bits of the start code prefix (>= 12 leading zeros is not a code) instead of decoding
    stale bytes as coefficients: the neighbours' coefficient lists, records and pictures must stay intact, and
    so must the pictures of the damaged stream before the cut."""
    full = [synth.generate(synth.SEED0 + 400 + i)[0] for i in range(5)]
    streams = [np.asarray(f).copy() for f in full]
    cuts = {}
    for i, frac in ((0, 0.4), (2, 0.7), (4, 0.15)):
        sc = [p for p, c in _start_codes(full[i]) if 1 <= c <= 0xAF]
        last = sc[-1]                                                   # last slice of the last picture
        cut = last + 4 + max(3, int((len(full[i]) - last - 4) * frac))
        streams[i] = np.asarray(full[i][:cut]).copy()
        cuts[i] = cut
    ctx = espflix_b200.Context(n_streams=len(streams), max_pictures=12, es_capacity=sum(len(s) for s in streams) + 4096, fields=False)
    blob, off = ctx.pack(streams)
    for _ in range(2):                                                  # twice: the second pass runs over a used list buffer
        ctx.submit_es(blob, off)
        ctx.index()
        ctx.decode_all(12)
        got = ctx.read_latest_i420()
        for i, f in enumerate(full):
            want = oracle.decode_es(f)
            base = ctx.stream_info(i)[1]
            prev = ctx.read_frame_i420(i, ((base + 12) & 1) ^ 1)
            assert np.array_equal(prev, want[10]), "stream %d picture 10: %s" % (i, _first_diff(prev, want[10]))
            if i not in cuts:
                assert np.array_equal(got[i], want[11]), "intact stream %d: %s" % (i, _first_diff(got[i], want[11]))
            else:                                                       # rows above the damaged slice are intact
                rows = 16 * 11
                assert np.array_equal(got[i][: 352 * rows], want[11][: 352 * rows]), "stream %d rows above the cut slice" % i
        ctx.reset()
    ctx.close()


def test_decode_all_to_host_hands_over_every_picture(oracle):
    """ef_decode_all_to_host = the decode loop with the reference's push_video() hand-over: every picture of every
    stream arrives on the host, exported between the reconstruction launches while the next picture is rebuilt
    (the two frame stores of a stream are overwritten two pictures later). Two submits in a row exercise the
    alternating staging buffers and the carried ping-pong phase."""
    n, pics = 7, 9
    batches = [[synth.generate(synth.SEED0 + 600 + 10 * b + i, n_pictures=pics, gop=pics)[0] for i in range(n)] for b in range(2)]
    ctx = espflix_b200.Context(n_streams=n, max_pictures=pics, es_capacity=1 << 22, fields=False)
    for b, streams in enumerate(batches):
        out = np.zeros((pics, n, 101376), dtype=np.uint8)
        blob, off = ctx.pack(streams)
        ctx.submit_es(blob, off)
        ctx.index()
        ctx.decode_all_to_host(pics, out)
        ctx.sync()
        for i, es in enumerate(streams):
            want = oracle.decode_es(es)
            for p in range(pics):
                assert np.array_equal(out[p, i], want[p]), "batch %d stream %d picture %d: %s" % (b, i, p, _first_diff(out[p, i], want[p]))
    ctx.close()


@pytest.mark.parametrize("rank", [1, 5, 7])
def test_rank_specific_seed_windows_are_bit_exact(oracle, rank):
    """SURVEY.md 4 "per-rank parity on a rank-specific slice": bench.py gives every rank its own window of the seed
    space (shard.stream_seed_index). The streams ranks > 0 decode in the scaling runs are checked against the oracle
    here on one GPU: all 64 distinct streams of that rank's window, last two pictures each."""
    import bench
    gen, streams = bench.make_streams(bench.DISTINCT, rank)
    gen0, _ = bench.make_streams(2, 0)
    assert not np.array_equal(gen[0][0][:4096], gen0[0][0][:4096])      # a different window from rank 0's
    ctx = espflix_b200.Context(n_streams=len(streams), max_pictures=bench.PICTURES, es_capacity=sum(len(s) for s in streams) + 4096, fields=False)
    blob, off = ctx.pack(streams)
    ctx.submit_es(blob, off)
    ctx.index()
    ctx.decode_all(bench.PICTURES)
    got = ctx.read_latest_i420()
    for i in range(len(streams)):
        want = oracle.decode_es(gen[i][0])
        assert np.array_equal(got[i], want[-1]), "rank %d stream %d: %s" % (rank, i, _first_diff(got[i], want[-1]))
        base = ctx.stream_info(i)[1]
        prev = ctx.read_frame_i420(i, ((base + bench.PICTURES) & 1) ^ 1)
        assert np.array_equal(prev, want[-2]), "rank %d stream %d previous picture" % (rank, i)
    ctx.close()
