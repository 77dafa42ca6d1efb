"""K0 (ef_scan_kernel, ef_prefix_kernel, ef_fill_kernel) on the start-code cases of tests/scan_cases.py: per-stream picture
counts and index totals against K0's rule, every decoded picture against the restatement and the reference's pins
(tests/golden/scan_pins.json), the picture pts of TS-wrapped cases, EF_ENOMEM exactly one past each index limit, the cases at
every batch shape K0's tiles meet, and the emulation cases cut at every packet boundary of a carrying context."""
import functools
import json
import os

import numpy as np
import pytest

import espflix_b200
from espflix_b200 import capi, synth
from tests import pts_cases
from tests import scan_cases as sc
from tests.harness import I420, error_code, sha

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "scan_pins.json")))
P, S = sc.LIMIT_PICTURES, sc.LIMIT_SLICES


def _in_limits(c):
    return not c.census.get("over")


@functools.lru_cache(maxsize=None)
def _want(es):
    """the pictures K0's rule gives the stream, as the restatement decodes them (an eos_code stream: the restatement's
    picture from the padding is not one of them)"""
    from tests.oracle_lib import Oracle
    n = sc.census_of(es)[0]
    return Oracle().decode_es(np.frombuffer(es, dtype=np.uint8))[:n] if n else np.zeros((0, I420), np.uint8)


def _check(name, es, got, pinned):
    want = _want(es)
    assert len(got) == want.shape[0], name
    for k, g in enumerate(got):
        assert np.array_equal(g, want[k]), "%s picture %d differs from the restatement" % (name, k)
        if pinned:
            assert sha(g) == PINS[name]["frame_sha256"][k], "%s picture %d differs from the reference's pin" % (name, k)


def _context(n, max_pictures=P, es_capacity=None):
    return espflix_b200.Context(n_streams=n, max_pictures=max_pictures, max_slices_per_picture=S,
                                es_capacity=es_capacity or (1 << 24), fields=False)


def _run(streams, misaligns, max_pictures=P):
    """one ES submit of the streams at the given base misalignments (None: packed back to back) -> (index_info, pictures of
    every stream)"""
    if misaligns is None:
        blob, off = espflix_b200.Context.pack(streams)
        idx = list(range(len(streams)))
    else:
        blob, off, idx = sc.pack(streams, misaligns)
    ctx = _context(len(off) - 1, max_pictures, int(off[-1]) + 4096)
    ctx.submit_es(blob, off)
    ctx.index()
    info = ctx.index_info()
    counts = [ctx.stream_info(i)[0] for i in idx]
    out = np.zeros((info["max_pictures"], len(off) - 1, I420), dtype=np.uint8)
    ctx.decode_all_to_host(info["max_pictures"], out)
    ctx.sync()
    ctx.close()
    return info, counts, [[out[p, i] for p in range(n)] for i, n in zip(idx, counts)]


def test_directed_cases_in_one_batch():
    cases = [c for c in sc.directed_cases() if _in_limits(c)]
    info, counts, got = _run([c.es for c in cases], [c.misalign for c in cases])
    census = [sc.census_of(c.es) for c in cases]
    assert info["total_pictures"] == sum(x[0] for x in census)
    assert info["total_slices"] == sum(x[1] for x in census)
    for c, n, g, x in zip(cases, counts, got, census):
        assert n == x[0], c.name
        _check(c.name, c.es, g, c.pinned)


@pytest.mark.parametrize("name", [c.name for c in sc.directed_cases() if c.name.startswith(("mat_", "tail_", "short", "lim_")) and _in_limits(c)])
def test_directed_case_alone(name):
    """one stream, based at its misalignment behind a filler stream (the cases past a limit: test_index_limits)"""
    c = {c.name: c for c in sc.directed_cases()}[name]
    info, counts, got = _run([c.es], [c.misalign])
    x = sc.census_of(c.es)
    assert counts[0] == x[0] and info["total_pictures"] == x[0] and info["total_slices"] == x[1]
    _check(c.name, c.es, got[0], c.pinned)


def test_geometry_every_offset_and_misalignment():
    cases = sc.geometry_cases()
    want = _want(sc.geometry_base())
    assert [sha(f) for f in want] == PINS["geo_base"]["frame_sha256"]
    for b in range(0, len(cases), 512):
        part = cases[b:b + 512]
        info, counts, got = _run([c.es for c in part], [c.misalign for c in part])
        assert info["total_pictures"] == 3 * len(part) and info["total_slices"] == sum(sc.census_of(c.es)[1] for c in part)
        for c, n, g in zip(part, counts, got):
            assert n == 3, c.name
            for k in range(3):
                assert np.array_equal(g[k], want[k]), "%s picture %d" % (c.name, k)


def test_index_limits():
    """EF_ENOMEM exactly one past max_pictures, max_pictures * max_slices_per_picture and max_seq (= max_pictures)"""
    for c in sc.limit_cases():
        blob, off, idx = sc.pack([c.es], [c.misalign])
        ctx = _context(len(off) - 1, es_capacity=int(off[-1]) + 4096)
        ctx.submit_es(blob, off)
        ctx.index()
        if c.census["over"]:
            assert error_code(ctx.index_info) == capi.EF_ENOMEM, c.name
        else:
            info = ctx.index_info()
            assert info["total_pictures"] == sc.census_of(c.es)[0], c.name
        ctx.close()


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1023, 1024, 1025, 2049])
def test_batch_shapes(n):
    """streams of 0 to max_pictures pictures (some without slices) and the directed cases, in ef_prefix_kernel's 1,024-stream
    tiles and ef_fill_kernel's (picture, stream) grid"""
    pool = sc.batch_pool() + [c.es for c in sc.directed_cases() if _in_limits(c)]
    streams = [pool[(k * 7) % len(pool)] for k in range(n)]
    info, counts, got = _run(streams, None)
    assert info["total_pictures"] == sum(sc.census_of(s)[0] for s in streams)
    assert info["total_slices"] == sum(sc.census_of(s)[1] for s in streams)
    assert info["max_pictures"] == max(sc.census_of(s)[0] for s in streams)
    for k, (s, g) in enumerate(zip(streams, got)):
        _check("stream %d" % k, s, g, False)


def _ts_cases():
    return [c for c in sc.directed_cases() if _in_limits(c) and sc.census_of(c.es)[0]]


def test_ts_wrapped_picture_pts():
    cases = _ts_cases()
    ts = [synth.wrap_ts(np.frombuffer(c.es, dtype=np.uint8), sc.unit_offsets(c.es)) for c in cases]
    ctx = _context(len(cases), es_capacity=sum(t.size for t in ts) + 4096)
    ctx.enable_pts()
    ctx.submit_ts(*ctx.pack(ts))
    ctx.index()
    ctx.index_info()
    pic, _ = ctx.picture_pts()
    for i, (c, t) in enumerate(zip(cases, ts)):
        n = ctx.stream_info(i)[0]
        assert n == sc.census_of(c.es)[0], c.name
        assert [int(v) for v in pic[i, :n]] == pts_cases.picture_pts(t), c.name
    ctx.close()


def _carry_run(per_stream, n_pictures=P):
    """per_stream[s]: the TS chunks of stream s, one per submit; the last submit ends every stream -> per stream the SHA-256
    of every picture and its pts"""
    n = len(per_stream)
    ctx = _context(n, n_pictures)
    ctx.enable_pts()
    ctx.enable_carry(65536)
    frames, pts = [[] for _ in range(n)], [[] for _ in range(n)]
    K = max(len(c) for c in per_stream)
    for k in range(K):
        ctx.submit_ts(*ctx.pack([c[k] if k < len(c) else b"" for c in per_stream]))
        if k == K - 1:
            ctx.end_streams(np.ones(n, dtype=np.uint8))
        ctx.index()
        ctx.index_info()
        counts = [ctx.stream_info(s)[0] for s in range(n)]
        for p in range(max(counts)):
            ctx.decode_picture(p)
            for s in range(n):
                if p < counts[s]:
                    frames[s].append(sha(ctx.read_frame_i420(s, (ctx.stream_info(s)[1] + p + 1) & 1)))
        pic, _ = ctx.picture_pts()
        for s in range(n):
            pts[s] += [int(v) for v in pic[s, :counts[s]]]
    ctx.close()
    return frames, pts


def test_emulation_cases_cut_at_every_packet():
    """each emulation case in two submits cut before every packet (a stream per cut): the pictures and pts equal the uncut
    stream's, and the pictures the restatement's"""
    cases = [c for c in sc.directed_cases() if c.name.startswith("mat_")]
    per_stream, whole, owner = [], [], []
    for c in cases:
        t = bytes(synth.wrap_ts(np.frombuffer(c.es, dtype=np.uint8), sc.unit_offsets(c.es)))
        whole.append([t])
        for k in range(len(t) // 188 + 1):
            per_stream.append([t[:188 * k], t[188 * k:]])
            owner.append(len(whole) - 1)
    ref_frames, ref_pts = _carry_run(whole)
    for c, f in zip(cases, ref_frames):
        assert f == [sha(x) for x in _want(c.es)], c.name
    frames, pts = _carry_run(per_stream)
    for s, o in enumerate(owner):
        assert frames[s] == ref_frames[o] and pts[s] == ref_pts[o], "%s cut %d" % (cases[o].name, s)
