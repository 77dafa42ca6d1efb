"""The CUDA decode path on the syntax-level streams of tests/syntax_cases.py: every picture of every stream against the
restatement and, for the pinned cases, against what the unmodified reference computed (tests/golden/syntax_pins.json).
The same streams run under several schedules: all cases in one batch (warp pairs mix sizes, picture types and
densities), one K1a launch per picture index, each directed case alone in a one-stream context, and submits cut at
picture boundaries (the carried vector parameters, sequence state and ping-pong phase)."""
import functools
import json
import os

import numpy as np
import pytest

import espflix_b200
from tests import syntax_cases as sc
from tests.harness import I420, check_picture, decode_es_batch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "syntax_pins.json")))
NAMES = sc.case_names()


@functools.lru_cache(maxsize=None)
def _case(name):
    return sc.outside_case() if name == "outside" else sc.make(name)


@pytest.fixture(scope="module")
def want(oracle):
    """restatement pictures of every case"""
    return {n: oracle.decode_es(_case(n)[0]) for n in NAMES + ["outside"]}


@pytest.mark.parametrize("rec_pics", [None, "1"])
def test_whole_batch_in_one_context(want, monkeypatch, rec_pics):
    if rec_pics is None:
        monkeypatch.delenv("EF_REC_PICS", raising=False)
    else:
        monkeypatch.setenv("EF_REC_PICS", rec_pics)
    out, counts = decode_es_batch([_case(n)[0] for n in NAMES], 12)
    for i, name in enumerate(NAMES):
        assert counts[i] == want[name].shape[0], name
        for k in range(counts[i]):
            check_picture(PINS, name, k, out[k, i], want[name][k])


@pytest.mark.parametrize("name", list(sc.DIRECTED))
def test_directed_case_alone(want, name):
    """a one-stream context: a grid of a few CTAs and a different slice-to-lane schedule"""
    out, counts = decode_es_batch([_case(name)[0]], want[name].shape[0])
    assert counts[0] == want[name].shape[0]
    for k in range(counts[0]):
        check_picture(PINS, name, k, out[k, 0], want[name][k])


def test_submits_cut_at_picture_boundaries(want):
    """every stream cut into three submits at seeded picture boundaries: the vector parameters of the last P header
    (pictures of type 3 / 4), the sequence state and the frame-store phase carry from one submit to the next"""
    rng = sc.Rng(0xC07)
    cuts = []
    for name in NAMES:
        n = want[name].shape[0]
        a = rng.int(1, n - 2)
        cuts.append((0, a, rng.int(a + 1, n - 1), n))
    ctx = espflix_b200.Context(n_streams=len(NAMES), max_pictures=12, max_slices_per_picture=12,
                               es_capacity=sum(len(_case(n)[0]) for n in NAMES) + 4096, fields=False)
    for part in range(3):
        streams = []
        for name, c in zip(NAMES, cuts):
            es, off = _case(name)[0], _case(name)[1]
            streams.append(es[off[c[part]]:off[c[part + 1]]])
        blob, off = ctx.pack(streams)
        ctx.submit_es(blob, off)
        ctx.index()
        n_pics = ctx.index_info()["max_pictures"]
        out = np.zeros((n_pics, len(NAMES), I420), dtype=np.uint8)
        ctx.decode_all_to_host(n_pics, out)
        ctx.sync()
        for i, (name, c) in enumerate(zip(NAMES, cuts)):
            assert ctx.stream_info(i)[0] == c[part + 1] - c[part], name
            for k in range(c[part], c[part + 1]):
                check_picture(PINS, name, k, out[k - c[part], i], want[name][k])
    ctx.close()


def test_windows_outside_the_frame_stay_isolated(want):
    """Macroblocks whose prediction window leaves the frame sideways, in the last picture of one stream of a batch.
    The device clamps the window into the frame where the reference reads the neighbouring strip bytes, so those
    macroblocks are not compared; every other macroblock of that picture and every other stream must be bit-exact."""
    names = [n for n in NAMES if n.startswith(("vector_", "small_"))] + ["outside"]
    out, counts = decode_es_batch([_case(n)[0] for n in names], 12)
    es, off, _, outside = _case("outside")
    last = len(off) - 2
    skip = np.zeros(I420, dtype=bool)
    yv = skip[:352 * 192].reshape(192, 352)
    cr = skip[352 * 192:352 * 192 + 176 * 96].reshape(96, 176)
    cb = skip[352 * 192 + 176 * 96:].reshape(96, 176)
    for mx, my in outside:
        yv[my * 16:my * 16 + 16, mx * 16:mx * 16 + 16] = True
        cr[my * 8:my * 8 + 8, mx * 8:mx * 8 + 8] = True
        cb[my * 8:my * 8 + 8, mx * 8:mx * 8 + 8] = True
    for i, name in enumerate(names):
        assert counts[i] == want[name].shape[0], name
        for k in range(counts[i]):
            if name == "outside" and k == last:
                got, ref = out[k, i].copy(), want[name][k].copy()
                got[skip] = ref[skip] = 0
                check_picture(PINS, name, k, got, ref)
            else:
                check_picture(PINS, name, k, out[k, i], want[name][k])
