"""The CUDA decode path on the block-level streams of tests/block_cases.py: every picture of every case against the
restatement and, for the cases inside the reference's domain, against what the unmodified reference computed
(tests/golden/block_pins.json). Three schedules: all cases in one batch, each case alone in a one-stream context, and one
record picture per reconstruction launch (EF_REC_PICS=1)."""
import functools
import hashlib
import json
import os

import numpy as np
import pytest

import espflix_b200
from tests import block_cases as bc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "block_pins.json")))
NAMES = bc.case_names()
I420 = 352 * 192 * 3 // 2


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@functools.lru_cache(maxsize=None)
def _case(name):
    return bc.make(name)


@pytest.fixture(scope="module")
def want(oracle):
    """restatement pictures of every case"""
    return {n: oracle.decode_es(_case(n)[0]) for n in NAMES}


def _where(got, ref):
    """plane, macroblock (mx, my) and block of the first differing byte of two I420 pictures"""
    i = int(np.nonzero(got != ref)[0][0])
    if i < 352 * 192:
        x, y = i % 352, i // 352
        return "Y mb (%d, %d) block %d, got %d want %d" % (x // 16, y // 16, (x >> 3 & 1) | (y >> 3 & 1) << 1, got[i], ref[i])
    j = (i - 352 * 192) % (176 * 96)
    plane, blk = ("Cr", 4) if i < 352 * 192 + 176 * 96 else ("Cb", 5)
    return "%s mb (%d, %d) block %d, got %d want %d" % (plane, j % 176 // 8, j // 176 // 8, blk, got[i], ref[i])


def _check(name, k, got, ref):
    if not np.array_equal(got, ref):
        pytest.fail("%s picture %d differs from the restatement: %d bytes, first at %s" % (name, k, int((got != ref).sum()), _where(got, ref)))
    if name in PINS:
        assert sha(got) == PINS[name]["frame_sha256"][k], "%s picture %d differs from the reference's pin" % (name, k)


def _decode(streams, n_pictures):
    """one submit of every stream, every picture to the host: out[picture][stream]"""
    ctx = espflix_b200.Context(n_streams=len(streams), max_pictures=12, max_slices_per_picture=12,
                               es_capacity=sum(len(s) for s in streams) + 4096, fields=False)
    blob, off = ctx.pack(streams)
    ctx.submit_es(blob, off)
    ctx.index()
    counts = [ctx.stream_info(i)[0] for i in range(len(streams))]
    out = np.zeros((n_pictures, len(streams), I420), dtype=np.uint8)
    ctx.decode_all_to_host(n_pictures, out)
    ctx.sync()
    ctx.close()
    return out, counts


@pytest.mark.parametrize("rec_pics", [None, "1"])
def test_all_cases_in_one_batch(want, monkeypatch, rec_pics):
    if rec_pics is None:
        monkeypatch.delenv("EF_REC_PICS", raising=False)
    else:
        monkeypatch.setenv("EF_REC_PICS", rec_pics)
    n = max(w.shape[0] for w in want.values())
    out, counts = _decode([_case(name)[0] for name in NAMES], n)
    for i, name in enumerate(NAMES):
        assert counts[i] == want[name].shape[0], name
        for k in range(counts[i]):
            _check(name, k, out[k, i], want[name][k])


@pytest.mark.parametrize("name", NAMES)
def test_case_alone(want, name):
    """a one-stream context: a grid of a few CTAs, so the warp pairs meet other work orders"""
    out, counts = _decode([_case(name)[0]], want[name].shape[0])
    assert counts[0] == want[name].shape[0]
    for k in range(counts[0]):
        _check(name, k, out[k, 0], want[name][k])
