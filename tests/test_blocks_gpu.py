"""The CUDA decode path on the block-level streams of tests/block_cases.py: every picture of every case against the
restatement and, for the cases inside the reference's domain, against what the unmodified reference computed
(tests/golden/block_pins.json). Three schedules: all cases in one batch, each case alone in a one-stream context, and one
record picture per reconstruction launch (EF_REC_PICS=1)."""
import functools
import json
import os

import pytest

from tests import block_cases as bc
from tests.harness import check_picture, decode_es_batch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "block_pins.json")))
NAMES = bc.case_names()


@functools.lru_cache(maxsize=None)
def _case(name):
    return bc.make(name)


@pytest.fixture(scope="module")
def want(oracle):
    """restatement pictures of every case"""
    return {n: oracle.decode_es(_case(n)[0]) for n in NAMES}


@pytest.mark.parametrize("rec_pics", [None, "1"])
def test_all_cases_in_one_batch(want, monkeypatch, rec_pics):
    if rec_pics is None:
        monkeypatch.delenv("EF_REC_PICS", raising=False)
    else:
        monkeypatch.setenv("EF_REC_PICS", rec_pics)
    n = max(w.shape[0] for w in want.values())
    out, counts = decode_es_batch([_case(name)[0] for name in NAMES], n)
    for i, name in enumerate(NAMES):
        assert counts[i] == want[name].shape[0], name
        for k in range(counts[i]):
            check_picture(PINS, name, k, out[k, i], want[name][k])


@pytest.mark.parametrize("name", NAMES)
def test_case_alone(want, name):
    """a one-stream context: a grid of a few CTAs, so the warp pairs meet other work orders"""
    out, counts = decode_es_batch([_case(name)[0]], want[name].shape[0])
    assert counts[0] == want[name].shape[0]
    for k in range(counts[0]):
        check_picture(PINS, name, k, out[k, 0], want[name][k])
