"""ef_trick_build against the restatement (tests/trick_cases.py): video_fwd.ts and video_rwd.ts byte for byte, and the argument checks."""

import numpy as np
import pytest

from tests import restart_cases, trick_cases
from tests.oracle_lib import Oracle

pytestmark = pytest.mark.gpu


def _capi():
    from espflix_b200 import capi
    return capi


def _synth_main(seed, n_pictures, gop, slices=12, flags=0, qscale=None):
    from espflix_b200 import synth
    kw = {} if qscale is None else {"qscale": qscale}
    es, off = synth.generate(synth.SEED0 + seed, n_pictures=n_pictures, gop=gop, slices=slices, flags=flags, **kw)
    return bytes(synth.wrap_ts(es, off))


def _seq_before_p(seed=77, n_pictures=40, gop=12, at=5):
    """a sequence header repeated at the start of P picture `at`'s PES: it does not start a segment"""
    from espflix_b200 import synth
    es, off = synth.generate(synth.SEED0 + seed, n_pictures=n_pictures, gop=gop)
    es = bytes(es)
    seq = es[:es.index(b"\x00\x00\x01\xb8")]
    pics = [es[off[k]:off[k + 1]] for k in range(n_pictures)]
    pics[at] = seq + pics[at]
    new = b"".join(pics)
    noff = np.cumsum([0] + [len(p) for p in pics]).astype(np.uint32)
    return bytes(synth.wrap_ts(np.frombuffer(new, np.uint8), noff))


def _cases():
    from espflix_b200 import synth
    return {
        "vmedia": trick_cases.fixture("vmedia"),
        "splash": trick_cases.fixture("splash"),
        "slices1": _synth_main(1, 31, 12, slices=1),
        "slices5": _synth_main(2, 46, 12, slices=5),
        "matrices": _synth_main(3, 30, 12, flags=synth.MATRICES),
        "biglevels": _synth_main(4, 16, 12, flags=synth.BIGLEVELS),
        "gop1": _synth_main(5, 17, 1),
        "gop13": _synth_main(6, 44, 13),
        "audio": restart_cases.program(210, 33, 90000, audio=dict(seed=21, frames=60)),
        "seq_before_p": _seq_before_p(),
    }


@pytest.fixture(scope="module")
def cases():
    return _cases()


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@pytest.mark.parametrize("qscale", [1, trick_cases.DEFAULT_QSCALE, 31])
def test_trick_build_equals_restatement(cases, oracle, qscale):
    names = list(cases)
    got = _capi().trick_build([cases[n] for n in names], qscale=qscale)       # every main in one call
    for n, (fwd, rwd) in zip(names, got):
        want_f, want_r, _ = trick_cases.restate(cases[n], oracle, qscale)
        assert fwd == want_f, "%s: fwd differs at byte %s" % (n, _first_diff(fwd, want_f))
        assert rwd == want_r, "%s: rwd differs at byte %s" % (n, _first_diff(rwd, want_r))


def test_trick_build_one_main_per_call(cases, oracle):
    for n in ("vmedia", "gop13", "seq_before_p"):
        (fwd, rwd), = _capi().trick_build([cases[n]])
        want_f, want_r, _ = trick_cases.restate(cases[n], oracle)
        assert fwd == want_f and rwd == want_r, n


def test_big_levels_use_16_bit_escapes(cases, oracle):
    frames, pts, codes = trick_cases.source(cases["biglevels"], oracle)
    levels = trick_cases.quantise(trick_cases.fdct(trick_cases.picture_blocks(frames[0])), 1)
    assert (np.abs(levels[..., 1:]) > 127).any()


def _raw(blob, off, qscale, fcap, rcap):
    capi = _capi()
    lib = capi.load_library()
    blob = np.ascontiguousarray(np.frombuffer(bytes(blob), np.uint8) if len(blob) else np.zeros(1, np.uint8))
    off = np.ascontiguousarray(off, dtype=np.uint64)
    n = off.size - 1
    fo, ro = np.zeros(n + 1, np.uint64), np.zeros(n + 1, np.uint64)
    fwd, rwd = np.full(max(fcap, 1), 0xAB, np.uint8), np.full(max(rcap, 1), 0xAB, np.uint8)
    rc = lib.ef_trick_build(0, blob.ctypes.data, off.ctypes.data, n, qscale, fwd.ctypes.data, fcap, fo.ctypes.data, rwd.ctypes.data, rcap, ro.ctypes.data)
    return rc, fo, ro, fwd, rwd


def test_enomem_sizing_contract(cases, oracle):
    capi = _capi()
    mains = [cases["splash"], cases["gop1"]]
    blob, off = capi.Context.pack(mains)
    want = [trick_cases.restate(m, oracle)[:2] for m in mains]
    need_f = sum(len(w[0]) for w in want)
    for fcap, rcap in ((0, 0), (need_f - 1, need_f), (need_f, need_f - 188)):
        rc, fo, ro, fwd, rwd = _raw(blob, off, trick_cases.DEFAULT_QSCALE, fcap, rcap)
        assert rc == capi.EF_ENOMEM
        assert list(fo) == [0, len(want[0][0]), need_f] and list(ro) == list(fo)
        assert (fwd == 0xAB).all() and (rwd == 0xAB).all()
    rc, fo, ro, fwd, rwd = _raw(blob, off, trick_cases.DEFAULT_QSCALE, need_f, need_f)
    assert rc == capi.EF_OK
    assert fwd.tobytes() == want[0][0] + want[1][0] and rwd.tobytes() == want[0][1] + want[1][1]


def test_einval(cases):
    capi = _capi()
    m = cases["splash"]
    blob, off = capi.Context.pack([m])
    for q in (0, 32, -1):
        assert _raw(blob, off, q, 1 << 20, 1 << 20)[0] == capi.EF_EINVAL
    assert _raw(blob[:len(m) - 4], np.array([0, len(m) - 4]), 8, 1 << 20, 1 << 20)[0] == capi.EF_EINVAL    # not a multiple of 188
    null = bytes([0x47, 0x1F, 0xFF, 0x10]) + b"\xff" * 184
    no_seq = capi.Context.pack([m, null * 4])
    assert _raw(no_seq[0], no_seq[1], 8, 1 << 20, 1 << 20)[0] == capi.EF_EINVAL                          # no sequence header
    empty = capi.Context.pack([m, b""])
    assert _raw(empty[0], empty[1], 8, 1 << 20, 1 << 20)[0] == capi.EF_EINVAL
    with pytest.raises(capi.EspflixError):
        capi.trick_build([m], qscale=40)


def test_stage_times_are_reported(cases):
    capi = _capi()
    capi.trick_build([cases["vmedia"]])
    ms = capi.trick_stage_ms()
    assert all(t > 0 for t in ms), ms


def _first_diff(a, b):
    n = min(len(a), len(b))
    d = np.nonzero(np.frombuffer(a[:n], np.uint8) != np.frombuffer(b[:n], np.uint8))[0]
    return int(d[0]) if d.size else ("length %d vs %d" % (len(a), len(b)))
