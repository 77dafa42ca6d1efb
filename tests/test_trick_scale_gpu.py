"""ef_trick_build past its first batch and on the encoder's rare codes (tests/trick_scale_cases.py): in every scenario each main's
fwd and rwd equal the restatement byte for byte, and the host plan restated in trick_scale_cases.plan() shows the scenario reached the
path it is named for."""
import numpy as np
import pytest

from tests import trick_cases as tc, trick_scale_cases as sc
from tests.oracle_lib import Oracle

pytestmark = pytest.mark.gpu


def _capi():
    from espflix_b200 import capi
    return capi


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def _first_diff(a, b):
    n = min(len(a), len(b))
    d = np.nonzero(np.frombuffer(a[:n], np.uint8) != np.frombuffer(b[:n], np.uint8))[0]
    return int(d[0]) if d.size else ("length %d vs %d" % (len(a), len(b)))


def _check(mains, oracle, qscale=tc.DEFAULT_QSCALE, want=None, got=None):
    got = got if got is not None else _capi().trick_build(mains, qscale=qscale)
    assert len(got) == len(mains)
    for k, (m, (fwd, rwd)) in enumerate(zip(mains, got)):
        wf, wr = want[k] if want is not None else tc.restate(m, oracle, qscale)[:2]
        assert fwd == wf, "main %d: fwd differs at byte %s" % (k, _first_diff(fwd, wf))
        assert rwd == wr, "main %d: rwd differs at byte %s" % (k, _first_diff(rwd, wr))
    return got


def test_many_segments(oracle):
    mains = sc.many_segments()
    sc.check_many_segments(sc.plan(mains, oracle))
    _check(mains, oracle)


def test_many_mains(oracle):
    mains = sc.many_mains()
    sc.check_many_mains(sc.plan(mains, oracle))
    _check(mains, oracle)


def test_padded_segments(oracle):
    small = sc.intra_main(sc.flat_run(40, 2))
    m = sc.padded_main()
    sc.check_padded(sc.plan([m], oracle))
    _check([m], oracle, want=[tc.restate(small, oracle)[:2]])          # null packets leave the restatement as it is


def test_context_grows_for_a_later_batch(oracle):
    mains = sc.multi_pes_mains()
    sc.check_multi_pes(sc.plan(mains, oracle))
    _check(mains, oracle)


@pytest.mark.parametrize("rec_pics", ["1", "3"])
def test_decode_in_pieces(oracle, monkeypatch, rec_pics):
    monkeypatch.setenv("EF_REC_PICS", rec_pics)
    mains = [tc.fixture("vmedia"), tc.fixture("splash")] + sc.multi_pes_mains() + sc.many_segments()
    p = sc.plan(mains, oracle, rec_pics=int(rec_pics))
    assert max(p["pieces"]) > 1
    _check(mains, oracle)


@pytest.mark.parametrize("qscale", [1, tc.DEFAULT_QSCALE, 31])
def test_adversarial(oracle, qscale):
    m = sc.adversarial_main()
    (fwd, rwd), = _check([m], oracle, qscale)
    frames, _, _ = tc.source(m, oracle)
    pics = sc.fwd_pictures(fwd)
    for k, j in enumerate(sc.ADV_PICTURES):
        assert np.array_equal(sc.parse_picture(pics[k]), sc.trick_levels(frames[j].tobytes(), qscale)), (qscale, j)
    if qscale == sc.RESIDUE_QSCALE:
        (fwd, _), = _check([sc.residue_main()], oracle, qscale)
        assert [(14 + len(p)) % 184 for p in sc.fwd_pictures(fwd)] == sorted(sc.RESIDUE_FRAMES)


@pytest.mark.parametrize("name", ["dropped_slice", "mid_row", "next_picture"])
def test_segment_cuts_keep_the_continuous_decode(oracle, name):
    _check([sc.cut_cases()[name]], oracle)


def test_long_main_of_multi_row_slices(oracle):
    """more pictures than one segment holds, in ffmpeg's slices: the main must be cut at its I pictures to build at all"""
    m = sc.long_main()
    sc.check_long(sc.plan([m], oracle))
    _check([m], oracle)


def test_batch_composition_changes_no_file(oracle):
    mains = [sc.adversarial_main(), sc.residue_main()] + list(sc.cut_cases().values()) + \
        [sc.intra_main(sc.flat_run(1 + j % 20, 40 + j)) for j in range(20)] + [tc.fixture("splash")]
    together = _capi().trick_build(mains)
    want = [tc.restate(m, oracle)[:2] for m in mains]
    _check(mains, oracle, want=want, got=together)
    _check(mains[::-1], oracle, want=want[::-1])
    for m, w in zip(mains, want):
        _check([m], oracle, want=[w])


def test_library_add_trick_adversarial_title(oracle):
    """the adversarial main as a title given its trick files on the device, against a twin added with the files trick_build returns"""
    import espflix_b200
    capi = _capi()
    m = sc.adversarial_main()
    (fwd, rwd), = _check([m], oracle)
    ctxs = []
    for k in range(2):
        ctx = espflix_b200.Context(n_streams=1, max_pictures=64, max_slices_per_picture=12, es_capacity=1 << 20, fields=False)
        ctx.enable_pts()
        ctxs.append(ctx)
    built, twin = ctxs
    assert built.library_add(capi.build_video_idx(m, b"", b""), m) == 0
    built.library_add_trick(0)
    assert twin.library_add(capi.build_video_idx(m, fwd, rwd), m, fwd, rwd) == 0
    assert built.library_read(0, -1) == twin.library_read(0, -1)
    assert built.library_read(0, 2) == fwd and built.library_read(0, 0) == rwd
    for ctx in ctxs:
        ctx.close()
