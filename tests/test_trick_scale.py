"""The trick encoder's rare codes and ef_trick_build's host plan on the CPU (tests/trick_scale_cases.py): the adversarial main reaches
the clamp, the escape forms, the longest runs and the largest DC steps; an independent MPEG-1 reader gives back exactly the levels
of every restated picture; the quantiser meets its definition for every coefficient the FDCT can reach; the mux ends PES on every
awkward residue; every planned segment decodes from reset to the frames of a continuous decode; and every GPU scenario reaches the
path it is named for."""
import numpy as np
import pytest

from tests import pts_cases, trick_cases as tc, trick_scale_cases as sc
from tests.oracle_lib import Oracle

@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@pytest.fixture(scope="module")
def adversarial(oracle):
    m = sc.adversarial_main()
    frames, _, _ = tc.source(m, oracle)
    return m, frames


def _runs(levels):
    out = set()
    for b in levels.reshape(-1, 64):
        nz = np.nonzero(b[1:])[0] + 1
        out.update((nz - np.concatenate([[0], nz[:-1]]) - 1).tolist())
    return out


def _dc_steps(levels):
    """{(component 0 luma / 1 chroma, DC difference)} of a picture's levels [12, 22, 6, 64]"""
    out = set()
    for row in levels:
        pred = [128, 128, 128]
        for mb in row:
            for b in range(6):
                c = 0 if b < 4 else b - 3
                out.add((min(c, 1), int(mb[b, 0]) - pred[c]))
                pred[c] = int(mb[b, 0])
    return out


def test_adversarial_main_reaches_the_rare_codes(adversarial):
    _, frames = adversarial
    lv = [sc.trick_levels(frames[j].tobytes(), 1) for j in sc.ADV_PICTURES]
    ac = set().union(*(set(np.unique(x[..., 1:]).tolist()) for x in lv))
    assert {255, -255, 128, -128, 127, -127} <= ac
    zz1 = set().union(*(set(np.unique(x[..., 1]).tolist()) for x in lv))
    assert {40, 41, -40, -41} <= zz1                        # run 0: the last table level and the first escaped one
    assert {31, 32, 62} <= set().union(*(_runs(x) for x in lv))
    steps = set().union(*(_dc_steps(x) for x in lv))
    assert {(0, 255), (0, -255), (1, 255), (1, -255)} <= steps


@pytest.mark.parametrize("qscale", [1, tc.DEFAULT_QSCALE, 31])
def test_reader_gives_back_the_levels(oracle, adversarial, qscale):
    m, frames = adversarial
    fwd, rwd = tc.restate(m, oracle, qscale)[:2]
    pics = sc.fwd_pictures(fwd)
    assert len(pics) == len(sc.ADV_PICTURES) and sc.fwd_pictures(rwd) == pics[::-1]
    for k, j in enumerate(sc.ADV_PICTURES):
        assert np.array_equal(sc.parse_picture(pics[k]), sc.trick_levels(frames[j].tobytes(), qscale)), (qscale, j)
    largest = max(len(b) for p in pics for _, b in sc.slices(p)[1])
    assert largest < sc.SLICE_BYTES, largest
    if qscale == 1:
        assert largest > 12000                              # the noise picture: 12,966 bytes when written, of 29,440
        oracle.stats_reset()
        assert len(oracle.decode_ts(fwd, max_frames=8)) == len(sc.ADV_PICTURES)
        assert oracle.stats().escapes16 > 0


def test_reader_rejects_the_forbidden_escape():
    """-128 in the 8-bit escape form (0x80 is the 16-bit form's prefix) does not read back as -128"""
    es = tc.encode_picture(sc.flat(128), 1, tc.header_bytes(1, 3))
    head, sl = sc.slices(es)
    good = sc.parse_picture(es)
    assert (good[..., 1:] == 0).all()
    # first macroblock of slice 1, block 0: DC "100" (size 0), then escape run 0 level -128 in 8 bits, then end of block
    bits = "00001" + "0" + "1" + "1" + "100" + "000001" + "000000" + "10000000" + "10"
    rest = "".join(format(b, "08b") for b in sl[0][1][4:])[5 + 1 + 2 + 3 + 2:]
    allbits = bits + rest
    allbits += "0" * (-len(allbits) % 8)
    bad = head + bytes([0, 0, 1, 1]) + int(allbits, 2).to_bytes(len(allbits) // 8, "big") + b"".join(b for _, b in sl[1:])
    with pytest.raises(AssertionError, match="16-bit escape of a level that fits 8 bits"):
        sc.parse_picture(bad)


def test_quantiser_meets_its_definition_everywhere():
    """every F the FDCT can reach (DC 0..2,040, AC within FDCT_BOUNDS), every qscale and every matrix entry"""
    dc_max = int(tc.fdct(np.full((8, 8), 255))[0, 0])
    ac_max = (tc.FDCT_BOUNDS["col_acc"] + 32768) >> 16
    assert dc_max == 2040 and int(tc.fdct(np.zeros((8, 8), np.int64))[0, 0]) == 0
    F = np.arange(-ac_max, ac_max + 1, dtype=np.int64)
    blocks = np.repeat(F[:, None], 64, axis=1).reshape(-1, 8, 8)
    Q = tc.INTRA_Q[tc.ZIGZAG][1:]
    A = 16 * np.abs(F)[:, None]
    for q in range(1, 32):
        lv = tc.quantise(blocks, q)[:, 1:]
        a = np.abs(lv)
        qQ = q * Q[None, :]
        clamped = a == 255
        assert ((2 * a - 1) * qQ <= A)[~clamped & (a > 0)].all() and (A < (2 * a + 1) * qQ)[~clamped].all()
        assert ((A >= 509 * qQ) == clamped).all()                         # round(8 |F| / qQ) >= 255
        assert (np.sign(lv) == np.where(a > 0, np.sign(F)[:, None], 0)).all()
    dc = np.arange(0, dc_max + 1, dtype=np.int64)
    b = np.zeros((dc.size, 8, 8), np.int64)
    b[:, 0, 0] = dc
    got = tc.quantise(b, 1)[:, 0]
    assert np.array_equal(got, np.minimum(np.floor(dc / 8 + 0.5).astype(np.int64), 255))


def test_mux_ends_pes_on_every_residue(oracle):
    fwd, _ = tc.restate(sc.residue_main(), oracle, sc.RESIDUE_QSCALE)[:2]
    pics = sc.fwd_pictures(fwd)
    assert [(14 + len(p)) % 184 for p in pics] == sorted(sc.RESIDUE_FRAMES)
    assert sc.residue_search(182) == sc.RESIDUE_FRAMES[182]
    starts = [k for k in range(len(fwd) // 188) if fwd[k * 188 + 1] & 0x40] + [len(fwd) // 188]
    last = [fwd[(s - 1) * 188:s * 188] for s in starts[1:]]
    assert [p[3] & 0x30 for p in last] == [0x10, 0x30, 0x30, 0x30]          # residue 0: no adaptation field
    assert [p[4] for p in last[1:]] == [182, 1, 0]                           # residue 1: 182 stuffing; 182: flags only; 183: length only
    assert last[2][5] == 0
    assert pts_cases.picture_pts(fwd) == tc.select(pts_cases.picture_pts(sc.residue_main()))[1]


@pytest.mark.parametrize("name", ["dropped_slice", "mid_row", "next_picture", "vmedia", "splash"])
def test_segments_decode_as_the_continuous_decode(oracle, name):
    """the planned segments, each decoded from reset, give the continuous decode's frames; the fixtures (ffmpeg's slices, each
    across several rows) are still cut at their I pictures; in the cut cases a cut before main picture 14 or 15 (which a rule
    that looks at one picture would make) does not"""
    m = tc.fixture(name) if name in ("vmedia", "splash") else sc.cut_cases()[name]
    p = sc.plan([m], oracle)
    full = oracle.decode_ts(m, max_frames=128)
    k = 0
    for _, a, b, n in p["segs"]:
        d = oracle.decode_ts(m[a * 188:b * 188], max_frames=128)
        assert len(d) == n and all(np.array_equal(d[i], full[k + i]) for i in range(n)), (name, a)
        k += n
    assert k == len(full)
    if name in ("vmedia", "splash"):
        assert len(p["segs"]) >= 6 and max(n for _, _, _, n in p["segs"]) <= 12
        return
    assert k == 20
    starts = [s for s in range(len(m) // 188) if m[s * 188 + 1] & 0x40] + [len(m) // 188]
    cuts = {a for _, a, _, _ in p["segs"]}
    assert starts[14] not in cuts and starts[15] not in cuts and starts[16] in cuts and starts[13] in cuts
    for s in (14, 15):
        d = oracle.decode_ts(m[starts[s] * 188:starts[16] * 188], max_frames=8)
        assert not np.array_equal(d[15 - s], full[15]), (name, s)


def test_every_other_main_cuts_at_every_picture(oracle):
    for m in (sc.adversarial_main(), sc.residue_main(), sc.many_segments()[0]):
        p = sc.plan([m], oracle)
        assert all(n == 1 for _, _, _, n in p["segs"]) and len(p["segs"]) == len(pts_cases.picture_pts(m))


def test_null_padding_keeps_the_restatement(oracle):
    m = sc.intra_main([(11 * k) % 256 for k in range(31)])
    padded = sc.pad(sc.pad(m, 20, 3000), 4, 500)
    assert tc.restate(padded, oracle)[:2] == tc.restate(m, oracle)[:2]


# -- the scenarios of tests/test_trick_scale_gpu.py reach their paths ------------------------------------------------------------
def test_scenarios_reach_their_paths(oracle):
    sc.check_many_segments(sc.plan(sc.many_segments(), oracle))
    sc.check_many_mains(sc.plan(sc.many_mains(), oracle))
    sc.check_padded(sc.plan([sc.padded_main()], oracle))
    p = sc.plan(sc.multi_pes_mains(), oracle, rec_pics=3)
    sc.check_multi_pes(p)
    assert max(p["pieces"]) > 1
    for rec in (1, 3):
        assert max(sc.plan([tc.fixture("vmedia"), tc.fixture("splash")], oracle, rec_pics=rec)["pieces"]) > 1
