"""The encoded-title rule (tests/encode_cases.py) on the CPU: the restated video.ts decodes, through the oracle, to exactly the
reconstructions the rule predicted from, stays inside the reference's defined clamp domain, keeps its syntax and placement rules,
and its motion search finds the motion that is there."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import encode_cases as ec
from tests import pts_cases
from tests import trick_cases as tc
from tests.oracle_lib import Oracle, have_ref, ref_decode_ts


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def _cases(oracle):
    return {
        "static": (ec.translated(1, 6, (0, 0), grain=0.0), {}),
        "integer": (ec.translated(2, 6, (4, -2)), {}),
        "half": (ec.translated(3, 6, (1, 3)), {}),
        "cut": (ec.scene_cut(4, 6, 3), {}),
        "edge": (ec.translated(5, 4, (14, -14)), {}),
        "noise_q1": (ec.noise(7, 3), dict(qscale_i=1, qscale_p=1)),
        "noise_q31": (ec.noise(7, 3), dict(qscale_i=31, qscale_p=31)),
        "checker_q1": (ec.checkerboard(3, cell=1), dict(qscale_i=1, qscale_p=1)),
        "checker_q31": (ec.checkerboard(3, cell=8, phase=1), dict(qscale_i=31, qscale_p=31)),
        "vmedia_q1": (ec.fixture_pictures("vmedia", oracle)[:14], dict(qscale_i=1, qscale_p=1)),
        "splash_q31": (ec.fixture_pictures("splash", oracle)[:14], dict(qscale_i=31, qscale_p=31, gop=5)),
    }


@pytest.mark.parametrize("name", ["static", "integer", "half", "cut", "edge", "noise_q1", "noise_q31", "checker_q1", "checker_q31",
                                  "vmedia_q1", "splash_q31"])
def test_restatement_decodes_to_its_reconstructions(oracle, name):
    pics, params = _cases(oracle)[name]
    oracle.stats_reset()
    ts, es, rec, infos = ec.encode_title(pics, oracle, **params)
    assert oracle.stats().pin_out_of_domain == 0
    frames = oracle.decode_ts(ts, max_frames=len(pics) + 1)
    assert len(frames) == len(pics) and np.array_equal(frames, rec)
    p = dict(ec.DEFAULT_PARAMS, **params)
    assert pts_cases.picture_pts(ts) == [p["pts0"] + k * p["pts_step"] for k in range(len(pics))]
    es_all, _ = pts_cases.demux(ts)
    assert es_all == b"".join(es)
    assert es_all.count(b"\x00\x00\x01\xb3") == (len(pics) + p["gop"] - 1) // p["gop"]
    for k, e in enumerate(es):                                  # every GOP opens with a sequence header, P pictures with their header
        if k % p["gop"] == 0:
            assert e.startswith(tc.header_bytes(p["aspect"], p["rate"]))
        else:
            assert e[:4] == b"\x00\x00\x01\x00" and len(e) > ec.P_HEADER_BYTES
            assert ((e[4] << 2) | (e[5] >> 6)) == k % p["gop"] and (e[5] >> 3) & 7 == 2


@pytest.mark.parametrize("name", ["integer", "half", "cut", "edge", "noise_q1", "checker_q31"])
def test_vectors_and_skips_are_legal(oracle, name):
    pics, params = _cases(oracle)[name]
    infos = ec.encode_title(pics, oracle, **params)[3]
    for info in infos:
        if info is None:
            continue
        h, v = info["h"], info["v"]
        assert ec.legal(ec._MX, ec._MY, h, v).all()
        sk = info["skipped"].reshape(12, 22)
        assert not sk[:, 0].any() and not sk[:, -1].any()
        assert not (sk.ravel() & ((h != 0) | (v != 0) | info["intra"] | (info["cbp"] != 0))).any()


def _interior(info, key):
    return info[key].reshape(12, 22)[2:-2, 2:-2]


@pytest.mark.parametrize("step", [(4, -2), (-6, 2), (14, 0), (0, -8)])
def test_search_finds_whole_pixel_translations(oracle, step):
    """picture k is picture k - 1 moved by `step` half-pels (whole pixels): every interior macroblock predicts it with -step"""
    pics = ec.translated(20 + step[0], 4, step, grain=0.0)
    for info in ec.encode_title(pics, oracle)[3][1:]:
        assert (_interior(info, "h") == -step[0]).all() and (_interior(info, "v") == -step[1]).all()
        assert not _interior(info, "intra").any()


@pytest.mark.parametrize("step", [(1, 1), (-1, 1), (1, 0), (0, -1), (-1, -1)])
def test_search_finds_half_pel_translations(oracle, step):
    """picture k is the decoder's half-pel prediction of picture k - 1's source at `step`: every interior macroblock gets step"""
    pics = ec.halfpel_chain(20, 4, step)
    for info in ec.encode_title(pics, oracle)[3][1:]:
        assert (_interior(info, "h") == step[0]).all() and (_interior(info, "v") == step[1]).all()
        assert not _interior(info, "intra").any()


def test_static_clip_skips(oracle):
    pics = ec.translated(1, 6, (0, 0), grain=0.0)
    infos = ec.encode_title(pics, oracle)[3]
    for info in infos[1:]:
        assert _interior(info, "skipped").all() and info["skipped"].reshape(12, 22)[:, 1:-1].all()


def test_scene_cut_turns_intra(oracle):
    infos = ec.encode_title(ec.scene_cut(4, 6, 3), oracle)[3]
    assert not any(info["intra"].any() for info in infos[1:3])
    assert _interior(infos[3], "intra").all()
    assert not infos[4]["intra"].any()


@pytest.mark.parametrize("gop", [1, 5, 12])
def test_index_and_trick_plan_see_every_gop(oracle, gop):
    """make_index's table holds one sequence header per GOP, each at a video PES start; the trick build's segment plan cuts at every
    one, since every picture writes every macroblock"""
    from tests import trick_scale_cases
    pics = ec.translated(2, 26, (2, -1))
    ts, es, _, _ = ec.encode_title(pics, oracle, gop=gop)
    n_gops = (len(pics) + gop - 1) // gop
    pos = [int(p) for p in oracle.make_index(ts)["seq_pos"]]
    pes_start = np.cumsum([0] + [(14 + len(e) + 183) // 184 for e in es])[:-1]
    assert pos == [int(pes_start[k]) for k in range(0, len(pics), gop)]
    pk = np.frombuffer(ts, np.uint8).reshape(-1, 188)
    assert all(int(pk[p, 1]) & 0x40 and (((int(pk[p, 1]) & 0x1F) << 8) | int(pk[p, 2])) == 0x100 for p in pos)
    segs = trick_scale_cases.plan([ts], oracle)["segs"]
    assert [(a, n) for _, a, _, n in segs] == [(pos[g], min(gop, len(pics) - g * gop)) for g in range(n_gops)]


_PINS = json.load(open(os.path.join(tc.ROOT, "tests", "golden", "encode_pins.json")))


@pytest.fixture(scope="module")
def pin_cases(oracle):
    return {name: (pics, params) for name, pics, params in ec.pin_cases(oracle)}


@pytest.mark.parametrize("name", sorted(_PINS))
def test_restatement_equals_pins(oracle, pin_cases, name):
    """the restated file, its picture sizes and quality are pinned (tools/make_encode_golden.py), and the oracle decodes it to the
    frames the unmodified reference decoder gave for it"""
    pin = _PINS[name]
    pics, params = pin_cases[name]
    oracle.stats_reset()
    ts, es, rec, _ = ec.encode_title(pics, oracle, **params)
    assert oracle.stats().pin_out_of_domain == 0
    assert hashlib.sha256(ts).hexdigest() == pin["ts_sha256"]
    assert [len(e) for e in es] == pin["picture_bytes"]
    psnr = [min(tc.psnr(a, b), 99.0) for a, b in zip(pics, rec)]
    assert round(min(psnr), 2) == pin["min_psnr_db"] and round(float(np.mean(psnr)), 2) == pin["mean_psnr_db"]
    assert hashlib.sha256(oracle.decode_ts(ts, max_frames=len(pics) + 1).tobytes()).hexdigest() == pin["ref_decode_sha256"]


def test_pinned_defaults_keep_35_db():
    """the default quantisers are the largest of 8 and 16 that keep every picture of both fixtures at or above 35 dB"""
    q = ec.DEFAULT_PARAMS["qscale_p"]
    assert q == ec.DEFAULT_PARAMS["qscale_i"] == 8
    assert min(_PINS["vmedia/q%d" % q]["min_psnr_db"], _PINS["splash/q%d" % q]["min_psnr_db"]) >= 35.0


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref (the unmodified reference) is not built")
@pytest.mark.parametrize("name", ["vmedia/q1", "halfpel", "cut", "noise/q1", "checker/q31"])
def test_reference_decodes_restatement(oracle, pin_cases, name):
    pics, params = pin_cases[name]
    ts, _, rec, _ = ec.encode_title(pics, oracle, **params)
    _, frames = ref_decode_ts(ts)
    assert np.array_equal(frames, rec)
