"""The SBC encoder and the audio mux restated (tests/sbc_encode_cases.py), checked without a GPU: the CRC on the fixtures, the analysis
tables, the frame length, the decoded level and SNR, the pins of the unmodified reference decoder, and the interleave."""
import hashlib
import json
import math
import os

import numpy as np
import pytest

from tests import pts_cases
from tests import sbc_cases as sc
from tests import sbc_encode_cases as se
from tests import trick_cases as tc

DELAY = 73                 # the analysis + synthesis filterbank delay in samples, measured below once for every case
SKIP = 2 * 128             # the reference decodes frame 0 twice (decode_audio(), video.cpp:966-973)
PINS = os.path.join(se.ROOT, "tests", "golden", "sbc_encode_pins.json")


def _stripped(ts):
    return b"".join(ts[k:k + 188] for k in range(0, len(ts), 188) if (((ts[k + 1] << 8) | ts[k + 2]) & 0x1FFF) not in (0x101, 0x102))


@pytest.mark.parametrize("name", ["splash", "vmedia"])
def test_crc_reproduces_every_fixture_frame(oracle, name):
    es = bytes(oracle.demux_audio_ts(np.frombuffer(tc.fixture(name), np.uint8)))
    fb = 8 + 2 * es[2]
    frames = [es[k:k + fb] for k in range(0, len(es) - fb + 1, fb)]
    assert len(frames) * fb == len(es) and len(frames) in (1240, 750)
    assert all(se.crc8(f[1:3] + f[4:8]) == f[3] for f in frames)


def test_analysis_tables():
    from tools import gen_sbc_tables as g
    for k in range(8):
        for i in range(16):
            assert se.MATRIX[k][i] == round(32768 * math.cos((k + 0.5) * (i - 4) * math.pi / 8))
            # the synthesis matrix's closed form at the same angle: cos((i' + 4)(k + 1/2) pi / 8), i' = i - 8 (a half turn apart below 8)
            c = math.cos(((i - 8) % 16 + 4) * (k + 0.5) * math.pi / 8)
            assert abs(se.MATRIX[k][i] / 32768 - (c if i >= 8 else -c)) < 1e-4
    assert list(se.WINDOW) == [-v for row in g.WINDOW for v in row]
    # the synthesis tables the decoder uses are the same constants
    src = open(os.path.join(se.ROOT, "espflix_b200", "csrc", "ef_sbc_tables.h")).read()
    body = src.split("ef_sbc_window[10][8] = {")[1].split("};")[0]
    assert [int(v) for v in body.replace("{", " ").replace("}", " ").replace(",", " ").split()] == [-v for v in se.WINDOW]


def _all_cases(oracle):
    out = {}
    for name, x in se.pcm_cases().items():
        for bp in (28, 128):
            out["%s_bp%d" % (name, bp)] = (x, dict(bitpool=bp))
    for f, a, b in se.sweep():
        out["sweep_f%d_a%d_bp%d" % (f, a, b)] = (se.sweep_pcm(f), dict(frequency=f, allocation=a, bitpool=b))
    for name, (fq, bp) in (("splash", (3, 28)), ("vmedia", (1, 20))):
        out["fixture_" + name] = (se.fixture_pcm(name, oracle)[0], dict(frequency=fq, bitpool=bp))
    return out


@pytest.fixture(scope="module")
def cases(oracle):
    return _all_cases(oracle)


def test_frame_length_and_no_wrap(cases):
    wraps_clamped = 0
    for name, (x, p) in cases.items():
        p = dict(se.DEFAULTS, **p)
        info = []
        s = se.encode(x, p["frequency"], p["allocation"], p["bitpool"], info=info)
        assert len(s) == se.n_frames(len(x)) * se.frame_bytes(p["bitpool"]), name
        for sf, a, q in info:
            assert a["total"] == p["bitpool"], (name, sf)
            for sb in range(8):
                L = a["bits"][sb]
                if L:
                    assert q[:, sb].min() >= 0 and q[:, sb].max() <= (1 << L) - 2
                    assert not any(sc.iquant_wraps(int(r), L, sf[sb]) for r in q[:, sb]), (name, sb)
                    wraps_clamped += L == 16 and sf[sb] == 15
    assert wraps_clamped, "no case reaches L = 16 at s = 15"


def test_square_and_clipped_reach_the_clamp():
    for name in ("square", "clipped"):
        info = []
        se.encode(se.pcm_cases()[name], bitpool=128, info=info)
        assert any(a["bits"][sb] == 16 and sf[sb] == 15 for sf, a, q in info for sb in range(8)), name


def _level(x, y):
    """(gain in dB, SNR in dB) of the decoded y against x, aligned by DELAY, frames 0 and 1 skipped"""
    n = min(len(x) - SKIP, len(y) - SKIP - DELAY)
    xx = x[SKIP:SKIP + n].astype(np.float64)
    yy = y[SKIP + DELAY:SKIP + DELAY + n].astype(np.float64)
    g = np.dot(yy, xx) / np.dot(xx, xx)
    return 20 * np.log10(g), 10 * np.log10(np.dot(xx, xx) / np.sum((yy - xx) ** 2))


def test_delay_is_the_same_for_every_signal(oracle):
    rng = np.random.default_rng(73)
    for fq in range(4):
        x = rng.normal(0, 3000, 20000).astype(np.int16)
        y = oracle.sbc_decode(np.frombuffer(se.encode(x, fq, 0, 128), np.uint8))
        corr = [np.dot(y[SKIP + d:SKIP + d + 15000].astype(float), x[SKIP:SKIP + 15000].astype(float)) for d in range(200)]
        assert int(np.argmax(corr)) == DELAY


@pytest.mark.parametrize("fq", range(4))
def test_passband_gain(oracle, fq):
    fs = se.FS_HZ[fq]
    for f0 in (fs / 64, fs / 16, fs * 3 / 16, fs * 5 / 16, fs * 7 / 16):
        x = se.sine(fs // 2, f0, fs, 8000)
        y = oracle.sbc_decode(np.frombuffer(se.encode(x, fq, 0, 128), np.uint8))
        gain, _ = _level(x, y)
        assert abs(gain) <= 0.1, (fq, f0, gain)


def test_snr_at_the_defaults(oracle):
    """a -6 dBFS 1 kHz sine at 48 kHz, bit pool 28, loudness: 64.4 dB"""
    x = se.sine(48000, 1000, 48000, 16384)
    _, snr = _level(x, oracle.sbc_decode(np.frombuffer(se.encode(x), np.uint8)))
    assert snr >= 40, snr


def test_splash_reencode_snr(oracle):
    """splash's own decoded audio, encoded again at its header (48 kHz, bit pool 28): 49.1 dB against it (vmedia's at 32 kHz, bit
    pool 20: 25.1 dB)"""
    x, _ = se.fixture_pcm("splash", oracle)
    _, snr = _level(x, oracle.sbc_decode(np.frombuffer(se.encode(x), np.uint8)))
    assert snr >= 45, snr


def _pin(pcm):
    return hashlib.sha256(np.ascontiguousarray(pcm, dtype=np.int16).tobytes()).hexdigest()[:32]


def ref_defined(n_bytes, bitpool):
    """whether the reference's TS path defines the PCM of an SBC stream: frames of at most the 64 bytes decode_audio() probes the
    frame size on (video.cpp:966-973), and none straddling the end of its 4 KB ring (video.cpp:957)"""
    fb = se.frame_bytes(bitpool)
    return fb <= 64 and (4096 % fb == 0 or n_bytes + 264 <= 4096)


ES_LIMIT = 4096 - 264       # the most SBC bytes the reference's ring takes in one push_audio() without wrapping


def es_frames(n_bytes, bitpool):
    """frames of a stream handed whole to the reference's push_audio() -> decode_audio() -> sbc_decoder() chain where its TS path
    leaves the PCM undefined: the whole frames that fit ES_LIMIT (the decoder is causal, so they pin a prefix of the stream)"""
    fb = se.frame_bytes(bitpool)
    return min(n_bytes // fb, ES_LIMIT // fb)


def test_decode_equals_reference_pins(oracle, cases):
    """the oracle's decode of every restated stream equals the reference's: of the whole stream through its TS path where that is
    defined, else of the stream's first es_frames() frames handed to its decoder directly"""
    pins = json.load(open(PINS))
    assert set(pins) == set(cases) | {"title_with_audio"}
    for name, (x, p) in cases.items():
        p = dict(se.DEFAULTS, **p)
        s = se.encode(x, p["frequency"], p["allocation"], p["bitpool"])
        assert hashlib.sha256(s).hexdigest()[:32] == pins[name]["sbc"], name
        if not s:
            continue
        if ref_defined(len(s), p["bitpool"]):
            assert _pin(oracle.sbc_decode(np.frombuffer(s, np.uint8))) == pins[name]["pcm"], name
        else:
            k = es_frames(len(s), p["bitpool"])
            assert pins[name]["es_frames"] == k > 0, name
            part = s[:k * se.frame_bytes(p["bitpool"])]
            assert _pin(oracle.sbc_decode(np.frombuffer(part, np.uint8))) == pins[name]["pcm_es"], name


def cli_title(oracle):
    """the pictures and 48 kHz PCM of the title ef_indexer_cli --encode ... --audio is checked on"""
    pics = ec_module().translated(2, 24, (2, -1))
    pcm = se.sine(48000 * 2 + 333, 523, 48000, 9000)
    return pics, pcm


def ec_module():
    from tests import encode_cases
    return encode_cases


def cli_title_ts(oracle):
    """its video.ts with audio, restated"""
    pics, pcm = cli_title(oracle)
    return se.mux(ec_module().encode_title(pics, oracle)[0], se.encode(pcm))


def test_title_with_audio_plays_as_the_reference_plays_it(oracle):
    """the reference's TS path plays the restated title with audio (what ef_indexer_cli --encode --audio writes) with the sound the
    oracle decodes from it, and its pictures are the video-only title's"""
    pins = json.load(open(PINS))
    ts = cli_title_ts(oracle)
    assert hashlib.sha256(ts).hexdigest()[:32] == pins["title_with_audio"]["ts"]
    es = oracle.demux_audio_ts(np.frombuffer(ts, np.uint8))
    assert bytes(es) == se.encode(cli_title(oracle)[1])
    assert _pin(oracle.sbc_decode(es)) == pins["title_with_audio"]["pcm"]
    pics, _ = cli_title(oracle)
    assert np.array_equal(oracle.decode_ts(ts, max_frames=40), ec_module().encode_title(pics, oracle)[2])


# ---- mux ---------------------------------------------------------------------------------------------------------------------------------
def _check_mux(video, sbc, oracle, **params):
    p = dict(se.DEFAULTS, **params)
    out = se.mux(video, sbc, **p)
    pk = [out[k:k + 188] for k in range(0, len(out), 188)]
    pid = [((d[1] << 8) | d[2]) & 0x1FFF for d in pk]
    assert b"".join(d for d, q in zip(pk, pid) if q != 0x102) == video
    assert bytes(oracle.demux_audio_ts(np.frombuffer(out, np.uint8))) == sbc
    assert pts_cases.picture_pts(out) == pts_cases.picture_pts(video)
    # every audio PES sits in (v_{j-1}, v_j] of the video PES start after it
    starts = se.video_starts(video)
    fpp = se.frames_per_pes(p["bitpool"], p["frames_per_pes"])
    k, vids_seen = 0, 0
    for d, q in zip(pk, pid):
        if q == 0x102 and d[1] & 0x40:
            a = se.audio_pts(k, p["frequency"], fpp, p["pts0"])
            if vids_seen < len(starts):
                assert starts[vids_seen][1] >= a
            if vids_seen:
                assert starts[vids_seen - 1][1] < a
            k += 1
        elif q == 0x100 and d[1] & 0x40 and d[3] & 0x10:               # a video PES start as se.video_starts() counts them
            vids_seen += 1
    assert k == len(se.audio_pes(sbc, **p))
    return out


@pytest.mark.parametrize("name", ["splash", "vmedia"])
def test_mux_on_stripped_fixtures(oracle, name):
    video = _stripped(tc.fixture(name))
    pcm = np.random.default_rng(1).integers(-9000, 9000, 48000 * 4).astype(np.int16)
    sbc = se.encode(pcm)
    out = _check_mux(video, sbc, oracle)
    assert se.audio_pes(sbc)[1][0] == 1920 and len(se.audio_pes(sbc)[0][1]) == 14 + 512
    assert _check_mux(video, b"", oracle) == video


def test_mux_on_encoded_and_trick_files(oracle):
    from tests import encode_cases as ec
    ts = ec.encode_title(ec.translated(2, 14, (2, -1)), oracle)[0]
    fwd, rwd, _ = tc.restate(ts, oracle)
    sbc = se.encode(se.sine(48000, 440, 48000, 5000))
    for v in (ts, fwd, rwd):
        _check_mux(v, sbc, oracle)
        _check_mux(v, sbc, oracle, frames_per_pes=1, pts0=3000)
        _check_mux(v, sbc[:64 * 11], oracle, frames_per_pes=3)


def test_mux_keeps_other_pids_in_place(oracle):
    from tests import encode_cases as ec
    ts = ec.encode_title(ec.translated(2, 6, (2, -1)), oracle)[0]
    pat = bytes([0x47, 0x40, 0x00, 0x10]) + b"\xff" * 184
    other = bytes([0x47, 0x00, 0x30, 0x10]) + b"\x55" * 184
    pk = [ts[k:k + 188] for k in range(0, len(ts), 188)]
    video = pat + b"".join(p + (other if i % 3 == 0 else b"") for i, p in enumerate(pk))
    sbc = se.encode(se.sine(20000, 700, 48000, 5000))
    out = _check_mux(video, sbc, oracle)
    assert out[:188] == pat


def test_mux_rejects():
    sbc = se.encode(np.zeros(1280, np.int16))
    video = _stripped(tc.fixture("splash"))
    with pytest.raises(ValueError):
        se.mux(tc.fixture("splash"), sbc)
    with pytest.raises(ValueError):
        se.mux(video, sbc, pts0=(1 << 33) - 1)
    with pytest.raises(ValueError):
        se.mux(video[:-1], sbc)
    with pytest.raises(ValueError):
        se.mux(video, sbc[:-1])
