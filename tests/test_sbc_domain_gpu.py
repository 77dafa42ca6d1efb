"""The device's SBC decoder across its whole frame-header domain (tests/sbc_cases.py): every directed stream in one
ef_audio_decode batch against the oracle and the reference's pins (tests/golden/sbc_pins.json), the same streams through
the decoder context cut at seeded and at placed packets (ef_decode_audio and ef_decode_audio_async), and out-of-domain
bit pools and joint-stereo frames inside a 4,096-stream batch."""
import json
import os

import numpy as np
import pytest

import espflix_b200
from tests import audio_cases
from tests import sbc_cases as sc
from tests.carry_cases import cut
from tests.harness import submits
from tests.test_audio_async_gpu import _pair

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PINS = json.load(open(os.path.join(G, "sbc_pins.json")))


def _frame_size(es):
    """the frame size the probe learns: 8 + 2 * total of frame 0, -1 rejected, -2 outside the domain, 0 empty"""
    if not len(es):
        return 0
    a = sc._hdr_alloc(bytes(es))
    return -1 if a is None else a["total"] if a["total"] < 0 else 8 + 2 * a["total"]


def _check(oracle, name, es, r):
    want = oracle.sbc_decode(es)
    fs = _frame_size(es)
    assert r["frame_size"] == fs, name
    if isinstance(want, int):
        assert want == fs and r["n_frames"] == 0, name
        return
    assert r["n_frames"] == len(es) // fs and r["pcm"].size == want.size, name
    assert np.array_equal(r["pcm"], want), "%s: first diff at %s" % (name, np.nonzero(r["pcm"] != want)[0][:4])
    assert np.array_equal(r["pdm"], oracle.pdm(want)), name
    if name in PINS and not name.startswith("kind_m3_b8_"):
        assert sc.pin_of(r["pcm"], r["pdm"], sc.ref_undefined_frames(es)) == PINS[name], name


def test_every_directed_stream_in_one_batch(oracle):
    ss = sc.streams()
    names = list(ss)
    res = espflix_b200.audio_decode([ss[n] for n in names])
    for n, r in zip(names, res):
        _check(oracle, n, ss[n], r)
    assert sum(1 for n in names if n in PINS) == len(PINS)


def _ts(i, es):
    return audio_cases.mux_audio_ts(es, pid=0x101 if i % 2 else 0x102, pes_bytes=[61, 188, 333, 1024, 2000][i % 5])


@pytest.mark.parametrize("mode", ["async", "alternate"])
def test_directed_streams_cut_at_seeded_packets(oracle, mode):
    """every directed stream through two contexts, one calling ef_decode_audio, the other ef_decode_audio_async (or both
    alternately): each stream's TS cut at its own seeded packets over 5 submits; concatenated, equal to the whole call"""
    ss = sc.streams()
    names = list(ss)
    K = 5
    chunks = []
    for i, n in enumerate(names):
        t = _ts(i, ss[n])
        r = np.random.RandomState(7100 + i)
        chunks.append(cut(t, sorted(r.randint(0, t.size // 188 + 1, size=K - 1).tolist())))
    got = _pair(submits(chunks), mode=mode, es_capacity=1 << 24)
    whole = espflix_b200.audio_decode([ss[n] for n in names])
    for s, n in enumerate(names):
        assert sum(g[s]["n_frames"] for g in got) == whole[s]["n_frames"], n
        assert np.array_equal(np.concatenate([g[s]["pcm"] for g in got]).astype(np.int16), whole[s]["pcm"]), n
        assert np.array_equal(np.concatenate([g[s]["pdm"] for g in got]).astype(np.uint16), whole[s]["pdm"]), n
        _check(oracle, n, ss[n], whole[s])


def test_cuts_placed_on_purpose(oracle):
    """cuts inside a 264-byte frame (263 bytes held), just before and after a bit-pool-200 header, between an out-of-domain
    frame and the next, and inside frame 0 of a stream whose frame 0 is outside the domain. Each piece is muxed on its own,
    so the audio is cut exactly there; per call, the frames decoded are those the hold-back restatement predicts."""
    ss = sc.streams()
    names = sorted(sc.PLACED_CUTS)
    chunks, pieces = [], []
    for i, n in enumerate(names):
        es = ss[n]
        edges = [0] + sc.PLACED_CUTS[n] + [es.size]
        pieces.append(edges)
        chunks.append([_ts(i, es[a:b]) for a, b in zip(edges[:-1], edges[1:])])
    K = max(len(c) for c in chunks)
    chunks = [c + [np.zeros(0, dtype=np.uint8)] * (K - len(c)) for c in chunks]
    got = _pair(submits(chunks), mode="alternate", es_capacity=1 << 22)
    whole = espflix_b200.audio_decode([ss[n] for n in names])
    for s, n in enumerate(names):
        es, edges = ss[n], pieces[s]
        done = 0
        fs = max(_frame_size(es), 0)
        for k, g in enumerate(got):
            if k + 1 < len(edges) - 1:                     # before the last piece: the hold-back rule
                c = edges[k + 1]
                want = (c - sc.held(es, c)) // fs if fs else 0
                assert done + g[s]["n_frames"] == want, (n, k)
            done += g[s]["n_frames"]
        assert done == max(whole[s]["n_frames"], 0), n
        assert np.array_equal(np.concatenate([g[s]["pcm"] for g in got]).astype(np.int16), whole[s]["pcm"]), n
        _check(oracle, n, es, whole[s])
    assert any(sc.held(ss["max_snr_zero"], c) == 263 for c in sc.PLACED_CUTS["max_snr_zero"])


def test_out_of_domain_streams_in_a_full_batch(oracle):
    """one stream with a bit pool of 255 and one with a mode-3 / 16-block frame among 4,096: the call returns, both
    report -2 or re-synthesise as the oracle does, and every other stream equals its output in a batch without them"""
    ss = sc.streams()
    names = [n for n in ss if not n.startswith("kind_")]
    base = [ss[names[k % len(names)]] for k in range(4094)]
    bad = [ss["kind_bp255_first"], ss["kind_m3_b16_middle"]]
    batch = base[:1000] + [bad[0]] + base[1000:3000] + [bad[1]] + base[3000:]
    got = espflix_b200.audio_decode(batch)
    ref = espflix_b200.audio_decode(base)
    assert got[1000]["frame_size"] == -2 and got[1000]["n_frames"] == 0
    _check(oracle, "kind_m3_b16_middle", bad[1], got[3001])
    rest = got[:1000] + got[1001:3001] + got[3002:]
    for k, (a, b) in enumerate(zip(rest, ref)):
        assert a["frame_size"] == b["frame_size"] and a["n_frames"] == b["n_frames"], k
        assert np.array_equal(a["pcm"], b["pcm"]) and np.array_equal(a["pdm"], b["pdm"]), k
