"""Synthetic stream cases shared by the CPU and GPU parity tests (SURVEY.md 8d), and the random frames of the video and
presentation cases the C restatement and the unmodified reference are compared on (tests/golden/ref_pins.json)."""
import numpy as np

from espflix_b200 import synth

# (name, kwargs) — the coverage set adds what the reference's own fixtures lack (SURVEY.md §4)
COVERAGE = [
    ("bench12", dict(n_pictures=12, slices=12)),
    ("slices5", dict(n_pictures=12, slices=5)),
    ("slices1", dict(n_pictures=12, slices=1)),
    ("mbquant", dict(n_pictures=12, flags=synth.MBQUANT)),
    ("fullpel", dict(n_pictures=12, flags=synth.FULLPEL)),
    ("fcode3", dict(n_pictures=12, flags=synth.FCODE3)),
    ("biglevels", dict(n_pictures=6, gop=6, flags=synth.BIGLEVELS)),
    ("matrices", dict(n_pictures=12, flags=synth.MATRICES)),
    ("intra_in_p", dict(n_pictures=12, slices=5, flags=synth.INTRA_IN_P)),
    ("static", dict(n_pictures=12, flags=synth.STATIC, noise=0)),
    ("mixed_two_gops", dict(n_pictures=24, qscale=4, flags=synth.MBQUANT | synth.MATRICES | synth.INTRA_IN_P)),
    ("smooth_q6", dict(n_pictures=12, noise=0)),
]


def make(idx, kw):
    return synth.generate(synth.SEED0 + 1000 + idx, **kw)


def coverage_stream(idx):
    """(elementary stream, transport stream) of coverage case `idx`"""
    es, off = make(idx, COVERAGE[idx][1])
    return es, synth.wrap_ts(es, off)


def video_cases():
    """(key, call): composite fields and blits of random frames; `call` takes the oracle or the reference alike."""
    rng = np.random.default_rng(7)
    for ntsc in (1, 0):
        for fc in (0, 1, 2):
            fr = rng.integers(0, 249, 101376, dtype=np.uint8)
            yield "field/%d/%d" % (ntsc, fc), lambda v, fr=fr, ntsc=ntsc, fc=fc: v.field(fr, ntsc, fc)
        fr = rng.integers(0, 256, 101376, dtype=np.uint8)          # bytes above 248: dither carries cross bytes
        yield "field/%d/1/carry" % ntsc, lambda v, fr=fr, ntsc=ntsc: v.field(fr, ntsc, 1)
        for line, x, w in ((0, 0, 352), (191, 0, 352), (77, 16, 64), (100, 8, 344)):
            yield "blit/%d/%d/%d/%d" % (ntsc, line, x, w), lambda v, fr=fr, ntsc=ntsc, line=line, x=x, w=w: v.blit(fr, ntsc, line, x, w, 1)


PRESENTATION_CASES = [(0, 0, 0), (8, 0, 0), (-8, 0, 0), (176, 0, 0), (-344, 0, 0), (344, -1, 100), (0, 32, 0), (0, 5, 239), (0, 31, 17), (24, 1, 300)]


def presentation_cases():
    """(key, call): _hscroll two-frame scroll and the composite() overlay / progress bar / fade, both standards."""
    rng = np.random.default_rng(11)
    a, b = rng.integers(0, 249, 101376, dtype=np.uint8), rng.integers(0, 249, 101376, dtype=np.uint8)
    bm = rng.integers(0, 256, 1280, dtype=np.uint8)
    for ntsc in (1, 0):
        for hs, blend, prog in PRESENTATION_CASES:
            yield "%d/%d/%d/%d" % (ntsc, hs, blend, prog), lambda v, ntsc=ntsc, hs=hs, blend=blend, prog=prog: v.field_ex(a, b, ntsc, 1, hs, bm, blend, prog)

# Outside the reference's defined domain (its clamp table is indexed out of bounds when a sample
# leaves [-256,511], which any coefficient saturated at +-2048 causes): the CUDA path is compared
# with the oracle restatement only, which clamps every integer to [0,248].
UNPINNED = [
    ("overdrive", dict(n_pictures=6, gop=6, flags=synth.BIGLEVELS | synth.OVERDRIVE)),
]
