"""The restatement against what the UNMODIFIED reference computed on the syntax-level streams of tests/syntax_cases.py
(pinned as SHA-256 by tools/make_syntax_pins.py in tests/golden/syntax_pins.json), and proof that those streams reach the
syntax the motion-search generator never writes."""
import functools
import json
import os
from collections import Counter

import numpy as np
import pytest

from tests import syntax_cases as sc
from tests.harness import sha

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "syntax_pins.json")))
PINNED = [n for n in sc.case_names() if n not in sc.UNPINNED]

# what each directed case exists for: its census has to show it
DIRECTED_FEATURE = {
    "stuffing_after_escape": ("stuffing_after_escape_slice_start", "stuffing_after_escape_mid_slice"),
    "intra_abort": ("abort_intra",),
    "skip_run_across_rows": ("skip_run_gt33_across_rows",),
    "qscale0": ("qscale_0",),
    "matrices_1_255": ("matrix_entry_1", "matrix_entry_255"),
    "fcode7": ("f_code_7",),
    "vector_wrap": ("vector_wrap",),
    "pic_320x176": ("mb_width_lt22", "mb_height_lt12", "slice_rows_past_picture"),
    "pic_176x96": ("mb_width_lt22", "mb_height_lt12", "slice_rows_past_picture"),
    "slices_mid_row": ("slice_ends_mid_row", "rows_without_slice", "pictures_without_slices"),
    "type3_p_grammar": ("picture_type_3", "picture_type_4"),
    "q7_dc_bleed": ("q7_dc_outside_0_255",),
    "mb_384_entries": ("mb_entries_384",),
}

# every item the syntax set has to reach, over the PINNED cases (so that each is held to the reference)
FEATURES = [
    "stuffing", "stuffing_after_escape_slice_start", "stuffing_after_escape_mid_slice", "address_escape",
    "q6_first_increment", "skip_run_across_rows", "skip_run_gt33_across_rows", "i_picture_skipped_mbs",
    "slice_ends_mid_row", "rows_without_slice", "pictures_without_slices", "slices_out_of_order",
    "vector_wrap", "full_pel_mbs", "mf_zero_vector_08", "mb_type_12",
    "edge_window_xy0", "edge_window_xy1", "edge_window_xy2", "edge_window_xy3",
    "mb_entries_gt48", "mb_entries_384", "escape_run_ge32", "escape16_level0", "abort_intra", "abort_inter",
    "qscale_0", "matrix_entry_0", "matrix_entry_1", "matrix_entry_255", "q7_dc_outside_0_255",
    "mb_width_lt22", "mb_height_lt12", "slice_rows_past_picture", "sequence_header_mid_stream",
    "extra_information_slice", "picture_type_3", "picture_type_4",
] + ["f_code_%d" % f for f in range(1, 8)] + ["vector_wrap_f_code_%d" % f for f in range(1, 7)]


@functools.lru_cache(maxsize=None)
def case(name):
    return sc.make(name)


@pytest.mark.parametrize("name", PINNED)
def test_restatement_equals_reference_pins(oracle, name):
    es, _, _, _ = case(name)
    pin = PINS[name]
    assert sha(es) == pin["es_sha256"], "%s: the generator no longer writes the pinned stream" % name
    oracle.stats_reset()
    got = oracle.decode_es(es)
    assert oracle.stats().pin_out_of_domain == 0, "%s left the clamp table's domain" % name
    assert got.shape[0] == pin["frames"], name
    for k in range(got.shape[0]):
        assert sha(got[k]) == pin["frame_sha256"][k], "%s picture %d" % (name, k)


def test_pinned_cases_are_exactly_the_in_domain_ones(oracle):
    assert sorted(PINS) == sorted(PINNED)
    for name in sc.UNPINNED:
        oracle.stats_reset()
        oracle.decode_es(case(name)[0])
        assert oracle.stats().pin_out_of_domain > 0, "%s is inside the domain: pin it" % name


def test_ts_wrapping_round_trips(oracle):
    from espflix_b200 import synth
    for name in ("header_0", "small_1", "stuffing_after_escape", "type3_p_grammar"):
        es, off, _, _ = case(name)
        assert np.array_equal(oracle.demux_ts(synth.wrap_ts(es, off)), es), name


def test_syntax_set_reaches_the_missing_paths(oracle):
    total = Counter()
    for name in PINNED:
        total.update(case(name)[2])
    missing = [f for f in FEATURES if total[f] <= 0]
    assert not missing, "never emitted by a pinned case: %s" % missing
    for name, feats in DIRECTED_FEATURE.items():
        c = case(name)[2]
        assert all(c[f] > 0 for f in feats), (name, {f: c[f] for f in feats})
    # the same paths seen from the decoder's side
    oracle.stats_reset()
    for name in PINNED:
        oracle.decode_es(case(name)[0])
    s = oracle.stats()
    assert s.pictures[3] > 0 and s.pictures[4] > 0
    assert s.f_code[7] > 0 and s.full_pel_mbs > 0
    assert all(v > 0 for v in s.mocomp_xy)
    assert s.escapes16 > 0 and s.skipped > 0 and s.blocks_dc_only > 0
    assert all(s.mb_type[t] > 0 for t in (0x01, 0x02, 0x08, 0x0A, 0x11, 0x12, 0x1A))
    assert s.pin_out_of_domain == 0


def test_outside_case_puts_its_windows_in_the_last_picture_only():
    es, off, c, outside = sc.outside_case()
    assert outside and all(mx in (0, 21) for mx, my in outside)
    assert c["picture_type_2"] == len(off) - 2                         # I then P pictures; the windows are in the last
