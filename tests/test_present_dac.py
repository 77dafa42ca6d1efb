"""EF_FIELD_DAC8, CPU side: the playback order of tests/dac_cases.py pinned to the reference's own code. burst_pal() writes
line[i ^ 1] = b[i] (video.cpp:640-644) so that the DAC plays its burst table b in order; the oracle's burst0 / burst1 are the
tables pal_init builds and its field() the reference's line buffer. The DAC bytes over the burst span of a PAL line must then
be the high bytes of that line's table in order."""
import numpy as np
import pytest

from tests import dac_cases
from tests.oracle_lib import Oracle


def _tables(o):
    v = o.video(0)
    hi = lambda t: (np.array(t[:], dtype=np.int16).view(np.uint16)[:v.burst_width] >> 8).astype(np.uint8)   # noqa: E731
    return v, hi(v.burst0), hi(v.burst1)


@pytest.mark.parametrize("line", [100, 101, 10, 11])     # active and blanking lines of both burst phases
def test_pal_burst_plays_in_table_order(line):
    o = Oracle()
    v, b0, b1 = _tables(o)
    frame = np.random.RandomState(line).randint(0, 256, size=101376).astype(np.uint8)
    u16 = o.field(frame, 0, 1).reshape(v.line_count, v.line_width)
    got = dac_cases.dac8(u16[line])[v.burst_start:v.burst_start + v.burst_width]
    want = b0 if line % 2 == 0 else b1                   # the table alternates line by line (burst_pal())
    assert np.array_equal(got, want), "line %d: the DAC bytes over the burst are not the table in order" % line


def test_buffer_order_is_not_playback_order():
    """the same bytes read in buffer order are not the table: burst0's pattern (10 29 29 10) shows the pair swap. burst1's
    (29 29 10 10) reads the same either way, so only the burst0 phase tells the two orders apart."""
    o = Oracle()
    v, b0, b1 = _tables(o)
    assert not np.array_equal(b0, b0.reshape(-1, 2)[:, ::-1].reshape(-1))
    u16 = o.field(np.zeros(101376, np.uint8), 0, 1).reshape(v.line_count, v.line_width)
    for line in (100, 10):
        raw = (u16[line, v.burst_start:v.burst_start + v.burst_width] >> 8).astype(np.uint8)
        assert not np.array_equal(raw, b0)


@pytest.mark.parametrize("ntsc", [1, 0])
def test_field_size_and_levels(ntsc):
    """a DAC8 field is line_count x line_width bytes; sync plays as 0x00 and black as 0x18 (IRE(-40), IRE(7.5))"""
    o = Oracle()
    v = o.video(ntsc)
    u16 = o.field(np.zeros(101376, np.uint8), ntsc, 1)
    d = dac_cases.dac8(u16)
    assert d.dtype == np.uint8 and d.size == dac_cases.FIELD_BYTES[ntsc] == v.line_count * v.line_width
    line = d.reshape(v.line_count, v.line_width)[40]     # above the picture, above vsync_start: sync, burst, black
    assert (line[:v.hsync] == 0).all()
    black = 104 if ntsc else 140                         # the end of the burst (burst(): 64 + 40; burst_pal(): 96 + 44)
    assert (line[black:black + 8] == 0x18).all()
