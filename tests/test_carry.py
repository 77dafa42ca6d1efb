"""The hold-back rule of TS submits cut at any packet boundary (tests/carry_cases.py), checked without a GPU: for every program
of pts_cases.cases(), both fixtures, a program with custom quantiser matrices and one ending in a lone sequence header, cut
before every packet and at seeded packets, the complete pictures of the submits concatenate to the pictures of the whole ES
and their pts to the pts of the whole program."""
import pytest

from tests import carry_cases, pts_cases


@pytest.fixture(scope="module")
def programs():
    return carry_cases.programs()


def _check(name, ts, cuts):
    es, _ = pts_cases.demux(ts)
    st = carry_cases.run(ts, cuts)
    assert st.codes == pts_cases.picture_codes(es), name
    assert st.pts == pts_cases.picture_pts(ts), name
    assert st.held_sizes[-1] == 0 and st.held == b""
    return st


def test_cut_before_every_packet(programs):
    for name, ts in programs:
        _check(name, ts, list(range(1, len(ts) // 188)))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_cut_at_seeded_packets(programs, seed):
    for i, (name, ts) in enumerate(programs):
        _check(name, ts, carry_cases.seeded_cuts(ts, 1000 * seed + i))


def test_cuts_cover_the_hard_cases(programs):
    """cut before every packet, the corpus meets every case the rule has to get right"""
    split_code = inside_matrices = pes_after_code = no_picture = 0
    for name, ts in programs:
        cuts = list(range(1, len(ts) // 188))
        es, _ = pts_cases.demux(ts)
        offs, pes = carry_cases.es_cut_offsets(ts, cuts)
        pes = set(pes)
        codes = set(pts_cases.picture_codes(es))
        for o in offs:
            if any(es[o - k:o - k + 3] == b"\x00\x00\x01" and o - k + 4 <= len(es) for k in (1, 2, 3)):
                split_code += 1
            if (o - 1 in codes or o - 2 in codes) and o in pes:      # within the two bytes after a code byte, a PES start there
                pes_after_code += 1
            q = es.rfind(b"\x00\x00\x01\xb3", 0, o)
            if q >= 0 and es[q + 11] & 3 and q + 12 < o <= q + 12 + 128:   # load_intra / load_non_intra: inside the matrices
                inside_matrices += 1
        st = carry_cases.run(ts, cuts)
        no_picture += sum(1 for c in st.counts if c == 0)
    assert split_code and inside_matrices and pes_after_code and no_picture


def test_end_drops_a_headers_only_tail():
    ts = carry_cases.headers_tail_program()
    es, _ = pts_cases.demux(ts)
    tail = len(es) - es.rfind(b"\x00\x00\x01\xb3")
    st = carry_cases.Stream()
    st.feed(ts)
    assert st.held_sizes[-1] == tail                                 # the lone sequence header is held ...
    assert st.codes == pts_cases.picture_codes(es)                   # the sequence code completes the last picture
    st.feed(b"", end=True)                                           # ... and the end of the stream drops it
    assert st.held == b"" and st.codes == pts_cases.picture_codes(es)
    assert st.pts == pts_cases.picture_pts(ts)


def test_scan_rules():
    seq = b"\x00\x00\x01\xb3" + bytes(8)
    pic = b"\x00\x00\x01\x00" + bytes(4)
    sl = b"\x00\x00\x01\x01" + b"\x55" * 10
    # a picture with its slices is held until a later unit code arrives whole
    assert carry_cases.scan(seq + pic + sl) == ([], len(seq + pic + sl), len(seq) + 3)
    assert carry_cases.scan(seq + pic + sl + b"\x00\x00\x01") == ([], len(seq + pic + sl) + 3, len(seq) + 3)
    assert carry_cases.scan(seq + pic + sl + pic) == ([len(seq) + 3], len(pic), len(seq + pic + sl) + 3)
    # headers after a complete picture start the held unit; a GOP header after a sequence header continues it
    gop = b"\x00\x00\x01\xb8" + bytes(4)
    assert carry_cases.scan(pic + sl + seq + gop) == ([3], len(seq + gop), None)
    # no unit open: the last 3 bytes; a sequence end: nothing; the end of the stream completes the last unit
    assert carry_cases.scan(b"\x11" * 10) == ([], 3, None)
    assert carry_cases.scan(pic + sl + b"\x00\x00\x01\xb7" + pic) == ([3], 0, None)
    assert carry_cases.scan(seq + pic + sl, end=True) == ([len(seq) + 3], 0, None)
