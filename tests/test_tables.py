"""ISO 11172-2 tables used by the product (ef_iso11172_tables.h) against the enumeration of the
reference's VLC trees (player.cpp:59-148) committed in tests/golden/vlc_codes.json."""
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "espflix_b200", "csrc", "ef_iso11172_tables.h")


def _table(name):
    s = open(HDR).read()
    i = s.index("static const ef_vlc_code %s[]" % name)
    body = s[i:s.index("};", i)]
    return {m.group(1): int(m.group(2), 0) for m in re.finditer(r'\{"([01]+)", (-?(?:0x)?[0-9A-Fa-f]+)\}', body)}


def _u8(name):
    s = open(HDR).read()
    i = s.index("static const unsigned char %s[" % name)
    body = s[s.index("{", i):s.index("};", i)]
    return [int(x) for x in re.findall(r"\d+", body)]


def _gold():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "vlc_codes.json")))


def test_mb_level_tables_match_reference_trees():
    g = _gold()
    assert _table("ef_vlc_mba") == g["macroblock_address_increment"]
    assert _table("ef_vlc_mbtype_i") == g["macroblock_type_I"]
    assert _table("ef_vlc_mbtype_p") == g["macroblock_type_P"]
    assert _table("ef_vlc_cbp") == g["coded_block_pattern"]
    assert _table("ef_vlc_mv") == g["motion_vec"]


def test_dct_table_matches_reference_tree():
    ref = dict(_gold()["dct_coeff"])
    mine = _table("ef_vlc_dct")
    assert ref.pop("000001") == -1          # escape marker in the reference tree
    assert ref.pop("1") == 1                # dct_coeff_first form of (0,1)
    assert mine.pop("11") == 1              # dct_coeff_next form of (0,1)
    assert mine == ref and len(mine) == 110


def test_prefix_free():
    for name in ("ef_vlc_mba", "ef_vlc_mbtype_p", "ef_vlc_cbp", "ef_vlc_mv", "ef_vlc_dct", "ef_vlc_dc_luma", "ef_vlc_dc_chroma"):
        codes = sorted(_table(name))
        for a, b in zip(codes, codes[1:]):
            assert not b.startswith(a), (name, a, b)


def test_numeric_tables():
    zz = _u8("ef_zigzag")
    assert sorted(zz) == list(range(64)) and zz[:6] == [0, 1, 8, 16, 9, 2]
    q = _u8("ef_default_intra_q")
    assert q[0] == 8 and q[63] == 83 and len(q) == 64
    import math
    s = [1.0] + [math.sqrt(2) * math.cos(k * math.pi / 16) for k in range(1, 8)]
    assert _u8("ef_aan_prescale") == [int(math.floor(32 * s[i] * s[j] + 0.5)) for i in range(8) for j in range(8)]


def test_chroma_lut_closed_form():
    """The composite chroma LUTs (video.cpp:335-507; derivation espflix.cpp:1091-1180) have a closed form (described in
    csrc/ef_composite.cu): phases 48, 48 +- r(c), r(c) = sgn(128 - c) * ((16 |128 - c| + 11) / 22), clamped to [0, 127]."""
    import numpy as np

    def r(c):
        d = 128 - c
        q = (16 * abs(d) + 11) // 22
        return q if d >= 0 else -q

    def cl(x):
        return max(0, min(127, x))

    for name in ("ntsc", "pal"):
        t = np.fromfile(os.path.join(ROOT, "tests", "golden", "color_tab_%s.u32" % name), dtype=np.uint32)
        for c in range(256):
            rr = r(c)
            sin = (48 << 24) | (48 << 16) | (cl(48 + rr) << 8) | cl(48 - rr)
            cos = (cl(48 + rr) << 24) | (cl(48 - rr) << 16) | (48 << 8) | 48
            cosn = (cl(48 - rr) << 24) | (cl(48 + rr) << 16) | (48 << 8) | 48
            assert t[c] == sin and t[256 + c] == cos and t[512 + c] == (cos if name == "ntsc" else cosn), (name, c)
