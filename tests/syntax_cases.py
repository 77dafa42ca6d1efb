"""Syntax-level MPEG-1 streams: the grammar the reference decoder READS (player.cpp:658-724, 733-889, 999-1148,
1251-1316), written from seeded random choices. No pixel content and no motion search, so the streams reach what an
encoder never chooses: stuffing and escapes in the macroblock address, ignored first increments (Q6), skip runs across
rows and in I pictures, slices that end mid-row, rows and pictures without slices, vector predictor wrap, windows at the
frame edges, dense and aborted blocks, long-run and 16-bit escapes, quantiser_scale 0, matrix entries 0 / 1 / 255,
drifting intra DC predictors (Q7), small pictures, mid-stream sequence headers, extra_information_slice and pictures of
type 3 / 4 (parsed with the P tables and the last P header's vector parameters).

Every stream stays inside the reference's defined behaviour: only valid codes; every prediction window inside the
352 x 192 frame (small pictures get vectors into the part of the frame outside the picture); slices never overlap or
share a row; mb_width <= 22 and every macroblock row < 12; no run of 23 zero bits inside a slice (the reference would end
the slice there, the index kernel would see a start code). Whether samples stay inside the clamp table's domain is
decided by the restatement after generation (UNPINNED).

Random numbers come from splitmix64 and the VLC codes from tests/golden/vlc_codes.json (the reference's own trees), so
the streams do not depend on numpy or CPython versions."""
import json
import os
from collections import Counter

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_VLC = json.load(open(os.path.join(ROOT, "tests", "golden", "vlc_codes.json")))


def _inv(name):
    return {v: c for c, v in _VLC[name].items()}


MBA, TYPE_I, TYPE_P, CBP, MV = (_inv(n) for n in ("macroblock_address_increment", "macroblock_type_I", "macroblock_type_P",
                                                  "coded_block_pattern", "motion_vec"))
DCT = {(v >> 8, v & 255): c for c, v in _VLC["dct_coeff"].items() if v > 0}
ESCAPE = "000001"
LUMA_DC = ["100", "00", "01", "101", "110", "1110", "11110", "111110", "1111110"]          # dct_dc_size_luminance 0..8
CHROMA_DC = ["00", "01", "10", "110", "1110", "11110", "111110", "1111110", "11111110"]    # dct_dc_size_chrominance 0..8
M64 = (1 << 64) - 1


class Rng:
    """splitmix64"""

    def __init__(self, seed):
        self.s = seed & M64

    def next(self):
        self.s = (self.s + 0x9E3779B97F4A7C15) & M64
        z = self.s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        return z ^ (z >> 31)

    def int(self, lo, hi):                  # inclusive
        return lo + self.next() % (hi - lo + 1)

    def chance(self, p):
        return self.next() < int(p * 18446744073709551616)

    def pick(self, seq):
        return seq[self.next() % len(seq)]


def _b(v, n):
    return format(v & ((1 << n) - 1), "0%db" % n) if n else ""


# what each profile draws; directed cases override single knobs
BASE = dict(
    sizes=[(352, 192)], n_pictures=(6, 12), p_i=0.15, p_type34=0.0, p_seq_mid=0.0, p_matrices=0.0, matrix_extremes=0.0,
    p_row_gap=0.0, p_mid_end=0.0, p_zero_slices=0.0, span=(1, 1), p_past_rows=0.0, p_shuffle=0.0, p_extra=0.0,
    p_q6=0.0, p_skip=0.1, skip_max=4, p_long_skip=0.0, p_stuff=0.0, p_esc_stuff=0.0,
    qscale=(2, 12), p_q0=0.0, p_mquant=0.1, p_intra_in_p=0.05, p_mf=0.6, p_coded=0.7, p_zero_mv=0.05,
    fcodes=[1, 2, 3], p_fullpel=0.1, p_far=0.2, p_edge=0.1, p_wrap=0.3,
    p_cbp=0.5, coefs=(0, 6), p_dense=0.0, p_escape=0.05, p_long_run=0.0, p_esc16=0.0, p_abort=0.0, level_max=3,
    p_dc_only=0.3, p_dc_drift=0.0, outside_last=False, budget=900,
)
PROFILES = {
    "header": dict(p_type34=0.15, p_seq_mid=0.3, p_matrices=0.3, p_row_gap=0.15, p_mid_end=0.3, p_zero_slices=0.08,
                   span=(1, 3), p_shuffle=0.3, p_extra=0.3, p_q6=0.3, p_skip=0.35, skip_max=40, p_long_skip=0.3,
                   p_stuff=0.2, p_esc_stuff=0.5, p_q0=0.05),
    "dense": dict(p_cbp=0.9, coefs=(20, 64), p_dense=0.3, p_escape=0.15, p_long_run=0.05, p_esc16=0.05, p_abort=0.08,
                  qscale=(1, 2), p_q0=0.1, p_mquant=0.2, level_max=2, p_matrices=0.3, matrix_extremes=0.2),
    "vector": dict(fcodes=[1, 2, 3, 4, 5, 6, 7], p_fullpel=0.3, p_far=0.5, p_edge=0.35, p_wrap=0.8, p_mf=0.85,
                   p_zero_mv=0.1, p_type34=0.1, p_skip=0.15),
    "small": dict(sizes=[(320, 176), (176, 96), (16, 16), (200, 130), (96, 190), (352, 40), (33, 177)], p_past_rows=0.5,
                  p_row_gap=0.1, p_mid_end=0.2, span=(1, 3), p_skip=0.3, skip_max=30, p_long_skip=0.2, p_seq_mid=0.3,
                  fcodes=[1, 2, 3, 4], p_far=0.4, p_edge=0.3),
    "mixed": dict(p_type34=0.1, p_seq_mid=0.15, p_matrices=0.2, matrix_extremes=0.1, p_row_gap=0.05, p_mid_end=0.1,
                  span=(1, 2), p_extra=0.1, p_q6=0.1, p_skip=0.2, skip_max=30, p_long_skip=0.1, p_stuff=0.05,
                  p_esc_stuff=0.2, fcodes=[1, 2, 3, 4, 5, 6, 7], p_far=0.3, p_edge=0.2, p_cbp=0.6,
                  coefs=(0, 20), p_escape=0.1, p_long_run=0.02, p_esc16=0.02, p_abort=0.03, p_dc_drift=0.1),
}


class _Stream:
    def __init__(self, seed, knobs):
        self.r = Rng(seed)
        self.k = knobs
        self.out = []                       # ES as bit strings, each a whole number of bytes at start codes
        self.nbits = 0
        self.census = Counter()
        self.pic_off = []
        self.mbw = self.mbh = 0
        self.fp, self.rs = 0, 0             # last P header: full_pel_forward, forward_r_size
        self.have_p = False
        self.outside = []                   # (mx, my) of macroblocks whose window leaves the frame (last picture only)

    # ---- bit output ------------------------------------------------------------------------------------------------
    def put(self, s):
        self.out.append(s)
        self.nbits += len(s)

    def align(self):
        if self.nbits % 8:
            self.put("0" * (8 - self.nbits % 8))

    def start_code(self, c):
        self.align()
        self.put("0" * 23 + "1" + _b(c, 8))

    def es(self):
        self.align()
        s = "".join(self.out)
        return np.frombuffer(int(s, 2).to_bytes(len(s) // 8, "big"), dtype=np.uint8).copy() if s else np.zeros(0, np.uint8)

    # ---- headers (player.cpp:658-724) -------------------------------------------------------------------------------
    def sequence(self, size):
        r, k = self.r, self.k
        w, h = size
        self.start_code(0xB3)
        self.put(_b(w, 12) + _b(h, 12) + _b(1, 4) + _b(3, 4) + _b(0x3FFFF, 18) + "1" + _b(20, 10) + "0")
        self.qmax = [83, 16]                # largest entry of the intra / non-intra matrix in force (default intra: 83)
        for i in range(2):
            if r.chance(k["p_matrices"]):
                m = [r.int(1, 64) for _ in range(64)]
                if r.chance(k["matrix_extremes"]):
                    for _ in range(r.int(1, 8)):
                        m[r.int(0, 63)] = r.pick([0, 1, 255])
                self.census["matrix_loaded"] += 1
                self.census["matrix_entry_0"] += m.count(0)
                self.census["matrix_entry_1"] += m.count(1)
                self.census["matrix_entry_255"] += m.count(255)
                self.put("1" + "".join(_b(v, 8) for v in m))
                self.qmax[i] = max(m)
            else:
                self.put("0")
        self.mbw, self.mbh = (w + 15) >> 4, (h + 15) >> 4
        if self.mbw < 22:
            self.census["mb_width_lt22"] += 1
        if self.mbh < 12:
            self.census["mb_height_lt12"] += 1

    def gop(self, n):
        self.start_code(0xB8)
        self.put(_b((1 << 12) | (n & 63), 25) + "1" + "0" * 6)

    def picture(self, n, ptype):
        self.start_code(0x00)
        self.put(_b(n, 10) + _b(ptype, 3))
        self.census["picture_type_%d" % ptype] += 1
        if ptype in (1, 2):
            self.put(_b(0xFFFF, 16))
        if ptype == 2:
            self.fp = 1 if self.r.chance(self.k["p_fullpel"]) else 0
            f_code = self.r.pick(self.k["fcodes"])
            self.rs = f_code - 1
            self.put(_b(self.fp, 1) + _b(f_code, 3))
            self.census["f_code_%d" % f_code] += 1
            self.census["full_pel_pictures"] += self.fp
            self.have_p = True

    # ---- slice (player.cpp:1251-1316) -------------------------------------------------------------------------------
    def address(self, inc, first, c):
        """macroblock_address_increment `inc`, possibly with stuffing, escapes, or an escape followed by stuffing
        (the reference then adds 34: it skips stuffing only before the first escape, player.cpp:1268-1275)"""
        r, k = self.r, self.k
        s = ""
        if r.chance(k["p_stuff"]):
            n = r.int(1, 3)
            s += MBA[34] * n
            c["stuffing"] += n
        if inc >= 67 and (inc - 34) % 33 == 0 and r.chance(k["p_esc_stuff"]):
            e = (inc - 34) // 33
            s += MBA[35] * e + MBA[34]
            c["address_escape"] += e
            c["stuffing_after_escape_" + ("slice_start" if first else "mid_slice")] += 1
            return s
        e = (inc - 1) // 33
        c["address_escape"] += e
        return s + MBA[35] * e + MBA[inc - 33 * e]

    def window_ok(self, mx, my, h, v):
        """prediction window of macroblock (mx, my) with vector (h, v) in half pels: inside the 352 x 192 frame,
        luma (predict(), player.cpp:882) and chroma (Q3)"""
        hx, hy = mx * 32 + h, my * 32 + v
        if hx < 0 or hy < 0 or (hx >> 1) + 16 + (hx & 1) > 352 or (hy >> 1) + 16 + (hy & 1) > 192:
            return False
        cx, cy = hx >> 1, hy >> 1
        return (cx >> 1) + 8 + (cx & 1) <= 176 and (cy >> 1) + 8 + (cy & 1) <= 96

    def vector(self, mx, my, pred, c, outside):
        """target vector (stored units) for a macroblock with motion_forward, its window inside the frame"""
        r, k, fp, rs = self.r, self.k, self.fp, self.rs
        lo, hi = -(16 << rs), (16 << rs) - 1
        if outside and (mx == 21 or (mx == 0 and my >= 1)):     # leaves the frame sideways by 1..15 half pels
            h = r.int(1, 15) if mx == 21 else -r.int(1, 15)
            t = (h >> fp, 0)
            if lo <= t[0] <= hi and (t[0] << fp) != 0:
                return t
        for _ in range(8):
            if r.chance(k["p_zero_mv"]):
                t = (0, 0)
            elif r.chance(k["p_edge"]):                  # window touching the right or bottom frame edge
                ex = r.pick([0, 1])
                hx = 2 * (336 - ex) + ex if r.chance(0.5) else r.int(0, 671)
                hy = 2 * (176 - r.pick([0, 1])) + r.pick([0, 1]) if r.chance(0.5) else r.int(0, 351)
                if (hy >> 1) + 16 + (hy & 1) > 192:
                    hy -= 2
                t = ((hx - mx * 32) >> fp, (hy - my * 32) >> fp)
            elif r.chance(k["p_far"]):
                t = ((r.int(0, 671) - mx * 32) >> fp, (r.int(0, 351) - my * 32) >> fp)
            else:
                t = (pred[0] + r.int(-6, 6), pred[1] + r.int(-6, 6))
            t = (min(hi, max(lo, t[0])), min(hi, max(lo, t[1])))
            if self.window_ok(mx, my, t[0] << fp, t[1] << fp):
                return t
        return (0, 0)

    def mv_component(self, p, t, c):
        """code so that motion_vector() (player.cpp:891) turns predictor p into t; wraps when it has to or by choice"""
        rs = self.rs
        rng = 16 << rs
        d = t - p
        alt = d - (32 << rs) if d > 0 else d + (32 << rs)
        if abs(d) > rng or (abs(alt) <= rng and self.r.chance(self.k["p_wrap"])):
            d = alt
        assert abs(d) <= rng
        if not -(16 << rs) <= p + d <= (16 << rs) - 1:
            c["vector_wrap"] += 1
            c["vector_wrap_f_code_%d" % (rs + 1)] += 1
        if d == 0:
            return MV[0]
        if rs == 0:
            return MV[d]
        a = abs(d) - 1
        code = (a >> rs) + 1
        return MV[code if d > 0 else -code] + _b(a & ((1 << rs) - 1), rs)

    def coef(self, run, level, first, c, force_escape=False, force16=False):
        if not force_escape and not force16:
            if run == 0 and abs(level) == 1:
                return ("1" if first else "11") + ("1" if level < 0 else "0")
            if (run, abs(level)) in DCT:
                return DCT[(run, abs(level))] + ("1" if level < 0 else "0")
        c["escape"] += 1
        if run >= 32:
            c["escape_run_ge32"] += 1
        s = ESCAPE + _b(run, 6)
        if 1 <= abs(level) <= 127 and not force16:
            return s + _b(level, 8)
        c["escape16"] += 1
        if level == 0:
            c["escape16_level0"] += 1
        return s + ("00000000" + _b(level, 8) if level >= 0 else "10000000" + _b(level + 256, 8))

    def dc(self, blk, pred, c, drift, dc_only):
        """dct_dc_size + differential (player.cpp:1010-1068); returns (bits, new predictor)"""
        r = self.r
        if drift:
            target = r.pick([r.int(-120, -1), r.int(256, 400)])
        elif not 0 <= pred <= 255:
            target = r.int(16, 235)
        else:
            target = r.int(16, 235) if r.chance(0.5) else pred + r.int(-20, 20)
        diff = max(-255, min(255, target - pred))
        size = abs(diff).bit_length()
        tab = LUMA_DC if blk < 4 else CHROMA_DC
        s = tab[size]
        if size:
            s += _b(diff if diff > 0 else diff + (1 << size) - 1, size)
        dcv = pred + diff
        if dc_only and not 0 <= dcv <= 255:
            c["q7_dc_outside_0_255"] += 1
        return s, dcv

    def block(self, intra, q, c, dense):
        """coefficients of one block, end of block or an abort (n > 63: no end of block, the next block follows,
        player.cpp:1100-1104); returns (bits, list entries, aborted)"""
        for _ in range(32):
            t = Counter()
            res = self._block(intra, q, t, dense)
            if "0" * 23 not in res[0]:
                c.update(t)
                return res
        raise RuntimeError("no block without a start-code emulation")

    def _block(self, intra, q, c, dense):
        # The sum of the dequantised magnitudes is kept under the budget, which keeps every sample of the inverse transform
        # well inside the clamp table's domain (a coefficient moves a sample by at most about |v| / 4)
        r, k = self.r, self.k
        budget, wmax = k["budget"], self.qmax[0 if intra else 1]
        n = 1 if intra else 0
        s, entries = "", 0
        if dense:
            target = 64 - n
        else:
            target = r.int(*k["coefs"])
            if not intra:
                target = max(1, target)
        abort = r.chance(k["p_abort"])
        lm = k["level_max"]
        while True:
            if n > 0 and (entries >= target or n >= 64):
                if abort and n < 64:
                    run = r.int(64 - n, min(63, 64 - n + 10))
                    s += self.coef(run, r.pick([-1, 1]), False, c, force_escape=run > 31 or r.chance(0.5))
                    c["abort_" + ("intra" if intra else "inter")] += 1
                    return s, entries, True
                return s + "10", entries, False
            if dense:
                run = 0
            elif r.chance(k["p_long_run"]) and n + 32 <= 63:
                run = r.int(32, 63 - n)
            else:
                run = min(r.int(0, 3) if r.chance(0.8) else r.int(0, 20), 63 - n)
            level = r.int(1, lm) * r.pick([-1, 1])
            if r.chance(k["p_escape"]):
                level = r.int(1, 40) * r.pick([-1, 1])
            # 16-bit escapes: an odd run ends the run field in a 1, so a level byte of 0 leaves fewer than 23 zeros
            force16 = not dense and n + (run | 1) <= 63 and r.chance(k["p_esc16"])
            if force16:
                run |= 1
                level = r.pick([0, 0, 1, -1, r.int(128, 160), -r.int(128, 160)])
            v = (2 * abs(level) + 1) * q * wmax // 16
            if v > budget:
                level = 1 if level > 0 else -1 if level < 0 else 0
                v = 3 * q * wmax // 16
                if v > budget and n > 0 and not dense:
                    target = entries
                    continue
            budget -= v
            s += self.coef(run, level, n == 0, c, force_escape=run > 31 or r.chance(k["p_escape"]), force16=force16)
            n += run + 1
            entries += 1

    def macroblock(self, mx, my, ptype, st, c, outside_ok):
        r, k = self.r, self.k
        if ptype == 1:
            mb_type = 0x11 if r.chance(k["p_mquant"]) else 0x01
        else:
            intra = r.chance(k["p_intra_in_p"])
            mf = not intra and r.chance(k["p_mf"])
            coded = intra or not mf or r.chance(k["p_coded"])
            q = r.chance(k["p_mquant"])
            mb_type = 0x01 if intra else (0x08 if mf else 0) | (0x02 if coded else 0)
            if q and (intra or coded):
                mb_type |= 0x10
            if mb_type == 0:
                mb_type = 0x02
            c["mb_type_%02x" % mb_type] += 1
        s = (TYPE_I if ptype == 1 else TYPE_P)[mb_type]
        if mb_type & 0x10:
            st["q"] = 0 if r.chance(k["p_q0"]) else r.int(*k["qscale"])
            c["qscale_0"] += st["q"] == 0
            s += _b(st["q"], 5)
        intra = mb_type & 1
        if intra:
            st["mv"] = (0, 0)
        else:
            st["dc"] = [128, 128, 128]
            if mb_type & 0x08:
                t = self.vector(mx, my, st["mv"], c, outside_ok and r.chance(0.5))
                s += self.mv_component(st["mv"][0], t[0], c) + self.mv_component(st["mv"][1], t[1], c)
                st["mv"] = t
                h, v = t[0] << self.fp, t[1] << self.fp
                if (h, v) == (0, 0):
                    c["mf_zero_vector_%02x" % mb_type] += 1
                if not self.window_ok(mx, my, h, v):
                    self.outside.append((mx, my))
                else:
                    hx, hy = mx * 32 + h, my * 32 + v
                    if (hx >> 1) + 16 + (hx & 1) == 352 or (hy >> 1) + 16 + (hy & 1) == 192:
                        c["edge_window_xy%d" % ((hx & 1) | (hy & 1) << 1)] += 1
                c["full_pel_mbs"] += self.fp
            else:
                st["mv"] = (0, 0)
        if mb_type & 0x02:
            cbp = 63 if r.chance(k["p_dense"]) else r.int(1, 63)
            s += CBP[cbp]
        else:
            cbp = 63 if intra else 0
        dense = cbp == 63 and r.chance(k["p_dense"])
        entries = 0
        for b in range(6):
            if not cbp & (32 >> b):
                continue
            if intra:
                comp = 0 if b < 4 else b - 3
                dc_only = r.chance(k["p_dc_only"]) and not dense
                bits, st["dc"][comp] = self.dc(b, st["dc"][comp], c, dc_only and r.chance(k["p_dc_drift"]), dc_only)
                s += bits
                if dc_only:
                    s += "10"
                    continue
            bits, e, _ = self.block(intra, st["q"], c, dense)
            s += bits
            entries += e
        c["mb_entries_max"] = max(c["mb_entries_max"], entries)
        if entries > 48:
            c["mb_entries_gt48"] += 1
        if entries == 384:
            c["mb_entries_384"] += 1
        return s

    def slice(self, row, end, ptype, c, outside_ok):
        """macroblocks from address row * mb_width up to (not including) address `end`"""
        r, k, mbw = self.r, self.k, self.mbw
        st = {"q": 0 if r.chance(k["p_q0"]) else r.int(*k["qscale"]), "mv": (0, 0), "dc": [128, 128, 128]}
        c["qscale_0"] += st["q"] == 0
        s = _b(st["q"], 5)
        while r.chance(k["p_extra"]):
            s += "1" + _b(r.int(1, 255), 8)
            c["extra_information_slice"] += 1
        s += "0"
        addr = row * mbw
        first = 1
        if r.chance(k["p_q6"]):
            first = r.pick([67, 100]) if r.chance(k["p_esc_stuff"]) else r.int(2, 140)
        if first != 1:
            c["q6_first_increment"] += 1
        s += self.address(first, True, c)
        while True:
            s += self.macroblock(addr % mbw, addr // mbw, ptype, st, c, outside_ok)
            room = end - 1 - addr
            if room <= 0:
                break
            inc = 1
            if r.chance(k["p_skip"]) and room >= 2:
                inc = r.int(2, min(room, k["skip_max"] + 1))
                if r.chance(k["p_long_skip"]) and room >= 34:
                    inc = r.pick([67, 100]) if room >= 67 and r.chance(0.5) else r.int(34, min(room, 120))
                    inc = min(inc, room)
            if inc > 1:
                st["mv"], st["dc"] = (0, 0), [128, 128, 128]
                c["skipped_mbs"] += inc - 1
                if ptype == 1:
                    c["i_picture_skipped_mbs"] += inc - 1
                if (addr + 1) // mbw != (addr + inc) // mbw:          # K1b walks the run back across a row
                    c["skip_run_across_rows"] += 1
                    if inc - 1 > 33:
                        c["skip_run_gt33_across_rows"] += 1
            s += self.address(inc, False, c)
            addr += inc
        return s

    def picture_slices(self, ptype, last):
        r, k = self.r, self.k
        mbw, mbh = self.mbw, self.mbh
        if r.chance(k["p_zero_slices"]):
            self.census["pictures_without_slices"] += 1
            return
        rows_limit = 12 if r.chance(k["p_past_rows"]) and mbh < 12 else mbh
        slices, row = [], 0
        while row <= min(mbh, 11) and row < rows_limit:
            if r.chance(k["p_row_gap"]):
                self.census["rows_without_slice"] += 1
                row += 1
                continue
            span = min(r.int(*k["span"]), rows_limit - row)
            end = (row + span) * mbw
            if r.chance(k["p_mid_end"]) and mbw > 1:
                end -= r.int(1, mbw - 1)
                self.census["slice_ends_mid_row"] += 1
            if row + span > mbh:
                self.census["slice_rows_past_picture"] += 1
            slices.append((row, end))
            row += span
        if len(slices) > 1 and r.chance(k["p_shuffle"]):
            for i in range(len(slices) - 1, 0, -1):
                j = r.int(0, i)
                slices[i], slices[j] = slices[j], slices[i]
            self.census["slices_out_of_order"] += 1
        for row, end in slices:
            for attempt in range(64):
                c = Counter()
                saved = len(self.outside)
                body = self.slice(row, end, ptype, c, last and k["outside_last"] and ptype == 2)
                if "0" * 23 not in body:
                    break
                del self.outside[saved:]
            else:
                raise RuntimeError("no slice without a start-code emulation")
            self.start_code(row + 1)
            self.put(body)
            mx = c.pop("mb_entries_max", 0)
            self.census.update(c)
            self.census["mb_entries_max"] = max(self.census["mb_entries_max"], mx)
            self.census["slices"] += 1


def generate(seed, knobs):
    """-> (es uint8 array, picture offsets uint32[n+1], census Counter, [(mx, my) windows outside the frame])"""
    k = dict(BASE)
    k.update(knobs)
    g = _Stream(seed, k)
    r = g.r
    n = r.int(*k["n_pictures"])
    size = r.pick(k["sizes"])
    for p in range(n):
        g.pic_off.append(g.nbits // 8 + (1 if g.nbits % 8 else 0))
        if p == 0 or r.chance(k["p_seq_mid"]):
            if p:
                size = r.pick(k["sizes"])
                g.census["sequence_header_mid_stream"] += 1
            g.sequence(size)
            g.gop(p)
        if p == 0 or r.chance(k["p_i"]):
            ptype = 1
        elif g.have_p and r.chance(k["p_type34"]):
            ptype = r.pick([3, 4])
        else:
            ptype = 2
        if k.get("ptypes"):
            ptype = k["ptypes"][p % len(k["ptypes"])]
        g.picture(p, ptype)
        g.picture_slices(1 if ptype == 1 else 2, p == n - 1)
    es = g.es()
    off = np.array(g.pic_off + [es.size], dtype=np.uint32)
    return es, off, g.census, g.outside


# ---- the case list --------------------------------------------------------------------------------------------------
SEED0 = 0x53594E54          # "SYNT"

DIRECTED = {
    "stuffing_after_escape": dict(p_q6=0.6, p_stuff=0.3, p_esc_stuff=1.0, p_skip=0.3, p_long_skip=0.7, skip_max=2, span=(2, 4)),
    "intra_abort": dict(p_i=1.0, p_abort=0.5, coefs=(3, 30), p_cbp=1.0, p_dc_only=0.1, qscale=(1, 3)),
    "skip_run_across_rows": dict(span=(3, 6), p_skip=0.4, p_long_skip=0.8, skip_max=30, p_i=0.3),
    "qscale0": dict(p_q0=0.5, p_mquant=0.5, coefs=(2, 30), p_esc16=0.05),
    "matrices_1_255": dict(p_matrices=1.0, matrix_extremes=1.0, p_seq_mid=0.4, qscale=(1, 2), coefs=(1, 10), level_max=1),
    "fcode7": dict(fcodes=[7], p_fullpel=0.5, p_far=0.8, p_edge=0.4, p_mf=0.9),
    "vector_wrap": dict(fcodes=[1, 2, 3, 4, 5, 6], p_wrap=1.0, p_far=0.7, p_mf=0.95, p_zero_mv=0.0, p_skip=0.0),
    "pic_320x176": dict(sizes=[(320, 176)], p_past_rows=1.0, p_skip=0.3, skip_max=30, p_far=0.4, p_edge=0.3),
    "pic_176x96": dict(sizes=[(176, 96)], p_past_rows=1.0, span=(1, 4), p_skip=0.3, skip_max=30, p_far=0.5, p_edge=0.3),
    "slices_mid_row": dict(p_mid_end=0.7, p_row_gap=0.3, p_zero_slices=0.2, span=(1, 2), p_shuffle=0.5, p_extra=0.5),
    "type3_p_grammar": dict(ptypes=[1, 2, 3, 2, 4, 3, 3, 2], n_pictures=(8, 8), fcodes=[2, 3, 5], p_fullpel=0.5),
    "q7_dc_bleed": dict(p_i=0.5, p_dc_only=0.8, p_dc_drift=0.5, p_intra_in_p=0.3),
    "mb_384_entries": dict(p_dense=0.6, p_cbp=1.0, coefs=(30, 64), level_max=1, qscale=(1, 2), p_coded=1.0,
                           p_mf=0.5, p_intra_in_p=0.0, p_escape=0.0),
}
# Outside the reference's defined domain (samples leave [-256, 511]): compared with the restatement only.
OUT_OF_DOMAIN = {
    "overdrive": dict(budget=1 << 30, qscale=(12, 31), level_max=12, p_escape=0.3, p_esc16=0.1, coefs=(2, 20), p_matrices=0.5),
}
UNPINNED = list(OUT_OF_DOMAIN)
RANDOM = [(p, i) for p in ("header", "dense", "vector", "small", "mixed") for i in range(8)]


def case_names():
    return ["%s_%d" % (p, i) for p, i in RANDOM] + list(DIRECTED) + UNPINNED


def knobs_of(name):
    if name in DIRECTED:
        return DIRECTED[name]
    if name in OUT_OF_DOMAIN:
        return OUT_OF_DOMAIN[name]
    p, _ = name.rsplit("_", 1)
    return PROFILES[p]


def seed_of(name):
    h = 0
    for ch in name.encode():
        h = (h * 131 + ch) & M64
    return SEED0 ^ h


def make(name):
    return generate(seed_of(name), knobs_of(name))


def outside_case():
    """A stream whose last picture has macroblocks with windows that leave the frame sideways (the device clamps into
    the frame, the reference reads the neighbouring strip bytes): -> (es, off, census, [(mx, my)])"""
    return generate(SEED0 + 7, dict(n_pictures=(6, 6), p_mf=0.9, p_skip=0.0, p_i=0.0, outside_last=True))

