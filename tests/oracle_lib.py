"""tests/oracle_lib.py — loads the CPU checkers under oracle/ (TEST INFRASTRUCTURE). Only tests,
__graft_entry__.smoke() and bench.py's cpu_baseline/reference legs import this."""
import ctypes
import json
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I420 = 101376
FRAME = 101376
REF_DECODE = os.path.join(ROOT, "oracle", "_ref", "efref_decode")
REF_VIDEO = os.path.join(ROOT, "oracle", "_ref", "libefref_vid.so")
REF_INDEX = os.path.join(ROOT, "oracle", "_ref", "libefref_idx.so")
IDX_PAD = [36, 37, 38, 39, 68, 69, 70, 71, 100, 101, 102, 103]      # padding bytes of idx_hdr (indeterminate in the reference)


class _Video(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in "ntsc line_width line_count hsync hsync_long hsync_short burst_start burst_width active_start".split()] + \
               [("color_tab", ctypes.c_uint32 * 768), ("burst0", ctypes.c_int16 * 64), ("burst1", ctypes.c_int16 * 64)]


class _Stats(ctypes.Structure):
    _fields_ = [("pictures", ctypes.c_uint64 * 8), ("f_code", ctypes.c_uint64 * 8)] + \
               [(n, ctypes.c_uint64) for n in "slices skipped blocks blocks_dc_only escapes escapes16 saturated q2_zero full_pel_mbs".split()] + \
               [("mb_type", ctypes.c_uint64 * 32), ("mocomp_xy", ctypes.c_uint64 * 4), ("pin_out_of_domain", ctypes.c_uint64)]


class Oracle:
    """The C restatement (oracle/libef_oracle.so)."""

    def __init__(self):
        self.lib = ctypes.CDLL(os.path.join(ROOT, "oracle", "libef_oracle.so"))
        L, VP = self.lib, ctypes.c_void_p
        L.efo_demux_ts.restype = ctypes.c_size_t
        L.efo_demux_ts.argtypes = [VP, ctypes.c_size_t, VP, ctypes.c_size_t, VP, VP, ctypes.c_size_t, VP]
        L.efo_decode_es.restype = ctypes.c_long
        L.efo_decode_es.argtypes = [VP, ctypes.c_size_t, ctypes.c_int, VP, ctypes.c_size_t, VP]
        L.efo_decode_ts.restype = ctypes.c_long
        L.efo_decode_ts.argtypes = [VP, ctypes.c_size_t, VP, ctypes.c_size_t]
        L.efo_idct.argtypes = [VP]
        L.efo_i420_to_strips.argtypes = [VP, VP]
        L.efo_strips_to_i420.argtypes = [VP, VP]
        L.efo_video_init.argtypes = [VP, ctypes.c_int]
        L.efo_blit.argtypes = [VP, VP, VP, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.efo_field.argtypes = [VP, VP, ctypes.c_int, VP]
        L.efo_field_ex.argtypes = [VP, VP, VP, ctypes.c_int, ctypes.c_int, VP, ctypes.c_int, ctypes.c_int, VP]
        L.efo_stats_get.argtypes = [VP]
        L.efo_coverage.restype = ctypes.c_int
        L.efo_coverage.argtypes = [VP, ctypes.c_int]
        L.efo_walk.restype = ctypes.c_long
        L.efo_walk.argtypes = [VP, ctypes.c_size_t, VP, VP, ctypes.c_size_t, VP]
        L.efo_paced_schedule.restype = ctypes.c_long
        L.efo_paced_schedule.argtypes = [VP, VP, ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_long, VP, VP]
        L.efo_paced_schedule_ex.restype = ctypes.c_long
        L.efo_paced_schedule_ex.argtypes = [VP, VP, ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_long, ctypes.c_long, VP, VP, VP]
        L.efo_make_index.restype = ctypes.c_int
        L.efo_make_index.argtypes = [VP, ctypes.c_size_t, VP, VP, ctypes.c_int, VP, VP]
        L.efo_pts2seq.restype = ctypes.c_int
        L.efo_pts2seq.argtypes = [VP, VP, ctypes.c_int, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint32, VP, ctypes.c_int]
        L.efo_build_idx.restype = ctypes.c_size_t
        L.efo_build_idx.argtypes = [VP, VP, VP, ctypes.c_size_t]
        L.efo_demux_audio_ts.restype = ctypes.c_size_t
        L.efo_demux_audio_ts.argtypes = [VP, ctypes.c_size_t, VP, ctypes.c_size_t]
        L.efo_sbc_decode.restype = ctypes.c_long
        L.efo_sbc_bits.restype = ctypes.c_int
        L.efo_sbc_bits.argtypes = [VP, ctypes.c_size_t, VP]
        L.efo_sbc_decode.argtypes = [VP, ctypes.c_size_t, VP, ctypes.c_size_t]
        L.efo_pdm.argtypes = [VP, ctypes.c_size_t, VP]
        self._video = {}

    # -- audio (oracle/ef_oracle_audio.c) --------------------------------------------------------------
    def demux_audio_ts(self, ts):
        ts = np.ascontiguousarray(np.frombuffer(bytes(ts), dtype=np.uint8))
        es = np.empty(ts.size + 16, dtype=np.uint8)
        n = self.lib.efo_demux_audio_ts(ts.ctypes.data, ts.size, es.ctypes.data, es.size)
        return es[:n].copy()

    def sbc_decode(self, es):
        """-> PCM int16 array, or the negative code of efo_sbc_decode"""
        es = np.ascontiguousarray(np.frombuffer(bytes(es), dtype=np.uint8))
        cap = (es.size // 8 + 2) * 128
        pcm = np.zeros(cap, dtype=np.int16)
        n = self.lib.efo_sbc_decode(es.ctypes.data if es.size else pcm.ctypes.data, es.size, pcm.ctypes.data, cap)
        return int(n) if n < 0 else pcm[:n].copy()

    def sbc_bits(self, frame):
        """-> (sum of the 8 sample widths or -1 / -2, the 8 widths) of one SBC frame's header, scale factors and bit allocation"""
        d = np.ascontiguousarray(np.frombuffer(bytes(frame), dtype=np.uint8))
        buf = np.zeros(max(d.size, 1), dtype=np.uint8)
        buf[:d.size] = d
        bits = np.zeros(8, dtype=np.int32)
        total = self.lib.efo_sbc_bits(buf.ctypes.data, d.size, bits.ctypes.data)
        return int(total), [int(b) for b in bits]

    def pdm(self, pcm):
        pcm = np.ascontiguousarray(pcm, dtype=np.int16)
        out = np.zeros(2 * pcm.size, dtype=np.uint16)
        self.lib.efo_pdm(pcm.ctypes.data, pcm.size, out.ctypes.data)
        return out

    def demux_ts(self, ts):
        ts = np.ascontiguousarray(np.frombuffer(bytes(ts), dtype=np.uint8))
        es = np.empty(ts.size + 16, dtype=np.uint8)
        n = self.lib.efo_demux_ts(ts.ctypes.data, ts.size, es.ctypes.data, es.size, None, None, 0, None)
        return es[:n].copy()

    def decode_es(self, es, has_pts=True, max_frames=256):
        es = np.ascontiguousarray(np.frombuffer(bytes(es), dtype=np.uint8))
        out = np.zeros((max_frames, I420), dtype=np.uint8)
        n = self.lib.efo_decode_es(es.ctypes.data, es.size, 1 if has_pts else 0, out.ctypes.data, max_frames, None)
        assert n <= max_frames
        return out[:n]

    def decode_ts(self, ts, max_frames=256):
        ts = np.ascontiguousarray(np.frombuffer(bytes(ts), dtype=np.uint8))
        out = np.zeros((max_frames, I420), dtype=np.uint8)
        n = self.lib.efo_decode_ts(ts.ctypes.data, ts.size, out.ctypes.data, max_frames)
        assert n <= max_frames
        return out[:n]

    def idct(self, coeffs):
        b = np.ascontiguousarray(coeffs, dtype=np.int32).copy()
        self.lib.efo_idct(b.ctypes.data)
        return b

    def i420_to_strips(self, i420):
        i420 = np.ascontiguousarray(i420, dtype=np.uint8)
        out = np.zeros(FRAME, dtype=np.uint8)
        self.lib.efo_i420_to_strips(i420.ctypes.data, out.ctypes.data)
        return out

    def strips_to_i420(self, strips):
        strips = np.ascontiguousarray(strips, dtype=np.uint8)
        out = np.zeros(I420, dtype=np.uint8)
        self.lib.efo_strips_to_i420(strips.ctypes.data, out.ctypes.data)
        return out

    def video(self, ntsc):
        if ntsc not in self._video:
            v = _Video()
            self.lib.efo_video_init(ctypes.byref(v), 1 if ntsc else 0)
            self._video[ntsc] = v
        return self._video[ntsc]

    def field(self, i420, ntsc, frame_counter):
        v = self.video(ntsc)
        strips = self.i420_to_strips(i420)
        out = np.zeros(v.line_width * v.line_count, dtype=np.uint16)
        self.lib.efo_field(ctypes.byref(v), strips.ctypes.data, frame_counter, out.ctypes.data)
        return out

    def paced(self, frames, pts, ntsc, frame_counter0, max_fields, want_fields=True, modes=None, tail_fields=0, want_hscroll=False):
        """push_video + video_isr of the unmodified reference under the instant-decoder model.
        Returns (fields, flip_field[], flip_line[], field stream or None[, hscroll per field])."""
        g = self.init(ntsc)
        frames = np.ascontiguousarray(frames, dtype=np.uint8)
        pts = np.ascontiguousarray(pts, dtype=np.int64)
        n = len(pts)
        ff, fl = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.int32)
        out = np.zeros(max_fields * g[0] * g[1], dtype=np.uint16) if want_fields else None
        md = None if modes is None else np.ascontiguousarray(modes, dtype=np.int32)
        hs = np.zeros(max_fields + 1, dtype=np.int16)
        r = self.lib.efref_paced_ex(frames.ctypes.data, n, pts.ctypes.data, None if md is None else md.ctypes.data, frame_counter0, max_fields, tail_fields,
                                    out.ctypes.data if want_fields else None, ff.ctypes.data, fl.ctypes.data, hs.ctypes.data)
        assert r >= 0, "reference pacing harness timed out"
        res = (int(r), ff, fl, (out[:r * g[0] * g[1]] if want_fields else None))
        return res + (hs[:r].copy(),) if want_hscroll else res

    def field_ex(self, i420_a, i420_b, ntsc, frame_counter, hscroll=0, bitmap=None, blend=0, progress=0):
        v = self.video(ntsc)
        sa, sb = self.i420_to_strips(i420_a), self.i420_to_strips(i420_b)
        out = np.zeros(v.line_width * v.line_count, dtype=np.uint16)
        bm = None if bitmap is None else np.ascontiguousarray(bitmap, dtype=np.uint8)
        self.lib.efo_field_ex(ctypes.byref(v), sa.ctypes.data, sb.ctypes.data, frame_counter, hscroll,
                              None if bm is None else bm.ctypes.data, blend, progress, out.ctypes.data)
        return out

    def blit(self, i420, ntsc, line, x, width, frame_counter):
        v = self.video(ntsc)
        strips = self.i420_to_strips(i420)
        out = np.zeros(2 * 352 + 160, dtype=np.uint16)
        self.lib.efo_blit(ctypes.byref(v), strips.ctypes.data, out.ctypes.data, line, x, width, frame_counter)
        return out

    def coverage(self, max_pictures):
        """uint8 [pictures, 264]: the macroblocks (row * 22 + column) each of the first pictures of the last decode wrote: 2 from
        its own codes, 1 by a skip's copy, 0 not at all"""
        out = np.zeros((8, 264), dtype=np.uint8)
        n = self.lib.efo_coverage(out.ctypes.data, min(max_pictures, 8))
        return out[:min(n, max_pictures, 8)].copy()

    def walk(self, es):
        """the markers the decoder's marker walk dispatches on an ES: ([(bit position of the prefix, code)], (pictures, slices,
        sequence headers))"""
        es = np.frombuffer(bytes(es), dtype=np.uint8) if isinstance(es, (bytes, bytearray)) else np.ascontiguousarray(es, dtype=np.uint8)
        cap = es.size // 3 + 8                              # a marker takes at least 3 bytes, the padding adds 2
        pos, code = np.zeros(cap, np.uint64), np.zeros(cap, np.uint8)
        counts = np.zeros(3, np.int64)
        n = self.lib.efo_walk(es.ctypes.data, es.size, pos.ctypes.data, code.ctypes.data, cap, counts.ctypes.data)
        assert n <= cap
        return [(int(p), int(c)) for p, c in zip(pos[:n], code[:n])], tuple(int(x) for x in counts)

    def stats_reset(self):
        self.lib.efo_stats_reset()

    def stats(self):
        s = _Stats()
        self.lib.efo_stats_get(ctypes.byref(s))
        return s

    def paced_schedule(self, pts, ntsc, frame_counter0, max_fields=1 << 20, modes=None, tail_fields=0, want_hscroll=False):
        """push_video pacing, instant-decoder model: (fields, flip_field[], flip_line[][, hscroll per field])"""
        pts = np.ascontiguousarray(pts, dtype=np.int64)
        ff, fl = np.zeros(len(pts), dtype=np.uint32), np.zeros(len(pts), dtype=np.int32)
        md = None if modes is None else np.ascontiguousarray(modes, dtype=np.int32)
        hs = np.zeros(min(max_fields, 1 << 16) + 1, dtype=np.int16)
        n = self.lib.efo_paced_schedule_ex(pts.ctypes.data, None if md is None else md.ctypes.data, len(pts), 1 if ntsc else 0, frame_counter0,
                                           min(max_fields, 1 << 16), tail_fields, ff.ctypes.data, fl.ctypes.data, hs.ctypes.data)
        return (int(n), ff, fl, hs[:n].copy()) if want_hscroll else (int(n), ff, fl)

    # -- trick-mode index (indexer/indexer.cpp) ----------------------------------------------------------
    def make_index(self, ts):
        ts = np.ascontiguousarray(np.frombuffer(bytes(ts), dtype=np.uint8))
        cap = ts.size // 188 + 1
        pts, pos = np.zeros(cap, dtype=np.int64), np.zeros(cap, dtype=np.uint32)
        first, last = ctypes.c_int64(), ctypes.c_int64()
        n = self.lib.efo_make_index(ts.ctypes.data, ts.size, pts.ctypes.data, pos.ctypes.data, cap, ctypes.byref(first), ctypes.byref(last))
        return {"first_pts": first.value, "last_pts": last.value, "seq_pts": pts[:n].copy(), "seq_pos": pos[:n].copy()}

    def pts2seq(self, seq_pts, seq_pos, first_pts, last_pts, bin_size):
        seq_pts = np.ascontiguousarray(seq_pts, dtype=np.int64)
        seq_pos = np.ascontiguousarray(seq_pos, dtype=np.uint32)
        n = self.lib.efo_pts2seq(seq_pts.ctypes.data, seq_pos.ctypes.data, len(seq_pts), first_pts, last_pts, bin_size, None, 0)
        out = np.zeros(max(n, 1), dtype=np.uint32)
        self.lib.efo_pts2seq(seq_pts.ctypes.data, seq_pos.ctypes.data, len(seq_pts), first_pts, last_pts, bin_size, out.ctypes.data, n)
        return out[:n].copy()

    def build_idx(self, files):
        bufs = [np.ascontiguousarray(np.frombuffer(bytes(f), dtype=np.uint8)) for f in files]
        ptrs = (ctypes.c_void_p * 3)(*[b.ctypes.data for b in bufs])
        lens = (ctypes.c_size_t * 3)(*[b.size for b in bufs])
        cap = 104 + 4 * sum(b.size // 188 + 2 for b in bufs) + (1 << 22)
        out = np.zeros(cap, dtype=np.uint8)
        n = self.lib.efo_build_idx(ptrs, lens, out.ctypes.data, cap)
        assert n
        return out[:n].tobytes()


def have_ref():
    return os.path.exists(REF_DECODE) and os.path.exists(REF_VIDEO)


def ref_decode_ts(ts, loops=1, dump=True, timeout=300):
    """Run the UNMODIFIED reference decoder (oracle/_ref/efref_decode, one process per call, Q11)."""
    with tempfile.TemporaryDirectory() as d:
        tin, tout = os.path.join(d, "in.ts"), os.path.join(d, "out.i420")
        with open(tin, "wb") as f:
            f.write(bytes(ts))
        r = subprocess.run([REF_DECODE, tin, tout if dump else "-", str(loops)], capture_output=True, timeout=timeout, check=True)
        info = json.loads(r.stdout)
        frames = np.fromfile(tout, dtype=np.uint8).reshape(-1, I420) if dump else None
        return info, frames


class RefVideo:
    """The UNMODIFIED reference composite code (oracle/_ref/libefref_vid.so)."""

    def __init__(self):
        self.lib = ctypes.CDLL(REF_VIDEO)
        VP = ctypes.c_void_p
        self.lib.efref_field.restype = ctypes.c_long
        self.lib.efref_field.argtypes = [VP, VP, ctypes.c_int, ctypes.c_int, VP]
        self.lib.efref_blit.argtypes = [VP, ctypes.c_int, VP, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        self.lib.efref_field_ex.restype = ctypes.c_long
        self.lib.efref_field_ex.argtypes = [VP, VP, ctypes.c_int, ctypes.c_int, VP, ctypes.c_int, ctypes.c_int, VP]
        self.lib.efref_paced.restype = ctypes.c_long
        self.lib.efref_paced.argtypes = [VP, ctypes.c_int, VP, VP, ctypes.c_int, ctypes.c_int, VP, VP, VP]
        self.lib.efref_paced_ex.restype = ctypes.c_long
        self.lib.efref_paced_ex.argtypes = [VP, ctypes.c_int, VP, VP, ctypes.c_int, ctypes.c_int, ctypes.c_int, VP, VP, VP, VP]
        self.std = None

    def init(self, ntsc):
        if self.std != ntsc:
            self.lib.efref_video_init(1 if ntsc else 0)
            self.std = ntsc
        g = (ctypes.c_int * 8)()
        self.lib.efref_geometry(g)
        return list(g)

    def field(self, i420, ntsc, frame_counter):
        g = self.init(ntsc)
        i420 = np.ascontiguousarray(i420, dtype=np.uint8)
        out = np.zeros(g[0] * g[1], dtype=np.uint16)
        self.lib.efref_field(i420.ctypes.data, None, frame_counter, 0, out.ctypes.data)
        return out

    def paced(self, frames, pts, ntsc, frame_counter0, max_fields, want_fields=True, modes=None, tail_fields=0, want_hscroll=False):
        """push_video + video_isr of the unmodified reference under the instant-decoder model.
        Returns (fields, flip_field[], flip_line[], field stream or None[, hscroll per field])."""
        g = self.init(ntsc)
        frames = np.ascontiguousarray(frames, dtype=np.uint8)
        pts = np.ascontiguousarray(pts, dtype=np.int64)
        n = len(pts)
        ff, fl = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.int32)
        out = np.zeros(max_fields * g[0] * g[1], dtype=np.uint16) if want_fields else None
        md = None if modes is None else np.ascontiguousarray(modes, dtype=np.int32)
        hs = np.zeros(max_fields + 1, dtype=np.int16)
        r = self.lib.efref_paced_ex(frames.ctypes.data, n, pts.ctypes.data, None if md is None else md.ctypes.data, frame_counter0, max_fields, tail_fields,
                                    out.ctypes.data if want_fields else None, ff.ctypes.data, fl.ctypes.data, hs.ctypes.data)
        assert r >= 0, "reference pacing harness timed out"
        res = (int(r), ff, fl, (out[:r * g[0] * g[1]] if want_fields else None))
        return res + (hs[:r].copy(),) if want_hscroll else res

    def field_ex(self, i420_a, i420_b, ntsc, frame_counter, hscroll=0, bitmap=None, blend=0, progress=0):
        g = self.init(ntsc)
        a = np.ascontiguousarray(i420_a, dtype=np.uint8)
        b = np.ascontiguousarray(i420_b, dtype=np.uint8)
        bm = None if bitmap is None else np.ascontiguousarray(bitmap, dtype=np.uint8)
        out = np.zeros(g[0] * g[1], dtype=np.uint16)
        self.lib.efref_field_ex(a.ctypes.data, b.ctypes.data, frame_counter, hscroll, None if bm is None else bm.ctypes.data, blend, progress, out.ctypes.data)
        return out

    def blit(self, i420, ntsc, line, x, width, frame_counter):
        self.init(ntsc)
        i420 = np.ascontiguousarray(i420, dtype=np.uint8)
        out = np.zeros(2 * 352 + 160, dtype=np.uint16)
        self.lib.efref_blit(i420.ctypes.data, frame_counter, out.ctypes.data, line, x, width)
        return out


def have_ref_index():
    return os.path.exists(REF_INDEX)


class RefIndexer:
    """The UNMODIFIED reference index builder (oracle/_ref/libefref_idx.so; indexer/indexer.cpp)."""

    def __init__(self):
        self.lib = ctypes.CDLL(REF_INDEX)
        VP = ctypes.c_void_p
        self.lib.efref_make_index.restype = ctypes.c_int
        self.lib.efref_make_index.argtypes = [ctypes.c_char_p, VP, VP, ctypes.c_int, VP, VP]
        self.lib.efref_build_idx.argtypes = [ctypes.c_char_p] * 4

    def make_index(self, ts):
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "in.ts")
            open(p, "wb").write(bytes(ts))
            cap = len(bytes(ts)) // 188 + 1
            pts, pos = np.zeros(cap, dtype=np.int64), np.zeros(cap, dtype=np.uint32)
            first, last = ctypes.c_int64(), ctypes.c_int64()
            n = self.lib.efref_make_index(p.encode(), pts.ctypes.data, pos.ctypes.data, cap, ctypes.byref(first), ctypes.byref(last))
            return {"first_pts": first.value, "last_pts": last.value, "seq_pts": pts[:n].copy(), "seq_pos": pos[:n].copy()}

    def build_idx(self, files):
        """video.idx as the reference tool writes it, padding bytes zeroed."""
        with tempfile.TemporaryDirectory() as d:
            paths = []
            for k, f in enumerate(files):
                paths.append(os.path.join(d, "s%d.ts" % k))
                open(paths[-1], "wb").write(bytes(f))
            self.lib.efref_build_idx(paths[0].encode(), paths[1].encode(), paths[2].encode(), d.encode())
            img = bytearray(open(os.path.join(d, "video.idx"), "rb").read())
            for b in IDX_PAD:
                img[b] = 0
            return bytes(img)
