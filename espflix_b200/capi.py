"""espflix_b200/capi.py — ctypes binding of include/espflix_b200.h. Fails loudly when the CUDA
library is missing or no GPU is present: there is no CPU path in the product."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
FRAME_BYTES = 101376
I420_BYTES = 101376
EF_OK, EF_EINVAL, EF_ECUDA, EF_ENOMEM, EF_ESTATE = 0, -1, -2, -3, -4


class EspflixError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("espflix_b200 error %d: %s" % (code, msg))
        self.code = code


class _Config(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int), ("n_streams", ctypes.c_int), ("max_pictures", ctypes.c_int),
                ("max_slices_per_picture", ctypes.c_int), ("es_capacity", ctypes.c_size_t), ("fields", ctypes.c_int)]


def lib_path():
    """The CUDA library. EF_LIB (a file name inside the package directory, or an absolute path) selects a tuning
    variant built by espflix_b200.build.build_variant(); the product is always libespflix_b200.so."""
    override = os.environ.get("EF_LIB")
    if override:
        return override if os.path.isabs(override) else os.path.join(_HERE, override)
    return os.path.join(_HERE, "libespflix_b200.so")


_lib = None
_VP, _I, _U64P = ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)

_SIGNATURES = {
    "ef_last_error": (ctypes.c_char_p, []),
    "ef_version": (ctypes.c_char_p, []),
    "ef_create": (_I, [ctypes.POINTER(_VP), ctypes.POINTER(_Config)]),
    "ef_destroy": (None, [_VP]),
    "ef_reset": (_I, [_VP]),
    "ef_submit_es_host": (_I, [_VP, _VP, _VP, _VP]),
    "ef_submit_es_device": (_I, [_VP, _VP, _VP, _VP]),
    "ef_submit_ts_host": (_I, [_VP, _VP, _VP, _VP]),
    "ef_submit_ts_device": (_I, [_VP, _VP, _VP, _VP]),
    "ef_index": (_I, [_VP, _VP]),
    "ef_index_info": (_I, [_VP, ctypes.POINTER(_I), _U64P, _U64P, _U64P]),
    "ef_stream_info": (_I, [_VP, _I, ctypes.POINTER(_I), ctypes.POINTER(_I)]),
    "ef_decode_picture": (_I, [_VP, _I, _VP]),
    "ef_decode_all": (_I, [_VP, _I, _VP]),
    "ef_decode_all_to_host": (_I, [_VP, _I, _VP, _I, _VP]),
    "ef_read_frame": (_I, [_VP, _I, _I, _VP]),
    "ef_read_frame_i420": (_I, [_VP, _I, _I, _VP]),
    "ef_write_frame_i420": (_I, [_VP, _I, _I, _VP]),
    "ef_write_frame": (_I, [_VP, _I, _I, _VP]),
    "ef_frame_device_ptr": (_I, [_VP, _I, _I, ctypes.POINTER(_VP)]),
    "ef_read_latest_i420": (_I, [_VP, _I, _I, _VP, _VP]),
    "ef_read_latest_i420_async": (_I, [_VP, _I, _I, _VP, _VP]),
    "ef_sync": (_I, [_VP, _VP]),
    "ef_video_init": (_I, [_VP, _I]),
    "ef_video_geometry": (_I, [_VP, ctypes.POINTER(_I), ctypes.POINTER(_I)]),
    "ef_composite_field": (_I, [_VP, _I, _I, _VP]),
    "ef_video_set_scroll": (_I, [_VP, _I]),
    "ef_video_set_overlay": (_I, [_VP, _VP, _I, _I]),
    "ef_read_field": (_I, [_VP, _I, _VP]),
    "ef_video_isr": (_I, [_VP, _I, _I, _VP]),
    "ef_blit": (_I, [_VP, _I, _I, _VP, _I, _I, _I, _I]),
    "ef_launch_count": (ctypes.c_uint64, [_VP]),
    "ef_host_alloc": (_I, [ctypes.POINTER(_VP), ctypes.c_size_t]),
    "ef_host_free": (None, [_VP]),
    "ef_set_profiling": (_I, [_VP, _I]),
    "ef_stage_ms": (_I, [_VP, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]),
    "ef_tsidx_scan": (_I, [_I, _VP, _VP, _I, ctypes.c_uint32, _VP, _VP, _VP]),
    "ef_idct_tc_run": (_I, [_I, _VP, _I, _VP, _VP, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), _I]),
    "ef_audio_demux_ts": (_I, [_I, _VP, _VP, _I, _VP, ctypes.c_uint64, _VP]),
    "ef_audio_decode": (_I, [_I, _VP, _VP, _I, _VP, _VP, ctypes.c_uint64, _VP]),
    "ef_audio_enable": (_I, [_VP]),
    "ef_decode_audio": (_I, [_VP, _VP, _VP, _VP, ctypes.c_uint64, _VP, _VP]),
    "ef_pts_enable": (_I, [_VP]),
    "ef_picture_pts": (_I, [_VP, _I, _I, _I, _VP, _VP]),
    "ef_tsidx_samples": (_I, [_I, _VP, _VP, _I, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint32, _VP, ctypes.c_uint32, _VP]),
}


def load_library():
    """Load libespflix_b200.so (built in-tree by __graft_entry__.build()). Raises if absent."""
    global _lib
    if _lib is None:
        p = lib_path()
        if not os.path.exists(p):
            raise EspflixError(EF_ECUDA, "CUDA library %s is not built (run __graft_entry__.build()); no CPU fallback exists" % p)
        lib = ctypes.CDLL(p)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data
    return int(a)          # raw (device) address


class Context:
    """One GPU's worth of independent decoders (see include/espflix_b200.h)."""

    def __init__(self, n_streams, max_pictures=12, max_slices_per_picture=12, es_capacity=None, device=0, fields=True):
        self.lib = load_library()
        if es_capacity is None:
            es_capacity = n_streams * max_pictures * 32768
        cfg = _Config(device, n_streams, max_pictures, max_slices_per_picture, es_capacity, 1 if fields else 0)
        self._h = _VP()
        self.n_streams, self.max_pictures = n_streams, max_pictures
        self._check(self.lib.ef_create(ctypes.byref(self._h), ctypes.byref(cfg)))

    def _check(self, rc):
        if rc != EF_OK:
            raise EspflixError(rc, self.lib.ef_last_error().decode("utf-8", "replace"))

    def close(self):
        if self._h:
            self.lib.ef_destroy(self._h)
            self._h = _VP()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self._check(self.lib.ef_reset(self._h))

    # -- submit -----------------------------------------------------------------------------
    @staticmethod
    def pack(streams):
        """list of bytes-like -> (blob uint8 array, offsets uint64 array)"""
        off = np.zeros(len(streams) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(s) for s in streams])
        blob = np.frombuffer(b"".join(bytes(s) for s in streams), dtype=np.uint8).copy() if int(off[-1]) else np.zeros(1, np.uint8)
        return blob, off

    def submit_es(self, blob, off, stream=0, device=False):
        fn = self.lib.ef_submit_es_device if device else self.lib.ef_submit_es_host
        self._check(fn(self._h, _ptr(blob), _ptr(off), stream))

    def submit_ts(self, blob, off, stream=0, device=False):
        fn = self.lib.ef_submit_ts_device if device else self.lib.ef_submit_ts_host
        self._check(fn(self._h, _ptr(blob), _ptr(off), stream))

    def index(self, stream=0):
        self._check(self.lib.ef_index(self._h, stream))

    def index_info(self):
        mp, tp, ts, eb = _I(), ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
        self._check(self.lib.ef_index_info(self._h, ctypes.byref(mp), ctypes.byref(tp), ctypes.byref(ts), ctypes.byref(eb)))
        return {"max_pictures": mp.value, "total_pictures": tp.value, "total_slices": ts.value, "es_bytes": eb.value}

    def stream_info(self, s):
        a, b = _I(), _I()
        self._check(self.lib.ef_stream_info(self._h, s, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    # -- decode -----------------------------------------------------------------------------
    def decode_picture(self, pic, stream=0):
        self._check(self.lib.ef_decode_picture(self._h, pic, stream))

    def decode_all(self, n_pictures, stream=0):
        self._check(self.lib.ef_decode_all(self._h, n_pictures, stream))

    def decode_all_to_host(self, n_pictures, out, stream=0, strips=False):
        """every picture of the submit to out[n_pictures][n_streams][I420 or strips] (pinned host memory; complete after sync())"""
        self._check(self.lib.ef_decode_all_to_host(self._h, n_pictures, _ptr(out), 1 if strips else 0, stream))

    def read_frame(self, s, fb=-1):
        out = np.empty(FRAME_BYTES, dtype=np.uint8)
        self._check(self.lib.ef_read_frame(self._h, s, fb, out.ctypes.data))
        return out

    def read_frame_i420(self, s, fb=-1):
        out = np.empty(I420_BYTES, dtype=np.uint8)
        self._check(self.lib.ef_read_frame_i420(self._h, s, fb, out.ctypes.data))
        return out

    def write_frame_i420(self, s, fb, data):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        assert data.size == I420_BYTES
        self._check(self.lib.ef_write_frame_i420(self._h, s, fb, data.ctypes.data))

    def read_latest_i420(self, first=0, count=None, out=None, stream=0):
        count = self.n_streams - first if count is None else count
        if out is None:
            out = np.empty((count, I420_BYTES), dtype=np.uint8)
        self._check(self.lib.ef_read_latest_i420(self._h, first, count, _ptr(out), stream))
        return out

    def read_latest_i420_async(self, first, count, out, stream=0):
        self._check(self.lib.ef_read_latest_i420_async(self._h, first, count, _ptr(out), stream))

    def sync(self, stream=0):
        self._check(self.lib.ef_sync(self._h, stream))

    def frame_device_ptr(self, s, fb):
        p = _VP()
        self._check(self.lib.ef_frame_device_ptr(self._h, s, fb, ctypes.byref(p)))
        return p.value

    def decode_sequence(self, streams, ts=False):
        """Convenience used by the parity tests: submit, index, then decode picture by picture,
        returning for every stream the list of I420 frames in presentation (push_video) order."""
        blob, off = self.pack(streams)
        (self.submit_ts if ts else self.submit_es)(blob, off)
        self.index()
        info = self.index_info()
        frames = [[] for _ in streams]
        counts = [self.stream_info(i)[0] for i in range(len(streams))]
        for p in range(info["max_pictures"]):
            self.decode_picture(p)
            for i in range(len(streams)):
                if p < counts[i]:
                    base = self.stream_info(i)[1]
                    frames[i].append(self.read_frame_i420(i, (base + p + 1) & 1))
        return frames

    # -- composite --------------------------------------------------------------------------
    def video_init(self, ntsc):
        self._check(self.lib.ef_video_init(self._h, 1 if ntsc else 0))

    def geometry(self):
        w, n = _I(), _I()
        self._check(self.lib.ef_video_geometry(self._h, ctypes.byref(w), ctypes.byref(n)))
        return w.value, n.value

    def composite_field(self, fb=-1, frame_counter=0, stream=0):
        self._check(self.lib.ef_composite_field(self._h, fb, frame_counter, stream))

    def set_scroll(self, hscroll):
        self._check(self.lib.ef_video_set_scroll(self._h, hscroll))

    def set_overlay(self, bitmap, blend, progress):
        if bitmap is not None:
            bitmap = np.ascontiguousarray(bitmap, dtype=np.uint8)
            assert bitmap.size == 1280
        self._check(self.lib.ef_video_set_overlay(self._h, _ptr(bitmap), blend, progress))

    def read_field(self, s):
        w, n = self.geometry()
        out = np.empty(w * n, dtype=np.uint16)
        self._check(self.lib.ef_read_field(self._h, s, out.ctypes.data))
        return out

    def video_isr(self, s, line):
        w, _ = self.geometry()
        out = np.empty(w, dtype=np.uint16)
        self._check(self.lib.ef_video_isr(self._h, s, line, out.ctypes.data))
        return out

    def blit(self, s, fb, line, x, width, frame_counter, dst=None):
        if dst is None:
            dst = np.zeros(2 * 352 + 160, dtype=np.uint16)
        self._check(self.lib.ef_blit(self._h, s, fb, dst.ctypes.data, line, x, width, frame_counter))
        return dst

    # -- audio ------------------------------------------------------------------------------
    def enable_audio(self):
        """from now on every TS submit also demuxes the stream's audio (PID 0x101 / 0x102)"""
        self._check(self.lib.ef_audio_enable(self._h))

    def decode_audio(self, end=None, pdm=True, pcm_out=None, pdm_out=None, stream=0):
        """ef_decode_audio: the frames of every stream that became decodable with the current submit -> list of dicts as
        audio_decode() (frame_size, n_frames, pcm, pdm). end: per-stream flags (or True for all) that end the stream after
        this call. pcm_out / pdm_out: preallocated (pinned) int16 / uint16 arrays large enough for the call; without them
        a sizing call comes first."""
        n = self.n_streams
        if end is True:
            end = np.ones(n, dtype=np.uint8)
        elif end is not None:
            end = np.ascontiguousarray(end, dtype=np.uint8)
            assert end.size == n
        info = np.zeros(n, dtype=_AUDIO_INFO)
        if pcm_out is None:
            self._check(self.lib.ef_decode_audio(self._h, _ptr(end), info.ctypes.data, None, 0, None, stream))
            total = int(info["n_frames"].sum()) * 128
            pcm_out = np.zeros(max(total, 1), dtype=np.int16)
            pdm_out = np.zeros(max(2 * total, 1), dtype=np.uint16) if pdm else None
        elif not pdm:
            pdm_out = None
        self._check(self.lib.ef_decode_audio(self._h, _ptr(end), info.ctypes.data, _ptr(pcm_out), pcm_out.size, _ptr(pdm_out), stream))
        out = []
        for i in info:
            a, k = int(i["pcm_offset"]), int(i["n_frames"]) * 128
            out.append({"frame_size": int(i["frame_size"]), "n_frames": int(i["n_frames"]), "pcm": pcm_out[a:a + k].copy(),
                        "pdm": None if pdm_out is None else pdm_out[2 * a:2 * (a + k)].copy()})
        return out

    # -- presentation timestamps -----------------------------------------------------------------
    def enable_pts(self):
        """from now on every TS submit also lists its video PES starts, and every index() resolves the pts of every picture"""
        self._check(self.lib.ef_pts_enable(self._h))

    def picture_pts(self, first=0, count=None, n_pictures=None):
        """ef_picture_pts for the submit the last index() made current -> (int64[count, n_pictures] pts of every picture, -1
        past a stream's pictures; int64[count] pts of every stream's most recent picture over all submits, get_pts())"""
        count = self.n_streams - first if count is None else count
        n_pictures = self.max_pictures if n_pictures is None else n_pictures
        pic = np.full((max(count, 0), n_pictures), -1, dtype=np.int64)
        last = np.full(max(count, 0), -1, dtype=np.int64)
        self._check(self.lib.ef_picture_pts(self._h, first, count, n_pictures, _ptr(pic) if pic.size else None, _ptr(last) if last.size else None))
        return pic, last

    def launch_count(self):
        return int(self.lib.ef_launch_count(self._h))

    def set_profiling(self, on=True):
        self._check(self.lib.ef_set_profiling(self._h, 1 if on else 0))

    def stage_ms(self):
        """(K0 index, K1a parse, K1b reconstruction) milliseconds of the last ef_index / ef_decode_* (synchronises)."""
        a, b, c = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.ef_stage_ms(self._h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
        return a.value, b.value, c.value


# -- trick-mode index (indexer/indexer.cpp; SURVEY.md 8f-4) ---------------------------------------------
IDX_BIN = 90000 // 12            # merge_index(): one sample per 1/12 s
_TSIDX_INFO = np.dtype([("first_pts", "<i8"), ("last_pts", "<i8"), ("n_seq", "<u4"), ("n_samples", "<u4")])


def _check_rc(lib, rc):
    if rc != 0:
        raise EspflixError(rc, lib.ef_last_error().decode("utf-8", "replace"))


def tsidx_scan(files, bin_size=IDX_BIN, device=0):
    """make_index() for a list of transport streams (bytes-like, lengths multiples of 188). Returns one dict per
    file: first_pts, last_pts, seq_pts (int64 array), seq_pos (uint32 array), n_samples."""
    lib = load_library()
    blob, off = Context.pack(files)
    n_packets = int(off[-1]) // 188
    info = np.zeros(len(files), dtype=_TSIDX_INFO)
    spts = np.zeros(max(n_packets, 1), dtype=np.int64)
    spos = np.zeros(max(n_packets, 1), dtype=np.uint32)
    blob = np.ascontiguousarray(blob)
    _check_rc(lib, lib.ef_tsidx_scan(device, blob.ctypes.data if blob.size else spts.ctypes.data, off.ctypes.data, len(files), bin_size,
                                     info.ctypes.data, spts.ctypes.data, spos.ctypes.data))
    out = []
    for f in range(len(files)):
        p0, n = int(off[f]) // 188, int(info[f]["n_seq"])
        out.append({"first_pts": int(info[f]["first_pts"]), "last_pts": int(info[f]["last_pts"]), "n_samples": int(info[f]["n_samples"]),
                    "seq_pts": spts[p0:p0 + n].copy(), "seq_pos": spos[p0:p0 + n].copy()})
    return out


def tsidx_samples(seq_pts, seq_pos, first_pts, last_pts, bin_size=IDX_BIN, device=0):
    """pts2seq(): uint32 packet number per bin."""
    lib = load_library()
    seq_pts = np.ascontiguousarray(seq_pts, dtype=np.int64)
    seq_pos = np.ascontiguousarray(seq_pos, dtype=np.uint32)
    n = ctypes.c_uint32(0)
    cap = 0 if len(seq_pts) == 0 or last_pts < first_pts else (last_pts - first_pts) // bin_size + 1
    out = np.zeros(max(cap, 1), dtype=np.uint32)
    _check_rc(lib, lib.ef_tsidx_samples(device, seq_pts.ctypes.data, seq_pos.ctypes.data, len(seq_pts), first_pts, last_pts, bin_size,
                                        out.ctypes.data, cap, ctypes.byref(n)))
    return out[:n.value].copy()


def idct_tc_run(coefs, L, repeats=5, device=0):
    """The tensor-core (wgmma) IDCT experiment (include/espflix_b200.h): coefs int32 [n][64], L float64 [64][64] -> (out int32 [n][64], prep_ms, mma_ms)"""
    lib = load_library()
    coefs = np.ascontiguousarray(coefs, dtype=np.int32)
    L = np.ascontiguousarray(L, dtype=np.float64)
    out = np.zeros_like(coefs)
    a, b = ctypes.c_float(), ctypes.c_float()
    _check_rc(lib, lib.ef_idct_tc_run(device, coefs.ctypes.data, coefs.shape[0], L.ctypes.data, out.ctypes.data, ctypes.byref(a), ctypes.byref(b), repeats))
    return out, a.value, b.value


# -- audio (src/sbc_decoder.cpp, espflix.ino pdm_second_order; SURVEY.md 8f-3) ------------------------------------------
_AUDIO_INFO = np.dtype([("frame_size", "<i4"), ("n_frames", "<u4"), ("pcm_offset", "<u8")])


def audio_demux_ts(files, device=0):
    """The bytes push_audio() receives (PID 0x101 / 0x102) for a list of transport streams -> list of uint8 arrays."""
    lib = load_library()
    blob, off = Context.pack(files)
    es = np.zeros(max(int(off[-1]), 1), dtype=np.uint8)
    es_off = np.zeros(len(files) + 1, dtype=np.uint64)
    _check_rc(lib, lib.ef_audio_demux_ts(device, blob.ctypes.data, off.ctypes.data, len(files), es.ctypes.data, es.size, es_off.ctypes.data))
    return [es[int(es_off[i]):int(es_off[i + 1])].copy() for i in range(len(files))]


def audio_decode(streams, pdm=True, device=0):
    """decode_audio() for a list of SBC byte streams -> list of dicts: frame_size, n_frames, pcm (int16), pdm (uint16 or None)."""
    lib = load_library()
    blob, off = Context.pack(streams)
    info = np.zeros(len(streams), dtype=_AUDIO_INFO)
    _check_rc(lib, lib.ef_audio_decode(device, blob.ctypes.data, off.ctypes.data, len(streams), info.ctypes.data, None, 0, None))
    n = int(sum(int(i["n_frames"]) for i in info)) * 128
    pcm = np.zeros(max(n, 1), dtype=np.int16)
    pd = np.zeros(max(2 * n, 1), dtype=np.uint16) if pdm else None
    _check_rc(lib, lib.ef_audio_decode(device, blob.ctypes.data, off.ctypes.data, len(streams), info.ctypes.data, pcm.ctypes.data, pcm.size,
                                       None if pd is None else pd.ctypes.data))
    out = []
    for i in info:
        a, k = int(i["pcm_offset"]), int(i["n_frames"]) * 128
        out.append({"frame_size": int(i["frame_size"]), "n_frames": int(i["n_frames"]), "pcm": pcm[a:a + k].copy(),
                    "pdm": None if pd is None else pd[2 * a:2 * (a + k)].copy()})
    return out


def build_video_idx(video_ts, fwd_ts, rev_ts, device=0):
    """merge_index(): the video.idx image (header + three sample arrays) for main / fast-forward / rewind
    streams; struct padding is zero (the reference leaves it indeterminate)."""
    recs = tsidx_scan([video_ts, fwd_ts, rev_ts], IDX_BIN, device)
    hdr = bytearray(104)
    hdr[0:8] = np.array([ord("I") | (ord("D") << 8) | (ord("X") << 16), 3], dtype="<u4").tobytes()
    body = b""
    for k, r in enumerate(recs):
        smp = tsidx_samples(r["seq_pts"], r["seq_pos"], r["first_pts"], r["last_pts"], IDX_BIN, device)
        o = 8 + 32 * k
        hdr[o:o + 16] = np.array([r["first_pts"], r["last_pts"]], dtype="<i8").tobytes()
        hdr[o + 16:o + 28] = np.array([IDX_BIN, 1 if k == 0 else 15, len(smp)], dtype="<u4").tobytes()
        body += smp.astype("<u4").tobytes()
    return bytes(hdr) + body
