"""espflix_b200/capi.py — ctypes binding of include/espflix_b200.h. Fails loudly when the CUDA
library is missing or no GPU is present: there is no CPU path in the product."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
FRAME_BYTES = 101376
I420_BYTES = 101376
EF_OK, EF_EINVAL, EF_ECUDA, EF_ENOMEM, EF_ESTATE = 0, -1, -2, -3, -4
EF_FIELD_U16, EF_FIELD_DAC8 = 0, 1          # ef_present_format: the uint16 DMA line buffer, or the bytes the video DAC plays


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
    "ef_decode_audio_async": (_I, [_VP, _VP, _VP, _VP, ctypes.c_uint64, _VP, _VP]),
    "ef_audio_wait": (_I, [_VP]),
    "ef_pts_enable": (_I, [_VP]),
    "ef_picture_pts": (_I, [_VP, _I, _I, _I, _VP, _VP]),
    "ef_present_enable": (_I, [_VP, _VP]),
    "ef_present_picture": (_I, [_VP, _I, _VP, _VP, ctypes.c_uint64, _VP, _VP]),
    "ef_present_idle": (_I, [_VP, _VP, _VP, ctypes.c_uint64, _VP, _VP]),
    "ef_present_picture_async": (_I, [_VP, _I, _VP, _VP, ctypes.c_uint64, _VP, _VP]),
    "ef_present_idle_async": (_I, [_VP, _VP, _VP, ctypes.c_uint64, _VP, _VP]),
    "ef_present_wait": (_I, [_VP, ctypes.POINTER(_I)]),
    "ef_present_format": (_I, [_VP, _I]),
    "ef_present_overlay": (_I, [_VP, _I, _I, _VP, _VP, _VP, _VP]),
    "ef_present_font": (_I, [_VP, _VP, _VP, _I]),
    "ef_present_clock": (_I, [_VP, _I, _I, _VP, _VP, _VP]),
    "ef_restart_streams": (_I, [_VP, _I, _I, _VP]),
    "ef_carry_enable": (_I, [_VP, ctypes.c_uint32]),
    "ef_end_streams": (_I, [_VP, _I, _I, _VP]),
    "ef_carry_info": (_I, [_VP, _I, _I, _VP, _VP]),
    "ef_tsidx_samples": (_I, [_I, _VP, _VP, _I, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint32, _VP, ctypes.c_uint32, _VP]),
    "ef_library_add": (_I, [_VP, _VP, ctypes.c_uint64, _VP, _VP, ctypes.POINTER(_I)]),
    "ef_library_command": (_I, [_VP, _I, _I, _I, _I, ctypes.c_int64]),
    "ef_library_submit": (_I, [_VP, ctypes.c_uint32, _VP, _VP]),
    "ef_library_info": (_I, [_VP, _I, _I, _VP]),
    "ef_trick_build": (_I, [_I, _VP, _VP, _I, _I, _VP, ctypes.c_uint64, _VP, _VP, ctypes.c_uint64, _VP]),
    "ef_trick_stage_ms": (_I, [ctypes.POINTER(ctypes.c_float)] * 4),
    "ef_library_add_trick": (_I, [_VP, _I, _I]),
    "ef_library_read": (_I, [_VP, _I, _I, _VP, ctypes.c_uint64, _U64P]),
    "ef_library_add_poster": (_I, [_VP, _I, _VP, ctypes.c_uint64]),
    "ef_library_nv_read": (_I, [_VP, _I, _I, _I, _VP]),
    "ef_library_nv_write": (_I, [_VP, _I, _I, _I, _VP]),
    "ef_library_keys": (_I, [_VP, _VP, _VP, _VP]),
    "ef_encode_build": (_I, [_I, _VP, _VP, _I, _VP, _VP, ctypes.c_uint64, _VP]),
    "ef_encode_stage_ms": (_I, [ctypes.POINTER(ctypes.c_float)] * 5),
    "ef_encode_build_rate": (_I, [_I, _VP, _VP, _I, _VP, _VP, _VP, ctypes.c_uint64, _VP, _VP, _VP]),
    "ef_sbc_encode": (_I, [_I, _VP, _VP, _I, _VP, _VP, ctypes.c_uint64, _VP]),
    "ef_mux_audio": (_I, [_I, _VP, _VP, _VP, _VP, _I, _VP, _VP, ctypes.c_uint64, _VP]),
    "ef_audio_encode_stage_ms": (_I, [ctypes.POINTER(ctypes.c_float)] * 4),
}

# ef_library_command's commands and ef_library_info's stream states (include/espflix_b200.h)
LIB_PLAY_AT, LIB_PLAY, LIB_SKIP, LIB_FAST_FORWARD, LIB_REWIND, LIB_PAUSE, LIB_RESUME, LIB_STOP, LIB_NAV, LIB_NAV_STEP, LIB_MENU = range(11)
LIB_IDLE, LIB_PLAYING, LIB_PAUSED, LIB_STOPPED, LIB_ENDED, LIB_POSTER = range(6)
LIB_POSTER_FILE = 3              # ef_library_status.file of a stream on its poster, ef_library_read's part for poster.ts
# ef_library_keys: the remote's keys (the HID codes of the reference's key_event()) and the done codes it reports
KEY_MENU, KEY_PLAY, KEY_SELECT, KEY_RIGHT, KEY_LEFT, KEY_DOWN, KEY_UP = 16, 19, 40, 79, 80, 81, 82
KEY_DONE_NOTHING, KEY_DONE_ENDED = 0x0F, 0x10
LIBRARY_STATUS = np.dtype([("title", "<i4"), ("speed", "<i4"), ("state", "<i4"), ("file", "<i4"), ("cursor", "<u8"), ("pos", "<i8")])


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
        self.field_format = EF_FIELD_U16
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

    def decode_audio_async(self, pcm, pdm=None, info=None, end=None, stream=0):
        """ef_decode_audio_async: decode_audio() into CUDA tensors, returning once the work is enqueued on `stream` (a
        torch.cuda.Stream or a raw handle). pcm: int16 tensor of pcm_cap samples; pdm: None or uint16 tensor of 2 * pcm_cap
        words; info: None or an int32 tensor [n_streams, 4] that receives the ef_audio_info rows (see audio_info()).
        Returns info. audio_wait() says whether the call fit."""
        import torch
        n = self.n_streams
        if info is None:
            info = torch.zeros((n, 4), dtype=torch.int32, device=pcm.device)
        for t, dt, what in ((pcm, torch.int16, "pcm"), (pdm, torch.uint16, "pdm"), (info, torch.int32, "info")):
            if t is not None and not (t.is_cuda and t.dtype == dt and t.is_contiguous()):
                raise TypeError("%s must be a contiguous CUDA %s tensor" % (what, dt))
        assert info.numel() == 4 * n
        if end is True:
            end = np.ones(n, dtype=np.uint8)
        elif end is not None:
            end = np.ascontiguousarray(end, dtype=np.uint8)
            assert end.size == n
        cap = pcm.numel() if pdm is None else min(pcm.numel(), pdm.numel() // 2)
        st = getattr(stream, "cuda_stream", stream)
        self._check(self.lib.ef_decode_audio_async(self._h, _ptr(end), info.data_ptr(), pcm.data_ptr(), cap,
                                                   None if pdm is None else pdm.data_ptr(), st))
        return info

    def audio_wait(self):
        """ef_audio_wait: waits for the last decode_audio_async -> EF_OK, or EF_ENOMEM when its samples exceeded pcm_cap
        (nothing decoded, no state changed)"""
        rc = self.lib.ef_audio_wait(self._h)
        if rc not in (EF_OK, EF_ENOMEM):
            self._check(rc)
        return rc

    @staticmethod
    def audio_info(info):
        """the int32 [n_streams, 4] info tensor of decode_audio_async -> numpy array of the ef_audio_info rows"""
        return np.ascontiguousarray(info.cpu().numpy()).view(_AUDIO_INFO).reshape(-1)

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

    # -- paced presentation ---------------------------------------------------------------------
    def enable_present(self, frame_counter0=None):
        """every stream gets its own display, starting at line 0 of field frame_counter0[s] (default 0); needs enable_pts()"""
        fc = None if frame_counter0 is None else np.ascontiguousarray(np.broadcast_to(frame_counter0, (self.n_streams,)), dtype=np.uint32)
        self._check(self.lib.ef_present_enable(self._h, _ptr(fc)))

    def present_format(self, fmt):
        """ef_present_format, before enable_present(): EF_FIELD_U16 (the default) has the present calls write the reference's
        uint16 DMA line buffer, EF_FIELD_DAC8 the bytes the video DAC plays (byte t of a line = sample t ^ 1's high byte). A DAC8
        context takes contiguous CUDA torch.uint8 tensors for `out`."""
        self._check(self.lib.ef_present_format(self._h, int(fmt)))
        self.field_format = int(fmt)

    def _dac8_out(self, out):
        """on a DAC8 context, out must be a contiguous CUDA uint8 tensor (TypeError otherwise) -> True"""
        if self.field_format != EF_FIELD_DAC8:
            return False
        import torch
        if not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous()):
            raise TypeError("out must be a contiguous CUDA torch.uint8 tensor on an EF_FIELD_DAC8 context")
        return True

    def _present(self, call, out, stream):
        info = np.zeros(self.n_streams, dtype=PRESENT_INFO)
        if out is None:
            dst, cap = None, 0
        else:
            if not self._dac8_out(out):
                assert out.is_cuda and str(out.dtype) == "torch.uint16" and out.is_contiguous()
            w, n = self.geometry()
            dst, cap = out.data_ptr(), out.numel() // (w * n)       # whole fields only
        self._check(call(dst, cap, info.ctypes.data, stream))
        return info

    def present_picture(self, pic, modes=None, out=None, stream=0):
        """ef_present_picture: decode picture index `pic` and push it on every stream that has it. out: CUDA uint16 tensor of
        whole fields, uint8 on a DAC8 context (None: sizing call). Returns info (PRESENT_INFO per stream)."""
        md = None if modes is None else np.ascontiguousarray(np.broadcast_to(modes, (self.n_streams,)), dtype=np.uint8)
        return self._present(lambda d, c, i, st: self.lib.ef_present_picture(self._h, pic, _ptr(md), d, c, i, st), out, stream)

    def present_idle(self, n_fields, out=None, stream=0):
        """ef_present_idle: every display runs on until it has emitted n_fields[s] more fields"""
        nf = np.ascontiguousarray(np.broadcast_to(n_fields, (self.n_streams,)), dtype=np.uint32)
        return self._present(lambda d, c, i, st: self.lib.ef_present_idle(self._h, nf.ctypes.data, d, c, i, st), out, stream)

    def _present_async(self, call, out, info):
        import torch
        if info is None:
            info = torch.zeros((self.n_streams, 8), dtype=torch.int32, device=out.device)
        checks = ((info, torch.int32, "info"),) if self._dac8_out(out) else ((out, torch.uint16, "out"), (info, torch.int32, "info"))
        for t, dt, what in checks:
            if not (t.is_cuda and t.dtype == dt and t.is_contiguous()):
                raise TypeError("%s must be a contiguous CUDA %s tensor" % (what, dt))
        assert info.numel() == 8 * self.n_streams
        w, n = self.geometry()
        self._check(call(out.data_ptr(), out.numel() // (w * n), info.data_ptr()))      # whole fields only
        return info

    def present_picture_async(self, pic, out, info=None, modes=None, stream=0):
        """ef_present_picture_async: present_picture() into the CUDA uint16 (DAC8: uint8) tensor `out`, returning once the work is enqueued on
        `stream` (a torch.cuda.Stream or a raw handle). info: None or an int32 tensor [n_streams, 8] that receives the
        ef_present_info rows (see present_info()). Returns info. present_wait() says how far the chain of async calls got."""
        md = None if modes is None else np.ascontiguousarray(np.broadcast_to(modes, (self.n_streams,)), dtype=np.uint8)
        st = getattr(stream, "cuda_stream", stream)
        return self._present_async(lambda d, c, i: self.lib.ef_present_picture_async(self._h, pic, _ptr(md), d, c, i, st), out, info)

    def present_idle_async(self, n_fields, out, info=None, stream=0):
        """ef_present_idle_async: present_idle() into the CUDA uint16 tensor `out`, enqueued on `stream`. Returns info."""
        nf = np.ascontiguousarray(np.broadcast_to(n_fields, (self.n_streams,)), dtype=np.uint32)
        st = getattr(stream, "cuda_stream", stream)
        return self._present_async(lambda d, c, i: self.lib.ef_present_idle_async(self._h, nf.ctypes.data, d, c, i, st), out, info)

    def present_wait(self):
        """ef_present_wait: waits for the chain of async present calls -> (EF_OK, or EF_ENOMEM when a call exceeded its buffer;
        the calls that took effect)"""
        k = _I()
        rc = self.lib.ef_present_wait(self._h, ctypes.byref(k))
        if rc not in (EF_OK, EF_ENOMEM):
            self._check(rc)
        return rc, k.value

    @staticmethod
    def present_info(info):
        """the int32 [n_streams, 8] info tensor of present_*_async -> numpy array of the PRESENT_INFO rows"""
        return np.ascontiguousarray(info.cpu().numpy()).view(PRESENT_INFO).reshape(-1)

    def present_overlay(self, bitmaps=None, blend=None, progress=None, set=None, first=0, count=None):
        """ef_present_overlay: stage overlay changes for streams [first, first + count); they latch at line 0 of the first field
        the next present call reaches. bitmaps: [count, 16, 80] uint8 (or one bitmap for all), blend / progress: int32 per stream or
        one for all, set: per-stream bits (1 bitmap, 2 blend, 4 progress; None = all three). None leaves that attribute unset."""
        count = self.n_streams - first if count is None else count

        bm = None if bitmaps is None else np.asarray(bitmaps, dtype=np.uint8).reshape(-1, 1280)
        keep = [None if a is None else np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=dt), shape))
                for a, dt, shape in ((bm, np.uint8, (count, 1280)), (blend, np.int32, (count,)), (progress, np.int32, (count,)), (set, np.uint8, (count,)))]
        ptrs = [None if a is None or a.size == 0 else a.ctypes.data for a in keep]
        self._check(self.lib.ef_present_overlay(self._h, first, count, *ptrs))

    def present_font(self, atlas, rights):
        """ef_present_font: the glyph atlas of the overlay's time text. atlas: [16, 1024] uint8 (the reference's _font8), rights:
        int16 glyph right edges (_font8_rights)."""
        a = np.ascontiguousarray(atlas, dtype=np.uint8).reshape(-1)
        r = np.ascontiguousarray(rights, dtype=np.int16).reshape(-1)
        if a.size != 16 * 1024:
            raise ValueError("the atlas is 16 x 1024 bytes")
        self._check(self.lib.ef_present_font(self._h, a.ctypes.data, r.ctypes.data, r.size))

    def present_clock(self, idx_hdrs, speed, flags, first=0, count=None):
        """ef_present_clock: update_progress() on streams [first, first + count) from the next present call on. idx_hdrs: [count, 104]
        uint8 video.idx headers (or one for all), speed: -1 / 0 / 1 per stream or one for all, flags: bit 0 on, bit 1 paused, bit 2
        zero _last_seconds."""
        count = self.n_streams - first if count is None else count
        h = np.ascontiguousarray(np.broadcast_to(np.asarray(idx_hdrs, dtype=np.uint8).reshape(-1, 104), (count, 104)))
        sp = np.ascontiguousarray(np.broadcast_to(np.asarray(speed, dtype=np.int8), (count,)))
        fl = np.ascontiguousarray(np.broadcast_to(np.asarray(flags, dtype=np.uint8), (count,)))
        ptrs = [a.ctypes.data if a.size else None for a in (h, sp, fl)]
        self._check(self.lib.ef_present_clock(self._h, first, count, *ptrs))

    # -- per-stream restart ----------------------------------------------------------------------
    def restart_streams(self, ops, first=0):
        """ef_restart_streams: ops[i] for stream first + i, between the current submit and the next one. 0 nothing, 1 the
        reference's MpegDecoder::reset() + video_reset() (a new title or a seek), 2 video_pause(0) (resume after a pause)."""
        ops = np.ascontiguousarray(ops, dtype=np.uint8).reshape(-1)
        self._check(self.lib.ef_restart_streams(self._h, first, ops.size, ops.ctypes.data if ops.size else None))

    # -- TS submits cut anywhere ------------------------------------------------------------------
    def enable_carry(self, max_carry):
        """ef_carry_enable: from the next submit, TS submits may be cut at any packet boundary; every stream holds up to
        max_carry bytes of its unfinished access unit between submits"""
        self._check(self.lib.ef_carry_enable(self._h, int(max_carry)))

    def end_streams(self, ends, first=0):
        """ef_end_streams: the streams first + i with ends[i] != 0 end with the pending submit (their last unit counts as
        complete at its index())"""
        ends = np.ascontiguousarray(ends, dtype=np.uint8).reshape(-1)
        self._check(self.lib.ef_end_streams(self._h, first, ends.size, ends.ctypes.data if ends.size else None))

    def carry_info(self, first=0, count=None):
        """ef_carry_info -> (uint32[count] bytes each stream holds after the current submit, uint8[count] flags: bit 0 = its held
        bytes exceeded max_carry)"""
        count = self.n_streams - first if count is None else count
        held = np.zeros(max(count, 1), dtype=np.uint32)
        flags = np.zeros(max(count, 1), dtype=np.uint8)
        self._check(self.lib.ef_carry_info(self._h, first, count, held.ctypes.data, flags.ctypes.data))
        return held[:count], flags[:count]

    # -- titles held in device memory ---------------------------------------------------------------
    def library_add(self, idx, main, fwd=None, rwd=None):
        """ef_library_add: copy one title to device memory -> its number. idx: the video.idx image; main / fwd / rwd: its
        transport streams (video.ts, video_fwd.ts, video_rwd.ts; the trick files may be None)"""
        keep = [None if f is None or len(f) == 0 else np.frombuffer(bytes(f), dtype=np.uint8) for f in (rwd, main, fwd)]
        ptrs = (ctypes.c_void_p * 3)(*[None if a is None else a.ctypes.data for a in keep])
        sizes = (ctypes.c_uint64 * 3)(*[0 if a is None else a.size for a in keep])
        im = np.frombuffer(bytes(idx), dtype=np.uint8)
        t = _I()
        self._check(self.lib.ef_library_add(self._h, im.ctypes.data if im.size else None, im.size, ptrs, sizes, ctypes.byref(t)))
        return t.value

    def library_add_trick(self, title, qscale=None):
        """ef_library_add_trick: build the fast-forward and rewind files of a title added with its main only, attach them and
        rewrite the fwd and rwd records and samples of its video.idx (qscale None: TRICK_QSCALE)"""
        self._check(self.lib.ef_library_add_trick(self._h, int(title), TRICK_QSCALE if qscale is None else int(qscale)))

    def library_read(self, title, what):
        """ef_library_read: a title's video.idx image (what -1), its rwd / main / fwd file (0 / 1 / 2) or its poster.ts (3) as bytes
        (b"" when absent)"""
        n = ctypes.c_uint64()
        rc = self.lib.ef_library_read(self._h, int(title), int(what), None, 0, ctypes.byref(n))
        if rc != EF_ENOMEM:
            self._check(rc)
            return b""
        out = np.zeros(n.value, dtype=np.uint8)
        self._check(self.lib.ef_library_read(self._h, int(title), int(what), out.ctypes.data, out.size, ctypes.byref(n)))
        return out.tobytes()

    def library_add_poster(self, title, poster):
        """ef_library_add_poster: attach a title's poster.ts (capi.encode_poster makes one) as its file 3"""
        a = np.frombuffer(bytes(poster), dtype=np.uint8)
        self._check(self.lib.ef_library_add_poster(self._h, int(title), a.ctypes.data if a.size else None, a.size))

    def library_nv_read(self, title, first=0, count=None):
        """ef_library_nv_read -> int64 saved positions of streams [first, first + count) on `title` (0: none saved)"""
        count = self.n_streams - first if count is None else count
        out = np.zeros(max(count, 1), dtype=np.int64)
        self._check(self.lib.ef_library_nv_read(self._h, int(title), first, count, out.ctypes.data))
        return out[:count]

    def library_nv_write(self, title, pos, first=0):
        """ef_library_nv_write: saved positions of streams [first, first + len(pos)) on `title`, e.g. kept by a service across sessions"""
        a = np.ascontiguousarray(pos, dtype=np.int64).reshape(-1)
        self._check(self.lib.ef_library_nv_write(self._h, int(title), first, a.size, a.ctypes.data if a.size else None))

    def library_command(self, cmd, first=0, count=1, title=0, arg=0):
        """ef_library_command: cmd (LIB_PLAY_AT ... LIB_MENU) on streams [first, first + count); title (PLAY_AT, NAV) and arg (main
        pts for PLAY_AT, seconds for SKIP, the step of NAV_STEP) as the header describes"""
        self._check(self.lib.ef_library_command(self._h, first, count, int(cmd), int(title), int(arg)))

    def library_submit(self, packets=0, per_stream=None, stream=0):
        """ef_library_submit: a TS submit of every PLAYING stream's next min(budget, packets left) packets; per_stream: one
        budget per stream (else `packets` for all)"""
        ps = None if per_stream is None else np.ascontiguousarray(np.broadcast_to(per_stream, (self.n_streams,)), dtype=np.uint32)
        st = getattr(stream, "cuda_stream", stream)
        self._check(self.lib.ef_library_submit(self._h, int(packets), _ptr(ps), st))

    def library_keys(self, keys, done=None, stream=0):
        """ef_library_keys: one iteration of the reference's loop() on every stream with keys[s] (KEY_*, 0 none), enqueued on `stream`
        (a torch.cuda.Stream or a raw handle). keys: n_streams bytes, a numpy array or a CUDA torch.uint8 tensor (a producer on the
        device); done: None or a CUDA torch.uint8 tensor of n_streams that receives each stream's done code. Returns done."""
        n = self.n_streams
        if isinstance(keys, np.ndarray) or not hasattr(keys, "data_ptr"):
            keys = np.ascontiguousarray(np.broadcast_to(keys, (n,)), dtype=np.uint8)
            kp = keys.ctypes.data
        else:
            import torch
            if not (keys.is_cuda and keys.dtype == torch.uint8 and keys.is_contiguous() and keys.numel() == n):
                raise TypeError("keys must be a contiguous CUDA torch.uint8 tensor of n_streams")
            kp = keys.data_ptr()
        if done is not None:
            import torch
            if not (done.is_cuda and done.dtype == torch.uint8 and done.is_contiguous() and done.numel() == n):
                raise TypeError("done must be a contiguous CUDA torch.uint8 tensor of n_streams")
        st = getattr(stream, "cuda_stream", stream)
        self._check(self.lib.ef_library_keys(self._h, kp, None if done is None else done.data_ptr(), st))
        return done

    def library_info(self, first=0, count=None):
        """ef_library_info -> LIBRARY_STATUS rows (title, speed, state, file, cursor, pos) of streams [first, first + count)"""
        count = self.n_streams - first if count is None else count
        out = np.zeros(max(count, 1), dtype=LIBRARY_STATUS)
        self._check(self.lib.ef_library_info(self._h, first, count, out.ctypes.data))
        return out[:count]

    def launch_count(self):
        return int(self.lib.ef_launch_count(self._h))

    def set_profiling(self, on=True):
        self._check(self.lib.ef_set_profiling(self._h, 1 if on else 0))

    def stage_ms(self):
        """(K0 index, K1a parse, K1b reconstruction) milliseconds of the last ef_index / ef_decode_* (synchronises)."""
        a, b, c = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.ef_stage_ms(self._h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
        return a.value, b.value, c.value


PRESENT_INFO = np.dtype([("first", "<u8"), ("n_fields", "<u4"), ("frame_counter", "<u4"), ("flip_field", "<u4"), ("flip_line", "<i4"),
                         ("flags", "<i4"), ("pad", "<i4")])


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


TRICK_QSCALE = 8                 # ef_trick_build's default quantiser scale (tests/trick_cases.DEFAULT_QSCALE)


def trick_build(mains, qscale=TRICK_QSCALE, device=0):
    """ef_trick_build: video_fwd.ts and video_rwd.ts of every main (bytes-like transport streams) -> [(fwd bytes, rwd bytes), ...]"""
    lib = load_library()
    blob, off = Context.pack(mains)
    n = len(mains)
    fo, ro = np.zeros(n + 1, dtype=np.uint64), np.zeros(n + 1, dtype=np.uint64)
    cap = int(off[-1]) + 188 * 1024          # intra pictures at 1/15 of the rate: the main's size is a generous first guess
    for _ in range(2):
        fwd, rwd = np.zeros(cap, dtype=np.uint8), np.zeros(cap, dtype=np.uint8)
        rc = lib.ef_trick_build(device, blob.ctypes.data, off.ctypes.data, n, int(qscale), fwd.ctypes.data, fwd.size, fo.ctypes.data,
                                rwd.ctypes.data, rwd.size, ro.ctypes.data)
        need = max(int(fo[-1]), int(ro[-1]))
        if rc != EF_ENOMEM or need <= cap:
            break
        cap = need
    _check_rc(lib, rc)
    return [(fwd[int(fo[i]):int(fo[i + 1])].tobytes(), rwd[int(ro[i]):int(ro[i + 1])].tobytes()) for i in range(n)]


class EncodeParams(ctypes.Structure):
    """ef_encode_params (include/espflix_b200.h)"""
    _fields_ = [("gop", ctypes.c_int), ("qscale_i", ctypes.c_int), ("qscale_p", ctypes.c_int), ("search", ctypes.c_int),
                ("aspect", ctypes.c_int), ("rate", ctypes.c_int), ("pts0", ctypes.c_int64), ("pts_step", ctypes.c_uint32)]


# ef_encode_build's defaults (tests/encode_cases.DEFAULT_PARAMS, where the measurement behind the quantisers is): GOP 12 as ffmpeg's
# mpeg1video and both fixtures; qscale 8 / 8, the largest that keeps every picture of both fixtures at or above 35 dB; search 7:
# forward_f_code 1 reaches -8..7.5 pixels; aspect 1 (square samples), rate 2 and a pts step of 3,750: 24 pictures per second on the
# 90 kHz clock.
ENCODE_DEFAULTS = dict(gop=12, qscale_i=8, qscale_p=8, search=7, aspect=1, rate=2, pts0=0, pts_step=3750)
PICTURE_BYTES = 101376


def encode_build(titles, device=0, **params):
    """ef_encode_build: video.ts of every title (a uint8 array of shape (n, 101376): 352 x 192 I420 pictures in display order)
    -> [bytes, ...]"""
    lib = load_library()
    p = dict(ENCODE_DEFAULTS, **params)
    arrs = [np.ascontiguousarray(np.asarray(t, dtype=np.uint8).reshape(-1, PICTURE_BYTES)) for t in titles]
    n = len(arrs)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([a.shape[0] for a in arrs])
    blob = np.concatenate(arrs) if n else np.zeros((1, PICTURE_BYTES), np.uint8)
    if blob.size == 0:
        blob = np.zeros((1, PICTURE_BYTES), np.uint8)
    par = EncodeParams(**{k: int(v) for k, v in p.items()})
    to = np.zeros(n + 1, dtype=np.uint64)
    cap = int(off[-1]) * 16384 + 188 * 64    # about twice the bytes per picture of the defaults on the fixtures; retried once when short
    for _ in range(2):
        ts = np.zeros(cap, dtype=np.uint8)
        rc = lib.ef_encode_build(device, blob.ctypes.data, off.ctypes.data, n, ctypes.byref(par), ts.ctypes.data, ts.size, to.ctypes.data)
        if rc != EF_ENOMEM or int(to[-1]) <= cap:
            break
        cap = int(to[-1])
    _check_rc(lib, rc)
    return [ts[int(to[i]):int(to[i + 1])].tobytes() for i in range(n)]


# make_video()'s poster: ffmpeg ... -bf 0 -q 2 poster.ts (indexer.cpp:306), one I picture at quantiser scale 2
POSTER_PARAMS = dict(gop=1, qscale_i=2)


def encode_poster(picture_i420, device=0):
    """poster.ts of one 352 x 192 I420 picture (101,376 bytes): ef_encode_build of that picture with gop 1 and qscale_i 2, the
    other parameters ENCODE_DEFAULTS -> bytes"""
    pic = np.asarray(picture_i420, dtype=np.uint8).reshape(-1)
    if pic.size != PICTURE_BYTES:
        raise EspflixError(EF_EINVAL, "a poster is one picture of %d bytes, not %d" % (PICTURE_BYTES, pic.size))
    return encode_build([pic.reshape(1, PICTURE_BYTES)], device=device, **POSTER_PARAMS)[0]


class RateParams(ctypes.Structure):
    """ef_rate_params (include/espflix_b200.h)"""
    _fields_ = [("bit_rate", ctypes.c_uint32), ("vbv_bits", ctypes.c_uint32), ("qmin", ctypes.c_int), ("qmax", ctypes.c_int)]


# ef_encode_build_rate's defaults: the reference's make_video() "-b:v 1500k -maxrate 1500k -bufsize 0.25M -qmin 3" (the quantisers
# up to 31, MPEG-1's largest)
ENCODE_RATE_DEFAULTS = dict(bit_rate=1500000, vbv_bits=250000, qmin=3, qmax=31)


def encode_build_rate(titles, device=0, **params):
    """ef_encode_build_rate: video.ts of every title encoded to a bit rate and buffer size -> [(ts bytes, pic_q uint8 [n], pic_bytes
    uint32 [n]), ...]; params: those of ENCODE_DEFAULTS (qscale_i / qscale_p are not read) and ENCODE_RATE_DEFAULTS"""
    lib = load_library()
    unknown = set(params) - set(ENCODE_DEFAULTS) - set(ENCODE_RATE_DEFAULTS)
    if unknown:
        raise TypeError("unknown parameters %s" % sorted(unknown))
    par = EncodeParams(**{k: int(v) for k, v in dict(ENCODE_DEFAULTS, **{k: v for k, v in params.items() if k in ENCODE_DEFAULTS}).items()})
    rp = RateParams(**{k: int(v) for k, v in dict(ENCODE_RATE_DEFAULTS, **{k: v for k, v in params.items() if k in ENCODE_RATE_DEFAULTS}).items()})
    arrs = [np.ascontiguousarray(np.asarray(t, dtype=np.uint8).reshape(-1, PICTURE_BYTES)) for t in titles]
    n = len(arrs)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([a.shape[0] for a in arrs])
    blob = np.concatenate(arrs) if n and off[-1] else np.zeros((1, PICTURE_BYTES), np.uint8)
    to = np.zeros(n + 1, dtype=np.uint64)
    q = np.zeros(max(int(off[-1]), 1), dtype=np.uint8)
    nb = np.zeros(max(int(off[-1]), 1), dtype=np.uint32)
    cap = int(off[-1]) * 16384 + 188 * 64
    for _ in range(2):
        ts = np.zeros(cap, dtype=np.uint8)
        rc = lib.ef_encode_build_rate(device, blob.ctypes.data, off.ctypes.data, n, ctypes.byref(par), ctypes.byref(rp), ts.ctypes.data, ts.size,
                                      to.ctypes.data, q.ctypes.data, nb.ctypes.data)
        if rc != EF_ENOMEM or int(to[-1]) <= cap:
            break
        cap = int(to[-1])
    _check_rc(lib, rc)
    return [(ts[int(to[i]):int(to[i + 1])].tobytes(), q[int(off[i]):int(off[i + 1])].copy(), nb[int(off[i]):int(off[i + 1])].copy())
            for i in range(n)]


def encode_stage_ms():
    """(upload, search, code, reconstruction, mux) device milliseconds of the last encode_build on this thread"""
    lib = load_library()
    v = [ctypes.c_float() for _ in range(5)]
    _check_rc(lib, lib.ef_encode_stage_ms(*[ctypes.byref(x) for x in v]))
    return tuple(x.value for x in v)


class AudioParams(ctypes.Structure):
    """ef_audio_params (include/espflix_b200.h)"""
    _fields_ = [("frequency", ctypes.c_int), ("allocation", ctypes.c_int), ("bitpool", ctypes.c_int), ("frames_per_pes", ctypes.c_int),
                ("pts0", ctypes.c_int64)]


# ef_sbc_encode / ef_mux_audio defaults: the reference's make_video() audio (48 kHz, mono, 192 kbit/s: bit pool 28 makes 64-byte frames,
# 375 a second; loudness allocation as ffmpeg's encoder; -pes_payload_size 512: 8 frames per PES)
AUDIO_ENCODE_DEFAULTS = dict(frequency=3, allocation=0, bitpool=28, frames_per_pes=0, pts0=0)


def sbc_encode(pcms, device=0, **params):
    """ef_sbc_encode: SBC of every mono int16 PCM stream -> [bytes, ...]"""
    lib = load_library()
    par = AudioParams(**{k: int(v) for k, v in dict(AUDIO_ENCODE_DEFAULTS, **params).items()})
    arrs = [np.ascontiguousarray(np.asarray(x, dtype=np.int16).reshape(-1)) for x in pcms]
    off = np.zeros(len(arrs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([a.size for a in arrs])
    blob = np.concatenate(arrs + [np.zeros(1, np.int16)])
    so = np.zeros(len(arrs) + 1, dtype=np.uint64)
    rc = lib.ef_sbc_encode(device, blob.ctypes.data, off.ctypes.data, len(arrs), ctypes.byref(par), None, 0, so.ctypes.data)
    if rc != EF_ENOMEM:
        _check_rc(lib, rc)
    out = np.zeros(max(int(so[-1]), 1), dtype=np.uint8)
    _check_rc(lib, lib.ef_sbc_encode(device, blob.ctypes.data, off.ctypes.data, len(arrs), ctypes.byref(par), out.ctypes.data, out.size,
                                     so.ctypes.data))
    return [out[int(so[i]):int(so[i + 1])].tobytes() for i in range(len(arrs))]


def mux_audio(videos, sbcs, device=0, **params):
    """ef_mux_audio: every video transport stream with its SBC interleaved on PID 0x102 -> [bytes, ...]"""
    lib = load_library()
    if len(videos) != len(sbcs):
        raise ValueError("one SBC stream per video")
    par = AudioParams(**{k: int(v) for k, v in dict(AUDIO_ENCODE_DEFAULTS, **params).items()})
    tb, to = Context.pack(videos)
    sb, so = Context.pack(sbcs)
    oo = np.zeros(len(videos) + 1, dtype=np.uint64)
    args = (device, tb.ctypes.data, to.ctypes.data, sb.ctypes.data, so.ctypes.data, len(videos), ctypes.byref(par))
    rc = lib.ef_mux_audio(*args, None, 0, oo.ctypes.data)
    if rc != EF_ENOMEM:
        _check_rc(lib, rc)
    out = np.zeros(max(int(oo[-1]), 1), dtype=np.uint8)
    _check_rc(lib, lib.ef_mux_audio(*args, out.ctypes.data, out.size, oo.ctypes.data))
    return [out[int(oo[i]):int(oo[i + 1])].tobytes() for i in range(len(videos))]


def audio_encode_stage_ms():
    """(upload, encode, download) device milliseconds of the last sbc_encode and the host milliseconds of the last mux_audio on this
    thread"""
    lib = load_library()
    v = [ctypes.c_float() for _ in range(4)]
    _check_rc(lib, lib.ef_audio_encode_stage_ms(*[ctypes.byref(x) for x in v]))
    return tuple(x.value for x in v)


def encode_title(pictures, pcm, rate=None, device=0, **params):
    """a title's video.ts with audio: encode_build of its pictures, sbc_encode of its PCM and mux_audio of both. params: those of
    ENCODE_DEFAULTS and AUDIO_ENCODE_DEFAULTS (pts0 is the video's; the audio's is audio_pts0, default the same). rate: None for the
    fixed quantisers, else a dict of ENCODE_RATE_DEFAULTS' fields ({} for the defaults) for encode_build_rate; the audio is not
    counted in the video's bucket, as ffmpeg's -b:v does not count it. An integer rate is the sequence header's picture-rate code, as
    it was before rate control existed."""
    if rate is not None and not isinstance(rate, dict):
        params["rate"], rate = rate, None
    vp = {k: v for k, v in params.items() if k in ENCODE_DEFAULTS}
    ap = {k: v for k, v in params.items() if k in AUDIO_ENCODE_DEFAULTS and k != "pts0"}
    unknown = set(params) - set(ENCODE_DEFAULTS) - set(AUDIO_ENCODE_DEFAULTS) - {"audio_pts0"}
    if unknown:
        raise TypeError("unknown parameters %s" % sorted(unknown))
    ap["pts0"] = params.get("audio_pts0", vp.get("pts0", 0))
    if rate is None:
        video = encode_build([pictures], device=device, **vp)[0]
    else:
        video = encode_build_rate([pictures], device=device, **vp, **dict(rate))[0][0]
    sbc = sbc_encode([pcm], device=device, **ap)[0]
    return mux_audio([video], [sbc], device=device, **ap)[0]


def trick_stage_ms():
    """(decode, gather, encode, mux) device milliseconds of the last trick_build on this thread"""
    lib = load_library()
    v = [ctypes.c_float() for _ in range(4)]
    _check_rc(lib, lib.ef_trick_stage_ms(*[ctypes.byref(x) for x in v]))
    return tuple(x.value for x in v)


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
