"""Directed SBC frames across the decoder's whole frame-header domain (csrc/ef_audio.cu, oracle/ef_oracle_audio.c): each
frame's header, scale factors and samples are chosen, not drawn.

  alloc()      plain-Python restatement of the reference's bit allocation (sbc_decoder.cpp:141-231) with an explicit
               iteration cap, reporting the branches it took; a bit pool above MAX_BITPOOL is -2 (outside the domain)
  frame()      one frame, every header field an argument, raw samples bit-packed by that allocation
  iquant()     IQUANT (sbc_decoder.cpp:257-265) with the 32-bit wrap of the compiled reference
  streams()    the directed streams, each under 4,096 bytes of audio, so that the reference's 4 KB ring never wraps
               (quirk Q13, tools/make_audio_golden.py) and every byte it reads past the end of a stream is a zero:
                 alloc_*     every bit pool 0..128 x 4 frequencies x both allocation modes over SF_SETS
                 iquant_*    raw 0, 1, 2^w - 2, 2^w - 1 at every width 1..16 and scale factors 0, 7, 14, 15
                 max_*       264-byte frames at bit pool 128
                 overrun_*   frames whose allocation reads past the frame into the next one and past the end of the stream
                 kind_*      every header kind as frame 0, as a middle frame, as the last frame and twice in a row
  census()     what the streams reach, so each test can assert it
"""
import numpy as np

MAX_BITPOOL = 128
CAP = 10 ** 6                                             # iterations of the slice loop alloc() runs before giving up
OFFSET8 = [[-2, 0, 0, 0, 0, 0, 0, 1], [-3, 0, 0, 0, 0, 0, 1, 2], [-4, 0, 0, 0, 0, 0, 1, 2], [-4, 0, 0, 0, 0, 0, 1, 2]]
ES_LIMIT = 3800                                           # + the 264 bytes a last frame may read: inside the 4 KB ring


def bitneed(frequency, allocation, sf):
    if allocation:
        return list(sf)
    out = []
    for sb, s in enumerate(sf):
        if s == 0:
            out.append(-5)
        else:
            n = s - OFFSET8[frequency][sb]
            out.append(n // 2 if n > 0 else n)
    return out


def alloc(frequency, allocation, bitpool, sf, bounded=True, cap=CAP):
    """-> dict(total, bits, branches, iterations). total -2 for a bit pool above MAX_BITPOOL when bounded; unbounded,
    the loop runs as the reference wrote it and total is None when it has not finished after `cap` iterations."""
    if bounded and bitpool > MAX_BITPOOL:
        return dict(total=-2, bits=[0] * 8, branches=set(), iterations=0)
    need = bitneed(frequency, allocation, sf)
    br = set()
    bitcount, slicecount, bitslice = 0, 0, max(0, max(need)) + 1
    it = 0
    while True:
        it += 1
        if it > cap:
            return dict(total=None, bits=[0] * 8, branches=br, iterations=it - 1)
        bitslice -= 1
        bitcount += slicecount
        slicecount = 0
        for n in need:
            if bitslice + 1 < n < bitslice + 16:
                slicecount += 1
            elif n == bitslice + 1:
                slicecount += 2
        if not bitcount + slicecount < bitpool:
            break
    if bitcount + slicecount == bitpool:
        br.add("exact")
        bitcount += slicecount
        bitslice -= 1
    else:
        br.add("overshoot")
    bits = [0 if n < bitslice + 2 else min(n - bitslice, 16) for n in need]
    for sb in range(8):
        if bitcount >= bitpool:
            break
        if 2 <= bits[sb] < 16:
            bits[sb] += 1
            bitcount += 1
            br.add("plus1")
        elif need[sb] == bitslice + 1:
            if bitpool > bitcount + 1:
                bits[sb] = 2
                bitcount += 2
                br.add("plus2")
            else:
                br.add("plus2_refused")
    for sb in range(8):
        if bitcount >= bitpool:
            break
        if bits[sb] < 16:
            if bits[sb] == 0:
                br.add("raise0")
            bits[sb] += 1
            bitcount += 1
        else:
            br.add("saturated16")
    return dict(total=sum(bits), bits=bits, branches=br, iterations=it)


def iquant(raw, level, scale):
    """((2 raw + 1) << scale) as the reference's int (32-bit wrap), divided by 2^level - 1 (C truncation), minus 2^scale"""
    v = ((2 * raw + 1) << scale) & 0xFFFFFFFF
    v = v - (1 << 32) if v >= 1 << 31 else v
    d = (1 << level) - 1
    q = abs(v) // d
    return (q if v >= 0 else -q) - (1 << scale)


def iquant_wraps(raw, level, scale):
    return (2 * raw + 1) << scale >= 1 << 31


def header(frequency=2, blocks=16, mode=0, allocation=0, subbands=8, bitpool=28, sync=0x9C, crc=0):
    return bytes([sync, (frequency << 6) | ((blocks // 4 - 1) << 4) | (mode << 2) | (allocation << 1) | (1 if subbands == 8 else 0), bitpool, crc])


def frame(sf, raw=None, size=None, frequency=2, blocks=16, mode=0, allocation=0, subbands=8, bitpool=28, sync=0x9C, crc=0, fill=0):
    """header + scale factors + raw[16][8] packed MSB first at the widths alloc() gives (raw values are masked to them),
    then `fill` bytes up to `size` (default: exactly the bytes the bit loader reads, 8 + 2 * total)"""
    a = alloc(frequency, allocation, bitpool, sf)
    bits = a["bits"] if a["total"] is not None and a["total"] >= 0 else [0] * 8
    out = bytearray(header(frequency, blocks, mode, allocation, subbands, bitpool, sync, crc))
    out += bytes([(sf[k] << 4) | sf[k + 1] for k in range(0, 8, 2)])
    if raw is not None and sum(bits):
        w = np.array(bits, dtype=np.int64)
        r = np.asarray(raw, dtype=np.int64).reshape(16, 8) & ((1 << w) - 1)
        j = np.arange(16)
        sel = j[None, None, :] < w[None, :, None]                       # [blk][sb][bit] bit j of a w-bit value, MSB first
        vals = (r[:, :, None] >> np.clip(w[None, :, None] - 1 - j[None, None, :], 0, 15)) & 1
        out += np.packbits(vals[np.broadcast_to(sel, vals.shape)].astype(np.uint8)).tobytes()
    want = 8 + 2 * max(a["total"] or 0, 0) if size is None else size
    out = out[:want]
    out += bytes([fill]) * (want - len(out))
    return bytes(out)


def _raws(bits, salt):
    """chosen samples: for each width the four extremes 0, 1, 2^w - 2, 2^w - 1 in turn, and a ramp between them"""
    r = np.zeros((16, 8), dtype=np.int64)
    for sb, w in enumerate(bits):
        if not w:
            continue
        top = (1 << w) - 1
        for blk in range(16):
            k = (blk + salt + sb) % 8
            r[blk, sb] = [0, 1, max(top - 1, 0), top][k] if k < 4 else (top * (k - 3) * (salt + 7) // 41) % (top + 1)
    return r


# ---- scale-factor sets of the allocation sweep ---------------------------------------------------------------------------
def _sf_sets():
    s = {"zero": [0] * 8, "all15": [15] * 8, "ascending": [1, 3, 5, 7, 9, 11, 13, 15], "descending": [15, 13, 11, 9, 7, 5, 3, 1],
         "ramp8": list(range(8, 16)), "tie_max": [12, 3, 12, 5, 12, 7, 1, 12], "tie_all9": [9] * 8,
         "slice_pairs": [10, 9, 9, 10, 9, 2, 0, 9], "slice_steps": [14, 13, 13, 12, 12, 12, 0, 1], "near_loud": [15, 14, 15, 14, 15, 14, 15, 14]}
    for v in (1, 8, 15):
        for sb in range(8):
            x = [0] * 8
            x[sb] = v
            s["onehot%d_sb%d" % (v, sb)] = x
    return s


SF_SETS = _sf_sets()
FREQUENCIES = range(4)
ALLOCATIONS = (0, 1)


def _pack_stream(frames_bytes, fs):
    """frames laid out every fs bytes: a frame longer than fs is cut (its bit loader reads on into the next frame)"""
    out = bytearray()
    for f in frames_bytes:
        out += f[:fs] + bytes(max(0, fs - len(f)))
    return np.frombuffer(bytes(out), dtype=np.uint8).copy()


def _alloc_streams():
    out = {}
    for fq in FREQUENCIES:
        for al in ALLOCATIONS:
            for bp in range(MAX_BITPOOL + 1):
                items = sorted(SF_SETS.items(), key=lambda kv: (-alloc(fq, al, bp, kv[1])["total"], kv[0]))
                k, part = 0, 0
                while k < len(items):
                    fs = 8 + 2 * alloc(fq, al, bp, items[k][1])["total"]
                    n = max(1, ES_LIMIT // fs)
                    chunk = items[k:k + n]
                    fr = [frame(sf, _raws(alloc(fq, al, bp, sf)["bits"], i + part), frequency=fq, allocation=al, bitpool=bp) for i, (_, sf) in enumerate(chunk)]
                    out["alloc_f%d_a%d_bp%d_%d" % (fq, al, bp, part)] = _pack_stream(fr, fs)
                    k += n
                    part += 1
    return out


def _find(width, scale):
    """a (frequency, allocation, bit pool, scale factors, subband) whose allocation gives `width` to a subband of scale factor
    `scale`: the first hit of a fixed search"""
    bases = [[0] * 8, [15] * 8, [8] * 8, [1, 3, 5, 7, 9, 11, 13, 15], [15, 13, 11, 9, 7, 5, 3, 1], [3] * 8, [12] * 8]
    for base in bases:
        for sb in (0, 7, 3):
            sf = list(base)
            sf[sb] = scale
            for al in ALLOCATIONS:
                for fq in (2, 0):
                    for bp in range(MAX_BITPOOL + 1):
                        if alloc(fq, al, bp, sf)["bits"][sb] == width:
                            return fq, al, bp, sf, sb
    return None


IQUANT_SCALES = (0, 7, 14, 15)


def _iquant_streams():
    out = {}
    for w in range(1, 17):
        for s in IQUANT_SCALES:
            hit = _find(w, s)
            assert hit is not None, (w, s)
            fq, al, bp, sf, sb = hit
            top = (1 << w) - 1
            fr = []
            for salt in range(3):
                r = _raws(alloc(fq, al, bp, sf)["bits"], salt)
                for blk in range(16):
                    r[blk, sb] = [0, 1, max(top - 1, 0), top][(blk + salt) % 4]
                fr.append(frame(sf, r, frequency=fq, allocation=al, bitpool=bp))
            out["iquant_w%d_sf%d" % (w, s)] = _pack_stream(fr, len(fr[0]))
    return out


def _max_streams():
    out = {}
    for name, fq, al, sf in (("snr_zero", 2, 1, [0] * 8), ("loud_zero", 0, 0, [0] * 8), ("snr_15", 3, 1, [15] * 8)):
        assert alloc(fq, al, MAX_BITPOOL, sf)["total"] == 128
        fr = [frame(sf, _raws([16] * 8, k), frequency=fq, allocation=al, bitpool=MAX_BITPOOL) for k in range(ES_LIMIT // 264)]
        out["max_" + name] = _pack_stream(fr, 264)
    return out


def _overrun_streams():
    """frame 0 sets a small frame size; later frames ask for more bits and read into the frames after them, the last
    ones past the end of the stream (bytes there read as zero)"""
    out = {}
    base = [6, 9, 4, 11, 7, 3, 10, 5]
    for name, bp0, big, at in (("bp28_to_40", 28, 40, (1, 2, 6, 11)), ("bp12_to_128", 12, 128, (3, 9, 10, 11)), ("bp2_to_97", 2, 97, (5, 11))):
        fs = 8 + 2 * alloc(2, 0, bp0, base)["total"]
        fr = []
        for k in range(12):
            bp = big if k in at else bp0
            sf = base if k % 3 else [15 - x for x in base]
            fr.append(frame(sf, _raws(alloc(2, 0, bp, sf)["bits"], k), bitpool=bp))
        out["overrun_" + name] = _pack_stream(fr, fs)
    return out


# every header kind: (name, header fields), applied to a frame of a consistent mono / 16-block / 8-subband stream
KINDS = [("sync", dict(sync=0x00)), ("sub4", dict(subbands=4))] + \
        [("m3_b%d" % b, dict(mode=3, blocks=b)) for b in (4, 8, 12, 16)] + \
        [("m%d_b%d" % (m, b), dict(mode=m, blocks=b)) for m in (1, 2) for b in (4, 8, 12, 16)] + \
        [("mono_b%d" % b, dict(blocks=b)) for b in (4, 8, 12)] + \
        [("bp%d" % p, dict(bitpool=p)) for p in (129, 200, 255)]
PLACES = {"first": (0,), "middle": (5,), "last": (11,), "twice": (5, 6)}
KIND_FRAMES = 12
KIND_BASE = dict(frequency=2, allocation=0, bitpool=28)
KIND_SF = [5, 9, 7, 11, 6, 4, 8, 2]


def kind_stream(kind, place):
    fields = dict(KINDS)[kind]
    a = alloc(2, 0, 28, KIND_SF)
    fs = 8 + 2 * a["total"]
    fr = []
    for k in range(KIND_FRAMES):
        f = bytearray(frame(KIND_SF, _raws(a["bits"], k), **KIND_BASE))
        if k in PLACES[place]:
            kw = dict(KIND_BASE)
            kw.update(fields)
            f[:4] = header(**kw)
        fr.append(bytes(f))
    return _pack_stream(fr, fs), fs


def _kind_streams():
    return {"kind_%s_%s" % (k, p): kind_stream(k, p)[0] for k, _ in KINDS for p in PLACES}


_CACHE = {}


def streams():
    """name -> audio bytes of every directed stream (built once per process)"""
    if not _CACHE:
        for part in (_alloc_streams(), _iquant_streams(), _max_streams(), _overrun_streams(), _kind_streams()):
            _CACHE.update(part)
        assert all(s.size <= ES_LIMIT for s in _CACHE.values())
    return _CACHE


def frames_of(es):
    """(offset, bytes to the end of the stream) of every frame the decoder reads: frame 0 at 0, then every frame_size bytes"""
    es = bytes(es)
    if len(es) < 4:
        return []
    a = _hdr_alloc(es)
    if a is None or a["total"] < 0:
        return [0]
    fs = 8 + 2 * a["total"]
    return list(range(0, len(es) - fs + 1, fs))


def _hdr_alloc(d):
    """the restatement of one frame's header: None for a rejected frame, total -2 outside the domain, else alloc()"""
    if len(d) < 4 or d[0] != 0x9C:
        return None
    b1 = d[1]
    fq, blocks, mode, al, sub, bp = (b1 >> 6) & 3, 4 * (((b1 >> 4) & 3) + 1), (b1 >> 2) & 3, (b1 >> 1) & 1, 8 if b1 & 1 else 4, d[2]
    if sub == 4:
        return None
    if mode != 0 or blocks != 16 or bp > MAX_BITPOOL:
        return dict(total=-2, bits=[0] * 8, branches=set())
    sf = []
    for k in range(4):
        x = d[4 + k] if 4 + k < len(d) else 0
        sf += [x >> 4, x & 15]
    return alloc(fq, al, bp, sf)


def frame_info(es):
    """per frame read by the decoder: (offset, alloc() or None when rejected, the scale factors)"""
    es = bytes(es)
    out = []
    for off in frames_of(es):
        d = es[off:]
        sf = [(d[4 + k // 2] >> (0 if k & 1 else 4)) & 15 if 4 + k // 2 < len(d) else 0 for k in range(8)]
        out.append((off, _hdr_alloc(d), sf))
    return out


def ref_undefined_frames(es):
    """frames whose PCM the reference leaves undefined: a frame decoded while a 4-subband header is in force (the
    4-subband frame itself, and a bad-sync frame after it, which leaves that header in place) synthesises nothing and
    emits mono[128] uninitialised. Frame numbers count decoded frames (the probe not included)."""
    es = bytes(es)
    out, sub4 = [], False
    for k, off in enumerate(frames_of(es)):
        d = es[off:]
        if len(d) >= 4 and d[0] == 0x9C:
            sub4 = not d[1] & 1
        if sub4:
            out.append(k)
    return out


def ref_defined(es):
    """whether the reference's output is defined for a stream handed to it whole: no frame it reads (probe or decode)
    has a mode other than mono with 12 or 16 blocks (256 samples into mono[128]) or a bit pool above 128 (no end)"""
    es = bytes(es)
    for off in frames_of(es):
        d = es[off:]
        if len(d) >= 4 and d[0] == 0x9C and d[1] & 1:
            mode, blocks = (d[1] >> 2) & 3, 4 * (((d[1] >> 4) & 3) + 1)
            if d[2] > MAX_BITPOOL or (mode != 0 and blocks > 8):
                return False
    return True


def census(names=None):
    """what the directed streams reach: widths, allocation branches, IQUANT extremes (width, scale factor, which of 0, 1,
    2^w - 2, 2^w - 1), the (width, scale factor) pairs whose IQUANT wraps, frame sizes, overruns"""
    ss = streams()
    names = list(ss) if names is None else names
    c = dict(widths=set(), branches=set(), iquant=set(), wraps=set(), frame_sizes=set(), overruns=0, past_end=0)
    for n in names:
        es = bytes(ss[n])
        fi = frame_info(es)
        fs = fi[1][0] - fi[0][0] if len(fi) > 1 else None
        for off, a, sf in fi:
            if a is None or a["total"] < 0:
                continue
            c["widths"].update(a["bits"])
            c["branches"] |= a["branches"]
            need = 8 + 2 * a["total"]
            if fs is not None and need > fs:
                c["overruns"] += 1
            if off + need > len(es):
                c["past_end"] += 1
            c["frame_sizes"].add(need)
            raws = unpack(es[off:], a["bits"])
            for sb in range(8):
                w = a["bits"][sb]
                if not w:
                    continue
                col = set(int(x) for x in raws[:, sb])
                top = (1 << w) - 1
                for tag, v in (("0", 0), ("1", 1), ("top-1", top - 1), ("top", top)):
                    if v in col:
                        c["iquant"].add((w, sf[sb], tag))
                if any(iquant_wraps(r, w, sf[sb]) for r in col):
                    c["wraps"].add((w, sf[sb]))
    return c


def unpack(d, bits):
    """raw samples [16][8] a frame's bit loader reads (bytes past the end read as zero)"""
    total = sum(bits)
    need = 8 + 2 * total
    buf = bytes(d[8:need]) + bytes(max(0, need - max(len(d), 8)))
    v = np.concatenate([np.unpackbits(np.frombuffer(buf, dtype=np.uint8)), np.zeros(16, dtype=np.uint8)]).astype(np.int64)
    w = np.tile(np.array(bits, dtype=np.int64), 16)
    start = np.concatenate([[0], np.cumsum(w)[:-1]])
    j = np.arange(16)
    take = v[start[:, None] + j[None, :]] * (j[None, :] < w[:, None])
    val = (take << np.clip(w[:, None] - 1 - j[None, :], 0, 15)).sum(axis=1)
    return val.reshape(16, 8)


# ---- pins (tools/make_sbc_pins.py writes them, tests/test_sbc_domain.py and the GPU test read them) ---------------------
PINNED_KINDS = ("sync", "sub4", "m3_b8")


def pinned_names():
    """the directed streams pinned against the reference: allocation, IQUANT, 264-byte and overrun streams, and the
    bad-sync, 4-subband and mode-3 / 8-block kinds (the only other kinds whose output the reference defines: modes 1 / 2
    with 4 or 8 blocks and mono with 4 to 12 blocks are outside the domain and emit part of mono[128] uninitialised)"""
    return [n for n in streams() if not n.startswith("kind_") or n.split("_", 1)[1].rsplit("_", 1)[0] in PINNED_KINDS]


def _h(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:32]


def pin_of(pcm, pdm, undefined_frames):
    """pin of one stream's output: PCM with the reference's undefined frames zeroed, and PDM up to the first of them"""
    und = [[k * 128, (k + 1) * 128] for k in undefined_frames if (k + 1) * 128 <= pcm.size]
    p = np.array(pcm, dtype=np.int16)
    for a, b in und:
        p[a:b] = 0
    words = 2 * (und[0][0] if und else pcm.size)
    return {"samples": int(pcm.size), "pcm": _h(p), "undefined": und, "pdm_words": words, "pdm": _h(np.asarray(pdm, dtype=np.uint16)[:words])}


# ---- cuts placed on purpose for the streaming tests ------------------------------------------------------------------------
def _fs(name):
    return frame_info(streams()[name])[1][0]


def _placed_cuts():
    fs = 8 + 2 * alloc(2, 0, 28, KIND_SF)["total"]
    return {
        "max_snr_zero": [263, 3 * 264 + 263, 7 * 264 + 1, 9 * 264 + 263],            # inside 264-byte frames: 263 bytes held
        "kind_bp200_middle": [5 * fs + 3, 5 * fs + 4, 6 * fs],                       # just before and just after its header
        "kind_bp255_twice": [5 * fs + 4, 7 * fs],
        "kind_m3_b16_middle": [6 * fs, 6 * fs + 1],                                   # between the out-of-domain frame and the next
        "kind_m1_b12_last": [11 * fs, 11 * fs + 4],
        "kind_sub4_twice": [5 * fs, 7 * fs],
        "kind_mono_b4_first": [4, 8, fs + 3],                                         # frame 0 out of the domain: everything discarded
        "overrun_bp12_to_128": [3 * _fs("overrun_bp12_to_128") + 9, 10 * _fs("overrun_bp12_to_128")],
    }


class _Lazy(dict):
    def __missing__(self, key):
        self.update(_placed_cuts())
        return dict.__getitem__(self, key)

    def __iter__(self):
        if not len(self):
            self.update(_placed_cuts())
        return dict.__iter__(self)


PLACED_CUTS = _Lazy()


def held(es, cut):
    """bytes a stream holds back after its first `cut` bytes (stream not ended): all of them while the probe lacks its
    bytes (8, and 8 + 2 * total for an accepted frame 0), none once frame 0 is rejected or out of the domain, else
    everything from the first frame not decodable (its frame-size bytes and its bit loader's 8 + 2 * total bytes)"""
    es = bytes(es)[:cut]
    if len(es) < 8:
        return len(es)
    a = _hdr_alloc(es)
    if a is None or a["total"] < 0:
        return 0
    fs = 8 + 2 * a["total"]
    if len(es) < fs:
        return len(es)
    k = 0
    while (k + 1) * fs <= len(es):
        b = _hdr_alloc(es[k * fs:])
        if b is not None and b["total"] >= 0 and k * fs + 8 + 2 * b["total"] > len(es):
            break
        k += 1
    return len(es) - k * fs
