"""Helpers the test modules share (TEST INFRASTRUCTURE): hashing, error codes, cutting TS into submits, presenting contexts
and their calls, overlay staging, the paced-presentation driver that checks a context call by call against the
restatement, and the decode-and-compare helpers of the block- and syntax-level streams. Nothing here is collected as a
test; torch is imported only where a device buffer is needed, so CPU tests can use the module too."""
import hashlib

import numpy as np

from tests import overlay_cases as oc
from tests import present_cases as pc

I420 = 352 * 192 * 3 // 2


def sha(a):
    """SHA-256 hex digest of a bytes object or of an array's bytes"""
    return hashlib.sha256(a if isinstance(a, bytes) else np.ascontiguousarray(a).tobytes()).hexdigest()


def error_code(fn):
    """the code of the EspflixError fn() raises"""
    import pytest

    import espflix_b200
    with pytest.raises(espflix_b200.EspflixError) as e:
        fn()
    return e.value.code


def submits(per_stream, empty=b"", n=0):
    """per-stream lists of TS chunks -> per-submit lists of every stream's chunk: at least n submits, a stream that has no
    chunk left gets `empty`"""
    K = max([n] + [len(c) for c in per_stream])
    return [[c[k] if k < len(c) else empty for c in per_stream] for k in range(K)]


# ---- presentation ----------------------------------------------------------------------------------------------------------
def presenting_context(n, ntsc, fc0=None, max_pictures=13, es_capacity=None, carry=None, font=None):
    """a context with PTS and paced presentation enabled; carry: ef_carry_enable(carry) first; font: (atlas, rights) to load"""
    import espflix_b200
    ctx = espflix_b200.Context(n_streams=n, max_pictures=max_pictures, max_slices_per_picture=12,
                               es_capacity=es_capacity or n * max_pictures * 40000, fields=False)
    ctx.enable_pts()
    if carry is not None:
        ctx.enable_carry(carry)
    ctx.video_init(ntsc)
    ctx.enable_present(fc0)
    if font is not None:
        ctx.present_font(*font)
    return ctx


def host_fields(fields):
    """fields [n, samples] (uint16 on the device) -> numpy uint16"""
    import torch
    return fields.view(torch.int16).cpu().numpy().view(np.uint16)


def present_call(ctx, fn, device=False):
    """fn(out): a present call. A sizing call, then the call into a buffer of exactly that size; the sizing call must report
    what the call did -> (info, fields [total, samples] uint16: on the host, or on the device when `device`)"""
    import torch
    w, nl = ctx.geometry()
    info = fn(None)
    total = int(info["n_fields"].sum())
    out = torch.empty(max(total, 1) * w * nl, dtype=torch.uint16, device="cuda")
    got = fn(out)
    assert (got == info).all()                          # the sizing call reported what the call did
    fields = out[:total * w * nl].view(total, w * nl)
    return got, fields if device else host_fields(fields)


def overlay_arrays(cmds):
    """overlay_cases' commands, one per stream (None: nothing set) -> ef_present_overlay's (bitmap, blend, progress, set)"""
    n = len(cmds)
    bm, bl, pr, st = np.zeros((n, 1280), np.uint8), np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint8)
    for s, c in enumerate(cmds):
        if not c:
            continue
        if c["bitmap"] is not None:
            bm[s], st[s] = oc.bitmap(c["bitmap"]), st[s] | 1
        if c["blend"] is not None:
            bl[s], st[s] = c["blend"], st[s] | 2
        if c["progress"] is not None:
            pr[s], st[s] = c["progress"], st[s] | 4
    return bm, bl, pr, st


def stage_overlay(ctx, disps, cmds):
    """one ef_present_overlay call for every stream, and the same changes in the restatement's displays"""
    for d, c in zip(disps, cmds):
        oc.stage(d, c)
    ctx.present_overlay(*overlay_arrays(cmds))


class Paced:
    """Drives a presenting context over TS submits and present calls, and the restatement alongside it: one display and one
    renderer per stream (present_cases' or overlay_cases'), and frames[s][g], stream s's decoded picture g (counted since
    `seen` was last zeroed). Every call checks the info against the restatement: the sizing call's info, consecutive frame
    counters, each pushed picture's flip (flags 0) and no flip on a stream without a picture. Per stream it keeps the pts and
    flip of every pushed picture, the SHA-256 of every field the device emitted (dev) and of the restatement's rendering of
    it (want), and the SHA-256 of the whole field stream."""

    def __init__(self, ctx, disps, rends, frames):
        n = len(disps)
        self.ctx, self.disp, self.rend, self.frames, self.n = ctx, disps, rends, frames, n
        self.seen = [0] * n
        self.dev = [[] for _ in range(n)]
        self.want = [[] for _ in range(n)]
        self.stream_hash = [hashlib.sha256() for _ in range(n)]
        self.flips = [[] for _ in range(n)]
        self.pts = [[] for _ in range(n)]
        self.fc = [d.F for d in disps]

    def render(self, s, fields):
        """the restatement's rendering of the fields a call emitted on stream s"""
        return [self.rend[s].field(f) for f in fields]

    def collect(self, info, host, want):
        """one call's info and fields (host [total, samples]) against want[s], the fields the restatement emitted"""
        for s in range(self.n):
            a, k = int(info[s]["first"]), int(info[s]["n_fields"])
            assert k == len(want[s]), (s, k, len(want[s]))
            if k:
                assert int(info[s]["frame_counter"]) == self.fc[s] & pc.M32    # consecutive frame counters over all calls
            self.fc[s] += k
            for j, f in enumerate(self.render(s, want[s])):
                b = host[a + j].tobytes()
                self.stream_hash[s].update(b)
                self.dev[s].append(hashlib.sha256(b).hexdigest())
                self.want[s].append(hashlib.sha256(f.tobytes()).hexdigest())

    def submit(self, chunk, mode_of=None, ends=None, use_async=False, before_call=None):
        """one TS submit (ef_end_streams(ends) before ef_index when any end) and a present call per picture index,
        synchronous or asynchronous. mode_of(s, g): the mode of stream s's picture g (None: 0). before_call(p, pushes): called
        before picture index p is pushed; pushes[s]: stream s has that picture."""
        import torch

        from espflix_b200 import capi
        ctx = self.ctx
        ctx.submit_ts(*ctx.pack(chunk))
        if ends is not None and any(ends):
            ctx.end_streams(np.array(ends, dtype=np.uint8))
        ctx.index()
        npics = ctx.index_info()["max_pictures"]
        counts = [ctx.stream_info(s)[0] for s in range(self.n)]
        pic_pts, _ = ctx.picture_pts()
        for p in range(npics):
            pushes = [p < c for c in counts]
            if before_call:
                before_call(p, pushes)
            modes = [mode_of(s, self.seen[s] + p) if mode_of and pushes[s] else 0 for s in range(self.n)]
            want = [[] for _ in range(self.n)]
            for s in range(self.n):
                if pushes[s]:
                    g = self.seen[s] + p
                    self.rend[s].decoded(g, self.frames[s][g])
                    want[s], _, _ = self.disp[s].push(int(pic_pts[s, p]), modes[s])
                    self.pts[s].append(int(pic_pts[s, p]))
            if use_async:
                w, nl = ctx.geometry()
                total = int(ctx.present_picture(p, modes)["n_fields"].sum())        # synchronous sizing call
                out = torch.empty(max(total, 1) * w * nl, dtype=torch.uint16, device="cuda")
                info_t = ctx.present_picture_async(p, out, modes=modes)
                assert ctx.present_wait() == (capi.EF_OK, 1)
                info = ctx.present_info(info_t)
                host = host_fields(out[:total * w * nl].view(total, w * nl))
            else:
                info, host = present_call(ctx, lambda o: ctx.present_picture(p, modes, o))
            for s in range(self.n):
                if pushes[s]:
                    self.flips[s].append((int(info[s]["flip_field"]), int(info[s]["flip_line"])))
                    assert self.flips[s][-1] == (self.disp[s].F, self.disp[s].L - 1)
                    assert int(info[s]["flags"]) == 0
                else:
                    assert int(info[s]["flip_line"]) == -1 and int(info[s]["n_fields"]) == 0
            self.collect(info, host, want)
        self.seen = [a + b for a, b in zip(self.seen, counts)]

    def idle(self, n_fields, before_call=None):
        """one ef_present_idle of n_fields (one per stream, or one for all); before_call(): called first"""
        if before_call:
            before_call()
        n_fields = [int(x) for x in np.broadcast_to(n_fields, (self.n,))]
        want = [self.disp[s].idle(n_fields[s]) for s in range(self.n)]
        self.collect(*present_call(self.ctx, lambda o: self.ctx.present_idle(n_fields, o)), want)

    def check(self):
        """every field the device emitted equals the restatement's rendering"""
        for s in range(self.n):
            assert len(self.dev[s]) == len(self.want[s])
            bad = [i for i, (a, b) in enumerate(zip(self.dev[s], self.want[s])) if a != b]
            assert not bad, "stream %d: fields %s differ from the restatement" % (s, bad[:8])


# ---- audio -----------------------------------------------------------------------------------------------------------------
def audio_results(info, pcm, pdm):
    """ef_decode_audio_async's info and device PCM / PDM -> ef_decode_audio's per-stream results"""
    import torch

    import espflix_b200
    out = []
    for i in espflix_b200.Context.audio_info(info):
        a, k = int(i["pcm_offset"]), int(i["n_frames"]) * 128
        out.append({"frame_size": int(i["frame_size"]), "n_frames": int(i["n_frames"]),
                    "pcm": pcm[a:a + k].view(torch.int16).cpu().numpy(), "pdm": pdm[2 * a:2 * (a + k)].view(torch.int16).cpu().numpy().view(np.uint16)})
    return out


def same_audio(a, b, what):
    """two calls' per-stream audio results are equal"""
    assert len(a) == len(b)
    for s, (x, y) in enumerate(zip(a, b)):
        assert x["frame_size"] == y["frame_size"] and x["n_frames"] == y["n_frames"], "%s stream %d" % (what, s)
        assert np.array_equal(x["pcm"].astype(np.int16), y["pcm"].astype(np.int16)), "%s stream %d: PCM" % (what, s)
        assert np.array_equal(x["pdm"].astype(np.uint16), y["pdm"].astype(np.uint16)), "%s stream %d: PDM" % (what, s)


# ---- block- and syntax-level streams ---------------------------------------------------------------------------------------
def decode_es_batch(streams, n_pictures):
    """one ES submit of every stream, every picture to the host: (out[picture][stream], pictures per stream)"""
    import espflix_b200
    ctx = espflix_b200.Context(n_streams=len(streams), max_pictures=12, max_slices_per_picture=12,
                               es_capacity=sum(len(s) for s in streams) + 4096, fields=False)
    blob, off = ctx.pack(streams)
    ctx.submit_es(blob, off)
    ctx.index()
    counts = [ctx.stream_info(i)[0] for i in range(len(streams))]
    out = np.zeros((n_pictures, len(streams), I420), dtype=np.uint8)
    ctx.decode_all_to_host(n_pictures, out)
    ctx.sync()
    ctx.close()
    return out, counts


def first_difference(got, ref):
    """plane, macroblock (mx, my) and block of the first differing byte of two I420 pictures"""
    i = int(np.nonzero(got != ref)[0][0])
    if i < 352 * 192:
        x, y = i % 352, i // 352
        return "Y mb (%d, %d) block %d, got %d want %d" % (x // 16, y // 16, (x >> 3 & 1) | (y >> 3 & 1) << 1, got[i], ref[i])
    j = (i - 352 * 192) % (176 * 96)
    plane, blk = ("Cr", 4) if i < 352 * 192 + 176 * 96 else ("Cb", 5)
    return "%s mb (%d, %d) block %d, got %d want %d" % (plane, j % 176 // 8, j // 176 // 8, blk, got[i], ref[i])


def check_picture(pins, name, k, got, ref):
    """picture k of case `name` equals the restatement's and, for a pinned case, the reference's pin"""
    import pytest
    if not np.array_equal(got, ref):
        pytest.fail("%s picture %d differs from the restatement: %d bytes, first at %s" % (name, k, int((got != ref).sum()), first_difference(got, ref)))
    if name in pins:
        assert sha(got) == pins[name]["frame_sha256"][k], "%s picture %d differs from the reference's pin" % (name, k)
