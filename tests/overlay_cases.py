"""The overlay of paced presentation, restated in Python (TEST INFRASTRUCTURE): tests/present_cases.py's Display with the
overlay state of composite() (video.cpp:839-887) staged between calls the way ef_present_overlay stages it.

The rule: changes staged before a call latch at line 0 of the first field that starts at or after the position (F, L) where
the call begins, F when L == 0 and F + 1 otherwise. A call that starts at an unchanged position latches at the same field,
so a call that never draws that line only defers the latch to the next call, which latches its own changes there too:
the field of a change is the latch field of the first call after it. Every field is drawn with the state latched at its
line 0; a latched blend b > 0 counts down at every field end (video.cpp:1193-1194).

Two rejected rules are restated beside it so that tests can show the pins tell them apart: "start_line" takes effect from
the line where the call starts drawing (field F when its overlay lines come at or after L, even where an earlier call has
already emitted F), "first_emitted" from the first field the call emits (pending while a call emits none)."""
import hashlib

import numpy as np

from tests import present_cases as pc

M32 = pc.M32
ZERO = np.zeros(1280, dtype=np.uint8)


def overlay_blend(b, blend_fc, fc):
    """_video_composite_blend on field fc after b was latched at field blend_fc"""
    d = (fc - blend_fc) & M32
    return b if b <= 0 else 0 if d >= b else b - d


class OverlayDisplay(pc.Display):
    """Display with an overlay. Fields come out as Display's tuples; overlays() gives each emitted field's
    (blend, progress, bitmap) once the calls are made."""

    def __init__(self, ntsc, frame_counter0=0, rule="line0"):
        super().__init__(ntsc, frame_counter0)
        self.fc0 = frame_counter0 & M32
        self.rule = rule
        self.overlay_top = self.bottom + 2
        self.pending = {}
        self.events = []                                # (latch field, changes) in the order they latch
        self.emitted = []                               # frame counters of every emitted field

    def stage(self, bitmap=None, blend=None, progress=None):
        """ef_present_overlay for this stream: the last write wins per attribute"""
        if blend is not None:
            assert blend >= -1
            self.pending["blend"] = int(blend)
        if progress is not None:
            self.pending["progress"] = int(progress)
        if bitmap is not None:
            self.pending["bitmap"] = np.ascontiguousarray(bitmap, dtype=np.uint8).reshape(1280).copy()

    def _call(self, fn, *a):
        F, L = self.F, self.L
        fields = fn(*a)
        out = fields[0] if isinstance(fields, tuple) else fields
        if self.pending:
            if self.rule == "line0":
                g = F + (0 if L == 0 else 1)
            elif self.rule == "start_line":
                g = F + (0 if L <= self.overlay_top else 1)
            else:
                g = out[0][0] if out else None
            if g is not None:
                self.events.append((g & M32, self.pending))
                self.pending = {}
        self.emitted += [f[0] for f in out]
        return fields

    def push(self, pts, mode=0):
        return self._call(super().push, pts, mode)

    def idle(self, n):
        return self._call(super().idle, n)

    def overlays(self):
        """(blend, progress, bitmap) of every emitted field, in emission order"""
        ev = sorted(((g - self.fc0) & M32, i, ch) for i, (g, ch) in enumerate(self.events))
        out = []
        for fc in self.emitted:
            rel = (fc - self.fc0) & M32
            b, bfc, prog, bm = 0, 0, 0, ZERO
            for g, _, ch in ev:
                if g > rel:
                    break
                if "blend" in ch:
                    b, bfc = ch["blend"], (g + self.fc0) & M32
                prog = ch.get("progress", prog)
                bm = ch.get("bitmap", bm)
            out.append((overlay_blend(b, bfc, fc), prog, bm))
        return out


class OverlayRenderer(pc.Renderer):
    """K2's field for an emitted field tuple and its overlay (via the C restatement)"""

    def field(self, f, ov=(0, 0, ZERO)):
        fc, cur, h = f
        blend, progress, bitmap = ov
        if cur < 0:
            return pc.blank_field(self.o.field_ex(self.store[0], self.store[1], self.ntsc, fc, 0, bitmap, blend, progress), self.ntsc)
        return self.o.field_ex(self.store[cur], self.store[cur ^ 1], self.ntsc, fc, h, bitmap, blend, progress)


def bitmap(seed):
    """a deterministic 16 x 80 bitmap of arbitrary bytes (composite() scales each by at most 63: no sample overflows)"""
    return np.random.default_rng(seed).integers(0, 256, size=1280, dtype=np.uint8)


def _cmd(bm=None, blend=None, progress=None):
    return {"bitmap": bm, "blend": blend, "progress": progress}


def cases():
    """the pinned cases, both standards: name -> dict(ntsc, fc0, segments [(synth seed, pts of its pictures)], modes, tail_fields,
    cmds (one per push: bitmap seed / blend / progress, None = not set), tail_cmds {t: cmd staged for field last flip + 1 + t}).
    A segment after the first is a new submit after ef_reset (video_reset() before its first push)."""
    out = {}
    for ntsc in (1, 0):
        std = "ntsc" if ntsc else "pal"
        rising = lambda n, base=129003: [base + 3003 * k for k in range(n)]            # noqa: E731
        # show_progress(180) at the first push (line 0 of the first field), progress and time bitmap every push, the whole fade
        out[std + "_fade"] = dict(ntsc=ntsc, fc0=1, segments=[(101, rising(12))], modes=[0] * 11 + [1], tail_fields=165,
                                  cmds=[_cmd(1, 180, 10)] + [_cmd(1 + k // 2 if k % 2 == 0 else None, None, 10 + 19 * k) for k in range(1, 12)],
                                  tail_cmds={})
        # blend -1 (always), 1, 5, 31, 32 (full), 0 (off); progress at 0, 240, below 0 and above 240
        out[std + "_blends"] = dict(ntsc=ntsc, fc0=3, segments=[(102, rising(10))], modes=[0] * 10, tail_fields=12,
                                    cmds=[_cmd(2, -1, 0), _cmd(None, None, 240), _cmd(3, 1, -7), _cmd(None, 5, 241), _cmd(4, 31, 1 << 30),
                                          _cmd(None, 32, -(1 << 31)), _cmd(5, 0, 239), _cmd(None, 5, 1), _cmd(6, None, 2), _cmd(None, -1, 120)],
                                    tail_cmds={})
        # changes before a mode-1 push that flips at line 1 (it emits nothing: they latch with the next call's)
        out[std + "_mode1"] = dict(ntsc=ntsc, fc0=5, segments=[(103, rising(8))], modes=[0, 0, 0, 1, 0, 0, 1, 0], tail_fields=6,
                                   cmds=[_cmd(7, 40, 20), _cmd(None, None, 30), _cmd(8, None, None), _cmd(9, 12, 60), _cmd(10, None, 61),
                                         _cmd(None, 33, 62), _cmd(11, 7, None), _cmd(None, None, 200)],
                                   tail_cmds={})
        # changes between idle runs in the tail (position line active_bottom), and the poster scroll with the overlay on
        out[std + "_tail_poster"] = dict(ntsc=ntsc, fc0=7, segments=[(104, rising(5))], modes=[0, 0, 0, 0, 3], tail_fields=17,
                                         cmds=[None, _cmd(12, -1, 100), None, None, _cmd(None, 20, None)],
                                         tail_cmds={0: _cmd(13, None, None), 1: _cmd(None, 9, 150), 4: _cmd(14, None, 5), 5: _cmd(None, -1, None),
                                                    9: _cmd(15, 3, 240)})
        # a late frame (re-latch of the timing), then ef_reset between pushes: the overlay survives both
        late = rising(8)
        late[5] -= 4 * 3003
        out[std + "_late_reset"] = dict(ntsc=ntsc, fc0=2, segments=[(105, late), (106, rising(3, 900000))], modes=[0] * 11, tail_fields=30,
                                        cmds=[None, None, None, _cmd(16, 60, 90), None, _cmd(None, None, 100), _cmd(17, None, None), None,
                                              _cmd(None, 25, None), None, _cmd(18, None, 3)],
                                        tail_cmds={})
    return out


def segment_ts(seed, pts):
    """a synthetic stream as TS with one video PES per picture, starting at its start code and carrying pts[k]"""
    from espflix_b200 import synth
    from tests import pts_cases
    es = bytes(synth.generate(synth.SEED0 + seed, n_pictures=len(pts), gop=6)[0])
    codes = pts_cases.picture_codes(es)
    assert len(codes) == len(pts)
    return pts_cases.wrap(es, [0] + [c - 3 for c in codes[1:]], ["pts"] * len(pts), [int(v) for v in pts], seed=seed + 1000)


def stage(disp, cmd):
    if cmd:
        disp.stage(None if cmd["bitmap"] is None else bitmap(cmd["bitmap"]), cmd["blend"], cmd["progress"])


def restate(case, rule="line0"):
    """the case through OverlayDisplay: (display, [("push", k, fields) / ("idle", None, fields)] in call order)"""
    d = OverlayDisplay(case["ntsc"], case["fc0"], rule)
    fields, k, last = [], 0, None
    for si, (_, pts) in enumerate(case["segments"]):
        if si:
            d.reset()
        for p in pts:
            stage(d, case["cmds"][k])
            f, last, _ = d.push(int(p), case["modes"][k])
            fields.append(("push", k, f))
            k += 1
    total = (last + 1 + case["tail_fields"] - case["fc0"]) & M32         # as present_cases.schedule: the tail after the last flip
    while len(d.emitted) < total:
        stage(d, case["tail_cmds"].get((d.F + (0 if d.L == 0 else 1) - last - 1) & M32))
        fields.append(("idle", None, d.idle(1)))
    return d, fields


def rendered(case, frames, oracle, rule="line0"):
    """the case's field stream as K2 draws the restatement: (SHA-256 of the whole stream, per-field SHA-256, blend of every
    field). frames[i]: the decoded pictures of segment i; ef_reset zero-fills the frame stores before a later segment."""
    d, calls = restate(case, rule)
    ovs = d.overlays()
    r = OverlayRenderer(oracle, case["ntsc"])
    seg = [(si, j) for si, (_, pts) in enumerate(case["segments"]) for j in range(len(pts))]
    whole, per, i = hashlib.sha256(), [], 0
    for kind, k, fields in calls:
        if kind == "push":
            si, j = seg[k]
            if si and j == 0:
                r.reset()
            r.decoded(j, frames[si][j])
        for f in fields:
            b = r.field(f, ovs[i]).tobytes()
            whole.update(b)
            per.append(hashlib.sha256(b).hexdigest())
            i += 1
    return whole.hexdigest(), per, [int(b) for b, _, _ in ovs]


def overlay_band(template, bitmaps, blend, progress, ntsc):
    """composite() restated in torch for many fields at once: the 16 lines from active_bottom + 2 of every field (int32
    [fields, 16, W]) from the same lines with the overlay off (template [16, W]), the bitmap (uint8 [fields, 1280]), blend and
    progress (int [fields]) each field is drawn with"""
    import torch
    x0 = (160 if ntsc else 280) + 16                    # blit start + 16 (video.cpp:845-853)
    n, w = blend.shape[0], template.shape[1]
    blend = blend.to(torch.int32).view(n, 1, 1)
    scale = torch.where((blend == -1) | (blend >= 32), torch.full_like(blend, 63), (63 * blend) >> 5)
    out = template.to(torch.int32).unsqueeze(0).repeat(n, 1, 1)
    bm = bitmaps.to(torch.int32).view(n, 16, 80).repeat_interleave(2, dim=2)
    out[:, :, x0:x0 + 160] = 0x1800 + bm * scale
    step = torch.arange(480, device=template.device).view(1, 1, 480) // 4 * 2
    bar = 0x1800 + torch.where(step < progress.to(torch.int64).view(n, 1, 1), scale << 8, scale << 7)
    out[:, 3:9, x0 + 176:x0 + 656] = bar.expand(n, 6, 480)
    return torch.where(blend != 0, out, template.to(torch.int32).unsqueeze(0).expand(n, 16, w))
