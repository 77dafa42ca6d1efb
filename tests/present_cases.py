"""Paced presentation, restated in Python (TEST INFRASTRUCTURE): the display of one stream under the instant-decoder model
of efo_paced_schedule_ex, cut into pushes and idle runs the way ef_present_picture / ef_present_idle cut it.

A push of (pts, mode) at the display's position (frame counter F, next line L) first runs push_video's arithmetic
(video.cpp:1023-1057), then draws lines from (F, L) until the flip (video_isr, video.cpp:1122-1198): the first line below
vsync_start that is not an active line of a presented frame, once F >= _next_frame_time. animate() (video.cpp:1076-1088)
runs at the flip and at the end of every field. The fields a run emits are those whose line active_bottom - 1 it draws.
Flips happen on blank lines only, so a field's picture lines never straddle a change of state: each emitted field is one
K2 field of (current store, other store, hscroll, F).

Frame stores follow the device: picture k of a stream (counted over all submits since the last reset) lives in store
(k + 1) & 1, and a reset zero-fills both stores."""
import numpy as np

EASD = (0, 8, 16, 24, 48, 72, 104, 136, 176, 216, 248, 280, 304, 328, 336, 344)   # _easd, video.cpp:1077
M32 = 0xFFFFFFFF


def geometry(ntsc):
    """(line_count, active_top, active_bottom, vsync_start), video.cpp:1135-1137"""
    lines = 262 if ntsc else 312
    top = 32 if ntsc else 64
    return lines, top, top + 192, lines - (3 if ntsc else 8)


def hscroll_of(ai):
    """_hscroll after an animate() call that left _animate_index at ai"""
    return -EASD[-ai] if ai < 0 else EASD[ai]


def animate(ai, n):
    """_animate_index after n animate() calls"""
    return 0 if abs(ai) <= n else ai - n if ai > 0 else ai + n


class Display:
    """One stream's display. Fields come out as tuples (frame_counter, current store or -1 before any flip, hscroll)."""

    def __init__(self, ntsc, frame_counter0=0):
        self.ntsc = ntsc
        self.lines, self.top, self.bottom, self.vsync = geometry(ntsc)
        self.F, self.L = frame_counter0 & M32, 0
        self.pts_origin, self.fc_origin = 0, 0          # _pts_origin, _video_frame_counter_origin
        self.cur = -1                                   # current frame store; -1: no frame presented yet
        self.ai = 0                                     # _animate_index (_hscroll = hscroll_of(ai), _animate is 0 between pushes)
        self.pictures = 0                               # pictures pushed since the last reset: picture k goes to store (k + 1) & 1
        self.out_of_domain = False

    def reset(self):
        """video_reset() (video.cpp:1070-1074): the next push latches a new origin. Position, store and scroll stay."""
        self.fc_origin = 0
        self.pictures = 0

    def _fields(self, first, n):
        """n fields from offset `first` (0 = the field at self.F), with the field-end animate() calls in between"""
        return [((self.F + first + j) & M32, self.cur, hscroll_of(animate(self.ai, first + j))) for j in range(n)]

    def push(self, pts, mode=0):
        """-> (emitted fields, flip frame counter, flip line); (None, None) for an unpushed picture (pts -1, mode 0)"""
        store = (self.pictures + 1) & 1
        self.pictures += 1
        if pts == -1 and mode == 0:                     # flush_picture() skips it (player.cpp:692-702): outside the domain
            self.out_of_domain = True
            return [], None, None
        F, L = self.F, self.L
        vp = (abs(pts) // (1500 if self.ntsc else 1800) * (1 if pts >= 0 else -1)) & M32    # C division truncates towards zero
        if self.fc_origin == 0:
            self.pts_origin, self.fc_origin = vp, F
        d = (vp - self.pts_origin + self.fc_origin) & M32
        anim = 0
        if mode:
            d, anim = F, mode
        late = (F - d) & M32
        if d < F and (late if late < 1 << 31 else late - (1 << 32)) > 2:
            self.fc_origin = 0                          # more than two fields late (int late, video.cpp:1047): re-latch at the next push
        # the flip: the first eligible line at or after (F, L)
        if d <= F:
            lo = [(0, self.vsync)] if self.cur == -1 else [(0, self.top), (self.bottom, self.vsync)]
            fl = next((max(L, a) for a, b in lo if max(L, a) < b), None)
            ff = 0 if fl is not None else 1
            if fl is None:
                fl = 0
        else:
            ff, fl = d - F, 0                           # fields from F to the flip
        first = 0 if L <= self.bottom - 1 else 1
        last = ff if fl >= self.bottom - 1 else ff - 1
        fields = self._fields(first, max(0, last - first + 1))
        ai = animate(self.ai, ff)
        if anim == 2:
            ai = -16
        elif anim == 3:
            ai = 16
        self.ai = animate(ai, 1)
        self.F, self.L = (F + ff) & M32, fl + 1
        self.cur = store
        return fields, (F + ff) & M32, fl

    def idle(self, n):
        """the display runs on with nothing pending until it has emitted n more fields"""
        if n <= 0:
            return []
        first = 0 if self.L <= self.bottom - 1 else 1
        fields = self._fields(first, n)
        end = first + n - 1
        self.ai = animate(self.ai, end)
        self.F, self.L = (self.F + end) & M32, self.bottom
        return fields


def schedule(pts, modes, ntsc, frame_counter0, tail_fields):
    """efo_paced_schedule_ex through the push / idle cut: (fields, flip_field, flip_line, hscroll per field, fields per
    push, the whole field list). The idle run after the last push emits the rest of the field holding the last flip and
    tail_fields more."""
    d = Display(ntsc, frame_counter0)
    out, ff, fl, per = [], [], [], []
    for p, m in zip(pts, modes):
        f, a, b = d.push(int(p), int(m))
        out += f
        per.append(len(f))
        ff.append(a)
        fl.append(b)
    end = (ff[-1] + 1 + tail_fields - frame_counter0) & M32
    out += d.idle(end - len(out))
    return len(out), ff, fl, [h for _, _, h in out], per, out


def irregular_cases():
    """(pts, ntsc, frame_counter0, modes, tail_fields) of 24 schedules with jitter, repeated and decreasing PTS (late
    frames, 'resetting v timing') and long gaps, both standards"""
    rng = np.random.default_rng(2024)
    for case in range(24):
        ntsc = case % 2
        n = int(rng.integers(2, 14))
        step = rng.choice([3003, 3003, 3003, 1501, 6006, 0, -4000, 45045], size=n)
        pts = (129003 + np.cumsum(step)).astype(np.int64)
        pts = np.maximum(pts, 0)
        fc0 = int(rng.integers(0, 4)) if case < 8 else int(rng.integers(1, 100000))
        modes = np.where(rng.random(n) < 0.2, rng.integers(1, 4, size=n), 0).astype(np.int32)      # 1 at once, 2 / 3 poster scroll
        tail = int(rng.integers(0, 20))
        yield pts, ntsc, fc0, modes, tail


def irregular_programs():
    """the 24 irregular schedules as TS programs, one PES per picture carrying the pinned pts:
    [(case, ts, pts, ntsc, frame_counter0, modes, tail_fields)]"""
    from tests.overlay_cases import segment_ts
    return [(case, segment_ts(200 + case, pts), [int(v) for v in pts], ntsc, fc0, [int(m) for m in modes], tail)
            for case, (pts, ntsc, fc0, modes, tail) in enumerate(irregular_cases())]


def synth_ts(seed, n):
    """synthetic stream `seed` of n pictures as TS"""
    from espflix_b200 import synth
    es, off = synth.generate(synth.SEED0 + seed, n_pictures=n)
    return synth.wrap_ts(es, off)


def blank_field(field, ntsc):
    """a field with no frame presented (video.cpp:1140): active lines are blanking lines, which repeat with period 2"""
    lines, top, bottom, _ = geometry(ntsc)
    f = field.reshape(lines, -1).copy()
    for i in range(top, bottom):
        f[i] = f[top - 2 + ((i - top) & 1)]
    return f.reshape(-1)


class Renderer:
    """K2's field for an emitted field tuple, from the pictures a stream's stores hold (via the C restatement)"""

    def __init__(self, oracle, ntsc):
        self.o, self.ntsc = oracle, ntsc
        self.store = [np.zeros(101376, dtype=np.uint8), np.zeros(101376, dtype=np.uint8)]
        self._blank = None

    def reset(self):
        self.store = [np.zeros(101376, dtype=np.uint8), np.zeros(101376, dtype=np.uint8)]

    def decoded(self, k, i420):
        """picture k (counted since the last reset) was decoded"""
        self.store[(k + 1) & 1] = i420

    def field(self, f):
        fc, cur, h = f
        if cur < 0:
            if self._blank is None:
                self._blank = blank_field(self.o.field_ex(self.store[0], self.store[1], self.ntsc, 0), self.ntsc)
            return self._blank
        return self.o.field_ex(self.store[cur], self.store[cur ^ 1], self.ntsc, fc, h)
