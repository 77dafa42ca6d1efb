"""The clock of paced presentation, restated in Python (TEST INFRASTRUCTURE): ESPFlix::update_progress() (espflix.cpp:862-874)
with idx_hdr::pts2pts (espflix.cpp:589-604) and show_time() / Render (espflix.cpp:62-174), as ef_present_clock runs it per stream.

All arithmetic is C's: int64 products, division truncating toward zero, and the (int) casts wrapping to 32 bits. Python's // and
% round toward minus infinity, so they are not used on values that may be negative.

The model: during the push of picture k, get_pts() is pts(k) (flush_picture(), player.cpp:692-700), so update_progress() runs
once at the start of the present call that pushes k; a stream with no picture at that index, and an idle call, read the stream's
most recent pts (ef_picture_pts's last_pts). What it stages latches by the overlay's rule (tests/overlay_cases.py)."""
import functools
import hashlib
import json
import os
import struct

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FONT = os.path.join(GOLDEN, "font8.bin")
PINS = os.path.join(GOLDEN, "clock_pins.json")
STOP, PAUSE, PLAY, FFWD, RWND = 0x18, 0x19, 0x1A, 0x1B, 0x1C          # enum Icon, espflix.cpp:53-59
COLOR = 240                                                             # Render::_color
PROGRESS_WIDTH = 240                                                    # VIDEO_COMPOSITE_PROGRESS_WIDTH


def c_div(a, b):
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def c_mod(a, b):
    return a - b * c_div(a, b)


def to_int(v):
    """C's (int) of an int64 on the targets the reference runs on: the low 32 bits"""
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def font():
    """tests/golden/font8.bin -> (atlas uint8 [16, 1024], rights int16 [n]): the reference's _font8 and _font8_rights"""
    raw = open(FONT, "rb").read()
    return np.frombuffer(raw[:16 * 1024], dtype=np.uint8).reshape(16, 1024), np.frombuffer(raw[16 * 1024:], dtype="<i2").astype(np.int16)


def header(video, fwd, rwd):
    """the 104-byte video.idx header (idx_hdr) with records (first_pts, last_pts); bin_size, trick_speed and sample_count are
    not read by the clock and carry arbitrary values"""
    recs = b"".join(struct.pack("<qqIII4x", f, l, 90000 * (i + 1), (1, 8, 8)[i], 77 + i) for i, (f, l) in enumerate((video, fwd, rwd)))
    return struct.pack("<II", 0x00584449, 3) + recs


def parse_header(h):
    v = struct.unpack_from("<qq", h, 8), struct.unpack_from("<qq", h, 40), struct.unpack_from("<qq", h, 72)
    return v


def pts2pts(hdr, pts, speed):
    (vf, vl), (ff, fl), (rf, rl) = parse_header(hdr)
    if speed == 1:
        return vf + c_div((pts - ff) * (vl - vf), fl - ff)
    if speed == -1:
        return vl - c_div((pts - rf) * (vl - vf), rl - rf)
    return pts


def time_text(s, icon):
    """show_time()'s sprintf (espflix.cpp:165-171) with C's / and %"""
    m = c_div(s, 60)
    h = c_div(m, 60)
    if h:
        return "%c %d:%02d:%02d" % (icon, h, c_mod(m, 60), c_mod(s, 60))
    return "%c   %02d:%02d" % (icon, c_mod(m, 60), c_mod(s, 60))


def text_width(text, rights):
    return sum(int(rights[ord(c) - 0x18]) - (int(rights[ord(c) - 0x19]) if ord(c) > 0x18 else 0) for c in text)


def render(text, atlas, rights):
    """erase(), then draw_text(0, 0, text) into the 80 x 16 bitmap, written the way the reference writes it: glyph by glyph, row
    by row, through p32(); rows are contiguous, so x >= 80 lands in the next row; bytes past the bitmap are dropped"""
    out = [0] * 1280
    x = 0
    for ch in text:
        c = ord(ch) - 0x18
        left = int(rights[c - 1]) if c else 0
        w = int(rights[c]) - left
        for y in range(16):
            for j in range(w):
                L = y * 80 + x + j
                if L >= 1280:
                    continue
                p = int(atlas[y, left + j])
                if p:
                    out[L] = (COLOR * p + (255 - p) * out[L]) >> 8
        x += w
    return np.array(out, dtype=np.uint8)


@functools.lru_cache(maxsize=4096)
def _rendered(text):
    atlas, rights = font()
    return render(text, atlas, rights)


def icon_of(speed, paused):
    return (PAUSE if paused else PLAY) if speed == 0 else FFWD if speed == 1 else RWND


class Clock:
    """one stream's clock: its header, speed, flags and _last_seconds. step() is update_progress() without its commit."""

    def __init__(self):
        self.hdr, self.speed, self.flags, self.last_seconds = header((0, 1), (0, 1), (0, 1)), 0, 0, 0

    def set(self, hdr, speed, flags):
        self.hdr, self.speed, self.flags = bytes(hdr), int(speed), int(flags) & 3
        if flags & 4:
            self.last_seconds = 0

    @property
    def on(self):
        return bool(self.flags & 1)

    def step(self, pts, atlas=None, rights=None):
        """-> (bitmap or None when the second did not change, progress, seconds); None when the clock is off. atlas None: the
        font of tests/golden/font8.bin, each text rendered once"""
        if not self.on:
            return None
        main = pts2pts(self.hdr, pts, self.speed)
        seconds = to_int(c_div(main, 90000))
        text = time_text(seconds, icon_of(self.speed, self.flags & 2))
        bm = None
        if seconds != self.last_seconds:
            bm = _rendered(text) if atlas is None else render(text, atlas, rights)
        return bm, to_int(c_div(main * PROGRESS_WIDTH, parse_header(self.hdr)[0][1])), seconds

    def commit(self, stepped):
        if stepped is not None:
            self.last_seconds = stepped[2]


# ---- the pinned cases: a sequence of update_progress() calls each, on a fresh player (_last_seconds 0, bitmap erased) ----------
# a step: (header, speed, paused, zero_last_seconds, get_pts())
H_MAIN = header((3003, 90000 * 3700), (900, 900 + 3 * 90000 * 370), (1000, 1000 + 7 * 90000 * 529))      # a 1 h 1 min 40 s title
H_ODD = header((5, 10 ** 9 + 7), (-17, 333331), (12, 3 * 7 * 11 * 13 * 1001))                        # map_pts truncates
H_LONG = header((0, 90000 * 400 * 3600), (0, 90000 * 1000), (0, 90000 * 999))                       # 400 hours


def _seq(hdr, speed, paused, pts_list, zero=()):
    return [(hdr, speed, paused, i in zero, p) for i, p in enumerate(pts_list)]


def cases():
    S = 90000
    return {
        "icon_play": _seq(H_MAIN, 0, 0, [62 * S + 5]),
        "icon_pause": _seq(H_MAIN, 0, 1, [62 * S + 5]),
        "icon_ffwd": _seq(H_MAIN, 1, 0, [900 + 3 * 62 * S]),
        "icon_rwnd": _seq(H_MAIN, -1, 0, [1000 + 7 * 5 * S]),
        "zero_seconds_last_zero": _seq(H_MAIN, 0, 0, [0, 45000, -1]),
        "zero_seconds_last_nonzero": _seq(H_MAIN, 0, 0, [7 * S, 0]),
        "seconds_59_60_3599_3600": _seq(H_MAIN, 0, 0, [59 * S, 60 * S, 3599 * S, 3600 * S, 3600 * S + 89999]),
        "hours_one_digit": _seq(H_MAIN, 0, 0, [(3600 + 2 * 60 + 3) * S]),
        "hours_two_digits": _seq(H_LONG, 0, 0, [(10 * 3600 + 11 * 60 + 12) * S]),
        "hours_three_digits_wrap": _seq(H_LONG, 0, 0, [(100 * 3600 + 1) * S, (388 * 3600 + 58 * 60 + 59) * S]),
        "negative_pts_minus_one": _seq(H_MAIN, 0, 0, [-1]),
        "negative_rewind_past_end": _seq(H_MAIN, -1, 0, [1000 + 7 * 90000 * 529 + 7 * 5 * S + 3, 1000 + 7 * 90000 * 529 + 7 * 3725 * S + 11]),
        "negative_ffwd_before_start": _seq(H_MAIN, 1, 0, [900 - 3 * 3 * S - 1, 900 - 3 * 3725 * S - 2, -1]),
        "negative_hours_paused": _seq(H_LONG, 0, 1, [-(3 * 3600 + 62) * S - 1, -(36 * S)]),
        "trick_truncation_ffwd": _seq(H_ODD, 1, 0, [-18, -17, 0, 1, 333330, 333331, 333332, 10 ** 7]),
        "trick_truncation_rwnd": _seq(H_ODD, -1, 0, [11, 12, 13, 3 * 7 * 11 * 13 * 1001 + 1, -(10 ** 6), 10 ** 8]),
        "progress_below_zero_above_240": _seq(H_MAIN, 0, 0, [-90000 * 40, 90000 * 3700, 90000 * 3700 + 1, 90000 * 7401]),
        "last_seconds_quirk": [(H_MAIN, 0, 0, False, 10 * S), (H_MAIN, 0, 0, False, 0), (H_MAIN, 0, 0, False, 4 * S),
                               (H_MAIN, 0, 1, True, 4 * S), (H_MAIN, 0, 0, True, 0), (H_MAIN, 0, 0, False, 0),
                               (H_MAIN, 1, 0, False, 900 + 3 * 4 * S), (H_MAIN, 0, 0, True, 4 * S + 1)],
        "speed_changes": [(H_MAIN, 0, 0, False, 100 * S), (H_MAIN, 1, 0, False, 900 + 3 * 100 * S), (H_MAIN, 1, 0, False, 900 + 3 * 160 * S),
                          (H_MAIN, -1, 0, False, 1000 + 7 * (3700 - 160) * S), (H_MAIN, 0, 1, True, 160 * S), (H_MAIN, 0, 0, False, 161 * S)],
    }


def restate(steps, atlas, rights):
    """-> one (sha256 of the bitmap, progress, _last_seconds) per step"""
    clk, bm, out = Clock(), np.zeros(1280, dtype=np.uint8), []
    for hdr, speed, paused, zero, pts in steps:
        clk.set(hdr, speed, 1 | (2 if paused else 0) | (4 if zero else 0))
        r = clk.step(pts, atlas, rights)
        clk.commit(r)
        if r[0] is not None:
            bm = r[0]
        out.append((hashlib.sha256(bm.tobytes()).hexdigest(), r[1], clk.last_seconds))
    return out


def pins():
    return json.load(open(PINS))
