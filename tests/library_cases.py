"""tests/library_cases.py — the title library (ef_library_*) restated in Python (TEST INFRASTRUCTURE): ESPFlix's play / skip /
fast_forward / rewind / play_pause / get_index / save_pos (espflix.cpp:787-859) with idx_hdr::pts2pts and pts2offset
(espflix.cpp:589-629), and the Streamer reads of every submit (espflix.cpp:723-747).

All arithmetic is C's. pts2offset's quirks are kept: the pts is clamped to [video.first_pts, video.last_pts]; at speed 0 the
int64 difference is divided by bin_size before the uint32 cast; at speed 1 the uint32 cast comes before the two unsigned
divisions; at speed -1 first_pts is subtracted a second time and the difference wraps in uint32; every min() is unsigned. The
sample read is at byte pts2offset(pos, speed) of video.idx, and the byte offset played is the sample x 188.

Commands (one per ESPFlix method) -> the restart op the library runs with it:
  PLAY_AT(title, pos)  nav(title) with pos, then play_pause() from NAV                 1
  PLAY                 play(nav, 0, get_index(0, pos) * 188)                           1
  SKIP(s)              skip(s): pos += (int)(s * 90000), unclamped; then PLAY             1
  FAST_FORWARD/REWIND  play at speed +-1 from get_index(+-1, pos)                      1
  PAUSE                a PLAYING stream becomes PAUSED                                  0
  RESUME               video_pause(0): a PAUSED stream plays on from its cursor         2
  STOP                 the stream gets no more bytes                                   0
Every command but PLAY_AT and RESUME first saves pos = pts2pts(get_pts(), speed) on a PLAYING stream (save_pos). A submit gives
every PLAYING stream min(budget, packets left) packets from its cursor; the stream whose cursor reaches the end of its file ends
with that submit, with pos = pts2pts(0, speed) (save_pos(0) at DONE).

loop_command() restates the pause handshake of ESPFlix::loop() (espflix.cpp:906-939), which runs in the reference's UI thread:
which command a key turns into once the decoder has paused."""
import os
import struct

M32 = 0xFFFFFFFF
HDR = 104
PLAY_AT, PLAY, SKIP, FAST_FORWARD, REWIND, PAUSE, RESUME, STOP = range(8)
IDLE, PLAYING, PAUSED, STOPPED, ENDED = range(5)
OP = {PLAY_AT: 1, PLAY: 1, SKIP: 1, FAST_FORWARD: 1, REWIND: 1, PAUSE: 0, RESUME: 2, STOP: 0}
NAMES = ["PLAY_AT", "PLAY", "SKIP", "FAST_FORWARD", "REWIND", "PAUSE", "RESUME", "STOP"]


def c_div(a, b):
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def to_i32(v):
    v &= M32
    return v - (1 << 32) if v >= 1 << 31 else v


def parse(idx):
    """video.idx image -> dict of the three records: (first, last, bin_size, trick_speed, sample_count)"""
    sig, n = struct.unpack_from("<II", idx, 0)
    recs = [struct.unpack_from("<qqIII", idx, 8 + 32 * k) for k in range(3)]
    return {"sig": sig, "len": n, "video": recs[0], "fwd": recs[1], "rwd": recs[2]}


def header(video, fwd, rwd):
    """a 104-byte idx_hdr from three (first, last, bin_size, trick_speed, sample_count) records"""
    return struct.pack("<II", 0x00584449, 3) + b"".join(struct.pack("<qqIII4x", *r) for r in (video, fwd, rwd))


def image(video, fwd, rwd, samples):
    """a video.idx image: the header, then the main, fwd and rwd samples (uint32 each) back to back"""
    return header(video, fwd, rwd) + struct.pack("<%dI" % len(samples), *samples)


def pts2pts(h, pts, speed):
    vf, vl = h["video"][:2]
    if speed == 1:
        ff, fl = h["fwd"][:2]
        return vf + c_div((pts - ff) * (vl - vf), fl - ff)
    if speed == -1:
        rf, rl = h["rwd"][:2]
        return vl - c_div((pts - rf) * (vl - vf), rl - rf)
    return pts


def pts2offset(h, pts, speed, signed_fwd=False, single_first=False):
    """idx_hdr::pts2offset. The keyword arguments are the two mistakes the pins must catch: a signed division at speed 1, and
    subtracting first_pts only once at speed -1."""
    vf, vl, vbin, _, vn = h["video"]
    pts = max(min(pts, vl), vf)
    if speed == 1:
        _, _, fbin, ftrick, fn = h["fwd"]
        off = c_div(pts - vf, ftrick * fbin) & M32 if signed_fwd else (((pts - vf) & M32) // ftrick) // fbin
        off = min((fn - 1) & M32, off) + vn
    elif speed == -1:
        _, _, rbin, rtrick, rn = h["rwd"]
        d = (vl - pts) if single_first else (vl - pts) - vf
        off = ((d & M32) // rtrick) // rbin
        off = min((rn - 1) & M32, off) + vn + h["fwd"][4]
    else:
        off = c_div(pts - vf, vbin) & M32
        off = min((vn - 1) & M32, off)
    return (off * 4 + HDR) & M32


def get_index(idx, pos, speed, **kw):
    """(byte offset read in video.idx, the uint32 sample there)"""
    at = pts2offset(parse(idx), pos, speed, **kw)
    return at, struct.unpack_from("<I", idx, at)[0]


class Title:
    def __init__(self, idx, main, fwd=None, rwd=None):
        self.idx, self.hdr = bytes(idx), parse(idx)
        self.files = [rwd, main, fwd]                    # _vid_names order: speed + 1
        self.sizes = [0 if f is None else len(f) for f in self.files]


class Stream:
    """one stream's title, speed, state, file, cursor and pos (ef_library_status)"""

    def __init__(self):
        self.title, self.speed, self.state, self.file, self.cursor, self.pos = -1, 0, IDLE, 1, 0, 0

    def status(self):
        return (self.title, self.speed, self.state, self.file, self.cursor, self.pos)

    def _play(self, titles, speed, **kw):
        at, sample = get_index(titles[self.title].idx, self.pos, speed, **kw)
        self.speed, self.file, self.cursor, self.state = speed, speed + 1, sample * 188, PLAYING
        return at

    def command(self, titles, cmd, title=0, arg=0, last_pts=-1, clamp_skip=False, **kw):
        """one command, get_pts() = last_pts -> (restart op, byte offset read in video.idx or None)"""
        if cmd == PLAY_AT:
            self.title, self.pos = title, arg
            return 1, self._play(titles, 0, **kw)
        t = titles[self.title]
        if cmd != RESUME and self.state == PLAYING:
            self.pos = pts2pts(t.hdr, last_pts, self.speed)
        if cmd == PLAY:
            return 1, self._play(titles, 0, **kw)
        if cmd == SKIP:
            self.pos += to_i32(arg * 90000)
            if clamp_skip:                               # a mistake the pins must catch: the reference keeps pos unclamped
                vf, vl = t.hdr["video"][:2]
                self.pos = max(min(self.pos, vl), vf)
            return 1, self._play(titles, 0, **kw)
        if cmd == FAST_FORWARD:
            return 1, self._play(titles, 1, **kw)
        if cmd == REWIND:
            return 1, self._play(titles, -1, **kw)
        if cmd == PAUSE:
            if self.state == PLAYING:
                self.state = PAUSED
            return 0, None
        if cmd == RESUME:
            self.state = PLAYING
            return 2, None
        self.state = STOPPED
        return 0, None

    def submit(self, titles, budget):
        """-> (file, first byte, packets, ends) of this submit's run, or None for a stream that gets nothing"""
        if self.state != PLAYING:
            return None
        t = titles[self.title]
        size = t.sizes[self.file]
        left = (size - self.cursor) // 188 if self.cursor < size else 0
        take = min(budget, left)
        run = (self.file, min(self.cursor, size), take, take == left)
        self.cursor += take * 188
        if take == left:
            self.state, self.pos = ENDED, pts2pts(t.hdr, 0, self.speed)
        return run


def check_command(titles, st, cmd, title=0, arg=0):
    """the EF_EINVAL cases of ef_library_command -> True when the command is refused"""
    if cmd == PLAY_AT:
        return not 0 <= title < len(titles)
    if st.state == IDLE or (cmd == RESUME and st.state != PAUSED):
        return True
    if cmd == SKIP and not -2 ** 31 <= arg < 2 ** 31:
        return True
    t = titles[st.title]
    return (cmd == FAST_FORWARD and t.sizes[2] == 0) or (cmd == REWIND and t.sizes[0] == 0)


# ---- ESPFlix::loop()'s pause handshake (espflix.cpp:906-939, the UI thread) -------------------------------------------------------
# A key while PLAYING sets _pending and pauses the decoder; once it has paused, loop() saves pos (save_pos) and runs the method
# _pending names. While _speed != 0 every pending action but DONE becomes play_pause() from NAV, i.e. PLAY.
P_NONE, P_NAV, P_DONE, P_REWIND, P_FAST_FORWARD, P_SKIP_FORWARD, P_SKIP_BACK = range(7)


def loop_command(pending, speed):
    """-> (command, arg) the library takes for what loop() does once the decoder paused with _pending at _speed"""
    if speed and pending != P_DONE:
        return PLAY, 0
    return {P_NAV: (STOP, 0), P_DONE: (STOP, 0), P_REWIND: (REWIND, 0), P_FAST_FORWARD: (FAST_FORWARD, 0),
            P_SKIP_FORWARD: (SKIP, 30), P_SKIP_BACK: (SKIP, -30), P_NONE: (PAUSE, 0)}[pending]


# ---- the pinned scripts (tests/golden/library_pins.json, written by tools/make_library_golden.py) ----------------------------------
PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "library_pins.json")
DONE = 8                                    # a script step only: the end of the title, save_pos(0) (espflix.cpp:906-911)
NOTHING = 0xFFFFFFFF


def restate(idx, steps, **kw):
    """a script of (cmd, arg, get_pts()) on one title -> per step the file played (-1 none), its byte offset, the video.idx byte
    read (NOTHING: none), _speed and pos, as tools/ref_library_harness.cpp reports them"""
    titles = [Title(idx, b"")]
    st, out = Stream(), []
    for cmd, arg, pts in steps:
        at = None
        if cmd == DONE:
            st.state, st.pos = ENDED, pts2pts(titles[0].hdr, 0, st.speed)
            op = 0
        else:
            op, at = st.command(titles, cmd, 0, arg, pts, **kw)
        played = op == 1
        out.append({"file": st.file if played else -1, "offset": (st.cursor & M32) if played else 0,
                    "idx_at": NOTHING if at is None else at, "speed": st.speed, "pos": st.pos})
    return out


def pinned_cases():
    """name -> (video.idx image, [(cmd, arg, get_pts())])"""
    fixture = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_idx_fixture.bin"), "rb").read()
    vf, vl = parse(fixture)["video"][:2]
    ff, fl = parse(fixture)["fwd"][:2]
    rf, rl = parse(fixture)["rwd"][:2]
    S = 90000

    def synth(video, fwd, rwd):
        n = video[4] + fwd[4] + rwd[4]
        return image(video, fwd, rwd, [(7919 * i + 13) % 100003 for i in range(n)])

    cases = {}
    for tag, p in (("minus_one", -1), ("before_first", vf - 1), ("at_first", vf), ("inside", (vf + vl) // 2), ("at_last", vl),
                   ("past_last", vl + 10 * S)):
        cases["fixture_play_at_" + tag] = (fixture, [(PLAY_AT, p, -1), (FAST_FORWARD, 0, -1), (PLAY, 0, ff + 5), (REWIND, 0, p),
                                                     (PLAY, 0, rf + 77), (PAUSE, 0, p), (RESUME, 0, p), (STOP, 0, p), (PLAY, 0, p)])
    cases["fixture_trick_positions"] = (fixture, [(PLAY_AT, vf, -1), (FAST_FORWARD, 0, vf + S), (FAST_FORWARD, 0, fl), (REWIND, 0, fl + S),
                                                  (REWIND, 0, rl), (REWIND, 0, rf - 1), (PLAY, 0, rf), (FAST_FORWARD, 0, ff - S)])
    cases["fixture_skips_past_both_ends"] = (fixture, [(PLAY_AT, vf + S, -1)] + [(SKIP, 30, vl + S)] * 4 + [(SKIP, -30, -1)] * 3 +
                                             [(PAUSE, 0, vf + 2 * S), (SKIP, -1000, 0), (SKIP, 2000, 0), (SKIP, -30, vf), (SKIP, 30, vl)])
    cases["fixture_skip_int_product_wraps"] = (fixture, [(PLAY_AT, vf, -1), (SKIP, 30000, vf), (SKIP, -30000, vf), (SKIP, 2 ** 31 - 1, vf),
                                                         (SKIP, -2 ** 31, vf)])
    cases["fixture_done"] = (fixture, [(PLAY_AT, vf, -1), (DONE, 0, vl), (PLAY, 0, 0), (FAST_FORWARD, 0, ff + S), (DONE, 0, 0), (PLAY, 0, 0),
                                       (REWIND, 0, vl), (DONE, 0, 0), (PLAY, 0, 0)])
    # rwd: (last - pts) - first wraps in uint32 when first_pts is large; a single subtraction would give another sample
    wrap = synth((5 * 10 ** 9, 5 * 10 ** 9 + 3600 * S, 7500, 1, 43200), (5 * 10 ** 9, 5 * 10 ** 9 + 240 * S, 7500, 15, 2880),
                 (5 * 10 ** 9 + 11, 5 * 10 ** 9 + 240 * S, 7500, 15, 2880))
    cases["rwd_wrap"] = (wrap, [(PLAY_AT, 5 * 10 ** 9 + k * 600 * S, -1) for k in range(7)] +
                         [(REWIND, 0, 5 * 10 ** 9 + 11 + k * 1111) for k in range(6)] + [(PLAY, 0, 5 * 10 ** 9 + 20 * S)])
    # fwd: the uint32 cast of pts - first truncates a difference of 2^32 or more; a signed division would not
    big = synth((0, 2 ** 34, 7500, 1, 300000), (0, 2 ** 34 // 15, 7500, 15, 300000), (1, 2 ** 34 // 15, 7500, 15, 2000))
    cases["fwd_truncation"] = (big, [(PLAY_AT, 2 ** 32 + 5 * S, -1), (FAST_FORWARD, 0, 2 ** 32 + 5 * S), (PLAY, 0, 2 ** 28), (FAST_FORWARD, 0, 2 ** 28 + 3 * S),
                                     (REWIND, 0, 2 ** 27), (PLAY_AT, 2 ** 33 + 1, -1), (FAST_FORWARD, 0, 2 ** 33 + 1)])
    # the unsigned min() against sample_count - 1 on every record
    few = synth((1000, 1000 + 3600 * S, 7500, 1, 5), (1000, 1000 + 240 * S, 7500, 15, 3), (1000, 1000 + 240 * S, 7500, 15, 2))
    cases["min_clamps"] = (few, [(PLAY_AT, 1000 + k * 900 * S, -1) for k in range(5)] + [(FAST_FORWARD, 0, 1000 + 60 * S), (REWIND, 0, 1000 + 60 * S),
                                                                                        (PLAY, 0, 1000 + 200 * S), (SKIP, -7200, 0)])
    return cases


# ---- seeded command scripts ----------------------------------------------------------------------------------------------------
def script(rng, n_titles, steps, trick=lambda t: (True, True)):
    """a random valid command for one stream per step, given its restated state: [(cmd, title, arg)] generator helper. trick(t) ->
    (has rwd, has fwd). Returns a function st -> (cmd, title, arg)."""
    def pick(st):
        if st.state == IDLE or rng.random() < 0.08:
            t = int(rng.integers(n_titles))
            return PLAY_AT, t, int(rng.integers(-90000, 90000 * 60))
        choices = [PLAY, SKIP, PAUSE, STOP, SKIP]
        has_rwd, has_fwd = trick(st.title)
        if has_fwd:
            choices.append(FAST_FORWARD)
        if has_rwd:
            choices.append(REWIND)
        if st.state == PAUSED:
            choices += [RESUME, RESUME]
        cmd = choices[int(rng.integers(len(choices)))]
        return cmd, 0, int(rng.integers(-60, 60)) if cmd == SKIP else 0
    return pick
