"""tests/nav_cases.py — the title library's poster menu restated in Python (TEST INFRASTRUCTURE), on top of tests/library_cases.py:
ESPFlix::nav(), menu(), set_state(), load_poster() and the NVS resume (espflix.cpp:704-720, 763-785, 851-859, 906-939, 1060-1069;
espflix.ino:160-178) as ef_library_command's EF_LIB_NAV / EF_LIB_NAV_STEP / EF_LIB_MENU, the POSTER state, the count kernel's rule
for a poster and the saved-position table nv[title][stream].

nav(s, i): dir = 0 before the first nav, else old title - i; mode = 1 (dir 0), 2 (dir < 0), 3 (dir > 0); title = i, pos = nv[i][s],
state POSTER, file 3 from byte 0, restart op 1 and a blend of 0 staged (hide_progress()); speed stays.
  NAV (title i)   from IDLE or POSTER: nav(s, i)
  NAV_STEP (k)    from POSTER: nav(s, title + k); outside [0, titles): nothing at all (nav()'s early return)
  MENU            PLAYING: pos = pts2pts(get_pts(), speed), nv[title][s] = pos, then at speed 0 nav(s, title), at speed +-1 play
                  at speed 0 from pos (op 1, no poster); PAUSED / STOPPED / ENDED: nav(s, title), no write; POSTER: nothing
A submit gives a POSTER stream packets of file 3 until its end, which ends the stream (end flag) and carries its mode; the stream
stays POSTER with its pos. The other commands keep library_cases' rules on a POSTER stream.

The keyword arguments of Stream.command / Stream.submit are the mistakes the pins must catch (tests/test_nav.py)."""
import os
import struct

from tests import library_cases as lc

PLAY_AT, PLAY, SKIP, FAST_FORWARD, REWIND, PAUSE, RESUME, STOP = range(8)
NAV, NAV_STEP, MENU = 8, 9, 10
IDLE, PLAYING, PAUSED, STOPPED, ENDED, POSTER = range(6)
POSTER_FILE = 3
DONE = 11                                   # a script step only: the title's bytes ran out (loop()'s DONE branch)


class Title(lc.Title):
    """a title with its poster.ts as file 3"""

    def __init__(self, idx, main, fwd=None, rwd=None, poster=None):
        super().__init__(idx, main, fwd, rwd)
        self.files.append(poster)
        self.sizes.append(0 if poster is None else len(poster))


def new_nv(n_titles, n_streams):
    """the saved-position table, nv[title][stream], every entry 0 (nv_read's default)"""
    return [[0] * n_streams for _ in range(n_titles)]


class Stream(lc.Stream):
    """one stream's library state and the mode of its latest nav"""

    def __init__(self):
        super().__init__()
        self.mode = 0

    def _nav(self, nv, s, i, flip_dir=False):
        d = 0 if self.title == -1 else self.title - i
        m = 1 if d == 0 else 2 if d < 0 else 3
        if flip_dir and m > 1:                       # a mistake: the scroll the other way
            m = 5 - m
        self.mode = m
        self.title, self.pos, self.state, self.file, self.cursor = i, nv[i][s], POSTER, POSTER_FILE, 0

    def command(self, titles, cmd, title=0, arg=0, last_pts=-1, nv=None, s=0, flip_dir=False, nv_on_pause=False, step_clamp=False,
                trick_menu_poster=False, **kw):
        """one command -> (restart op, whether a blend of 0 is staged). nv: the table, s: this stream's index in it"""
        if cmd == NAV:
            self._nav(nv, s, title, flip_dir)
            return 1, True
        if cmd == NAV_STEP:
            i = self.title + arg
            if not 0 <= i < len(titles):
                if not step_clamp:
                    return 0, False
                i = min(max(i, 0), len(titles) - 1)
            self._nav(nv, s, i, flip_dir)
            return 1, True
        if cmd == MENU:
            if self.state == POSTER:
                return 0, False
            if self.state == PLAYING:
                self.pos = lc.pts2pts(titles[self.title].hdr, last_pts, self.speed)
                nv[self.title][s] = self.pos
                if self.speed and not trick_menu_poster:
                    self._play(titles, 0, **kw)
                    return 1, False
            self._nav(nv, s, self.title, flip_dir)
            return 1, True
        was = self.state
        op, _ = super().command(titles, cmd, title, arg, last_pts, **kw)
        if nv_on_pause and cmd == PAUSE and was == PLAYING:
            nv[self.title][s] = self.pos
        return op, False

    def submit(self, titles, budget, poster_ends=False):
        """-> (file, first byte, packets, ends) of this submit's run, or None; a POSTER stream reads its poster to the end once"""
        if self.state != POSTER:
            return super().submit(titles, budget)
        size = titles[self.title].sizes[POSTER_FILE]
        if self.cursor >= size:
            return None
        left = (size - self.cursor) // 188
        take = min(budget, left)
        run = (POSTER_FILE, self.cursor, take, take == left)
        self.cursor += take * 188
        if take == left and poster_ends:             # a mistake: the poster's end as a title's end
            self.state, self.pos = ENDED, lc.pts2pts(titles[self.title].hdr, 0, self.speed)
        return run

    def end_mode(self, run):
        """the mode a submit carries for this stream: its nav's mode when the run ends the poster, else 0"""
        return self.mode if run is not None and run[0] == POSTER_FILE and run[3] else 0


def check_command(titles, st, cmd, title=0, arg=0):
    """the EF_EINVAL cases of ef_library_command with the poster commands -> True when the command is refused"""
    def no_poster(i):
        return titles[i].sizes[POSTER_FILE] == 0
    if cmd == NAV:
        return not 0 <= title < len(titles) or st.state not in (IDLE, POSTER) or no_poster(title)
    if cmd == PLAY_AT:
        return lc.check_command(titles, st, cmd, title, arg)
    if st.state == IDLE:
        return True
    if cmd == NAV_STEP:
        if st.state != POSTER or not -2 ** 31 <= arg < 2 ** 31:
            return True
        i = st.title + arg
        return 0 <= i < len(titles) and no_poster(i)
    if cmd == MENU:
        return st.state != POSTER and not (st.state == PLAYING and st.speed) and no_poster(st.title)
    if cmd > MENU or cmd < 0:
        return True
    return lc.check_command(titles, st, cmd, title, arg)


def loop_command(pending, speed):
    """loop_command() of library_cases with the poster menu: a pending NAV (menu() while PLAYING) and the end of a title (DONE) both
    become MENU, at every speed; every other pending key as library_cases.loop_command"""
    if pending in (lc.P_NAV, lc.P_DONE):
        return MENU, 0
    return lc.loop_command(pending, speed)


# ---- the pinned scripts (tests/golden/nav_pins.json, written by tools/make_nav_golden.py) -------------------------------------------
PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nav_pins.json")


def restate(idxs, steps, **kw):
    """a script of (cmd, arg, get_pts()) on one stream over titles with the video.idx images idxs -> per step the file a restart
    played (-1 none) and its byte offset, the mode of a nav (-1 none), the NVS writes, title, speed, state, pos and the saved
    position of every title, as tools/ref_nav_harness.cpp reports them. Every poster is read to its end after the step, as
    load_poster() does before it returns."""
    titles = [Title(idx, b"", poster=bytes(188 * 3)) for idx in idxs]
    nv = new_nv(len(titles), 1)
    st, out = Stream(), []
    submit_kw = {"poster_ends": kw.pop("poster_ends", False)}
    nv_on_pause = kw.get("nv_on_pause", False)
    for cmd, arg, pts in steps:
        before = [row[0] for row in nv]
        if cmd == DONE:                              # the submit that ends the title, then MENU from ENDED (the host's DONE)
            st.state, st.pos = ENDED, lc.pts2pts(titles[st.title].hdr, 0, st.speed)
            if nv_on_pause:                          # the mistake writes NVS at DONE too
                nv[st.title][0] = st.pos
            op, hide = st.command(titles, MENU, nv=nv, **kw)
        else:
            op, hide = st.command(titles, cmd, 0 if cmd != NAV else arg, arg if cmd != NAV else 0, pts, nv=nv, **kw)
        played = op == 1
        rec = {"file": st.file if played else -1, "offset": (st.cursor & lc.M32) if played else 0, "mode": st.mode if hide else -1,
               "writes": sum(1 for a, row in zip(before, nv) if row[0] != a), "title": st.title, "speed": st.speed,
               "state": st.state, "pos": st.pos, "nv": [row[0] for row in nv]}
        if st.state == POSTER:
            st.submit(titles, 1 << 30, **submit_kw)
            rec["state"] = st.state
        out.append(rec)
    return out


def pinned_cases():
    """name -> ([video.idx image per title], [(cmd, arg, get_pts())])"""
    fixture = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_idx_fixture.bin"), "rb").read()
    h = lc.parse(fixture)
    vf, vl = h["video"][:2]
    ff = h["fwd"][0]
    rf = h["rwd"][0]
    S = 90000
    # a second image: the fixture's records with its first_pts moved, so that titles map pts differently
    shifted = bytearray(fixture)
    for k in range(3):
        a, b = struct.unpack_from("<qq", fixture, 8 + 32 * k)
        struct.pack_into("<qq", shifted, 8 + 32 * k, a + 7 * S, b + 7 * S)
    row = [fixture, bytes(shifted), fixture, bytes(shifted)]
    cases = {}
    cases["row_ends_and_jumps"] = (row, [(NAV, 0, -1), (NAV_STEP, -1, -1), (NAV_STEP, 1, -1), (NAV_STEP, 1, -1), (NAV_STEP, 1, -1),
                                         (NAV_STEP, 1, -1), (NAV_STEP, -3, -1), (NAV_STEP, 2, -1), (NAV_STEP, 5, -1), (NAV, 3, -1),
                                         (NAV, 0, -1), (NAV_STEP, -5, -1), (NAV, 0, -1)])
    cases["menu_playing_speed0"] = (row, [(NAV, 1, -1), (PLAY, 0, -1), (MENU, 0, vf + 17 * S), (PLAY, 0, -1), (MENU, 0, vf + 40 * S),
                                          (NAV_STEP, 1, -1), (NAV_STEP, -1, -1), (PLAY, 0, -1), (MENU, 0, vl + S), (PLAY, 0, -1)])
    cases["menu_trick_modes"] = (row, [(NAV, 2, -1), (PLAY, 0, -1), (FAST_FORWARD, 0, vf + 5 * S), (MENU, 0, ff + 3 * S),
                                       (MENU, 0, vf + 30 * S), (PLAY, 0, -1), (REWIND, 0, vf + 60 * S), (MENU, 0, rf + 7 * S),
                                       (PAUSE, 0, vf + 9 * S), (MENU, 0, -1), (PLAY, 0, -1)])
    cases["pause_then_menu"] = (row, [(NAV, 0, -1), (PLAY, 0, -1), (MENU, 0, vf + 30 * S), (PLAY, 0, -1), (PAUSE, 0, vf + 50 * S),
                                      (MENU, 0, -1), (PLAY, 0, -1), (PAUSE, 0, vf + 70 * S), (RESUME, 0, -1), (MENU, 0, vf + 75 * S),
                                      (PLAY, 0, -1)])
    cases["done"] = (row, [(NAV, 3, -1), (PLAY, 0, -1), (MENU, 0, vf + 40 * S), (PLAY, 0, -1), (DONE, 0, vl), (PLAY, 0, -1),
                           (FAST_FORWARD, 0, vf + 44 * S), (DONE, 0, 0), (PLAY, 0, -1), (REWIND, 0, vf + 50 * S), (DONE, 0, 0)])
    cases["menu_from_nav"] = (row, [(NAV, 1, -1), (MENU, 0, -1), (MENU, 0, vf), (NAV_STEP, 1, -1), (MENU, 0, -1), (PLAY, 0, -1),
                                    (MENU, 0, vf + 3 * S), (MENU, 0, -1)])
    cases["both_directions"] = (row, [(NAV, 0, -1), (PLAY, 0, -1), (MENU, 0, vf + S), (NAV_STEP, 1, -1), (PLAY, 0, -1),
                                      (MENU, 0, vf + 12 * S), (NAV_STEP, 2, -1), (PLAY, 0, -1), (MENU, 0, vf + 23 * S), (NAV_STEP, -2, -1),
                                      (NAV_STEP, -1, -1), (PLAY, 0, -1), (MENU, 0, vf + 2 * S), (NAV_STEP, 3, -1), (NAV_STEP, -2, -1),
                                      (PLAY, 0, -1)])
    return cases


# ---- seeded scripts --------------------------------------------------------------------------------------------------------------
def script(rng, n_titles, trick=lambda t: (True, True)):
    """-> pick(st): a random command (cmd, title, arg) for one stream given its restated state, valid or not (the refused ones are
    checked for EF_EINVAL), browsing posters and playing titles"""
    def pick(st):
        u = rng.random()
        if st.state == IDLE:
            return (NAV, int(rng.integers(n_titles)), 0) if u < 0.8 else (PLAY_AT, int(rng.integers(n_titles)), int(rng.integers(0, 90000 * 4)))
        if st.state == POSTER:
            if u < 0.45:
                return NAV_STEP, 0, int(rng.choice([-1, 1, -1, 1, 2, -3, 5]))
            if u < 0.55:
                return NAV, int(rng.integers(n_titles)), 0
            if u < 0.65:
                return MENU, 0, 0
            return PLAY, 0, 0
        if u < 0.3:
            return MENU, 0, 0
        if u < 0.35:
            return NAV_STEP, 0, 1                    # refused outside POSTER
        cmd, title, arg = lc.script(rng, n_titles, 1, trick)(st)
        return cmd, title, arg
    return pick
