"""tests/keys_cases.py — the remote restated in Python (TEST INFRASTRUCTURE), on top of tests/nav_cases.py: one ESPFlix::loop()
iteration (espflix.cpp:886-1010) per stream with the key key_event() produced (espflix.cpp:1020-1040), as ef_library_keys runs it.

  1. An ENDED stream (the decoder ran out of bytes: _pending == DONE) takes the pause branch first, also with key 0:
     nav_cases.loop_command(P_DONE) = MENU, i.e. nav(s, title). A title without a poster stays ENDED and ignores the key.
  2. The key on the state step 1 left. On a PLAYING stream a key sets _pending and pauses; the pause resolves at once and
     nav_cases.loop_command(pending, speed) names the command. On the poster, PLAY / SELECT is play_pause() from NAV (PLAY) and
     RIGHT / LEFT is nav(_nav +- 1) (NAV_STEP); on a PAUSED stream MENU is menu(), PLAY / SELECT play_pause() (RESUME), RIGHT / LEFT
     fast_forward() / rewind(); on STOPPED only MENU acts. A command nav_cases.check_command refuses does nothing.
The commands run by nav_cases.Stream.command. What loop() leaves on screen: a nav hides the progress (blend 0), play() shows it at 180
(speed 0) or -1 (speed +-1), a pause and a resume show it at 180. _last_seconds becomes 0 where play_pause() runs (PLAY / SELECT,
and every pending action at speed +-1) and in the pause branch's NONE case.

The keyword arguments of Stream.key are the mistakes the pins must catch (tests/test_keys.py)."""
import os
import random
import struct

from tests import library_cases as lc
from tests import nav_cases as nc

KEY_MENU, KEY_PLAY, KEY_SELECT, KEY_RIGHT, KEY_LEFT, KEY_DOWN, KEY_UP = 16, 19, 40, 79, 80, 81, 82
KEYS = (KEY_MENU, KEY_PLAY, KEY_SELECT, KEY_RIGHT, KEY_LEFT, KEY_DOWN, KEY_UP)
NOTHING, ENDED_BIT = 0x0F, 0x10                 # done codes: no command ran; the DONE branch ran first
# key_event()'s table: the Apple remote's 7-bit code (bits 8..14 of the NEC code) -> key
APPLE = {0x40: KEY_MENU, 0x7A: KEY_PLAY, 0x3A: KEY_SELECT, 0x60: KEY_RIGHT, 0x10: KEY_LEFT, 0x30: KEY_DOWN, 0x50: KEY_UP}
NEC = {k: 0x07EE0000 | (a << 8) | 0x9B for a, k in APPLE.items()}
NEC_OTHER = 0x07EE2F9B                           # a code key_event() maps to no key (7-bit code 0x2F)
# the pending action a key leaves on a PLAYING stream (espflix.cpp:957-1004)
PENDING = {KEY_MENU: lc.P_NAV, KEY_PLAY: lc.P_NONE, KEY_SELECT: lc.P_NONE, KEY_RIGHT: lc.P_FAST_FORWARD, KEY_LEFT: lc.P_REWIND,
           KEY_UP: lc.P_SKIP_FORWARD, KEY_DOWN: lc.P_SKIP_BACK}


def key_of(nec):
    """key_event(): the key of a NEC code, 0 for none or an unknown code"""
    return APPLE.get((nec >> 8) & 0x7F, 0) if nec else 0


class Stream(nc.Stream):
    """one stream's library state; key() is one loop() iteration"""

    def key(self, titles, key, last_pts=-1, nv=None, s=0, ff_continues=False, up_paused=False, trick_blend_180=False,
            no_zero_on_play=False, done_needs_key=False, **kw):
        """one iteration with `key`, get_pts() = last_pts -> dict: done code, restart op, blend staged (None: none), whether
        _last_seconds is zeroed, whether a nav ran, NVS writes"""
        r = {"done": NOTHING, "op": 0, "blend": None, "zero": False, "nav": False, "writes": 0}
        no_poster = self.state != nc.IDLE and titles[self.title].sizes[nc.POSTER_FILE] == 0
        if self.state == nc.IDLE or (self.state == nc.ENDED and no_poster):
            return r
        if self.state == nc.ENDED and not (done_needs_key and key == 0):
            cmd, _ = nc.loop_command(lc.P_DONE, self.speed)
            r["op"], _ = self.command(titles, cmd, nv=nv, s=s, **kw)
            r["done"] |= ENDED_BIT
            r["blend"], r["nav"] = 0, True
        play, side, vert = key in (KEY_PLAY, KEY_SELECT), key in (KEY_RIGHT, KEY_LEFT), key in (KEY_UP, KEY_DOWN)
        sign = 1 if key in (KEY_RIGHT, KEY_UP) else -1
        cmd, arg = None, 0
        if self.state == nc.POSTER:
            if play:
                cmd = nc.PLAY
            elif side:
                cmd, arg = nc.NAV_STEP, sign
            r["zero"] = play
        elif self.state == nc.PLAYING and key in PENDING:
            cmd, arg = nc.loop_command(PENDING[key], self.speed)
            if ff_continues and self.speed and side:
                cmd, arg = (nc.FAST_FORWARD if sign > 0 else nc.REWIND), 0
            r["zero"] = play or self.speed != 0
        elif self.state == nc.PAUSED:
            if key == KEY_MENU:
                cmd = nc.MENU
            elif play:
                cmd = nc.RESUME
            elif side:
                cmd = nc.FAST_FORWARD if sign > 0 else nc.REWIND
            elif vert and up_paused:
                cmd, arg = nc.SKIP, 30 * sign
            r["zero"] = play
        elif self.state == nc.STOPPED:
            cmd = nc.MENU if key == KEY_MENU else None
            r["zero"] = play
        if no_zero_on_play and play:
            r["zero"] = False
        if cmd == nc.NAV_STEP and not 0 <= self.title + arg < len(titles):
            cmd = None                                   # nav()'s early return
        if cmd is not None and nc.check_command(titles, self, cmd, 0, arg):
            cmd = None
        if cmd is None:
            return r
        was = self.state
        op, hide = self.command(titles, cmd, 0, arg, last_pts, nv=nv, s=s, **kw)
        r["op"] = 1 if 1 in (r["op"], op) else op
        r["done"] = (r["done"] & ~0xF) | cmd
        r["writes"] = int(cmd == nc.MENU and was == nc.PLAYING)
        if hide:
            r["blend"], r["nav"] = 0, True
        elif self.state == nc.PLAYING and cmd != nc.RESUME:
            r["blend"] = 180 if self.speed == 0 or trick_blend_180 else -1
        elif cmd in (nc.PAUSE, nc.RESUME):
            r["blend"] = 180
        return r

    def end(self, titles):
        """the submit that reaches the end of a PLAYING stream's file: ENDED with pos = pts2pts(0, speed)"""
        if self.state == nc.PLAYING:
            self.state, self.pos = nc.ENDED, lc.pts2pts(titles[self.title].hdr, 0, self.speed)


def titles_of(idxs):
    """restated titles over video.idx images: every file present (one packet), a poster"""
    return [nc.Title(idx, bytes(188), bytes(188), bytes(188), bytes(188 * 3)) for idx in idxs]


# ---- the pinned scripts (tests/golden/keys_pins.json, written by tools/make_keys_golden.py) -------------------------------------------
PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "keys_pins.json")
STATE = {nc.PLAYING: 1, nc.PAUSED: 2, nc.POSTER: 5}


def restate(idxs, steps, sentinel, **kw):
    """a script of (nec, ended, get_pts()) on one stream, from init_service()'s nav(0) -> per step what tools/ref_keys_harness.cpp
    reports: file played (-1 none), its offset, the mode of the last nav (-1 none), NVS writes, title, speed, state, blend and
    _last_seconds (sentinel: not written in the step), pos and the saved position of every title"""
    titles = titles_of(idxs)
    nv = nc.new_nv(len(titles), 1)
    st, out = Stream(), []
    st.command(titles, nc.NAV, 0, nv=nv)
    st.submit(titles, 1 << 30)
    for nec, ended, pts in steps:
        if ended:
            st.end(titles)
        r = st.key(titles, key_of(nec), pts, nv=nv, **kw)
        played = r["op"] == 1 and st.state in (nc.PLAYING, nc.POSTER)
        out.append([st.file if played else -1, (st.cursor & lc.M32) if played else 0, st.mode if r["nav"] else -1, r["writes"], st.title,
                    st.speed, STATE.get(st.state, -1), sentinel if r["blend"] is None else r["blend"], 0 if r["zero"] else sentinel, st.pos]
                   + [row[0] for row in nv])
        if st.state == nc.POSTER:
            st.submit(titles, 1 << 30)
    return out


def pinned_cases():
    """name -> ([video.idx image per title], [(nec, ended, get_pts())])"""
    fixture = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_idx_fixture.bin"), "rb").read()
    h = lc.parse(fixture)
    vf, vl = h["video"][:2]
    S = 90000
    shifted = bytearray(fixture)
    for k in range(3):
        a, b = struct.unpack_from("<qq", fixture, 8 + 32 * k)
        struct.pack_into("<qq", shifted, 8 + 32 * k, a + 7 * S, b + 7 * S)
    row = [fixture, bytes(shifted), fixture]
    P, M, R, L, U, D = (NEC[k] for k in (KEY_PLAY, KEY_MENU, KEY_RIGHT, KEY_LEFT, KEY_UP, KEY_DOWN))
    every = [NEC[k] for k in KEYS] + [0, NEC_OTHER]
    # the states, reached from the poster of title 1: (prefix of steps, get_pts() of the key)
    states = {"poster": ([(R, 0, -1)], -1), "play0": ([(R, 0, -1), (P, 0, -1)], vf + 40 * S),
              "ffwd": ([(R, 0, -1), (P, 0, -1), (R, 0, vf + 20 * S)], vf + 9 * S), "rwnd": ([(R, 0, -1), (P, 0, -1), (L, 0, vf + 50 * S)], vf + 61 * S),
              "paused": ([(R, 0, -1), (P, 0, -1), (P, 0, vf + 33 * S)], vf + 35 * S)}
    cases = {}
    for tag, (prefix, pts) in states.items():
        for nec in every:
            cases["%s_%08x" % (tag, nec)] = (row, prefix + [(nec, 0, pts), (0, 0, pts), (P, 0, pts + 3 * S)])
    for tag, (prefix, _) in states.items():
        if tag.startswith("play") or tag in ("ffwd", "rwnd"):
            for nec in every:
                cases["done_%s_%08x" % (tag, nec)] = (row, prefix + [(nec, 1, 0), (R, 0, -1), (P, 0, -1)])
    cases["row_ends"] = (row, [(L, 0, -1), (L, 0, -1), (R, 0, -1), (R, 0, -1), (R, 0, -1), (R, 0, -1), (L, 0, -1), (M, 0, -1), (P, 0, -1),
                               (M, 0, vf + 12 * S), (R, 0, -1), (R, 0, -1), (NEC[KEY_SELECT], 0, -1)])
    cases["skips_past_both_ends"] = (row, [(P, 0, -1)] + [(U, 0, vl - 40 * S)] * 3 + [(U, 0, vl + S)] * 2 + [(D, 0, vf + 10 * S)] * 3 +
                                     [(D, 0, vf - S), (D, 0, 0), (P, 0, vf), (U, 0, -1), (D, 0, -1)])
    for seed in range(6):
        rng = random.Random(seed)
        idxs = [fixture, bytes(shifted)] * (1 + seed % 2)
        steps, playing = [], False
        for _ in range(48):
            u = rng.random()
            nec = 0 if u < 0.12 else NEC_OTHER if u < 0.16 else NEC[rng.choice(KEYS)]
            ended = int(rng.random() < 0.12)
            pts = rng.choice([-1, 0, vf + rng.randrange(0, 120) * S + rng.randrange(S), vl + rng.randrange(-5, 5) * S])
            steps.append((nec, ended, pts))
        cases["seeded_%d" % seed] = (idxs, steps)
    return cases

