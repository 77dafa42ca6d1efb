"""tests/restart_cases.py — the per-stream restart (ef_restart_streams) restated in Python, and the programs it is pinned on.

A restart with op 1 is what the reference's player does on play / skip / fast_forward / rewind / load_poster:
MpegDecoder::reset() with its video_reset() (player.cpp:439-453, video.cpp:1070-1074). Between one program and the next:
  * get_pts() reads -1 until the next picture; the carried _pts stays, so a program whose first video PES has no PTS
    gives its first pictures the previous program's last PTS;
  * the audio demux gate shuts (the next program's audio bytes before its first PES start are dropped), the SBC ring and the
    learned frame size are cleared (bytes held back are dropped, the next frame is probed and so decoded twice), while the
    SBC filter memory, the last subband samples and the delta-sigma modulator carry on. A probe that fails the sync byte
    still re-synthesises the last subband samples into the filter memory (sbc_decoder.cpp:343-372);
  * the display latches a new origin at the next push; position, frame stores, store phase, scroll and overlay stay.
Op 2, video_pause(0) (video.cpp:1060-1068), clears the display origin only.

decoder_cases() are the programs of tools/ref_restart_harness.cpp's decoder run (pts of every push, get_pts() after every
program, PCM and PDM); paced_cases() the field streams of its paced run. tests/golden/restart_pins.json holds what the
unmodified reference produced on them (tools/make_restart_golden.py)."""
import hashlib

import numpy as np

from tests import audio_cases, overlay_cases as oc, present_cases as pc, pts_cases

M32 = pc.M32


# -- programs -----------------------------------------------------------------------------------------------------------
def _synth_es(seed, n_pictures, gop):
    from espflix_b200 import synth
    return bytes(synth.generate(synth.SEED0 + seed, n_pictures=n_pictures, gop=gop)[0])


def program(seed, n_pictures, first_pts, first_kind="pts", audio=None):
    """a TS program: synthetic video with one PES per picture (the first of kind first_kind, the others with rising PTS) and,
    when audio = dict(seed, frames, bad_first, cut, drop_packets), SBC audio on PID 0x101 interleaved with it. cut: audio bytes
    left off the end (a partial frame); drop_packets: audio packets left off the start (continuation bytes before the first
    PES start)."""
    es = _synth_es(seed, n_pictures, n_pictures)
    codes = pts_cases.picture_codes(es)
    kinds = [first_kind] + ["pts"] * (len(codes) - 1)
    video = pts_cases.wrap(es, [0] + [c - 3 for c in codes[1:]], kinds, [first_pts + 3003 * k for k in range(len(codes))], seed=seed + 500)
    vp = [video[i:i + 188] for i in range(0, len(video), 188)]
    if not audio:
        return video
    sbc = audio_cases.sbc_stream(audio["seed"], audio["frames"], bad_frames=(0,) if audio.get("bad_first") else ())
    if audio.get("cut"):
        sbc = sbc[:sbc.size - audio["cut"]]
    ats = audio_cases.mux_audio_ts(sbc, pes_bytes=640, first_pts=first_pts)
    ap = [bytes(ats[i:i + 188]) for i in range(0, ats.size, 188)][audio.get("drop_packets", 0):]
    out, j = [], 0
    for i, v in enumerate(vp):                  # audio packets spread evenly over the video packets
        out.append(v)
        while j < len(ap) and j * len(vp) <= (i + 1) * len(ap):
            out.append(ap[j])
            j += 1
    out += ap[j:]
    return b"".join(out)


def decoder_cases():
    """name -> [program TS bytes]; a restart (op 1) before every program but the first"""
    A = lambda seed, frames=40, **kw: dict(seed=seed, frames=frames, **kw)       # noqa: E731
    return {
        # the second program's first video PES has no PTS: its first picture takes the first program's last PTS
        "carry_no_pts": [program(201, 7, 300000, audio=A(11)), program(202, 6, 900000, first_kind="none", audio=A(12))],
        # audio bytes held back at the restart (the first program ends in mid-frame) and continuation bytes before the next
        # program's first audio PES start
        "held_back": [program(203, 6, 45000, audio=A(13, 37, cut=23)), program(204, 8, 7000000, audio=A(14, 44, drop_packets=2)),
                      program(205, 5, 123456, first_kind="none", audio=A(15, 30, cut=61))],
        # a program whose first audio frame is rejected, restarted straight after it, then a good one
        "rejected_first": [program(206, 6, 90000, audio=A(16)), program(207, 5, 180000, audio=A(17, 20, bad_first=True)),
                           program(208, 6, 270000, audio=A(18, 33))],
        # the same title restarted at a later picture (a seek): pts jump back
        "seek_back": [program(209, 9, 2000000, audio=A(19, 50)), program(209, 9, 1000000, audio=A(19, 50, drop_packets=3))],
    }


def paced_cases():
    """name -> dict(ntsc, fc0, op, segments [(synth seed, pts)], modes, tail_fields, cmds, tail_cmds): the restart `op` (1 reset,
    2 video_pause(0)) before the first push of every later segment, show_progress(180)-style overlays staged at restarts"""
    out = {}
    rising = lambda n, base: [base + 3003 * k for k in range(n)]                       # noqa: E731
    ov = lambda k: oc._cmd(k, 180, 20)                                                  # noqa: E731
    for ntsc in (1, 0):
        std = "ntsc" if ntsc else "pal"
        # a new title whose pts lie far below the old ones
        out[std + "_new_title"] = dict(ntsc=ntsc, fc0=4, op=1, segments=[(301, rising(6, 9000000)), (302, rising(6, 90000))], modes=[0] * 12,
                                       tail_fields=20, cmds=[ov(1)] + [None] * 5 + [ov(2)] + [None] * 5, tail_cmds={})
        # load_poster: a restart, then the poster pushed with mode 2 / 3 (the scroll) after a title
        out[std + "_poster"] = dict(ntsc=ntsc, fc0=9, op=1, segments=[(303, rising(5, 500000)), (304, rising(1, 77777)), (305, rising(1, 1234))],
                                    modes=[0] * 5 + [2, 3], tail_fields=30, cmds=[None] * 7, tail_cmds={})
        # play_pause: video_pause(0) after a run, pts continuing after a gap (the display waited while paused)
        out[std + "_resume"] = dict(ntsc=ntsc, fc0=2, op=2, segments=[(306, rising(5, 60000)), (307, rising(5, 60000 + 3003 * 5 + 40 * 1500))],
                                    modes=[0] * 10, tail_fields=8, cmds=[None] * 5 + [oc._cmd(None, None, 120)] + [None] * 4, tail_cmds={})
    return out


# -- the restatement ------------------------------------------------------------------------------------------------------
def decoder_restate(programs, carry_reset=False):
    """-> dict(pic_pts [per program, per picture], last [get_pts() after each program], pushes [pts of every push_video of the
    reference: every program's pictures but its last, all of the last program's (flush_picture(1))]).
    carry_reset: the rejected rule that also clears the carried PTS."""
    carry, pic_all, last, pushes = -1, [], [], []
    for i, ts in enumerate(programs):
        if carry_reset and i:
            carry = -1
        es, pes = pts_cases.demux(ts)
        valid = [(o, p) for o, p in pes if p >= 0]
        pics = []
        for x in pts_cases.picture_codes(es):
            v = [p for o, p in valid if o <= x + 2]
            pics.append(v[-1] if v else carry)
        if valid:
            carry = valid[-1][1]
        pic_all.append(pics)
        last.append(pics[-1] if pics else -1)
        pushes += pics if i == len(programs) - 1 else pics[:-1]
    return dict(pic_pts=pic_all, last=last, pushes=pushes)


def _frames(sbc, fs=64):
    """whole frames of a demuxed SBC stream of frame size fs (audio_cases' streams: bitpool 28 gives 64)"""
    n = len(sbc) // fs
    return [bytes(sbc[k * fs:(k + 1) * fs]) for k in range(n)]


def audio_restate_runs(oracle, runs, fs):
    """the general form of audio_restate for streams of one frame size fs: runs[i] = the SBC bytes one program delivered
    between two restarts (submits without a restart between them simply concatenate). -> (pcm per run, pdm of everything).
    A run's bytes are cut to whole frames except for the last run, which ends the stream (the whole-stream checker decodes
    whole frames only as well); each run after the first decodes its first frame twice."""
    spliced, owner = [], []
    for i, b in enumerate(runs):
        fr = _frames(b, fs)
        if not fr:
            continue
        if spliced:
            spliced.append(fr[0])
            owner.append((i, False))
        spliced += fr
        owner += [(i, True)] * len(fr)
    pcm = oracle.sbc_decode(b"".join(spliced))
    assert not isinstance(pcm, int) and pcm.size == 128 * len(spliced), pcm
    pcms = [[] for _ in runs]
    for k, (i, keep) in enumerate(owner):
        if keep:
            pcms[i].append(pcm[128 * k:128 * (k + 1)])
    pcms = [np.concatenate(p) if p else np.zeros(0, np.int16) for p in pcms]
    return pcms, oracle.pdm(np.concatenate(pcms))


def idle_resume_cases():
    """video_pause(0) after an idle run (ef_present_idle while the stream is paused, then op 2 and the rest of the title).
    Restatement only: the reference's display runs only while a picture is pending in the instant-decoder harness, so it
    cannot be pinned there; the idle run and video_pause(0) are each pinned on their own (tests/golden/pacing_pins.json
    tails, the *_resume cases here)."""
    out = {}
    rising = lambda n, base: [base + 3003 * k for k in range(n)]                       # noqa: E731
    for ntsc in (1, 0):
        std = "ntsc" if ntsc else "pal"
        out[std + "_idle_resume"] = dict(ntsc=ntsc, fc0=6, op=2, segments=[(308, rising(4, 80000)), (309, rising(4, 80000 + 3003 * 4 + 90 * 1500))],
                                         modes=[0] * 8, tail_fields=6, cmds=[None] * 4 + [oc._cmd(3, 180, 33)] + [None] * 3, tail_cmds={},
                                         idle_before=[0, 37])
    return out


def audio_restate(oracle, programs, zero_state=False):
    """-> (pcm per program, pdm of the whole run). Every program's audio as the reference's demux lets it through after a
    restart (efo_demux_audio_ts starts with the gate shut), whole frames only; restarted programs decode their first frame
    twice with the filter memory carried. Restated through the whole-stream checker on one spliced stream: each later
    program's first frame appears twice (its probe) and the probe's 128 samples are cut out again; a program whose first frame
    is rejected contributes that frame only (the probe re-synthesises, nothing is output, nothing after it decodes).
    zero_state: the rejected rule that starts every program's audio from zero, as end_of_stream does."""
    if zero_state:
        pcms = []
        for ts in programs:
            p = oracle.sbc_decode(oracle.demux_audio_ts(ts))
            pcms.append(np.zeros(0, np.int16) if isinstance(p, int) else p)
        return pcms, np.concatenate([oracle.pdm(p) for p in pcms])
    spliced, owner = [], []                       # frames of the spliced stream; owner: (program, counts in the output)
    for i, ts in enumerate(programs):
        fr = _frames(oracle.demux_audio_ts(ts))
        if not fr:
            continue
        if fr[0][0] != 0x9C:
            spliced.append(fr[0])
            owner.append((i, False))
            continue
        if spliced:
            spliced.append(fr[0])
            owner.append((i, False))
        for f in fr:
            spliced.append(f)
            owner.append((i, True))
    pcm = oracle.sbc_decode(b"".join(spliced))
    assert not isinstance(pcm, int) and pcm.size == 128 * len(spliced), pcm
    pcms = [[] for _ in programs]
    for k, (i, keep) in enumerate(owner):
        if keep:
            pcms[i].append(pcm[128 * k:128 * (k + 1)])
    pcms = [np.concatenate(p) if p else np.zeros(0, np.int16) for p in pcms]
    return pcms, oracle.pdm(np.concatenate(pcms))


def paced_restate(case, frames, oracle, zero_stores=False):
    """the case through the overlay restatement with restarts: (fields, flip fields, SHA-256 of the rendered field stream).
    frames[i]: the decoded pictures of segment i. zero_stores: the rejected rule that zero-fills the frame stores and
    restarts the store phase (as ef_reset)."""
    d = oc.OverlayDisplay(case["ntsc"], case["fc0"])
    calls, k, last, flips = [], 0, None, []
    for si, (_, pts) in enumerate(case["segments"]):
        if si:
            if case.get("idle_before") and case["idle_before"][si]:
                calls.append((None, d.idle(case["idle_before"][si])))
            d.fc_origin = 0
            if zero_stores:
                d.pictures = 0
        for p in pts:
            oc.stage(d, case["cmds"][k])
            f, last, _ = d.push(int(p), case["modes"][k])
            flips.append(last)
            calls.append((k, f))
            k += 1
    total = (last + 1 + case["tail_fields"] - case["fc0"]) & M32
    calls.append((None, d.idle(total - len(d.emitted))))
    ovs = d.overlays()
    r = oc.OverlayRenderer(oracle, case["ntsc"])
    seg = [(si, j) for si, (_, pts) in enumerate(case["segments"]) for j in range(len(pts))]
    whole, i = hashlib.sha256(), 0
    for kk, fields in calls:
        if kk is not None:
            si, j = seg[kk]
            if zero_stores and si and j == 0:
                r.reset()
            r.decoded(j if zero_stores else kk, frames[si][j])
        for f in fields:
            whole.update(r.field(f, ovs[i]).tobytes())
            i += 1
    return len(d.emitted), flips, whole.hexdigest()
