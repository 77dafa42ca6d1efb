"""Synthetic SBC streams and an audio transport-stream muxer for the audio tests (SURVEY.md 8f-3). The SBC decoder
does not check the CRC, so any 0x9C-synced mono / 8-subband / 16-block header followed by scale factors and sample
bits is a decodable frame: random frames exercise bit allocation (both modes, all four frequencies), every sample
width 2..16 and the 32-bit wrap-around of the reference's arithmetic. `consistent` streams repeat one header and one
set of scale factors, so every frame consumes exactly the frame size the reference learns from the first one."""
import numpy as np


def sbc_stream(seed, n_frames, bitpool=28, allocation=0, frequency=2, consistent=True, bad_frames=(), loud=False):
    r = np.random.RandomState(seed)
    frame_bytes = 8 + 2 * bitpool                        # header 4 + scale factors 4 + 16 blocks x bitpool bits (when the pool is used up)
    out = np.zeros(n_frames * frame_bytes, dtype=np.uint8)
    sf0 = r.randint(8 if loud else 1, 16 if loud else 12, size=8)
    for k in range(n_frames):
        f = out[k * frame_bytes:(k + 1) * frame_bytes]
        f[0] = 0x9C if k not in bad_frames else 0x00
        f[1] = (frequency << 6) | (3 << 4) | (0 << 2) | (allocation << 1) | 1
        f[2] = bitpool
        f[3] = r.randint(0, 256)                         # CRC: ignored
        sf = sf0 if consistent else r.randint(0, 16, size=8)
        for sb in range(0, 8, 2):
            f[4 + sb // 2] = (int(sf[sb]) << 4) | int(sf[sb + 1])
        f[8:] = r.randint(0, 256, size=frame_bytes - 8)
    return out


def mux_audio_ts(es, pid=0x101, pes_bytes=1024, first_pts=90000, drop_pts_on=()):
    """188-byte TS packets, one PES per `pes_bytes` of audio, PTS on every PES except the indices in drop_pts_on."""
    es = bytes(es)
    pkts, cc, pos, pes_index = [], 0, 0, 0
    while pos < len(es):
        chunk = es[pos:pos + pes_bytes]
        pos += len(chunk)
        with_pts = pes_index not in drop_pts_on
        pts = first_pts + pes_index * 3600
        hdr = bytearray(b"\x00\x00\x01\xC0") + (len(chunk) + (8 if with_pts else 3)).to_bytes(2, "big")
        if with_pts:
            hdr += bytes([0x80, 0x80, 5, 0x21 | ((pts >> 29) & 0x0E), (pts >> 22) & 0xFF, 0x01 | ((pts >> 14) & 0xFE), (pts >> 7) & 0xFF, 0x01 | ((pts << 1) & 0xFE)])
        else:
            hdr += bytes([0x80, 0x00, 0])
        payload = bytes(hdr) + chunk
        first = True
        while payload:
            n = min(184, len(payload))
            head = bytearray([0x47, (0x40 if first else 0) | (pid >> 8), pid & 0xFF, 0x10 | cc])
            if n < 184:                                  # stuff with an adaptation field
                stuff = 184 - n
                head[3] |= 0x20
                head += bytes([stuff - 1]) + (bytes([0x00]) + b"\xFF" * (stuff - 2) if stuff > 1 else b"")
            pkts.append(bytes(head) + payload[:n])
            payload = payload[n:]
            cc = (cc + 1) & 15
            first = False
        pes_index += 1
    return np.frombuffer(b"".join(pkts), dtype=np.uint8).copy()


AUDIO_CASES = ["bp28", "snr_bp12_f0", "bp60_loud", "rejected_frames", "muted_pes", "pid102"]


def synthetic_case(case):
    """(elementary stream, transport stream) of a synthetic audio case"""
    kw = {"bp28": dict(bitpool=28), "snr_bp12_f0": dict(bitpool=12, allocation=1, frequency=0), "bp60_loud": dict(bitpool=60, loud=True, frequency=3),
          "rejected_frames": dict(bitpool=28, bad_frames=(3, 4, 17)), "muted_pes": dict(bitpool=28), "pid102": dict(bitpool=28, frequency=1)}[case]
    es = sbc_stream(1000 + len(case), 40, **kw)
    return es, mux_audio_ts(es, pid=0x102 if case == "pid102" else 0x101, drop_pts_on=(1,) if case == "muted_pes" else ())


def synthetic_batch():
    """51 streams: rejected frames, inconsistent scale factors, loud, empty, shorter than a frame, no sync byte"""
    streams = []
    for i in range(48):
        streams.append(sbc_stream(5000 + i, 3 + i % 11, bitpool=[2, 7, 12, 28, 31, 60, 97, 120][i % 8], allocation=i & 1, frequency=i % 4,
                                  consistent=i % 3 != 0, bad_frames=(2, 5) if i % 5 == 0 else (), loud=i % 7 == 0))
    streams.append(np.zeros(0, dtype=np.uint8))                          # empty
    streams.append(sbc_stream(1, 1)[:40].copy())                         # shorter than its frame
    streams.append(np.full(200, 0x55, dtype=np.uint8))                   # no sync byte at all: rejected
    return streams


def overrun_stream(seed):
    """a stream whose frames 1, 2, 6, 7, 9 and 23 ask for a larger bit pool than frame 0's and read into the next frame"""
    es = sbc_stream(seed, 24, bitpool=28, consistent=False, bad_frames=(3, 4, 11))
    for k in (1, 2, 6, 7, 9, 23):
        es[k * 64 + 2] = 40                              # bit pool 40: 8 + 2 * 40 bytes read
    return es
