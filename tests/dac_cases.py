"""EF_FIELD_DAC8 restated in numpy (TEST INFRASTRUCTURE): what the video DAC plays of a field the reference's DMA line buffer
holds. The I2S unit sends the two 16-bit halves of each word in swapped order, so buffer sample t ^ 1 plays at time t, and
only its high byte reaches the 8-bit DAC (levels IRE(x) << 8, video.cpp:520)."""
import numpy as np

FIELD_BYTES = {1: 262 * 912, 0: 312 * 1136}             # NTSC 238,944, PAL 354,432


def dac8(u16):
    """uint16 samples (one or more lines, fields or field rows: every line has an even length) -> the DAC's bytes in playback
    order, same shape: byte t of a line = u16[t ^ 1] >> 8"""
    a = np.asarray(u16, dtype=np.uint16)
    assert a.shape[-1] % 2 == 0
    return (a.reshape(-1, 2)[:, ::-1] >> 8).astype(np.uint8).reshape(a.shape)
