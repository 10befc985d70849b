"""BYR5 (12-bit packed Bayer) frames for the tests: packing, the restated unpack of Codec/frame.c:5473
ConvertBYR5ToFrame16s, and the reference encoder's call on a packed frame."""
import numpy as np

import parity_util as pu

COLOR_FORMAT_BYR5 = 105          # Codec/color.h:128

# component rows of a packed row in phase order (frame.c:5614-5640): index of R, G1, G2, B
ORDER = {0: (0, 1, 2, 3), 1: (1, 0, 3, 2), 2: (2, 0, 3, 1), 3: (3, 1, 2, 0)}


def random_components(rng, pw, ph, kind="random"):
    """Four component rows per plane row as (4, ph, pw) 12-bit samples in the frame's order.  kind "extreme": only 0 and
    4095 (with every component taking both values), "random": uniform."""
    if kind == "extreme":
        return np.where(rng.integers(0, 2, (4, ph, pw)) == 0, 0, 4095).astype(np.uint16)
    if kind == "natural":           # smooth gradients + texture + mild noise, a little different per component
        yy, xx = np.mgrid[0:ph, 0:pw].astype(np.float32)
        out = np.empty((4, ph, pw), np.uint16)
        for k, (a, b) in enumerate(((37.0, 23.0), (41.0, 29.0), (43.0, 31.0), (29.0, 47.0))):
            v = 2000 + 1200 * np.sin(xx / a) * np.cos(yy / b) + 400 * np.sin((xx + 2 * yy) / 5.0) * (xx > pw / 2)
            out[k] = np.clip(v + rng.normal(0, 20.0, v.shape), 0, 4095).astype(np.uint16)
        return out
    return rng.integers(0, 4096, (4, ph, pw)).astype(np.uint16)


def pack(comps, pitch=None):
    """(4, ph, pw) 12-bit samples -> (ph, pitch) uint8 packed rows: 4 pw high bytes, then 2 pw bytes of low nibbles
    (sample 2i: low nibble of byte i, 2i + 1: high nibble)."""
    _, ph, pw = comps.shape
    s = comps.transpose(1, 0, 2).reshape(ph, 4 * pw).astype(np.uint16)
    out = np.zeros((ph, pitch or 6 * pw), np.uint8)
    out[:, :4 * pw] = (s >> 4).astype(np.uint8)
    lo = (s & 15).astype(np.uint8)
    out[:, 4 * pw:6 * pw] = lo[:, 0::2] | (lo[:, 1::2] << 4)
    return out


def components(frame, pw):
    """The inverse of pack: (ph, >= 6 pw) uint8 -> (4, ph, pw) 12-bit samples."""
    hi = frame[:, :4 * pw].astype(np.uint16)
    nib = frame[:, 4 * pw:6 * pw]
    lo = np.empty_like(hi)
    lo[:, 0::2] = nib & 15
    lo[:, 1::2] = nib >> 4
    s = (hi << 4) | lo
    return s.reshape(frame.shape[0], 4, pw).transpose(1, 0, 2)


def planes(frame, pw, phase, height=None):
    """The four int16 planes G, R-G, B-G, dG of ConvertBYR5ToFrame16s (SIMD loop, frame.c:5642-5668).  height: the
    codec's plane height; plane rows at or beyond the frame's rows repeat its last row (srcrow = display_height - 1)."""
    c = components(frame, pw).astype(np.int32)
    if height is not None and height > c.shape[1]:
        c = np.concatenate([c, np.repeat(c[:, -1:], height - c.shape[1], axis=1)], axis=1)
    r, g1, g2, b = (c[i] for i in ORDER[phase])
    gg = (g1 + g2) >> 1
    mid = 1 << 12
    out = [gg, (r - gg + mid) >> 1, (b - gg + mid) >> 1, (g1 - g2 + mid) >> 1]
    return [np.ascontiguousarray(p.astype(np.int16)) for p in out]


def ref_encode(ref_lib, frame, pw, ph, phase, quality=4):
    """The reference's EncodeSample on a packed frame of ph plane rows (display height ph; the encoder pads the plane
    height to its own multiple).  Returns (bands, divisors, prescale, sample bytes) as pu.ref_encode_frame."""
    ref_lib.ref_set_bayer_format(phase)
    try:
        return pu.ref_encode_frame(ref_lib, np.ascontiguousarray(frame[:, :6 * pw]), pw, ph, COLOR_FORMAT_BYR5, 1, 4, quality)
    finally:
        ref_lib.ref_set_bayer_format(-1)
