"""Every encode source and every decode output of the library, described once for the tests.

SOURCES[name] (the CFB_PIXEL_* name, "-alpha" for the RGBA 4:4:4:4 codec of a 16-bit RGBA source): how a test builds a frame
of that source, the int16 planes the reference encoder transforms from it, and how the oracle forms its coded bands.
OUTPUTS[name] (the CFB_PIXEL_* name, "-alpha" for the B64A frame of an RGBA 4:4:4:4 codec): the numpy restatement of the
frame the reference decoder writes from the reconstructed planes, the bytes of one row, the reference's DECODED_FORMAT_*
code and its reduced-resolution rules.  The restatements are pinned to the reference decoder
on the CPU (test_output16.py, test_output_v210.py, test_output_byr4.py, test_reduced_res_outputs.py, test_rgba64.py)."""
import ctypes as C
from functools import partial
from typing import Callable, NamedTuple, Optional

import numpy as np

import byr4_out_util as b4
import oracle_lib as ol
import parity_util as pu

CANARY = 0xA5                                             # fill of output buffers: bytes nobody writes keep it
HALF, QUARTER = 2, 3                                      # DECODED_RESOLUTION_HALF / _QUARTER
COLOR_FORMAT_B64A, COLOR_FORMAT_RG64 = 30, 121            # Codec/color.h:96 / :161
ALPHA_DC_OFFSET, ALPHA_GAIN = 256, 9400                   # Codec/codec.h:164-165


# ================================================================ sources
def yuyv_to_uyvy(frame):
    out = np.empty_like(frame)
    out[:, 0::2] = frame[:, 1::2]
    out[:, 1::2] = frame[:, 0::2]
    return out


# ---------------------------------------------------------------- YU64 (16-bit packed 4:2:2 -> 10-bit planes)
def yu64_from_yuyv(frame8, rng):
    """16-bit packed Y0 C1 Y1 C3 frame whose top 8 bits are the given 8-bit frame and whose low bits are random."""
    f16 = (frame8.astype(np.uint16) << 8) | rng.integers(0, 256, frame8.shape).astype(np.uint16)
    return f16                                   # (height, 2 * width) uint16


def unpack_yu64(frame16, precision=10):
    """Codec/frame.c:1556 ConvertYU64ToFrame16s: sample >> (16 - precision); position 1 -> channel 1, position 3 -> channel 2."""
    s = (frame16 >> (16 - precision)).astype(np.int16)
    return [np.ascontiguousarray(s[:, 0::2]), np.ascontiguousarray(s[:, 1::4]), np.ascontiguousarray(s[:, 3::4])]


# ---------------------------------------------------------------- V210 (10-bit packed 4:2:2)
def pack_v210(y, cb, cr):
    """y (h, w), cb / cr (h, w/2) 10-bit -> (h, pitch/4) uint32: component stream Cb Y Cr Y ..., three per word at bits
    0, 10, 20 (Codec/convert.c:3365), rows padded to a multiple of 128 bytes (48 pixels)."""
    h, w = y.shape
    comp = np.zeros((h, 2 * w), np.uint32)
    comp[:, 0::4], comp[:, 1::4], comp[:, 2::4], comp[:, 3::4] = cb, y[:, 0::2], cr, y[:, 1::2]
    nwords = ((w + 47) // 48) * 32
    padded = np.zeros((h, nwords * 3), np.uint32)
    padded[:, :2 * w] = comp
    return (padded[:, 0::3] | (padded[:, 1::3] << 10) | (padded[:, 2::3] << 20)).astype(np.uint32)


def v210_from_yuyv(frame8, rng):
    """10-bit planes whose top 8 bits are the given 8-bit YUYV frame (random low bits) and their V210 packing.
    Returns (words, [Y, ch1, ch2]) with ch1 = Cr (second chroma), ch2 = Cb as ConvertV210ToFrame16s assigns them."""
    h, w2 = frame8.shape
    w = w2 // 2
    y = (frame8[:, 0::2].astype(np.uint32) << 2) | rng.integers(0, 4, (h, w)).astype(np.uint32)
    cb = (frame8[:, 1::4].astype(np.uint32) << 2) | rng.integers(0, 4, (h, w // 2)).astype(np.uint32)
    cr = (frame8[:, 3::4].astype(np.uint32) << 2) | rng.integers(0, 4, (h, w // 2)).astype(np.uint32)
    return pack_v210(y, cb, cr), [y.astype(np.int16), cr.astype(np.int16), cb.astype(np.int16)]


# ---------------------------------------------------------------- RG48 (packed 16-bit RGB -> 4:4:4, 12 bit)
def synthetic_rg48(rng, width, height, kind="natural"):
    if kind == "random":
        return rng.integers(0, 65536, (height, width * 3)).astype(np.uint16)
    if kind == "extreme":
        return np.where(rng.integers(0, 2, (height, width * 3)) == 0, 0, 65535).astype(np.uint16)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float32)
    f = np.empty((height, width * 3), np.uint16)
    for c, (a, b) in enumerate(((37.0, 23.0), (51.0, 31.0), (29.0, 47.0))):
        v = 30000 + 20000 * np.sin(xx / a) * np.cos(yy / b) + 6000 * np.sin((xx + 2 * yy) / 5.0) * (xx > width / 2)
        v += rng.normal(0, 300.0, v.shape)
        f[:, c::3] = np.clip(v, 0, 65535).astype(np.uint16)
    return f


def unpack_rg48(frame16, precision=12):
    """Codec/frame.c:5968 ConvertRGB48ToFrame16s, default branch (:6130-6164): plane0 = G, plane1 = R, plane2 = B,
    each `>> (16 - precision)`."""
    sh = 16 - precision
    r, g, b = frame16[:, 0::3], frame16[:, 1::3], frame16[:, 2::3]
    return [np.ascontiguousarray((x >> sh).astype(np.int16)) for x in (g, r, b)]


# ---------------------------------------------------------------- 10-bit packed RGB (one 32-bit word per pixel)
RGB30_FORMATS = {          # name: (COLOR_FORMAT_* of Codec/color.h, byte swapped, bit position of R, G, B)
    "RG30": (122, False, (0, 10, 20)),
    "R210": (123, True, (20, 10, 0)),
    "AR10": (124, False, (20, 10, 0)),
    "AB10": (125, False, (0, 10, 20)),
    "DPX0": (128, True, (22, 12, 2)),
}


def pack_rgb30(name, r, g, b):
    """10-bit r, g, b planes (h, w) -> (h, w) uint32 words in the layout of Codec/spatial.c:2118-2268."""
    _, swap, (pr, pg, pb) = RGB30_FORMATS[name]
    words = ((r.astype(np.uint32) << pr) | (g.astype(np.uint32) << pg) | (b.astype(np.uint32) << pb)).astype(np.uint32)
    return words.byteswap() if swap else words


def rgb30_planes(r, g, b, precision=12):
    """planes the reference transforms: G, R, B at `precision` bits (value << (precision - 10))."""
    sh = precision - 10
    return [(g.astype(np.int32) << sh).astype(np.int16), (r.astype(np.int32) << sh).astype(np.int16), (b.astype(np.int32) << sh).astype(np.int16)]


# ---------------------------------------------------------------- B64A / RG64 (16-bit RGBA -> 4:4:4 or 4:4:4:4, 12 bit)
# word of each plane (G, R, B, A) inside a pixel of four 16-bit words
RGBA64_WORDS = {"B64A": (2, 1, 3, 0), "RG64": (1, 0, 2, 3)}


def alpha_curve(a16):
    """The encoder's alpha curve on 16-bit samples (Codec/frame.c:6697-6706, :5942-5951): a = A >> 4, and 0 < a < 4095
    -> ((a * 223 + 128) >> 8) + 256; 0 and 4095 pass through."""
    a = (a16.astype(np.int32) >> 4)
    mid = (a > 0) & (a < 4095)
    return np.where(mid, ((a * 223 + 128) >> 8) + 256, a).astype(np.int16)


def unpack_rgba64(frame16, name, alpha):
    """(height, 4 * width) uint16 -> planes G, R, B (+ A) at 12 bits, as ConvertBGRA64ToFrame_4444_16s (B64A, frame.c:6569)
    and ConvertRGBA64ToFrame16s (RG64, frame.c:5737, default branch) produce them."""
    g, r, b, a = RGBA64_WORDS[name]
    planes = [np.ascontiguousarray((frame16[:, k::4] >> 4).astype(np.int16)) for k in (g, r, b)]
    if alpha:
        planes.append(np.ascontiguousarray(alpha_curve(frame16[:, a::4])))
    return planes


def synthetic_alpha(rng, width, height):
    """16-bit alpha that covers the curve: 8 x 8 blocks of raw 0-15 (a = 0), 16-31 (a = 1, the lowest curved input),
    65504-65519 (a = 4094, the highest), 65520-65535 (a = 4095), a ramp over the whole range and uniform noise."""
    kind = np.repeat(np.repeat(rng.integers(0, 6, ((height + 7) // 8, (width + 7) // 8)), 8, 0), 8, 1)[:height, :width]
    lo = rng.integers(0, 16, (height, width))
    yy, xx = np.mgrid[0:height, 0:width]
    ramp = ((xx * 97 + yy * 61) * 16) % 65536
    choices = [lo, 16 + lo, 65504 + lo, 65520 + lo, ramp, rng.integers(0, 65536, (height, width))]
    out = np.zeros((height, width), np.int64)
    for k, v in enumerate(choices):
        out = np.where(kind == k, v, out)
    return out.astype(np.uint16)


def synthetic_rgba64(rng, width, height, kind, name):
    """(height, 4 * width) uint16 frame in the word order of `name` (B64A / RG64): colours as synthetic_rg48, alpha from
    synthetic_alpha."""
    rgb = synthetic_rg48(rng, width, height, kind)
    g, r, b, a = RGBA64_WORDS[name]
    f = np.empty((height, 4 * width), np.uint16)
    f[:, r::4], f[:, g::4], f[:, b::4] = rgb[:, 0::3], rgb[:, 1::3], rgb[:, 2::3]
    f[:, a::4] = synthetic_alpha(rng, width, height)
    return f


# ---------------------------------------------------------------- BYR4 (16-bit Bayer, curve applied -> 4 planes, 12 bit)
def mosaic_from_rg48(frame16, fmt=0):
    """Bayer mosaic (height x width uint16) sampled from a packed RGB frame; fmt = BAYER_FORMAT_* phase."""
    r, g, b = frame16[:, 0::3], frame16[:, 1::3], frame16[:, 2::3]
    h, w = r.shape
    m = np.empty((h, w), np.uint16)
    # quad positions (line, col): RED_GRN: r g / g b ; GRN_RED: g r / b g ; GRN_BLU: g b / r g ; BLU_GRN: b g / g r
    lay = {0: ("r", "g", "g", "b"), 1: ("g", "r", "b", "g"), 2: ("g", "b", "r", "g"), 3: ("b", "g", "g", "r")}[fmt]
    src = {"r": r, "g": g, "b": b}
    m[0::2, 0::2] = src[lay[0]][0::2, 0::2]; m[0::2, 1::2] = src[lay[1]][0::2, 1::2]
    m[1::2, 0::2] = src[lay[2]][1::2, 0::2]; m[1::2, 1::2] = src[lay[3]][1::2, 1::2]
    return m


def synthetic_mosaic(rng, w, h, kind, phase=0):
    """(h, w) uint16 Bayer mosaic: "natural" (sampled from a smooth RGB frame), "random", "extreme" (0 / 65535),
    "constant"."""
    if kind == "natural":
        return mosaic_from_rg48(synthetic_rg48(rng, w, h, "natural"), phase)
    if kind == "extreme":
        return np.where(rng.integers(0, 2, (h, w)) == 0, 0, 65535).astype(np.uint16)
    if kind == "constant":
        return np.full((h, w), 0x8120, np.uint16)
    return rng.integers(0, 65536, (h, w)).astype(np.uint16)


def bayer_log90_curve(precision=12):
    """The default encode curve of Codec/frame.c:5208-5245: curve[i] = (int)(lin2log((float)i / 16384, 90) * 4095) with
    lin2log (Common/AVIExtendedHeader.h:153) evaluated in double and rounded to float, 1 << 14 entries, curve[0] = 0."""
    i = np.arange(1 << 14, dtype=np.float32) / np.float32(1 << 14)
    v = (np.log10(i.astype(np.float64) * (np.float64(np.float32(90.0)) - 1.0) + 1.0) / np.log10(np.float64(np.float32(90.0)))).astype(np.float32)
    curve = (v * np.float32((1 << precision) - 1)).astype(np.int32)
    curve[0] = 0
    return curve.astype(np.uint16)


def unpack_byr4(bayer16, fmt=0, precision=12, curve=None):
    """Codec/frame.c:4993 ConvertBYR4ToFrame16s: planes G, R-G, B-G, dG.  curve=None: encode_curve_preset branch
    (:5040-5200, samples >> 4); else the table branch (:5206-5420): sample -> curve[sample >> 2]."""
    sh = 16 - precision
    if curve is None:
        conv = lambda a: (a >> sh).astype(np.int32)
    else:
        conv = lambda a: curve[(a >> 2).astype(np.int64)].astype(np.int32)
    q0 = conv(bayer16[0::2, 0::2]); q1 = conv(bayer16[0::2, 1::2])
    q2 = conv(bayer16[1::2, 0::2]); q3 = conv(bayer16[1::2, 1::2])
    r, g1, g2, b = {0: (q0, q1, q2, q3), 1: (q1, q0, q3, q2), 2: (q2, q0, q3, q1), 3: (q3, q1, q2, q0)}[fmt]
    mid = 1 << 12
    gg = (g1 + g2) >> 1
    planes = [gg, (r - gg + mid) >> 1, (b - gg + mid) >> 1, (g1 - g2 + mid) >> 1]
    return [np.ascontiguousarray(p.astype(np.int16)) for p in planes]


# ---------------------------------------------------------------- BYR5 (12-bit packed Bayer -> 4 planes, 12 bit)
# component rows of a packed row in phase order (frame.c:5614-5640): index of R, G1, G2, B
BYR5_ORDER = {0: (0, 1, 2, 3), 1: (1, 0, 3, 2), 2: (2, 0, 3, 1), 3: (3, 1, 2, 0)}


def byr5_random_components(rng, pw, ph, kind="random"):
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


def byr5_pack(comps, pitch=None):
    """(4, ph, pw) 12-bit samples -> (ph, pitch) uint8 packed rows: 4 pw high bytes, then 2 pw bytes of low nibbles
    (sample 2i: low nibble of byte i, 2i + 1: high nibble)."""
    _, ph, pw = comps.shape
    s = comps.transpose(1, 0, 2).reshape(ph, 4 * pw).astype(np.uint16)
    out = np.zeros((ph, pitch or 6 * pw), np.uint8)
    out[:, :4 * pw] = (s >> 4).astype(np.uint8)
    lo = (s & 15).astype(np.uint8)
    out[:, 4 * pw:6 * pw] = lo[:, 0::2] | (lo[:, 1::2] << 4)
    return out


def byr5_components(frame, pw):
    """The inverse of byr5_pack: (ph, >= 6 pw) uint8 -> (4, ph, pw) 12-bit samples."""
    hi = frame[:, :4 * pw].astype(np.uint16)
    nib = frame[:, 4 * pw:6 * pw]
    lo = np.empty_like(hi)
    lo[:, 0::2] = nib & 15
    lo[:, 1::2] = nib >> 4
    s = (hi << 4) | lo
    return s.reshape(frame.shape[0], 4, pw).transpose(1, 0, 2)


def byr5_planes(frame, pw, phase, height=None):
    """The four int16 planes G, R-G, B-G, dG of ConvertBYR5ToFrame16s (SIMD loop, frame.c:5642-5668).  height: the
    codec's plane height; plane rows at or beyond the frame's rows repeat its last row (srcrow = display_height - 1)."""
    c = byr5_components(frame, pw).astype(np.int32)
    if height is not None and height > c.shape[1]:
        c = np.concatenate([c, np.repeat(c[:, -1:], height - c.shape[1], axis=1)], axis=1)
    r, g1, g2, b = (c[i] for i in BYR5_ORDER[phase])
    gg = (g1 + g2) >> 1
    mid = 1 << 12
    out = [gg, (r - gg + mid) >> 1, (b - gg + mid) >> 1, (g1 - g2 + mid) >> 1]
    return [np.ascontiguousarray(p.astype(np.int16)) for p in out]


# ---------------------------------------------------------------- the table
def coded_region(pyr):
    """The coded bands of a pyramid: LL3 and every highpass band (the LL of levels 1 and 2 is not coded)."""
    return {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}


def _planar_bands(nchan, frame, planes, quant):
    pyr = pu.forward_pyramid_planes(ol.oracle(), planes, quant.table(nchan), tuple(quant.prescale), quant.midpoint_prequant)
    return coded_region(pyr)


def _packed_422_bands(fmt, frame, planes, quant):
    return pu.oracle_forward_422(ol.oracle(), frame, quant, fmt)


class Source(NamedTuple):
    frame: Callable         # (rng, w, h, kind) -> (packed frame, planes the reference encoder transforms; None for 8-bit 4:2:2)
    nchan: int
    precision: int
    bands: Callable         # (frame, planes, quant) -> the oracle's coded-region bands {(c, level, name): array}


def _source(frame, nchan, precision, packed_422=None):
    """packed_422: the oracle's 4:2:2 format (0 YUYV, 1 UYVY) when it transforms the packed frame itself."""
    bands = partial(_planar_bands, nchan) if packed_422 is None else partial(_packed_422_bands, packed_422)
    return Source(frame, nchan, precision, bands)


def _yuyv_frame(uyvy, rng, w, h, kind):
    f8 = pu.synthetic_yuyv(rng, w, h, kind)
    return (yuyv_to_uyvy(f8) if uyvy else f8), None


def _yu64_frame(rng, w, h, kind):
    f16 = yu64_from_yuyv(pu.synthetic_yuyv(rng, w, h, kind), rng)
    return f16, unpack_yu64(f16)


def _v210_frame(rng, w, h, kind):
    return v210_from_yuyv(pu.synthetic_yuyv(rng, w, h, kind), rng)


def _rg48_frame(planar, rng, w, h, kind):
    rg = synthetic_rg48(rng, w, h, kind)
    planes = unpack_rg48(rg)
    return (np.ascontiguousarray(np.concatenate(planes, axis=0)) if planar else rg), planes


def _rgb30_frame(name, rng, w, h, kind):
    """Uniform 10-bit samples whatever the kind."""
    r, g, b = (rng.integers(0, 1024, (h, w)).astype(np.uint32) for _ in range(3))
    return pack_rgb30(name, r, g, b), rgb30_planes(r, g, b)


def _rgba64_frame(name, alpha, rng, w, h, kind):
    f = synthetic_rgba64(rng, w, h, kind, name)
    return f, unpack_rgba64(f, name, alpha)


def _byr4_frame(rng, w, h, kind):
    """Phase 0, curve already applied."""
    m = synthetic_mosaic(rng, w, h, kind)
    return m, unpack_byr4(m, 0)


def _byr5_frame(rng, w, h, kind):
    """Phase 0; w x h Bayer samples, planes of w / 2 x h / 2."""
    f = byr5_pack(byr5_random_components(rng, w // 2, h // 2, kind))
    return f, byr5_planes(f, w // 2, 0)


SOURCES = {
    "YUYV": _source(partial(_yuyv_frame, False), 3, 10, packed_422=0),
    "UYVY": _source(partial(_yuyv_frame, True), 3, 10, packed_422=1),
    "YU64": _source(_yu64_frame, 3, 10),
    "V210": _source(_v210_frame, 3, 10),
    "RG48": _source(partial(_rg48_frame, False), 3, 12),
    **{n: _source(partial(_rgb30_frame, n), 3, 12) for n in RGB30_FORMATS},
    "PLANAR16": _source(partial(_rg48_frame, True), 3, 12),
    **{n + suffix: _source(partial(_rgba64_frame, n, alpha), 3 + alpha, 12)
       for n in RGBA64_WORDS for suffix, alpha in (("", False), ("-alpha", True))},
    "BYR4": _source(_byr4_frame, 4, 12),
    "BYR5": _source(_byr5_frame, 4, 12),
}


# ================================================================ outputs
def row16u_tail_col(band_width):
    """First band column produced by the scalar tail of Codec/InvertHorizontalStrip16s.c:16571 InvertHorizontalStrip16sToRow16u
    (8-column SSE2 loop up to post_column = width - width % 8 - 16, one more group of 7 columns with the SIMD rule)."""
    return (band_width - band_width % 8 - 16) + 7


def row16u(plane, precision):
    """The reference's unsigned 16-bit row output of one reconstructed channel: max(v, 0) << (16 - precision), limited to
    ((1 << precision) - 1) << shift where its SSE2 loop runs (the `protection` clamp) and to 65535 in the scalar tail and
    at the right border (SATURATE_16U)."""
    s = 16 - precision
    v = np.maximum(plane.astype(np.int64), 0) << s
    hi = np.full(plane.shape[1], ((1 << precision) - 1) << s, np.int64)
    hi[2 * row16u_tail_col(plane.shape[1] // 2):] = 65535
    return np.minimum(v, hi[None, :]).astype(np.uint16)


def pack_yu64(planes, precision=10):
    """[Y, ch1, ch2] int16 planes -> packed Y0 C1 Y1 C3 (height x 2*width uint16), Codec/decoder.c:26351-26366."""
    y, c1, c3 = [row16u(p, precision) for p in planes]
    h, w = y.shape
    out = np.zeros((h, 2 * w), np.uint16)
    out[:, 0::2] = y
    out[:, 1::4] = c1
    out[:, 3::4] = c3
    return out


def pack_rg48(planes, precision=12):
    """[G, R, B] int16 planes -> packed R G B (height x 3*width uint16), Codec/wavelet.c:4947 TransformInverseRGB444ToRGB48."""
    g, r, b = [row16u(p, precision) for p in planes]
    h, w = g.shape
    out = np.zeros((h, 3 * w), np.uint16)
    out[:, 0::3], out[:, 1::3], out[:, 2::3] = r, g, b
    return out


def b64a_tail_col(band_width):
    """First band column produced by the scalar code of Codec/InvertHorizontalStrip16s.c:13298 InvertHorizontalStrip16sRGB2B64A:
    its 8-column SSE2 loop runs up to post_column = width - width % 8 (:13319) and always leaves the right border column."""
    return band_width - band_width % 8 if band_width % 8 else band_width - 1


def pack_b64a(planes, precision=12):
    """[G, R, B] int16 planes -> 16-bit A R G B words (height x 4*width uint16) as the reference's decoder writes them for
    DECODED_FORMAT_B64A (Codec/decoder.c:26862 -> InvertHorizontalStrip16s.c:13298 InvertHorizontalStrip16sRGB2B64A): alpha is
    0xfff << 4 (:13385); colour samples are limited to the 12-bit maximum where its SSE2 loop runs (:13387 limiterRGB) and to
    65535 in the scalar tail and at the right border (SATURATE_16U)."""
    s = 16 - precision
    top = ((1 << precision) - 1) << s
    h, w = planes[0].shape
    hi = np.full(w, top, np.int64)
    hi[2 * b64a_tail_col(w // 2):] = 65535
    g, r, b = [np.minimum(np.maximum(p.astype(np.int64), 0) << s, hi[None, :]).astype(np.uint16) for p in planes]
    out = np.full((h, 4 * w), top, np.uint16)
    out[:, 1::4], out[:, 2::4], out[:, 3::4] = r, g, b
    return out


def alpha_out(plane):
    """B64A alpha word of an RGBA 4:4:4:4 sample from the reconstructed channel-3 plane.  The reference decoder takes such a
    sample with an alpha output through its active-metadata path (Codec/bayer.c:7144-7147): the ...ToRow16u sample >> 4,
    i.e. the 12-bit sample limited to [0, 4095] in every column, then ((a - 256) << 3) * 9400 >> 12 limited to [0, 65535]
    (bayer.c:16215-16224 Convert4444LinesToOutput)."""
    a = np.clip(plane.astype(np.int64), 0, 4095)
    return np.clip(((a - ALPHA_DC_OFFSET) * (8 * ALPHA_GAIN)) >> 12, 0, 65535).astype(np.uint16)


def pack_b64a_alpha(planes, precision=12):
    """[G, R, B, A] int16 planes -> the reference decoder's B64A frame of an RGBA 4:4:4:4 sample: the colour samples of its
    RG48 frame (pack_rg48, the ...ToRow16u rule) and the de-companded alpha (alpha_out), A R G B per pixel."""
    rg = pack_rg48(planes[:3], precision)
    h, w = planes[0].shape
    out = np.empty((h, 4 * w), np.uint16)
    out[:, 0::4] = alpha_out(planes[3])
    out[:, 1::4], out[:, 2::4], out[:, 3::4] = rg[:, 0::3], rg[:, 1::3], rg[:, 2::3]
    return out


def pack_rgb30_output(name, planes, precision=12):
    """[G, R, B] int16 planes -> the reference decoder's 10-bit packed RGB words (height x width uint32) for
    DECODED_FORMAT_RG30 / R210 / DPX0 / AR10 / AB10 (Codec/decoder.c:26893 -> InvertHorizontalStrip16s.c:14812
    InvertHorizontalStrip16sRGB2RG30): every sample limited to [0, 2^precision - 1] (:14892 limiterRGB; its scalar code
    clamps alike), >> 2 (:15552), packed as on the encode side.  NOTE the reference's lowpass decode adds a format-dependent
    offset to LL3 (decoder.c:12270-12316: 6 for these formats, 0 for RG48 / B64A), so its bands differ between output
    formats; that offset is applied by the host's band decode, upstream of the transform."""
    top = (1 << precision) - 1
    g, r, b = [(np.clip(p.astype(np.int64), 0, top) >> (precision - 10)).astype(np.uint32) for p in planes]
    return pack_rgb30(name, r, g, b)


# ---------------------------------------------------------------- V210 output
def v210_row_bytes(w):
    """Bytes of one V210 row: ceil(W / 6) groups of 16 bytes (the last one partial when W % 6 != 0)."""
    return (w + 5) // 6 * 16


def v210_natural_pitch(w):
    """cfb_layout.frame_pitch of a V210 codec: rows padded to 48 pixels = 128 bytes."""
    return (w + 47) // 48 * 128


def pack_v210_components(y, cr, cb):
    """10-bit components y (h, w), cr / cb (h, w/2) -> V210 words (h, 4 * ceil(W / 6)) uint32 as
    Codec/convert.c:13526 ConvertPlanarYUVToV210 writes them: Cb0 Y0 Cr0 | Y1 Cb1 Y2 | Cr1 Y3 Cb2 | Y4 Cr2 Y5 at bits 0 / 10 / 20.
    The partial last group of W % 6 != 0 follows its scalar loop (:13889-13965), which keeps the previous components
    where a column is past the width.  At W % 6 == 4 that loop reads one Cb sample past the row (X, not reproducible);
    this restatement puts Cb1 there, as the library does."""
    y, cr, cb = [np.asarray(a, np.uint32) for a in (y, cr, cb)]
    h, w = y.shape
    full, rem = w // 6, w % 6
    ng = full + (rem > 0)
    comp = np.zeros((h, ng, 12), np.uint32)
    for p in range(3):
        comp[:, :full, 4 * p] = cb[:, p:3 * full:3]
        comp[:, :full, 4 * p + 1] = y[:, 2 * p:6 * full:6]
        comp[:, :full, 4 * p + 2] = cr[:, p:3 * full:3]
        comp[:, :full, 4 * p + 3] = y[:, 2 * p + 1:6 * full:6]
    if rem:
        c = 6 * full
        cb0, y0, cr0, y1 = cb[:, c // 2], y[:, c], cr[:, c // 2], y[:, c + 1]
        if rem == 2:
            tail = [cb0, y0, cr0, y1, cb0, y0, cr0, y1, cb0, y1, cr0, y0]
        else:
            cb1, y2, cr1, y3 = cb[:, c // 2 + 1], y[:, c + 2], cr[:, c // 2 + 1], y[:, c + 3]
            tail = [cb0, y0, cr0, y1, cb1, y2, cr1, y3, cb1, y3, cr1, y2]
        comp[:, full, :] = np.stack(tail, axis=1)
    words = comp[:, :, 0::3] | (comp[:, :, 1::3] << 10) | (comp[:, :, 2::3] << 20)
    return words.reshape(h, 4 * ng).astype(np.uint32)


def pack_v210_output(planes, precision=10):
    """[Y, ch1, ch2] int16 planes of a 4:2:2 decode -> the reference decoder's V210 words (decoder.c:26303 ->
    InvertHorizontalStrip16s.c:6490 -> convert.c:16126 ConvertYUVStripPlanarToV210 with precision 16): every component is
    the ...ToRow16u sample of YU64 (row16u) >> 6; Cb = channel 2, Cr = channel 1."""
    y, cr, cb = [row16u(p, precision) >> 6 for p in planes]
    return pack_v210_components(y, cr, cb)


def v210_x_mask(w):
    """Per-word mask (4 * ceil(W / 6),) that clears the one field the reference does not determine: X, bits 20-29 of word 2
    of the last group when W % 6 == 4."""
    m = np.full(4 * ((w + 5) // 6), 0xFFFFFFFF, np.uint32)
    if w % 6 == 4:
        m[-2] = ~np.uint32(0x3FF << 20)
    return m


def v210_agree(w, pitch):
    """The bytes of a (h, pitch) V210 frame two reference decodes must agree on (pu.ref_decode's `agree`): every row's
    words except X."""
    m = np.zeros(pitch, np.uint8)
    m[:v210_row_bytes(w)] = v210_x_mask(w).view(np.uint8)
    return m


def v210_frame_words(buf, w, h):
    """The V210 words of a frame buffer (h rows of `pitch` bytes, any dtype) -> (h, 4 * ceil(W / 6)) uint32."""
    b = np.ascontiguousarray(buf).view(np.uint8).reshape(h, -1)
    return np.ascontiguousarray(b[:, :v210_row_bytes(w)]).view("<u4")


# ---------------------------------------------------------------- BYR4 output of a Bayer sample
def restore_table(base=90.0):
    """decoder->BYR4LinearRestore for a log encode curve (Codec/decoder.c:10714-10785, default base 90):
    (int)(CURVE_LOG2LIN((float)j / 16384.0f, base) * 65535.0f), CURVE_LOG2LIN = (pow(b, i) - 1) / (b - 1) in double
    returned as float (Common/AVIExtendedHeader.h:115-123), limited to [0, 65535]."""
    j = (np.arange(16384, dtype=np.float32) / np.float32(16384.0)).astype(np.float64)
    b = np.float64(np.float32(base))
    lin = ((np.power(b, j) - 1.0) / (b - 1.0)).astype(np.float32)
    return np.clip((lin * np.float32(65535.0)).astype(np.int64), 0, 65535).astype(np.uint16)


def rows16u(planes, precision=12):
    """The four RawBayer16 rows of the reference's final level: row16u of every channel."""
    return [np.ascontiguousarray(row16u(p, precision)) for p in planes]


def mosaic_from_rows(rows, phase, restore=None):
    """orc_bayer_to_byr4 on four (ph, pw) uint16 planes -> (2 ph, 2 pw) uint16 mosaic.  restore: the 16384-entry table
    (linear restore, encode_curve_preset == 0) or None (& 0xfffe, encode_curve_preset == 1)."""
    g, rg, bg, gd = [np.ascontiguousarray(r, np.uint16) for r in rows]
    ph, pw = g.shape
    out = np.zeros((2 * ph, 2 * pw), np.uint16)
    fn = b4.load_oracle_bayer().orc_bayer_to_byr4
    fn.restype = None
    vp = C.c_void_p
    tab = None if restore is None else np.ascontiguousarray(restore, np.uint16)
    assert tab is None or tab.size == 16384
    fn(vp(g.ctypes.data), vp(rg.ctypes.data), vp(bg.ctypes.data), vp(gd.ctypes.data), C.c_int(pw * 2), C.c_int(pw), C.c_int(ph),
       C.c_int(phase), vp(tab.ctypes.data) if tab is not None else None, vp(out.ctypes.data), C.c_int(pw * 4))
    return out


def pack_byr4(planes, precision=12, phase=0, restore=None):
    """[G, R-G, B-G, dG] int16 planes -> the reference decoder's BYR4 mosaic: the ...ToRow16u rows (row16u), then
    oracle/cfhd_oracle_bayer.c orc_bayer_to_byr4 at `phase` with the linear restore table or the & 0xfffe rule."""
    return mosaic_from_rows(rows16u(planes, precision), phase, restore)


UNIT4 = [[[1, 1, 1, 1]] * 3] * 4


def oracle_byr4(bands, divisors, prescale, phase, restore=None):
    """{(c, level, name)} QUANTISED coded-region bands of the four channels -> the BYR4 mosaic the reference decodes."""
    planes = pu.inverse_pyramid(ol.oracle(), bands, divisors, prescale, nchan=4)
    return pack_byr4(planes, 12, phase, restore)


# ---------------------------------------------------------------- reduced-resolution outputs
# Numpy restatements of the reference decoder's conversion of a lowpass image to pixels:
#   YU64, half (LL1)         decoder.c:22883 CopyLowpass16sToBuffer -> frame.c:11146 ConvertLowpass16sToYUV64
#   10-bit RGB, quarter      decoder.c:17000 ConvertQuarterFrameToBuffer -> convert.c:16869 ConvertUnpacked16sRowToRGB30
# and the routine the reference names for RG48 at quarter resolution (convert.c:17415 ConvertUnpacked16sRowToRGB48), which its
# decoder does not follow on LL2 values above 16383 (test_reduced_res_outputs.py), so the library does not decode it.
def yu64_half(planes, precision=10):
    """[Y, ch1, ch2] LL1 images -> packed Y0 C1 Y1 C2 words (h x 2w uint16): the scalar loop of ConvertLowpass16sToYUV64
    (its MMX block is compiled out), min(max(ll, 0), 4095) << 4 at 10 bits (16383 << 2 at 12)."""
    s = 16 - precision - 2
    y, c1, c2 = [np.minimum(np.maximum(p.astype(np.int64), 0), 0xFFFF >> s) << s for p in planes]
    h, w = y.shape
    out = np.zeros((h, 2 * w), np.uint16)
    out[:, 0::2], out[:, 1::4], out[:, 3::4] = y, c1, c2
    return out


def rg48_quarter(planes, precision=12):
    """[G, R, B] LL2 images -> packed R G B (h x 3w uint16) as the scalar loop of ConvertUnpacked16sRowToRGB48 writes them
    (its SSE2 block is compiled out): min(max(ll << (16 - precision - 2), 0), 65535)."""
    s = 16 - precision - 2
    g, r, b = [np.minimum(np.maximum(p.astype(np.int64), 0) << s, 65535) for p in planes]
    h, w = g.shape
    out = np.zeros((h, 3 * w), np.uint16)
    out[:, 0::3], out[:, 1::3], out[:, 2::3] = r, g, b
    return out


def rgb10_simd(x, shift):
    """The SSE2 loop of ConvertUnpacked16sRowToRGB30 on int16 values: subs_epu16(adds_epi16(x, 0x4000), 0x4000), slli_epi16
    by `shift`, srli_epi16 by 6.  The saturating add does not saturate values below -0x4000, so they do not go to 0."""
    a = np.clip(x.astype(np.int64) + 0x4000, -32768, 32767) & 0xFFFF       # adds_epi16, as unsigned lanes
    v = np.maximum(a - 0x4000, 0)                                            # subs_epu16
    return ((v << shift) & 0xFFFF) >> 6


def rgb10_tail(x, shift):
    """The scalar tail of ConvertUnpacked16sRowToRGB30: min(max(x << shift, 0), 65535) >> 6."""
    return np.minimum(np.maximum(x.astype(np.int64), 0) << shift, 65535) >> 6


def rgb10_quarter(name, planes, precision=12):
    """[G, R, B] LL2 images -> the 10-bit RGB words (h x w uint32) of `name` (RGB30_FORMATS): the SSE2 rule in the columns
    below width - width % 8, the scalar rule right of them, packed as the full-resolution words."""
    s = 16 - precision - 2
    w = planes[0].shape[1]
    post = w - w % 8

    def conv(p):
        out = rgb10_tail(p, s)
        out[:, :post] = rgb10_simd(p[:, :post], s)
        return out.astype(np.uint32)

    g, r, b = [conv(p) for p in planes]
    return pack_rgb30(name, r, g, b)


def ref_decode_reduced(ref_lib, sample, width, height, decoded_format, num_channels, resolution, bytes_per_pixel):
    """Codec-level reference decode at `resolution` (ref_set_decode_resolution + ref_decode_sample_bands, through
    pu.ref_decode).  Returns (the decoded frame, h x w * bytes_per_pixel
    bytes of the reduced size, the bytes right of it in those rows, the rows below it, the dequantised bands the decoder
    held; the LL of the lowest reconstructed level is the image it converted)."""
    out, bands = pu.ref_decode(ref_lib, sample, width, height, decoded_format, num_channels, width * bytes_per_pixel,
                               resolution=resolution)
    ll = bands[(0, resolution - 1, "LL")]
    h, w = ll.shape
    rb = w * bytes_per_pixel
    return out[:h, :rb].copy(), out[:h, rb:], out[h:], bands


def ref_decode_api(ref_lib, sample, width, height, fourcc, resolution, bytes_per_pixel):
    """Public-API reference decode (CFHD_PrepareToDecode with decodedResolution, CFHD_DecodeSample) into a buffer of
    full-size rows; returns (return code, buffer, (decoded width, decoded height))."""
    out = np.zeros((height, width * bytes_per_pixel), np.uint8)
    dims = np.zeros(2, np.int32)
    fn = ref_lib.ref_decode_sample_res
    fn.restype = C.c_int
    rc = fn(sample.ctypes.data_as(C.c_void_p), C.c_int64(sample.size), width, height, fourcc, resolution,
            out.ctypes.data_as(C.c_void_p), width * bytes_per_pixel, dims.ctypes.data_as(C.c_void_p))
    return rc, out, (int(dims[0]), int(dims[1]))


def lowpass_images(bands, resolution, nchan=3):
    return [bands[(c, resolution - 1, "LL")] for c in range(nchan)]


def block_rg48(width, height, block, seed):
    """A packed RG48 frame of 0 / 65535 blocks of block x block pixels per channel: sharp edges the wavelet rings at, so
    that LL2 leaves [0, 16383] on both sides (the quarter-resolution clamps)."""
    rng = np.random.default_rng(seed)
    g = np.where(rng.integers(0, 2, (height // block + 1, width // block + 1, 3)) == 0, 0, 65535).astype(np.uint16)
    img = np.repeat(np.repeat(g, block, 0), block, 1)[:height, :width]
    return np.ascontiguousarray(img.reshape(height, 3 * width))


def reduced_coded_bands(bands, resolution, nchan=3):
    """The coded-region bands a reduced decode reads (LL3 and the highpass of levels 3 .. resolution), from a dump of the
    bands the reference decoder held."""
    lowest = resolution          # half: levels 3 and 2; quarter: level 3
    return {k: v for k, v in bands.items() if k[0] < nchan and k[1] >= lowest and (k[2] != "LL" or k[1] == 3)}


# ---------------------------------------------------------------- the table
class Output(NamedTuple):
    expected: Optional[Callable]   # (planes, precision, ...) -> the frame the reference decoder writes; None: no exact rule
    row_bytes: Callable            # frame width -> bytes of one row
    decoded_format: int            # the reference's DECODED_FORMAT_* (Codec/decoder.h, == COLOR_FORMAT_*; 0: none)
    reduced: dict = {}             # DECODED_RESOLUTION_* -> rule (planes = the lowpass images, precision) -> frame


def _bpp(n):
    return lambda w: n * w


OUTPUTS = {
    # 8-bit 4:2:2: the reference dithers; tests bound it by pu.yuyv_envelope / pu.lowpass_to_422
    "YUYV": Output(None, _bpp(2), pu.COLOR_FORMAT_YUYV),
    "UYVY": Output(None, _bpp(2), pu.COLOR_FORMAT_UYVY),
    "YU64": Output(pack_yu64, _bpp(4), 12, {HALF: yu64_half}),
    "V210": Output(pack_v210_output, v210_row_bytes, 10),
    "RG48": Output(pack_rg48, _bpp(6), pu.COLOR_FORMAT_RG48, {QUARTER: rg48_quarter}),
    "B64A": Output(pack_b64a, _bpp(8), COLOR_FORMAT_B64A),
    "B64A-alpha": Output(pack_b64a_alpha, _bpp(8), COLOR_FORMAT_B64A),
    **{n: Output(partial(pack_rgb30_output, n), _bpp(4), RGB30_FORMATS[n][0],
                 {QUARTER: partial(rgb10_quarter, n)}) for n in RGB30_FORMATS},
    "BYR4": Output(pack_byr4, _bpp(2), pu.COLOR_FORMAT_BYR4),
    # the int16 planes themselves, each at its own width, stacked
    "PLANAR16": Output(None, _bpp(2), 0),
    "BYR5": Output(None, _bpp(3), pu.COLOR_FORMAT_BYR5),
}
