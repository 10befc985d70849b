"""Reduced-resolution outputs of the deep formats (test infrastructure): numpy restatements of the reference decoder's
conversion of a lowpass image to pixels, and the reference probes that pin them.

  YU64, half (LL1)         decoder.c:22883 CopyLowpass16sToBuffer -> frame.c:11146 ConvertLowpass16sToYUV64
  10-bit RGB, quarter      decoder.c:17000 ConvertQuarterFrameToBuffer -> convert.c:16869 ConvertUnpacked16sRowToRGB30
and the routine the reference names for RG48 at quarter resolution (convert.c:17415 ConvertUnpacked16sRowToRGB48), which its
decoder does not follow on LL2 values above 16383 (test_reduced_res_outputs.py), so the library does not decode it.
"""
import ctypes as C

import numpy as np

import parity_util as pu

DECODED_FORMAT_YU64, DECODED_FORMAT_RG48 = 12, 120          # Codec/color.h
HALF, QUARTER = 2, 3                                         # DECODED_RESOLUTION_HALF / _QUARTER
CANARY = 0xA5


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
    """[G, R, B] LL2 images -> the 10-bit RGB words (h x w uint32) of `name` (parity_util.RGB30_FORMATS): the SSE2 rule in
    the columns below width - width % 8, the scalar rule right of them, packed as the full-resolution words."""
    s = 16 - precision - 2
    w = planes[0].shape[1]
    post = w - w % 8

    def conv(p):
        out = rgb10_tail(p, s)
        out[:, :post] = rgb10_simd(p[:, :post], s)
        return out.astype(np.uint32)

    g, r, b = [conv(p) for p in planes]
    return pu.pack_rgb30(name, r, g, b)


def rgb10_decoded_format(name):
    return pu.RGB30_FORMATS[name][0]


def ref_decode_reduced(ref_lib, sample, width, height, decoded_format, num_channels, resolution, bytes_per_pixel):
    """Codec-level reference decode at `resolution` (ref_set_decode_resolution + ref_decode_sample_bands).  Returns (the
    decoded frame, h x w * bytes_per_pixel bytes of the reduced size, the bytes right of it in those rows, the rows below it,
    the dequantised bands the decoder held; the LL of the lowest reconstructed level is the image it converted)."""
    fn = ref_lib.ref_set_decode_resolution
    fn.argtypes, fn.restype = [C.c_int], None
    fn(resolution)
    try:
        out, bands = pu.ref_decode_sample_raw(ref_lib, sample, width, height, decoded_format, num_channels,
                                              width * bytes_per_pixel)
    finally:
        fn(1)
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
