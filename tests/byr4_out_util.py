"""BYR4 output of a Bayer sample for the tests: the restated decode "decoder bands -> BYR4 mosaic" (the ...ToRow16u rows of
parity_util.row16u, then oracle/cfhd_oracle_bayer.c orc_bayer_to_byr4), the restated linear-restore table, and the
reference's own encode (oracle/ref_probe.cpp) and decode (oracle/ref_probe_bayer.cpp) of a mosaic."""
import ctypes as C
import os
import subprocess

import numpy as np

import byr5_util as bu
import oracle_lib as ol
import parity_util as pu

DECODED_FORMAT_BYR4 = pu.COLOR_FORMAT_BYR4      # Codec/decoder.h: DECODED_FORMAT_* == COLOR_FORMAT_*


def load_oracle_bayer():
    """oracle/liboracle_bayer.so (oracle/bayer.mk), built on first use like oracle_lib.load_oracle."""
    path = os.path.join(ol.ORACLE_DIR, "liboracle_bayer.so")
    if not os.path.exists(path):
        subprocess.check_call(["make", "-s", "-C", ol.ORACLE_DIR, "-f", "bayer.mk", "liboracle_bayer.so"])
    return C.CDLL(path)


def ref_bayer_available():
    return os.path.exists(os.path.join(ol.ORACLE_DIR, "_ref", "libcfhd_ref_bayer.so"))


def load_ref_bayer():
    """oracle/_ref/libcfhd_ref_bayer.so: the decoder probe, linked to the unmodified reference of oracle/_ref."""
    return C.CDLL(os.path.join(ol.ORACLE_DIR, "_ref", "libcfhd_ref_bayer.so"))


def restore_table(base=90.0):
    """decoder->BYR4LinearRestore for a log encode curve (Codec/decoder.c:10714-10785, default base 90):
    (int)(CURVE_LOG2LIN((float)j / 16384.0f, base) * 65535.0f), CURVE_LOG2LIN = (pow(b, i) - 1) / (b - 1) in double
    returned as float (Common/AVIExtendedHeader.h:115-123), limited to [0, 65535]."""
    j = (np.arange(16384, dtype=np.float32) / np.float32(16384.0)).astype(np.float64)
    b = np.float64(np.float32(base))
    lin = ((np.power(b, j) - 1.0) / (b - 1.0)).astype(np.float32)
    return np.clip((lin * np.float32(65535.0)).astype(np.int64), 0, 65535).astype(np.uint16)


def rows16u(planes, precision=12):
    """The four RawBayer16 rows of the reference's final level: parity_util.row16u of every channel."""
    return [np.ascontiguousarray(pu.row16u(p, precision)) for p in planes]


def mosaic_from_rows(rows, phase, restore=None):
    """orc_bayer_to_byr4 on four (ph, pw) uint16 planes -> (2 ph, 2 pw) uint16 mosaic.  restore: the 16384-entry table
    (linear restore, encode_curve_preset == 0) or None (& 0xfffe, encode_curve_preset == 1)."""
    g, rg, bg, gd = [np.ascontiguousarray(r, np.uint16) for r in rows]
    ph, pw = g.shape
    out = np.zeros((2 * ph, 2 * pw), np.uint16)
    fn = load_oracle_bayer().orc_bayer_to_byr4
    fn.restype = None
    vp = C.c_void_p
    tab = None if restore is None else np.ascontiguousarray(restore, np.uint16)
    assert tab is None or tab.size == 16384
    fn(vp(g.ctypes.data), vp(rg.ctypes.data), vp(bg.ctypes.data), vp(gd.ctypes.data), C.c_int(pw * 2), C.c_int(pw), C.c_int(ph),
       C.c_int(phase), vp(tab.ctypes.data) if tab is not None else None, vp(out.ctypes.data), C.c_int(pw * 4))
    return out


def oracle_byr4(bands, divisors, prescale, phase, restore=None):
    """{(c, level, name)} QUANTISED coded-region bands of the four channels -> the BYR4 mosaic the reference decodes."""
    planes = pu.inverse_pyramid(ol.oracle(), bands, divisors, prescale, nchan=4)
    return mosaic_from_rows(rows16u(planes), phase, restore)


UNIT4 = [[[1, 1, 1, 1]] * 3] * 4


def synthetic_mosaic(rng, w, h, kind, phase=0):
    """(h, w) uint16 Bayer mosaic: "natural" (sampled from a smooth RGB frame), "random", "extreme" (0 / 65535),
    "constant"."""
    if kind == "natural":
        return pu.mosaic_from_rg48(pu.synthetic_rg48(rng, w, h, "natural"), phase)
    if kind == "extreme":
        return np.where(rng.integers(0, 2, (h, w)) == 0, 0, 65535).astype(np.uint16)
    if kind == "constant":
        return np.full((h, w), 0x8120, np.uint16)
    return rng.integers(0, 65536, (h, w)).astype(np.uint16)


def ref_encode_byr4(ref_lib, mosaic, phase, preset=1, quality=4):
    """The reference's EncodeSample on a BYR4 mosaic (plane dimensions and a doubled pitch, EncoderSDK/SampleEncoder.cpp:494);
    preset 1: curve already applied (samples >> 4), 0: the encoder applies its log-90 curve.  Returns pu.ref_encode_frame's
    (bands, divisors, prescale, sample)."""
    h, w = mosaic.shape
    ref_lib.ref_set_bayer_format(phase)
    ref_lib.ref_set_bayer_curve_preset(preset)
    try:
        two = np.ascontiguousarray(mosaic).reshape(h // 2, 2 * w)
        return pu.ref_encode_frame(ref_lib, two.view(np.uint8), w // 2, h // 2, pu.COLOR_FORMAT_BYR4, 1, 4, quality)
    finally:
        ref_lib.ref_set_bayer_curve_preset(1)
        ref_lib.ref_set_bayer_format(-1)


def ref_encode_byr5(ref_lib, packed, pw, ph, phase, quality=4):
    return bu.ref_encode(ref_lib, packed, pw, ph, phase, quality)


def _ref_decode_byr4_once(sample, w, h, phase, preset):
    out = np.zeros((h, 2 * w), np.uint8)
    dims, quant, state = np.zeros(36, np.int32), np.zeros(48, np.int32), np.zeros(3, np.int32)
    cap = w * h * 16
    b = np.zeros(cap, np.int16)
    table = np.zeros(16384, np.uint16)
    sample = np.ascontiguousarray(sample)
    vp = C.c_void_p
    rc = load_ref_bayer().ref_decode_bayer_bands(vp(sample.ctypes.data), C.c_int64(sample.size), w, h, DECODED_FORMAT_BYR4, 4, phase, preset,
                                                 vp(out.ctypes.data), 2 * w, vp(dims.ctypes.data), vp(quant.ctypes.data),
                                                 vp(b.ctypes.data), C.c_int64(cap), vp(state.ctypes.data), vp(table.ctypes.data))
    assert rc == 0, f"reference decode failed ({rc})"
    bands, pos = {}, 0
    for c in range(4):
        for k in range(3):
            bw, bh = int(dims[(c * 3 + k) * 3]), int(dims[(c * 3 + k) * 3 + 1])
            for bi in range(4):
                bands[(c, k + 1, pu.BAND_NAMES[bi])] = b[pos:pos + bw * bh].reshape(bh, bw).copy()
                pos += bw * bh
    return out.view(np.uint16), bands, (int(state[0]), int(state[1])), table if state[2] else None


def ref_decode_byr4(sample, w, h, phase, preset):
    """The reference decoder on a Bayer sample -> DECODED_FORMAT_BYR4 at full resolution, with the Bayer phase and curve
    mode set on the decoder (the sample itself does not carry them).  Returns (mosaic (h, w) uint16, dequantised bands the
    decoder held, (phase, preset) the decoder held after the decode, its restore table or None).  Repeated until two
    consecutive decodes agree, as parity_util.ref_decode_sample_raw (the reference's threaded decoder races on a busy host)."""
    prev = None
    for _ in range(8):
        cur = _ref_decode_byr4_once(sample, w, h, phase, preset)
        if prev is not None and np.array_equal(prev[0], cur[0]) and all(np.array_equal(prev[1][k], cur[1][k]) for k in cur[1]):
            return cur
        prev = cur
    return prev
