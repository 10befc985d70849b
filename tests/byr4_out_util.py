"""The Bayer checkers for the tests: the oracle's Bayer library (oracle/bayer.mk), the reference's decoder probe
(oracle/ref_probe_bayer.cpp) and the reference encoder's calls on BYR4 and BYR5 frames (oracle/ref_probe.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as ol
import parity_util as pu


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


def ref_decode_byr4(sample, w, h, phase, preset):
    """The reference decoder on a Bayer sample -> DECODED_FORMAT_BYR4 at full resolution, with the Bayer phase and curve
    mode set on the decoder (the sample itself does not carry them), through pu.ref_decode.  Returns (mosaic (h, w) uint16,
    dequantised bands the decoder held, (phase, preset) the decoder held after the decode, its restore table or None)."""
    out, bands, used, table = pu.ref_decode(load_ref_bayer(), sample, w, h, pu.COLOR_FORMAT_BYR4, 4, 2 * w,
                                            bayer=(phase, preset))
    return out.view(np.uint16), bands, used, table


def ref_encode_byr5(ref_lib, frame, pw, ph, phase, quality=4):
    """The reference's EncodeSample on a packed BYR5 frame of ph plane rows (display height ph; the encoder pads the plane
    height to its own multiple).  Returns (bands, divisors, prescale, sample bytes) as pu.ref_encode_frame."""
    ref_lib.ref_set_bayer_format(phase)
    try:
        return pu.ref_encode_frame(ref_lib, np.ascontiguousarray(frame[:, :6 * pw]), pw, ph, pu.COLOR_FORMAT_BYR5, 1, 4, quality)
    finally:
        ref_lib.ref_set_bayer_format(-1)
