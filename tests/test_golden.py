"""Oracle vs the committed golden vectors (generated from the reference itself by
tests/golden/make_golden.py).  Runs on CPU, needs neither /root/reference nor oracle/_ref."""
import glob
import os

import numpy as np
import pytest

import oracle_lib as ol
import parity_util as pu

_ALL = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "*.npz")))
GOLDEN = [p for p in _ALL if os.path.basename(p).startswith("qbist_")]                 # progressive
GOLDEN_FIELDS = [p for p in _ALL if os.path.basename(p).startswith("interlaced_")]     # interlaced sources


def load_golden(path):
    z = np.load(path)
    bands = {}
    for k in z.files:
        if k.startswith("b_"):
            _, c, lvl, name = k.split("_")
            bands[(int(c), int(lvl), name)] = z[k]
    return z["frame"], z["divisors"].tolist(), tuple(int(v) for v in z["prescale"]), int(z["quality"]), bands


def test_golden_present():
    assert len(GOLDEN) >= 3


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_reproduces_golden(path):
    frame, div, prescale, quality, bands = load_golden(path)
    pyr = pu.forward_pyramid_422(ol.oracle(), frame, div, prescale, fmt=0)
    for key, want in bands.items():
        assert np.array_equal(pyr[key], want), f"band {key}"


def load_golden_decoder_side(path):
    z = np.load(path)
    bands = {}
    for k in z.files:
        if k.startswith("d_"):
            _, c, lvl, name = k.split("_")
            bands[(int(c), int(lvl), name)] = z[k]
    return bands, z["decoded_yuy2"]


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_inverse_inside_reference_decoder_envelope(path):
    """Oracle inverse pyramid applied to the bands the reference's decoder held, against the frame the
    reference's DecodeSample produced.  The reference's 8-bit reduction is dithered with rand(), so every
    byte must be one of the two values the oracle's 10-bit reconstruction allows."""
    frame, div, prescale, quality, _ = load_golden(path)
    bands, dec = load_golden_decoder_side(path)
    planes = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, prescale)
    a, b = pu.yuyv_envelope(planes)
    ok = (dec == a) | (dec == b)
    assert ok.all(), f"{(~ok).sum()} bytes outside the dither envelope"
    assert pu.psnr(dec[:, 0::2], frame[:, 0::2]) > 45.0


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_reduced_resolution_decode(path):
    """Half / quarter resolution decode (decoder.c:26078, :11818): the oracle's partial inverse pyramid must give the
    reference decoder's own lowpass images LL1 / LL2 bit for bit, its half-resolution packing must equal the frame
    CFHD_DecodeSample returned at CFHD_DECODED_RESOLUTION_HALF byte for byte, and the quarter-resolution packing
    (CopyQuarterRowToBuffer, temporal.c:11362) must stay within the rounding of the SDK's quarter-resolution output,
    which the public API renders through its 16-bit active-metadata path and re-dithers."""
    z = np.load(path)
    _, _, prescale, _, _ = load_golden(path)
    bands, _ = load_golden_decoder_side(path)
    for stop, name, unsigned in ((1, "half", False), (2, "quarter", True)):
        planes = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, prescale, stop_level=stop)
        for c in range(3):
            assert np.array_equal(planes[c], z[f"r_{c}_{stop}_LL"]), f"LL{stop} channel {c}"
        got = pu.lowpass_to_422(planes, unsigned)
        want = z[f"decoded_{name}_yuy2"]
        assert got.shape == want.shape
        if name == "half":
            assert np.array_equal(got, want)
        else:
            d = np.abs(got.astype(np.int32) - want.astype(np.int32))
            assert (d > 2).mean() < 2e-3 and d.max() <= 16 and d.mean() < 0.6, (d.max(), d.mean())


def test_interlaced_golden_present():
    assert len(GOLDEN_FIELDS) >= 2


@pytest.mark.parametrize("path", GOLDEN_FIELDS, ids=[os.path.basename(p) for p in GOLDEN_FIELDS])
def test_oracle_reproduces_interlaced_golden(path):
    """Field transform at level 1 (TransformForwardFrameYUV, wavelet.c:6076): every band the reference's EncodeSample
    produced for an interlaced source, the HL band in its difference-coded form."""
    frame, div, prescale, quality, bands = load_golden(path)
    assert div[0][0][1] != div[0][0][2]          # the interlaced schedule (LH * 3/2, HL * 2/3) was in force
    pyr = pu.forward_pyramid_422(ol.oracle(), frame, div, prescale, fmt=0, interlaced=True)
    for key, want in bands.items():
        assert np.array_equal(pyr[key], want), f"band {key}"


@pytest.mark.parametrize("path", GOLDEN_FIELDS, ids=[os.path.basename(p) for p in GOLDEN_FIELDS])
def test_oracle_interlaced_inverse_inside_reference_decoder_envelope(path):
    frame, div, prescale, quality, enc_bands = load_golden(path)
    bands, dec = load_golden_decoder_side(path)
    for c in range(3):
        # the decoder integrates HL after dequantising it (decoder.c:20822): its band is cumsum(coded) * divisor
        want = (np.cumsum(enc_bands[(c, 1, "HL")].astype(np.int64), axis=1) * div[c][0][2]).astype(np.int16)
        assert np.array_equal(bands[(c, 1, "HL")], want)
        hl = bands[(c, 1, "HL")].astype(np.int32)
        hl[:, 1:] -= hl[:, :-1].copy()
        bands[(c, 1, "HL")] = hl.astype(np.int16)        # back to the coded (differenced) form inverse_pyramid expects
    planes = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, prescale, interlaced=True)
    a, b = pu.yuyv_envelope(planes)
    ok = (dec == a) | (dec == b)
    assert ok.all(), f"{(~ok).sum()} bytes outside the dither envelope"
    assert pu.psnr(dec[:, 0::2], frame[:, 0::2]) > 45.0


@pytest.mark.parametrize("path", GOLDEN_FIELDS, ids=[os.path.basename(p) for p in GOLDEN_FIELDS])
def test_integrate_hl_matches_reference_decoder(path):
    """The decoder-side level-1 HL band is integrate_hl of the dequantised encoder band, and the oracle's inverse of the
    decoder's bands as they are (hl_integrated=True, unit divisors) lies inside the dither envelope of its frame.  This
    anchors the GPU tests of the integrated-HL decode mode to the reference."""
    frame, div, prescale, quality, enc_bands = load_golden(path)
    bands, dec = load_golden_decoder_side(path)
    for c in range(3):
        want = pu.integrate_hl(pu.dequantize(enc_bands[(c, 1, "HL")], div[c][0][2]))
        assert want.dtype == np.int16
        assert np.array_equal(bands[(c, 1, "HL")], want), f"channel {c}"
    planes = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, prescale, interlaced=True, hl_integrated=True)
    a, b = pu.yuyv_envelope(planes)
    ok = (dec == a) | (dec == b)
    assert ok.all(), f"{(~ok).sum()} bytes outside the dither envelope"


def test_integrate_hl_wraps_in_int16():
    """`line[x] += line[x-1]` on int16 samples: the running sum wraps modulo 2^16 instead of saturating."""
    hl = np.array([[30000, 30000, -20000, -30000, -30000, 5]], np.int16)
    want = (np.cumsum(hl.astype(np.int64), axis=1) + 32768) % 65536 - 32768
    got = pu.integrate_hl(hl)
    assert got.dtype == np.int16 and np.array_equal(got, want)
