"""BYR5 (12-bit packed Bayer -> the four half-resolution 12-bit planes of BYR4): the restated unpack of formats.byr5_planes and the
oracle pyramid against the reference's real encoder, and the layout and quantisation of the C ABI."""
import numpy as np
import pytest

import formats as fm
import byr4_out_util as b4
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")


def test_layout_byr5(pkg):
    w, h = 720, 96                                  # Bayer samples; planes 360 x 48
    lay = pkg.layout_for(pkg.FrameDesc(w, h, pkg.PIXEL_BYR5))
    assert lay.num_channels == 4 and lay.precision == 12
    assert lay.frame_pitch == 3 * w and lay.frame_bytes == 3 * w * (h // 2)
    by4 = pkg.layout_for(pkg.FrameDesc(w, h, pkg.PIXEL_BYR4))
    assert lay.coded_bytes == by4.coded_bytes and lay.total_bytes == by4.total_bytes
    for bad in (712, 200):                          # Bayer widths are multiples of 16
        with pytest.raises(pkg.CfbError):
            pkg.layout_for(pkg.FrameDesc(bad, h, pkg.PIXEL_BYR5))


def test_pack_roundtrip():
    rng = np.random.default_rng(5)
    comps = fm.byr5_random_components(rng, 104, 3)
    frame = fm.byr5_pack(comps, pitch=6 * 104 + 16)
    assert np.array_equal(fm.byr5_components(frame, 104), comps)
    # byte layout: high bytes of the first sample, then the nibble pair of samples 0 and 1
    assert frame[0, 0] == comps[0, 0, 0] >> 4
    assert frame[0, 4 * 104] == (comps[0, 0, 0] & 15) | ((comps[0, 0, 1] & 15) << 4)


@needs_ref
@pytest.mark.parametrize("phase", [0, 1, 2, 3])
@pytest.mark.parametrize("size,kind", [((512, 128), "random"), ((208, 96), "extreme"), ((720, 100), "random"),
                                       ((1040, 112), "random")])
def test_oracle_byr5_pyramid_matches_reference_encoder(pkg, size, kind, phase):
    """Every band of the reference's EncodeSample on a BYR5 frame equals the oracle pyramid of the restated planes.
    720 x 100: 50 plane rows, which the encoder pads to 56 by repeating the last packed row; 208 / 720 / 1040 wide: plane
    widths that are not multiples of 64 (nor of 32 for 208 and 720)."""
    w, h = size
    pw, ph = w // 2, h // 2
    rng = np.random.default_rng(w * 7 + h + phase)
    frame = fm.byr5_pack(fm.byr5_random_components(rng, pw, ph, kind))
    bands_ref, div, prescale, _ = b4.ref_encode_byr5(ol.load_ref(), frame, pw, ph, phase)
    assert prescale[0] == [0, 2, 2]
    coded_h = bands_ref[(0, 1, "LL")].shape[0] * 2
    assert coded_h == (ph + 7) // 8 * 8
    q = pkg.quant_for_quality(pkg.FrameDesc(w, coded_h * 2, pkg.PIXEL_BYR5), 4)
    assert q.table(4) == div
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.byr5_planes(frame, pw, phase, height=coded_h), div, tuple(prescale[0]))
    for key, want in bands_ref.items():
        assert np.array_equal(pyr[key], want), f"band {key}"


@needs_ref
@pytest.mark.parametrize("quality", [1, 2, 3, 4, 5, 6])
def test_quant_schedule_byr5_matches_reference(pkg, quality):
    """cfb_quant_for_source on BYR5 equals the divisors and prescales the reference encoder used (precision 12,
    `3 << 25` in the fixed quality, chroma at full resolution); they are those of BYR4."""
    w, h = 512, 128
    rng = np.random.default_rng(quality)
    frame = fm.byr5_pack(fm.byr5_random_components(rng, w // 2, h // 2))
    _, div, prescale, _ = b4.ref_encode_byr5(ol.load_ref(), frame, w // 2, h // 2, 0, quality=quality)
    q = pkg.quant_for_quality(pkg.FrameDesc(w, h, pkg.PIXEL_BYR5), quality)
    assert q.table(4) == div
    assert list(q.prescale) == prescale[0]
    assert q.table(4) == pkg.quant_for_quality(pkg.FrameDesc(w, h, pkg.PIXEL_BYR4), quality).table(4)
    if quality == 4:                                # ChromaFullRes: channel 1 shares the luma divisors
        assert div[0][0] == div[1][0] == [1, 96, 96, 144]
