"""BYR4 (BASELINE config 5: 16-bit Bayer -> four half-resolution 12-bit planes): CPU gate against the reference's
real encoder (curve applied), GPU parity of the forward path and the planar inverse."""
import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")


@needs_ref
@pytest.mark.parametrize("fmt", [0, 1, 2, 3])
def test_oracle_byr4_pyramid_matches_reference_encoder(pkg, fmt):
    w, h = 512, 128                      # Bayer dimensions; planes are 256 x 64
    ref_lib = ol.load_ref()
    bayer = fm.mosaic_from_rg48(pu.qbist_rg48(ref_lib, w, h, 1), fmt)
    ref_lib.ref_set_bayer_format(fmt)
    try:
        # the SDK passes the plane dimensions and a doubled pitch (EncoderSDK/SampleEncoder.cpp:268-269, :494)
        two_lines_per_row = np.ascontiguousarray(bayer).reshape(h // 2, 2 * w)          # pitch = 2 Bayer lines
        bands_ref, div, prescale, _ = pu.ref_encode_frame(ref_lib, two_lines_per_row.view(np.uint8), w // 2, h // 2,
                                                          pu.COLOR_FORMAT_BYR4, 1, 4, 4)
    finally:
        ref_lib.ref_set_bayer_format(-1)
    assert prescale[0] == [0, 2, 2]
    q = pkg.quant_for_quality(pkg.FrameDesc(w, h, pkg.PIXEL_BYR4), 4)
    assert q.table(4) == div
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_byr4(bayer, fmt), div, tuple(prescale[0]))
    for key, want in bands_ref.items():
        assert np.array_equal(pyr[key], want), f"band {key}"


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(512, 128), (1152, 192), (3840, 2160)])
@pytest.mark.parametrize("fmt", [0, 1, 2, 3])
def test_forward_byr4_vs_oracle(pkg, size, fmt):
    w, h = size
    if (w, h) == (3840, 2160) and fmt not in (0, 2):
        pytest.skip("large size covered by two phases")
    rng = np.random.default_rng(w + fmt)
    bayer = rng.integers(0, 65536, (h, w)).astype(np.uint16) if fmt % 2 else fm.mosaic_from_rg48(fm.synthetic_rg48(rng, w, h, "natural"), fmt)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        codec.set_bayer_phase(fmt)
        coded = codec.forward_host([bayer], quant)[0]
        got = codec.unpack_coded(coded)
        pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_byr4(bayer, fmt), quant.table(4), tuple(quant.prescale))
        for key, want in pyr.items():
            if key[2] == "LL" and key[1] != 3:
                continue
            if not np.array_equal(got[key], want):
                bad = np.argwhere(got[key] != want)
                raise AssertionError(f"band {key}: {len(bad)} mismatches, first {bad[:4].tolist()}")
        # planar inverse of the same coefficients == oracle inverse (4 channels)
        coded_bands = {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}
        want_planes = pu.inverse_pyramid(ol.oracle(), coded_bands, quant.table(4), tuple(quant.prescale), nchan=4)
        ph, pw = h // 2, w // 2
        out = np.zeros((4 * ph, w), np.int16)           # planes stacked at the frame's luma pitch (2*w bytes)
        codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [out])
        for c in range(4):
            assert np.array_equal(out[c * ph:(c + 1) * ph, :pw], want_planes[c]), f"inverse channel {c}"


@needs_ref
@pytest.mark.parametrize("fmt", [0, 1, 2, 3])
def test_oracle_byr4_default_curve_matches_reference_encoder(pkg, fmt):
    """BYR4 WITHOUT the curve-applied flag: the reference builds its default encode curve (log base 90, frame.c:5208-5245)
    and maps every sample through it; formats.bayer_log90_curve restates the table."""
    w, h = 512, 128
    ref_lib = ol.load_ref()
    rng = np.random.default_rng(fmt)
    bayer = fm.mosaic_from_rg48(pu.qbist_rg48(ref_lib, w, h, 1), fmt)
    bayer = (bayer.astype(np.uint32) | rng.integers(0, 16, bayer.shape).astype(np.uint32)).astype(np.uint16)   # use the low bits too
    ref_lib.ref_set_bayer_format(fmt)
    ref_lib.ref_set_bayer_curve_preset(0)
    try:
        two_lines_per_row = np.ascontiguousarray(bayer).reshape(h // 2, 2 * w)
        bands_ref, div, prescale, _ = pu.ref_encode_frame(ref_lib, two_lines_per_row.view(np.uint8), w // 2, h // 2,
                                                          pu.COLOR_FORMAT_BYR4, 1, 4, 4)
    finally:
        ref_lib.ref_set_bayer_curve_preset(1)
        ref_lib.ref_set_bayer_format(-1)
    curve = fm.bayer_log90_curve()
    assert curve[0] == 0 and curve[-1] <= 4095 and np.all(np.diff(curve.astype(np.int32)) >= 0)
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_byr4(bayer, fmt, curve=curve), div, tuple(prescale[0]))
    for key, want in bands_ref.items():
        assert np.array_equal(pyr[key], want), f"band {key}"


@pytest.mark.gpu
@pytest.mark.parametrize("size,fmt", [((512, 128), 0), ((1152, 192), 1), ((512, 128), 2), ((3840, 2160), 3)])
def test_forward_byr4_with_encode_curve(pkg, size, fmt):
    """cfb_codec_set_bayer_curve: the table lookup fused into the load == oracle planes built with the same table;
    clearing the curve restores the curve-applied path."""
    w, h = size
    rng = np.random.default_rng(w + 10 * fmt)
    bayer = rng.integers(0, 65536, (h, w)).astype(np.uint16)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    curve = fm.bayer_log90_curve()
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        codec.set_bayer_phase(fmt)
        for cv in (curve, None):
            codec.set_bayer_curve(cv)
            got = codec.unpack_coded(codec.forward_host([bayer], quant)[0])
            pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_byr4(bayer, fmt, curve=cv), quant.table(4), tuple(quant.prescale))
            for key, want in pyr.items():
                if key[2] == "LL" and key[1] != 3:
                    continue
                assert np.array_equal(got[key], want), f"curve {'on' if cv is not None else 'off'} band {key}"
