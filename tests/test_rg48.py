"""RG48 (BASELINE config 4: packed 16-bit RGB -> RGB 4:4:4 at 12 bits): CPU gate against the reference's real
encoder, GPU parity of the forward path through the C ABI."""
import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")


@needs_ref
@pytest.mark.parametrize("size", [(256, 64), (640, 96)])
def test_oracle_rg48_pyramid_matches_reference_encoder(pkg, size):
    w, h = size
    ref_lib = ol.load_ref()
    frame = pu.qbist_rg48(ref_lib, w, h, 1)
    bands_ref, div, prescale, _ = pu.ref_encode_frame(ref_lib, frame.view(np.uint8), w, h, pu.COLOR_FORMAT_RG48, 1, 3, 4)
    assert prescale[0] == [0, 2, 2]
    assert div[0] == [[1, 96, 96, 144], [1, 24, 24, 12], [1, 24, 24, 12]]        # BASELINE.md, 12-bit FS1, channel 0
    assert div[1] == [[1, 192, 192, 288], [1, 24, 24, 12], [1, 24, 24, 12]]
    q = pkg.quant_for_quality(pkg.FrameDesc(w, h, pkg.PIXEL_RG48), 4)
    assert q.table(3) == div and list(q.prescale) == prescale[0]
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_rg48(frame), div, tuple(prescale[0]))
    for key, want in bands_ref.items():
        assert np.array_equal(pyr[key], want), f"band {key}"


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(256, 64), (288, 48), (640, 96), (1920, 1080)])
@pytest.mark.parametrize("kind", ["natural", "random", "extreme"])
def test_forward_rg48_vs_oracle(pkg, size, kind):
    w, h = size
    rng = np.random.default_rng(w + h)
    frame = fm.synthetic_rg48(rng, w, h, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        coded = codec.forward_host([frame, frame], quant)
        assert np.array_equal(coded[0], coded[1])
        got = codec.unpack_coded(coded[0])
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_rg48(frame), quant.table(3), tuple(quant.prescale))
    for key, want in pyr.items():
        if key[2] == "LL" and key[1] != 3:
            continue
        if not np.array_equal(got[key], want):
            bad = np.argwhere(got[key] != want)
            raise AssertionError(f"band {key}: {len(bad)} mismatches, first {bad[:4].tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(256, 64), (640, 96)])
def test_inverse_rg48_planar16_vs_oracle(pkg, size):
    """12-bit 4:4:4 decode path: descale at levels 3 and 2, divisors > 255 (generic dequant path)."""
    w, h = size
    rng = np.random.default_rng(w)
    frame = fm.synthetic_rg48(rng, w, h, "natural")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    pyr = pu.forward_pyramid_planes(orc, fm.unpack_rg48(frame), quant.table(3), tuple(quant.prescale))
    coded_bands = {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}
    want = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        out = np.zeros((3 * h, w), np.int16)
        codec.inverse_host([codec.pack_coded(coded_bands)], quant, pkg.PIXEL_PLANAR16, [out])
    for c in range(3):
        got = out[c * h:(c + 1) * h]
        assert np.array_equal(got, want[c]), f"channel {c}: {np.argwhere(got != want[c])[:4].tolist()}"
    # round trip fidelity at 12 bits (G plane)
    g12 = fm.unpack_rg48(frame)[0].astype(np.float64)
    mse = np.mean((out[0:h].astype(np.float64) - g12) ** 2)
    assert 10 * np.log10(4095.0 ** 2 / mse) > 45.0
