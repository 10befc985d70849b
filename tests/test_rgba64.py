"""16-bit RGBA sources (B64A, RG64) as RGB 4:4:4 or RGBA 4:4:4:4, and the B64A output of an RGBA sample: the layout and
quantisation of the C ABI, and the unpack / alpha rules of rgba_util pinned to the reference's real encoder and decoder
(oracle/_ref; skipped when it is absent)."""
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
import rgba_util as ru
from gpu_fixtures import pkg  # noqa: F401

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")
FORMATS = ("B64A", "RG64")


def _desc(pkg, w, h, name, alpha):
    return pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + name), pkg.FRAME_ALPHA if alpha else 0)


@pytest.mark.parametrize("name", FORMATS)
@pytest.mark.parametrize("alpha", [False, True])
def test_layout_rgba64(pkg, name, alpha):
    lay = pkg.layout_for(_desc(pkg, 328, 48, name, alpha))
    assert lay.num_channels == (4 if alpha else 3) and lay.precision == 12
    assert lay.frame_pitch == 328 * 8 and lay.frame_bytes == 328 * 8 * 48
    for c in range(lay.num_channels):
        assert (lay.band[c][0][1].width, lay.band[c][0][1].height) == (164, 24)
    rg = pkg.layout_for(pkg.FrameDesc(328, 48, pkg.PIXEL_RG48))
    assert lay.coded_bytes == rg.coded_bytes * lay.num_channels // 3
    with pytest.raises(pkg.CfbError):
        pkg.layout_for(_desc(pkg, 324, 48, name, alpha))          # 4:4:4 widths are multiples of 8


@pytest.mark.parametrize("fmt", ["YUYV", "RG48", "BYR4", "RG30", "V210", "PLANAR16"])
def test_alpha_flag_ignored_by_other_formats(pkg, fmt):
    w, h = 480, 96
    f = getattr(pkg, "PIXEL_" + fmt)
    plain, flagged = pkg.layout_for(pkg.FrameDesc(w, h, f)), pkg.layout_for(pkg.FrameDesc(w, h, f, pkg.FRAME_ALPHA))
    assert bytes(plain) == bytes(flagged)
    qa, qb = pkg.quant_for_quality(pkg.FrameDesc(w, h, f), 4), pkg.quant_for_quality(pkg.FrameDesc(w, h, f, pkg.FRAME_ALPHA), 4)
    assert bytes(qa) == bytes(qb)


def test_positional_frame_desc(pkg):
    d = pkg.FrameDesc(256, 64, pkg.PIXEL_RG48)
    assert (d.width, d.height, d.pixel_format, d.flags) == (256, 64, pkg.PIXEL_RG48, 0)


def test_alpha_curve_edges():
    curve = lambda a: ((a * 223 + 128) >> 8) + 256
    raw = np.array([0, 15, 16, 31, 4096, 65503, 65504, 65519, 65520, 65535], np.uint16)
    want = [0, 0, 257, 257, curve(256), curve(4093), curve(4094), curve(4094), 4095, 4095]
    assert fm.alpha_curve(raw).tolist() == want and want[2] == curve(1)


@needs_ref
@pytest.mark.parametrize("name", FORMATS)
@pytest.mark.parametrize("alpha", [False, True])
def test_quant_matches_reference_encoder(pkg, name, alpha):
    """Per-channel divisors and prescale, every fixed quality: B64A reaches the quantiser as COLOR_FORMAT_B64A (30), below
    COLOR_FORMAT_BAYER, so its channels 1-3 take the chroma table; RG64 (121) takes the luma table for every channel."""
    w, h = 256, 64
    frame = fm.synthetic_rgba64(np.random.default_rng(5), w, h, "natural", name)
    ref_lib = ol.load_ref()
    for quality in range(1, 7):
        _, div, prescale, _ = ru.ref_encode(ref_lib, frame, w, h, name, alpha, quality)
        q = pkg.quant_for_quality(_desc(pkg, w, h, name, alpha), quality)
        assert q.table(4 if alpha else 3) == div, quality
        assert list(q.prescale) == prescale == [0, 2, 2]


@needs_ref
@pytest.mark.parametrize("size", [(256, 64), (328, 48), (640, 96)])
@pytest.mark.parametrize("name", FORMATS)
@pytest.mark.parametrize("alpha", [False, True])
def test_oracle_pyramid_matches_reference_encoder(size, name, alpha):
    w, h = size
    frame = fm.synthetic_rgba64(np.random.default_rng(w + h), w, h, "natural", name)
    planes = fm.unpack_rgba64(frame, name, alpha)
    if alpha:       # the frame exercises both ends of the curve and the values it keeps
        a = planes[3]
        assert (a == 0).any() and (a == 257).any() and (a == 4095).any() and (a == ((4094 * 223 + 128) >> 8) + 256).any()
    bands_ref, div, prescale, _ = ru.ref_encode(ol.load_ref(), frame, w, h, name, alpha)
    pyr = pu.forward_pyramid_planes(ol.oracle(), planes, div, tuple(prescale))
    assert len(bands_ref) == 12 * len(planes)
    for key, want in bands_ref.items():
        assert np.array_equal(pyr[key], want), f"band {key}"


@needs_ref
@pytest.mark.skipif((os.cpu_count() or 1) > 8, reason="the reference's active-metadata output path sizes its row workers by "
                    "the online CPU count and, with many of them, returns rows that its own transform has not finished")
@pytest.mark.parametrize("size", [(640, 96), (328, 48), (256, 64), (200, 48), (1016, 64)])
@pytest.mark.parametrize("kind", ["natural", "extreme"])
def test_oracle_b64a_alpha_matches_reference_decoder(size, kind):
    """B64A and RG48 frames of an RGBA 4:4:4:4 sample.  The widths put band columns in the 8-column loops, their tails and
    the right border column; 0/65535 noise separates the 12-bit limit of the ...ToRow16u loop from its scalar saturation."""
    w, h = size
    ref_lib, orc = ol.load_ref(), ol.oracle()
    frame = fm.synthetic_rgba64(np.random.default_rng(w + len(kind)), w, h, kind, "B64A")
    _, _, prescale, sample = ru.ref_encode(ref_lib, frame, w, h, "B64A", True)
    out, bands = ru.ref_decode_fresh(sample, w, h, fm.OUTPUTS["B64A"].decoded_format, 4, w * 8, decodes=5)
    planes = pu.inverse_pyramid(orc, bands, [[[1] * 4] * 3] * 4, tuple(prescale), nchan=4)
    got = out.view(np.uint16).reshape(h, 4 * w)
    want = fm.pack_b64a_alpha(planes)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5].tolist()
    alpha = got[:, 0::4]
    assert (alpha == 0).any() and (alpha == 65535).any() and ((alpha > 0) & (alpha < 65535)).any()
    if kind == "extreme":
        assert (got[:, 1::4] == 0xFFF0).any() and (got[:, 1::4] == 65535).any()
    out48, bands48 = ru.ref_decode_fresh(sample, w, h, fm.OUTPUTS["RG48"].decoded_format, 4, w * 6)
    for key in bands:
        assert np.array_equal(bands48[key], bands[key]), key
    assert np.array_equal(out48.view(np.uint16).reshape(h, 3 * w), fm.pack_rg48(planes[:3]))
