"""10-bit packed RGB outputs (RG30 / AB10 / AR10 / R210 / DPX0) of the final inverse level for RGB 4:4:4 codecs on the GPU
(SURVEY 8f rank 2).  The rule (formats.pack_rgb30_output) is pinned to the reference's decoder in test_output16.py."""
import hashlib

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

FORMATS = {"RG30": "PIXEL_RG30", "AB10": "PIXEL_AB10", "AR10": "PIXEL_AR10", "R210": "PIXEL_R210", "DPX0": "PIXEL_DPX0"}


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(256, 64), (328, 48), (200, 48), (640, 96), (1920, 1080)])
@pytest.mark.parametrize("kind", ["natural", "extreme"])
def test_gpu_rgb30_outputs_vs_oracle(pkg, size, kind):
    w, h = size
    rng = np.random.default_rng(w + h)
    frame = fm.synthetic_rg48(rng, w, h, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    pyr = pu.forward_pyramid_planes(orc, fm.unpack_rg48(frame), quant.table(3), tuple(quant.prescale))
    coded_bands = {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}
    planes = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        coded = codec.pack_coded(coded_bands)
        for name, attr in FORMATS.items():
            want = fm.pack_rgb30_output(name, planes)
            outs = [np.zeros((h, w), np.uint32) for _ in range(2)]
            codec.inverse_host([coded, coded], quant, getattr(pkg, attr), outs)
            assert np.array_equal(outs[0], want), (name, np.argwhere(outs[0] != want)[:5].tolist())
            assert np.array_equal(outs[1], want), name
        # a padded output pitch
        wide = np.zeros((h, w + 4), np.uint32)
        codec.inverse_host([coded], quant, pkg.PIXEL_DPX0, [wide])
        assert np.array_equal(wide[:, :w], fm.pack_rgb30_output("DPX0", planes)) and not wide[:, w:].any()


@pytest.mark.gpu
def test_gpu_rgb30_round_trip_of_a_10bit_source(pkg):
    """Encode an R210 frame, decode to R210: the 10-bit samples come back within the quantiser's error, and exactly where
    nothing was quantised away (a flat frame)."""
    w, h = 640, 96
    r = np.full((h, w), 300, np.uint32); g = np.full((h, w), 512, np.uint32); b = np.full((h, w), 700, np.uint32)
    frame = fm.pack_rgb30("R210", r, g, b)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_R210)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.forward_host([frame.view(np.uint8).reshape(h, 4 * w)], quant)[0]
        out = np.zeros((h, w), np.uint32)
        codec.inverse_host([coded], quant, pkg.PIXEL_R210, [out])
    assert np.array_equal(out, frame)


@pytest.mark.gpu
def test_gpu_rgb30_output_needs_a_444_codec(pkg):
    desc = pkg.FrameDesc(256, 64, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        with pytest.raises(pkg.CfbError):
            codec.inverse_host([coded], quant, pkg.PIXEL_RG30, [np.zeros((64, 256), np.uint32)])


@pytest.mark.gpu
def test_gpu_rgb30_vs_reference_decoder(pkg):
    """The bands the reference decoder held for a Qbist RG48 sample and the hashes of the five 10-bit frames it wrote
    (golden/)."""
    w, h = 640, 96
    with pkg.Context(0) as ctx, pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_RG48), 1) as codec:
        for name, attr in FORMATS.items():
            bands, prescale, want = pu.reference_decoded("rg48", name)
            unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
            out = np.zeros((h, w), np.uint32)
            codec.inverse_host([codec.pack_coded(bands)], unit, getattr(pkg, attr), [out])
            assert hashlib.sha256(out.tobytes()).hexdigest() == want, name
