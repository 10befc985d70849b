"""B64A output of the final inverse level for RGB 4:4:4 codecs (SURVEY 8f rank 2: "decode to RG48 / B64A") on the GPU.
The rule (formats.pack_b64a) is pinned to the reference's decoder in test_output16.py; here the CUDA path is compared
with the oracle and, where oracle/_ref travelled, with the reference decoder's own frame."""
import hashlib

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(256, 64), (328, 48), (200, 48), (640, 96), (720, 480), (1920, 1080)])
@pytest.mark.parametrize("kind", ["natural", "extreme"])
def test_gpu_b64a_output_vs_oracle(pkg, size, kind):
    w, h = size
    rng = np.random.default_rng(w + h)
    frame = fm.synthetic_rg48(rng, w, h, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    pyr = pu.forward_pyramid_planes(orc, fm.unpack_rg48(frame), quant.table(3), tuple(quant.prescale))
    coded_bands = {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}
    planes = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale))
    want = fm.pack_b64a(planes)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        coded = codec.pack_coded(coded_bands)
        outs = [np.zeros((h, 4 * w), np.uint16) for _ in range(2)]
        codec.inverse_host([coded, coded], quant, pkg.PIXEL_B64A, outs)
        assert np.array_equal(outs[0], want), np.argwhere(outs[0] != want)[:5].tolist()
        assert np.array_equal(outs[1], want)
        # the RG48 output of the same codec afterwards: the two stagings do not disturb each other
        rg = np.zeros((h, 3 * w), np.uint16)
        codec.inverse_host([coded], quant, pkg.PIXEL_RG48, [rg])
        assert np.array_equal(rg, fm.pack_rg48(planes))
        # a padded output pitch
        wide = np.zeros((h, 4 * w + 8), np.uint16)
        codec.inverse_host([coded], quant, pkg.PIXEL_B64A, [wide])
        assert np.array_equal(wide[:, :4 * w], want) and not wide[:, 4 * w:].any()


@pytest.mark.gpu
def test_gpu_b64a_needs_a_444_codec(pkg):
    desc = pkg.FrameDesc(256, 64, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        with pytest.raises(pkg.CfbError):
            codec.inverse_host([coded], quant, pkg.PIXEL_B64A, [np.zeros((64, 4 * 256), np.uint16)])


@pytest.mark.gpu
def test_gpu_b64a_vs_reference_decoder(pkg):
    """The bands the reference decoder held for a Qbist RG48 sample and the hash of the B64A frame it wrote (golden/)."""
    w, h = 640, 96
    bands, prescale, want = pu.reference_decoded("rg48", "B64A")
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_RG48), 1) as codec:
        out = np.zeros((h, 4 * w), np.uint16)
        codec.inverse_host([codec.pack_coded(bands)], unit, pkg.PIXEL_B64A, [out])
    assert hashlib.sha256(out.tobytes()).hexdigest() == want
