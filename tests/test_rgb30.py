"""10-bit packed RGB sources (RG30, AB10, AR10, R210, DPX0): the reference transforms them directly
(wavelet.c:3597 TransformForwardSpatialRGB30).  CPU: the oracle's planar pyramid on G, R, B << 2 reproduces every band of
the reference's EncodeSample for each layout.  GPU: CUDA forward (field extraction fused into the load) vs the oracle."""
import importlib

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")
NAMES = sorted(fm.RGB30_FORMATS)


def _rgb(rng, w, h, kind):
    if kind == "random":
        return [rng.integers(0, 1024, (h, w)).astype(np.uint32) for _ in range(3)]
    f = fm.synthetic_rg48(rng, w, h, "natural").reshape(h, w, 3)
    return [(f[:, :, i] >> 6).astype(np.uint32) for i in range(3)]


@needs_ref
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("size,quality", [((512, 128), 4), ((208, 56), 2)])
def test_oracle_rgb30_matches_reference_encoder(name, size, quality):
    w, h = size
    ref_lib = ol.load_ref()
    f = pu.qbist_rg48(ref_lib, w, h).reshape(h, w, 3)
    r, g, b = [(f[:, :, i] >> 6).astype(np.uint32) for i in range(3)]
    words = fm.pack_rgb30(name, r, g, b)
    bands, div, prescale, _ = pu.ref_encode_frame(ref_lib, words.view(np.uint8).reshape(h, w * 4), w, h,
                                                  fm.RGB30_FORMATS[name][0], 1, 3, quality)
    assert prescale[0] == [0, 2, 2]
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.rgb30_planes(r, g, b), div, tuple(prescale[0]))
    for key, want in bands.items():
        if not (key[2] == "LL" and key[1] != 3):
            assert np.array_equal(pyr[key], want), f"{name} band {key}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("size,kind", [((256, 64), "natural"), ((208, 56), "random"), ((1928, 120), "natural"), ((3840, 2160), "random")])
def test_cuda_rgb30_vs_oracle(name, size, kind):
    pkg = importlib.import_module("cineform-sdk_b200")
    w, h = size
    rng = np.random.default_rng(w + h)
    r, g, b = _rgb(rng, w, h, kind)
    words = fm.pack_rgb30(name, r, g, b)
    desc = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + name))
    quant = pkg.quant_for_quality(desc, 4)
    rg48_quant = pkg.quant_for_quality(pkg.FrameDesc((w + 7) // 8 * 8, h, pkg.PIXEL_RG48), 4)
    assert quant.table(3) == rg48_quant.table(3)            # same schedule as RG48 (ChromaFullRes, 12 bit)
    want = pu.forward_pyramid_planes(ol.oracle(), fm.rgb30_planes(r, g, b), quant.table(3), tuple(quant.prescale), quant.midpoint_prequant)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        codec.forward_host([words], quant, [coded])
        got = codec.unpack_coded(coded)
        for key in sorted(want):
            if key[2] == "LL" and key[1] != 3:
                continue
            if not np.array_equal(got[key], want[key]):
                bad = np.argwhere(got[key] != want[key])
                raise AssertionError(f"{name} band {key}: {bad.shape[0]} mismatches, first {bad[:4].tolist()}")
        planes = pu.inverse_pyramid(ol.oracle(), {k: v for k, v in want.items() if not (k[2] == "LL" and k[1] != 3)},
                                    quant.table(3), tuple(quant.prescale))
        out = np.zeros((3 * h, w), np.int16)
        codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [out])
        for c in range(3):
            assert np.array_equal(out[c * h:(c + 1) * h], planes[c]), f"{name} decoded plane {c}"
