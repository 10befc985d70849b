"""Interlaced (field) transform of the 16-bit / 10-bit 4:2:2 sources (YU64, V210): the reference converts them to planes
and runs Codec/filter.c:273 FilterFrameQuant16s, whose LL / LH come out of FilterHorizontalRowQuant16s (midpoint
divisor / 2, spatial.c:5856) -- not the packed 8-bit path's quantiser.  CPU: the oracle's planar field transform is pinned to
the reference's real encoder (progressive = 0); GPU: k_fwd_422_fields<SrcYU64 / SrcV210> through the C ABI against the oracle, then the
inverse back to planes."""
import importlib

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")


def planar_fields_pyramid(orc, planes, div, prescale, midpoint=2):
    """level 1 = planar field transform, levels 2, 3 = the ordinary spatial levels on its LL"""
    out = {}
    for c, plane in enumerate(planes):
        ll, lh, hl, hh = orc.fwd_fields_plane(plane, div[c][0], midpoint)
        out[(c, 1, "LL")], out[(c, 1, "LH")], out[(c, 1, "HL")], out[(c, 1, "HH")] = ll, lh, hl, hh
        for k in (1, 2):
            ll, lh, hl, hh = orc.fwd_level(ll, 1 if prescale[k] == 2 else 0, div[c][k], midpoint)
            out[(c, k + 1, "LL")], out[(c, k + 1, "LH")], out[(c, k + 1, "HL")], out[(c, k + 1, "HH")] = ll, lh, hl, hh
    return out


def make_source(fmt, w, h, rng, kind):
    frame8 = pu.synthetic_yuyv(rng, w, h, kind)
    frame8[1::2] = np.roll(frame8[1::2], 12, axis=1)            # the two fields differ
    if fmt == "yu64":
        f16 = fm.yu64_from_yuyv(frame8, rng)
        return f16, fm.unpack_yu64(f16), pu.COLOR_FORMAT_YU64
    words, planes = fm.v210_from_yuyv(frame8, rng)
    return words, planes, pu.COLOR_FORMAT_V210


@needs_ref
# 208 / 240: chroma rows of 104 / 120 samples = six / seven SSE2 groups + a scalar tail (no midpoint there)
@pytest.mark.parametrize("fmt,size", [("yu64", (256, 64)), ("yu64", (208, 48)), ("yu64", (704, 96)), ("yu64", (1920, 1080)),
                                      ("v210", (192, 48)), ("v210", (240, 48)), ("v210", (768, 96))])
@pytest.mark.parametrize("kind", ["natural", "random"])
def test_oracle_planar_fields_match_reference_encoder(fmt, size, kind):
    w, h = size
    ref_lib, orc = ol.load_ref(), ol.oracle()
    rng = np.random.default_rng(w + h + len(kind))
    src, planes, color_format = make_source(fmt, w, h, rng, kind)
    ref_lib.ref_set_interlaced(1)
    try:
        bands_ref, div, prescale, _ = pu.ref_encode_frame(ref_lib, src.view(np.uint8), w, h, color_format, 0, 3, 4)
    finally:
        ref_lib.ref_set_interlaced(0)
    pyr = planar_fields_pyramid(orc, planes, div, tuple(prescale[0]))
    for key, want in bands_ref.items():
        if not (key[2] == "LL" and key[1] != 3):
            assert np.array_equal(pyr[key], want), f"band {key}: {np.argwhere(pyr[key] != want)[:4].tolist()}"


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,size", [("yu64", (256, 64)), ("yu64", (208, 48)), ("yu64", (704, 96)), ("yu64", (1920, 1080)), ("yu64", (3840, 2160)),
                                      ("v210", (192, 48)), ("v210", (240, 48)), ("v210", (768, 96)), ("v210", (1920, 1080))])
@pytest.mark.parametrize("kind", ["natural", "random"])
def test_cuda_planar_fields_vs_oracle(fmt, size, kind):
    pkg = importlib.import_module("cineform-sdk_b200")
    w, h = size
    if fmt == "v210" and w % 48:
        w = (w // 48) * 48
    orc = ol.oracle()
    rng = np.random.default_rng(w * 3 + h + len(kind))
    src, planes, _ = make_source(fmt, w, h, rng, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YU64 if fmt == "yu64" else pkg.PIXEL_V210)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    want = planar_fields_pyramid(orc, planes, quant.table(3), tuple(quant.prescale), quant.midpoint_prequant)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        codec.set_interlaced(True)
        coded = [np.zeros(codec.layout.coded_bytes, np.uint8) for _ in range(2)]
        codec.forward_host([src, src[::-1].copy()], quant, coded)
        got = codec.unpack_coded(coded[0])
        for key in sorted(want):
            if key[2] == "LL" and key[1] != 3:
                continue
            assert np.array_equal(got[key], want[key]), f"band {key}: {np.argwhere(got[key] != want[key])[:4].tolist()}"
        # and back: planes of the inverse field transform equal the oracle's inverse of the same bands
        coded_bands = {k: v for k, v in want.items() if not (k[2] == "LL" and k[1] != 3)}
        planes_back = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale), interlaced=True)
        out = np.zeros((3 * h, w), np.int16)
        codec.inverse_host([coded[0]], quant, pkg.PIXEL_PLANAR16, [out])
        for c, pl in enumerate([out[0:h, :w], out[h:2 * h, :w // 2], out[2 * h:3 * h, :w // 2]]):
            assert np.array_equal(pl, planes_back[c]), f"plane {c}"
        if kind == "natural":
            assert pu.psnr(np.clip(planes_back[0], 0, 1023) >> 2, planes[0] >> 2) > 38.0
