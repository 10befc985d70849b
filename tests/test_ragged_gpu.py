"""Frame widths that are not a multiple of the kernels' lane granularity (720, 1440, 208 ... wide: band widths such as
45 or 13 at level 3).  Forward == oracle == the reference encoder's bands (checked on CPU in test_pyramid_cpu), inverse
== oracle, through every format family and the reduced-resolution / interlaced variants."""
import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401

pytestmark = pytest.mark.gpu
SIZES = [(720, 480), (1440, 1080), (208, 48), (176, 144), (400, 56), (272, 64), (304, 96), (2000, 120)]


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("kind", ["natural", "random"])
def test_ragged_422_roundtrip_vs_oracle(pkg, ctx, size, kind):
    w, h = size
    rng = np.random.default_rng(w + h)
    frame = pu.synthetic_yuyv(rng, w, h, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4 if kind == "natural" else 2)
    orc = ol.oracle()
    want = pu.oracle_forward_422(orc, frame, quant, 0)
    planes = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale))
    with pkg.Codec(ctx, desc, 2) as codec:
        coded = [np.zeros(codec.layout.coded_bytes, np.uint8) for _ in range(2)]
        codec.forward_host([frame, frame[::-1].copy()], quant, coded)
        pu.assert_bands(codec.unpack_coded(coded[0]), want)
        got = pu.planar16(codec, pkg, coded[0], quant, w, h)
        for c in range(3):
            assert np.array_equal(got[c], planes[c]), f"inverse channel {c}"
        out = np.zeros_like(frame)
        codec.inverse_host([coded[0]], quant, pkg.PIXEL_YUYV, [out])
        a, b = pu.yuyv_envelope(planes)
        assert ((out == a) | (out == b)).all()
        # sparse transfer format and reduced-resolution decode on the same geometry
        sp, sizes = codec.forward_host_sparse([frame], quant)
        assert np.array_equal(pkg.sparse_expand(codec.layout, sp[0]), coded[0])
        for res, stop in ((pkg.RESOLUTION_HALF, 1), (pkg.RESOLUTION_QUARTER, 2)):
            codec.set_decode_resolution(res)
            rw, rh = codec.decoded_size()
            red = np.zeros((rh, rw * 2), np.uint8)
            codec.inverse_host([coded[0]], quant, pkg.PIXEL_YUYV, [red])
            lows = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale), stop_level=stop)
            assert np.array_equal(red, pu.lowpass_to_422(lows, unsigned_shift=(stop == 2)))
        codec.set_decode_resolution(pkg.RESOLUTION_FULL)


@pytest.mark.parametrize("size", [(720, 480), (208, 48), (400, 56)])
def test_ragged_interlaced_and_yu64(pkg, ctx, size):
    w, h = size
    rng = np.random.default_rng(w * 2 + h)
    orc = ol.oracle()
    frame = pu.synthetic_yuyv(rng, w, h, "natural")
    frame[1::2] = np.roll(frame[1::2], 6, axis=1)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    want = pu.oracle_forward_422(orc, frame, quant, 0, interlaced=True)
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_interlaced(True)
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        codec.forward_host([frame], quant, [coded])
        pu.assert_bands(codec.unpack_coded(coded), want)
        planes = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale), interlaced=True)
        got = pu.planar16(codec, pkg, coded, quant, w, h)
        for c in range(3):
            assert np.array_equal(got[c], planes[c])
    frame16 = fm.yu64_from_yuyv(frame, rng)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YU64)
    quant = pkg.quant_for_quality(desc, 4)
    want = pu.forward_pyramid_planes(orc, fm.unpack_yu64(frame16), quant.table(3), tuple(quant.prescale), quant.midpoint_prequant)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        codec.forward_host([frame16], quant, [coded])
        pu.assert_bands(codec.unpack_coded(coded), want)


@pytest.mark.parametrize("shape,prescale", [((24, 18), 0), ((30, 94), 0), ((32, 94), 2), ((26, 50), 2), ((48, 90), 0), ((270, 180), 2), ((540, 360), 0)])
def test_ragged_single_level(pkg, ctx, shape, prescale):
    """Free-standing planes whose width is 2, 4 or 6 past a multiple of 8 (band widths 9, 25, 45, 90, 180)."""
    h, w = shape
    rng = np.random.default_rng(h * w)
    plane = rng.integers(0, 4096, (h, w)).astype(np.int16)
    div = [1, 12, 12, 6]
    orc = ol.oracle()
    want = orc.fwd_level(plane, 1 if prescale == 2 else 0, div, 2)
    got = ctx.level_forward(plane, prescale, div)
    for b in range(4):
        if not np.array_equal(got[b], want[b]):
            bad = np.argwhere(got[b] != want[b])
            raise AssertionError(f"band {b}: {bad.shape[0]} mismatches, columns {sorted(set(bad[:, 1].tolist()))}")
    deq = [want[0]] + [pu.dequantize(want[b], div[b]) for b in (1, 2, 3)]
    back = ctx.level_inverse(want, prescale, div)
    ref = orc.inv_level(*deq, 2 if prescale == 2 else 0)
    if not np.array_equal(back, ref):
        bad = np.argwhere(back != ref)
        raise AssertionError(f"inverse: {bad.shape[0]} mismatches, columns {sorted(set(bad[:, 1].tolist()))}")
