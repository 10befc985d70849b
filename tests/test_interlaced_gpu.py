"""GPU parity tests of the interlaced (field transform) level 1, through the C ABI:
forward == oracle == the reference's EncodeSample bands (golden), inverse == oracle and inside the reference
decoder's dither envelope."""
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401
from test_golden import GOLDEN_FIELDS, load_golden, load_golden_decoder_side

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("path", GOLDEN_FIELDS, ids=[os.path.basename(p) for p in GOLDEN_FIELDS])
def test_forward_reproduces_reference_encoder_bands(pkg, ctx, path):
    frame, div, prescale, quality, bands = load_golden(path)
    h, w2 = frame.shape
    desc = pkg.FrameDesc(w2 // 2, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, quality, interlaced=True)
    assert quant.table(3) == div
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_interlaced(True)
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        codec.forward_host([frame], quant, [coded])
        got = codec.unpack_coded(coded)
    coded_bands = {k: v for k, v in bands.items() if not (k[2] == "LL" and k[1] != 3)}
    assert set(got) == set(coded_bands)
    pu.assert_bands(got, coded_bands)


@pytest.mark.parametrize("path", GOLDEN_FIELDS, ids=[os.path.basename(p) for p in GOLDEN_FIELDS])
def test_inverse_of_reference_decoder_bands(pkg, ctx, path):
    """Bands as the reference's decoder held them (HL put back into its coded, differenced form): 16-bit planes equal
    the oracle's, 8-bit output inside the decoder's dither envelope and within 1 LSB of the frame it produced."""
    frame, div, prescale, quality, _ = load_golden(path)
    bands, dec = load_golden_decoder_side(path)
    for c in range(3):
        hl = bands[(c, 1, "HL")].astype(np.int32)
        hl[:, 1:] -= hl[:, :-1].copy()
        bands[(c, 1, "HL")] = hl.astype(np.int16)
    h, w2 = frame.shape
    w = w2 // 2
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    want = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, prescale, interlaced=True)
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_interlaced(True)
        coded = codec.pack_coded(bands)
        got = pu.planar16(codec, pkg, coded, unit, w, h)
        out = np.zeros((h, w2), np.uint8)
        codec.inverse_host([coded], unit, pkg.PIXEL_YUYV, [out])
    for c in range(3):
        assert np.array_equal(got[c], want[c]), f"channel {c}"
    a, b = pu.yuyv_envelope(want)
    assert ((out == a) | (out == b)).all()
    assert np.abs(out.astype(int) - dec.astype(int)).max() <= 1


@pytest.mark.parametrize("size", [(192, 48), (256, 64), (448, 120), (704, 96), (1920, 1080), (3840, 2160)])
@pytest.mark.parametrize("kind,fmt_name", [("natural", "YUYV"), ("random", "YUYV"), ("natural", "UYVY")])
def test_field_transform_vs_oracle(pkg, ctx, size, kind, fmt_name):
    """Forward and inverse against the oracle on synthetic interlaced content, strips and borders of every width class;
    then the round trip through our own forward + inverse."""
    w, h = size
    fmt = getattr(pkg, "PIXEL_" + fmt_name)
    uyvy = fmt_name == "UYVY"
    rng = np.random.default_rng(w * 5 + h + (7 if uyvy else 0))
    frame = pu.synthetic_yuyv(rng, w, h, kind)
    frame[1::2] = np.roll(frame[1::2], 8, axis=1)           # the two fields differ
    if uyvy:
        frame = fm.yuyv_to_uyvy(frame)
    desc = pkg.FrameDesc(w, h, fmt)
    quant = pkg.quant_for_quality(desc, 4 if kind == "natural" else 2, interlaced=True)
    orc = ol.oracle()
    want_bands = pu.oracle_forward_422(orc, frame, quant, 1 if uyvy else 0, interlaced=True)
    want_planes = pu.inverse_pyramid(orc, want_bands, quant.table(3), tuple(quant.prescale), interlaced=True)
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_interlaced(True)
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        codec.forward_host([frame], quant, [coded])
        pu.assert_bands(codec.unpack_coded(coded), want_bands)
        got = pu.planar16(codec, pkg, coded, quant, w, h)
        for c in range(3):
            assert np.array_equal(got[c], want_planes[c]), f"inverse channel {c}"
        out = np.zeros_like(frame)
        codec.inverse_host([coded], quant, fmt, [out])
        a, b = pu.yuyv_envelope(want_planes, uyvy=uyvy)
        assert ((out == a) | (out == b)).all()
        if kind == "natural":
            yo = 1 if uyvy else 0
            assert pu.psnr(out[:, yo::2], frame[:, yo::2]) > 40.0
        # switching the flag off restores the progressive transform on the same codec
        codec.set_interlaced(False)
        q2 = pkg.quant_for_quality(desc, 4)
        codec.forward_host([frame], q2, [coded])
        pu.assert_bands(codec.unpack_coded(coded), pu.oracle_forward_422(orc, frame, q2, 1 if uyvy else 0))


def test_interlaced_batch_device_resident(pkg, ctx):
    """Batch of 4 different frames in one launch == 4 single-frame results (frame index plumbing of the carries)."""
    w, h = 704, 96
    rng = np.random.default_rng(99)
    frames = []
    for i in range(4):
        f = pu.synthetic_yuyv(rng, w, h, "natural")
        f[1::2] = np.roll(f[1::2], 4 + 2 * i, axis=1)
        frames.append(f)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    with pkg.Codec(ctx, desc, 4) as codec:
        codec.set_interlaced(True)
        coded = [np.zeros(codec.layout.coded_bytes, np.uint8) for _ in range(4)]
        codec.forward_host(frames, quant, coded)
        outs = [np.zeros_like(frames[0]) for _ in range(4)]
        codec.inverse_host(coded, quant, pkg.PIXEL_YUYV, outs)
        for i in range(4):
            one = np.zeros(codec.layout.coded_bytes, np.uint8)
            codec.forward_host([frames[i]], quant, [one])
            assert np.array_equal(one, coded[i])
            o1 = np.zeros_like(frames[0])
            codec.inverse_host([one], quant, pkg.PIXEL_YUYV, [o1])
            assert np.array_equal(o1, outs[i])


def test_final_level_kernel_launches(pkg, ctx):
    """The library's kernel_launches counter: the interlaced final level counts k_fields_carry + k_inv_fields, the
    progressive one its single kernel.  With the HL band already integrated (the reference decoder's bands) there are no
    row carries to compute, so k_fields_carry does not run and k_inv_fields is the one launch."""
    w, h = 256, 64
    frame = pu.synthetic_yuyv(np.random.default_rng(5), w, h, "natural")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    deltas = {}
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        for mode in (pkg.PROGRESSIVE, pkg.INTERLACED, pkg.INTERLACED_HL_INTEGRATED):
            codec.set_interlaced(mode)
            codec.forward_host([frame], quant, [coded])
            codec.set_level_mask(7, 1)
            before = ctx.stats()["kernel_launches"]
            codec.inverse_host([coded], quant, pkg.PIXEL_YUYV, [np.zeros_like(frame)])
            deltas[mode] = ctx.stats()["kernel_launches"] - before
            codec.set_level_mask(7, 7)
    assert deltas == {pkg.PROGRESSIVE: 1, pkg.INTERLACED: 2, pkg.INTERLACED_HL_INTEGRATED: 1}


def test_interlaced_rejected_for_non_422(pkg, ctx):
    """The field transform exists for 4:2:2 sources only: every other input format refuses it."""
    for name in ("RG48", "BYR4", "PLANAR16", "RG30", "AB10", "AR10", "R210", "DPX0", "B64A", "RG64"):
        for flags in ((0, pkg.FRAME_ALPHA) if name in ("B64A", "RG64") else (0,)):
            with pkg.Codec(ctx, pkg.FrameDesc(256, 96, getattr(pkg, "PIXEL_" + name), flags), 1) as codec:
                with pytest.raises(pkg.CfbError) as ei:
                    codec.set_interlaced(True)
                assert ei.value.code == 102, name      # CFB_ERROR_UNSUPPORTED
