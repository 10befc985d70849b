"""16-bit packed outputs of the final inverse level (SURVEY 8 row a16): YU64 from 4:2:2 samples and RG48 from RGB 4:4:4
samples.  Neither uses dither, so the whole chain is bit-exact: the oracle rule (formats.row16u, restating
Codec/InvertHorizontalStrip16s.c:16571 incl. its SSE2-loop / scalar-tail saturation difference) is pinned to the
reference's real decoder on the CPU, and the CUDA path is compared with both on the GPU."""
import hashlib

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")


def _sample_422(ref_lib, w, h, kind):
    rng = np.random.default_rng(w + len(kind))
    frame = pu.qbist_yuy2(ref_lib, w, h, 2) if kind == "qbist" else pu.synthetic_yuyv(rng, w, h, kind)
    _, div, prescale, sample = pu.ref_encode_frame(ref_lib, frame, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, 4)
    return sample, prescale[0]


def _sample_444(ref_lib, w, h, kind):
    rng = np.random.default_rng(w + len(kind))
    frame = pu.qbist_rg48(ref_lib, w, h, 1) if kind == "qbist" else fm.synthetic_rg48(rng, w, h, kind)
    _, div, prescale, sample = pu.ref_encode_frame(ref_lib, frame.view(np.uint8), w, h, pu.COLOR_FORMAT_RG48, 1, 3, 4)
    return sample, prescale[0]


@needs_ref
@pytest.mark.parametrize("size", [(640, 96), (704, 96), (208, 48), (720, 480)])
@pytest.mark.parametrize("kind", ["qbist", "extreme"])
def test_oracle_yu64_matches_reference_decoder(size, kind):
    w, h = size
    ref_lib, orc = ol.load_ref(), ol.oracle()
    sample, prescale = _sample_422(ref_lib, w, h, kind)
    out, bands = pu.ref_decode(ref_lib, sample, w, h, fm.OUTPUTS["YU64"].decoded_format, 3, w * 4)
    planes = pu.inverse_pyramid(orc, bands, pu.UNIT_DIVISORS, tuple(prescale))
    want = fm.pack_yu64(planes)
    got = out.view(np.uint16).reshape(h, 2 * w)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5].tolist()
    if kind == "extreme":       # the case that separates the two saturation rules
        assert (got == 65535).any() and (got == 0xFFC0).any()


@needs_ref
@pytest.mark.parametrize("size", [(640, 96), (328, 48), (720, 480)])
@pytest.mark.parametrize("kind", ["qbist", "extreme"])
def test_oracle_rg48_matches_reference_decoder(size, kind):
    w, h = size
    if kind == "extreme" and w * h > 100000:
        pytest.skip("0/65535 noise at this size does not fit the probe's sample buffer")
    ref_lib, orc = ol.load_ref(), ol.oracle()
    sample, prescale = _sample_444(ref_lib, w, h, kind)
    out, bands = pu.ref_decode(ref_lib, sample, w, h, fm.OUTPUTS["RG48"].decoded_format, 3, w * 6)
    planes = pu.inverse_pyramid(orc, bands, pu.UNIT_DIVISORS, tuple(prescale))
    want = fm.pack_rg48(planes)
    got = out.view(np.uint16).reshape(h, 3 * w)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5].tolist()


@needs_ref
@pytest.mark.parametrize("size", [(640, 96), (328, 48), (256, 64), (200, 48), (1016, 64), (720, 480)])
@pytest.mark.parametrize("kind", ["qbist", "extreme"])
def test_oracle_b64a_matches_reference_decoder(size, kind):
    """B64A from an RGB 4:4:4 sample: the same reconstructed planes as RG48, a constant alpha and one limit for all columns."""
    w, h = size
    if kind == "extreme" and w * h > 100000:
        pytest.skip("0/65535 noise at this size does not fit the probe's sample buffer")
    ref_lib, orc = ol.load_ref(), ol.oracle()
    sample, prescale = _sample_444(ref_lib, w, h, kind)
    out, bands = pu.ref_decode(ref_lib, sample, w, h, fm.OUTPUTS["B64A"].decoded_format, 3, w * 8)
    planes = pu.inverse_pyramid(orc, bands, pu.UNIT_DIVISORS, tuple(prescale))
    want = fm.pack_b64a(planes)
    got = out.view(np.uint16).reshape(h, 4 * w)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5].tolist()
    if kind == "extreme":       # both saturation rules occur: the SSE2 loop's 12-bit limit and the scalar code's 65535
        assert (got[:, 1::4] == 0xFFF0).any() and (got[:, 1::4] == 65535).any()
        assert not (got[:, :8 * fm.b64a_tail_col(w // 2)] == 65535).any()


@needs_ref
@pytest.mark.parametrize("size", [(640, 96), (328, 48), (256, 64), (200, 48), (1016, 64), (720, 480)])
@pytest.mark.parametrize("kind", ["qbist", "extreme"])
def test_oracle_rgb30_outputs_match_reference_decoder(size, kind):
    """The five 10-bit packed RGB outputs of an RGB 4:4:4 sample: truncation of the limited 12-bit sample, one rule for all
    columns.  The bands are the ones the decoder held for THAT output format (its lowpass decode adds a per-format offset)."""
    w, h = size
    if kind == "extreme" and w * h > 100000:
        pytest.skip("0/65535 noise at this size does not fit the probe's sample buffer")
    ref_lib, orc = ol.load_ref(), ol.oracle()
    sample, prescale = _sample_444(ref_lib, w, h, kind)
    rg48_bands = pu.ref_decode(ref_lib, sample, w, h, fm.OUTPUTS["RG48"].decoded_format, 3, w * 6)[1]
    for name, (fmt, _, _) in fm.RGB30_FORMATS.items():
        out, bands = pu.ref_decode(ref_lib, sample, w, h, fmt, 3, w * 4)
        planes = pu.inverse_pyramid(orc, bands, pu.UNIT_DIVISORS, tuple(prescale))
        want = fm.pack_rgb30_output(name, planes)
        got = out.view(np.uint32).reshape(h, w)
        assert np.array_equal(got, want), (name, np.argwhere(got != want)[:5].tolist())
        # the host-side offset of the lowpass decode: the coded bands are the RG48 decode's except for a constant on LL3
        # (6 where the reference's threaded lowpass decode applies it, decoder.c:12308; 0 otherwise)
        for key in bands:
            delta = bands[key].astype(np.int32) - rg48_bands[key].astype(np.int32)
            if key[2] != "LL":
                assert not delta.any(), key
            elif key[1] == 3:
                assert delta.min() == delta.max() and int(delta.min()) in (0, 6), (key, int(delta.min()), int(delta.max()))


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(256, 64), (640, 96), (704, 96), (720, 480), (1920, 1080), (3840, 2160)])
@pytest.mark.parametrize("kind", ["natural", "extreme"])
def test_gpu_yu64_output_vs_oracle(pkg, size, kind):
    w, h = size
    rng = np.random.default_rng(w + h)
    frame = pu.synthetic_yuyv(rng, w, h, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    coded_bands = pu.oracle_forward_422(orc, frame, quant, 0)
    want = fm.pack_yu64(pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale)))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        coded = codec.pack_coded(coded_bands)
        outs = [np.zeros((h, 2 * w), np.uint16) for _ in range(2)]
        codec.inverse_host([coded, coded], quant, pkg.PIXEL_YU64, outs)
    assert np.array_equal(outs[0], want), np.argwhere(outs[0] != want)[:5].tolist()
    assert np.array_equal(outs[1], want)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(256, 64), (328, 48), (640, 96), (720, 480), (1920, 1080), (3840, 2160)])
@pytest.mark.parametrize("kind", ["natural", "extreme"])
def test_gpu_rg48_output_vs_oracle(pkg, size, kind):
    w, h = size
    rng = np.random.default_rng(w + h)
    if (w, h) == (3840, 2160):
        tile = fm.synthetic_rg48(rng, w // 2, h // 2, kind)
        frame = np.tile(tile.reshape(h // 2, w // 2, 3), (2, 2, 1)).reshape(h, w * 3).copy()
    else:
        frame = fm.synthetic_rg48(rng, w, h, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    pyr = pu.forward_pyramid_planes(orc, fm.unpack_rg48(frame), quant.table(3), tuple(quant.prescale))
    coded_bands = {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}
    want = fm.pack_rg48(pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale)))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        out = np.zeros((h, 3 * w), np.uint16)
        codec.inverse_host([codec.pack_coded(coded_bands)], quant, pkg.PIXEL_RG48, [out])
    assert np.array_equal(out, want), np.argwhere(out != want)[:5].tolist()
    if kind == "natural":       # config 4 round trip: 12-bit fidelity of the decoded RG48 frame
        mse = np.mean(((out >> 4).astype(np.float64) - (frame >> 4).astype(np.float64)) ** 2)
        assert 10 * np.log10(4095.0 ** 2 / mse) > 45.0


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(640, 96), (1920, 1080)])
def test_gpu_16bit_outputs_vs_reference_decoder(pkg, size):
    """End of the chain: the reference encodes and decodes a Qbist frame (its real entropy coder in between); our inverse,
    fed the bands its decoder held, reproduces its YU64 / RG48 frames byte for byte.  At 640x96 the reference's bands and
    frame hashes are stored under golden/ (make_golden.py decoded_outputs); the 1920x1080 case needs oracle/_ref."""
    w, h = size
    if size != (640, 96) and not ol.ref_available():
        pytest.skip("oracle/_ref not built (reference absent)")
    for fmt, kind, sampler, dfmt, bpp, cfb_src, cfb_out in (
            ("YU64", "yuy2", _sample_422, fm.OUTPUTS["YU64"].decoded_format, 4, "PIXEL_YUYV", "PIXEL_YU64"),
            ("RG48", "rg48", _sample_444, fm.OUTPUTS["RG48"].decoded_format, 6, "PIXEL_RG48", "PIXEL_RG48")):
        if size == (640, 96):
            bands, prescale, want = pu.reference_decoded(kind, fmt)
        else:
            ref_lib = ol.load_ref()
            sample, prescale = sampler(ref_lib, w, h, "qbist")
            ref_out, bands = pu.ref_decode(ref_lib, sample, w, h, dfmt, 3, w * bpp)
            bands = {k: v for k, v in bands.items() if not (k[2] == "LL" and k[1] != 3)}    # the coded region: LL3 + highpass
            want = hashlib.sha256(np.ascontiguousarray(ref_out).tobytes()).hexdigest()
        desc = pkg.FrameDesc(w, h, getattr(pkg, cfb_src))
        unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
        with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
            out = np.zeros((h, w * bpp // 2), np.uint16)
            codec.inverse_host([codec.pack_coded(bands)], unit, getattr(pkg, cfb_out), [out])
        assert hashlib.sha256(out.tobytes()).hexdigest() == want, fmt
