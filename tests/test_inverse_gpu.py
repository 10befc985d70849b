"""GPU parity tests of the inverse path (fused dequantisation + 3 inverse levels), through the C ABI."""
import hashlib
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401
from test_golden import GOLDEN, load_golden, load_golden_decoder_side

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("size", [(192, 48), (256, 64), (320, 56), (704, 96), (1920, 1080)])
@pytest.mark.parametrize("kind", ["natural", "random"])
def test_inverse_planar16_vs_oracle(pkg, ctx, size, kind):
    """Quantised bands produced by the oracle's forward -> our inverse (dequant fused) == oracle inverse."""
    w, h = size
    rng = np.random.default_rng(w + h)
    frame = pu.synthetic_yuyv(rng, w, h, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    coded_bands = pu.oracle_forward_422(orc, frame, quant, 0)
    want = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale))
    with pkg.Codec(ctx, desc, 1) as codec:
        got = pu.planar16(codec, pkg, codec.pack_coded(coded_bands), quant, w, h)
    pu.check_planes(got, want)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_inverse_golden_decoder_bands(pkg, ctx, path):
    """Bands exactly as the reference's decoder held them -> our inverse: the 16-bit planes equal the oracle's
    and the 8-bit YUYV output lies inside the reference decoder's dither envelope (and within 1 LSB of the
    frame the reference actually produced)."""
    frame, div, prescale, quality, _ = load_golden(path)
    bands, dec = load_golden_decoder_side(path)
    h, w2 = frame.shape
    w = w2 // 2
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    orc = ol.oracle()
    want = pu.inverse_pyramid(orc, bands, pu.UNIT_DIVISORS, prescale)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(bands)
        pu.check_planes(pu.planar16(codec, pkg, coded, unit, w, h), want)
        out = np.zeros((h, w2), np.uint8)
        codec.inverse_host([coded], unit, pkg.PIXEL_YUYV, [out])
    a, b = pu.yuyv_envelope(want)
    ok = (out == a) | (out == b)
    assert ok.all(), f"{(~ok).sum()} bytes outside the reference's dither envelope"
    assert np.abs(out.astype(int) - dec.astype(int)).max() <= 1


@pytest.mark.parametrize("fmt", [0, 1])
def test_roundtrip_psnr_and_uyvy(pkg, ctx, fmt):
    w, h = 1920, 1080
    rng = np.random.default_rng(12)
    frame = pu.synthetic_yuyv(rng, w, h, "natural")
    if fmt:
        frame = fm.yuyv_to_uyvy(frame)
    pf = pkg.PIXEL_UYVY if fmt else pkg.PIXEL_YUYV
    desc = pkg.FrameDesc(w, h, pf)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.forward_host([frame], quant)[0]
        out = np.zeros_like(frame)
        codec.inverse_host([coded], quant, pf, [out])
    yo = 1 if fmt else 0
    # the synthetic frame carries sigma=2 noise, which FILMSCAN1 does not preserve: ~47.5 dB luma here
    assert pu.psnr(out[:, yo::2], frame[:, yo::2]) > 45.0        # luma PSNR, as TestCFHD reports it
    assert pu.psnr(out, frame) > 44.0


def test_roundtrip_4k_batch(pkg, ctx, monkeypatch):
    """The step bench.py times: 16 distinct 3840x2160 frames in one launch sequence, forward then inverse to 8-bit YUYV and
    to PLANAR16.  A batch of 16 gives every level other rows per warp than a single frame does (th = 16 / 16 / 8 forward,
    8 / 16 / 16 inverse on a 132-SM H100: the final level's TMA ring wraps twice), and frame 15 uses the last tensor map of
    the batch.  Run with the split the device picks and with CFB_TH = 16 and 12: every frame's coefficients and decoded
    outputs equal those of the frame processed alone at th = 4; frames 0 and 15 equal the oracle."""
    w, h, n = 3840, 2160, 16
    rng = np.random.default_rng(5)
    base = pu.synthetic_yuyv(rng, w, h, "natural")
    frames = [np.roll(base, (8 * i, 64 * i), axis=(0, 1)).copy() for i in range(n)]
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    oracle = {}
    for i in (0, n - 1):
        bands = pu.oracle_forward_422(orc, frames[i], quant, 0)
        planes = pu.inverse_pyramid(orc, bands, quant.table(3), tuple(quant.prescale))
        oracle[i] = (bands, planes, pu.yuyv_envelope(planes))

    def digest(a):
        return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()

    def planar(a):
        return [a[0:h, :w], a[h:2 * h, :w // 2], a[2 * h:3 * h, :w // 2]]

    monkeypatch.setenv("CFB_TH", "4")
    alone = []
    with pkg.Codec(ctx, desc, 1) as codec:
        for f in frames:
            coded = codec.forward_host([f], quant)[0]
            o8 = np.zeros_like(f)
            codec.inverse_host([coded], quant, pkg.PIXEL_YUYV, [o8])
            o16 = np.zeros((3 * h, w), np.int16)
            codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [o16])
            alone.append((digest(coded), digest(o8), digest(o16)))
    for th in (None, "16", "12"):
        if th is None:
            monkeypatch.delenv("CFB_TH")
        else:
            monkeypatch.setenv("CFB_TH", th)
        what = f"th={th or 'device default'}"
        with pkg.Codec(ctx, desc, n) as codec:
            coded = codec.forward_host(frames, quant)
            for i, c in enumerate(coded):
                if i in oracle:
                    pu.assert_bands(codec.unpack_coded(c), oracle[i][0], f"{what} frame {i}")
                assert digest(c) == alone[i][0], f"{what} frame {i}: coefficients differ from the frame coded alone"
            outs = [np.zeros_like(f) for f in frames]
            codec.inverse_host(coded, quant, pkg.PIXEL_YUYV, outs)
            for i, (f, o) in enumerate(zip(frames, outs)):
                if i in oracle:
                    a, b = oracle[i][2]
                    assert ((o == a) | (o == b)).all(), f"{what} frame {i}: outside the dither envelope"
                assert digest(o) == alone[i][1], f"{what} frame {i}: 8-bit output differs from the frame decoded alone"
                assert pu.psnr(o[:, 0::2], f[:, 0::2]) > 45.0
            del outs
            outs = [np.zeros((3 * h, w), np.int16) for _ in range(n)]
            codec.inverse_host(coded, quant, pkg.PIXEL_PLANAR16, outs)
            for i, o in enumerate(outs):
                if i in oracle:
                    pu.check_planes(planar(o), oracle[i][1], f"{what} frame {i} PLANAR16")
                assert digest(o) == alone[i][2], f"{what} frame {i}: planes differ from the frame decoded alone"
            del outs, coded


def _reduced(codec, pkg, coded, quant, res, fmt):
    """Decode `coded` at a reduced resolution: returns (packed 8-bit frame, [Y, V, U] int16 lowpass planes)."""
    codec.set_decode_resolution(res)
    try:
        w, h = codec.decoded_size()
        out = np.zeros((h, w * 2), np.uint8)
        codec.inverse_host([coded], quant, fmt, [out])
        pl = np.zeros((3 * h, w), np.int16)
        codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [pl])
    finally:
        codec.set_decode_resolution(pkg.RESOLUTION_FULL)
    return out, [pl[0:h, :w], pl[h:2 * h, :w // 2], pl[2 * h:3 * h, :w // 2]]


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_reduced_resolution_golden(pkg, ctx, path):
    """CFHD_DECODED_RESOLUTION_HALF / _QUARTER: lowpass images equal the reference decoder's own LL1 / LL2, the
    half-resolution frame equals what CFHD_DecodeSample returned byte for byte, the quarter-resolution frame equals
    the oracle's CopyQuarterRowToBuffer restatement."""
    z = np.load(path)
    frame, _, prescale, _, _ = load_golden(path)
    bands, _ = load_golden_decoder_side(path)
    h, w2 = frame.shape
    desc = pkg.FrameDesc(w2 // 2, h, pkg.PIXEL_YUYV)
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(bands)
        for res, stop, name in ((pkg.RESOLUTION_HALF, 1, "half"), (pkg.RESOLUTION_QUARTER, 2, "quarter")):
            out, planes = _reduced(codec, pkg, coded, unit, res, pkg.PIXEL_YUYV)
            pu.check_planes(planes, [z[f"r_{c}_{stop}_LL"] for c in range(3)])
            assert np.array_equal(out, pu.lowpass_to_422(planes, unsigned_shift=(stop == 2)))
            if name == "half":
                assert np.array_equal(out, z["decoded_half_yuy2"])
        # and the codec still decodes at full resolution afterwards
        full = np.zeros((h, w2), np.uint8)
        codec.inverse_host([coded], unit, pkg.PIXEL_YUYV, [full])
        assert np.abs(full.astype(int) - z["decoded_yuy2"].astype(int)).max() <= 1


@pytest.mark.parametrize("size", [(192, 48), (448, 120), (1920, 1080), (3840, 2160)])
@pytest.mark.parametrize("fmt_name", ["YUYV", "UYVY"])
def test_reduced_resolution_vs_oracle(pkg, ctx, size, fmt_name):
    """Random (adversarial: negative and > 4095 lowpass values occur) coefficients: both shift rules and byte orders."""
    w, h = size
    fmt = getattr(pkg, "PIXEL_" + fmt_name)
    rng = np.random.default_rng(w * 3 + h)
    frame = pu.synthetic_yuyv(rng, w, h, "random")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 3)
    orc = ol.oracle()
    coded_bands = pu.oracle_forward_422(orc, frame, quant, 0)
    # push the lowpass images out of the 8-bit range in places: scale LL3 of every channel
    for c in range(3):
        ll = coded_bands[(c, 3, "LL")].astype(np.int32)
        coded_bands[(c, 3, "LL")] = np.clip((ll - 8000) * 3, -32768, 32767).astype(np.int16)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(coded_bands)
        for res, stop in ((pkg.RESOLUTION_HALF, 1), (pkg.RESOLUTION_QUARTER, 2)):
            want = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale), stop_level=stop)
            out, planes = _reduced(codec, pkg, coded, quant, res, fmt)
            pu.check_planes(planes, want)
            assert np.array_equal(out, pu.lowpass_to_422(want, unsigned_shift=(stop == 2), uyvy=(fmt_name == "UYVY")))
            assert out.min() == 0                    # negative lowpass values occur (clamped / wrapped by the two rules)
