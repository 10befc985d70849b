"""Reduced-resolution decodes to the deep outputs (CPU): the numpy restatements in formats.py -- YU64 at half resolution,
the 10-bit RGB words at quarter resolution -- equal byte for byte the frames the reference decoder writes from the lowpass
images it held (ref_set_decode_resolution + ref_decode_sample_bands), and the oracle's inverse of the bands it read gives
those lowpass images.  The golden fixtures keep the rules pinned where oracle/_ref is absent.  RG48 at half and at quarter
resolution: the reference decoder does not write what the routines it names would, so the library leaves them unsupported;
the tests below record what it writes instead."""
import glob
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reduced_*.npz")))
RGB_SIZES = [(640, 96), (200, 64), (328, 48), (256, 64), (1016, 48)]         # LL2 widths 160, 50, 82, 64, 254
YUV_SIZES = [(640, 96), (336, 48), (208, 48), (720, 64), (1296, 48)]         # LL1 chroma widths 160, 84, 52, 180, 324


def _rgb_sample(ref_lib, w, h, kind, nchan):
    """An RGB 4:4:4 (nchan 3) or RGBA 4:4:4:4 (nchan 4) sample; "blocks" drives LL2 out of [0, 16383] on both sides."""
    import rgba_util as ru
    if nchan == 4:
        frame = fm.synthetic_rgba64(np.random.default_rng(w + h), w, h, "extreme", "B64A")
        return ru.ref_encode(ref_lib, frame, w, h, "B64A", True)[2:]
    frame = fm.block_rg48(w, h, 2, w) if kind == "blocks" else fm.synthetic_rg48(np.random.default_rng(w + h), w, h, kind)
    _, _, prescale, sample = pu.ref_encode_frame(ref_lib, frame.view(np.uint8), w, h, pu.COLOR_FORMAT_RG48, 1, 3,
                                                 1 if kind == "blocks" else 4)
    return prescale[0], sample


def _yuv_sample(ref_lib, w, h, kind, fmt):
    rng = np.random.default_rng(w + h)
    frame = pu.synthetic_yuyv(rng, w, h, kind)
    if fmt == "UYVY":
        frame, cf = fm.yuyv_to_uyvy(frame), pu.COLOR_FORMAT_UYVY
    elif fmt == "YU64":
        frame, cf = fm.yu64_from_yuyv(frame, rng).view(np.uint8), pu.COLOR_FORMAT_YU64
    elif fmt == "V210":
        frame, cf = fm.v210_from_yuyv(frame, rng)[0].view(np.uint8), pu.COLOR_FORMAT_V210
    else:
        cf = pu.COLOR_FORMAT_YUYV
    _, _, prescale, sample = pu.ref_encode_frame(ref_lib, frame, w, h, cf, 0, 3, 4)
    return prescale[0], sample


def _check_oracle(bands, prescale, res, nchan=3):
    """The oracle's inverse of the bands the decoder read gives the lowpass images it converted."""
    planes = pu.inverse_pyramid(ol.oracle(), fm.reduced_coded_bands(bands, res, nchan), [[[1] * 4] * 3] * nchan,
                                tuple(prescale), nchan=nchan, stop_level=res - 1)
    for c in range(nchan):
        assert np.array_equal(planes[c], bands[(c, res - 1, "LL")]), f"channel {c}"


def _assert_equal(got, want, what):
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{what}: {bad.shape[0]} differ, first {bad[:5].tolist()}"


# ------------------------------------------------------------------------------------------------ reference decoder
@needs_ref
@pytest.mark.parametrize("size", RGB_SIZES, ids=[f"{w}x{h}" for w, h in RGB_SIZES])
@pytest.mark.parametrize("kind", ["natural", "blocks", "rgba"])
def test_quarter_rgb_rules_match_reference_decoder(size, kind):
    w, h = size
    ref_lib = ol.load_ref()
    nchan = 4 if kind == "rgba" else 3
    prescale, sample = _rgb_sample(ref_lib, w, h, kind, nchan)
    for name in fm.RGB30_FORMATS:
        got, right, below, bands = fm.ref_decode_reduced(ref_lib, sample, w, h, fm.OUTPUTS[name].decoded_format, nchan,
                                                        fm.QUARTER, 4)
        ll = fm.lowpass_images(bands, fm.QUARTER)
        _assert_equal(got.view(np.uint32), fm.OUTPUTS[name].reduced[fm.QUARTER](ll), f"{name} {w}x{h} {kind}")
        assert not right.any() and not below.any()
        _check_oracle(bands, prescale, fm.QUARTER, nchan)
    if kind == "blocks":        # both clamps of either rule occur in the data
        v = np.concatenate([p.ravel() for p in ll]).astype(np.int64)
        assert (v < 0).any() and (v > 16383).any()


@needs_ref
@pytest.mark.parametrize("size", YUV_SIZES, ids=[f"{w}x{h}" for w, h in YUV_SIZES])
@pytest.mark.parametrize("fmt", ["YUYV", "UYVY", "YU64", "V210"])
def test_half_yu64_rule_matches_reference_decoder(size, fmt):
    w, h = size
    if fmt == "V210" and w % 48:
        pytest.skip("V210 sources are multiples of 48 pixels wide")
    ref_lib = ol.load_ref()
    for kind in ("natural", "extreme"):
        prescale, sample = _yuv_sample(ref_lib, w, h, kind, fmt)
        got, right, below, bands = fm.ref_decode_reduced(ref_lib, sample, w, h, fm.OUTPUTS["YU64"].decoded_format, 3, fm.HALF, 4)
        ll = fm.lowpass_images(bands, fm.HALF)
        _assert_equal(got.view(np.uint16), fm.OUTPUTS["YU64"].reduced[fm.HALF](ll), f"{fmt} {w}x{h} {kind}")
        assert not right.any() and not below.any()


@needs_ref
def test_limits_are_reached():
    """The data of the pins above reaches YU64's 0 and 4095 limits and both quarter-resolution clamps."""
    ref_lib = ol.load_ref()
    _, sample = _yuv_sample(ref_lib, 640, 96, "extreme", "YUYV")
    bands = fm.ref_decode_reduced(ref_lib, sample, 640, 96, fm.OUTPUTS["YU64"].decoded_format, 3, fm.HALF, 4)[3]
    v = np.concatenate([p.ravel() for p in fm.lowpass_images(bands, fm.HALF)]).astype(np.int64)
    assert (v < 0).any() and (v > 4095).any()
    frame = fm.OUTPUTS["YU64"].reduced[fm.HALF](fm.lowpass_images(bands, fm.HALF))
    assert (frame == 0).any() and (frame == 4095 << 4).any()


@needs_ref
@pytest.mark.parametrize("size", [(640, 96), (200, 64), (328, 48)])
def test_public_api_quarter_rgb10(size):
    """CFHD_DecodeSample at CFHD_DECODED_RESOLUTION_QUARTER takes the same path: the same frame, top-left in the buffer."""
    w, h = size
    ref_lib = ol.load_ref()
    _, sample = _rgb_sample(ref_lib, w, h, "blocks", 3)
    rc, out, dims = fm.ref_decode_api(ref_lib, sample, w, h, ol.fourcc("r210"), fm.QUARTER, 4)
    got, _, _, bands = fm.ref_decode_reduced(ref_lib, sample, w, h, fm.OUTPUTS["R210"].decoded_format, 3, fm.QUARTER, 4)
    assert rc == 0 and dims == (w // 4, h // 4)
    assert np.array_equal(out[:h // 4, :w // 4 * 4], got)
    assert np.array_equal(got.view(np.uint32), fm.OUTPUTS["R210"].reduced[fm.QUARTER](fm.lowpass_images(bands, fm.QUARTER)))


@needs_ref
def test_quarter_rg48_is_not_the_named_routine():
    """Why RG48 at quarter resolution stays unsupported.  ConvertUnpacked16sRowToRGB48 writes min(max(ll << 2, 0), 65535),
    and the decoder does on LL2 values up to 16383; above 16383 it writes 65535 at 640 x 96 but 65528 at 200 x 64 and
    328 x 48, which that routine cannot produce."""
    ref_lib = ol.load_ref()
    above = {}
    for w, h in ((640, 96), (200, 64), (328, 48)):
        _, sample = _rgb_sample(ref_lib, w, h, "blocks", 3)
        got, _, _, bands = fm.ref_decode_reduced(ref_lib, sample, w, h, fm.OUTPUTS["RG48"].decoded_format, 3, fm.QUARTER, 6)
        g, r, b = fm.lowpass_images(bands, fm.QUARTER)
        x = np.zeros((h // 4, 3 * (w // 4)), np.int64)
        x[:, 0::3], x[:, 1::3], x[:, 2::3] = r, g, b
        got, named = got.view(np.uint16), fm.OUTPUTS["RG48"].reduced[fm.QUARTER]([g, r, b])
        assert (x > 16383).any() and np.array_equal(got[x <= 16383], named[x <= 16383])
        above[(w, h)] = set(got[x > 16383].tolist())
    assert above[(640, 96)] == {65535} and above[(200, 64)] == {65528} and above[(328, 48)] == {65528}


@needs_ref
@pytest.mark.parametrize("size", [(640, 96), (336, 48)])
def test_public_api_half_yu64(size):
    w, h = size
    ref_lib = ol.load_ref()
    _, sample = _yuv_sample(ref_lib, w, h, "extreme", "YUYV")
    rc, out, dims = fm.ref_decode_api(ref_lib, sample, w, h, ol.fourcc("YU64"), fm.HALF, 4)
    got, _, _, bands = fm.ref_decode_reduced(ref_lib, sample, w, h, fm.OUTPUTS["YU64"].decoded_format, 3, fm.HALF, 4)
    assert rc == 0 and dims == (w // 2, h // 2)
    assert np.array_equal(out[:h // 2, :w // 2 * 4], got)
    assert np.array_equal(got.view(np.uint16), fm.OUTPUTS["YU64"].reduced[fm.HALF](fm.lowpass_images(bands, fm.HALF)))


@needs_ref
@pytest.mark.parametrize("size", [(640, 96), (200, 64), (328, 48)])
def test_half_rg48_is_not_the_named_routine(size):
    """Why RG48 at half resolution stays unsupported.  The reference decoder does not write ConvertLowpass16sRGB48ToRGB48's
    (uint16)(ll << 2): on out-of-range LL1 values it clamps instead of wrapping, and when the LL1 width is not a multiple of
    8 (200 x 64, 328 x 48) it writes the R and B samples of other columns."""
    w, h = size
    ref_lib = ol.load_ref()
    _, sample = _rgb_sample(ref_lib, w, h, "extreme", 3)
    got, _, _, bands = fm.ref_decode_reduced(ref_lib, sample, w, h, fm.OUTPUTS["RG48"].decoded_format, 3, fm.HALF, 6)
    g, r, b = [p.astype(np.int64) for p in fm.lowpass_images(bands, fm.HALF)]
    got = got.view(np.uint16)
    wrap = np.zeros(got.shape, np.int64)
    wrap[:, 0::3], wrap[:, 1::3], wrap[:, 2::3] = (r << 2) & 0xFFFF, (g << 2) & 0xFFFF, (b << 2) & 0xFFFF
    clamp = np.zeros(got.shape, np.int64)
    clamp[:, 0::3], clamp[:, 1::3], clamp[:, 2::3] = [np.clip(x << 2, 0, 65535) for x in (r, g, b)]
    assert not np.array_equal(got, wrap)
    assert np.array_equal(got, clamp) == ((w // 2) % 8 == 0)


# ------------------------------------------------------------------------------------------------ the rules themselves
def test_rgb10_simd_and_tail_rules_are_not_vacuous():
    """The SSE2 rule and the scalar tail agree on every value an LL2 image of a 12-bit source reaches, and differ below
    -0x4000, where the saturating add leaves the value unsaturated; the restatement applies each to its own columns."""
    x = np.arange(-32768, 32768, dtype=np.int64)
    simd, tail = fm.rgb10_simd(x, 2), fm.rgb10_tail(x, 2)
    assert np.array_equal(simd[x >= -0x4000], tail[x >= -0x4000])
    assert (simd[x < -0x4000] != 0).any() and not tail[x < 0].any()
    assert simd[x == 16383] == 1023 and simd[x == 32767] == 1023 and tail[x == 32767] == 1023
    plane = np.full((1, 12), -20000, np.int16)
    words = fm.OUTPUTS["RG30"].reduced[fm.QUARTER]([plane, plane, plane])
    assert (words[0, :8] != 0).all() and not words[0, 8:].any()


def test_quarter_and_yu64_clamps_are_not_vacuous():
    v = np.array([[-5, 0, 1, 4095, 4096, 16383, 16384, 32767]], np.int16)
    assert fm.OUTPUTS["RG30"].reduced[fm.QUARTER]([v, v, v])[0].tolist() == [(x << 20) | (x << 10) | x for x in (0, 0, 0, 255, 256, 1023, 1023, 1023)]
    assert fm.OUTPUTS["YU64"].reduced[fm.HALF]([v, v[:, ::2], v[:, 1::2]])[0, 0::2].tolist() == [0, 0, 16, 65520, 65520, 65520, 65520, 65520]


def test_golden_present():
    assert sorted(os.path.basename(p).split("_")[1] + "_" + os.path.basename(p).split("_")[2] for p in GOLDEN) == \
        ["rgb10_quarter", "yu64_half"]


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_golden_frames_follow_the_rules(path):
    """The stored decoder bands -> oracle inverse -> the lowpass images the decoder held -> the rule -> the stored frame."""
    z = np.load(path)
    res = fm.HALF if "_half_" in path else fm.QUARTER
    fmts = sorted({k.split("_")[1] for k in z.files if k.startswith("frame_")})
    for fmt in fmts:
        bands = {(int(c), int(k), b): z[key] for key in z.files if key.startswith(f"d_{fmt}_")
                 for c, k, b in [key.split("_")[2:]]}
        ll = [z[f"ll_{fmt}_{c}"] for c in range(3)]
        planes = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, tuple(int(v) for v in z["prescale"]),
                                    stop_level=res - 1)
        for c in range(3):
            assert np.array_equal(planes[c], ll[c]), (fmt, c)
        want = fm.OUTPUTS[fmt].reduced[res](ll)
        assert np.array_equal(z[f"frame_{fmt}"], want), fmt
