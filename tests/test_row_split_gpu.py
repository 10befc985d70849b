"""Bit-exact parity at explicit rows-per-warp splits.

Every transform kernel gives each warp `th` consecutive rows of a band (FwdParams / InvParams .th), and the level-1 kernels
stream those rows through TMA rings that wrap once a warp (or a CTA) has more row chunks than stages.  The library picks
`th` at every launch from the SM count and the batch size (pick_th, cfb_api.cu), so the split an ordinary test exercises
depends on the GPU it runs on and on how many frames it batches.  CFB_TH overrides that choice at every launch: these
tests compute the oracle result of a geometry once and require it at every split in TH -- the production candidates,
odd splits, two rows per warp, and more rows than most bands have -- independently of the device.

The band heights of the geometries (68 / 34 / 17, 100 / 50 / 25, 28 / 14 / 7, and 540 / 270 / 135 at 1920x1080) lie on
both sides of every th, so every level has interior warps, short last warps and warps with a single strip of rows."""
import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import TH, ctx, pkg, splits  # noqa: F401
from test_gop2 import _oracle_blocks
from test_interlaced_planar import make_source, planar_fields_pyramid

pytestmark = pytest.mark.gpu

SIZES = [(1024, 136), (720, 200), (208, 56)]


def _assert_in_envelope(out, env, what):
    a, b = env
    ok = (out == a) | (out == b)
    if not ok.all():
        bad = np.argwhere(~ok)
        raise AssertionError(f"{what}: {bad.shape[0]} bytes outside the dither envelope, rows {sorted(set(bad[:, 0].tolist()))[:12]}")


def _assert_same_at_every_split(outs, what):
    """8-bit outputs carry a deterministic dither: every split must give the bytes of the th = 4 split."""
    for th, o in outs.items():
        for i, (x, y) in enumerate(zip(o, outs[4])):
            assert np.array_equal(x, y), f"{what} output {i} at th={th} differs from th=4: rows {sorted(set(np.argwhere(x != y)[:, 0].tolist()))[:12]}"


# ------------------------------------------------------------------------------------------------ packed 8-bit 4:2:2
@pytest.mark.parametrize("size", SIZES + [(1920, 1080)])
def test_422_at_every_split(pkg, ctx, splits, size):
    """YUYV / UYVY forward (k_fwd_422_tma, k_fwd_plane); the inverse of the oracle's bands to PLANAR16 (k_inv_plane), YUYV /
    UYVY (k_inv_422_tma) and YU64 (its kInvOutYU64 instantiation); half and quarter resolution (k_inv_plane, k_lowpass_422)."""
    w, h = size
    rng = np.random.default_rng(w + h)
    frame = pu.synthetic_yuyv(rng, w, h, "random")
    frame_u = fm.yuyv_to_uyvy(frame)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    want = pu.oracle_forward_422(orc, frame, quant, 0)
    want_u = pu.oracle_forward_422(orc, frame_u, quant, 1)
    table, prescale = quant.table(3), tuple(quant.prescale)
    planes = pu.inverse_pyramid(orc, want, table, prescale)
    yu64 = fm.pack_yu64(planes)
    envs = {pkg.PIXEL_YUYV: pu.yuyv_envelope(planes), pkg.PIXEL_UYVY: pu.yuyv_envelope(planes, uyvy=True)}
    lows = {stop: pu.inverse_pyramid(orc, want, table, prescale, stop_level=stop) for stop in (1, 2)}
    lows8 = {stop: pu.lowpass_to_422(lows[stop], unsigned_shift=(stop == 2)) for stop in (1, 2)}
    out8 = {}
    with pkg.Codec(ctx, desc, 1) as codec, pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_UYVY), 1) as codec_u:
        coded = codec.pack_coded(want)
        for th in splits():
            what = f"{w}x{h} th={th}"
            pu.assert_bands(codec.unpack_coded(codec.forward_host([frame], quant)[0]), want, what + " YUYV forward")
            pu.assert_bands(codec_u.unpack_coded(codec_u.forward_host([frame_u], quant)[0]), want_u, what + " UYVY forward")
            pu.check_planes(pu.planar16(codec, pkg, coded, quant, w, h), planes, what + " PLANAR16")
            o16 = np.zeros((h, 2 * w), np.uint16)
            codec.inverse_host([coded], quant, pkg.PIXEL_YU64, [o16])
            assert np.array_equal(o16, yu64), f"{what} YU64: rows {sorted(set(np.argwhere(o16 != yu64)[:, 0].tolist()))[:12]}"
            out8[th] = []
            for fmt, env in envs.items():
                o = np.zeros((h, 2 * w), np.uint8)
                codec.inverse_host([coded], quant, fmt, [o])
                _assert_in_envelope(o, env, f"{what} 8-bit format {fmt}")
                out8[th].append(o)
            for res, stop in ((pkg.RESOLUTION_HALF, 1), (pkg.RESOLUTION_QUARTER, 2)):
                codec.set_decode_resolution(res)
                try:
                    rw, rh = codec.decoded_size()
                    red = np.zeros((rh, 2 * rw), np.uint8)
                    codec.inverse_host([coded], quant, pkg.PIXEL_YUYV, [red])
                    pu.check_planes(pu.planar16(codec, pkg, coded, quant, rw, rh), lows[stop], f"{what} lowpass {stop}")
                finally:
                    codec.set_decode_resolution(pkg.RESOLUTION_FULL)
                assert np.array_equal(red, lows8[stop]), f"{what} reduced-resolution frame {stop}"
    _assert_same_at_every_split(out8, f"{w}x{h}")


@pytest.mark.parametrize("size", SIZES)
def test_interlaced_at_every_split(pkg, ctx, splits, size):
    """Field transform forward (k_fwd_422_fields<Src422>) and inverse to planes and to 8-bit YUYV (k_fields_carry, k_inv_fields)."""
    w, h = size
    rng = np.random.default_rng(w * 2 + h)
    frame = pu.synthetic_yuyv(rng, w, h, "natural")
    frame[1::2] = np.roll(frame[1::2], 6, axis=1)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    orc = ol.oracle()
    want = pu.oracle_forward_422(orc, frame, quant, 0, interlaced=True)
    planes = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale), interlaced=True)
    env = pu.yuyv_envelope(planes)
    out8 = {}
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_interlaced(True)
        for th in splits():
            what = f"interlaced {w}x{h} th={th}"
            coded = codec.forward_host([frame], quant)[0]
            pu.assert_bands(codec.unpack_coded(coded), want, what)
            pu.check_planes(pu.planar16(codec, pkg, coded, quant, w, h), planes, what + " PLANAR16")
            o = np.zeros_like(frame)
            codec.inverse_host([coded], quant, pkg.PIXEL_YUYV, [o])
            _assert_in_envelope(o, env, what + " YUYV")
            out8[th] = [o]
    _assert_same_at_every_split(out8, f"interlaced {w}x{h}")


@pytest.mark.parametrize("fmt", ["yu64", "v210"])
@pytest.mark.parametrize("size", SIZES)
def test_16bit_and_10bit_422_sources_at_every_split(pkg, ctx, splits, size, fmt):
    """YU64 / V210 sources, progressive (k_fwd_422_src) and interlaced (k_fwd_422_fields<SrcYU64 / SrcV210>), and back to planes."""
    w, h = size
    if fmt == "v210":
        w = w // 48 * 48                                     # whole V210 groups: 1008, 720, 192
    rng = np.random.default_rng(w * 3 + h)
    src, src_planes, _ = make_source(fmt, w, h, rng, "natural")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YU64 if fmt == "yu64" else pkg.PIXEL_V210)
    orc = ol.oracle()
    cases = []
    for interlaced in (False, True):
        quant = pkg.quant_for_quality(desc, 4, interlaced=interlaced)
        table, prescale = quant.table(3), tuple(quant.prescale)
        pyramid = planar_fields_pyramid if interlaced else pu.forward_pyramid_planes
        want = {k: v for k, v in pyramid(orc, src_planes, table, prescale, quant.midpoint_prequant).items() if not (k[2] == "LL" and k[1] != 3)}
        cases.append((interlaced, quant, want, pu.inverse_pyramid(orc, want, table, prescale, interlaced=interlaced)))
    with pkg.Codec(ctx, desc, 1) as codec:
        for th in splits():
            for interlaced, quant, want, planes in cases:
                what = f"{fmt} {w}x{h} {'interlaced' if interlaced else 'progressive'} th={th}"
                codec.set_interlaced(interlaced)
                coded = codec.forward_host([src], quant)[0]
                pu.assert_bands(codec.unpack_coded(coded), want, what)
                pu.check_planes(pu.planar16(codec, pkg, coded, quant, w, h), planes, what + " PLANAR16")


# ------------------------------------------------------------------------------------------------ RGB 4:4:4 and Bayer
@pytest.mark.parametrize("size", SIZES)
def test_rg48_at_every_split(pkg, ctx, splits, size):
    """RG48 forward (k_fwd_tma<SrcRG48> and its border launch: its CTA ring starts a second round at th >= 7); inverse to
    PLANAR16, RG48, B64A and the five 10-bit RGB outputs (k_inv_plane, k_inv_444)."""
    w, h = size
    rng = np.random.default_rng(w + h)
    frame = fm.synthetic_rg48(rng, w, h, "natural")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(3), tuple(quant.prescale)
    orc = ol.oracle()
    want = {k: v for k, v in pu.forward_pyramid_planes(orc, fm.unpack_rg48(frame), table, prescale).items() if not (k[2] == "LL" and k[1] != 3)}
    planes = pu.inverse_pyramid(orc, want, table, prescale)
    outputs = [("RG48", pkg.PIXEL_RG48, np.uint16, 3, fm.pack_rg48(planes)), ("B64A", pkg.PIXEL_B64A, np.uint16, 4, fm.pack_b64a(planes))]
    outputs += [(name, getattr(pkg, "PIXEL_" + name), np.uint32, 1, fm.pack_rgb30_output(name, planes)) for name in sorted(fm.RGB30_FORMATS)]
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(want)
        for th in splits():
            what = f"RG48 {w}x{h} th={th}"
            pu.assert_bands(codec.unpack_coded(codec.forward_host([frame], quant)[0]), want, what)
            out = np.zeros((3 * h, w), np.int16)
            codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [out])
            pu.check_planes([out[c * h:(c + 1) * h] for c in range(3)], planes, what + " PLANAR16")
            for name, fmt, dtype, per_pixel, expect in outputs:
                o = np.zeros((h, per_pixel * w), dtype)
                codec.inverse_host([coded], quant, fmt, [o])
                assert np.array_equal(o, expect), f"{what} {name} output: rows {sorted(set(np.argwhere(o != expect)[:, 0].tolist()))[:12]}"


@pytest.mark.parametrize("size", SIZES)
def test_byr4_at_every_split(pkg, ctx, splits, size):
    """BYR4 forward, all four Bayer phases, with and without the encode curve (k_fwd_tma<SrcBYR4<LUT>> and its border
    launch); the four-plane inverse of phase 0.  `size` is the plane size: the mosaic is twice as wide and high."""
    pw, ph = size
    w, h = 2 * pw, 2 * ph
    rng = np.random.default_rng(w + h)
    bayer = rng.integers(0, 65536, (h, w)).astype(np.uint16)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(4), tuple(quant.prescale)
    orc = ol.oracle()
    curve = fm.bayer_log90_curve()
    cases = [(fmt, cv, pu.forward_pyramid_planes(orc, fm.unpack_byr4(bayer, fmt, curve=cv), table, prescale))
             for fmt in range(4) for cv in (None, curve)]
    coded_bands = {k: v for k, v in cases[0][2].items() if not (k[2] == "LL" and k[1] != 3)}
    planes = pu.inverse_pyramid(orc, coded_bands, table, prescale, nchan=4)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(coded_bands)
        for th in splits():
            for fmt, cv, want in cases:
                codec.set_bayer_phase(fmt)
                codec.set_bayer_curve(cv)
                got = codec.unpack_coded(codec.forward_host([bayer], quant)[0])
                pu.assert_bands(got, want, f"BYR4 {w}x{h} phase {fmt} curve {'on' if cv is not None else 'off'} th={th}")
            out = np.zeros((4 * ph, w), np.int16)               # planes stacked at the frame's pitch (2 * w bytes)
            codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [out])
            pu.check_planes([out[c * ph:(c + 1) * ph, :pw] for c in range(4)], planes, f"BYR4 {w}x{h} th={th} PLANAR16")


@pytest.mark.parametrize("size", SIZES)
def test_rgb30_sources_at_every_split(pkg, ctx, splits, size):
    """The five 10-bit packed RGB sources (k_fwd_rgb30, one launch per channel): the planes, hence the bands, are the same
    for every layout."""
    w, h = size
    rng = np.random.default_rng(w + h)
    r, g, b = [rng.integers(0, 1024, (h, w)).astype(np.uint32) for _ in range(3)]
    names = sorted(fm.RGB30_FORMATS)
    quant = pkg.quant_for_quality(pkg.FrameDesc(w, h, pkg.PIXEL_RG30), 4)
    want = pu.forward_pyramid_planes(ol.oracle(), fm.rgb30_planes(r, g, b), quant.table(3), tuple(quant.prescale), quant.midpoint_prequant)
    codecs = [pkg.Codec(ctx, pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + name)), 1) for name in names]
    try:
        for th in splits():
            for name, codec in zip(names, codecs):
                got = codec.unpack_coded(codec.forward_host([fm.pack_rgb30(name, r, g, b)], quant)[0])
                pu.assert_bands(got, want, f"{name} {w}x{h} th={th}")
    finally:
        for codec in codecs:
            codec.close()


# ------------------------------------------------------------------------------------------------ building blocks
@pytest.mark.parametrize("size", SIZES)
def test_single_level_at_every_split(pkg, ctx, splits, size):
    """cfb_level_forward / _inverse on free-standing planes (k_fwd_plane, k_inv_plane): a signed plane inside the range the
    forward audits (|x| <= 2500, test_range_audit.py) and a non-negative prescaled one, which is also inverted."""
    w, h = size
    rng = np.random.default_rng(w * 7 + h)
    div = [1, 12, 12, 6]
    orc = ol.oracle()
    signed = rng.integers(-2500, 2501, (h, w)).astype(np.int16)
    plane = rng.integers(0, 4096, (h, w)).astype(np.int16)
    want_signed = orc.fwd_level(signed, 0, div, 2)
    want = orc.fwd_level(plane, 1, div, 2)
    back = orc.inv_level(*([want[0]] + [pu.dequantize(want[b], div[b]) for b in (1, 2, 3)]), 2)
    for th in splits():
        what = f"level {w}x{h} th={th}"
        pu.check_planes(ctx.level_forward(signed, 0, div), want_signed, what + " signed forward")
        assert ctx.range_status() == 0
        pu.check_planes(ctx.level_forward(plane, 2, div), want, what + " prescaled forward")
        pu.check_planes([ctx.level_inverse(want, 2, div)], [back], what + " inverse")


@pytest.mark.parametrize("size", [(1024, 136), (704, 200), (256, 56)])
def test_gop2_at_every_split(pkg, ctx, splits, size):
    """cfb_gop2_forward_host / _inverse_host (two-frame GOP: level 1 of both frames, temporal Haar, three more levels):
    every coded band equals the oracle composition's, the decoded frames lie inside the dither envelope of its inverse.
    Widths are multiples of 64 (the GOP layout's chroma bands are whole 16-coefficient groups)."""
    w, h = size
    rng = np.random.default_rng(w + 3 * h)
    fa = pu.synthetic_yuyv(rng, w, h, "natural")
    fb = np.roll(fa, 2, axis=0).copy()
    fb[:, 0::2] = np.clip(fb[:, 0::2].astype(np.int32) + rng.integers(-3, 4, (h, w)), 16, 235).astype(np.uint8)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    gq = pkg.gop2_quant_for_quality(desc, 4, False)
    quant = [[[int(gq.divisor[c][k][b]) for b in range(4)] for k in range(6)] for c in range(3)]
    prescale = [[int(v) for v in gq.prescale] + [0, 0]] * 3
    orc = ol.oracle()
    level1, temporal, level = _oracle_blocks()
    want = pu.gop2_pyramid(level1, temporal, level, fa, fb, quant, prescale)
    envs = [pu.yuyv_envelope(p) for p in pu.gop2_inverse_planes(orc, want, quant, prescale)]
    out8 = {}
    with pkg.Codec(ctx, desc, 2) as codec:
        g = codec.gop2_layout()
        for th in splits():
            what = f"GOP-2 {w}x{h} th={th}"
            coded = codec.gop2_forward_host(fa, fb, gq)
            for (c, k, b), wv in sorted(want.items()):
                if k != 2:                                   # the temporal bands are device scratch, not coded
                    got = codec.gop2_band_view(g, coded, c, k, b)
                    assert np.array_equal(got, wv), f"{what} (channel, wavelet, band) {(c, k, b)}"
            out8[th] = codec.gop2_inverse_host(coded, gq, pkg.PIXEL_YUYV, fa.shape)
            for o, env, name in zip(out8[th], envs, "AB"):
                _assert_in_envelope(o, env, f"{what} frame {name}")
    _assert_same_at_every_split(out8, f"GOP-2 {w}x{h}")


# ------------------------------------------------------------------------------------------------ divisors > 255
@pytest.mark.parametrize("interlaced", [False, True])
def test_422_final_level_divisors_above_255(pkg, ctx, splits, interlaced):
    """Level-1 highpass divisors on both sides of 255: the final 4:2:2 level then dequantises with full multiplies
    (the SMALLDQ = false instantiations of k_inv_422_tma; k_inv_fields dequantises alike for every divisor).
    The coefficients come from the oracle's forward under the same table, so the dequantised values stay in int16."""
    w, h = 720, 200
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    base = pkg.quant_for_quality(desc, 4, interlaced=interlaced)
    biggest = max(d for q in range(1, 7) for per_c in pkg.quant_for_quality(desc, q).table(3) for per_k in per_c for d in per_k)
    print(f"largest divisor of the built-in 4:2:2 schedules: {biggest}")
    table = base.table(3)
    for c, level1 in enumerate(([1, 255, 256, 1000], [1, 1000, 255, 256], [1, 256, 1000, 255])):
        table[c][0] = level1
    quant = pkg.make_quant(table, tuple(base.prescale), base.midpoint_prequant)
    rng = np.random.default_rng(255 + interlaced)
    frame = pu.synthetic_yuyv(rng, w, h, "random")
    if interlaced:
        frame[1::2] = np.roll(frame[1::2], 6, axis=1)
    orc = ol.oracle()
    want = pu.oracle_forward_422(orc, frame, quant, 0, interlaced=interlaced)
    assert max(int(np.abs(want[(c, 1, "LH")]).max()) for c in range(3)) > 0
    planes = pu.inverse_pyramid(orc, want, table, tuple(quant.prescale), interlaced=interlaced)
    env = pu.yuyv_envelope(planes)
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_interlaced(interlaced)
        coded = codec.pack_coded(want)
        for th in splits((4, 16)):
            what = f"{'interlaced' if interlaced else 'progressive'} th={th}"
            pu.check_planes(pu.planar16(codec, pkg, coded, quant, w, h), planes, what + " PLANAR16")
            o = np.zeros_like(frame)
            codec.inverse_host([coded], quant, pkg.PIXEL_YUYV, [o])
            _assert_in_envelope(o, env, what + " YUYV")
            if not interlaced:
                o16 = np.zeros((h, 2 * w), np.uint16)
                codec.inverse_host([coded], quant, pkg.PIXEL_YU64, [o16])
                assert np.array_equal(o16, fm.pack_yu64(planes)), what + " YU64"
