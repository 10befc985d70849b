"""Inverse levels 3 and 2 in one pass (k_inv_l32 + k_inv_l32_border, cfb_inverse_l32.inl).

A full or half-resolution decode that runs both levels (inverse mask bits 1 and 2) rebuilds LL2 in registers instead of
writing it to the pyramid and reading it back.  The same codec decodes the same coefficients in two launches when its
inverse mask runs one level per call (4, then 2, then 1): LL2 then goes through the pyramid's scratch region, which keeps
it between calls.  Both must give the same bytes, and the oracle's result, at every rows-per-warp split."""
import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401

pytestmark = pytest.mark.gpu


def _decode(codec, coded, quant, fmt, outs, masks=(7,)):
    """Decode `coded` into `outs` with the inverse masks run one after the other (7: one call, fused levels 3 + 2)."""
    try:
        for m in masks:
            codec.set_level_mask(7, m)
            codec.inverse_host(coded, quant, fmt, outs)
    finally:
        codec.set_level_mask(7, 7)
    return outs


def _fused_and_split(codec, coded, quant, fmt, shape, dtype):
    a = _decode(codec, coded, quant, fmt, [np.zeros(shape, dtype) for _ in coded])
    b = _decode(codec, coded, quant, fmt, [np.zeros(shape, dtype) for _ in coded], masks=(4, 2, 1))
    return a, b


def _assert_same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), f"{what} frame {i}: fused and two-launch decodes differ, rows {sorted(set(np.argwhere(x != y)[:, 0].tolist()))[:12]}"


def _ths(monkeypatch, values):
    for th in values:
        monkeypatch.setenv("CFB_TH", str(th))
        yield th
    monkeypatch.delenv("CFB_TH", raising=False)


# ------------------------------------------------------------------------------------------------ 4:2:2
@pytest.mark.parametrize("size", [(1920, 1080), (256, 48), (1024, 136)])
def test_422_oracle_and_two_launch(pkg, ctx, monkeypatch, size):
    """PLANAR16, YUYV and YU64 of the oracle's bands: the fused decode equals the oracle and the two-launch decode at
    rows-per-warp 2, 3, 4, 8 and 64.  256x48 has the fewest rows a codec takes (level 3: 6 rows)."""
    w, h = size
    rng = np.random.default_rng(w * 7 + h)
    frame = pu.synthetic_yuyv(rng, w, h, "random")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    want = pu.oracle_forward_422(orc, frame, quant, 0)
    planes = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale))
    yu64 = fm.pack_yu64(planes)
    env = pu.yuyv_envelope(planes)
    with pkg.Codec(ctx, desc, 1) as codec:
        assert codec.layout.band[0][2][0].height >= 3
        coded = [codec.pack_coded(want)]
        for th in _ths(monkeypatch, (2, 3, 4, 8, 64)):
            what = f"{w}x{h} th={th}"
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_PLANAR16, (3 * h, w), np.int16)
            _assert_same(a, b, what + " PLANAR16")
            pu.check_planes([a[0][0:h, :w], a[0][h:2 * h, :w // 2], a[0][2 * h:3 * h, :w // 2]], planes, what + " PLANAR16")
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_YU64, (h, 2 * w), np.uint16)
            _assert_same(a, b, what + " YU64")
            assert np.array_equal(a[0], yu64), what + " YU64 against the oracle"
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_YUYV, (h, 2 * w), np.uint8)
            _assert_same(a, b, what + " YUYV")
            assert ((a[0] == env[0]) | (a[0] == env[1])).all(), what + " YUYV outside the oracle's dither envelope"


def test_422_4k_batch_of_16(pkg, ctx, monkeypatch):
    """The benchmark's launch: 16 3840x2160 frames in one call, YUYV and PLANAR16, fused against two launches."""
    w, h, n = 3840, 2160, 16
    rng = np.random.default_rng(16)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    base = pu.synthetic_yuyv(rng, w, h, "natural")
    frames = [np.roll(base, 37 * i, axis=(0, 1)) for i in range(n)]
    with pkg.Codec(ctx, desc, n) as codec:
        coded = [codec.forward_host([f], quant)[0].copy() for f in frames]
        for th in _ths(monkeypatch, (2, 4, 16)):
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_YUYV, (h, 2 * w), np.uint8)
            _assert_same(a, b, f"4K x16 th={th} YUYV")
        a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_PLANAR16, (3 * h, w), np.int16)
        _assert_same(a, b, "4K x16 PLANAR16")


@pytest.mark.parametrize("size", [(720, 200), (208, 56)])
def test_ragged_width_falls_back(pkg, ctx, size):
    """Level-2 chroma bands of 90 / 26 columns are not whole lanes: the two launches run (k_inv_plane + its edge kernel),
    and the decode still equals the oracle."""
    w, h = size
    rng = np.random.default_rng(w + 3 * h)
    frame = pu.synthetic_yuyv(rng, w, h, "random")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    want = pu.oracle_forward_422(orc, frame, quant, 0)
    planes = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale))
    with pkg.Codec(ctx, desc, 1) as codec:
        assert codec.layout.band[1][1][0].width % 4 != 0
        coded = [codec.pack_coded(want)]
        a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_PLANAR16, (3 * h, w), np.int16)
        _assert_same(a, b, f"{w}x{h} PLANAR16")
        pu.check_planes([a[0][0:h, :w], a[0][h:2 * h, :w // 2], a[0][2 * h:3 * h, :w // 2]], planes, f"{w}x{h} PLANAR16")


def test_422_interlaced(pkg, ctx, monkeypatch):
    """Interlaced samples differ at level 1 only: levels 3 and 2 run fused before k_inv_fields."""
    w, h = 1024, 136
    rng = np.random.default_rng(5)
    frame = pu.synthetic_yuyv(rng, w, h, "natural")
    frame[1::2] = np.roll(frame[1::2], 6, axis=1)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    orc = ol.oracle()
    want = pu.oracle_forward_422(orc, frame, quant, 0, interlaced=True)
    planes = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale), interlaced=True)
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_interlaced(True)
        coded = [codec.forward_host([frame], quant)[0].copy()]
        for th in _ths(monkeypatch, (2, 3, 8)):
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_PLANAR16, (3 * h, w), np.int16)
            _assert_same(a, b, f"interlaced th={th} PLANAR16")
            pu.check_planes([a[0][0:h, :w], a[0][h:2 * h, :w // 2], a[0][2 * h:3 * h, :w // 2]], planes, f"interlaced th={th}")
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_YUYV, (h, 2 * w), np.uint8)
            _assert_same(a, b, f"interlaced th={th} YUYV")


def test_half_resolution(pkg, ctx, monkeypatch):
    """Half resolution: LL1 of the fused pass, as 8-bit YUYV (k_lowpass_422) and as PLANAR16, equals the oracle's."""
    w, h = 1024, 136
    rng = np.random.default_rng(11)
    frame = pu.synthetic_yuyv(rng, w, h, "random")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    want = pu.oracle_forward_422(orc, frame, quant, 0)
    low = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale), stop_level=1)
    low8 = pu.lowpass_to_422(low, unsigned_shift=False)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = [codec.pack_coded(want)]
        codec.set_decode_resolution(pkg.RESOLUTION_HALF)
        try:
            rw, rh = codec.decoded_size()
            for th in _ths(monkeypatch, (2, 3, 64)):
                a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_YUYV, (rh, 2 * rw), np.uint8)
                _assert_same(a, b, f"half th={th} YUYV")
                assert np.array_equal(a[0], low8), f"half th={th} YUYV against the oracle"
                pu.check_planes(pu.planar16(codec, pkg, coded[0], quant, rw, rh), low, f"half th={th} PLANAR16")
        finally:
            codec.set_decode_resolution(pkg.RESOLUTION_FULL)


# ------------------------------------------------------------------------------------------------ RGB 4:4:4, Bayer
def test_rg48_level3_prescaled(pkg, ctx, monkeypatch):
    """12-bit RGB: level 3 is prescaled too (k_inv_l32<2, 2, ...>).  PLANAR16 and RG48 against the oracle and two launches."""
    w, h = 1024, 136
    rng = np.random.default_rng(48)
    frame = fm.synthetic_rg48(rng, w, h, "natural")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(3), tuple(quant.prescale)
    assert prescale[2] == 2 and prescale[1] == 2
    orc = ol.oracle()
    want = {k: v for k, v in pu.forward_pyramid_planes(orc, fm.unpack_rg48(frame), table, prescale).items() if not (k[2] == "LL" and k[1] != 3)}
    planes = pu.inverse_pyramid(orc, want, table, prescale)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = [codec.pack_coded(want)]
        for th in _ths(monkeypatch, (2, 3, 4, 8, 64)):
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_PLANAR16, (3 * h, w), np.int16)
            _assert_same(a, b, f"RG48 th={th} PLANAR16")
            pu.check_planes([a[0][c * h:(c + 1) * h] for c in range(3)], planes, f"RG48 th={th} PLANAR16")
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_RG48, (h, 3 * w), np.uint16)
            _assert_same(a, b, f"RG48 th={th} RG48")
            assert np.array_equal(a[0], fm.pack_rg48(planes)), f"RG48 th={th} RG48 against the oracle"


def test_byr4_planes(pkg, ctx, monkeypatch):
    """BYR4: four planes, PLANAR16 against the oracle and two launches."""
    pw, ph = 512, 72
    w, h = 2 * pw, 2 * ph
    rng = np.random.default_rng(4)
    bayer = rng.integers(0, 65536, (h, w)).astype(np.uint16)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(4), tuple(quant.prescale)
    orc = ol.oracle()
    bands = pu.forward_pyramid_planes(orc, fm.unpack_byr4(bayer, 0), table, prescale)
    coded_bands = {k: v for k, v in bands.items() if not (k[2] == "LL" and k[1] != 3)}
    planes = pu.inverse_pyramid(orc, coded_bands, table, prescale, nchan=4)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = [codec.pack_coded(coded_bands)]
        for th in _ths(monkeypatch, (2, 3, 8)):
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_PLANAR16, (4 * ph, w), np.int16)
            _assert_same(a, b, f"BYR4 th={th} PLANAR16")
            pu.check_planes([a[0][c * ph:(c + 1) * ph, :pw] for c in range(4)], planes, f"BYR4 th={th} PLANAR16")


# ------------------------------------------------------------------------------------------------ saturation, launches
def test_ll2_saturates(pkg, ctx, monkeypatch):
    """Extreme level-3 bands drive LL2 past int16: the fused pass must saturate it to [-32768, 32767] exactly where the
    int16 store of the level-3 launch does.  The quarter-resolution PLANAR16 decode shows LL2 as that store leaves it."""
    w, h = 1024, 136
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    rng = np.random.default_rng(32767)
    with pkg.Codec(ctx, desc, 1) as codec:
        lay = codec.layout
        buf = np.zeros(lay.coded_bytes, np.uint8)
        for c in range(3):
            for k in range(3):
                for b in range(4):
                    if b == 0 and k != 2:
                        continue
                    v = codec.band_view(buf, c, k, b)
                    if k == 2:
                        v[:] = rng.choice(np.array([-32767, -20000, 0, 20000, 32767], np.int16), v.shape)
                    else:
                        v[:] = rng.integers(-40, 41, v.shape).astype(np.int16)
        coded = [buf]
        codec.set_decode_resolution(pkg.RESOLUTION_QUARTER)
        try:
            qw, qh = codec.decoded_size()
            ll2 = pu.planar16(codec, pkg, buf, quant, qw, qh)
        finally:
            codec.set_decode_resolution(pkg.RESOLUTION_FULL)
        assert any((p == 32767).any() for p in ll2) and any((p == -32768).any() for p in ll2), "LL2 does not saturate"
        for th in _ths(monkeypatch, (2, 3, 16)):
            a, b = _fused_and_split(codec, coded, quant, pkg.PIXEL_PLANAR16, (3 * h, w), np.int16)
            _assert_same(a, b, f"saturated LL2 th={th} PLANAR16")


@pytest.mark.parametrize("res", ["full", "half"])
def test_kernel_launches(pkg, ctx, res):
    """The fused pass counts its two launches: a full progressive 4:2:2 inverse is 3 launches (fused main + border rows +
    the final level), a half-resolution 8-bit one 3 too (fused main + border rows + k_lowpass_422)."""
    w, h = 1920, 1080
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    rng = np.random.default_rng(3)
    frame = pu.synthetic_yuyv(rng, w, h, "natural")
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.forward_host([frame], quant)[0].copy()
        if res == "half":
            codec.set_decode_resolution(pkg.RESOLUTION_HALF)
        rw, rh = codec.decoded_size()
        before = ctx.stats()["kernel_launches"]
        codec.inverse_host([coded], quant, pkg.PIXEL_YUYV, [np.zeros((rh, 2 * rw), np.uint8)])
        assert ctx.stats()["kernel_launches"] - before == 3
        codec.set_decode_resolution(pkg.RESOLUTION_FULL)
