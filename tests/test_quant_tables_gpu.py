"""Quantisation with a distinct divisor per channel, level and band, at every midpoint rule, on the GPU.

Every transform kernel quantises in its stores and dequantises in its loads, picking the divisor of a band by channel,
level and band index; border rows and ragged edges have their own stores (border_rows in k_fwd_422_l12_border and the
k_fwd_tma_border launches, k_fwd_plane_edge, k_inv_plane_edge, the border rows of k_inv_plane).  These tests
run every forward source and every inverse output under the tables of test_quant_tables.py -- LH != HL != HH, four
distinct channels, distinct levels, midpoint_prequant 2, 3, 8 and 0, LL divisors > 1 -- and compare bit for bit with the
oracle (8-bit outputs: inside the reference's dither envelope).

T_SMALL keeps every inverse launch on the dp2a dequantiser, T_BIG (one divisor above 255 at every level) puts every
launch on the full multiply: launch_inv_plane, launch_inv_422 and launch_inv_444 (cfb_inverse.cu) instantiate
SMALLDQ = dq_small(), true only when every highpass divisor of the launch's channels is <= 255.  With T_BIG the inverse runs
k_inv_plane<2, false> (prescaled levels 2 and 3) and k_inv_444<false, RG48 / B64A / B64AAlpha / RGB10>; with T_SMALL the
RGB final level runs k_inv_444<true, RG48 / B64A / B64AAlpha / RGB10>, which the built-in quality-4 schedule (level-1
chroma HH 288) never reaches.
The dequantised values of every inverse case fit int16, where the reference's (short)(v * quant) is well defined."""
import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401
from test_quant_tables import (MIDPOINTS, SIZES, frame_byr4, frame_interlaced, frame_rg48, frame_yuyv,
                               fwd_422, fwd_planes, int16_safe, rgb30_components, source_422, table, with_ll)

pytestmark = pytest.mark.gpu

SMALL_SIZES = SIZES[:3]
TABLE_NAMES = ["small", "big"]


def _in_envelope(out, env, what):
    a, b = env
    ok = (out == a) | (out == b)
    if not ok.all():
        bad = np.argwhere(~ok)
        raise AssertionError(f"{what}: {bad.shape[0]} bytes outside the dither envelope, rows {sorted(set(bad[:, 0].tolist()))[:12]}")


def _equal(got, want, what):
    assert got.shape == want.shape, f"{what}: shape {got.shape}, want {want.shape}"
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        raise AssertionError(f"{what}: {bad.shape[0]} mismatches, rows {sorted(set(bad[:, 0].tolist()))[:12]}, first {bad[:4].tolist()}")


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", SIZES)
def test_forward_yuyv_uyvy(pkg, ctx, size, name):
    """Packed 8-bit 4:2:2: 1024x136 takes the fused level-1/2 kernel (k_fwd_422_l12_tma and its border launch), the other
    widths k_fwd_422_tma + k_fwd_plane (720x200: chroma LL3 45 wide, an edge kernel).  The packed filter never
    quantises LL, whatever its divisor."""
    w, h = size
    orc = ol.oracle()
    frame = frame_yuyv(w, h)
    frame_u = fm.yuyv_to_uyvy(frame)
    t = table(name)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 1) as cy, pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_UYVY), 1) as cu:
        for m in MIDPOINTS:
            for tt in ((t, with_ll(t)) if m == 2 else (t,)):
                quant = pkg.make_quant(tt, (0, 2, 0), m)
                what = f"{w}x{h} {name} g={m}{' LL>1' if tt is not t else ''}"
                pu.assert_bands(cy.unpack_coded(cy.forward_host([frame], quant)[0]), fwd_422(orc, frame, tt, (0, 2, 0), m), what + " YUYV")
                pu.assert_bands(cu.unpack_coded(cu.forward_host([frame_u], quant)[0]), fwd_422(orc, frame_u, tt, (0, 2, 0), m, uyvy=True), what + " UYVY")


@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", SMALL_SIZES)
def test_forward_interlaced_yuyv(pkg, ctx, size, name):
    """Packed field transform (k_fwd_422_fields<Src422>): LH through the ordinary quantiser, HL rounded with divisor / g
    (plain_midpoint) before its row difference."""
    w, h = size
    orc = ol.oracle()
    frame = frame_interlaced(w, h)
    t = table(name)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 1) as codec:
        codec.set_interlaced(True)
        for m in MIDPOINTS:
            quant = pkg.make_quant(t, (0, 2, 0), m)
            pu.assert_bands(codec.unpack_coded(codec.forward_host([frame], quant)[0]),
                            fwd_422(orc, frame, t, (0, 2, 0), m, interlaced=True), f"interlaced {w}x{h} {name} g={m}")


@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("fmt", ["yu64", "v210"])
@pytest.mark.parametrize("size", SMALL_SIZES)
def test_forward_yu64_v210(pkg, ctx, size, fmt, name):
    """16-bit / 10-bit 4:2:2 sources, progressive (k_fwd_422_src: level 1 is the planar filter, which quantises LL when
    its divisor is > 1, as does level 3 of a 10-bit source) and interlaced (k_fwd_422_fields<SrcYU64 / SrcV210>: LH rounds with
    divisor / 2 at every g).  An interlaced codec refuses a level-1 LL divisor > 1 with CFB_ERROR_UNSUPPORTED and
    goes on working."""
    w, h = size
    if fmt == "v210":
        w = w // 48 * 48
    orc = ol.oracle()
    src, planes = source_422(fmt, w, h)
    t = table(name)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + fmt.upper())), 1) as codec:
        for m in MIDPOINTS:
            for interlaced in (False, True):
                codec.set_interlaced(interlaced)
                for tt in ((t, with_ll(t)) if not interlaced else (t,)):
                    quant = pkg.make_quant(tt, (0, 2, 0), m)
                    what = f"{fmt} {w}x{h} {name} g={m} {'interlaced' if interlaced else 'progressive'}{' LL>1' if tt is not t else ''}"
                    pu.assert_bands(codec.unpack_coded(codec.forward_host([src], quant)[0]),
                                    fwd_planes(orc, planes, tt, (0, 2, 0), m, interlaced=interlaced), what)
        codec.set_interlaced(True)
        with pytest.raises(pkg.CfbError) as e:
            codec.forward_host([src], pkg.make_quant(with_ll(t), (0, 2, 0), 3))
        assert e.value.code == 102                                     # CFB_ERROR_UNSUPPORTED
        quant = pkg.make_quant(t, (0, 2, 0), 3)
        pu.assert_bands(codec.unpack_coded(codec.forward_host([src], quant)[0]),
                        fwd_planes(orc, planes, t, (0, 2, 0), 3, interlaced=True), f"{fmt} interlaced after the refusal")


@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", SMALL_SIZES)
def test_forward_rgb(pkg, ctx, size, name):
    """RG48 (k_fwd_tma<SrcRG48> + its border launch), the five 10-bit RGB sources (k_fwd_rgb30, one launch per channel)
    and PLANAR16 (k_fwd_plane on caller planes, signed filter at levels 2 and 3).  Level 1 quantises LL when its divisor
    is > 1; the prescaled level 3 of 12-bit sources does not."""
    w, h = size
    orc = ol.oracle()
    t = table(name)
    frame = frame_rg48(w, h)
    rg_planes = fm.unpack_rg48(frame)
    r, g, b = rgb30_components(w, h)
    rgb_planes = fm.rgb30_planes(r, g, b)
    p16 = np.ascontiguousarray(np.concatenate(rg_planes, axis=0))                 # the same planes, stacked
    names = sorted(fm.RGB30_FORMATS)
    codecs = {n: pkg.Codec(ctx, pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + n)), 1) for n in names + ["RG48", "PLANAR16"]}
    try:
        for m in MIDPOINTS:
            for tt in ((t, with_ll(t)) if m == 3 else (t,)):
                quant = pkg.make_quant(tt, (0, 2, 2), m)
                what = f"{w}x{h} {name} g={m}{' LL>1' if tt is not t else ''}"
                cd = codecs["RG48"]
                pu.assert_bands(cd.unpack_coded(cd.forward_host([frame], quant)[0]), fwd_planes(orc, rg_planes, tt, (0, 2, 2), m), what + " RG48")
                cd = codecs["PLANAR16"]
                pu.assert_bands(cd.unpack_coded(cd.forward_host([p16], quant)[0]), fwd_planes(orc, rg_planes, tt, (0, 2, 2), m), what + " PLANAR16")
                want = fwd_planes(orc, rgb_planes, tt, (0, 2, 2), m)
                for n in names:
                    cd = codecs[n]
                    pu.assert_bands(cd.unpack_coded(cd.forward_host([fm.pack_rgb30(n, r, g, b)], quant)[0]), want, f"{what} {n}")
    finally:
        for cd in codecs.values():
            cd.close()


@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", SMALL_SIZES)
def test_forward_byr4(pkg, ctx, size, name):
    """BYR4 (k_fwd_tma<SrcBYR4<LUT>> + its border launch): four channels with four distinct divisor rows, phases 0
    and 3, with and without the encode curve.  `size` is the plane size; the mosaic is twice as wide and high."""
    pw, ph = size
    w, h = 2 * pw, 2 * ph
    orc = ol.oracle()
    bayer = frame_byr4(w, h)
    curve = fm.bayer_log90_curve()
    t = table(name, 4)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_BYR4), 1) as codec:
        for m in MIDPOINTS:
            for tt in ((t, with_ll(t)) if m == 8 else (t,)):
                quant = pkg.make_quant(tt, (0, 2, 2), m)
                for phase in (0, 3):
                    for cv in (None, curve):
                        codec.set_bayer_phase(phase)
                        codec.set_bayer_curve(cv)
                        what = f"BYR4 {w}x{h} {name} g={m} phase {phase} curve {'on' if cv is not None else 'off'}{' LL>1' if tt is not t else ''}"
                        pu.assert_bands(codec.unpack_coded(codec.forward_host([bayer], quant)[0]),
                                        fwd_planes(orc, fm.unpack_byr4(bayer, phase, curve=cv), tt, (0, 2, 2), m), what)


@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", [(720, 200), (208, 56)])
def test_level_api(pkg, ctx, size, name):
    """cfb_level_forward_* at prescale 0 (signed plane, LL quantised when its divisor is > 1) and 2 (non-negative plane),
    every row of the table at every midpoint; cfb_level_inverse_* of the rows with LL divisor 1."""
    w, h = size
    orc = ol.oracle()
    rng = np.random.default_rng(w + h)
    planes = {0: rng.integers(-2500, 2501, (h, w)).astype(np.int16), 2: rng.integers(0, 4096, (h, w)).astype(np.int16)}
    t = table(name, 4)
    rows = [row for per_c in t for row in per_c] + [row for per_c in with_ll(t) for row in per_c]
    for prescale, plane in planes.items():
        for m in MIDPOINTS:
            for div in rows:
                want = orc.fwd_level(plane, 1 if prescale == 2 else 0, div, m)
                got = ctx.level_forward(plane, prescale, div, m)
                for b in range(4):
                    _equal(got[b], want[b], f"level {w}x{h} prescale {prescale} g={m} divisors {div} band {pu.BAND_NAMES[b]}")
                if div[0] == 1 and m == 2:
                    deq = [want[0]] + [pu.dequantize(want[b], div[b]) for b in (1, 2, 3)]
                    assert all(int(np.abs(want[b].astype(np.int64)).max()) * div[b] <= 32767 for b in (1, 2, 3))
                    _equal(ctx.level_inverse(want, prescale, div), orc.inv_level(*deq, prescale), f"level inverse {w}x{h} prescale {prescale} divisors {div}")


def _gop2_table(t):
    """Six wavelets per channel, each with its own divisors: frame A / B level 1 (0 / 1), temporal (2, unquantised),
    the temporal highpass (3) and lowpass levels (4, 5)."""
    rot = lambda row: [1, row[3], row[1], row[2]]
    return [[per_c[0], rot(per_c[0]), [1, 1, 1, 1], per_c[1], rot(per_c[1]), per_c[2]] for per_c in t]


@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", [(704, 200), (256, 56)])
def test_gop2(pkg, ctx, size, name):
    """cfb_gop2_forward_host / _inverse_host under make_gop2_quant with distinct per-wavelet divisors at every midpoint:
    every coded band equals the oracle composition's, and the decoded frames lie inside the dither envelope of the
    oracle's inverse (oracle as in test_gop2.py)."""
    from test_gop2 import _oracle_blocks
    w, h = size
    rng = np.random.default_rng(w + 3 * h)
    fa = pu.synthetic_yuyv(rng, w, h, "random")
    fb = np.roll(fa, 2, axis=0).copy()
    fb[:, 0::2] = np.clip(fb[:, 0::2].astype(np.int32) + rng.integers(-9, 10, (h, w)), 0, 255).astype(np.uint8)
    orc = ol.oracle()
    _, temporal, _ = _oracle_blocks()
    div = _gop2_table(table(name))
    prescale6 = [0, 0, 0, 0, 2, 0]
    prescale = [prescale6 + [0, 0]] * 3
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 2) as codec:
        g = codec.gop2_layout()
        for m in MIDPOINTS:
            gq = pkg.make_gop2_quant(div, prescale6, m)
            level1 = lambda f, c, q: orc.fwd_level_422(f, c, 0, q, 10, m)
            level = lambda p, pre, q: orc.fwd_level(p, 1 if pre == 2 else 0, q, m)
            want = pu.gop2_pyramid(level1, temporal, level, fa, fb, div, prescale)
            cbuf = codec.gop2_forward_host(fa, fb, gq)
            for (c, k, b), wv in sorted(want.items()):
                if k != 2:
                    _equal(codec.gop2_band_view(g, cbuf, c, k, b), wv, f"GOP-2 {w}x{h} {name} g={m} (channel, wavelet, band) {(c, k, b)}")
            if m == 2:
                assert all(int(np.abs(v.astype(np.int64)).max()) * div[c][k][b] <= 32767 for (c, k, b), v in want.items() if k != 2 and b)
                outs = codec.gop2_inverse_host(cbuf, gq, pkg.PIXEL_YUYV, fa.shape)
                for o, planes, fr in zip(outs, pu.gop2_inverse_planes(orc, want, div, prescale), "AB"):
                    _in_envelope(o, pu.yuyv_envelope(planes), f"GOP-2 {w}x{h} {name} frame {fr}")


# ------------------------------------------------------------------------------------------------ inverse
@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", SIZES)
def test_inverse_422(pkg, ctx, size, name):
    """The oracle's coefficients of the same table, to PLANAR16 (k_inv_plane at every level), YUYV / UYVY / YU64 / V210
    (k_inv_422_tma), half and quarter resolution (k_inv_plane, k_lowpass_422)."""
    w, h = size
    orc = ol.oracle()
    t = table(name)
    want = fwd_422(orc, frame_yuyv(w, h), t, (0, 2, 0), 2)
    assert int16_safe(want, t)
    quant = pkg.make_quant(t, (0, 2, 0), 2)
    planes = pu.inverse_pyramid(orc, want, t, (0, 2, 0))
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 1) as codec:
        cbuf = codec.pack_coded(want)
        what = f"{w}x{h} {name}"
        pu.check_planes(pu.planar16(codec, pkg, cbuf, quant, w, h), planes, what + " PLANAR16")
        for fmt, uyvy in ((pkg.PIXEL_YUYV, False), (pkg.PIXEL_UYVY, True)):
            o = np.zeros((h, 2 * w), np.uint8)
            codec.inverse_host([cbuf], quant, fmt, [o])
            _in_envelope(o, pu.yuyv_envelope(planes, uyvy=uyvy), f"{what} 8-bit {'UYVY' if uyvy else 'YUYV'}")
        o16 = np.zeros((h, 2 * w), np.uint16)
        codec.inverse_host([cbuf], quant, pkg.PIXEL_YU64, [o16])
        _equal(o16, fm.pack_yu64(planes), what + " YU64")
        buf = np.zeros((h, fm.v210_natural_pitch(w)), np.uint8)
        codec.inverse_host([cbuf], quant, pkg.PIXEL_V210, [buf])
        _equal(fm.v210_frame_words(buf, w, h), fm.pack_v210_output(planes), what + " V210")
        for res, stop in ((pkg.RESOLUTION_HALF, 1), (pkg.RESOLUTION_QUARTER, 2)):
            low = pu.inverse_pyramid(orc, want, t, (0, 2, 0), stop_level=stop)
            codec.set_decode_resolution(res)
            try:
                rw, rh = codec.decoded_size()
                red = np.zeros((rh, 2 * rw), np.uint8)
                codec.inverse_host([cbuf], quant, pkg.PIXEL_YUYV, [red])
                pu.check_planes(pu.planar16(codec, pkg, cbuf, quant, rw, rh), low, f"{what} lowpass {stop}")
            finally:
                codec.set_decode_resolution(pkg.RESOLUTION_FULL)
            _equal(red, pu.lowpass_to_422(low, unsigned_shift=(stop == 2)), f"{what} reduced-resolution frame {stop}")


@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", SMALL_SIZES)
def test_inverse_interlaced(pkg, ctx, size, name):
    """Inverse field transform (k_fields_carry, k_inv_fields) to PLANAR16 and 8-bit YUYV."""
    w, h = size
    orc = ol.oracle()
    t = table(name)
    want = fwd_422(orc, frame_interlaced(w, h), t, (0, 2, 0), 2, interlaced=True)
    assert int16_safe(want, t)
    quant = pkg.make_quant(t, (0, 2, 0), 2)
    planes = pu.inverse_pyramid(orc, want, t, (0, 2, 0), interlaced=True)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 1) as codec:
        codec.set_interlaced(True)
        cbuf = codec.pack_coded(want)
        pu.check_planes(pu.planar16(codec, pkg, cbuf, quant, w, h), planes, f"interlaced {w}x{h} {name} PLANAR16")
        o = np.zeros((h, 2 * w), np.uint8)
        codec.inverse_host([cbuf], quant, pkg.PIXEL_YUYV, [o])
        _in_envelope(o, pu.yuyv_envelope(planes), f"interlaced {w}x{h} {name} YUYV")


@pytest.mark.parametrize("name", TABLE_NAMES)
@pytest.mark.parametrize("size", SMALL_SIZES)
def test_inverse_rgb(pkg, ctx, size, name):
    """RG48 coefficients to PLANAR16 (k_inv_plane), RG48, B64A and the five 10-bit RGB outputs (k_inv_444<SMALLDQ,
    RG48 / B64A / RGB10>); the BYR4 four-plane inverse to PLANAR16; RGBA 4:4:4:4 coefficients to B64A with the
    de-companded alpha of channel 3 (k_inv_444<SMALLDQ, B64AAlpha>)."""
    w, h = size
    orc = ol.oracle()
    t = table(name)
    want = fwd_planes(orc, fm.unpack_rg48(frame_rg48(w, h)), t, (0, 2, 2), 2)
    assert int16_safe(want, t)
    quant = pkg.make_quant(t, (0, 2, 2), 2)
    planes = pu.inverse_pyramid(orc, want, t, (0, 2, 2))
    outputs = [("RG48", pkg.PIXEL_RG48, np.uint16, 3, fm.pack_rg48(planes)), ("B64A", pkg.PIXEL_B64A, np.uint16, 4, fm.pack_b64a(planes))]
    outputs += [(n, getattr(pkg, "PIXEL_" + n), np.uint32, 1, fm.pack_rgb30_output(n, planes)) for n in sorted(fm.RGB30_FORMATS)]
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_RG48), 1) as codec:
        cbuf = codec.pack_coded(want)
        out = np.zeros((3 * h, w), np.int16)
        codec.inverse_host([cbuf], quant, pkg.PIXEL_PLANAR16, [out])
        pu.check_planes([out[c * h:(c + 1) * h] for c in range(3)], planes, f"RG48 {w}x{h} {name} PLANAR16")
        for n, fmt, dtype, per_pixel, expect in outputs:
            o = np.zeros((h, per_pixel * w), dtype)
            codec.inverse_host([cbuf], quant, fmt, [o])
            _equal(o, expect, f"RG48 {w}x{h} {name} {n} output")
    t4 = table(name, 4)
    bw, bh = 2 * w, 2 * h
    want4 = fwd_planes(orc, fm.unpack_byr4(frame_byr4(bw, bh), 0), t4, (0, 2, 2), 2)
    assert int16_safe(want4, t4)
    planes4 = pu.inverse_pyramid(orc, want4, t4, (0, 2, 2), nchan=4)
    with pkg.Codec(ctx, pkg.FrameDesc(bw, bh, pkg.PIXEL_BYR4), 1) as codec:
        out = np.zeros((4 * h, bw), np.int16)
        codec.inverse_host([codec.pack_coded(want4)], pkg.make_quant(t4, (0, 2, 2), 2), pkg.PIXEL_PLANAR16, [out])
        pu.check_planes([out[c * h:(c + 1) * h, :w] for c in range(4)], planes4, f"BYR4 {bw}x{bh} {name} PLANAR16")
    rgba = fm.unpack_rgba64(fm.synthetic_rgba64(np.random.default_rng(w * 19 + h), w, h, "random", "B64A"), "B64A", True)
    want_a = fwd_planes(orc, rgba, t4, (0, 2, 2), 2)
    assert int16_safe(want_a, t4)
    planes_a = pu.inverse_pyramid(orc, want_a, t4, (0, 2, 2), nchan=4)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_B64A, pkg.FRAME_ALPHA), 1) as codec:
        o = np.zeros((h, 4 * w), np.uint16)
        codec.inverse_host([codec.pack_coded(want_a)], pkg.make_quant(t4, (0, 2, 2), 2), pkg.PIXEL_B64A, [o])
        _equal(o, fm.pack_b64a_alpha(planes_a), f"RGBA {w}x{h} {name} B64A output")


# ------------------------------------------------------------------------------------------------ sparse transfer
@pytest.mark.parametrize("size", [(720, 200), (1920, 1080)])
def test_sparse_at_unit_divisors(pkg, ctx, size):
    """Every divisor 1 on random and extreme content (a batch of 3 distinct frames): the densest coefficients the
    library produces, near kSparseMaxChunk per block.  forward_host_sparse equals the dense forward and the host's
    compaction of it byte for byte (k_sparse_pack), and inverse_host_sparse equals inverse_host (k_sparse_unpack)."""
    w, h = size
    rng = np.random.default_rng(w + h)
    frames = [pu.synthetic_yuyv(rng, w, h, "random"), pu.synthetic_yuyv(rng, w, h, "extreme"), pu.synthetic_yuyv(rng, w, h, "random")]
    quant = pkg.make_quant(pu.UNIT_DIVISORS, (0, 2, 0), 2)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 3) as codec:
        dense = codec.forward_host(frames, quant)
        sparse, sizes = codec.forward_host_sparse(frames, quant)
        words = np.concatenate([d.view(np.int16) for d in dense]).astype(np.int32)
        for v in (-128, -127, 127, 128):
            assert (words == v).any(), f"value {v} never occurs"
        assert (words > 128).any() and (words < -128).any()
        for d, s, n in zip(dense, sparse, sizes):
            x = d.view(np.int16).astype(np.int32)
            blocks = np.zeros((x.size + 8191) // 8192 * 8192, np.int32)            # the format's blocks of 8192 words
            blocks[:x.size] = x
            blocks = blocks.reshape(-1, 8192)
            nz = (blocks != 0).sum(axis=1)
            i = int(np.argmax(nz))
            esc = int(((blocks[i] < -127) | (blocks[i] > 127)).sum())
            assert nz[i] >= 0.9 * 8192 and esc > nz[i] // 2, (int(nz[i]), esc)
            assert pkg.sparse_bytes(s) == n
            assert np.array_equal(pkg.sparse_compact(codec.layout, d), s[:n])
            assert np.array_equal(pkg.sparse_expand(codec.layout, s), d)
        out_d = [np.zeros((h, w * 2), np.uint8) for _ in frames]
        out_s = [np.zeros((h, w * 2), np.uint8) for _ in frames]
        codec.inverse_host(dense, quant, pkg.PIXEL_YUYV, out_d)
        codec.inverse_host_sparse(sparse, quant, pkg.PIXEL_YUYV, out_s)
        for a, b in zip(out_d, out_s):
            assert np.array_equal(a, b)
