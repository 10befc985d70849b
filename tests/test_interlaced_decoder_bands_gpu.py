"""GPU tests of the interlaced inverse on the bands the reference's entropy decoder hands over: level-1 HL already
integrated along its rows (Codec/decoder.c:20822-20836) and every highpass band dequantised, decoded with
INTERLACED_HL_INTEGRATED (mode 2, what the SDK shim runs), against the oracle, the reference decoder's frame and the
INTERLACED decode (mode 1) of the coded, difference-coded band.  Also the shim's sparse hand-over: per-band buffers
compacted by cfb_sparse_compact_bands and decoded by cfb_inverse_host_sparse."""
import os

import numpy as np
import pytest

import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401
from test_golden import GOLDEN, GOLDEN_FIELDS, load_golden, load_golden_decoder_side
from test_gop2 import _oracle_blocks

pytestmark = pytest.mark.gpu

LUMA_STRIP, CHROMA_STRIP = 120, 60      # band columns per inverse strip (kInvStrip) and its chroma half
LUMA_HALO, CHROMA_HALO = 4, 2           # columns a strip loads left of its first output column


def interlaced_frame(rng, w, h, kind, shift=8):
    f = pu.synthetic_yuyv(rng, w, h, kind)
    f[1::2] = np.roll(f[1::2], shift, axis=1)           # the two fields differ
    return f


def with_hl(bands, hls):
    out = dict(bands)
    for c, hl in enumerate(hls):
        out[(c, 1, "HL")] = hl
    return out


def integrated(bands):
    """Level-1 HL integrated along its rows, every other band as it is."""
    return with_hl(bands, [pu.integrate_hl(bands[(c, 1, "HL")]) for c in range(3)])


def differenced(hl):
    d = hl.astype(np.int32)
    d[:, 1:] -= d[:, :-1].copy()
    return d.astype(np.int16)


def decoder_form(bands, table):
    """What the reference's FSM decoder leaves: every highpass band dequantised with int16 wrap (decoder.c:20551), then
    the level-1 HL band integrated; decoded with unit divisors."""
    out = {k: v if k[2] == "LL" else pu.dequantize(v, table[k[0]][k[1] - 1][pu.BAND_NAMES.index(k[2])])
           for k, v in bands.items()}
    return integrated(out)


def decode(pkg, codec, bands, quant, mode, fmt):
    """Full-resolution decode of one band set in the given interlaced mode: [Y, V, U] planes or the packed 8-bit frame."""
    codec.set_interlaced(mode)
    coded = codec.pack_coded(bands)
    w, h = codec.desc.width, codec.desc.height
    if fmt == pkg.PIXEL_PLANAR16:
        return [p.copy() for p in pu.planar16(codec, pkg, coded, quant, w, h)]
    out = np.zeros((h, 2 * w), np.uint8)
    codec.inverse_host([coded], quant, fmt, [out])
    return out


def assert_in_envelope(out, planes, uyvy=False):
    a, b = pu.yuyv_envelope(planes, uyvy=uyvy)
    ok = (out == a) | (out == b)
    assert ok.all(), f"{(~ok).sum()} bytes outside the dither envelope, first {np.argwhere(~ok)[:4].tolist()}"


def forward_bands(pkg, ctx, frames, quant):
    w, h = frames[0].shape[1] // 2, frames[0].shape[0]
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), len(frames)) as codec:
        codec.set_interlaced(pkg.INTERLACED)
        coded = codec.forward_host(frames, quant)
        return [codec.unpack_coded(c) for c in coded]


# ------------------------------------------------------------------------------------------------ (a) golden
@pytest.mark.parametrize("path", GOLDEN_FIELDS, ids=[os.path.basename(p) for p in GOLDEN_FIELDS])
def test_golden_decoder_bands_as_handed_over(pkg, ctx, path):
    """The reference decoder's bands as they are (HL integrated and dequantised), unit divisors, mode 2: PLANAR16 equals the
    oracle, YUYV and UYVY lie inside the dither envelope, YUYV within 1 LSB of the reference decoder's frame."""
    frame, div, prescale, quality, _ = load_golden(path)
    bands, dec = load_golden_decoder_side(path)
    h, w = frame.shape[0], frame.shape[1] // 2
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    want = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, prescale, interlaced=True, hl_integrated=True)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 1) as codec:
        mode = pkg.INTERLACED_HL_INTEGRATED
        pu.check_planes(decode(pkg, codec, bands, unit, mode, pkg.PIXEL_PLANAR16), want, "PLANAR16")
        yuyv = decode(pkg, codec, bands, unit, mode, pkg.PIXEL_YUYV)
        uyvy = decode(pkg, codec, bands, unit, mode, pkg.PIXEL_UYVY)
    assert_in_envelope(yuyv, want)
    assert_in_envelope(uyvy, want, uyvy=True)
    assert np.abs(yuyv.astype(int) - dec.astype(int)).max() <= 1


# ------------------------------------------------------------------------------------------------ (b) three forms
SIZES = [(192, 48), (256, 64), (448, 120), (704, 96), (1920, 1080), (3840, 2160), (720, 480), (1440, 1080)]
CASES = [(s, k) for k in ("natural", "random") for s in SIZES] + [((720, 480), "hl_divisor_300"), ((1920, 1080), "hl_divisor_300")]


@pytest.mark.parametrize("size,kind", CASES, ids=[f"{w}x{h}-{k}" for (w, h), k in CASES])
def test_three_forms_agree(pkg, ctx, size, kind):
    """Our forward's bands decoded three ways give identical PLANAR16 and 8-bit bytes, all equal to the oracle:
    (i) mode 1 on the coded (differenced, quantised) bands with the real quant, (ii) mode 2 on integrate_hl of the
    quantised HL with the real quant, (iii) mode 2 on the decoder form with unit divisors.  hl_divisor_300: the level-1 HL
    divisors exceed 255, the range where the inverse kernels leave their byte-sized dequantiser."""
    w, h = size
    rng = np.random.default_rng(w * 3 + h)
    frame = interlaced_frame(rng, w, h, "random" if kind == "random" else "natural")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 2 if kind == "random" else 4, interlaced=True)
    if kind == "hl_divisor_300":
        for c, d in enumerate((300, 271, 257)):
            quant.divisor[c][0][2] = d
    table, prescale = quant.table(3), tuple(quant.prescale)
    q = forward_bands(pkg, ctx, [frame], quant)[0]
    want = pu.inverse_pyramid(ol.oracle(), q, table, prescale, interlaced=True)
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    forms = {"(i) coded, mode 1": (q, quant, pkg.INTERLACED),
             "(ii) integrated, mode 2": (integrated(q), quant, pkg.INTERLACED_HL_INTEGRATED),
             "(iii) decoder form, mode 2": (decoder_form(q, table), unit, pkg.INTERLACED_HL_INTEGRATED)}
    outs = {}
    with pkg.Codec(ctx, desc, 1) as codec:
        for name, (bands, qt, mode) in forms.items():
            pu.check_planes(decode(pkg, codec, bands, qt, mode, pkg.PIXEL_PLANAR16), want, name)
            outs[name] = decode(pkg, codec, bands, qt, mode, pkg.PIXEL_YUYV)
    first = outs["(i) coded, mode 1"]
    for name, out in outs.items():
        assert np.array_equal(out, first), f"{name}: 8-bit bytes differ from (i)"
    assert_in_envelope(first, want)


# ------------------------------------------------------------------------------------------------ (c) carries
def carry_rows(rng, rows, width, strip, halo):
    """Integrated HL rows inside +-2000 whose differences are large and alternate in sign, with a jump of +-1500 on the
    last column that the carry of each strip sums (strip - halo - 1: 115, 235, ... luma, 57, 117, ... chroma) and on the
    first column the next strip loads itself."""
    s = rng.integers(300, 1800, (rows, width)) * np.where(np.arange(width) % 2 == 0, 1, -1)[None, :]
    for end in range(strip - halo, width, strip):
        for col in (end - 1, end):
            s[:, col] = s[:, col - 1] + np.where(s[:, col - 1] > 0, -1500, 1500)
    assert np.abs(s).max() <= 2000
    return s.astype(np.int16)


@pytest.mark.parametrize("size", [(1920, 1080), (720, 480)])
def test_carry_across_strips_in_range(pkg, ctx, size):
    """Large alternating HL differences and +-1500 jumps at every strip boundary, prefix sums in range: mode 1 on the
    differenced rows and mode 2 on the integrated rows both equal the oracle."""
    w, h = size
    rng = np.random.default_rng(w + 5 * h)
    quant = pkg.quant_for_quality(pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 4, interlaced=True)
    prescale = tuple(quant.prescale)
    base = decoder_form(forward_bands(pkg, ctx, [interlaced_frame(rng, w, h, "natural")], quant)[0], quant.table(3))
    hls = []
    for c in range(3):
        bh, bw = base[(c, 1, "HL")].shape
        hls.append(carry_rows(rng, bh, bw, LUMA_STRIP if c == 0 else CHROMA_STRIP, LUMA_HALO if c == 0 else CHROMA_HALO))
    assert not np.array_equal(hls[1], hls[2])
    bands2 = with_hl(base, hls)
    bands1 = with_hl(base, [differenced(hl) for hl in hls])
    for c in range(3):
        assert np.array_equal(pu.integrate_hl(bands1[(c, 1, "HL")]), hls[c])
    want = pu.inverse_pyramid(ol.oracle(), bands2, pu.UNIT_DIVISORS, prescale, interlaced=True, hl_integrated=True)
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 1) as codec:
        for name, bands, mode in (("mode 1", bands1, pkg.INTERLACED), ("mode 2", bands2, pkg.INTERLACED_HL_INTEGRATED)):
            pu.check_planes(decode(pkg, codec, bands, unit, mode, pkg.PIXEL_PLANAR16), want, name)
            assert_in_envelope(decode(pkg, codec, bands, unit, mode, pkg.PIXEL_YUYV), want)


# ------------------------------------------------------------------------------------------------ (d) wrap-around
def wrapping_rows(rng, rows, width, strip, halo):
    """Differenced HL rows whose running sum crosses +-32768 many times: runs of 37 columns that climb or fall by
    6000 - 14000 per column, and +-30000 on the last carry column of each strip and the first column after it."""
    d = rng.integers(6000, 14000, (rows, width)) * np.where((np.arange(width) // 37) % 2 == 0, 1, -1)[None, :]
    for end in range(strip - halo, width, strip):
        d[:, end - 1:end + 1] = rng.choice([-30000, 30000], (rows, 2))
    assert np.abs(np.cumsum(d, axis=1)).max() > 4 * 32768
    return d.astype(np.int16)


@pytest.mark.parametrize("divisors", ["unit", "real"])
@pytest.mark.parametrize("size", [(1920, 1080), (720, 480)])
def test_wraparound_modes_agree(pkg, ctx, size, divisors):
    """HL rows whose running sum wraps around int16 several times, inside a strip and across strip boundaries: mode 1 on
    the differenced rows equals mode 2 on integrate_hl of them (the decoder's wrapping `line[x] += line[x-1]`).  Only the
    two GPU modes are compared: the reconstruction from such values leaves int16, where the reference's saturating
    inverse and the kernels' exact int32 arithmetic part ways, outside the parity claim against the oracle (DESIGN.md
    section 4, overflow semantics)."""
    w, h = size
    rng = np.random.default_rng(w + 7 * h)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    q = forward_bands(pkg, ctx, [interlaced_frame(rng, w, h, "natural")], quant)[0]
    if divisors == "unit":
        q, quant = decoder_form(q, quant.table(3)), pkg.make_quant(pu.UNIT_DIVISORS, tuple(quant.prescale))
    hls = []
    for c in range(3):
        bh, bw = q[(c, 1, "HL")].shape
        hls.append(wrapping_rows(rng, bh, bw, LUMA_STRIP if c == 0 else CHROMA_STRIP, LUMA_HALO if c == 0 else CHROMA_HALO))
    bands1 = with_hl(q, hls)
    bands2 = integrated(bands1)
    with pkg.Codec(ctx, desc, 1) as codec:
        for fmt in (pkg.PIXEL_PLANAR16, pkg.PIXEL_YUYV):
            a = decode(pkg, codec, bands1, quant, pkg.INTERLACED, fmt)
            b = decode(pkg, codec, bands2, quant, pkg.INTERLACED_HL_INTEGRATED, fmt)
            if fmt == pkg.PIXEL_PLANAR16:
                pu.check_planes(b, a, "mode 2 vs mode 1")
            else:
                assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ (e) batch and state
def test_batch_of_four_in_one_launch(pkg, ctx):
    """4 distinct frames in one mode-2 launch equal each frame decoded alone; frames 0 and 3 equal the oracle."""
    w, h = 720, 480
    rng = np.random.default_rng(44)
    frames = [interlaced_frame(rng, w, h, "natural", shift=4 + 2 * i) for i in range(4)]
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    table, prescale = quant.table(3), tuple(quant.prescale)
    qs = forward_bands(pkg, ctx, frames, quant)
    forms = [decoder_form(q, table) for q in qs]
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    with pkg.Codec(ctx, desc, 4) as codec:
        codec.set_interlaced(pkg.INTERLACED_HL_INTEGRATED)
        coded = [codec.pack_coded(b) for b in forms]
        p16 = [np.zeros((3 * h, w), np.int16) for _ in range(4)]
        p8 = [np.zeros((h, 2 * w), np.uint8) for _ in range(4)]
        codec.inverse_host(coded, unit, pkg.PIXEL_PLANAR16, p16)
        codec.inverse_host(coded, unit, pkg.PIXEL_YUYV, p8)
        for i in range(4):
            one16 = decode(pkg, codec, forms[i], unit, pkg.INTERLACED_HL_INTEGRATED, pkg.PIXEL_PLANAR16)
            one8 = decode(pkg, codec, forms[i], unit, pkg.INTERLACED_HL_INTEGRATED, pkg.PIXEL_YUYV)
            batch16 = [p16[i][0:h, :w], p16[i][h:2 * h, :w // 2], p16[i][2 * h:3 * h, :w // 2]]
            pu.check_planes(batch16, one16, f"frame {i}")
            assert np.array_equal(p8[i], one8), f"frame {i}"
            if i in (0, 3):
                pu.check_planes(one16, pu.inverse_pyramid(ol.oracle(), qs[i], table, prescale, interlaced=True), f"frame {i} oracle")


def test_mode_switches_leave_no_state(pkg, ctx):
    """One codec switched 0 -> 1 -> 2 -> 1 -> 0 over two different frames: every decode equals the oracle of its own mode
    and frame, so no carry of an earlier call is read (mode 1 after mode 2 must recompute them)."""
    w, h = 720, 480
    rng = np.random.default_rng(45)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    table, prescale = quant.table(3), tuple(quant.prescale)
    qs = forward_bands(pkg, ctx, [interlaced_frame(rng, w, h, "natural", shift=s) for s in (4, 10)], quant)
    orc = ol.oracle()
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    with pkg.Codec(ctx, desc, 1) as codec:
        for step, (mode, f) in enumerate([(pkg.PROGRESSIVE, 0), (pkg.INTERLACED, 1), (pkg.INTERLACED_HL_INTEGRATED, 0),
                                          (pkg.INTERLACED, 0), (pkg.PROGRESSIVE, 1)]):
            want = pu.inverse_pyramid(orc, qs[f], table, prescale, interlaced=mode != pkg.PROGRESSIVE)
            if mode == pkg.INTERLACED_HL_INTEGRATED:
                bands, qt = decoder_form(qs[f], table), unit
            else:
                bands, qt = qs[f], quant
            pu.check_planes(decode(pkg, codec, bands, qt, mode, pkg.PIXEL_PLANAR16), want, f"step {step}, mode {mode}, frame {f}")


# ------------------------------------------------------------------------------------------------ (f) reduced resolution
@pytest.mark.parametrize("size", [(720, 480), (1920, 1080)])
def test_reduced_resolution(pkg, ctx, size):
    """Half and quarter decodes in mode 2 (decoder form, unit divisors) equal mode 1 (coded bands, real quant) and the
    oracle's lowpass images LL1 / LL2, which do not depend on the level-1 transform."""
    w, h = size
    rng = np.random.default_rng(w + h)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    table, prescale = quant.table(3), tuple(quant.prescale)
    q = forward_bands(pkg, ctx, [interlaced_frame(rng, w, h, "natural")], quant)[0]
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    with pkg.Codec(ctx, desc, 1) as codec:
        for res, stop in ((pkg.RESOLUTION_HALF, 1), (pkg.RESOLUTION_QUARTER, 2)):
            lows = pu.inverse_pyramid(ol.oracle(), q, table, prescale, stop_level=stop)
            lows8 = pu.lowpass_to_422(lows, unsigned_shift=(stop == 2))
            codec.set_decode_resolution(res)
            rw, rh = codec.decoded_size()
            pitch = (2 * rw + 15) // 16 * 16            # output rows start 16-byte aligned (720 / 4 = 180 pixels: 360 bytes)
            for name, bands, qt, mode in (("mode 1", q, quant, pkg.INTERLACED),
                                          ("mode 2", decoder_form(q, table), unit, pkg.INTERLACED_HL_INTEGRATED)):
                codec.set_interlaced(mode)
                coded = codec.pack_coded(bands)
                pl = np.zeros((3 * rh, pitch // 2), np.int16)
                codec.inverse_host([coded], qt, pkg.PIXEL_PLANAR16, [pl])
                pu.check_planes([pl[0:rh, :rw], pl[rh:2 * rh, :rw // 2], pl[2 * rh:3 * rh, :rw // 2]], lows, f"{name} lowpass {stop}")
                out = np.zeros((rh, pitch), np.uint8)
                codec.inverse_host([coded], qt, pkg.PIXEL_YUYV, [out])
                assert np.array_equal(out[:, :2 * rw], lows8), f"{name} reduced-resolution frame {stop}"


# ------------------------------------------------------------------------------------------------ (g) GOP-2
@pytest.mark.parametrize("size", [(704, 96), (1920, 1080)])
def test_gop2_integrated_hl(pkg, ctx, size):
    """Interlaced two-frame GOP: the oracle's FIELDPLUS composition, decoded by cfb_gop2_inverse_host in mode 1, and the
    same pyramid with the wavelet-0 and wavelet-1 HL bands integrated, decoded in mode 2, give the same bytes."""
    w, h = size
    rng = np.random.default_rng(w + h + 1)
    fa = pu.synthetic_yuyv(rng, w, h, "natural")
    fb = np.roll(fa, 2, axis=0).copy()
    fb[:, 0::2] = np.clip(fb[:, 0::2].astype(np.int32) + rng.integers(-3, 4, (h, w)), 16, 235).astype(np.uint8)
    for f in (fa, fb):
        f[1::2] = np.roll(f[1::2], 8, axis=1)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    gq = pkg.gop2_quant_for_quality(desc, 4, True)
    quant = [[[int(gq.divisor[c][k][b]) for b in range(4)] for k in range(6)] for c in range(3)]
    prescale = [[int(v) for v in gq.prescale] + [0, 0]] * 3
    orc = ol.oracle()
    _, temporal, level = _oracle_blocks()
    want = pu.gop2_pyramid(lambda f, c, qq: orc.fwd_fields_422(f, c, 0, qq, 10, 2), temporal, level, fa, fb, quant, prescale)
    with pkg.Codec(ctx, desc, 2) as codec:
        g = codec.gop2_layout()
        coded = np.zeros(g.coded_bytes, np.uint8)
        for (c, k, b), v in want.items():
            if k != 2:
                codec.gop2_band_view(g, coded, c, k, b)[:] = v
        codec.set_interlaced(pkg.INTERLACED)
        a1, b1 = codec.gop2_inverse_host(coded, gq, pkg.PIXEL_YUYV, fa.shape)
        integ = coded.copy()
        for c in range(3):
            for k in (0, 1):
                view = codec.gop2_band_view(g, integ, c, k, 2)
                view[:] = pu.integrate_hl(view.copy())
        codec.set_interlaced(pkg.INTERLACED_HL_INTEGRATED)
        a2, b2 = codec.gop2_inverse_host(integ, gq, pkg.PIXEL_YUYV, fa.shape)
    assert np.array_equal(a2, a1) and np.array_equal(b2, b1)
    assert pu.psnr(a1[:, 0::2], fa[:, 0::2]) > 40.0 and pu.psnr(b1[:, 0::2], fb[:, 0::2]) > 40.0


# ------------------------------------------------------------------------------------------------ (h) pool
def test_pool_mode2_dense_and_sparse(pkg, ctx):
    """Pool.set_interlaced(INTERLACED_HL_INTEGRATED): dense and sparse inverse jobs of decoder-form bands give the bytes
    of the synchronous codec in mode 2."""
    w, h, n = 720, 480, 4
    rng = np.random.default_rng(46)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    qs = forward_bands(pkg, ctx, [interlaced_frame(rng, w, h, "natural", shift=2 + 2 * i) for i in range(n)], quant)
    forms = [decoder_form(q, quant.table(3)) for q in qs]
    unit = pkg.make_quant(pu.UNIT_DIVISORS, tuple(quant.prescale))
    with pkg.Codec(ctx, desc, 1) as codec:
        want = [decode(pkg, codec, b, unit, pkg.INTERLACED_HL_INTEGRATED, pkg.PIXEL_YUYV) for b in forms]
    with pkg.Pool([0], desc, slots=2, batch=2, queue_length=2 * n) as pool:
        pool.set_interlaced(pkg.INTERLACED_HL_INTEGRATED)
        lay = pool.layout
        dense, sparse = [], []
        for b in forms:
            d = pkg.pack_coded(lay, b)
            s = pkg.sparse_compact(lay, d)
            dense.append(pkg.pinned_empty(d.size)); dense[-1][:] = d
            sparse.append(pkg.pinned_empty(s.size)); sparse[-1][:] = s
        out_d = [pkg.pinned_empty((h, 2 * w)) for _ in range(n)]
        out_s = [pkg.pinned_empty((h, 2 * w)) for _ in range(n)]
        for i in range(n):
            pool.submit_inverse(2 * i, dense[i], unit, pkg.PIXEL_YUYV, out_d[i])
            pool.submit_inverse_sparse(2 * i + 1, sparse[i], unit, pkg.PIXEL_YUYV, out_s[i])
        assert [pool.wait() for _ in range(2 * n)] == list(range(2 * n))
    for i in range(n):
        assert np.array_equal(np.asarray(out_d[i]), want[i]), f"dense job {i}"
        assert np.array_equal(np.asarray(out_s[i]), want[i]), f"sparse job {i}"


# ------------------------------------------------------------------------------------------------ (i) sparse hand-over
def band_buffers(layout, bands, rng):
    """Each band in a buffer of its own, as the reference's decoder leaves wavelet->band[]: a row pitch wider than the
    layout's and garbage behind the band's width.  Returns views whose row stride is that pitch."""
    out = {}
    for c in range(3):
        for k in range(3):
            for b in range(4):
                if b == 0 and k != 2:
                    continue
                key = (c, k + 1, pu.BAND_NAMES[b])
                bl = layout.band[c][k][b]
                buf = rng.integers(-999, 999, (bl.height, bl.pitch // 2 + 8 * (1 + (c + k + b) % 3))).astype(np.int16)
                buf[:, :bl.width] = bands[key]
                out[key] = buf[:, :bl.width]
    return out


def _coded_region(bands):
    return {k: v for k, v in bands.items() if not (k[2] == "LL" and k[1] != 3)}


HANDOVER = GOLDEN + GOLDEN_FIELDS


@pytest.mark.parametrize("path", HANDOVER, ids=[os.path.basename(p) for p in HANDOVER])
def test_sparse_handover_of_decoder_bands(pkg, ctx, path):
    """The shim's CFHD_B200_DECODE_SPARSE hand-over: the golden decoder bands in per-band buffers, compacted by
    cfb_sparse_compact_bands and decoded by cfb_inverse_host_sparse, give byte for byte what cfb_inverse_host gives for the
    packed dense region (progressive fixtures in mode 0, interlaced ones in mode 2), for YUYV and PLANAR16; PLANAR16 also
    equals the oracle."""
    interlaced = path in GOLDEN_FIELDS
    frame, _, prescale, _, _ = load_golden(path)
    bands, _ = load_golden_decoder_side(path)
    bands = _coded_region(bands)
    h, w = frame.shape[0], frame.shape[1] // 2
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    want = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, prescale, interlaced=interlaced, hl_integrated=True)
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_interlaced(pkg.INTERLACED_HL_INTEGRATED if interlaced else pkg.PROGRESSIVE)
        lay = codec.layout
        sp = pkg.sparse_compact_bands(lay, band_buffers(lay, bands, np.random.default_rng(w + h)))
        dense = pkg.pack_coded(lay, bands)
        assert np.array_equal(pkg.sparse_expand(lay, sp), dense)
        for fmt, shape, dtype in ((pkg.PIXEL_YUYV, (h, 2 * w), np.uint8), (pkg.PIXEL_PLANAR16, (3 * h, w), np.int16)):
            out_d, out_s = np.zeros(shape, dtype), np.zeros(shape, dtype)
            codec.inverse_host([dense], unit, fmt, [out_d])
            codec.inverse_host_sparse([sp], unit, fmt, [out_s])
            assert np.array_equal(out_s, out_d), f"format {fmt}"
        pu.check_planes([out_d[0:h, :w], out_d[h:2 * h, :w // 2], out_d[2 * h:3 * h, :w // 2]], want, "PLANAR16")


@pytest.mark.parametrize("path", GOLDEN_FIELDS[-1:], ids=[os.path.basename(p) for p in GOLDEN_FIELDS[-1:]])
def test_sparse_handover_batch_of_three(pkg, ctx, path):
    """Three distinct band sets (the golden decoder bands, two with sparse perturbations of every highpass band) handed
    over as per-band buffers and decoded in one sparse mode-2 launch equal the dense batch and each dense frame alone."""
    frame, _, prescale, _, _ = load_golden(path)
    bands, _ = load_golden_decoder_side(path)
    bands = _coded_region(bands)
    h, w = frame.shape[0], frame.shape[1] // 2
    rng = np.random.default_rng(47)
    sets = [bands]
    for _ in range(2):
        b2 = dict(bands)
        for key, v in bands.items():
            if key[2] != "LL":
                b2[key] = np.where(rng.random(v.shape) < 0.03, v + rng.integers(-60, 60, v.shape), v).astype(np.int16)
        sets.append(b2)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    unit = pkg.make_quant(pu.UNIT_DIVISORS, prescale)
    with pkg.Codec(ctx, desc, 3) as codec:
        codec.set_interlaced(pkg.INTERLACED_HL_INTEGRATED)
        lay = codec.layout
        sp = [pkg.sparse_compact_bands(lay, band_buffers(lay, b, rng)) for b in sets]
        dense = [pkg.pack_coded(lay, b) for b in sets]
        out_d = [np.zeros((h, 2 * w), np.uint8) for _ in range(3)]
        out_s = [np.zeros((h, 2 * w), np.uint8) for _ in range(3)]
        codec.inverse_host(dense, unit, pkg.PIXEL_YUYV, out_d)
        codec.inverse_host_sparse(sp, unit, pkg.PIXEL_YUYV, out_s)
        for i in range(3):
            one = np.zeros((h, 2 * w), np.uint8)
            codec.inverse_host([dense[i]], unit, pkg.PIXEL_YUYV, [one])
            assert np.array_equal(out_s[i], one) and np.array_equal(out_d[i], one), f"frame {i}"
        assert not np.array_equal(out_s[0], out_s[1]) and not np.array_equal(out_s[1], out_s[2])
