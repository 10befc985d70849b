"""BYR4 output of the final inverse level on the GPU (k_inv_444, BYR4 instantiation: four channels, the Bayer reconstruction
fused into the writer): byte-identical to the reference decoder's frames (golden fixtures of make_golden_byr4_out.py) and to the
oracle's "bands -> mosaic" (formats.oracle_byr4) in all four phases and both curve modes, from BYR4 and BYR5 codecs, with
both dequantiser paths, at every rows-per-warp split, in batches, with a padded pitch left untouched (every entry point:
test_entry_points_gpu.py); the encode -> decode round trip; the documented rejections."""
import glob
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import TH, ctx, pkg  # noqa: F401
from test_output_byr4 import fixture_bands
from test_quant_tables import table as quant_table


pytestmark = pytest.mark.gpu

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decoded_byr4_*.npz")))
RESTORE = fm.restore_table()


def _decode(codec, pkg, coded, quant, w, h, phase, restore, pitch=None):
    """Host-API BYR4 decode of one coded buffer into a fm.CANARY-filled (h + 2, pitch) byte buffer; returns (mosaic, buffer)."""
    pitch = pitch or 2 * w
    buf = np.full((h + 2, pitch), fm.CANARY, np.uint8)
    codec.set_bayer_phase(phase)
    codec.set_bayer_decode_curve(restore)
    codec.inverse_host([coded], quant, pkg.PIXEL_BYR4, [buf])
    return np.ascontiguousarray(buf[:h, :2 * w]).view(np.uint16), buf


def _assert_mosaic(got, want, what):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {bad.shape[0]} samples differ, first (row, column) {bad[:5].tolist()}, "
                           f"got {got[tuple(bad[0])] if bad.size else 0} want {want[tuple(bad[0])] if bad.size else 0}")


def _assert_untouched(buf, w, h, what):
    assert (buf[:h, 2 * w:] == fm.CANARY).all(), f"{what}: row padding written"
    assert (buf[h:] == fm.CANARY).all(), f"{what}: rows past the frame written"


def _coded_bands(mosaic, phase, table, prescale):
    """Coded-region bands of a BYR4 mosaic (curve applied: samples >> 4) by the oracle's forward pyramid."""
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_byr4(mosaic, phase), table, prescale)
    return {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}


# ------------------------------------------------------------------------------------------------ reference frames
def test_golden_present():
    assert len(GOLDEN) == 4


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
@pytest.mark.parametrize("source", ["BYR4", "BYR5"])
def test_golden_bands_give_reference_frame(pkg, ctx, path, source):
    """The bands the reference decoder held -> its own frame, from a codec of either Bayer source.  208 x 100: the codec has
    the coded height 112, the reference wrote the first 100 rows."""
    z = np.load(path)
    w, h, ch = int(z["width"]), int(z["height"]), int(z["coded_height"])
    phase, preset = int(z["phase"]), int(z["preset"])
    unit = pkg.make_quant(fm.UNIT4, [int(v) for v in z["prescale"]])
    with pkg.Codec(ctx, pkg.FrameDesc(w, ch, getattr(pkg, "PIXEL_" + source)), 1) as codec:
        got, buf = _decode(codec, pkg, codec.pack_coded(fixture_bands(z)), unit, w, ch, phase, z["restore"] if preset == 0 else None)
    _assert_mosaic(got[:h], z["frame"], os.path.basename(path))
    _assert_untouched(buf, w, ch, os.path.basename(path))


# ------------------------------------------------------------------------------------------------ oracle parity
# mosaic sizes: one strip, ragged strips (plane widths 104, 360, 1352), two and more strips, 4K and 8K
CASES = [((192, 96), "random", "small"), ((208, 96), "extreme", "big"), ((720, 112), "random", "big"), ((512, 128), "constant", "small"),
         ((2704, 160), "extreme", "small"), ((3840, 2160), "natural", None), ((8192, 4320), "natural", None)]


@pytest.mark.parametrize("size,kind,tab", CASES, ids=[f"{s[0]}x{s[1]}-{k}-{t}" for s, k, t in CASES])
def test_byr4_output_vs_oracle(pkg, ctx, size, kind, tab):
    """4 phases x 2 curve modes (the large sizes: one combination each), the codec's own quantisation (tab None) or the tables
    of test_quant_tables (T_small: every divisor <= 255, the dp2a dequantiser; T_big: the full multiply), a padded pitch."""
    w, h = size
    rng = np.random.default_rng(w + 3 * h)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4) if tab is None else pkg.make_quant(quant_table(tab, 4), [0, 2, 2])
    table, prescale = quant.table(4), tuple(quant.prescale)
    combos = [(p, r) for p in range(4) for r in (None, RESTORE)] if w < 3840 else [(1, RESTORE)] if w == 8192 else [(2, None)]
    pitch = 2 * w + (0 if w >= 3840 else 48)
    with pkg.Codec(ctx, desc, 1) as codec:
        for phase, restore in combos:
            bands = _coded_bands(fm.synthetic_mosaic(rng, w, h, kind, phase), phase, table, prescale)
            want = fm.oracle_byr4(bands, table, prescale, phase, restore)
            got, buf = _decode(codec, pkg, codec.pack_coded(bands), quant, w, h, phase, restore, pitch)
            what = f"{w}x{h} {kind} phase {phase} {'restore' if restore is not None else 'applied'}"
            _assert_mosaic(got, want, what)
            _assert_untouched(buf, w, h, what)


@pytest.mark.parametrize("size", [(2048, 272), (1440, 400), (416, 112)])
def test_byr4_output_at_every_split(pkg, ctx, monkeypatch, size):
    """Level-1 band heights 68 / 100 / 28 lie on both sides of every th."""
    w, h = size
    rng = np.random.default_rng(w + h)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(4), tuple(quant.prescale)
    bands = _coded_bands(fm.synthetic_mosaic(rng, w, h, "random"), 3, table, prescale)
    wants = {mode: fm.oracle_byr4(bands, table, prescale, 3, restore) for mode, restore in (("applied", None), ("restore", RESTORE))}
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(bands)
        for th in TH:
            monkeypatch.setenv("CFB_TH", str(th))
            for mode, want in wants.items():
                got, buf = _decode(codec, pkg, coded, quant, w, h, 3, RESTORE if mode == "restore" else None)
                _assert_mosaic(got, want, f"{w}x{h} th={th} {mode}")
                _assert_untouched(buf, w, h, f"{w}x{h} th={th} {mode}")


@pytest.mark.parametrize("source", ["BYR4", "BYR5"])
def test_batch_of_4_equals_each_alone(pkg, ctx, source):
    w, h, n, phase = 1040, 112, 4, 2
    rng = np.random.default_rng(44)
    desc = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + source))
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(4), tuple(quant.prescale)
    kinds = ("random", "extreme", "natural", "random")
    with pkg.Codec(ctx, desc, n) as codec:
        bands = [_coded_bands(fm.synthetic_mosaic(rng, w, h, k, phase), phase, table, prescale) for k in kinds]
        coded = [codec.pack_coded(b) for b in bands]
        codec.set_bayer_phase(phase)
        codec.set_bayer_decode_curve(RESTORE)
        outs = [np.zeros((h, w), np.uint16) for _ in range(n)]
        codec.inverse_host(coded, quant, pkg.PIXEL_BYR4, outs)
        for i in range(n):
            alone, _ = _decode(codec, pkg, coded[i], quant, w, h, phase, RESTORE)
            _assert_mosaic(outs[i], alone, f"{source} frame {i} batch vs alone")
            _assert_mosaic(outs[i], fm.oracle_byr4(bands[i], table, prescale, phase, RESTORE), f"{source} frame {i} vs oracle")


# ------------------------------------------------------------------------------------------------ round trip
def test_round_trip_on_the_gpu(pkg, ctx):
    """BYR4 in, BYR4 out, curve applied by the application: the GPU's bands and mosaic are the oracle's.  What can be derived
    about the distance to the source: a constant mosaic comes back as v & 0xfff0 exactly (constant planes have zero highpass
    bands at every level, which quantise to zero, and the lowpass chain of a constant is exact; 12 bits survive), and where no
    sample saturates every output sample is a multiple of 16 (sums of 12-bit samples << 4).  The quantiser's error on other
    content has no bound derived here, so none is asserted."""
    w, h = 720, 112
    rng = np.random.default_rng(9)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(4), tuple(quant.prescale)
    with pkg.Codec(ctx, desc, 1) as codec:
        for phase in range(4):
            src = fm.synthetic_mosaic(rng, w, h, "natural", phase)
            codec.set_bayer_phase(phase)
            coded = codec.forward_host([src], quant)[0]
            bands = _coded_bands(src, phase, table, prescale)
            pu.assert_bands(codec.unpack_coded(coded), bands, f"phase {phase}")
            got, _ = _decode(codec, pkg, coded, quant, w, h, phase, None)
            _assert_mosaic(got, fm.oracle_byr4(bands, table, prescale, phase, None), f"round trip phase {phase}")
            assert got.max() < 65520 and got.min() > 0 and (got % 16 == 0).all()
        for v in (0, 0x0230, 0x8120, 0xffff):
            got, _ = _decode(codec, pkg, codec.forward_host([np.full((h, w), v, np.uint16)], quant)[0], quant, w, h, 3, None)
            assert (got == (v & 0xfff0)).all(), hex(v)


# ------------------------------------------------------------------------------------------------ rejections, launches
def test_rejections_leave_the_codec_usable(pkg, ctx):
    """What the BYR4 output does not cover is refused by the checks every output goes through: another codec family
    CFB_ERROR_BADFORMAT (3), as for every family-bound output; reduced resolution, the two-frame GOP and outputs the library
    does not write CFB_ERROR_UNSUPPORTED (102); a bad pitch or table CFB_ERROR_INVALID_ARGUMENT (1)."""
    w, h = 208, 96
    rng = np.random.default_rng(1)

    def code_of(fn):
        with pytest.raises(pkg.CfbError) as ei:
            fn()
        return ei.value.code

    # BYR4 out of codecs that are not Bayer, and the decode curve on them
    for fmt in ("YUYV", "RG48"):
        d = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + fmt))
        with pkg.Codec(ctx, d, 1) as c:
            q = pkg.quant_for_quality(d, 4)
            out = np.zeros((h, w), np.uint16)
            assert code_of(lambda: c.inverse_host([np.zeros(c.layout.coded_bytes, np.uint8)], q, pkg.PIXEL_BYR4, [out])) == 3, fmt
            assert code_of(lambda: c.set_bayer_decode_curve(RESTORE)) == 3, fmt
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(4), tuple(quant.prescale)
    bands = _coded_bands(fm.synthetic_mosaic(rng, w, h, "random"), 1, table, prescale)
    want = fm.oracle_byr4(bands, table, prescale, 1, RESTORE)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(bands)
        # 4:2:2 / 4:4:4 outputs from a Bayer codec (RG48: the host form finds first that 6 W H bytes do not fit the frame
        # staging); BYR5 is input only
        for fmt, shape, code in (("YU64", (h, 2 * w), 3), ("RG48", (h, 3 * w), 102), ("B64A", (h, 4 * w), 3), ("V210", (h, 2 * w), 3)):
            out = np.zeros(shape, np.uint16)
            assert code_of(lambda: codec.inverse_host([coded], quant, getattr(pkg, "PIXEL_" + fmt), [out])) == code, fmt
        assert code_of(lambda: codec.inverse_host([coded], quant, pkg.PIXEL_BYR5, [np.zeros((h // 2, 3 * w), np.uint8)])) == 102
        # reduced resolution, interlaced (refused when set on a Bayer codec), two-frame GOP
        for res in (pkg.RESOLUTION_HALF, pkg.RESOLUTION_QUARTER):
            codec.set_decode_resolution(res)
            try:
                assert code_of(lambda: codec.inverse_host([coded], quant, pkg.PIXEL_BYR4, [np.zeros((h, w), np.uint16)])) == 102
            finally:
                codec.set_decode_resolution(pkg.RESOLUTION_FULL)
        assert code_of(lambda: codec.set_interlaced(pkg.INTERLACED)) == 102
        assert code_of(lambda: pkg.gop2_quant_for_quality(desc, 4)) == 102
        # pitches below 2 W or not a multiple of 16; a table of the wrong length
        assert code_of(lambda: codec.inverse_host([coded], quant, pkg.PIXEL_BYR4, [np.zeros((h, w - 8), np.uint16)])) == 1
        assert code_of(lambda: codec.set_bayer_decode_curve(RESTORE[:4096])) == 1
        assert code_of(lambda: codec.set_bayer_phase(4)) == 1
        # still usable
        got, buf = _decode(codec, pkg, coded, quant, w, h, 1, RESTORE)
        _assert_mosaic(got, want, "after the rejections")


def test_final_level_is_one_launch(pkg, ctx):
    w, h = 720, 112
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        codec.set_level_mask(7, 1)
        before = ctx.stats()["kernel_launches"]
        codec.inverse_host([coded], quant, pkg.PIXEL_BYR4, [np.zeros((h, w), np.uint16)])
        assert ctx.stats()["kernel_launches"] - before == 1
        codec.set_level_mask(7, 7)
