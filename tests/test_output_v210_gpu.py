"""V210 output of the final 4:2:2 inverse level on the GPU (k_inv_422_tma, V210 instantiation): byte-identical to the
reference decoder's frames (golden fixtures, X masked) and to formats.pack_v210_output of the oracle's planes (X = Cb1
included), from YUYV, UYVY, YU64 and V210 codecs; consistent with the library's own YU64 output; bit-exact at every
rows-per-warp split, with padding and rows past the frame untouched (every entry point: test_entry_points_gpu.py); the
documented rejections; one launch for the final level."""
import glob
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import TH, ctx, pkg  # noqa: F401

pytestmark = pytest.mark.gpu

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decoded_v210_*.npz")))


def _decode(codec, pkg, coded, quant, w, h, pitch=None):
    """Host-API V210 decode of one coded buffer into a CANARY-filled (h + 2, pitch) buffer; returns (words, buffer)."""
    pitch = pitch or fm.v210_natural_pitch(w)
    buf = np.full((h + 2, pitch), fm.CANARY, np.uint8)
    codec.inverse_host([coded], quant, pkg.PIXEL_V210, [buf])
    return fm.v210_frame_words(buf[:h], w, h), buf


def _assert_words(got, want, what):
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{what}: {bad.shape[0]} words differ, first (row, word) {bad[:5].tolist()}"


def _assert_untouched(buf, w, h, what):
    assert (buf[:h, fm.v210_row_bytes(w):] == fm.CANARY).all(), f"{what}: row padding written"
    assert (buf[h:] == fm.CANARY).all(), f"{what}: rows past the frame written"


def _source(pkg, orc, fmt, w, h, kind, rng):
    """Coded-region bands of a frame in source format `fmt` (oracle forward) and that codec's quantisation."""
    desc = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + fmt))
    quant = pkg.quant_for_quality(desc, 4)
    frame = pu.synthetic_yuyv(rng, w, h, kind)
    table, prescale = quant.table(3), tuple(quant.prescale)
    if fmt in ("YUYV", "UYVY"):
        return desc, quant, pu.oracle_forward_422(orc, frame if fmt == "YUYV" else fm.yuyv_to_uyvy(frame), quant, int(fmt == "UYVY"))
    planes = fm.unpack_yu64(fm.yu64_from_yuyv(frame, rng)) if fmt == "YU64" else fm.v210_from_yuyv(frame, rng)[1]
    pyr = pu.forward_pyramid_planes(orc, planes, table, prescale, quant.midpoint_prequant)
    return desc, quant, {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}


# ------------------------------------------------------------------------------------------------ reference frames
def test_golden_present():
    assert len(GOLDEN) == 3


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_golden_bands_give_reference_frame(pkg, ctx, path):
    z = np.load(path)
    w, h = int(z["width"]), int(z["height"])
    bands = {(int(c), int(k), b): z[key] for key in z.files if key.startswith("d_") for c, k, b in [key.split("_")[1:]]}
    unit = pkg.make_quant(pu.UNIT_DIVISORS, [int(v) for v in z["prescale"]])
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), 1) as codec:
        got, buf = _decode(codec, pkg, codec.pack_coded(bands), unit, w, h)
    m = fm.v210_x_mask(w)
    _assert_words(got & m, fm.v210_frame_words(z["frame"], w, h) & m, os.path.basename(path))
    _assert_untouched(buf, w, h, os.path.basename(path))


# ------------------------------------------------------------------------------------------------ oracle parity
SIZES = [(192, 48), (208, 48), (720, 480), (1280, 720), (1440, 1080), (1920, 1080), (2048, 1080), (4096, 2160)]


@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
@pytest.mark.parametrize("fmt", ["YUYV", "UYVY", "YU64", "V210"])
def test_v210_output_vs_oracle(pkg, ctx, fmt, size):
    """Also the cross-check: on every whole group the V210 words are the library's own YU64 samples >> 6."""
    w, h = size
    if fmt == "V210" and w % 48:
        pytest.skip("V210 sources are multiples of 48 pixels wide")
    rng = np.random.default_rng(w + 7 * h)
    orc = ol.oracle()
    kinds = ["natural", "extreme"] if (fmt == "YUYV" and w * h <= 720 * 480) else ["natural"]
    for kind in kinds:
        desc, quant, bands = _source(pkg, orc, fmt, w, h, kind, rng)
        want = fm.pack_v210_output(pu.inverse_pyramid(orc, bands, quant.table(3), tuple(quant.prescale)))
        with pkg.Codec(ctx, desc, 1) as codec:
            coded = codec.pack_coded(bands)
            got, buf = _decode(codec, pkg, coded, quant, w, h)
            yu64 = np.zeros((h, 2 * w), np.uint16)
            codec.inverse_host([coded], quant, pkg.PIXEL_YU64, [yu64])
        _assert_words(got, want, f"{fmt} {w}x{h} {kind}")
        _assert_untouched(buf, w, h, f"{fmt} {w}x{h} {kind}")
        full = 4 * (w // 6)
        own = fm.pack_v210_components(yu64[:, 0::2] >> 6, yu64[:, 1::4] >> 6, yu64[:, 3::4] >> 6)
        _assert_words(got[:, :full], own[:, :full], f"{fmt} {w}x{h} {kind} vs YU64 >> 6")


def test_4k_batch_of_16(pkg, ctx):
    """16 distinct 3840x2160 frames decoded to V210 in one batch (frame 15 uses the batch's last tensor maps): every frame
    equals the same frame decoded alone, frames 0 and 15 equal the oracle."""
    w, h, n = 3840, 2160, 16
    rng = np.random.default_rng(5)
    base = pu.synthetic_yuyv(rng, w, h, "natural")
    frames = [np.roll(base, (8 * i, 64 * i), axis=(0, 1)).copy() for i in range(n)]
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    pitch = fm.v210_natural_pitch(w)
    with pkg.Codec(ctx, desc, n) as codec:
        coded = codec.forward_host(frames, quant)
        outs = [np.full((h, pitch), fm.CANARY, np.uint8) for _ in range(n)]
        codec.inverse_host(coded, quant, pkg.PIXEL_V210, outs)
        for i in range(n):
            alone, _ = _decode(codec, pkg, coded[i], quant, w, h)
            _assert_words(fm.v210_frame_words(outs[i], w, h), alone, f"frame {i} batch vs alone")
        for i in (0, n - 1):
            bands = codec.unpack_coded(coded[i])
            want = fm.pack_v210_output(pu.inverse_pyramid(orc, bands, quant.table(3), tuple(quant.prescale)))
            _assert_words(fm.v210_frame_words(outs[i], w, h), want, f"frame {i} vs oracle")


# ------------------------------------------------------------------------------------------------ rows per warp
@pytest.mark.parametrize("size", [(1024, 136), (720, 200), (208, 56), (224, 56), (1920, 1080)])
def test_v210_at_every_split(pkg, ctx, monkeypatch, size):
    """Level-1 band heights 68 / 100 / 28 / 28 / 540 lie on both sides of every th; widths cover W % 6 = 4, 0, 4, 2, 0."""
    w, h = size
    rng = np.random.default_rng(w + h)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    bands = pu.oracle_forward_422(orc, pu.synthetic_yuyv(rng, w, h, "random"), quant, 0)
    want = fm.pack_v210_output(pu.inverse_pyramid(orc, bands, quant.table(3), tuple(quant.prescale)))
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(bands)
        for th in TH:
            monkeypatch.setenv("CFB_TH", str(th))
            got, buf = _decode(codec, pkg, coded, quant, w, h)
            _assert_words(got, want, f"{w}x{h} th={th}")
            _assert_untouched(buf, w, h, f"{w}x{h} th={th}")


# ------------------------------------------------------------------------------------------------ rejections, launches
def test_rejections_leave_the_context_usable(pkg, ctx):
    import torch
    w, h = 208, 48
    rng = np.random.default_rng(1)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    bands = pu.oracle_forward_422(orc, pu.synthetic_yuyv(rng, w, h, "natural"), quant, 0)
    want = fm.pack_v210_output(pu.inverse_pyramid(orc, bands, quant.table(3), tuple(quant.prescale)))

    def code_of(fn):
        with pytest.raises(pkg.CfbError) as ei:
            fn()
        return ei.value.code

    # a codec that is not 4:2:2
    rdesc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    with pkg.Codec(ctx, rdesc, 1) as rc:
        rq = pkg.quant_for_quality(rdesc, 4)
        out = np.zeros((h, fm.v210_natural_pitch(w)), np.uint8)
        assert code_of(lambda: rc.inverse_host([np.zeros(rc.layout.coded_bytes, np.uint8)], rq, pkg.PIXEL_V210, [out])) == 3
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(bands)
        # reduced resolution and interlaced decodes
        for res in (pkg.RESOLUTION_HALF, pkg.RESOLUTION_QUARTER):
            codec.set_decode_resolution(res)
            try:
                rw, rh = codec.decoded_size()
                out = np.zeros((rh, fm.v210_natural_pitch(rw)), np.uint8)
                assert code_of(lambda: codec.inverse_host([coded], quant, pkg.PIXEL_V210, [out])) == 102
            finally:
                codec.set_decode_resolution(pkg.RESOLUTION_FULL)
        codec.set_interlaced(True)
        try:
            out = np.zeros((h, fm.v210_natural_pitch(w)), np.uint8)
            assert code_of(lambda: codec.inverse_host([coded], quant, pkg.PIXEL_V210, [out])) == 102
        finally:
            codec.set_interlaced(False)
        # pitches below ceil(W / 6) * 16 or not a multiple of 16
        d_pyr = torch.zeros(codec.layout.total_bytes, dtype=torch.uint8, device="cuda")
        d_pyr[:coded.size] = torch.from_numpy(coded).cuda()
        d_out = torch.full((h * 2 * fm.v210_natural_pitch(w),), fm.CANARY, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        for pitch in (fm.v210_row_bytes(w) - 16, fm.v210_row_bytes(w) + 8):
            assert code_of(lambda: codec.inverse_device([d_pyr.data_ptr()], quant, pkg.PIXEL_V210, [d_out.data_ptr()], pitch)) == 1
        out = np.zeros((h, fm.v210_row_bytes(w) - 16), np.uint8)
        assert code_of(lambda: codec.inverse_host([coded], quant, pkg.PIXEL_V210, [out])) == 1
        ctx.synchronize()
        assert (d_out.cpu().numpy() == fm.CANARY).all()
        # still usable: the smallest legal pitch works and gives the oracle's bytes
        got, buf = _decode(codec, pkg, coded, quant, w, h, pitch=fm.v210_row_bytes(w))
        _assert_words(got, want, "after the rejections")


def test_final_level_is_one_launch(pkg, ctx):
    w, h = 720, 96
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    bands = pu.oracle_forward_422(ol.oracle(), pu.synthetic_yuyv(np.random.default_rng(2), w, h, "natural"), quant, 0)
    with pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.pack_coded(bands)
        out = np.zeros((h, fm.v210_natural_pitch(w)), np.uint8)
        deltas = {}
        for mask in (1, 7):
            codec.set_level_mask(7, mask)
            for fmt in (pkg.PIXEL_V210, pkg.PIXEL_YU64):
                o = out if fmt == pkg.PIXEL_V210 else np.zeros((h, 2 * w), np.uint16)
                before = ctx.stats()["kernel_launches"]
                codec.inverse_host([coded], quant, fmt, [o])
                deltas[(mask, fmt)] = ctx.stats()["kernel_launches"] - before
        codec.set_level_mask(7, 7)
    assert deltas[(1, pkg.PIXEL_V210)] == 1
    assert deltas[(7, pkg.PIXEL_V210)] == deltas[(7, pkg.PIXEL_YU64)]
