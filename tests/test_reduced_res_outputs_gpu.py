"""Reduced-resolution decodes to the deep outputs on the GPU (k_lowpass_422<YU64>, k_lowpass_444): YU64 at half resolution
from 4:2:2 codecs (progressive and interlaced), the 10-bit RGB words at quarter resolution from RGB 4:4:4 and RGBA 4:4:4:4
codecs.  Byte-identical to the reference decoder's frames (golden fixtures) and to the rules of formats.py on
the oracle's lowpass images, at batch sizes 1 and 3, with the bytes between the row and the pitch and the rows past the
frame untouched (every entry point: test_entry_points_gpu.py); one conversion launch; the combinations that stay
unsupported are refused."""
import glob
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401

pytestmark = pytest.mark.gpu

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reduced_*.npz")))
RGB10 = list(fm.RGB30_FORMATS)


def _rule(fmt, res, ll):
    return fm.OUTPUTS[fmt].reduced[res](ll).view(np.uint8)


def _case(pkg, codec_kind, w, h, kind, seed):
    """(desc, quant, coded-region bands, resolution) of an oracle-encoded frame.  codec_kind: "422", "422i" (interlaced),
    "444" (RG48 source) or "4444" (B64A source with alpha)."""
    rng = np.random.default_rng(seed)
    orc = ol.oracle()
    if codec_kind.startswith("422"):
        desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
        quant = pkg.quant_for_quality(desc, 4)
        bands = pu.oracle_forward_422(orc, pu.synthetic_yuyv(rng, w, h, kind), quant, 0, interlaced=codec_kind == "422i")
        return desc, quant, bands, fm.HALF
    if codec_kind == "4444":
        desc = pkg.FrameDesc(w, h, pkg.PIXEL_B64A, pkg.FRAME_ALPHA)
        quant = pkg.quant_for_quality(desc, 4)
        planes = fm.unpack_rgba64(fm.synthetic_rgba64(rng, w, h, "natural", "B64A"), "B64A", True)
        nc = 4
    else:
        desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
        quant = pkg.quant_for_quality(desc, 1 if kind == "blocks" else 4)
        frame = fm.block_rg48(w, h, 2, seed) if kind == "blocks" else fm.synthetic_rg48(rng, w, h, kind)
        planes = fm.unpack_rg48(frame)
        nc = 3
    pyr = pu.forward_pyramid_planes(orc, planes, quant.table(nc), tuple(quant.prescale), quant.midpoint_prequant)
    return desc, quant, {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}, fm.QUARTER


def _want(fmt, quant, bands, res, nc):
    planes = pu.inverse_pyramid(ol.oracle(), bands, quant.table(nc), tuple(quant.prescale), nchan=nc, stop_level=res - 1)
    return _rule(fmt, res, planes[:3])


def _buffers(n, rh, pitch):
    return [np.full((rh + 2, pitch), fm.CANARY, np.uint8) for _ in range(n)]


def _check(buf, want, what):
    rh, rb = want.shape
    bad = np.argwhere(buf[:rh, :rb] != want)
    assert bad.size == 0, f"{what}: {bad.shape[0]} bytes differ, first (row, byte) {bad[:5].tolist()}"
    assert (buf[:rh, rb:] == fm.CANARY).all(), f"{what}: bytes between the row and the pitch written"
    assert (buf[rh:] == fm.CANARY).all(), f"{what}: rows past the frame written"


CASES = [   # (output formats, codec kind, sizes)
    (["YU64"], "422", [(640, 96), (336, 48), (208, 48), (1920, 1080)]),
    (["YU64"], "422i", [(640, 96), (336, 48)]),
    (RGB10, "444", [(640, 96), (200, 64), (328, 48), (1016, 48), (3840, 2160)]),
    (RGB10, "4444", [(256, 64), (328, 48)]),
]
PARAMS = [(f, k, s) for fmts, k, sizes in CASES for s in sizes for f in [fmts]]


# ------------------------------------------------------------------------------------------------ reference frames
def test_golden_present():
    assert len(GOLDEN) == 2


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_golden_bands_give_reference_frame(pkg, ctx, path):
    z = np.load(path)
    w, h = int(z["width"]), int(z["height"])
    res = fm.HALF if "_half_" in path else fm.QUARTER
    src = pkg.PIXEL_YUYV if res == fm.HALF else pkg.PIXEL_RG48
    unit = pkg.make_quant(pu.UNIT_DIVISORS, [int(v) for v in z["prescale"]])
    with pkg.Codec(ctx, pkg.FrameDesc(w, h, src), 1) as codec:
        codec.set_decode_resolution(res)
        for fmt in sorted({k.split("_")[1] for k in z.files if k.startswith("frame_")}):
            bands = {(int(c), int(k), b): z[key] for key in z.files if key.startswith(f"d_{fmt}_")
                     for c, k, b in [key.split("_")[2:]]}
            want = z[f"frame_{fmt}"].view(np.uint8)
            buf = _buffers(1, want.shape[0], want.shape[1] + 32)[0]
            codec.inverse_host([codec.pack_coded(bands)], unit, getattr(pkg, "PIXEL_" + fmt), [buf])
            _check(buf, want, f"{os.path.basename(path)} {fmt}")


# ------------------------------------------------------------------------------------------------ oracle, batches
@pytest.mark.parametrize("fmts,codec_kind,size", PARAMS, ids=[f"{k}-{w}x{h}" for _, k, (w, h) in PARAMS])
def test_reduced_output_vs_oracle(pkg, ctx, fmts, codec_kind, size):
    """Batch 1 and a batch of 3 distinct frames, host API; the 4:4:4 frames at 640 x 96 and below also with LL2 beyond
    [0, 16383] on both sides (0 / 65535 blocks at quality 1)."""
    w, h = size
    kinds = ["natural", "blocks"] if codec_kind == "444" and w * h <= 640 * 96 else ["natural"]
    for kind in kinds:
        cases = [_case(pkg, codec_kind, w, h, kind, w + h + i) for i in range(3)]
        desc, quant, _, res = cases[0]
        nc = 4 if codec_kind == "4444" else 3
        with pkg.Codec(ctx, desc, 3) as codec:
            if codec_kind == "422i":
                codec.set_interlaced(pkg.INTERLACED)
            codec.set_decode_resolution(res)
            rw, rh = codec.decoded_size()
            coded = [codec.pack_coded(c[2]) for c in cases]
            for fmt in fmts:
                wants = [_want(fmt, quant, c[2], res, nc) for c in cases]
                assert wants[0].shape == (rh, fm.OUTPUTS[fmt].row_bytes(rw))
                if kind == "blocks" and fmt == "RG30":
                    v = wants[0].view(np.uint32) & 0x3FF
                    assert (v == 0).any() and (v == 1023).any()
                pitch = (fm.OUTPUTS[fmt].row_bytes(rw) + 15) // 16 * 16 + 32
                one = _buffers(1, rh, pitch)
                codec.inverse_host(coded[:1], quant, getattr(pkg, "PIXEL_" + fmt), one)
                _check(one[0], wants[0], f"{fmt} {codec_kind} {w}x{h} {kind} alone")
                three = _buffers(3, rh, pitch)
                codec.inverse_host(coded, quant, getattr(pkg, "PIXEL_" + fmt), three)
                for i in range(3):
                    _check(three[i], wants[i], f"{fmt} {codec_kind} {w}x{h} {kind} batch frame {i}")


def test_rgb10_values_below_the_saturating_add(pkg, ctx):
    """LL2 values below -0x4000 (from an LL3 injected with zero highpass; a 12-bit source never produces them) take the
    SSE2 rule in the columns below width - width % 8 and the scalar rule right of them.  The LL2 images the conversion
    reads are the codec's own, from its PLANAR16 decode at quarter resolution."""
    w, h = 200, 64                                      # LL2 50 wide: columns 48, 49 are the scalar tail
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.make_quant(pu.UNIT_DIVISORS, [0, 2, 2])
    rng = np.random.default_rng(3)
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_decode_resolution(fm.QUARTER)
        rw, rh = codec.decoded_size()
        bands = {}
        for c in range(3):
            for k in (1, 2, 3):
                for b in ("LH", "HL", "HH"):
                    bl = codec.layout.band[c][k - 1][1]
                    bands[(c, k, b)] = np.zeros((bl.height, bl.width), np.int16)
            bl = codec.layout.band[c][2][0]
            bands[(c, 3, "LL")] = rng.integers(-20000, 20000, (bl.height, bl.width)).astype(np.int16)
        coded = codec.pack_coded(bands)
        planar = np.zeros((3 * rh, rw), np.int16)
        codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [planar])
        planes = [planar[c * rh:(c + 1) * rh] for c in range(3)]
        v = planar.astype(np.int64)
        assert (v[:, :48] < -0x4000).any() and (v[:, 48:] < -0x4000).any() and (v > 16383).any()
        for fmt in RGB10:
            want = _rule(fmt, fm.QUARTER, planes)
            buf = _buffers(1, want.shape[0], want.shape[1] + 16)[0]
            codec.inverse_host([coded], quant, getattr(pkg, "PIXEL_" + fmt), [buf])
            _check(buf, want, fmt)


# ------------------------------------------------------------------------------------------------ launches
@pytest.mark.parametrize("fmt,codec_kind", [("YU64", "422"), ("RG30", "444")])
def test_conversion_is_one_launch(pkg, ctx, fmt, codec_kind):
    """A reduced decode launches the levels it inverts (as the PLANAR16 decode, whose lowpass copy launches nothing) plus
    one conversion kernel for the whole batch."""
    w, h = 640, 96
    desc, quant, bands, res = _case(pkg, codec_kind, w, h, "natural", 5)
    with pkg.Codec(ctx, desc, 4) as codec:
        codec.set_decode_resolution(res)
        rw, rh = codec.decoded_size()
        coded = [codec.pack_coded(bands)] * 4
        deltas = {}
        for name in ("PLANAR16", fmt):
            outs = [np.zeros((rh * (3 if name == "PLANAR16" else 1), fm.OUTPUTS[name].row_bytes(rw)), np.uint8) for _ in range(4)]
            before = ctx.stats()["kernel_launches"]
            codec.inverse_host(coded, quant, getattr(pkg, "PIXEL_" + name), outs)
            deltas[name] = ctx.stats()["kernel_launches"] - before
    assert deltas[fmt] == deltas["PLANAR16"] + 1 and deltas["PLANAR16"] >= 1


# ------------------------------------------------------------------------------------------------ rejections
def test_unsupported_combinations_and_bad_pitch(pkg, ctx):
    """Still CFB_ERROR_UNSUPPORTED (102): RG48 at half and quarter resolution, the 10-bit RGB words at half resolution,
    YU64 at quarter resolution,
    V210, B64A and BYR4 at either.  A pitch below the row bytes: CFB_ERROR_INVALID_ARGUMENT (1).  The codec decodes
    correctly after each rejection."""
    import torch

    def code_of(fn):
        with pytest.raises(pkg.CfbError) as ei:
            fn()
        return ei.value.code

    checks = [("422", [("YU64", fm.QUARTER), ("V210", fm.HALF), ("V210", fm.QUARTER)], ("YU64", fm.HALF)),
              ("444", [("RG48", fm.HALF), ("RG48", fm.QUARTER), ("B64A", fm.HALF), ("B64A", fm.QUARTER)] +
               [(n, fm.HALF) for n in RGB10], ("AB10", fm.QUARTER))]
    for codec_kind, refused, good in checks:
        w, h = 336, 48
        desc, quant, bands, res = _case(pkg, codec_kind, w, h, "natural", 9)
        want = _want(good[0], quant, bands, good[1], 3)
        with pkg.Codec(ctx, desc, 1) as codec:
            coded = codec.pack_coded(bands)

            def decode_good():
                codec.set_decode_resolution(good[1])
                buf = _buffers(1, *want.shape)[0]
                codec.inverse_host([coded], quant, getattr(pkg, "PIXEL_" + good[0]), [buf])
                _check(buf, want, f"{good} after the rejections")

            for fmt, r in refused:
                codec.set_decode_resolution(r)
                rw, rh = codec.decoded_size()
                out = np.zeros((rh, rw * 8), np.uint8)
                assert code_of(lambda: codec.inverse_host([coded], quant, getattr(pkg, "PIXEL_" + fmt), [out])) == 102, (fmt, r)
                decode_good()
            codec.set_decode_resolution(good[1])
            rh, rb = want.shape
            d_pyr = torch.zeros(codec.layout.total_bytes, dtype=torch.uint8, device="cuda")
            d_pyr[:coded.size] = torch.from_numpy(coded).cuda()
            d_out = torch.full((2 * rh * rb,), fm.CANARY, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            short = (rb - 1) // 16 * 16
            assert code_of(lambda: codec.inverse_device([d_pyr.data_ptr()], quant, getattr(pkg, "PIXEL_" + good[0]),
                                                        [d_out.data_ptr()], short)) == 1
            out = np.zeros((rh, rb - 2), np.uint8)
            assert code_of(lambda: codec.inverse_host([coded], quant, getattr(pkg, "PIXEL_" + good[0]), [out])) == 1
            ctx.synchronize()
            assert (d_out.cpu().numpy() == fm.CANARY).all()
            decode_good()
    with pkg.Codec(ctx, pkg.FrameDesc(256, 96, pkg.PIXEL_BYR4), 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        quant = pkg.quant_for_quality(pkg.FrameDesc(256, 96, pkg.PIXEL_BYR4), 4)
        for r in (fm.HALF, fm.QUARTER):
            codec.set_decode_resolution(r)
            assert code_of(lambda: codec.inverse_host([coded], quant, pkg.PIXEL_BYR4, [np.zeros((96, 256), np.uint16)])) == 102
