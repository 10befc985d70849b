"""GPU parity tests of the forward path (level 1 packed 4:2:2 + levels 2,3 + fused quantisation),
called through the C ABI (include/cfhd_b200.h) and compared bit for bit with the oracle and with
the golden vectors produced by the reference itself."""
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401
from test_golden import GOLDEN, load_golden

pytestmark = pytest.mark.gpu


def _compare(got, want):
    assert set(want) <= set(got)
    for key in sorted(want):
        if not np.array_equal(got[key], want[key]):
            bad = np.argwhere(got[key] != want[key])
            raise AssertionError(f"band {key}: {bad.shape[0]} mismatches, first at {bad[:5].tolist()} "
                                 f"got {got[key][tuple(bad[0])]} want {want[key][tuple(bad[0])]}")


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_golden_vectors(pkg, ctx, path):
    frame, div, prescale, quality, bands = load_golden(path)
    h, w2 = frame.shape
    desc = pkg.FrameDesc(w2 // 2, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, quality)
    assert quant.table(3) == div
    with pkg.Codec(ctx, desc, 1) as codec:
        got = codec.unpack_coded(codec.forward_host([frame], quant)[0])
    want = {k: v for k, v in bands.items() if not (k[2] == "LL" and k[1] != 3)}
    _compare(got, want)


@pytest.mark.parametrize("size", [(192, 48), (256, 64), (320, 56), (704, 96), (1920, 1080)])
@pytest.mark.parametrize("kind", ["natural", "random", "extreme", "constant"])
@pytest.mark.parametrize("fmt", [0, 1])
def test_forward_422_vs_oracle(pkg, ctx, size, kind, fmt):
    w, h = size
    rng = np.random.default_rng(w * 31 + h + fmt)
    frame = pu.synthetic_yuyv(rng, w, h, kind)
    if fmt == 1:
        frame = fm.yuyv_to_uyvy(frame)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_UYVY if fmt else pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 1) as codec:
        got = codec.unpack_coded(codec.forward_host([frame], quant)[0])
    _compare(got, pu.oracle_forward_422(ol.oracle(), frame, quant, fmt))


@pytest.mark.parametrize("quality", [1, 2, 3, 5, 6])
def test_forward_422_qualities(pkg, ctx, quality):
    w, h = 512, 128
    rng = np.random.default_rng(quality)
    frame = pu.synthetic_yuyv(rng, w, h, "natural")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, quality)
    with pkg.Codec(ctx, desc, 1) as codec:
        got = codec.unpack_coded(codec.forward_host([frame], quant)[0])
    _compare(got, pu.oracle_forward_422(ol.oracle(), frame, quant, 0))


def test_forward_batch_and_pitch(pkg, ctx):
    """A batch of different frames in one launch, with a padded host pitch."""
    w, h, n = 640, 96, 5
    rng = np.random.default_rng(99)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    padded = [np.zeros((h, w * 2 + 64), np.uint8) for _ in range(n)]
    frames = []
    for p in padded:
        f = pu.synthetic_yuyv(rng, w, h, "natural")
        p[:, :w * 2] = f
        frames.append(f)
    with pkg.Codec(ctx, desc, n) as codec:
        views = [p[:, :] for p in padded]
        coded = codec.forward_host(views, quant)
        for f, cbuf in zip(frames, coded):
            _compare(codec.unpack_coded(cbuf), pu.oracle_forward_422(ol.oracle(), f, quant, 0))


def test_forward_4k_full_size(pkg, ctx):
    """BASELINE config 3 size: one 3840x2160 frame against the oracle + a second identical submission
    must give identical bytes (determinism), and a constant frame must give all-zero highpass bands."""
    w, h = 3840, 2160
    rng = np.random.default_rng(4)
    frame = pu.synthetic_yuyv(rng, w, h, "natural")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 2) as codec:
        a, b = codec.forward_host([frame, frame], quant)
        assert np.array_equal(a, b)
        _compare(codec.unpack_coded(a), pu.oracle_forward_422(ol.oracle(), frame, quant, 0))
        const = np.full((h, w * 2), 128, np.uint8)
        bands = codec.unpack_coded(codec.forward_host([const], quant)[0])
        for key, arr in bands.items():
            if key[2] != "LL":
                assert not arr.any(), key
            else:
                assert (arr == arr[0, 0]).all()


def test_invalid_arguments(pkg, ctx):
    desc = pkg.FrameDesc(256, 64, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 1) as codec:
        with pytest.raises(pkg.CfbError) as ei:
            codec.forward_host([np.zeros((64, 512), np.uint8)] * 2, quant)      # batch > max_batch
        assert ei.value.code == 1
    with pytest.raises(pkg.CfbError):
        pkg.Codec(ctx, pkg.FrameDesc(250, 64, pkg.PIXEL_YUYV), 1)


# kernel_launches per forward call, by source and level mask (1: level 1 only, 7: all three levels), 384 wide
_FWD_LAUNCHES = {"YUYV": (1, 3), "UYVY": (1, 3), "YU64": (1, 3), "V210": (1, 3), "PLANAR16": (1, 3),
                 "RG48": (2, 4), "B64A": (2, 4), "RG64": (2, 4), "RG30": (3, 5), "AB10": (3, 5), "AR10": (3, 5),
                 "R210": (3, 5), "DPX0": (3, 5), "BYR4": (2, 4)}
# 400 wide, the level-2 and level-3 planes of 4:2:2 are ragged: each level is k_fwd_plane plus its edge kernel
_FWD_LAUNCHES_400 = {"YUYV": (1, 5), "UYVY": (1, 5)}


@pytest.mark.parametrize("fmt_name", sorted(_FWD_LAUNCHES))
def test_forward_kernel_launches(pkg, ctx, fmt_name):
    """The library's kernel_launches counter for one forward call of every source, at level masks 1 and 7: progressive
    and interlaced 4:2:2, levels 1 + 2 fused (width a multiple of 32) or not, RGBA with and without alpha.  Every kernel
    that runs is counted: the border-row kernel of a TMA-fed level 1 (BYR4 as RG48 / RGBA) and the edge kernel of a
    ragged plane."""
    fmt = getattr(pkg, "PIXEL_" + fmt_name)
    widths = [384, 400] if fmt_name in ("YUYV", "UYVY") else [384]
    modes = [pkg.PROGRESSIVE, pkg.INTERLACED] if fmt_name in ("YUYV", "UYVY", "YU64", "V210") else [pkg.PROGRESSIVE]
    flags = [0, pkg.FRAME_ALPHA] if fmt_name in ("B64A", "RG64") else [0]
    for w in widths:
        for fl in flags:
            desc = pkg.FrameDesc(w, 96, fmt, fl)
            with pkg.Codec(ctx, desc, 1) as codec:
                lay = codec.layout
                frame = np.zeros((lay.frame_bytes // lay.frame_pitch, lay.frame_pitch), np.uint8)
                for mode in modes:
                    codec.set_interlaced(mode)
                    quant = pkg.quant_for_quality(desc, 4, interlaced=bool(mode))
                    for mask, want in zip((1, 7), (_FWD_LAUNCHES_400 if w == 400 else _FWD_LAUNCHES)[fmt_name]):
                        codec.set_level_mask(mask, 7)
                        before = ctx.stats()["kernel_launches"]
                        codec.forward_host([frame], quant)
                        assert ctx.stats()["kernel_launches"] - before == want, (w, fl, mode, mask)


@pytest.mark.parametrize("mode", [0, 1])
def test_gop2_forward_launch_count(pkg, ctx, mode):
    """cfb_gop2_forward_host: level 1 of each frame (1 each), the temporal transform (1 per channel), the range audit of
    the temporal highpass (1) and wavelets 3, 4, 5 (1 each)."""
    desc = pkg.FrameDesc(384, 96, pkg.PIXEL_YUYV)
    frame = np.zeros((96, 768), np.uint8)
    with pkg.Codec(ctx, desc, 2) as codec:
        codec.set_interlaced(mode)
        before = ctx.stats()["kernel_launches"]
        codec.gop2_forward_host(frame, frame, pkg.gop2_quant_for_quality(desc, 4, bool(mode)))
        assert ctx.stats()["kernel_launches"] - before == 2 + 3 + 1 + 3
