"""Forward levels 1 and 2 of progressive packed 8-bit 4:2:2 in one kernel (k_fwd_422_l12_tma, widths that are multiples
of 32) against the two-launch path on the same frames: level 1 alone (k_fwd_422_tma, LL1 to the scratch region), then
levels 2 and 3 (k_fwd_plane<3> reading LL1 back).  The coded region must be the same bytes -- at the 16-frame 4K batch the
benchmark times, at the device's own rows-per-warp split and at forced ones (CFB_TH), at the smallest height the layout
accepts (the level-2 band has 12 rows, so the top and bottom border ranges meet) and in UYVY byte order."""
import numpy as np
import pytest

import formats as fm
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401

pytestmark = pytest.mark.gpu


def _frames(w, h, n, seed):
    """n distinct frames: random bytes (every LL1 up to 4 * 255 << 2) and a natural picture, alternately"""
    rng = np.random.default_rng(seed)
    kinds = ("random", "natural")
    return [pu.synthetic_yuyv(rng, w, h, kinds[i % 2]) for i in range(n)]


def _fused_and_split(pkg, ctx, fmt, frames):
    """-> (coded regions of the full forward, coded regions of level 1 then levels 2 + 3), one array per frame"""
    import torch
    h, w2 = frames[0].shape
    w = w2 // 2
    desc = pkg.FrameDesc(w, h, fmt)
    quant = pkg.quant_for_quality(desc, 4)
    assert tuple(quant.prescale)[1] == 2                    # the fused kernel runs the prescaled level 2
    n = len(frames)
    with pkg.Codec(ctx, desc, n) as codec:
        lay = codec.layout
        stream = torch.cuda.ExternalStream(ctx.stream)
        with torch.cuda.stream(stream):
            d_frames = [torch.from_numpy(np.ascontiguousarray(f).reshape(-1)).cuda() for f in frames]
            d_pyr = [torch.zeros(lay.total_bytes, dtype=torch.uint8, device="cuda") for _ in range(n)]
        fp, pp = [t.data_ptr() for t in d_frames], [t.data_ptr() for t in d_pyr]
        ctx.synchronize()

        def run(*masks):
            with torch.cuda.stream(stream):
                for t in d_pyr:
                    t.fill_(0xA5)                           # stale bytes must not survive either path
            ctx.synchronize()
            for m in masks:
                codec.set_level_mask(m, 7)
                codec.forward_device(fp, lay.frame_pitch, quant, pp)
            ctx.synchronize()
            with torch.cuda.stream(stream):
                return [t[:lay.coded_bytes].cpu().numpy() for t in d_pyr]

        fused = run(7)
        split = run(1, 6)
        codec.set_level_mask(7, 7)
    return fused, split


def _assert_same(fused, split, what):
    for i, (a, b) in enumerate(zip(fused, split)):
        if not np.array_equal(a, b):
            bad = np.flatnonzero(a != b)
            raise AssertionError(f"{what} frame {i}: {bad.size} coded bytes differ, first at byte offsets {bad[:8].tolist()}")


@pytest.mark.parametrize("th", [None, 2, 3, 5, 8, 64])
def test_fused_equals_split_4k_batch(pkg, ctx, monkeypatch, th):
    """16 distinct 3840x2160 frames in one launch; th = None is the split pick_th chooses on this device"""
    if th is not None:
        monkeypatch.setenv("CFB_TH", str(th))
    frames = _frames(3840, 2160, 16, seed=12)
    fused, split = _fused_and_split(pkg, ctx, pkg.PIXEL_YUYV, frames)
    _assert_same(fused, split, f"4K x16 th={th}")


@pytest.mark.parametrize("size", [(256, 48), (96, 48), (288, 56), (1920, 1080)])
@pytest.mark.parametrize("th", [None, 2, 3, 64])
def test_fused_equals_split_small(pkg, ctx, monkeypatch, size, th):
    """The smallest height (12 level-2 rows), one strip with both image borders (96: the narrowest width whose level-3
    chroma band still has the 6 columns its border filter reads), a last strip of 4 lanes, and 1080p, in YUYV and UYVY"""
    if th is not None:
        monkeypatch.setenv("CFB_TH", str(th))
    w, h = size
    frames = _frames(w, h, 3, seed=w + h)
    for fmt, name, conv in ((pkg.PIXEL_YUYV, "YUYV", lambda f: f), (pkg.PIXEL_UYVY, "UYVY", fm.yuyv_to_uyvy)):
        fused, split = _fused_and_split(pkg, ctx, fmt, [conv(f) for f in frames])
        _assert_same(fused, split, f"{name} {w}x{h} th={th}")
