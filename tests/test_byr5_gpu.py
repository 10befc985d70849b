"""BYR5 (12-bit packed Bayer) on the GPU: k_fwd_tma<SrcBYR5> and its border launch against the reference's bands (golden
fixtures from make_golden_byr5.py) and the oracle pyramid of the restated planes, at widths whose segments sit 8 / 4 bytes
off a 16-byte boundary, padded pitches, batches, every rows-per-warp split, the sparse format, the pool, the four-plane
inverse and the error codes."""
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg, splits  # noqa: F401
from test_row_split_gpu import SIZES

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _oracle(frame, pw, phase, quant, height=None):
    return pu.forward_pyramid_planes(ol.oracle(), fm.byr5_planes(frame, pw, phase, height), quant.table(4), tuple(quant.prescale))


def _forward(pkg, codec, frames, quant, phase):
    codec.set_bayer_phase(phase)
    return [codec.unpack_coded(c) for c in codec.forward_host(frames, quant)]


@pytest.mark.parametrize("name", ["byr5_512x128_p1_q4", "byr5_208x100_p2_extreme_q4"])
def test_golden_byr5(pkg, ctx, name):
    """The reference's bands of a BYR5 frame, bit for bit.  208 x 100: the plane height 50 is padded to 56 by the encoder,
    which repeats the last packed row; the codec is given those rows."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    frame, phase, ch = z["frame"], int(z["phase"]), int(z["coded_height"])
    pw = frame.shape[1] // 6
    full = np.concatenate([frame, np.repeat(frame[-1:], ch - frame.shape[0], axis=0)])
    desc = pkg.FrameDesc(2 * pw, 2 * ch, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    assert quant.table(4) == z["divisors"].tolist() and list(quant.prescale) == z["prescale"][0].tolist()
    want = {tuple(int(v) if v.isdigit() else v for v in k.split("_")[1:]): z[k] for k in z.files if k.startswith("b_")}
    with pkg.Codec(ctx, desc, 1) as codec:
        got = _forward(pkg, codec, [full], quant, phase)[0]
        pu.assert_bands(got, want, name)
        for ph in range(4):
            pu.assert_bands(_forward(pkg, codec, [full], quant, ph)[0], _oracle(frame, pw, ph, quant, ch), f"{name} phase {ph}")


# Bayer sizes: plane widths 104, 360, 1352, 2656 (segments 8 / 4 bytes off 16-byte boundaries), 4096 (8K)
@pytest.mark.parametrize("size,phases", [((208, 96), (0, 1, 2, 3)), ((720, 112), (0, 1, 2, 3)), ((2704, 160), (1, 2)),
                                         ((5312, 128), (0, 3)), ((8192, 4320), (2,))])
def test_forward_byr5_vs_oracle(pkg, ctx, size, phases):
    w, h = size
    pw, ph = w // 2, h // 2
    rng = np.random.default_rng(w + h)
    frame = fm.byr5_pack(fm.byr5_random_components(rng, pw, ph, "random" if w < 8192 else "natural"))
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 1) as codec:
        for phase in phases:
            pu.assert_bands(_forward(pkg, codec, [frame], quant, phase)[0], _oracle(frame, pw, phase, quant), f"BYR5 {w}x{h} phase {phase}")


@pytest.mark.parametrize("size,extra", [((720, 112), 16), ((2704, 96), 48), ((208, 96), 400)])
def test_forward_byr5_padded_pitch(pkg, ctx, size, extra):
    """A frame pitch beyond 3 W bytes (a multiple of 16): the padding never enters the bands."""
    w, h = size
    pw, ph = w // 2, h // 2
    rng = np.random.default_rng(w * 3 + extra)
    frame = fm.byr5_pack(fm.byr5_random_components(rng, pw, ph), pitch=6 * pw + extra)
    frame[:, 6 * pw:] = rng.integers(0, 256, (ph, extra)).astype(np.uint8)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 1) as codec:
        for phase in range(4):
            pu.assert_bands(_forward(pkg, codec, [frame], quant, phase)[0], _oracle(frame, pw, phase, quant), f"pitch +{extra} phase {phase}")


def test_forward_byr5_batch_equals_single(pkg, ctx):
    """16 frames in one launch == each frame coded alone."""
    w, h = 1040, 112
    rng = np.random.default_rng(16)
    frames = [fm.byr5_pack(fm.byr5_random_components(rng, w // 2, h // 2, "extreme" if i % 5 == 0 else "random")) for i in range(16)]
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 16) as codec:
        codec.set_bayer_phase(3)
        batch = codec.forward_host(frames, quant)
        for i in range(16):
            assert np.array_equal(codec.forward_host([frames[i]], quant)[0], batch[i]), f"frame {i}"
        pu.assert_bands(codec.unpack_coded(batch[7]), _oracle(frames[7], w // 2, 3, quant), "batch frame 7")


@pytest.mark.parametrize("size", SIZES)
def test_byr5_at_every_split(pkg, ctx, splits, size):
    """Every rows-per-warp split of test_row_split_gpu, all four phases; `size` is the plane size."""
    pw, ph = size
    w, h = 2 * pw, 2 * ph
    rng = np.random.default_rng(w + h + 5)
    frame = fm.byr5_pack(fm.byr5_random_components(rng, pw, ph))
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    cases = [(phase, _oracle(frame, pw, phase, quant)) for phase in range(4)]
    with pkg.Codec(ctx, desc, 1) as codec:
        for th in splits():
            for phase, want in cases:
                pu.assert_bands(_forward(pkg, codec, [frame], quant, phase)[0], want, f"BYR5 {w}x{h} phase {phase} th={th}")


def test_byr5_sparse_inverse_and_pool(pkg, ctx):
    """forward_host_sparse expands to the dense coded region; the four-plane (PLANAR16) inverse equals the oracle's; a
    pool round gives the synchronous bytes."""
    w, h, phase = 720, 112, 1
    pw, ph = w // 2, h // 2
    rng = np.random.default_rng(77)
    frames = [fm.byr5_pack(fm.byr5_random_components(rng, pw, ph, "natural")) for _ in range(6)]
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    with pkg.Codec(ctx, desc, 1) as codec:
        codec.set_bayer_phase(phase)
        dense = [codec.forward_host([f], quant)[0] for f in frames]
        sp, _ = codec.forward_host_sparse([frames[0]], quant)
        assert np.array_equal(pkg.sparse_expand(codec.layout, sp[0]), dense[0])
        want = _oracle(frames[0], pw, phase, quant)
        coded_bands = {k: v for k, v in want.items() if not (k[2] == "LL" and k[1] != 3)}
        planes = pu.inverse_pyramid(orc, coded_bands, quant.table(4), tuple(quant.prescale), nchan=4)
        out = np.zeros((4 * ph, w), np.int16)           # planes stacked at a pitch of 2 W bytes
        codec.inverse_host([dense[0]], quant, pkg.PIXEL_PLANAR16, [out])
        pu.check_planes([out[c * ph:(c + 1) * ph, :pw] for c in range(4)], planes, "BYR5 PLANAR16")
    # the pool takes the Bayer phase 0 of a fresh codec: compare with phase 0
    with pkg.Codec(ctx, desc, 1) as codec:
        dense0 = [codec.forward_host([f], quant)[0] for f in frames]
    with pkg.Pool([0], desc, slots=2, batch=4, queue_length=8) as pool:
        lay = pool.layout
        pf = [pkg.pinned_empty(f.shape) for f in frames]
        pc = [pkg.pinned_empty(lay.coded_bytes) for _ in frames]
        for a, f in zip(pf, frames):
            a[:] = f
        for i in range(len(frames)):
            pool.submit_forward(i, pf[i], quant, pc[i])
        assert [pool.wait() for _ in frames] == list(range(len(frames)))
        for i in range(len(frames)):
            assert np.array_equal(np.asarray(pc[i]).view(np.uint8).reshape(-1), dense0[i]), f"pool frame {i}"


def test_byr5_launch_count(pkg, ctx):
    """Level 1 is two launches (main rows + border rows); levels 2 and 3 one each."""
    desc = pkg.FrameDesc(384, 96, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 1) as codec:
        frame = np.zeros((48, 3 * 384), np.uint8)
        for mask, want in ((1, 2), (7, 4)):
            codec.set_level_mask(mask, 7)
            before = ctx.stats()["kernel_launches"]
            codec.forward_host([frame], quant)
            assert ctx.stats()["kernel_launches"] - before == want, mask


def test_byr5_errors(pkg, ctx):
    for bad in (200, 712):                              # Bayer widths are multiples of 16
        with pytest.raises(pkg.CfbError) as ei:
            pkg.Codec(ctx, pkg.FrameDesc(bad, 96, pkg.PIXEL_BYR5), 1)
        assert ei.value.code == 102
    desc = pkg.FrameDesc(208, 96, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Codec(ctx, desc, 1) as codec:
        for pitch in (6 * 104 - 16, 6 * 104 + 8):       # below 3 W bytes, or not a multiple of 16
            with pytest.raises(pkg.CfbError) as ei:
                codec.forward_host([np.zeros((48, pitch), np.uint8)], quant)
            assert ei.value.code == 1, pitch
        with pytest.raises(pkg.CfbError) as ei:
            codec.set_interlaced(pkg.INTERLACED)
        assert ei.value.code == 102
        with pytest.raises(pkg.CfbError) as ei:
            codec.set_bayer_curve(fm.bayer_log90_curve())
        assert ei.value.code == 102
        coded = codec.forward_host([np.zeros((48, 6 * 104), np.uint8)], quant)[0]
        with pytest.raises(pkg.CfbError) as ei:
            codec.inverse_host([coded], quant, pkg.PIXEL_BYR5, [np.zeros((48, 6 * 104), np.uint8)])
        assert ei.value.code == 102
