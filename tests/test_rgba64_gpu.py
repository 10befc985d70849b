"""16-bit RGBA sources (B64A, RG64) on the GPU: forward level 1 of k_fwd_tma<SrcRGBA64> + levels 2, 3 for three and four
channels, and the four-channel final inverse, bit-exact against the oracle (rgba_util's rules are pinned to the reference
in test_rgba64.py) and against the reference's own bands and frames stored under golden/ (make_golden_rgba.py)."""
import hashlib

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
import rgba_util as ru
from gpu_fixtures import pkg, splits  # noqa: F401

pytestmark = pytest.mark.gpu
FORMATS = ("B64A", "RG64")


def _desc(pkg, w, h, name, alpha):
    return pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + name), pkg.FRAME_ALPHA if alpha else 0)


def _frame(w, h, kind, name):
    rng = np.random.default_rng(w + h + len(kind))
    if w * h > 4_000_000:       # 4K: a tiled quarter keeps the oracle cheap; every strip and row block still runs
        tile = fm.synthetic_rgba64(rng, w // 2, h // 2, kind, name)
        return np.tile(tile, (2, 2))
    return fm.synthetic_rgba64(rng, w, h, kind, name)


def _oracle_coded(frame, name, alpha, quant, nchan):
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_rgba64(frame, name, alpha), quant.table(nchan), tuple(quant.prescale))
    return fm.coded_region(pyr)


def _forward_vs_oracle(pkg, w, h, kind, name, alpha):
    frame = _frame(w, h, kind, name)
    desc = _desc(pkg, w, h, name, alpha)
    quant = pkg.quant_for_quality(desc, 4)
    nchan = 4 if alpha else 3
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        coded = codec.forward_host([frame, frame], quant)
        assert np.array_equal(coded[0], coded[1])
        got = codec.unpack_coded(coded[0])
    assert len(got) == 10 * nchan
    pu.assert_bands(got, _oracle_coded(frame, name, alpha, quant, nchan), f"{name} alpha={alpha} {w}x{h} {kind}")


@pytest.mark.parametrize("size", [(256, 64), (328, 48), (720, 480), (1920, 1080)])
@pytest.mark.parametrize("kind", ["natural", "random", "extreme"])
@pytest.mark.parametrize("name", FORMATS)
@pytest.mark.parametrize("alpha", [False, True])
def test_forward_vs_oracle(pkg, size, kind, name, alpha):
    _forward_vs_oracle(pkg, *size, kind, name, alpha)


@pytest.mark.parametrize("name", FORMATS)
def test_forward_4k_vs_oracle(pkg, name):
    _forward_vs_oracle(pkg, 3840, 2160, "natural", name, True)


@pytest.mark.parametrize("name", FORMATS)
@pytest.mark.parametrize("alpha", [False, True])
def test_forward_padded_pitch(pkg, name, alpha):
    w, h = 720, 96
    frame = _frame(w, h, "random", name)
    padded = np.zeros((h, 4 * w + 64), np.uint16)
    padded[:, :4 * w] = frame
    padded[:, 4 * w:] = 0xBEEF
    desc = _desc(pkg, w, h, name, alpha)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        got = codec.unpack_coded(codec.forward_host([padded], quant)[0])
    pu.assert_bands(got, _oracle_coded(frame, name, alpha, quant, 4 if alpha else 3), "padded pitch")


def test_forward_vs_reference_fixture(pkg):
    z = ru.load_fixture("rgba_b64a_256x64_q4.npz")
    frame = z["frame"]
    h, w = frame.shape[0], frame.shape[1] // 4
    desc = _desc(pkg, w, h, "B64A", True)
    quant = pkg.quant_for_quality(desc, 4)
    assert quant.table(4) == z["divisors"].tolist() and list(quant.prescale) == z["prescale"].tolist()
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        got = codec.unpack_coded(codec.forward_host([frame], quant)[0])
    want = ru.fixture_bands(z, "b")
    assert len(want) == 40
    pu.assert_bands(got, want, "reference bands")


def _decode_case(pkg, w, h, kind, name="B64A"):
    frame = _frame(w, h, kind, name)
    desc = _desc(pkg, w, h, name, True)
    quant = pkg.quant_for_quality(desc, 4)
    coded = _oracle_coded(frame, name, True, quant, 4)
    planes = pu.inverse_pyramid(ol.oracle(), coded, quant.table(4), tuple(quant.prescale), nchan=4)
    return desc, quant, coded, planes


@pytest.mark.parametrize("size", [(256, 64), (328, 48), (200, 48), (720, 480), (1920, 1080)])
@pytest.mark.parametrize("kind", ["natural", "extreme"])
def test_inverse_four_channels_vs_oracle(pkg, size, kind):
    w, h = size
    desc, quant, coded_bands, planes = _decode_case(pkg, w, h, kind)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        coded = codec.pack_coded(coded_bands)
        outs = [np.zeros((h, 4 * w), np.uint16) for _ in range(2)]
        codec.inverse_host([coded, coded], quant, pkg.PIXEL_B64A, outs)
        want = fm.pack_b64a_alpha(planes)
        assert np.array_equal(outs[0], want), np.argwhere(outs[0] != want)[:5].tolist()
        assert np.array_equal(outs[1], want)
        rg = np.zeros((h, 3 * w), np.uint16)
        codec.inverse_host([coded], quant, pkg.PIXEL_RG48, [rg])
        assert np.array_equal(rg, fm.pack_rg48(planes[:3]))
        r30 = np.zeros((h, w), np.uint32)
        codec.inverse_host([coded], quant, pkg.PIXEL_RG30, [r30])
        assert np.array_equal(r30, fm.pack_rgb30_output("RG30", planes[:3]))
        pl = np.zeros((4 * h, w), np.int16)
        codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [pl])
        pu.check_planes([pl[c * h:(c + 1) * h] for c in range(4)], planes, "PLANAR16")
        wide = np.zeros((h, 4 * w + 8), np.uint16)
        codec.inverse_host([coded], quant, pkg.PIXEL_B64A, [wide])
        assert np.array_equal(wide[:, :4 * w], want) and not wide[:, 4 * w:].any()


@pytest.mark.parametrize("name,w,h", [("decoded_rgba_b64a_328x48_q4.npz", 328, 48),
                                      ("decoded_rgba_b64a_200x48_extreme_q4.npz", 200, 48)])
def test_inverse_vs_reference_fixture(pkg, name, w, h):
    z = ru.load_fixture(name)
    bands = ru.fixture_bands(z, "d")
    unit = pkg.make_quant([[[1] * 4] * 3] * 4, z["prescale"].tolist())
    with pkg.Context(0) as ctx, pkg.Codec(ctx, _desc(pkg, w, h, "B64A", True), 1) as codec:
        coded = codec.pack_coded(bands)
        b64a = np.zeros((h, 4 * w), np.uint16)
        codec.inverse_host([coded], unit, pkg.PIXEL_B64A, [b64a])
        rg48 = np.zeros((h, 3 * w), np.uint16)
        codec.inverse_host([coded], unit, pkg.PIXEL_RG48, [rg48])
    assert hashlib.sha256(b64a.tobytes()).hexdigest() == str(z["sha256_B64A"])
    assert hashlib.sha256(rg48.tobytes()).hexdigest() == str(z["sha256_RG48"])


@pytest.mark.parametrize("name", FORMATS)
def test_three_channel_codec_decodes_as_rg48(pkg, name):
    """A B64A / RG64 source without FRAME_ALPHA is an RGB 4:4:4 codec: its coded region has the RG48 codec's layout and every
    output of the same bands is byte-identical to the RG48 codec's."""
    w, h = 328, 48
    frame = _frame(w, h, "natural", name)
    desc = _desc(pkg, w, h, name, False)
    quant = pkg.quant_for_quality(desc, 4)
    coded_bands = _oracle_coded(frame, name, False, quant, 3)
    outs = {}
    with pkg.Context(0) as ctx:
        for d in (desc, pkg.FrameDesc(w, h, pkg.PIXEL_RG48)):
            with pkg.Codec(ctx, d, 1) as codec:
                coded = codec.pack_coded(coded_bands)
                for fmt, shape, dt in ((pkg.PIXEL_B64A, (h, 4 * w), np.uint16), (pkg.PIXEL_RG48, (h, 3 * w), np.uint16),
                                       (pkg.PIXEL_RG30, (h, w), np.uint32)):
                    o = np.zeros(shape, dt)
                    codec.inverse_host([coded], quant, fmt, [o])
                    outs.setdefault(fmt, []).append(o)
    for fmt, (a, b) in outs.items():
        assert np.array_equal(a, b), fmt


@pytest.mark.parametrize("name", FORMATS)
def test_every_row_split(pkg, splits, name):
    """Forward (3 and 4 channels) and the four-channel B64A inverse at every rows-per-warp split (CFB_TH), 16 frames per
    launch for the forward, as the benchmark batches them."""
    w, h = 720, 200
    frame = _frame(w, h, "random", name)
    with pkg.Context(0) as ctx:
        for alpha in (False, True):
            desc = _desc(pkg, w, h, name, alpha)
            quant = pkg.quant_for_quality(desc, 4)
            want = _oracle_coded(frame, name, alpha, quant, 4 if alpha else 3)
            with pkg.Codec(ctx, desc, 16) as codec:
                for th in splits():
                    coded = codec.forward_host([frame] * 16, quant)
                    for i in (0, 15):
                        pu.assert_bands(codec.unpack_coded(coded[i]), want, f"th={th} alpha={alpha} frame {i}")
        desc, quant, coded_bands, planes = _decode_case(pkg, w, h, "natural", name)
        want = fm.pack_b64a_alpha(planes)
        with pkg.Codec(ctx, desc, 1) as codec:
            coded = codec.pack_coded(coded_bands)
            for th in splits():
                out = np.zeros((h, 4 * w), np.uint16)
                codec.inverse_host([coded], quant, pkg.PIXEL_B64A, [out])
                assert np.array_equal(out, want), f"th={th}"


@pytest.mark.parametrize("name", FORMATS)
def test_pool_and_sparse_match_dense(pkg, name):
    w, h, n = 720, 96, 6
    desc = _desc(pkg, w, h, name, True)
    quant = pkg.quant_for_quality(desc, 4)
    frames = [_frame(w, h, k, name) for k in ("natural", "random", "extreme")] * 2
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        dense = [codec.forward_host([f], quant)[0] for f in frames]
        dec = []
        for c in dense:
            o = np.zeros((h, 4 * w), np.uint16)
            codec.inverse_host([c], quant, pkg.PIXEL_B64A, [o])
            dec.append(o)
        sp, sizes = codec.forward_host_sparse(frames[:1], quant)
        assert np.array_equal(pkg.sparse_expand(codec.layout, sp[0]), dense[0])
        o = np.zeros((h, 4 * w), np.uint16)
        codec.inverse_host_sparse(sp, quant, pkg.PIXEL_B64A, [o])
        assert np.array_equal(o, dec[0])
    with pkg.Pool([0], desc, slots=2, batch=2, queue_length=8) as pool:
        lay = pool.layout
        pf = [pkg.pinned_empty((h, 4 * w), np.uint16) for _ in range(n)]
        pc = [pkg.pinned_empty(lay.coded_bytes) for _ in range(n)]
        ps = [pkg.pinned_empty(pkg.sparse_max_bytes(lay)) for _ in range(n)]
        po = [pkg.pinned_empty((h, 4 * w), np.uint16) for _ in range(n)]
        for i in range(n):
            pf[i][:] = frames[i]
            pool.submit_forward(i, pf[i], quant, pc[i])
        assert [pool.wait() for _ in range(n)] == list(range(n))
        for i in range(n):
            assert np.array_equal(pc[i], dense[i]), i
            pool.submit_forward_sparse(i, pf[i], quant, ps[i])
        assert [pool.wait() for _ in range(n)] == list(range(n))
        for i in range(n):
            assert np.array_equal(pkg.sparse_expand(lay, ps[i]), dense[i]), i
            pool.submit_inverse_sparse(i, ps[i], quant, pkg.PIXEL_B64A, po[i])
        assert [pool.wait() for _ in range(n)] == list(range(n))
        for i in range(n):
            assert np.array_equal(po[i], dec[i]), i
            po[i][:] = 0
            pool.submit_inverse(i, pc[i], quant, pkg.PIXEL_B64A, po[i])
        assert [pool.wait() for _ in range(n)] == list(range(n))
        for i in range(n):
            assert np.array_equal(po[i], dec[i]), i


@pytest.mark.parametrize("alpha", [False, True])
def test_error_cases(pkg, alpha):
    w, h = 256, 64
    desc = _desc(pkg, w, h, "RG64", alpha)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        with pytest.raises(pkg.CfbError) as e:          # RG64 is an input only
            codec.inverse_host([coded], quant, pkg.PIXEL_RG64, [np.zeros((h, 4 * w), np.uint16)])
        assert e.value.code == 102
        with pytest.raises(pkg.CfbError) as e:
            codec.set_interlaced(True)
        assert e.value.code == 102
        codec.set_decode_resolution(pkg.RESOLUTION_HALF)
        with pytest.raises(pkg.CfbError) as e:
            codec.inverse_host([coded], quant, pkg.PIXEL_B64A, [np.zeros((h // 2, 4 * w // 2), np.uint16)])
        assert e.value.code == 102
