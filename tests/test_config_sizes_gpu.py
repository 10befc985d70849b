"""Bit-exact parity at the sizes BASELINE.json quotes, through the C ABI:

  * the exact path bench.py's e2e leg times: the asynchronous pool with the sparse transfer format at 3840x2160,
    16 slots x batch 2, encode and decode jobs interleaved, incl. frames whose non-zero count exceeds the speculative
    value guess (second D2H) -- sparse == expand == dense == oracle bands, bit for bit;
  * full-resolution inverse (16-bit planes) at 3840x2160 against the oracle;
  * config 4 (3840x2160 RG48 -> RGB 4:4:4 12 bit) and config 5 (7680x4320 BYR4 -> 4 x 3840x2160 12 bit) against the oracle;
  * the north star's own frames: TestCFHD's Qbist sequence (seed 50, Example/TestCFHD.cpp:41,1149-1219) frames 1-10 at
    1920x1080 and 3840x2160 against the bands the UNMODIFIED reference's EncodeSample leaves behind (oracle/_ref travels
    to the GPU box with the snapshot; /root/reference itself is not needed at run time).
"""
import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")


# ------------------------------------------------------------------------------------------------ timed e2e path
def test_pool_sparse_4k_interleaved_bitexact(pkg):
    w, h = 3840, 2160
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    rng = np.random.default_rng(2160)
    base = [pu.synthetic_yuyv(rng, w, h, "natural") for _ in range(2)]
    dense_frame = pu.synthetic_yuyv(rng, w, h, "random")                 # nearly every coefficient non-zero
    n = 24
    frames = []
    for i in range(n):
        if i in (5, 6, 17):
            frames.append(np.roll(dense_frame, 32 * i, axis=1).copy())   # exceeds any value guess -> second D2H
        else:
            frames.append(np.roll(base[i & 1], (64 * i, 16 * i), axis=(0, 1)).copy())
    orc = ol.oracle()
    with pkg.Pool([0], desc, slots=16, batch=2, queue_length=80) as pool, pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        lay = pool.layout
        h_in = [pkg.pinned_empty((h, lay.frame_pitch)) for _ in range(n)]
        h_sp = [pkg.pinned_empty(pkg.sparse_max_bytes(lay)) for _ in range(n)]
        h_out = [pkg.pinned_empty((h, lay.frame_pitch)) for _ in range(n)]
        for a, f in zip(h_in, frames):
            a[:] = f
        for a in h_sp:
            a[:] = 0xEE                                                  # stale bytes must not survive in the used part
        # interleaved encode / decode exactly as bench.py's run_stream does: a frame's decode is submitted as soon as its
        # coefficients are back, while later encodes are still in flight
        FWD, INV = 0, 1 << 30
        next_f = done = inflight = 0
        order = []
        while done < n:
            while next_f < n and inflight < 64:
                pool.submit_forward_sparse(FWD | next_f, h_in[next_f], quant, h_sp[next_f])
                next_f += 1; inflight += 1
            r = pool.wait(); inflight -= 1
            order.append(r)
            if r & INV:
                done += 1
            else:
                pool.submit_inverse_sparse(INV | r, h_sp[r], quant, pkg.PIXEL_YUYV, h_out[r]); inflight += 1
        assert [r for r in order if not r & INV] == list(range(n))                    # in-order delivery per direction
        assert [r & ~INV for r in order if r & INV] == list(range(n))
        sizes = []
        for i in range(n):
            sp = np.asarray(h_sp[i])
            nbytes = pkg.sparse_bytes(sp)
            sizes.append(nbytes)
            dense = codec.forward_host([frames[i]], quant)[0]
            assert np.array_equal(pkg.sparse_expand(lay, sp[:nbytes]), dense), f"frame {i}: sparse != dense"
            assert np.array_equal(pkg.sparse_compact(lay, dense), sp[:nbytes]), f"frame {i}: bytes differ from the host packer"
            out = np.zeros((h, lay.frame_pitch), np.uint8)
            codec.inverse_host([dense], quant, pkg.PIXEL_YUYV, [out])
            assert np.array_equal(np.asarray(h_out[i]), out), f"frame {i}: pooled sparse decode != dense decode"
            if i in (0, 5, 23):                                                       # and both == the oracle
                want = pu.oracle_forward_422(orc, frames[i], quant, 0)
                pu.assert_bands(codec.unpack_coded(dense), want, f"frame {i}")
                planes = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale))
                a, b = pu.yuyv_envelope(planes)
                assert ((out == a) | (out == b)).all(), f"frame {i}: outside the reference's dither envelope"
        assert min(sizes[5], sizes[6], sizes[17]) > 2 * sizes[0]                      # dense frames: far beyond the speculative copy
        assert sizes[0] < lay.coded_bytes // 4


# ------------------------------------------------------------------------------------------------ inverse at 4K
@pytest.mark.parametrize("kind", ["natural", "random"])
def test_inverse_planar16_4k_vs_oracle(pkg, kind):
    w, h = 3840, 2160
    rng = np.random.default_rng(7 + len(kind))
    frame = pu.synthetic_yuyv(rng, w, h, kind)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    coded_bands = pu.oracle_forward_422(orc, frame, quant, 0)
    want = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        out = np.zeros((3 * h, w), np.int16)
        codec.inverse_host([codec.pack_coded(coded_bands)], quant, pkg.PIXEL_PLANAR16, [out])
        out8 = np.zeros((h, w * 2), np.uint8)
        codec.inverse_host([codec.pack_coded(coded_bands)], quant, pkg.PIXEL_YUYV, [out8])
    got = [out[0:h, :w], out[h:2 * h, :w // 2], out[2 * h:3 * h, :w // 2]]
    for c in range(3):
        assert np.array_equal(got[c], want[c]), f"channel {c}: {np.argwhere(got[c] != want[c])[:4].tolist()}"
    a, b = pu.yuyv_envelope(want)
    assert ((out8 == a) | (out8 == b)).all()


# ------------------------------------------------------------------------------------------------ config 4
@pytest.mark.parametrize("kind", ["natural", "extreme"])
def test_rg48_4k_vs_oracle(pkg, kind):
    w, h = 3840, 2160
    rng = np.random.default_rng(48)
    if kind == "natural":
        tile = fm.synthetic_rg48(rng, w // 2, h // 2, "natural")
        frame = np.tile(tile.reshape(h // 2, w // 2, 3), (2, 2, 1)).reshape(h, w * 3).copy()
        frame[::7, ::5] ^= 0x0155                                           # break the tile symmetry
    else:
        frame = fm.synthetic_rg48(rng, w, h, "extreme")
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_RG48)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    pyr = pu.forward_pyramid_planes(orc, fm.unpack_rg48(frame), quant.table(3), tuple(quant.prescale))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        coded = codec.forward_host([frame], quant)[0]
        pu.assert_bands(codec.unpack_coded(coded), pyr, "RG48 4K")
        if kind == "natural":
            coded_bands = {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}
            want = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale))
            out = np.zeros((3 * h, w), np.int16)
            codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [out])
            for c in range(3):
                assert np.array_equal(out[c * h:(c + 1) * h], want[c]), f"inverse channel {c}"


# ------------------------------------------------------------------------------------------------ config 5
@pytest.mark.parametrize("fmt,kind", [(0, "natural"), (3, "random")])
def test_byr4_8k_vs_oracle(pkg, fmt, kind):
    w, h = 7680, 4320
    rng = np.random.default_rng(8000 + fmt)
    if kind == "natural":
        tile = fm.mosaic_from_rg48(fm.synthetic_rg48(rng, w // 4, h // 4, "natural"), fmt)       # 1920 x 1080 mosaic
        bayer = np.tile(tile, (4, 4)).copy()
        bayer[::6, ::10] ^= 0x0230
    else:
        bayer = rng.integers(0, 65536, (h, w)).astype(np.uint16)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    pyr = pu.forward_pyramid_planes(orc, fm.unpack_byr4(bayer, fmt), quant.table(4), tuple(quant.prescale))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        codec.set_bayer_phase(fmt)
        coded = codec.forward_host([bayer], quant)[0]
        pu.assert_bands(codec.unpack_coded(coded), pyr, "BYR4 8K")
        if kind == "natural":
            coded_bands = {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}
            want = pu.inverse_pyramid(orc, coded_bands, quant.table(4), tuple(quant.prescale), nchan=4)
            ph, pw = h // 2, w // 2
            out = np.zeros((4 * ph, w), np.int16)
            codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [out])
            for c in range(4):
                assert np.array_equal(out[c * ph:(c + 1) * ph, :pw], want[c]), f"inverse channel {c}"


# ------------------------------------------------------------------------------------------------ the north star's frames
@needs_ref
@pytest.mark.parametrize("size", [(1920, 1080), (3840, 2160)])
def test_qbist_frames_1_to_10_vs_reference_encoder(pkg, size):
    """GPU bands == transform[c]->wavelet[k]->band[b] of the unmodified reference after its real EncodeSample, for the
    ten frames TestCFHD -D encodes (QBIST_SEED 50), FILMSCAN1, 4:2:2; batch of 10 through one launch sequence."""
    w, h = size
    ref_lib = ol.load_ref()
    frames = pu.qbist_yuy2_sequence(ref_lib, w, h, 10)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 10) as codec:
        coded = codec.forward_host(frames, quant)
        for i, f in enumerate(frames):
            bands_ref, div, prescale, sample = pu.ref_encode_frame(ref_lib, f, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, 4)
            assert div == quant.table(3) and prescale[0] == list(quant.prescale)
            if (w, h) == (1920, 1080):          # known-answer sample sizes of TestCFHD -D (BASELINE.md; metadata varies by ~100 B)
                kat = (592268, 587816, 287344, 529388, 490096, 461736, 402808, 362904, 262468, 259744)
                assert kat[i] - sample.size == 144, (i, sample.size)   # Codec-level sample = the SDK's minus its 144 metadata bytes
            pu.assert_bands(codec.unpack_coded(coded[i]), bands_ref, f"Qbist frame {i + 1} {w}x{h}")
