"""Sparse transfer format of the coded region: host conversion utilities (CPU) and GPU compaction/expansion."""
import numpy as np
import pytest

import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401


@pytest.mark.parametrize("density", [0.0, 0.02, 0.3, 1.0])
def test_host_compact_expand_roundtrip(pkg, density):
    lay = pkg.layout_for(pkg.FrameDesc(704, 96, pkg.PIXEL_YUYV))
    rng = np.random.default_rng(int(density * 100))
    words = lay.coded_bytes // 2
    dense = np.zeros(words, np.int16)
    nz = rng.random(words) < density
    dense[nz] = rng.integers(-3000, 3000, int(nz.sum())).astype(np.int16)
    dense[nz & (dense == 0)] = 7
    dense_u8 = dense.view(np.uint8)
    sp = pkg.sparse_compact(lay, dense_u8)
    assert pkg.sparse_bytes(sp) == sp.size
    hdr = sp[:16].view(np.uint32)
    nblocks = (words + 8191) // 8192
    assert hdr[0] == 0x32534643 and hdr[1] == words and hdr[2] == sp.size and hdr[3] == nblocks        # 'CFS2'
    table = sp[32:32 + 16 * nblocks].view(np.uint32).reshape(nblocks, 4)
    assert int(table[:, 2].sum()) == int((dense != 0).sum())
    assert int(table[:, 3].sum()) == int((np.abs(dense.astype(np.int32)) > 127).sum())
    back = pkg.sparse_expand(lay, sp)
    assert np.array_equal(back, dense_u8)
    if density == 0.0:
        assert sp.size < lay.coded_bytes // 500         # header + block table only
    bad = sp.copy(); bad[0] ^= 1
    with pytest.raises(pkg.CfbError):
        pkg.sparse_expand(lay, bad)


@pytest.mark.parametrize("size", [(704, 96), (720, 480), (1920, 1080)])
def test_host_compact_from_band_buffers(pkg, size):
    """cfb_sparse_compact_bands: one buffer per band with its own pitch and garbage behind the band's width (what an
    entropy decoder leaves in wavelet->band[]) gives the bytes cfb_sparse_compact gives for the clean dense region."""
    w, h = size
    lay = pkg.layout_for(pkg.FrameDesc(w, h, pkg.PIXEL_YUYV))
    rng = np.random.default_rng(w)
    bands, clean = {}, {}
    for c in range(lay.num_channels):
        for k in range(3):
            for b in range(4):
                if b == 0 and k != 2:
                    continue
                bl = lay.band[c][k][b]
                pitch_words = bl.pitch // 2 + 8 * ((c + k + b) % 3)             # some bands with a wider pitch than the layout's
                buf = rng.integers(-999, 999, (bl.height, pitch_words)).astype(np.int16)       # garbage everywhere ...
                data = np.where(rng.random((bl.height, bl.width)) < 0.07, rng.integers(-2000, 2000, (bl.height, bl.width)), 0).astype(np.int16)
                buf[:, :bl.width] = data                                        # ... except the band itself
                bands[(c, k + 1, pkg.BAND_NAMES[b])] = buf[:, :bl.width]        # a view: the row stride stays pitch_words
                clean[(c, k + 1, pkg.BAND_NAMES[b])] = data
    want = pkg.sparse_compact(lay, pkg.pack_coded(lay, clean))
    got = pkg.sparse_compact_bands(lay, bands)
    assert np.array_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("size,kind", [((704, 96), "natural"), ((704, 96), "random"), ((1920, 1080), "natural"), ((256, 64), "constant")])
def test_gpu_sparse_matches_dense(pkg, size, kind):
    w, h = size
    rng = np.random.default_rng(w)
    frames = [pu.synthetic_yuyv(rng, w, h, kind) for _ in range(3)]
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 3) as codec:
        dense = codec.forward_host(frames, quant)
        sparse, sizes = codec.forward_host_sparse(frames, quant)
        for d, s, n in zip(dense, sparse, sizes):
            assert pkg.sparse_bytes(s) == n
            assert np.array_equal(pkg.sparse_expand(codec.layout, s), d)                 # lossless
            assert np.array_equal(pkg.sparse_compact(codec.layout, d), s[:n])            # same bytes as the host packer
        out_d = [np.zeros((h, w * 2), np.uint8) for _ in frames]
        out_s = [np.zeros((h, w * 2), np.uint8) for _ in frames]
        codec.inverse_host(dense, quant, pkg.PIXEL_YUYV, out_d)
        codec.inverse_host_sparse(sparse, quant, pkg.PIXEL_YUYV, out_s)
        for a, b in zip(out_d, out_s):
            assert np.array_equal(a, b)
        if kind == "natural":
            assert sizes[0] < codec.layout.coded_bytes // 2
