"""The host packer and unpacker of the 'CFS2' sparse format (cfb_sparse_compact / cfb_sparse_expand) against the numpy
restatement in sparse_ref.py, on adversarial coded regions.  CPU only: this pins the reference and the host code to
each other before the GPU kernels are compared with either (test_sparse_kernels_gpu.py)."""
import numpy as np
import pytest

import sparse_ref as sr
from gpu_fixtures import pkg  # noqa: F401

# (source, width, height): the coded regions of the GPU test, with the last block 32 words, all but 32 words, or full
LAYOUTS = [("YUYV", 288, 208), ("YUYV", 224, 304), ("YUYV", 256, 48), ("RG48", 232, 56), ("RG48", 600, 152), ("BYR4", 240, 96)]
LAST_BLOCK = {(288, 208): 32, (224, 304): 8160, (256, 48): 8192, (232, 56): 32, (600, 152): 8160, (240, 96): 8192}


def _layout(pkg, src, w, h):
    return pkg.layout_for(pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + src)))


def _check_region(pkg, lay, name, dense):
    nwords = lay.coded_bytes // 2
    want = sr.compact(nwords, dense)
    got = pkg.sparse_compact(lay, dense.view(np.uint8))
    assert got.tobytes() == want, name                                   # byte for byte, padding included
    assert pkg.sparse_bytes(got) == len(want), name
    assert np.array_equal(sr.expand(nwords, want), dense), name
    assert np.array_equal(pkg.sparse_expand(lay, got).view(np.int16), dense), name
    return want


@pytest.mark.parametrize("src,w,h", LAYOUTS)
def test_reference_equals_host_packer(pkg, src, w, h):
    lay = _layout(pkg, src, w, h)
    nwords = lay.coded_bytes // 2
    assert nwords - (sr.nblocks(nwords) - 1) * sr.BLOCK_WORDS == LAST_BLOCK[(w, h)]
    rng = np.random.default_rng(w * 1000 + h)
    for name, dense in sr.catalogue(nwords, rng):
        _check_region(pkg, lay, name, dense)


def test_reference_equals_host_packer_4k(pkg):
    """2025 blocks: the empty runs reach 300 blocks, and every block kind sits in many positions."""
    lay = _layout(pkg, "YUYV", 3840, 2160)
    nwords = lay.coded_bytes // 2
    rng = np.random.default_rng(4)
    _check_region(pkg, lay, "blocks", sr.region(nwords, sr.BLOCK_KINDS, rng))
    _check_region(pkg, lay, "empty_runs", sr.empty_runs(nwords, rng))


@pytest.mark.parametrize("src,w,h", LAYOUTS)
def test_fully_escaped_region_size(pkg, src, w, h):
    """Every word escaped gives the largest chunk in every block: sparse_max_bytes exactly when the coded region is a whole
    number of blocks, less by what the partial last block does not hold otherwise."""
    lay = _layout(pkg, src, w, h)
    nwords = lay.coded_bytes // 2
    nb = sr.nblocks(nwords)
    sp = _check_region(pkg, lay, "escaped", sr.region(nwords, ["escaped"], np.random.default_rng(1)))
    table = np.frombuffer(sp, np.uint8)[32:32 + 16 * nb].view("<u4").reshape(nb, 4)
    assert (table[:-1, 1:] == (256, 8192, 8192)).all()
    last = nwords - (nb - 1) * sr.BLOCK_WORDS
    assert tuple(table[-1, 1:]) == (last // 32, last, last)
    assert sr.max_bytes(nwords) == pkg.sparse_max_bytes(lay)
    if last == sr.BLOCK_WORDS:
        assert len(sp) == pkg.sparse_max_bytes(lay)
    else:
        assert len(sp) == pkg.sparse_max_bytes(lay) - sr.MAX_CHUNK + sr.chunk_bytes(last // 32, last, last)


def test_escape_boundaries():
    """-128 is the escape byte and must be escaped; -127 and 127 are plain; 128, -32768 and 32767 are escaped."""
    nwords = sr.BLOCK_WORDS
    dense = np.zeros(nwords, np.int16)
    vals = np.array([-128, -127, 127, 128, -32768, 32767, -129, 1, -1], np.int16)
    dense[:vals.size] = vals
    sp = np.frombuffer(sr.compact(nwords, dense), np.uint8)
    c = sp[sr.chunks_offset(1):]
    assert c[:32].tolist() == [1] + [0] * 31
    assert c[32:36].view("<u4")[0] == (1 << vals.size) - 1
    assert c[36:45].view(np.int8).tolist() == [-128, -127, 127, -128, -128, -128, -128, 1, -1]
    assert c[48:58].view("<i2").tolist() == [-128, 128, -32768, 32767, -129]
    assert len(c) == 64 and not c[45:48].any() and not c[58:].any()
    assert np.array_equal(sr.expand(nwords, sp), dense)


def test_reference_rejects_non_canonical():
    """expand() refuses what no packer may write, so that a byte comparison through it cannot pass a wrong encoding."""
    nwords = sr.BLOCK_WORDS
    dense = np.zeros(nwords, np.int16)
    dense[5], dense[40] = 3, -200
    good = bytearray(sr.compact(nwords, dense))
    base = sr.chunks_offset(1)
    bad_plain = bytearray(good); bad_plain[base + 40] = 0                # a plain byte of 0 for a word marked non-zero
    bad_pad = bytearray(good); bad_pad[base + 42] = 1                    # value padding not zero
    bad_wide = bytearray(good); bad_wide[base + 44:base + 46] = np.int16(5).tobytes()     # an escape that fits a byte
    for bad in (bad_plain, bad_pad, bad_wide):
        with pytest.raises(sr.FormatError):
            sr.expand(nwords, bytes(bad))


def test_catalogue_is_adversarial():
    """The generator produces what its names promise (a generator gone quiet would make every comparison vacuous)."""
    rng = np.random.default_rng(0)
    esc = sr.block("escaped", rng)
    assert (esc != 0).all() and ((esc < -127) | (esc > 127)).all()
    assert {-32768, 32767, -128, 128, -129} == set(esc.tolist())
    assert len(sr._block_chunk(esc)[0]) == sr.MAX_CHUNK
    plain = sr.block("plain", rng)
    assert (plain != 0).all() and (np.abs(plain.astype(np.int32)) <= 127).all()
    assert set(sr.block("boundary", rng).tolist()) == {0, -128, -127, 127, 128}
    grp = sr.block("per_group", rng).reshape(256, 32)
    assert ((grp != 0).sum(axis=1) == 1).all()
    for p in sr.SINGLE_POSITIONS:
        assert np.flatnonzero(sr.block(f"single{p}", rng)).tolist() == [p]
    nwords = 17 * sr.BLOCK_WORDS - 32
    runs = sr.empty_runs(40 * sr.BLOCK_WORDS, rng).reshape(40, -1).any(axis=1)
    assert runs.tolist() == [True, False, True] + [False] * 31 + [True] + [False] * 4 + [True]
    names = [n for n, _ in sr.catalogue(nwords, rng)]
    assert len(names) == len(set(names))
