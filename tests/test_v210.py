"""V210 (10-bit packed 4:2:2) level-1 front end: CPU = the golden bands of the reference's EncodeSample are reproduced
from the unpacked planes by the oracle; GPU = CUDA forward through the C ABI (unpack fused into the load) vs golden and vs
the oracle for every lane phase, strip boundary and size class."""
import glob
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "v210_*.npz")))


def _load(path):
    z = np.load(path)
    bands = {}
    for k in z.files:
        if k.startswith("b_"):
            _, c, lvl, name = k.split("_")
            bands[(int(c), int(lvl), name)] = z[k]
    return z["words"], int(z["width"]), z["divisors"].tolist(), tuple(int(v) for v in z["prescale"]), int(z["quality"]), bands


def unpack_v210(words, w):
    """inverse of formats.pack_v210 -> [Y, ch1 = Cr, ch2 = Cb] int16 planes"""
    comp = np.zeros((words.shape[0], words.shape[1] * 3), np.int16)
    comp[:, 0::3], comp[:, 1::3], comp[:, 2::3] = words & 1023, (words >> 10) & 1023, (words >> 20) & 1023
    comp = comp[:, :2 * w]
    y = np.zeros((words.shape[0], w), np.int16)
    y[:, 0::2], y[:, 1::2] = comp[:, 1::4], comp[:, 3::4]
    return [y, np.ascontiguousarray(comp[:, 2::4]), np.ascontiguousarray(comp[:, 0::4])]


def test_golden_present():
    assert GOLDEN


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_reproduces_v210_golden(path):
    words, w, div, prescale, _, bands = _load(path)
    pyr = pu.forward_pyramid_planes(ol.oracle(), unpack_v210(words, w), div, prescale)
    for key, want in bands.items():
        if not (key[2] == "LL" and key[1] != 3):
            assert np.array_equal(pyr[key], want), f"band {key}"


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_cuda_v210_reproduces_reference_bands(pkg, path):
    words, w, div, prescale, quality, bands = _load(path)
    h = words.shape[0]
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_V210)
    quant = pkg.quant_for_quality(desc, quality)
    assert quant.table(3) == div
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        assert codec.layout.frame_pitch == words.shape[1] * 4
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        codec.forward_host([words], quant, [coded])
        pu.assert_bands(codec.unpack_coded(coded), bands)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(240, 64), (480, 96), (720, 480), (1440, 120), (1920, 1080), (3840, 2160)])
@pytest.mark.parametrize("kind", ["natural", "random"])
def test_cuda_v210_vs_oracle(pkg, size, kind):
    w, h = size
    rng = np.random.default_rng(w + 7 * h)
    if kind == "random":
        y, cb, cr = (rng.integers(0, 1024, (h, w)), rng.integers(0, 1024, (h, w // 2)), rng.integers(0, 1024, (h, w // 2)))
        words = fm.pack_v210(y.astype(np.uint32), cb.astype(np.uint32), cr.astype(np.uint32))
        planes = [y.astype(np.int16), cr.astype(np.int16), cb.astype(np.int16)]
    else:
        words, planes = fm.v210_from_yuyv(pu.synthetic_yuyv(rng, w, h, "natural"), rng)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_V210)
    quant = pkg.quant_for_quality(desc, 4)
    want = pu.forward_pyramid_planes(ol.oracle(), planes, quant.table(3), tuple(quant.prescale), quant.midpoint_prequant)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        coded = [np.zeros(codec.layout.coded_bytes, np.uint8) for _ in range(2)]
        codec.forward_host([words, words[::-1].copy()], quant, coded)
        pu.assert_bands(codec.unpack_coded(coded[0]), want)
