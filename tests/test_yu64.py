"""YU64 (16-bit packed 4:2:2) level-1 front end: CPU = oracle vs the golden bands of the reference's EncodeSample;
GPU = CUDA forward through the C ABI vs golden and vs the oracle at several sizes, then decode to 8-bit / planes."""
import glob
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "yu64_*.npz")))


def _load(path):
    z = np.load(path)
    bands = {}
    for k in z.files:
        if k.startswith("b_"):
            _, c, lvl, name = k.split("_")
            bands[(int(c), int(lvl), name)] = z[k]
    return z["frame16"], z["divisors"].tolist(), tuple(int(v) for v in z["prescale"]), int(z["quality"]), bands


def test_golden_present():
    assert GOLDEN


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_reproduces_yu64_golden(path):
    frame16, div, prescale, _, bands = _load(path)
    pyr = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_yu64(frame16), div, prescale)
    for key, want in bands.items():
        if not (key[2] == "LL" and key[1] != 3):
            assert np.array_equal(pyr[key], want), f"band {key}"


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_cuda_yu64_reproduces_reference_bands(pkg, path):
    frame16, div, prescale, quality, bands = _load(path)
    h, w2 = frame16.shape
    desc = pkg.FrameDesc(w2 // 2, h, pkg.PIXEL_YU64)
    quant = pkg.quant_for_quality(desc, quality)
    assert quant.table(3) == div
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        codec.forward_host([frame16], quant, [coded])
        pu.assert_bands(codec.unpack_coded(coded), bands)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(192, 48), (256, 64), (448, 120), (704, 96), (1920, 1080), (3840, 2160)])
@pytest.mark.parametrize("kind", ["natural", "random"])
def test_cuda_yu64_vs_oracle(pkg, size, kind):
    w, h = size
    rng = np.random.default_rng(w + 3 * h)
    if kind == "random":
        frame16 = rng.integers(0, 65536, (h, 2 * w)).astype(np.uint16)
    else:
        frame16 = fm.yu64_from_yuyv(pu.synthetic_yuyv(rng, w, h, "natural"), rng)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YU64)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    want = pu.forward_pyramid_planes(orc, fm.unpack_yu64(frame16), quant.table(3), tuple(quant.prescale), quant.midpoint_prequant)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        coded = [np.zeros(codec.layout.coded_bytes, np.uint8) for _ in range(2)]
        codec.forward_host([frame16, frame16[::-1].copy()], quant, coded)       # batch of two different frames
        got = codec.unpack_coded(coded[0])
        pu.assert_bands(got, want)
        # decode: 10-bit planes equal the oracle's inverse of the same bands; 8-bit output is the usual envelope
        coded_bands = {k: v for k, v in want.items() if not (k[2] == "LL" and k[1] != 3)}
        planes = pu.inverse_pyramid(orc, coded_bands, quant.table(3), tuple(quant.prescale))
        out = np.zeros((3 * h, w), np.int16)
        codec.inverse_host([coded[0]], quant, pkg.PIXEL_PLANAR16, [out])
        for c, pl in enumerate([out[0:h, :w], out[h:2 * h, :w // 2], out[2 * h:3 * h, :w // 2]]):
            assert np.array_equal(pl, planes[c]), f"plane {c}"
        if kind == "natural":
            src = fm.unpack_yu64(frame16)
            assert pu.psnr(np.clip(planes[0], 0, 1023) >> 2, src[0] >> 2) > 40.0
