"""V210 output of 4:2:2 samples (CPU): the numpy restatement formats.pack_v210_output, applied to the oracle's inverse of
the bands the reference decoder held, equals the V210 frame that decoder writes, byte for byte except the one field it
does not determine (X of the last group at W % 6 == 4).  Widths: 480 and 720 (W % 6 == 0; 720 also has ragged level-3
chroma), 704 and 1280 (W % 6 == 2), 640 and 208 (W % 6 == 4)."""
import glob
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decoded_v210_*.npz")))


def _sample_422(ref_lib, w, h, kind):
    rng = np.random.default_rng(w + len(kind))
    frame = pu.qbist_yuy2(ref_lib, w, h, 2) if kind == "qbist" else pu.synthetic_yuyv(rng, w, h, kind)
    _, _, prescale, sample = pu.ref_encode_frame(ref_lib, frame, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, 4)
    return sample, prescale[0]


@needs_ref
@pytest.mark.parametrize("size", [(480, 96), (720, 480), (704, 96), (1280, 96), (640, 96), (208, 48)])
@pytest.mark.parametrize("kind", ["qbist", "extreme"])
def test_v210_rule_matches_reference_decoder(size, kind):
    w, h = size
    ref_lib, orc = ol.load_ref(), ol.oracle()
    sample, prescale = _sample_422(ref_lib, w, h, kind)
    pitch = fm.v210_natural_pitch(w)
    out, bands = pu.ref_decode(ref_lib, sample, w, h, fm.OUTPUTS["V210"].decoded_format, 3, pitch, agree=fm.v210_agree(w, pitch))
    # the decoder's bands for V210 are those of a YU64 decode (the same LL3 constant, decoder.c:12274)
    yu64_bands = pu.ref_decode(ref_lib, sample, w, h, fm.OUTPUTS["YU64"].decoded_format, 3, w * 4)[1]
    for key in bands:
        assert np.array_equal(bands[key], yu64_bands[key]), key
    planes = pu.inverse_pyramid(orc, bands, pu.UNIT_DIVISORS, tuple(prescale))
    want = fm.pack_v210_output(planes)
    got = fm.v210_frame_words(out, w, h)
    m = fm.v210_x_mask(w)
    bad = np.argwhere((got & m) != (want & m))
    assert bad.size == 0, bad[:5].tolist()
    # the reference never writes between ceil(W / 6) * 16 and the pitch: those bytes keep the probe's zero fill
    assert not out[:, fm.v210_row_bytes(w):].any()
    if kind == "extreme":       # both ...ToRow16u limits (1023 << 6 in its SSE2 columns, 65535 in its tail) occur and map to 1023
        r16 = np.concatenate([fm.row16u(p, 10).ravel() for p in planes])
        assert (r16 == 65535).any() and (r16 == 0xFFC0).any()
        assert ((got >> 20) & 0x3FF).max() == 1023 and (got & 0x3FF).min() == 0


def test_partial_group_rules_are_not_vacuous():
    """The tail group rules differ from a plain continuation of the component stream, so the pin above tests them."""
    for w in (704, 640):
        rng = np.random.default_rng(w)
        y = rng.integers(0, 1024, (2, w))
        cr, cb = rng.integers(0, 1024, (2, w // 2)), rng.integers(0, 1024, (2, w // 2))
        words = fm.pack_v210_components(y, cr, cb)
        padded = fm.pack_v210(y, cb, cr)[:, :words.shape[1]]
        assert not np.array_equal(words[:, -4:], padded[:, -4:])
        assert np.array_equal(words[:, :-4], padded[:, :-4])


def test_golden_present():
    assert len(GOLDEN) == 3
    assert sorted(int(os.path.basename(p).split("_")[2].split("x")[0]) % 6 for p in GOLDEN) == [0, 2, 4]


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_reproduces_v210_golden(path):
    """The stored decoder bands -> oracle inverse -> pack_v210_output gives the stored reference frame (X masked)."""
    z = np.load(path)
    w, h = int(z["width"]), int(z["height"])
    bands = {(int(c), int(k), b): z[key] for key in z.files if key.startswith("d_") for c, k, b in [key.split("_")[1:]]}
    planes = pu.inverse_pyramid(ol.oracle(), bands, pu.UNIT_DIVISORS, tuple(int(v) for v in z["prescale"]))
    want = fm.pack_v210_output(planes)
    m = fm.v210_x_mask(w)
    assert np.array_equal(fm.v210_frame_words(z["frame"], w, h) & m, want & m)
    assert not z["frame"][:, fm.v210_row_bytes(w):].any()
