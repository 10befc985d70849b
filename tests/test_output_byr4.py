"""BYR4 output of a Bayer sample, CPU side: the restated decode "decoder bands -> mosaic" (formats.row16u per channel, then
oracle/cfhd_oracle_bayer.c orc_bayer_to_byr4) equals the reference decoder's DECODED_FORMAT_BYR4 frame byte for byte, live against
oracle/_ref and from the committed fixtures; the restated linear-restore table equals the one the reference built; and the
phase and curve mode really enter the expected frames."""
import glob
import os

import numpy as np
import pytest

import byr4_out_util as b4
import formats as fm
import oracle_lib as ol
import parity_util as pu

needs_ref = pytest.mark.skipif(not (ol.ref_available() and b4.ref_bayer_available()), reason="oracle/_ref not built (reference absent)")
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decoded_byr4_*.npz")))

# mosaic sizes; plane / level-1 band widths 96 / 48, 104 / 52, 120 / 60, 136 / 68, 256 / 128, 360 / 180: the ...ToRow16u scalar
# tail (band columns from w - w % 8 - 9 on) is 9, 13, 13, 13, 9 and 13 columns wide, next to an SSE2 loop of 2 .. 20 groups
SIZES = [(192, 96), (208, 96), (240, 112), (272, 96), (512, 128), (720, 112)]


def fixture_bands(z):
    return {(int(c), int(k), b): z[key] for key in z.files if key.startswith("d_") for c, k, b in [key.split("_")[1:]]}


def _mismatch(got, want):
    bad = np.argwhere(got != want)
    return f"{bad.shape[0]} samples differ, first (row, column) {bad[:5].tolist()}"


@needs_ref
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
@pytest.mark.parametrize("phase", [0, 1, 2, 3])
@pytest.mark.parametrize("preset", [0, 1], ids=["restore", "applied"])
def test_oracle_equals_reference_decoder(size, phase, preset):
    w, h = size
    ref = ol.load_ref()
    rng = np.random.default_rng(w + h + 4 * phase + preset)
    # extreme content drives the planes beyond 12 bits, so both ...ToRow16u limits and the [0, 65535] limits of the cell occur
    kind = ("natural", "extreme", "random")[(phase + preset + w // 16) % 3]
    _, _, prescale, sample = b4.ref_encode_byr4(ref, fm.synthetic_mosaic(rng, w, h, kind, phase), phase, preset)
    frame, bands, used, table = b4.ref_decode_byr4(sample, w, h, phase, preset)
    assert used == (phase, preset), "the decoder did not decode with the phase and curve mode under test"
    assert table is not None and np.array_equal(table, fm.restore_table())
    coded = {k: v for k, v in bands.items() if not (k[2] == "LL" and k[1] != 3)}
    want = fm.oracle_byr4(coded, fm.UNIT4, tuple(prescale[0]), phase, table if preset == 0 else None)
    assert np.array_equal(want, frame), f"{w}x{h} phase {phase} preset {preset} {kind}: " + _mismatch(want, frame)
    if kind == "extreme":
        rows = fm.rows16u(pu.inverse_pyramid(ol.oracle(), coded, fm.UNIT4, tuple(prescale[0]), nchan=4))
        assert any((r == 0xfff0).any() for r in rows) and any((r == 0xffff).any() for r in rows), "both ...ToRow16u limits occur"


@needs_ref
def test_oracle_equals_reference_decoder_byr5_padded_height():
    """A sample encoded from BYR5 at 208 x 100: the encoder pads the planes from 50 to 56 rows, the decoder writes 100 rows."""
    w, h, phase = 208, 100, 1
    ref = ol.load_ref()
    packed = fm.byr5_pack(fm.byr5_random_components(np.random.default_rng(3), w // 2, h // 2, "random"))
    _, _, prescale, sample = b4.ref_encode_byr5(ref, packed, w // 2, h // 2, phase)
    for preset in (0, 1):
        frame, bands, used, table = b4.ref_decode_byr4(sample, w, h, phase, preset)
        assert used == (phase, preset)
        coded = {k: v for k, v in bands.items() if not (k[2] == "LL" and k[1] != 3)}
        assert coded[(0, 1, "HH")].shape == (28, 52)
        want = fm.oracle_byr4(coded, fm.UNIT4, tuple(prescale[0]), phase, table if preset == 0 else None)
        assert want.shape == (112, w) and np.array_equal(want[:h], frame), _mismatch(want[:h], frame)


def test_fixtures_present():
    assert len(GOLDEN) == 4
    zs = [np.load(p) for p in GOLDEN]
    assert sorted(int(z["phase"]) for z in zs) == [0, 1, 2, 3] and {int(z["preset"]) for z in zs} == {0, 1}


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_equals_fixture(path):
    z = np.load(path)
    h, phase, preset = int(z["height"]), int(z["phase"]), int(z["preset"])
    if preset == 0:
        assert np.array_equal(z["restore"], fm.restore_table())
    want = fm.oracle_byr4(fixture_bands(z), fm.UNIT4, tuple(int(v) for v in z["prescale"]), phase, z["restore"] if preset == 0 else None)
    assert want.shape[0] == int(z["coded_height"]) and np.array_equal(want[:h], z["frame"]), _mismatch(want[:h], z["frame"])


def test_restore_table_shape():
    t = fm.restore_table().astype(np.int64)
    assert t[0] == 0 and t[-1] == 65516 and np.all(np.diff(t) >= 0)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_phase_and_curve_mode_enter_the_frame(path):
    """Not vacuous: with the fixture's content, any other phase and the other curve mode give another frame."""
    z = np.load(path)
    h, phase, preset = int(z["height"]), int(z["phase"]), int(z["preset"])
    bands, prescale = fixture_bands(z), tuple(int(v) for v in z["prescale"])
    table = fm.restore_table()
    for other in range(4):
        if other != phase:
            got = fm.oracle_byr4(bands, fm.UNIT4, prescale, other, table if preset == 0 else None)
            assert not np.array_equal(got[:h], z["frame"]), f"phase {other} gives the frame of phase {phase}"
    got = fm.oracle_byr4(bands, fm.UNIT4, prescale, phase, None if preset == 0 else table)
    assert not np.array_equal(got[:h], z["frame"]), "the other curve mode gives the same frame"
