"""Quantisation with a distinct divisor per channel, level and band, at every midpoint rule (CPU side).

The built-in schedules give LH and HL the same divisor at every progressive level, give both chroma channels the same
divisors, use midpoint rule 2 (detail bits 0) and keep every level-2 / level-3 divisor far below 256.  A kernel that
picked the wrong band's, channel's or level's divisor, ignored `midpoint_prequant`, or mis-dequantised with a divisor
above 255 would pass every test built on them.  This file defines the tables that tell those apart (shared with
test_quant_tables_gpu.py) and pins the oracle that the GPU tests compare against:

  * the oracle's level functions equal the reference's at rows of these tables, LL > 1 included, at all four midpoints;
  * the oracle pyramid equals the reference's real encoder at detail bits 1, 6 and 7 (midpoints 3, 8 and 0), progressive
    and interlaced, packed and planar;
  * every mutation of a table that a kernel could make -- two bands, two channels or two levels exchanged, another
    midpoint -- changes the oracle's result for the frames the GPU tests use, so those tests cannot pass vacuously.
"""
import copy
import importlib

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from test_interlaced_planar import make_source, planar_fields_pyramid

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")

# ------------------------------------------------------------------------------------------------ tables
# T_SMALL[c][k] = [LL, LH, HL, HH] of channel c (4 rows: BYR4 has four channels), level k + 1.  Every highpass divisor
# is <= 255, so every inverse launch takes the dp2a dequantiser (SMALLDQ = true).  Within a (channel, level) the three
# highpass divisors differ, at a (level, band) the four channels differ, and the levels differ; the table holds 1, 2, 3,
# primes (5, 7, 11, 13, 17, 19, 29, 31, 83, 97, 101, 131) and 255.  Levels 2 and 3 stay small enough that their bands
# keep non-zero values (test_tables_are_not_vacuous).
T_SMALL = [
    [[1, 2, 3, 5], [1, 19, 24, 31], [1, 60, 255, 97]],
    [[1, 11, 1, 6], [1, 40, 27, 22], [1, 120, 71, 200]],
    [[1, 4, 9, 13], [1, 29, 36, 45], [1, 83, 150, 64]],
    [[1, 7, 10, 17], [1, 33, 21, 50], [1, 101, 180, 131]],
]
# T_BIG: one highpass divisor per level above 255, on a different channel at each level, so every inverse launch (it
# takes the largest divisor of all channels of its level) runs the full-multiply dequantiser (SMALLDQ = false).
T_BIG = copy.deepcopy(T_SMALL)
T_BIG[2][0][3] = 1000           # level 1, channel 2, HH
T_BIG[1][1][2] = 256            # level 2, channel 1, HL
T_BIG[0][2][1] = 257            # level 3, channel 0, LH
TABLES = {"small": T_SMALL, "big": T_BIG}

# midpoint_prequant g of detail bits 0, 1, 6, 7 (quality bits 17-19): g = detail + 2, and 9 maps to 0 (quantize.c)
MIDPOINTS = (2, 3, 8, 0)
DETAIL_OF_MIDPOINT = {2: 0, 3: 1, 8: 6, 0: 7}


def table(name, nchan=3):
    return copy.deepcopy(TABLES[name][:nchan])


def with_ll(t):
    """LL divisors > 1: 3 or 5 at every level.  The unprescaled planar filter quantises LL with them (level 1 of planar
    sources, level 3 of 10-bit sources); the prescaled levels and the packed 4:2:2 filter leave LL alone."""
    t = copy.deepcopy(t)
    for c, row in enumerate(t):
        row[0][0], row[1][0], row[2][0] = (3, 5)[c % 2], 3, (5, 3)[c % 2]
    return t


# ------------------------------------------------------------------------------------------------ frames of the GPU tests
SIZES = [(1024, 136), (720, 200), (208, 56), (1920, 1080)]      # fused L1+L2 (W % 32 == 0), unfused, small, HD


def frame_yuyv(w, h):
    return pu.synthetic_yuyv(np.random.default_rng(w * 3 + h), w, h, "random")


def frame_interlaced(w, h):
    return pu.synthetic_yuyv(np.random.default_rng(w * 5 + h), w, h, "random")


def frame_rg48(w, h):
    return fm.synthetic_rg48(np.random.default_rng(w * 7 + h), w, h, "random")


def frame_byr4(w, h):
    """(w, h) is the mosaic size; the four planes are w/2 x h/2."""
    return np.random.default_rng(w * 11 + h).integers(0, 65536, (h, w)).astype(np.uint16)


def source_422(fmt, w, h):
    """YU64 / V210 source: (frame, [Y, ch1, ch2] 10-bit planes)."""
    src, planes, _ = make_source(fmt, w, h, np.random.default_rng(w * 13 + h + len(fmt)), "random")
    return src, planes


def rgb30_components(w, h):
    return [np.random.default_rng(w * 17 + h + i).integers(0, 1024, (h, w)).astype(np.uint32) for i in range(3)]


# ------------------------------------------------------------------------------------------------ oracle results
def coded(pyr):
    """The coded bands of a pyramid: LL3 and every highpass band."""
    return {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}


def fwd_422(orc, frame, t, prescale, midpoint, uyvy=False, interlaced=False):
    return coded(pu.forward_pyramid_422(orc, frame, t, prescale, int(uyvy), midpoint, interlaced=interlaced))


def fwd_planes(orc, planes, t, prescale, midpoint, interlaced=False):
    build = planar_fields_pyramid if interlaced else pu.forward_pyramid_planes
    return coded(build(orc, planes, t, prescale, midpoint))


def int16_safe(bands, t):
    """Every dequantised highpass value fits int16 (the reference's FSM stores (short)(v * quant): parity holds only
    there)."""
    for (c, lvl, name), v in bands.items():
        if name != "LL":
            d = t[c][lvl - 1][pu.BAND_NAMES.index(name)]
            m = int(np.abs(v.astype(np.int64)).max()) * max(d, 1)
            if m > 32767:
                return False
    return True


def differs(a, b):
    if isinstance(a, dict):
        return any(not np.array_equal(a[k], b[k]) for k in a)
    return any(not np.array_equal(x, y) for x, y in zip(a, b))


def mutations(t):
    """Every table a kernel reading the wrong divisor would effectively use: two highpass bands of one (channel, level)
    exchanged, two channels exchanged at one level, or one (channel, level) taking the next level's row."""
    nchan = len(t)
    for c in range(nchan):
        for k in range(3):
            for a, b in ((1, 2), (2, 3), (1, 3)):
                m = copy.deepcopy(t)
                m[c][k][a], m[c][k][b] = m[c][k][b], m[c][k][a]
                yield f"channel {c} level {k + 1} {pu.BAND_NAMES[a]}<->{pu.BAND_NAMES[b]}", m
            m = copy.deepcopy(t)
            m[c][k][1:] = t[c][(k + 1) % 3][1:]
            yield f"channel {c} level {k + 1} takes level {(k + 1) % 3 + 1}'s divisors", m
    for k in range(3):
        for a, b in ((1, 2), (0, 1)):
            m = copy.deepcopy(t)
            m[a][k], m[b][k] = m[b][k], m[a][k]
            yield f"level {k + 1} channels {a}<->{b}", m


# ------------------------------------------------------------------------------------------------ CPU tests
def test_launch_selection_preconditions():
    """T_SMALL keeps every launch on the dp2a dequantiser, T_BIG puts every launch on the full multiply (the rule of
    launch_inv_plane / launch_inv_422 / launch_inv_444, cfb_inverse.cu: dq_small() = every highpass divisor of the
    launch's channels <= 255), for 3 and 4 channels."""
    for nchan in (3, 4):
        for k in range(3):
            assert max(T_SMALL[c][k][b] for c in range(nchan) for b in (1, 2, 3)) <= 255
            assert max(T_BIG[c][k][b] for c in range(nchan) for b in (1, 2, 3)) > 255
    for t in (T_SMALL, T_BIG):
        for c in range(4):
            for k in range(3):
                assert len(set(t[c][k][1:])) == 3, (c, k)
                for b in (1, 2, 3):
                    assert len({t[cc][k][b] for cc in range(4)}) == 4, (k, b)
        assert len({tuple(t[0][k]) for k in range(3)}) == 3
    values = {d for per_c in T_SMALL for per_k in per_c for d in per_k[1:]}
    assert {1, 2, 3, 255} <= values and 97 in values


@needs_ref
@pytest.mark.parametrize("midpoint", MIDPOINTS)
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("shape", [(24, 64), (24, 100), (40, 240), (32, 482)])   # band widths 32 / 50 / 120 / 241
def test_fwd_level_rows_match_reference(midpoint, variant, shape):
    """ref_fwd_level (the plain and the prescaled planar filter) at every row of the tables, LL > 1 included: the oracle
    maps LL / LH / HL / HH to divisor 0 / 1 / 2 / 3, quantises LL only in the plain filter, and applies the midpoint
    in the SSE2 columns and the scalar tail alike."""
    orc, ref = ol.oracle(), ol.ref()
    h, w = shape
    plane = np.random.default_rng(w * 31 + h).integers(0, 4096, (h, w)).astype(np.int16)
    rows = {tuple(r) for t in (T_BIG, with_ll(T_SMALL)) for per_c in t for r in per_c}
    for quant in sorted(rows):
        bo = orc.fwd_level(plane, variant, list(quant), midpoint)
        br = ref.fwd_level(plane, variant, list(quant), midpoint)
        for b, (x, y) in enumerate(zip(bo, br)):
            assert np.array_equal(x, y), f"divisors {quant} band {pu.BAND_NAMES[b]}"


@needs_ref
@pytest.mark.parametrize("midpoint", MIDPOINTS)
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("shape", [(24, 128), (32, 208)])       # chroma band widths 32 (no scalar tail) / 52 (tail of 4)
def test_fwd_level_422_rows_match_reference(midpoint, fmt, shape):
    """ref_fwd_level_422 on YUYV / UYVY for channels 0, 1, 2, each with its own rows of the tables (LL > 1 included,
    which the packed filter must not quantise)."""
    orc, ref = ol.oracle(), ol.ref()
    h, w = shape
    frame = np.random.default_rng(h * w + fmt).integers(0, 256, (h, w * 2)).astype(np.uint8)
    for t in (T_BIG, with_ll(T_SMALL)):
        for c in range(3):
            for k in range(3):
                bo = orc.fwd_level_422(frame, c, fmt, t[c][k], midpoint=midpoint)
                br = ref.fwd_level_422(frame, c, fmt, t[c][k], midpoint=midpoint)
                for b, (x, y) in enumerate(zip(bo, br)):
                    assert np.array_equal(x, y), f"channel {c} divisors {t[c][k]} band {pu.BAND_NAMES[b]}"


def _ref_encode(ref_lib, src, w, h, color_format, sampling_444, quality, interlaced):
    ref_lib.ref_set_interlaced(int(interlaced))
    try:
        return pu.ref_encode_frame(ref_lib, src, w, h, color_format, sampling_444, 3, quality)
    finally:
        ref_lib.ref_set_interlaced(0)


@needs_ref
@pytest.mark.parametrize("detail", [1, 6, 7])
@pytest.mark.parametrize("case", ["yuyv", "yuyv-interlaced", "rg48", "yu64-interlaced", "v210-interlaced"])
def test_oracle_matches_reference_encoder_at_midpoint(detail, case):
    """The reference's real EncodeSample at quality 4 | detail << 17 (midpoint_prequant 3, 8, 0): its divisor table and
    midpoint equal cfb_quant_for_source's, and the oracle pyramid under that quantisation equals every band it left
    behind.  Covers the packed 8-bit path, the packed field transform (its HL rounds with divisor / g and no "- 1"), the
    planar field transform of 16-bit / 10-bit sources (LH rounds with divisor / 2 at every g) and 12-bit RGB."""
    pkg = importlib.import_module("cineform-sdk_b200")
    ref_lib, orc = ol.load_ref(), ol.oracle()
    quality = 4 | (detail << 17)
    g = {1: 3, 6: 8, 7: 0}[detail]
    interlaced = case.endswith("interlaced")
    if case.startswith("yuyv"):
        w, h = 448, 96
        src = pu.synthetic_yuyv(np.random.default_rng(detail), w, h, "natural")
        if interlaced:
            src[1::2] = np.roll(src[1::2], 6, axis=1)
        bands_ref, div, prescale, _ = _ref_encode(ref_lib, src, w, h, pu.COLOR_FORMAT_YUYV, 0, quality, interlaced)
        quant = pkg.quant_for_quality(pkg.FrameDesc(w, h, pkg.PIXEL_YUYV), quality, interlaced=interlaced)
        want = fwd_422(orc, src, quant.table(3), tuple(quant.prescale), quant.midpoint_prequant, interlaced=interlaced)
    elif case == "rg48":
        w, h = 320, 64
        frame = frame_rg48(w, h)
        bands_ref, div, prescale, _ = _ref_encode(ref_lib, frame.view(np.uint8), w, h, pu.COLOR_FORMAT_RG48, 1, quality, False)
        quant = pkg.quant_for_quality(pkg.FrameDesc(w, h, pkg.PIXEL_RG48), quality)
        want = fwd_planes(orc, fm.unpack_rg48(frame), quant.table(3), tuple(quant.prescale), quant.midpoint_prequant)
    else:
        fmt = case.split("-")[0]
        w, h = (208, 48) if fmt == "yu64" else (240, 48)      # chroma rows with a scalar tail
        src, planes, color_format = make_source(fmt, w, h, np.random.default_rng(detail + len(fmt)), "natural")
        bands_ref, div, prescale, _ = _ref_encode(ref_lib, src.view(np.uint8), w, h, color_format, 0, quality, True)
        quant = pkg.quant_for_quality(pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + fmt.upper())), quality, interlaced=True)
        want = fwd_planes(orc, planes, quant.table(3), tuple(quant.prescale), quant.midpoint_prequant, interlaced=True)
    assert quant.midpoint_prequant == g
    assert quant.table(3) == div and list(quant.prescale) == prescale[0]
    for key in want:
        assert np.array_equal(want[key], bands_ref[key]), f"{case} detail {detail} band {key}: {np.argwhere(want[key] != bands_ref[key])[:4].tolist()}"


def _cases_for_vacuity():
    """(name, forward(t, midpoint) -> coded bands, inverse(bands, t) -> planes, nchan) for the frames of the GPU tests."""
    orc = ol.oracle()
    out = []
    for w, h in SIZES:
        f = frame_yuyv(w, h)
        out.append((f"YUYV {w}x{h}", lambda t, m, f=f: fwd_422(orc, f, t, (0, 2, 0), m),
                    lambda b, t: pu.inverse_pyramid(orc, b, t, (0, 2, 0)), 3))
    w, h = 720, 200
    fi = frame_interlaced(w, h)
    out.append((f"interlaced YUYV {w}x{h}", lambda t, m: fwd_422(orc, fi, t, (0, 2, 0), m, interlaced=True),
                lambda b, t: pu.inverse_pyramid(orc, b, t, (0, 2, 0), interlaced=True), 3))
    _, planes = source_422("yu64", w, h)
    out.append((f"interlaced YU64 {w}x{h}", lambda t, m: fwd_planes(orc, planes, t, (0, 2, 0), m, interlaced=True), None, 3))
    rg = fm.unpack_rg48(frame_rg48(w, h))
    out.append((f"RG48 {w}x{h}", lambda t, m: fwd_planes(orc, rg, t, (0, 2, 2), m),
                lambda b, t: pu.inverse_pyramid(orc, b, t, (0, 2, 2)), 3))
    by = fm.unpack_byr4(frame_byr4(2 * w, 2 * h), 0)
    out.append((f"BYR4 {2 * w}x{2 * h}", lambda t, m: fwd_planes(orc, by, t, (0, 2, 2), m),
                lambda b, t: pu.inverse_pyramid(orc, b, t, (0, 2, 2), nchan=4), 4))
    return out


@pytest.mark.parametrize("name", ["small", "big"])
def test_tables_are_not_vacuous(name):
    """For the frames and sizes of the GPU tests: every coded band is non-zero, the dequantised values fit int16, and
    every mutation of the table (mutations()) or of the midpoint changes the oracle's forward result -- and, with the
    same coefficients, its inverse -- so a kernel that made it cannot match."""
    for what, fwd, inv, nchan in _cases_for_vacuity():
        t = table(name, nchan)
        results = {m: fwd(t, m) for m in MIDPOINTS}
        base = results[2]
        for key, v in base.items():
            assert np.any(v), f"{what}: band {key} is all zero"
        for a in MIDPOINTS:
            for b in MIDPOINTS:
                if a < b:
                    assert differs(results[a], results[b]), f"{what}: midpoints {a} and {b} give the same bands"
        if inv is not None:
            assert int16_safe(base, t), what
            planes = inv(base, t)
        for mut, m in mutations(t):
            assert differs(base, fwd(m, 2)), f"{what}: forward unchanged by {mut}"
            if inv is not None:
                assert differs(planes, inv(base, m)), f"{what}: inverse unchanged by {mut}"
