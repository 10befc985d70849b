"""Signed planes through the single-level transform (VERDICT round 1, weak 3).

The kernels compute in exact int32, the reference in saturating 16-bit chains; the oracle models the latter.  The two
agree while no chain input exceeds 8190.  Free-standing planes may be signed (the temporal highpass of a two-frame GOP),
so the forward level audits its input and REPORTS a violation (CFB_ERROR_RANGE = 103) instead of silently computing
something the reference would not: in-range signed planes must be bit-exact against the oracle's saturating model,
out-of-range ones must be rejected."""
import numpy as np
import pytest

import oracle_lib as ol
from gpu_fixtures import pkg  # noqa: F401

pytestmark = pytest.mark.gpu


def _check_exact(pkg, plane, prescale, div):
    orc = ol.oracle()
    want = orc.fwd_level(plane, 1 if prescale == 2 else 0, div, 2)
    with pkg.Context(0) as ctx:
        got = ctx.level_forward(plane, prescale, div)
        assert ctx.range_status() == 0
    for g, w_, name in zip(got, want, ("LL", "LH", "HL", "HH")):
        assert np.array_equal(g, w_), name


@pytest.mark.parametrize("shape", [(48, 64), (270, 480), (540, 960)])
@pytest.mark.parametrize("kind", ["random", "extremes", "checker"])
def test_signed_in_range_planes_match_the_saturating_oracle(pkg, shape, kind):
    """|x| <= 2500: horizontal outputs stay below 3.25 * 2500 = 8125 whatever the pattern (6-tap border filter)."""
    h, w = shape
    rng = np.random.default_rng(h + len(kind))
    if kind == "random":
        plane = rng.integers(-2500, 2501, (h, w))
    elif kind == "extremes":
        plane = rng.choice(np.array([-2500, 2500]), (h, w))
    else:
        plane = np.where((np.add.outer(np.arange(h), np.arange(w)) & 1) == 0, 2500, -2500)
    _check_exact(pkg, plane.astype(np.int16), 0, [1, 12, 12, 6])


@pytest.mark.parametrize("prescale", [0, 2])
def test_natural_temporal_difference_is_in_range(pkg, prescale):
    """What wavelet 3 of the two-frame GOP really sees: the difference of two lowpass images (+-4080 by range), smooth."""
    h, w = 540, 960
    y, x = np.mgrid[0:h, 0:w]
    a = 2040 + 2000 * np.sin(x / 37.0) * np.cos(y / 23.0)
    b = 2040 + 2000 * np.sin((x + 40) / 37.0) * np.cos((y - 9) / 23.0)
    _check_exact(pkg, (a - b).astype(np.int16), prescale, [1, 24, 24, 12])


@pytest.mark.parametrize("kind", ["full-range", "worst-case-4080", "one-sample"])
def test_out_of_range_planes_are_rejected(pkg, kind):
    h, w = 96, 256
    rng = np.random.default_rng(len(kind))
    if kind == "full-range":
        plane = rng.integers(-32768, 32768, (h, w))
    elif kind == "worst-case-4080":          # the declared range of a temporal highpass in its worst pattern: the window
        # (-M, -M, M, -M, M, M) gives a horizontal highpass of 4M / 8 + 2M = 10200 > 8190
        plane = np.tile(np.array([-4080, -4080, 4080, -4080, 4080, 4080]), w // 6 + 1)[:w][None, :].repeat(h, 0)
    else:
        plane = np.zeros((h, w), np.int64); plane[40, 100] = 9000
    plane = plane.astype(np.int16)
    with pkg.Context(0) as ctx:
        with pytest.raises(pkg.CfbError) as ei:
            ctx.level_forward(plane, 0, [1, 12, 12, 6])
        assert ei.value.code == 103
        assert ctx.range_status() == 0          # reported once, then cleared
        ok = ctx.level_forward(np.zeros((h, w), np.int16), 0, [1, 12, 12, 6])        # the context stays usable
        assert all(not b.any() for b in ok)
