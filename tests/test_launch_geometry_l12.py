"""Host-side model of the row schedule of the fused forward levels 1 + 2 of packed 4:2:2 (k_fwd_422_l12_tma,
cfb_forward_l12.inl): a warp owns level-2 rows [y0, y1) = level-1 rows [2 y0, 2 y1) and streams level-1 row pairs
2 y0 - 2 ... 2 y1 + 1 through its TMA ring.  For every band height and rows-per-warp value test_launch_geometry.py sweeps:
the streamed pairs lie inside the image, the ring's stages and parities are right and nothing is left in flight, every
level-1 and level-2 output row is written exactly once (by a main warp or by the border-row launch), and every row a warp emits
has the vertical state of the rows it depends on."""
import pytest

from test_launch_geometry import HEIGHTS, TH_MODEL, ceil_div, check_ring, warp_ring_events


def fused_warp_rows(oh2, th, wi):
    """Interior warp wi of a launch whose level-2 band has oh2 rows (level 1: 2 * oh2) -> (jfirst, jlast) and the rows it
    writes: level-1 LL/LH (LH only: LL1 stays in registers), level-1 HL/HH, level-2 LL/LH, level-2 HL/HH, each as a list of
    (row, first pair the state of that row depends on); None when it has no rows."""
    y0 = wi * th
    if y0 >= oh2:
        return None
    y1 = min(y0 + th, oh2)
    Jfirst, Jlast = max(y0 - 1, 0), min(y1, oh2 - 1)
    hlo2 = max(y0, 1)
    jfirst, jlast = 2 * Jfirst, 2 * Jlast + 1
    Y0, Y1 = 2 * y0, 2 * y1
    hlo1 = max(Y0, 1)
    low1, high1, low2, high2 = [], [], [], []
    for j in range(jfirst, jlast + 1):
        if Y0 <= j < Y1:                                    # emit_low
            low1.append((j, j))
        if j - 1 >= hlo1 and j <= Y1:                       # emit_high: HL/HH row j - 1 from pairs j - 2, j - 1, j
            high1.append((j - 1, j - 2))
        if j & 1:                                           # second LL1 row of level-2 pair J
            J = j >> 1
            if y0 <= J < y1:
                low2.append((J, 2 * J))
            if J - 1 >= hlo2:                               # level-2 HL/HH row J - 1 from pairs J - 2, J - 1, J
                high2.append((J - 1, 2 * (J - 2)))
    return (jfirst, jlast), low1, high1, low2, high2


@pytest.mark.parametrize("th", TH_MODEL)
def test_fused_rows_split_and_ring(th):
    for oh1 in HEIGHTS:
        if oh1 % 2 or oh1 < 6:
            continue                                        # the layout's heights are multiples of 8: LL1 rows are even
        oh2 = oh1 // 2
        n1 = {"low": [0] * oh1, "high": [0] * oh1}
        n2 = {"low": [0] * oh2, "high": [0] * oh2}
        warps = ceil_div(ceil_div(oh2, th), 4) * 4          # warps of the ceil(ceil(oh2 / th) / 4) CTA rows (launch_fwd_422_l12)
        for wi in range(warps):
            r = fused_warp_rows(oh2, th, wi)
            if r is None:
                assert wi >= ceil_div(oh2, th)
                continue
            (jfirst, jlast), low1, high1, low2, high2 = r
            assert 0 <= jfirst <= jlast <= oh1 - 1, (oh1, th, wi)           # streamed pairs inside the image
            assert jfirst % 2 == 0                                          # level-2 pairs start on an even LL1 row
            assert check_ring(warp_ring_events(jlast - jfirst + 1), jlast - jfirst + 1, lambda c: [c])[0] == \
                list(range(jlast - jfirst + 1))                             # stages, parities, nothing in flight at exit
            for rows, counts in ((low1, n1["low"]), (high1, n1["high"]), (low2, n2["low"]), (high2, n2["high"])):
                for row, needs in rows:
                    counts[row] += 1
            for row, needs in high1 + low1:
                assert needs >= jfirst, (oh1, th, wi, row)                  # the vertical state was built in this warp
            for row, needs in high2 + low2:
                assert needs >= jfirst, (oh1, th, wi, row)
        # k_fwd_422_l12_border: warps 0 / 1 -> first / last HL1,HH1 row; warps 2 / 3 -> first / last HL2,HH2 row, the latter
        # from LL1 rows 2 (oh2 - 3) ... 2 oh2 - 1 = input rows 4 (oh2 - 3) ... 4 oh2 - 1
        n1["high"][0] += 1; n1["high"][oh1 - 1] += 1
        n2["high"][0] += 1; n2["high"][oh2 - 1] += 1
        assert 4 * (oh2 - 3) >= 0 and 4 * oh2 - 1 <= 2 * oh1 - 1
        for name, counts in (("level 1", n1), ("level 2", n2)):
            for band, c in counts.items():
                bad = [i for i, v in enumerate(c) if v != 1]
                assert not bad, (oh1, th, name, band, bad[:8])

