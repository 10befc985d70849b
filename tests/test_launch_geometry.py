"""Host-side model of how the kernels partition a row among warps, lanes and the edge kernels (cfb_forward.cu lane_setup /
k_fwd_plane_edge, cfb_inverse.cu inv_lane writer rule / k_inv_plane_edge): for EVERY width the library accepts, each output column is
produced exactly once, border columns get the border filter exactly once, and every halo word a lane reads lies inside the
row.  The GPU parity tests exercise a few dozen widths; this covers all of them without a GPU.  The same for rows: how a
band's rows are split among warps and streamed through the TMA rings, for every band height."""
import functools

import numpy as np
import pytest

K_STRIP_IN, K_INV_STRIP = 256, 120


def forward_cover(width):
    """-> (columns written by the main kernel, by the edge kernel, lanes flagged right_border, halo reads)"""
    ow = width // 2
    main, halos, right_border = [], [], []
    nstrips = (width + K_STRIP_IN - 1) // K_STRIP_IN
    for strip in range(nstrips):
        for lane in range(32):
            col0 = strip * K_STRIP_IN + lane * 8
            if col0 + 8 > width:
                continue                                    # inactive: not all 8 input columns exist
            main += list(range(col0 // 2, col0 // 2 + 4))
            if col0 + 8 == width:
                right_border.append(col0 // 2 + 3)
            use_lh = lane == 0 and strip > 0
            use_rh = (col0 + 8 < width) and (lane == 31 or col0 + 16 > width)
            if use_lh:
                halos.append((col0 - 2, col0 - 1))
            if use_rh:
                halos.append((col0 + 8, col0 + 9))
            if not (use_rh or col0 + 8 == width):
                assert lane < 31 and col0 + 16 <= width      # right neighbour value comes from an ACTIVE lane
    edge = list(range((width // 8) * 4, ow))
    return main, edge, right_border, halos


@pytest.mark.parametrize("width", list(range(16, 4200, 2)))
def test_forward_row_partition(width):
    ow = width // 2
    main, edge, right_border, halos = forward_cover(width)
    assert sorted(main + edge) == list(range(ow))            # every output column exactly once
    assert len(edge) <= 3
    if width % 8 == 0:
        assert right_border == [ow - 1] and not edge          # the last full lane applies the border filter
    else:
        assert not right_border and edge[-1] == ow - 1        # the edge kernel owns the right border column
    for a, b in halos:
        assert 0 <= a and b < width                           # halo samples exist


def inverse_cover(bw):
    main = []
    nstrips = (bw + K_INV_STRIP - 1) // K_INV_STRIP
    right_border = []
    for strip in range(nstrips):
        for lane in range(32):
            col0 = strip * K_INV_STRIP - 4 + lane * 4
            active = 0 <= col0 < bw
            writer = active and 1 <= lane <= 30 and col0 + 4 <= bw
            if writer:
                main += list(range(col0, col0 + 4))
                if col0 + 4 == bw:
                    right_border.append(col0 + 3)
                else:
                    # its right tap is band column col0 + 4, loaded by the next lane (halo lane 31 included)
                    assert col0 + 4 < bw
            if active:
                # a partial lane loads 8 bytes from col0: must stay inside the band pitch ALIGN16(2 * bw)
                assert 2 * col0 + 8 <= (2 * bw + 15) // 16 * 16
    edge = list(range((bw // 4) * 4, bw))
    return main, edge, right_border


@pytest.mark.parametrize("bw", list(range(6, 2100)))
def test_inverse_row_partition(bw):
    main, edge, right_border = inverse_cover(bw)
    assert sorted(main + edge) == list(range(bw))
    assert len(edge) <= 3
    if bw % 4 == 0:
        assert right_border == [bw - 1] and not edge
    else:
        assert not right_border and edge[-1] == bw - 1


# ------------------------------------------------------------------------------------------------ rows
# The split of a band's rows among warps, and the TMA rings the level-1 kernels stream them through, for every band height
# 6 ... 1100 and every rows-per-warp value pick_th (cfb_api.cu) can return: its candidates 4 ... 16 and, through CFB_TH,
# any value >= 2.  The GPU tests pin a few heights at a few splits (test_row_split_gpu.py); this covers all of them.
TH_MODEL = list(range(2, 21)) + [64]
HEIGHTS = range(6, 1101)
K_TMA_STAGES = 4
INV_RINGS = [(2, 4)]     # (kInvRows, kInvStages) of k_inv_422_tma (cfb_inverse_tma.inl)


def ceil_div(a, b):
    return (a + b - 1) // b


def forward_warp_rows(oh, th, wi):
    """Interior warp wi of a forward level with `oh` output rows (cfb_forward_tma.inl:79-83 and :218-222, the register-fed
    kernels of cfb_forward.cu alike) -> (row pairs jfirst..jlast it streams, LL/LH rows it writes, HL/HH rows it writes),
    or None when it has no rows.  Row pair j feeds LL/LH row j when y0 <= j < y1 (emit_low) and HL/HH row j - 1 when
    j - 1 >= max(y0, 1) (emit_high, :132 / :275)."""
    y0 = wi * th
    if y0 >= oh:
        return None
    y1 = min(y0 + th, oh)
    jfirst, jlast = max(y0 - 1, 0), min(y1, oh - 1)
    hlo = max(y0, 1)
    return (jfirst, jlast), range(max(jfirst, y0), min(jlast + 1, y1)), range(max(jfirst - 1, hlo), jlast)


def inverse_warp_rows(H, th, wi):
    """Interior warp wi of an inverse level with `H` band rows (cfb_inverse.cu:328-329, cfb_inverse_tma.inl:89-90):
    the band rows it outputs, [y0, y1), or None.  Rows 0 and H - 1 belong to the border warps."""
    y0 = max(wi * th, 1)
    y1 = min((wi + 1) * th, H - 1)
    return range(y0, y1) if y0 < y1 else None


def check_ring(events, nchunks, rows_of, consumers=1):
    """Replays the events of one ring and checks the protocol.  events: ("issue", chunk, stage) = the producer's copy of a
    chunk into a stage; ("wait", chunk, stage, parity, consumer) = a consumer's wait on the stage's full barrier;
    ("read", row, chunk, consumer); ("release", stage, parity) = the producer's wait on the stage's empty barrier (CTA ring).
    Returns the rows each consumer read, in order."""
    issued = {}                                     # stage -> chunks copied into it, in order
    waited, where = set(), {}
    reads = {c: [] for c in range(consumers)}
    released = {}                                   # stage -> number of empty-barrier phases the producer waited for
    for ev in events:
        if ev[0] == "issue":
            _, chunk, stage = ev
            assert 0 <= chunk < nchunks and chunk not in where, ev           # each chunk once, none past the last row
            prev = issued.setdefault(stage, [])
            if prev:
                # the stage is overwritten only after every consumer has read every row of the chunk it held ...
                for c in range(consumers):
                    assert set(rows_of(prev[-1])) <= set(reads[c]), (ev, "stage re-issued before its chunk was consumed")
                # ... and, with an empty barrier, after the producer waited for exactly that consumption
                if consumers > 1:
                    assert released.get(stage, 0) == len(prev), (ev, "re-issued without waiting on the empty barrier")
            prev.append(chunk)
            where[chunk] = stage
        elif ev[0] == "wait":
            _, chunk, stage, parity, c = ev
            assert where.get(chunk) == stage, (ev, "waits for a chunk that was not issued into this stage")
            n = issued[stage].index(chunk)
            assert parity == n & 1, (ev, "parity of another phase")            # the n-th copy completes phase n
            waited.add((chunk, c))
        elif ev[0] == "read":
            _, row, chunk, c = ev
            assert (chunk, c) in waited and row in rows_of(chunk), ev
            reads[c].append(row)
        elif ev[0] == "release":
            _, stage, parity = ev
            n = released.get(stage, 0)                  # phase n of the empty barrier = consumption of the n-th copy
            assert parity == n & 1 and n < len(issued.get(stage, [])), (ev, "empty barrier: wrong phase")
            released[stage] = n + 1
    assert sorted(where) == list(range(nchunks))        # every chunk copied ...
    assert all((ch, c) in waited for ch in where for c in range(consumers))     # ... and waited for: nothing in flight at exit
    return reads


def warp_ring_events(nchunks):
    """cfb_forward_tma.inl:90-146 (k_fwd_422_tma), one ring per warp: chunk i = row pair jfirst + i.  Lane 0 issues the
    first kTmaStages pairs, and refills a stage right after the warp has read it."""
    ev = [("issue", s, s) for s in range(K_TMA_STAGES) if s < nchunks]
    stage, parity = 0, 0
    for i in range(nchunks):
        ev += [("wait", i, stage, parity, 0), ("read", i, i, 0)]
        if i + K_TMA_STAGES < nchunks:                  # jj + kTmaStages <= jlast
            ev.append(("issue", i + K_TMA_STAGES, stage))
        stage += 1
        if stage == K_TMA_STAGES:
            stage, parity = 0, parity ^ 1
    return ev


def cta_ring_events(nchunks, nwarps):
    """cfb_forward_tma.inl:230-279 (k_fwd_tma), one ring per CTA of channel warps (SrcRG48: 3, SrcBYR4: 4): every warp reads the
    stage, arrives on its empty barrier; the producer (warp 0, lane 0) waits for that phase before the refill."""
    ev = [("issue", s, s) for s in range(K_TMA_STAGES) if s < nchunks]
    stage, parity = 0, 0
    for j in range(nchunks):
        for w in range(nwarps):
            ev += [("wait", j, stage, parity, w), ("read", j, j, w)]
        if j + K_TMA_STAGES < nchunks:
            ev += [("release", stage, parity), ("issue", j + K_TMA_STAGES, stage)]
        stage += 1
        if stage == K_TMA_STAGES:
            stage, parity = 0, parity ^ 1
    return ev


def inv_ring_events(nrows, R, NS):
    """cfb_inverse_tma.inl:130-174: chunk k = rows qfirst + k*R ... (+ R - 1) of the nrows rows y0 - 1 ... y1 (relative to
    qfirst here).  After the first row of chunk k, lane 0 refills the previous stage with chunk k - 1 + NS."""
    ev = [("issue", s, s) for s in range(NS) if s * R < nrows]
    stage, parity, k = 0, 0, 0
    while k * R < nrows:
        ev.append(("wait", k, stage, parity, 0))
        for i in range(R):
            q = k * R + i
            if i > 0 and q > nrows - 1:                 # q > y1
                break
            ev.append(("read", q, k, 0))
            if i == 0 and k >= 1 and (k - 1 + NS) * R < nrows:
                ev.append(("issue", k - 1 + NS, NS - 1 if stage == 0 else stage - 1))
        stage += 1
        if stage == NS:
            stage, parity = 0, parity ^ 1
        k += 1
    return ev


@functools.lru_cache(maxsize=None)
def forward_rings_ok(nchunks):
    one = lambda c: [c]
    assert check_ring(warp_ring_events(nchunks), nchunks, one)[0] == list(range(nchunks))
    for nw in (3, 4):
        reads = check_ring(cta_ring_events(nchunks, nw), nchunks, one, nw)
        assert all(r == list(range(nchunks)) for r in reads.values())
    return True


@functools.lru_cache(maxsize=None)
def inverse_rings_ok(nrows):
    for R, NS in INV_RINGS:
        nchunks = ceil_div(nrows, R)
        reads = check_ring(inv_ring_events(nrows, R, NS), nchunks, lambda c: range(c * R, min(c * R + R, nrows)))
        assert reads[0] == list(range(nrows)), (R, NS, nrows)       # rows y0 - 1 ... y1, each once, in order
    return True


@pytest.mark.parametrize("th", TH_MODEL)
def test_forward_rows_split_and_rings(th):
    for oh in HEIGHTS:
        low, high = np.zeros(oh, np.int32), np.zeros(oh, np.int32)
        warps = ceil_div(ceil_div(oh, th), 4) * 4     # interior warps of gridDim.y - 1 CTA rows (cfb_forward.cu:1370)
        assert ceil_div(oh, th) <= warps              # every warp with rows exists; the CTA-ring kernels launch ceil(oh / th) CTA rows
        for wi in range(warps):
            r = forward_warp_rows(oh, th, wi)
            if r is None:
                assert wi >= ceil_div(oh, th)
                continue
            (jfirst, jlast), lo, hi = r
            low[lo.start:lo.stop] += 1
            high[hi.start:hi.stop] += 1
            forward_rings_ok(jlast - jfirst + 1)
        high[[0, oh - 1]] += 1                        # the border CTA row (k_fwd_422_tma, k_fwd_plane; k_fwd_tma_border<SRC> on a CTA row of its own)
        assert (low == 1).all(), (oh, np.flatnonzero(low != 1)[:8])
        assert (high == 1).all(), (oh, np.flatnonzero(high != 1)[:8])


@pytest.mark.parametrize("th", TH_MODEL)
def test_inverse_rows_split_and_ring(th):
    for H in HEIGHTS:
        out = np.zeros(H, np.int32)
        warps = ceil_div(ceil_div(H, th), 4) * 4      # cfb_inverse.cu:1011 inv_grid
        for wi in range(warps):
            rows = inverse_warp_rows(H, th, wi)
            if rows is None:
                continue
            out[rows.start:rows.stop] += 1
            inverse_rings_ok(rows.stop - (rows.start - 1) + 1)    # nrows = y1 - qfirst + 1
        out[[0, H - 1]] += 1                          # border warps
        assert (out == 1).all(), (H, np.flatnonzero(out != 1)[:8])


@pytest.mark.parametrize("rule", ["no refill", "refill one chunk behind", "skip parity flip"])
def test_ring_model_rejects_broken_schedules(rule):
    """The checker itself: schedules with the mistakes a ring can make are refused."""
    ev = warp_ring_events(11)
    if rule == "no refill":
        ev = [e for e in ev if not (e[0] == "issue" and e[1] >= K_TMA_STAGES)]
    elif rule == "refill one chunk behind":
        ev = [("issue", e[1] - 1, e[2]) if e[0] == "issue" and e[1] >= K_TMA_STAGES else e for e in ev]
    else:
        ev = [("wait", e[1], e[2], 0, e[4]) if e[0] == "wait" else e for e in ev]
    with pytest.raises(AssertionError):
        check_ring(ev, 11, lambda c: [c])
