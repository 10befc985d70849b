"""The frame pool (cfb_pool_*) against the synchronous codec on the same device, for every encode source and every decode
output, dense and sparse.

The synchronous entry points are pinned to the oracle and the reference elsewhere; what lies between the pool's queue and
the kernels is not: the grouping of queued jobs into one launch (same direction, sparse / dense mode, out_format, pitch
and quant table), the staging offsets and per-frame pointers of a batch, the output geometry and pitch of the download,
the speculative download of a sparse result and its tail, the pool-wide settings.  A mistake there gives wrong bytes or
an out-of-bounds copy with every kernel correct, so every job here must give the synchronous codec's bytes, including the
bytes between a row's end and the caller's pitch, and frames 0 and N - 1 of every source are also checked against the
oracle's bands, so the two paths cannot agree on a shared mistake.

Every source and output runs at a geometry whose level-3 bands are ragged (208 / 336 / 328 / 104-wide planes), with
N = 7 frames, batch 3 (two full batches and a short one), 2 slots and a queue of 4 (full queue, submit interleaved with
wait).  Outputs the synchronous codec refuses for a pool's format must fail in the pool with the same error code, and the
pool must keep working.  The pool's statistics must count exactly the frames and payload bytes of the jobs (the
speculative sparse download: at most the larger of the frame and the copy size documented in DESIGN.md section 5b)."""
import ctypes as C
import glob
import importlib
import math
import os

import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx  # noqa: F401
from test_output_byr4 import fixture_bands
from test_quant_tables import table as quant_table

pytestmark = pytest.mark.gpu

PKG = importlib.import_module("cineform-sdk_b200")
N, BATCH, SLOTS, QUEUE = 7, 3, 2, 4
RGB10 = ("RG30", "AB10", "AR10", "R210", "DPX0")
GOLDEN_BYR4 = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decoded_byr4_*.npz")))

# encode sources: (name, FrameDesc flags, width, height).  Level-3 bands 26 / 13 (4:2:2), 42 / 21 (V210), 41 (4:4:4) and
# 13 (Bayer planes of 104 x 48) wide: none a whole number of the kernels' lanes.
SOURCES = [("YUYV", 0, 208, 56), ("UYVY", 0, 208, 56), ("YU64", 0, 208, 56), ("V210", 0, 336, 56),
           ("RG48", 0, 328, 48)] + [(n, 0, 328, 48) for n in RGB10] + \
          [("PLANAR16", 0, 328, 48), ("B64A", 0, 328, 48), ("B64A", 1, 328, 48), ("RG64", 0, 328, 48), ("RG64", 1, 328, 48),
           ("BYR4", 0, 208, 96), ("BYR5", 0, 208, 96)]
SOURCE_IDS = [f"{n}{'-alpha' if f else ''}" for n, f, _, _ in SOURCES]

# every CFB_PIXEL_* value an inverse can be asked for (BYR5 is input only)
OUTPUTS = ["YUYV", "UYVY", "RG48", "BYR4", "PLANAR16", "YU64", "V210"] + list(RGB10) + ["B64A", "BYR5"]

# one pool per codec family; what the codec decodes at full resolution (include/cfhd_b200.h at cfb_inverse_device), every
# other output is refused by the codec and must be refused by the pool with the same code
FAMILIES = {"YUYV": (("YUYV", 0, 208, 56), {"YUYV", "UYVY", "YU64", "V210", "PLANAR16"}),
            "RG48": (("RG48", 0, 328, 48), {"RG48", "B64A", "PLANAR16"} | set(RGB10)),
            "B64A": (("B64A", 0, 328, 48), {"RG48", "B64A", "PLANAR16"} | set(RGB10)),
            "B64A-alpha": (("B64A", 1, 328, 48), {"RG48", "B64A", "PLANAR16"} | set(RGB10)),
            "BYR5": (("BYR5", 0, 208, 96), {"BYR4", "PLANAR16"})}
# reduced resolutions: (family, resolution) -> outputs the codec writes there
REDUCED = {("YUYV", PKG.RESOLUTION_HALF): {"YUYV", "UYVY", "YU64", "PLANAR16"},
           ("YUYV", PKG.RESOLUTION_QUARTER): {"YUYV", "UYVY", "PLANAR16"},
           ("RG48", PKG.RESOLUTION_HALF): {"PLANAR16"},
           ("RG48", PKG.RESOLUTION_QUARTER): {"PLANAR16"} | set(RGB10)}


# ------------------------------------------------------------------------------------------------ frames and the oracle
def _desc(name, flags, w, h):
    return PKG.FrameDesc(w, h, getattr(PKG, "PIXEL_" + name), flags)


def _key(name, flags):
    return name + ("-alpha" if flags else "")


def _frames(name, flags, w, h, n=N, seed=0):
    """Frames 0 .. n - 1 of a source (distinct content per frame) and their planes as the encoder unpacks them (Bayer:
    phase 0)."""
    rng = np.random.default_rng(seed + w * 7 + h + len(name) + 31 * flags)
    return [fm.SOURCES[_key(name, flags)].frame(rng, w, h, ("natural", "random", "extreme")[i % 3]) for i in range(n)]


def _pinned(a):
    p = PKG.pinned_empty(a.shape, a.dtype)
    p[:] = a
    return p


# ------------------------------------------------------------------------------------------------ running a queue
def _wait(pool):
    """(frame number, the job's own error code) of the oldest job, as cfb_pool_wait returns them."""
    n, e = C.c_uint32(), C.c_int()
    PKG._check(PKG.lib().cfb_pool_wait(pool.h, C.byref(n), C.byref(e)))
    return n.value, e.value


def _run(pool, submits, queue_length=QUEUE):
    """Submit callables in order with never more than queue_length jobs outstanding (submit blocks on a full queue);
    returns [(frame number, error code)] in delivery order."""
    out, k = [], 0
    while len(out) < len(submits):
        while k < len(submits) and k - len(out) < queue_length:
            submits[k]()
            k += 1
        out.append(_wait(pool))
    return out


def _guess_bound(lay, sizes):
    """The largest speculative sparse copy a frame can get (cfb_sparse.cu sparse_initial_guess / sparse_next_guess): the
    initial guess, or the largest frame so far + 1/8 + 64 KiB rounded to 256 bytes, never above cfb_sparse_max_bytes."""
    nwords = lay.coded_bytes // 2
    nblocks = (nwords + 8191) // 8192
    chunks_off = (32 + 16 * nblocks + 15) & ~15
    cap = PKG.sparse_max_bytes(lay)
    m = max(sizes)
    return max(chunks_off + nwords // 4, min((m + m // 8 + 65536 + 255) & ~255, cap))


def _planes(lay, res):
    """(width, height) of each PLANAR16 plane at a decode resolution."""
    kk = res - 1
    return [(lay.band[c][kk - 1][0].width, lay.band[c][kk - 1][0].height) if kk else
            (2 * lay.band[c][0][0].width, 2 * lay.band[c][0][0].height) for c in range(lay.num_channels)]


def _out_rows(lay, out, res, rh):
    return sum(ph for _, ph in _planes(lay, res)) if out == "PLANAR16" else rh


def _out_bytes(lay, out, res, rw, rh):
    """Bytes a decode writes into the caller's buffer: every row of the output, each PLANAR16 plane at its own width."""
    if out == "PLANAR16":
        return sum(2 * pw * ph for pw, ph in _planes(lay, res))
    return fm.OUTPUTS[out].row_bytes(rw) * rh


# ------------------------------------------------------------------------------------------------ 1. every source, forward
def _forward_through_pool(desc, frames, quant, sparse, devices=(0,), setup=None):
    """Encode `frames` through a pool; returns (delivery order, results, stats)."""
    with PKG.Pool(list(devices), desc, slots=SLOTS, batch=BATCH, queue_length=QUEUE) as pool:
        if setup:
            setup(pool)
        lay = pool.layout
        pf = [_pinned(f) for f in frames]
        po = [PKG.pinned_empty(PKG.sparse_max_bytes(lay) if sparse else lay.coded_bytes) for _ in frames]
        for o in po:
            o[:] = 0xEE                                   # stale bytes must not survive in the part a result owns
        submit = pool.submit_forward_sparse if sparse else pool.submit_forward
        order = _run(pool, [lambda i=i: submit(100 + i, pf[i], quant, po[i]) for i in range(len(frames))])
        return order, [np.array(o) for o in po], pool.stats()


def _check_forward(codec, key, frames, planes, quant, order, got, stats, sparse):
    lay = codec.layout
    n = len(frames)
    assert order == [(100 + i, 0) for i in range(n)], order
    dense, sizes = [], []
    for i, f in enumerate(frames):
        want = codec.forward_host([f], quant)[0]
        dense.append(want)
        if sparse:
            sp, sz = codec.forward_host_sparse([f], quant)
            nb = PKG.sparse_bytes(got[i])
            assert nb == sz[0], f"frame {i}: sparse size {nb}, synchronous {sz[0]}"
            assert np.array_equal(got[i][:nb], sp[0][:nb]), f"frame {i}: sparse bytes differ from the synchronous codec's"
            assert np.array_equal(PKG.sparse_expand(lay, got[i]), want), f"frame {i}: sparse_expand != dense coded region"
            sizes.append(nb)
        else:
            assert np.array_equal(got[i], want), f"frame {i}: coded region differs from the synchronous codec's"
    for i in (0, n - 1):
        pu.assert_bands(codec.unpack_coded(dense[i]), fm.SOURCES[key].bands(frames[i], planes[i], quant),
                        f"{key} frame {i} vs oracle")
    assert stats["frames_forward"] == n and stats["frames_inverse"] == 0, stats
    assert stats["h2d_bytes"] == n * lay.frame_bytes, stats
    if sparse:
        g = _guess_bound(lay, sizes)
        assert sum(sizes) <= stats["d2h_bytes"] <= sum(max(s, g) for s in sizes), (stats, sizes, g)
    else:
        assert stats["d2h_bytes"] == n * lay.coded_bytes, stats


@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
@pytest.mark.parametrize("src", SOURCES, ids=SOURCE_IDS)
def test_forward_every_source(ctx, src, sparse):
    name, flags, w, h = src
    desc = _desc(*src)
    quant = PKG.quant_for_quality(desc, 4)
    fp = _frames(*src)
    frames, planes = [f for f, _ in fp], [p for _, p in fp]
    order, got, stats = _forward_through_pool(desc, frames, quant, sparse)
    with PKG.Codec(ctx, desc, 1) as codec:
        assert codec.layout.num_channels == (4 if flags or name in ("BYR4", "BYR5") else 3)
        _check_forward(codec, _key(name, flags), frames, planes, quant, order, got, stats, sparse)


# ------------------------------------------------------------------------------------------------ 2. every decode output
def _sync_inverse(codec, coded, quant, fmt, buf, sparse):
    """The synchronous decode into a copy of buf; returns (bytes, error code)."""
    out = buf.copy()
    try:
        (codec.inverse_host_sparse if sparse else codec.inverse_host)([coded], quant, fmt, [out])
    except PKG.CfbError as e:
        return None, e.code
    return out, 0


def _decode_cell(ctx, family, out, res=PKG.RESOLUTION_FULL, devices=(0,)):
    """Every frame of the family's source, dense and sparse, at the tight pitch and a padded one (fm.CANARY-filled rows of
    the row bytes rounded to 16 + 48, two rows more than the frame): pool bytes == synchronous bytes, or the same error
    code from cfb_pool_wait, after which a PLANAR16 job on the same pool succeeds.  Returns whether the output was
    accepted."""
    src, _ = FAMILIES[family]
    desc = _desc(*src)
    quant = PKG.quant_for_quality(desc, 4)
    frames = [f for f, _ in _frames(*src, n=5, seed=1)]
    fmt = getattr(PKG, "PIXEL_" + out)
    with PKG.Codec(ctx, desc, 1) as codec:
        lay = codec.layout
        coded = [codec.forward_host([f], quant)[0] for f in frames]
        sparse = [codec.forward_host_sparse([f], quant)[0][0] for f in frames]
        sparse = [s[:PKG.sparse_bytes(s)].copy() for s in sparse]
        codec.set_decode_resolution(res)
        rw, rh = codec.decoded_size()
        rb = fm.OUTPUTS[out].row_bytes(rw)
        rows = _out_rows(lay, out, res, rh)
        shapes = [(rows, (rb + 15) & ~15), (rows + 2, ((rb + 15) & ~15) + 48)]
        jobs = [(i, sp, shape) for sp in (False, True) for shape in shapes for i in range(len(frames))]
        want = []
        for i, sp, shape in jobs:
            want.append(_sync_inverse(codec, sparse[i] if sp else coded[i], quant, fmt, np.full(shape, fm.CANARY, np.uint8), sp))
        codes = {e for _, e in want}
        assert len(codes) == 1, f"{out}: the synchronous codec accepts some jobs and refuses others: {codes}"
        code = codes.pop()
        extra = np.zeros((_out_rows(lay, "PLANAR16", res, rh), (fm.OUTPUTS["PLANAR16"].row_bytes(rw) + 15) & ~15), np.uint8)
        want_extra, e = _sync_inverse(codec, coded[0], quant, PKG.PIXEL_PLANAR16, extra, False)
        assert e == 0
        if out == "PLANAR16" and res == PKG.RESOLUTION_FULL:
            # and the oracle: the stacked planes of frame 0 are its inverse pyramid of the coded bands
            planes = pu.inverse_pyramid(ol.oracle(), codec.unpack_coded(coded[0]), quant.table(lay.num_channels),
                                        tuple(quant.prescale), nchan=lay.num_channels)
            buf, off = want[0][0].view(np.int16), 0
            for c, p in enumerate(planes):
                hc, wc = p.shape
                assert np.array_equal(buf[off:off + hc, :wc], p), f"{family} PLANAR16 channel {c} vs oracle"
                off += hc
    with PKG.Pool(list(devices), desc, slots=SLOTS, batch=BATCH, queue_length=QUEUE) as pool:
        pool.set_decode_resolution(res)
        pc = [_pinned(c) for c in coded]
        ps = [_pinned(s) for s in sparse]
        bufs = []
        for _, _, shape in jobs:
            b = PKG.pinned_empty(shape)
            b[:] = fm.CANARY
            bufs.append(b)
        subs = []
        for k, (i, sp, _) in enumerate(jobs):
            if sp:
                subs.append(lambda k=k, i=i: pool.submit_inverse_sparse(k, ps[i], quant, fmt, bufs[k]))
            else:
                subs.append(lambda k=k, i=i: pool.submit_inverse(k, pc[i], quant, fmt, bufs[k]))
        order = _run(pool, subs)
        assert [n for n, _ in order] == list(range(len(jobs))), order
        assert [e for _, e in order] == [code] * len(jobs), f"{out}: pool codes {[e for _, e in order]}, synchronous {code}"
        for k, (i, sp, shape) in enumerate(jobs):
            if code == 0:
                assert np.array_equal(np.array(bufs[k]), want[k][0]), \
                    f"{family} -> {out}: frame {i} {'sparse' if sp else 'dense'} pitch {shape[1]}: bytes differ from the synchronous codec's"
            else:
                assert (np.array(bufs[k]) == fm.CANARY).all(), f"{out}: a refused job wrote its output buffer"
        pe = PKG.pinned_empty(extra.shape)
        pe[:] = 0
        pool.submit_inverse(1000, pc[0], quant, PKG.PIXEL_PLANAR16, pe)
        assert _wait(pool) == (1000, 0)
        assert np.array_equal(np.array(pe), want_extra), "the job after the refused ones"
        st = pool.stats()
    ok = len(jobs) if code == 0 else 0
    assert st["frames_forward"] == 0 and st["frames_inverse"] == ok + 1, st
    payload = sum(sparse[i].size if sp else lay.coded_bytes for i, sp, _ in jobs) + lay.coded_bytes
    # every job is uploaded before its output is checked, a refused one too; a reduced-resolution decode uploads only the
    # bands it reads
    if res == PKG.RESOLUTION_FULL:
        assert st["h2d_bytes"] == payload, (st, payload)
    else:
        assert st["h2d_bytes"] <= payload, (st, payload)
    assert st["d2h_bytes"] == ok * _out_bytes(lay, out, res, rw, rh) + _out_bytes(lay, "PLANAR16", res, rw, rh), st
    return code == 0


@pytest.mark.parametrize("out", OUTPUTS)
@pytest.mark.parametrize("family", list(FAMILIES))
def test_decode_every_output(ctx, family, out):
    accepted = _decode_cell(ctx, family, out)
    assert accepted == (out in FAMILIES[family][1]), f"{family} -> {out}: accepted {accepted}"


@pytest.mark.parametrize("out", ["YUYV", "UYVY", "YU64", "V210", "PLANAR16", "RG48"] + list(RGB10))
@pytest.mark.parametrize("family,res", list(REDUCED), ids=[f"{f}-{'half' if r == PKG.RESOLUTION_HALF else 'quarter'}" for f, r in REDUCED])
def test_decode_reduced_resolution(ctx, family, res, out):
    accepted = _decode_cell(ctx, family, out, res)
    assert accepted == (out in REDUCED[(family, res)]), f"{family} -> {out} at resolution {res}: accepted {accepted}"


@pytest.mark.parametrize("family,res,wide", [("YUYV", PKG.RESOLUTION_FULL, "YU64"), ("YUYV", PKG.RESOLUTION_HALF, "YU64"),
                                             ("BYR5", PKG.RESOLUTION_FULL, "BYR4"), ("RG48", PKG.RESOLUTION_QUARTER, "RG30")])
def test_planar16_writes_each_plane_at_its_width(ctx, family, res, wide):
    """A PLANAR16 decode into host memory writes each plane at its own width, as the device form does.  The bytes right of
    a narrower plane (4:2:2 chroma, the Bayer planes, the lowpass planes of a reduced decode) keep the caller's fm.CANARY
    even after a wider output (`wide`) has filled the frame staging; they used to come back as that output's stale bytes,
    which differed with the staging's history.  Host, sparse host and pool forms; the planes are the oracle's."""
    src, _ = FAMILIES[family]
    desc = _desc(*src)
    quant = PKG.quant_for_quality(desc, 4)
    frame = _frames(*src, n=1, seed=2)[0][0]
    with PKG.Codec(ctx, desc, 1) as codec:
        lay = codec.layout
        coded = codec.forward_host([frame], quant)[0]
        sparse = codec.forward_host_sparse([frame], quant)[0][0]
        planes = pu.inverse_pyramid(ol.oracle(), codec.unpack_coded(coded), quant.table(lay.num_channels), tuple(quant.prescale),
                                    nchan=lay.num_channels, stop_level=res - 1)
        codec.set_decode_resolution(res)
        rw, rh = codec.decoded_size()
        geo = _planes(lay, res)
        assert [p.shape[::-1] for p in planes] == geo
        shape = (_out_rows(lay, "PLANAR16", res, rh) + 2, ((2 * rw + 15) & ~15) + 32)
        scratch = np.zeros((4 * rh, (8 * rw + 15) & ~15), np.uint8)
        results = {}
        for name, f, c in (("host", codec.inverse_host, coded), ("host-sparse", codec.inverse_host_sparse, sparse)):
            codec.inverse_host([coded], quant, getattr(PKG, "PIXEL_" + wide), [scratch])
            buf = np.full(shape, fm.CANARY, np.uint8)
            f([c], quant, PKG.PIXEL_PLANAR16, [buf])
            results[name] = buf
    with PKG.Pool([0], desc, slots=1, batch=1, queue_length=2) as pool:
        pool.set_decode_resolution(res)
        pc, ps, pw_ = _pinned(coded), _pinned(sparse), _pinned(scratch)
        for name, sub, c in (("pool", pool.submit_inverse, pc), ("pool-sparse", pool.submit_inverse_sparse, ps)):
            buf = PKG.pinned_empty(shape)
            buf[:] = fm.CANARY
            pool.submit_inverse(0, pc, quant, getattr(PKG, "PIXEL_" + wide), pw_)
            sub(1, c, quant, PKG.PIXEL_PLANAR16, buf)
            assert [_wait(pool), _wait(pool)] == [(0, 0), (1, 0)]
            results[name] = np.array(buf)
    for name, buf in results.items():
        off = 0
        for c, (p, (pw, ph)) in enumerate(zip(planes, geo)):
            rows = buf[off:off + ph]
            assert np.array_equal(np.ascontiguousarray(rows[:, :2 * pw]).view(np.int16), p), f"{name}: plane {c} vs oracle"
            assert (rows[:, 2 * pw:] == fm.CANARY).all(), f"{name}: bytes right of plane {c} ({pw} wide) written"
            off += ph
        assert (buf[off:] == fm.CANARY).all(), f"{name}: rows past the planes written"


# ------------------------------------------------------------------------------------------------ 3. mixed queues
def _launches(ctx, call):
    ctx.synchronize()
    before = ctx.stats()["kernel_launches"]
    call()
    ctx.synchronize()
    return ctx.stats()["kernel_launches"] - before


def test_mixed_queue_never_shares_a_launch(ctx):
    """One queue alternates jobs that must not share a launch: quant tables T_small and T_big (T_big puts the inverse on the
    full-multiply dequantiser), YUYV, UYVY (same pitch) and YU64 outputs, the natural and a padded pitch, dense and sparse,
    forward and inverse.
    Every job gives its synchronous bytes; the launch count is at least what one launch sequence per class and per `batch`
    jobs of that class needs (a class merged into another would go below it)."""
    w, h = 720, 112
    desc = PKG.FrameDesc(w, h, PKG.PIXEL_YUYV)
    q = {name: PKG.make_quant(quant_table(name, 3), (0, 2, 0), 2) for name in ("small", "big")}
    rng = np.random.default_rng(5)
    frames = [pu.synthetic_yuyv(rng, w, h, ("natural", "random")[i % 2]) for i in range(4)]
    padded = [np.pad(f, ((0, 0), (0, 64)), constant_values=77) for f in frames]
    # (direction, quant, out_format, pitch: natural / padded, sparse)
    base = ("inv", "small", "YUYV", "natural", False)
    variants = [("inv", "big", "YUYV", "natural", False), ("inv", "small", "UYVY", "natural", False),
                ("inv", "small", "YU64", "natural", False),
                ("inv", "small", "YUYV", "padded", False), ("inv", "small", "YUYV", "natural", True),
                ("fwd", "small", None, "natural", False), ("fwd", "big", None, "natural", False),
                ("fwd", "small", None, "padded", False), ("fwd", "small", None, "natural", True)]
    classes = []
    for v in variants:
        classes += [base, v]
    with PKG.Codec(ctx, desc, 1) as codec:
        lay = codec.layout
        coded = {t: [codec.forward_host([f], q[t])[0] for f in frames] for t in q}
        sparse = {t: [codec.forward_host_sparse([f], q[t])[0][0] for f in frames] for t in q}

        def out_shape(fmt, pitch):
            rb = fm.OUTPUTS[fmt].row_bytes(w)
            return (h, rb + (0 if pitch == "natural" else 96))

        jobs, want = [], []
        for k, (d, t, fmt, pitch, sp) in enumerate(classes):
            i = k % len(frames)
            if d == "fwd":
                src = frames[i] if pitch == "natural" else padded[i]
                if sp:
                    want.append(codec.forward_host_sparse([src], q[t])[0][0])
                else:
                    want.append(codec.forward_host([src], q[t])[0])
            else:
                buf = np.full(out_shape(fmt, pitch), fm.CANARY, np.uint8)
                src = sparse[t][i] if sp else coded[t][i]
                (codec.inverse_host_sparse if sp else codec.inverse_host)([src], q[t], getattr(PKG, "PIXEL_" + fmt), [buf])
                want.append(buf)
            jobs.append((d, t, fmt, pitch, sp, i))
        per_class = {}
        for c in set(classes):
            d, t, fmt, pitch, sp = c
            if d == "fwd":
                src = frames[0] if pitch == "natural" else padded[0]
                call = (lambda: codec.forward_host_sparse([src], q[t])) if sp else (lambda: codec.forward_host([src], q[t]))
            else:
                buf = np.zeros(out_shape(fmt, pitch), np.uint8)
                src = sparse[t][0] if sp else coded[t][0]
                f = codec.inverse_host_sparse if sp else codec.inverse_host
                call = lambda: f([src], q[t], getattr(PKG, "PIXEL_" + fmt), [buf])
            per_class[c] = _launches(ctx, call)
    with PKG.Pool([0], desc, slots=SLOTS, batch=BATCH, queue_length=8) as pool:
        pins, outs, subs = [], [], []
        for k, (d, t, fmt, pitch, sp, i) in enumerate(jobs):
            if d == "fwd":
                src = _pinned(frames[i] if pitch == "natural" else padded[i])
                o = PKG.pinned_empty(PKG.sparse_max_bytes(lay) if sp else lay.coded_bytes)
                o[:] = 0xEE
                sub = pool.submit_forward_sparse if sp else pool.submit_forward
                subs.append(lambda k=k, s=src, o=o, sub=sub, t=t: sub(k, s, q[t], o))
            else:
                src = _pinned(sparse[t][i] if sp else coded[t][i])
                o = PKG.pinned_empty(out_shape(fmt, pitch))
                o[:] = fm.CANARY
                sub = pool.submit_inverse_sparse if sp else pool.submit_inverse
                subs.append(lambda k=k, s=src, o=o, sub=sub, t=t, fmt=fmt: sub(k, s, q[t], getattr(PKG, "PIXEL_" + fmt), o))
            pins.append(src)
            outs.append(o)
        order = _run(pool, subs, queue_length=8)
        st = pool.stats()
    assert order == [(k, 0) for k in range(len(jobs))], order
    for k, (d, t, fmt, pitch, sp, i) in enumerate(jobs):
        got = np.array(outs[k])
        what = f"job {k} {(d, t, fmt, pitch, 'sparse' if sp else 'dense')}"
        if d == "fwd" and sp:
            n = PKG.sparse_bytes(got)
            assert n == PKG.sparse_bytes(want[k]) and np.array_equal(got[:n], want[k][:n]), what
        else:
            assert np.array_equal(got, want[k]), what
    counts = {c: classes.count(c) for c in set(classes)}
    least = sum(math.ceil(n / BATCH) * per_class[c] for c, n in counts.items())
    assert st["kernel_launches"] >= least, (st["kernel_launches"], least)
    assert st["frames_forward"] == sum(n for c, n in counts.items() if c[0] == "fwd")
    assert st["frames_inverse"] == sum(n for c, n in counts.items() if c[0] == "inv")


def test_identical_jobs_share_launches(ctx):
    """A run of identical decode jobs queued behind a busy slot goes out in batches: fewer launch sequences than jobs."""
    w, h, n = 1920, 1080, 9
    desc = PKG.FrameDesc(w, h, PKG.PIXEL_YUYV)
    quant = PKG.quant_for_quality(desc, 4)
    rng = np.random.default_rng(9)
    with PKG.Codec(ctx, desc, 1) as codec:
        frames = [pu.synthetic_yuyv(rng, w, h, "natural") for _ in range(3)]
        coded = [codec.forward_host([f], quant)[0] for f in frames]
        want = []
        for i in range(n):
            o = np.zeros((h, 2 * w), np.uint8)
            codec.inverse_host([coded[i % 3]], quant, PKG.PIXEL_YUYV, [o])
            want.append(o)
        one = _launches(ctx, lambda: codec.inverse_host([coded[0]], quant, PKG.PIXEL_YUYV, [np.zeros((h, 2 * w), np.uint8)]))
    with PKG.Pool([0], desc, slots=1, batch=4, queue_length=n) as pool:
        pc = [_pinned(c) for c in coded]
        po = [PKG.pinned_empty((h, 2 * w)) for _ in range(n)]
        for i in range(n):
            pool.submit_inverse(i, pc[i % 3], quant, PKG.PIXEL_YUYV, po[i])
        assert [_wait(pool) for _ in range(n)] == [(i, 0) for i in range(n)]
        st = pool.stats()
    for i in range(n):
        assert np.array_equal(np.array(po[i]), want[i]), f"frame {i}"
    assert st["frames_inverse"] == n
    assert math.ceil(n / 4) * one <= st["kernel_launches"] < n * one, (st["kernel_launches"], one)


# ------------------------------------------------------------------------------------------------ 4. Bayer settings
@pytest.mark.parametrize("path", GOLDEN_BYR4, ids=[os.path.basename(p) for p in GOLDEN_BYR4])
@pytest.mark.parametrize("source", ["BYR4", "BYR5"])
def test_pool_bayer_decode_golden(path, source):
    """The bands the reference decoder held, through a pool set to the fixture's phase and curve mode: its own frame, dense
    and sparse, with the row padding and the rows past the frame untouched."""
    z = np.load(path)
    w, h, ch = int(z["width"]), int(z["height"]), int(z["coded_height"])
    phase, preset = int(z["phase"]), int(z["preset"])
    desc = PKG.FrameDesc(w, ch, getattr(PKG, "PIXEL_" + source))
    unit = PKG.make_quant(fm.UNIT4, [int(v) for v in z["prescale"]])
    lay = PKG.layout_for(desc)
    bands = fixture_bands(z)
    coded = _pinned(PKG.pack_coded(lay, bands))
    sparse = _pinned(PKG.sparse_compact_bands(lay, bands))
    pitch = 2 * w + 48
    with PKG.Pool([0], desc, slots=1, batch=2, queue_length=4) as pool:
        pool.set_bayer_phase(phase)
        pool.set_bayer_decode_curve(z["restore"] if preset == 0 else None)
        outs = []
        for k, (sub, src) in enumerate(((pool.submit_inverse, coded), (pool.submit_inverse_sparse, sparse))):
            o = PKG.pinned_empty((ch + 2, pitch))
            o[:] = fm.CANARY
            sub(k, src, unit, PKG.PIXEL_BYR4, o)
            outs.append(o)
        assert [_wait(pool) for _ in outs] == [(0, 0), (1, 0)]
    for name, o in zip(("dense", "sparse"), outs):
        buf = np.array(o)
        got = np.ascontiguousarray(buf[:h, :2 * w]).view(np.uint16)
        bad = np.argwhere(got != z["frame"])
        assert bad.size == 0, f"{name}: {bad.shape[0]} samples differ from the reference decoder's, first {bad[:4].tolist()}"
        assert (buf[:ch, 2 * w:] == fm.CANARY).all() and (buf[ch:] == fm.CANARY).all(), f"{name}: bytes outside the frame written"


def test_pool_bayer_encode_with_curve(ctx):
    """A BYR4 pool at phase 2 with the log-90 encode curve gives the synchronous codec's bands at the same settings, and
    the oracle's (fm.unpack_byr4 with the curve); back to no curve and phase 0, the defaults' bands.  The settings a codec
    refuses are refused by the pool with the same code."""
    w, h = 208, 96
    desc = PKG.FrameDesc(w, h, PKG.PIXEL_BYR4)
    quant = PKG.quant_for_quality(desc, 4)
    curve = fm.bayer_log90_curve()
    rng = np.random.default_rng(90)
    frames = [fm.synthetic_mosaic(rng, w, h, ("natural", "random", "extreme")[i % 3]) for i in range(N)]

    def setup(phase, cv):
        def f(pool):
            pool.set_bayer_phase(phase)
            pool.set_bayer_curve(cv)
        return f

    with PKG.Codec(ctx, desc, 1) as codec:
        for phase, cv in ((2, curve), (0, None)):
            order, got, stats = _forward_through_pool(desc, frames, quant, False, setup=setup(phase, cv))
            codec.set_bayer_phase(phase)
            codec.set_bayer_curve(cv)
            assert order == [(100 + i, 0) for i in range(N)]
            for i, f in enumerate(frames):
                assert np.array_equal(got[i], codec.forward_host([f], quant)[0]), f"phase {phase} frame {i}"
            for i in (0, N - 1):
                want = pu.forward_pyramid_planes(ol.oracle(), fm.unpack_byr4(frames[i], phase, curve=cv), quant.table(4),
                                                 tuple(quant.prescale))
                pu.assert_bands(codec.unpack_coded(got[i]), want, f"phase {phase} curve {cv is not None} frame {i} vs oracle")
            assert stats["frames_forward"] == N
    codes = {}
    for what, d, call in (("phase 4", desc, lambda p: p.set_bayer_phase(4)),
                          ("short curve", desc, lambda p: p.set_bayer_curve(curve[:4096])),
                          ("BYR5 curve", PKG.FrameDesc(w, h, PKG.PIXEL_BYR5), lambda p: p.set_bayer_curve(curve)),
                          ("YUYV restore", PKG.FrameDesc(w, h, PKG.PIXEL_YUYV), lambda p: p.set_bayer_decode_curve(fm.restore_table()))):
        with PKG.Pool([0], d, slots=2, batch=1, queue_length=2) as pool:
            with pytest.raises(PKG.CfbError) as ei:
                call(pool)
            codes[what] = ei.value.code
    assert codes == {"phase 4": 1, "short curve": 1, "BYR5 curve": 102, "YUYV restore": 3}, codes


# ------------------------------------------------------------------------------------------------ 5. two devices
def _needs_two():
    if PKG.device_count() < 2:
        pytest.skip("needs two CUDA devices")


@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
def test_two_devices_forward_rgba(ctx, sparse):
    """RGBA 4:4:4:4 (B64A with alpha) frames round-robin over devices 0 and 1 give device 0's synchronous bands."""
    _needs_two()
    src = ("B64A", 1, 328, 48)
    desc = _desc(*src)
    quant = PKG.quant_for_quality(desc, 4)
    fp = _frames(*src)
    frames, planes = [f for f, _ in fp], [p for _, p in fp]
    order, got, stats = _forward_through_pool(desc, frames, quant, sparse, devices=(0, 1))
    with PKG.Codec(ctx, desc, 1) as codec:
        _check_forward(codec, "B64A-alpha", frames, planes, quant, order, got, stats, sparse)


@pytest.mark.parametrize("out", ["B64A", "RG30"])
def test_two_devices_decode(ctx, out):
    """RG48 coefficients decoded to B64A (its own staging) and RG30 on a pool over devices 0 and 1."""
    _needs_two()
    assert _decode_cell(ctx, "RG48", out, devices=(0, 1))
