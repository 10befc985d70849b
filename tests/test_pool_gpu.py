"""Frame pool (cfb_pool_*): EncoderPool semantics on GPU streams -- in-order delivery, bounded queue,
batched launches, results identical to the synchronous API / the oracle."""
import numpy as np
import pytest

import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

pytestmark = pytest.mark.gpu


def test_pool_forward_inverse_in_order(pkg):
    w, h, n = 704, 96, 23
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    rng = np.random.default_rng(3)
    frames = [pu.synthetic_yuyv(rng, w, h, "natural") for _ in range(n)]
    orc = ol.oracle()
    ndev = min(pkg.device_count(), 2)
    with pkg.Pool(list(range(ndev)), desc, slots=2, batch=4, queue_length=8) as pool:
        lay = pool.layout
        pf = [pkg.pinned_empty((h, w * 2)) for _ in range(n)]
        pc = [pkg.pinned_empty(lay.coded_bytes) for _ in range(n)]
        po = [pkg.pinned_empty((h, w * 2)) for _ in range(n)]
        for a, f in zip(pf, frames):
            a[:] = f
        # encode: submit all (queue_length 8 < n forces interleaved submit/collect), collect in order
        got, submitted = [], 0
        while len(got) < n:
            while submitted < n and submitted - len(got) < 8:
                pool.submit_forward(1000 + submitted, pf[submitted], quant, pc[submitted])
                submitted += 1
            got.append(pool.wait())
        assert got == [1000 + i for i in range(n)]
        # decode
        got, submitted = [], 0
        while len(got) < n:
            while submitted < n and submitted - len(got) < 8:
                pool.submit_inverse(submitted, pc[submitted], quant, pkg.PIXEL_YUYV, po[submitted])
                submitted += 1
            got.append(pool.wait())
        assert got == list(range(n))
        st = pool.stats()
        assert st["frames_forward"] == n and st["frames_inverse"] == n
        assert st["kernel_launches"] < 6 * n          # batching: fewer launches than one pyramid per frame
        # results == oracle
        with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
            for i in (0, 7, n - 1):
                want = pu.oracle_forward_422(orc, frames[i], quant, 0)
                bands = codec.unpack_coded(pc[i])
                for key in want:
                    assert np.array_equal(bands[key], want[key]), (i, key)
                planes = pu.inverse_pyramid(orc, want, quant.table(3), tuple(quant.prescale))
                a, b = pu.yuyv_envelope(planes)
                assert ((po[i] == a) | (po[i] == b)).all()


def test_pool_test_returns_not_finished_then_result(pkg):
    w, h = 256, 64
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    with pkg.Pool([0], desc, slots=1, batch=1, queue_length=2) as pool:
        f = pkg.pinned_empty((h, w * 2)); f[:] = 128
        c = pkg.pinned_empty(pool.layout.coded_bytes)
        pool.submit_forward(7, f, quant, c)
        r = None
        for _ in range(100000):
            r = pool.test()
            if r is not None:
                break
        assert r == 7
        with pytest.raises(pkg.CfbError):
            pool.wait()             # nothing outstanding -> invalid argument, as the reference's empty queue


def test_pool_interlaced_and_half_resolution(pkg):
    """Pool-wide modes: interlaced sources (field transform at level 1) and half-resolution decode through the
    asynchronous queue give the same bytes as the synchronous codec."""
    w, h, n = 448, 96, 6
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4, interlaced=True)
    rng = np.random.default_rng(11)
    frames = []
    for i in range(n):
        f = pu.synthetic_yuyv(rng, w, h, "natural")
        f[1::2] = np.roll(f[1::2], 4 + 2 * i, axis=1)
        frames.append(f)
    with pkg.Pool([0], desc, slots=2, batch=2, queue_length=8) as pool, pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        pool.set_interlaced(1)
        codec.set_interlaced(True)
        lay = pool.layout
        pf = [pkg.pinned_empty((h, w * 2)) for _ in range(n)]
        pc = [pkg.pinned_empty(lay.coded_bytes) for _ in range(n)]
        for a, f in zip(pf, frames):
            a[:] = f
        for i in range(n):
            pool.submit_forward(i, pf[i], quant, pc[i])
        assert [pool.wait() for _ in range(n)] == list(range(n))
        for i in range(n):
            one = np.zeros(lay.coded_bytes, np.uint8)
            codec.forward_host([frames[i]], quant, [one])
            assert np.array_equal(np.asarray(pc[i]), one), f"frame {i}"
        # half-resolution decode of the interlaced samples (LL1 does not depend on the level-1 transform type)
        pool.set_decode_resolution(pkg.RESOLUTION_HALF)
        codec.set_decode_resolution(pkg.RESOLUTION_HALF)
        rw, rh = codec.decoded_size()
        po = [pkg.pinned_empty((rh, rw * 2)) for _ in range(n)]
        for i in range(n):
            pool.submit_inverse(i, pc[i], quant, pkg.PIXEL_YUYV, po[i])
        assert [pool.wait() for _ in range(n)] == list(range(n))
        for i in range(n):
            want = np.zeros((rh, rw * 2), np.uint8)
            codec.inverse_host([np.asarray(pc[i])], quant, pkg.PIXEL_YUYV, [want])
            assert np.array_equal(np.asarray(po[i]), want), f"frame {i}"


def test_pool_two_devices_decode_matches_one_device(pkg):
    """A pool over devices 0 and 1 decodes YUYV frames (the final level's TMA ring, above the default shared-memory
    limit, on both devices) to the bytes of the synchronous codec on device 0."""
    if pkg.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    w, h, n = 704, 96, 8
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    rng = np.random.default_rng(17)
    frames = [pu.synthetic_yuyv(rng, w, h, "natural") for _ in range(n)]
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        coded = [codec.forward_host([f], quant)[0].copy() for f in frames]
        want = []
        for c in coded:
            out = np.zeros((h, w * 2), np.uint8)
            codec.inverse_host([c], quant, pkg.PIXEL_YUYV, [out])
            want.append(out)
    with pkg.Pool([0, 1], desc, slots=1, batch=1, queue_length=n) as pool:
        pc = [pkg.pinned_empty(c.size) for c in coded]
        po = [pkg.pinned_empty((h, w * 2)) for _ in range(n)]
        for a, c in zip(pc, coded):
            a[:] = c
        for i in range(n):
            pool.submit_inverse(i, pc[i], quant, pkg.PIXEL_YUYV, po[i])
        assert [pool.wait() for _ in range(n)] == list(range(n))
    for i in range(n):
        assert np.array_equal(np.asarray(po[i]), want[i]), f"frame {i}"
