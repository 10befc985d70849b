"""Every entry point of a decode writes the same frame: cfb_inverse_device, cfb_inverse_host, cfb_inverse_host_sparse and
both pool forms give the restatement in formats.OUTPUTS of the oracle's planes, at full resolution and at the reduced
resolutions, at a pitch wider than a row; the padding and the two rows past the frame keep the CANARY."""
import numpy as np
import pytest

import formats as fm
import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import ctx, pkg  # noqa: F401
from test_reduced_res_outputs_gpu import _case, _want

pytestmark = pytest.mark.gpu


def _v210(pkg, w, h):
    """A YUYV codec; a pitch 128 bytes wider than the codec's own."""
    rng = np.random.default_rng(w * 3 + h)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_YUYV)
    quant = pkg.quant_for_quality(desc, 4)
    orc = ol.oracle()
    bands = pu.oracle_forward_422(orc, pu.synthetic_yuyv(rng, w, h, "natural"), quant, 0)
    planes = pu.inverse_pyramid(orc, bands, quant.table(3), tuple(quant.prescale))
    return desc, quant, bands, None, fm.OUTPUTS["V210"].expected(planes), fm.v210_natural_pitch(w) + 128


def _byr4(pkg, w, h):
    """A BYR5 codec at the defaults (phase 0, `& 0xfffe`), which the pool's codecs keep; a pitch 64 bytes wider than a row."""
    rng = np.random.default_rng(w * 3 + h)
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR5)
    quant = pkg.quant_for_quality(desc, 4)
    table, prescale = quant.table(4), tuple(quant.prescale)
    orc = ol.oracle()
    bands = fm.coded_region(pu.forward_pyramid_planes(orc, fm.unpack_byr4(fm.synthetic_mosaic(rng, w, h, "random"), 0),
                                                      table, prescale))
    planes = pu.inverse_pyramid(orc, bands, table, prescale, nchan=4)
    return desc, quant, bands, None, fm.OUTPUTS["BYR4"].expected(planes), 2 * w + 64


def _reduced(out, codec_kind):
    """YU64 at half resolution of a 4:2:2 codec, the 10-bit words at quarter resolution of an RGB 4:4:4 ("444") or RGBA
    4:4:4:4 ("4444") codec; a pitch of the row rounded to 16 bytes + 64."""
    def case(pkg, w, h):
        desc, quant, bands, res = _case(pkg, codec_kind, w, h, "natural", 11)
        want = _want(out, quant, bands, res, 4 if codec_kind == "4444" else 3)
        return desc, quant, bands, res, want, (want.shape[1] + 15) // 16 * 16 + 64
    return case


CASES = [("V210", _v210, (208, 48)), ("V210", _v210, (224, 64)), ("V210", _v210, (720, 96)),
         ("BYR4", _byr4, (208, 96)), ("BYR4", _byr4, (720, 112)),
         ("YU64", _reduced("YU64", "422"), (336, 48)), ("RG30", _reduced("RG30", "444"), (328, 48)),
         ("DPX0", _reduced("DPX0", "444"), (200, 64)), ("AR10", _reduced("AR10", "4444"), (256, 64))]
IDS = ["V210-208x48", "V210-224x64", "V210-720x96", "BYR4-208x96", "BYR4-720x112",
       "YU64-422-336x48", "RG30-444-328x48", "DPX0-444-200x64", "AR10-4444-256x64"]


@pytest.mark.parametrize("out,case,size", CASES, ids=IDS)
def test_every_entry_point_gives_the_same_bytes(pkg, ctx, out, case, size):
    import torch
    w, h = size
    desc, quant, bands, res, want, pitch = case(pkg, w, h)
    fmt = getattr(pkg, "PIXEL_" + out)
    want = np.ascontiguousarray(want).view(np.uint8)
    rh, rb = want.shape
    results = {}
    with pkg.Codec(ctx, desc, 1) as codec:
        if res is not None:
            codec.set_decode_resolution(res)
        assert rb == fm.OUTPUTS[out].row_bytes(codec.decoded_size()[0])
        coded = codec.pack_coded(bands)
        sparse = pkg.sparse_compact_bands(codec.layout, bands)
        # device: the pyramid (coded region) in device memory, the frame written straight into a device buffer
        d_pyr = torch.zeros(codec.layout.total_bytes, dtype=torch.uint8, device="cuda")
        d_pyr[:coded.size] = torch.from_numpy(coded).cuda()
        d_out = torch.full(((rh + 2) * pitch,), fm.CANARY, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        codec.inverse_device([d_pyr.data_ptr()], quant, fmt, [d_out.data_ptr()], pitch)
        ctx.synchronize()
        results["device"] = d_out.cpu().numpy().reshape(rh + 2, pitch)
        buf = np.full((rh + 2, pitch), fm.CANARY, np.uint8)
        codec.inverse_host([coded], quant, fmt, [buf])
        results["host"] = buf
        buf = np.full((rh + 2, pitch), fm.CANARY, np.uint8)
        codec.inverse_host_sparse([sparse], quant, fmt, [buf])
        results["host-sparse"] = buf
    with pkg.Pool([0], desc, slots=1, batch=1, queue_length=4) as pool:
        if res is not None:
            pool.set_decode_resolution(res)
        pc = pkg.pinned_empty(coded.size)
        pc[:] = coded
        ps = pkg.pinned_empty(sparse.size)
        ps[:] = sparse
        for name, submit, src in (("pool", pool.submit_inverse, pc), ("pool-sparse", pool.submit_inverse_sparse, ps)):
            po = pkg.pinned_empty((rh + 2, pitch))
            po[:] = fm.CANARY
            submit(1, src, quant, fmt, po)
            assert pool.wait() == 1
            results[name] = np.array(po)
    for name, buf in results.items():
        what = f"{out} {w}x{h} {name}"
        bad = np.argwhere(buf[:rh, :rb] != want)
        assert bad.size == 0, f"{what}: {bad.shape[0]} bytes differ, first (row, byte) {bad[:5].tolist()}"
        assert (buf[:rh, rb:] == fm.CANARY).all(), f"{what}: row padding written"
        assert (buf[rh:] == fm.CANARY).all(), f"{what}: rows past the frame written"
