"""Final-level timing of the BYR4 output of a Bayer codec (development): each round times inverse level 1 of `batch` 8K
mosaics, device-resident, with CUDA events on the launching stream, alternating (a) the BYR4 output with the `& 0xfffe` rule,
(b) the BYR4 output through the linear-restore table (a gather of 64 table entries per lane and band row through the
read-only path) and (c) as a yardstick the PLANAR16 output of the same codec (the four planes the fused kernel never writes);
the card's name and power limit are read in the same call.
    python tools/byr4_out_ab.py --rounds 3
Every mode reads 2 W H bytes of level-1 bands and writes 2 W H bytes (141.6 MB per 8192 x 4320 frame together).  The gather's
cost depends on how far apart the samples of a warp lie in the table, so the rounds run on smooth and on uniformly random
mosaics.  The BYR4 frame of the first mosaic is checked against the PLANAR16 planes before timing."""
import argparse
import importlib
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_GBS = 3350.0        # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=8192)
    ap.add_argument("--height", type=int, default=4320)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--phase", type=int, default=1)
    a = ap.parse_args()
    import formats as fm
    pkg = importlib.import_module("cineform-sdk_b200")
    torch.cuda.init()
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    ctx = pkg.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    w, h, n = a.width, a.height, a.batch
    desc = pkg.FrameDesc(w, h, pkg.PIXEL_BYR4)
    quant = pkg.quant_for_quality(desc, 4)
    codec = pkg.Codec(ctx, desc, n)
    codec.set_bayer_phase(a.phase)
    lay = codec.layout
    restore = fm.restore_table()
    rng = np.random.default_rng(0)
    base = fm.mosaic_from_rg48(fm.synthetic_rg48(rng, w, h, "natural"), a.phase)
    with torch.cuda.stream(stream):
        d_pyr = {kind: [torch.zeros(lay.total_bytes, dtype=torch.uint8, device="cuda") for _ in range(n)] for kind in ("smooth", "random")}
        d_byr4 = [torch.zeros(2 * w * h, dtype=torch.uint8, device="cuda") for _ in range(n)]
        d_planes = [torch.zeros(4 * w * h, dtype=torch.uint8, device="cuda") for _ in range(n)]
        for kind in d_pyr:      # the pyramids of n distinct mosaics, by the library's own forward transform
            for i in range(n):
                m = np.roll(base, (8 * i, 64 * i), axis=(0, 1)) if kind == "smooth" else rng.integers(0, 65536, (h, w)).astype(np.uint16)
                d_m = torch.from_numpy(np.ascontiguousarray(m).reshape(-1).view(np.uint8)).cuda()
                codec.forward_device([d_m.data_ptr()], lay.frame_pitch, quant, [d_pyr[kind][i].data_ptr()])
                ctx.synchronize()
    # the full inverse once, so that LL1 (the pyramid's scratch region) holds what levels 3 and 2 reconstruct
    for kind in d_pyr:
        codec.inverse_device([t.data_ptr() for t in d_pyr[kind]], quant, pkg.PIXEL_PLANAR16, [t.data_ptr() for t in d_planes], 2 * w)
    ctx.synchronize()
    codec.set_level_mask(7, 1)      # from here on the final inverse level only
    out_ptrs = {"BYR4 applied": [t.data_ptr() for t in d_byr4], "BYR4 restore": [t.data_ptr() for t in d_byr4],
                "PLANAR16": [t.data_ptr() for t in d_planes]}

    def launch(kind, mode):
        codec.set_bayer_decode_curve(restore if mode == "BYR4 restore" else None)
        codec.inverse_device([t.data_ptr() for t in d_pyr[kind]], quant, pkg.PIXEL_PLANAR16 if mode == "PLANAR16" else pkg.PIXEL_BYR4,
                             out_ptrs[mode], 2 * w)

    # the fused output equals the Bayer reconstruction of the planes (smooth content, first frame, both curve modes)
    launch("smooth", "PLANAR16")
    ctx.synchronize()
    planes = d_planes[0].cpu().numpy().view(np.int16).reshape(2 * h, w)
    planes = [planes[c * (h // 2):(c + 1) * (h // 2), :w // 2] for c in range(4)]
    for mode, table in (("BYR4 applied", None), ("BYR4 restore", restore)):
        launch("smooth", mode)
        ctx.synchronize()
        got = d_byr4[0].cpu().numpy().view(np.uint16).reshape(h, w)
        assert np.array_equal(got, fm.mosaic_from_rows(fm.rows16u(planes), a.phase, table)), mode + " differs from the planes' reconstruction"
    for kind in d_pyr:              # warm-up
        for mode in out_ptrs:
            for _ in range(3):
                launch(kind, mode)
    ctx.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    mb = 4 * w * h * n / 1e6
    print(f"{card}, power limit {power}; {n} mosaics of {w}x{h} per launch, phase {a.phase}, {mb:.1f} MB of bands in + frame out per launch", flush=True)
    for r in range(a.rounds):
        for kind in d_pyr:
            for mode in out_ptrs:
                codec.set_bayer_decode_curve(restore if mode == "BYR4 restore" else None)       # uploads: outside the timed window
                fmt = pkg.PIXEL_PLANAR16 if mode == "PLANAR16" else pkg.PIXEL_BYR4
                pp = [t.data_ptr() for t in d_pyr[kind]]
                e0.record(stream)
                for _ in range(a.iters):
                    codec.inverse_device(pp, quant, fmt, out_ptrs[mode], 2 * w)
                e1.record(stream)
                ctx.synchronize()
                us = e0.elapsed_time(e1) / a.iters * 1000
                gbs = mb * 1e6 / (us * 1e-6) / 1e9
                print(f"round {r} {kind:6s} {mode:12s}: {us:7.1f} us per launch, {gbs:6.0f} GB/s algorithmic, "
                      f"{100 * gbs / HBM_GBS:4.1f} % of {HBM_GBS:.0f} GB/s", flush=True)


if __name__ == "__main__":
    main()
