"""Device-resident decode rate of the reduced-resolution outputs (development), with CUDA events on the codec's stream:
  4K RGB 4:4:4 12-bit (RG48 source) to the 10-bit RGB words (RG30) at quarter resolution, and at full resolution;
  4K 4:2:2 (YUYV source) to YU64 at half resolution, and at full resolution;
and the conversion kernel alone (inverse level mask 0: k_lowpass_444 / k_lowpass_422<YU64> only), with its bytes per launch
computed from the shapes (the three LL images read, the frame written) against the 3.35 TB/s HBM3 of the H100 SXM data
sheet.  The card's name and power limit are read in the same call.
    python tools/reduced_res_bench.py --batch 16 --iters 50 --rounds 3
RG48 at half and quarter resolution stays unsupported (include/cfhd_b200.h), so it is not timed."""
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
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import formats as fm
    import parity_util as pu
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
    rng = np.random.default_rng(0)
    configs = []        # (name, codec, quant, pyramids, outputs, format, pitch, resolution, conversion bytes per launch)
    for src, out_fmt, res, bpp in (("RG48", "RG30", pkg.RESOLUTION_QUARTER, 4), ("YUYV", "YU64", pkg.RESOLUTION_HALF, 4)):
        desc = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + src))
        quant = pkg.quant_for_quality(desc, 4)
        codec = pkg.Codec(ctx, desc, n)
        lay = codec.layout
        frame = fm.synthetic_rg48(rng, w, h, "natural") if src == "RG48" else pu.synthetic_yuyv(rng, w, h, "natural")
        with torch.cuda.stream(stream):
            pyr = [torch.zeros(lay.total_bytes, dtype=torch.uint8, device="cuda") for _ in range(n)]
            d_f = torch.from_numpy(np.ascontiguousarray(frame).reshape(-1).view(np.uint8)).cuda()
        torch.cuda.synchronize()
        for i in range(n):
            codec.forward_device([d_f.data_ptr()], lay.frame_pitch, quant, [pyr[i].data_ptr()])
        ctx.synchronize()
        for r in (pkg.RESOLUTION_FULL, res):
            codec.set_decode_resolution(r)
            rw, rh = codec.decoded_size()
            pitch = (rw * bpp + 15) // 16 * 16
            outs = [torch.zeros(rh * pitch, dtype=torch.uint8, device="cuda") for _ in range(n)]
            k = 0 if r == pkg.RESOLUTION_FULL else r - 2
            ll_bytes = sum(lay.band[c][k][0].width * lay.band[c][k][0].height * 2 for c in range(3))
            configs.append((f"{src}->{out_fmt} {'full' if r == pkg.RESOLUTION_FULL else ('half' if r == 2 else 'quarter')}",
                            codec, quant, pyr, outs, getattr(pkg, "PIXEL_" + out_fmt), pitch, r, (ll_bytes + rh * rw * bpp) * n))

    def run(cfg, mask):
        _, codec, quant, pyr, outs, fmt, pitch, r, _ = cfg
        codec.set_decode_resolution(r)
        codec.set_level_mask(7, mask)
        codec.inverse_device([t.data_ptr() for t in pyr], quant, fmt, [t.data_ptr() for t in outs], pitch)

    for cfg in configs:                 # warm-up; a full inverse leaves LL1 / LL2 in the scratch region for the mask-0 runs
        for _ in range(3):
            run(cfg, 7)
    ctx.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    print(f"{card}, power limit {power}; {n} frames of {w}x{h} per launch, device-resident", flush=True)
    for rnd in range(a.rounds):
        for cfg in configs:
            name, r, nbytes = cfg[0], cfg[7], cfg[8]
            modes = [("decode", 7)] + ([("conversion only", 0)] if r != pkg.RESOLUTION_FULL else [])
            for mode, mask in modes:
                e0.record(stream)
                for _ in range(a.iters):
                    run(cfg, mask)
                e1.record(stream)
                ctx.synchronize()
                us = e0.elapsed_time(e1) / a.iters * 1000
                line = f"round {rnd} {name:22s} {mode:16s}: {us:8.1f} us per batch, {n / (us * 1e-6):8.0f} frames/s"
                if mask == 0:
                    gbs = nbytes / (us * 1e-6) / 1e9
                    line += f", {nbytes / 1e6:.1f} MB, {gbs:6.0f} GB/s, {100 * gbs / HBM_GBS:4.1f} % of {HBM_GBS:.0f} GB/s"
                print(line, flush=True)
    for cfg in configs:
        cfg[1].set_level_mask(7, 7)


if __name__ == "__main__":
    main()
