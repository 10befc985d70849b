"""Level-1 timing of 12-bit packed Bayer (BYR5) against 16-bit Bayer (BYR4) on the same mosaics (development): each
round times forward level 1 of `batch` 8K frames of each source, device-resident, with CUDA events on the launching
stream, alternating the two sources; the card's name and power limit are read in the same call.
    python tools/byr5_ab.py --rounds 4
The BYR4 frames carry the BYR5 frames' 12-bit samples << 4 (curve applied), so both produce the same planes -- checked
once on the first frame before timing."""
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


def byr4_from_components(comps, phase):
    """The 16-bit mosaic whose quads hold the component samples << 4 (quad layout of formats.mosaic_from_rg48)."""
    import formats as fm
    _, ph, pw = comps.shape
    r, g1, g2, b = (comps[i] for i in fm.BYR5_ORDER[phase])
    lay = {0: (r, g1, g2, b), 1: (g1, r, b, g2), 2: (g1, b, r, g2), 3: (b, g1, g2, r)}[phase]
    m = np.empty((2 * ph, 2 * pw), np.uint16)
    m[0::2, 0::2], m[0::2, 1::2], m[1::2, 0::2], m[1::2, 1::2] = (x << 4 for x in lay)
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=8192)
    ap.add_argument("--height", type=int, default=4320)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--phase", type=int, default=0)
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
    rng = np.random.default_rng(0)
    pw, ph, n = a.width // 2, a.height // 2, a.batch
    comps = [fm.byr5_random_components(rng, pw, ph, "natural") for _ in range(n)]
    runs = {}
    for name in ("BYR5", "BYR4"):
        desc = pkg.FrameDesc(a.width, a.height, getattr(pkg, "PIXEL_" + name))
        quant = pkg.quant_for_quality(desc, 4)
        codec = pkg.Codec(ctx, desc, n)
        codec.set_bayer_phase(a.phase)
        lay = codec.layout
        frames = [fm.byr5_pack(c) if name == "BYR5" else byr4_from_components(c, a.phase) for c in comps]
        with torch.cuda.stream(stream):
            d_frames = [torch.from_numpy(f.reshape(-1).view(np.uint8)).cuda() for f in frames]
            d_pyr = [torch.zeros(lay.total_bytes, dtype=torch.uint8, device="cuda") for _ in range(n)]
        fp, pp = [t.data_ptr() for t in d_frames], [t.data_ptr() for t in d_pyr]
        codec.set_level_mask(1, 0)
        runs[name] = (codec, lay, quant, fp, pp, d_frames, d_pyr)
    # both sources give the same level-1 bands
    ctx.synchronize()
    ref = None
    for name, (codec, lay, quant, fp, pp, _, d_pyr) in runs.items():
        codec.forward_device(fp, lay.frame_pitch, quant, pp)
        ctx.synchronize()
        got = d_pyr[0][:lay.coded_bytes].cpu().numpy()
        ref = got if ref is None else ref
        assert np.array_equal(got, ref), "BYR5 and BYR4 level-1 bands differ"
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, (codec, lay, quant, fp, pp, *_) in runs.items():       # warm-up
        for _ in range(5):
            codec.forward_device(fp, lay.frame_pitch, quant, pp)
    ctx.synchronize()
    print(f"{card}, power limit {power}; {n} frames of {a.width}x{a.height} per launch, phase {a.phase}", flush=True)
    for r in range(a.rounds):
        for name, (codec, lay, quant, fp, pp, *_) in runs.items():
            e0.record(stream)
            for _ in range(a.iters):
                codec.forward_device(fp, lay.frame_pitch, quant, pp)
            e1.record(stream)
            ctx.synchronize()
            us = e0.elapsed_time(e1) / a.iters * 1000
            frame_mb = lay.frame_bytes * n / 1e6
            print(f"round {r} {name}: {us:.1f} us per launch ({us / n:.1f} us per frame), frame bytes {frame_mb:.1f} MB", flush=True)


if __name__ == "__main__":
    main()
