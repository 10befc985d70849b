"""Per-kernel A/B timing (development): times ONE pyramid level of the forward
or inverse path, device-resident, 16 x 4K frames per launch, CUDA events on the launching stream.  Kernel variants are
compared as two builds, each timed in its own process; the library reads CFB_TH (rows per warp):
    python tools/kernel_ab.py --level 1 --dir fwd
--levels 1,2 times several levels in one call (forward levels 1 + 2 of packed 4:2:2 then run as one fused kernel);
the algorithmic bytes are then those of the levels' separate launches added up, less LL1's write and read when levels 1
and 2 of a YUYV frame run fused (LL1 never leaves the chip: frame + 2P, the bytes of level 1 alone), and less LL2's write
and read when inverse levels 2 and 3 run fused (every level-2 band a multiple of 4 wide: P, the bytes of level 2 alone).
--dir inv --out-format YUYV / YU64 / V210 picks what the final 4:2:2 level writes (default: YUYV from a YUYV source, planes
otherwise); level 1 then counts 2P of bands in plus that packed frame out (3840x2160: 49.77 / 66.4 / 55.3 MB).
--format B64A / RG64 (--alpha: four channels, RGBA 4:4:4:4) and --out-format B64A / RG48 / RG30 time the 16-bit RGB(A)
paths and the 10-bit RGB words: forward level 1 of RGBA counts 8 bytes in + 4 x 2 out per pixel, the final inverse to B64A
4 x 2 in + 8 out.  --out-format PLANAR16 times the int16 planes of any source.  --interlaced makes level 1 the field
transform (4:2:2 sources: --dir inv --level 1 then times k_fields_carry + k_inv_fields)."""
import argparse
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--level", type=int, default=1)
    ap.add_argument("--levels", default=None, help="comma-separated levels timed together, e.g. 1,2 (overrides --level)")
    ap.add_argument("--dir", default="fwd", choices=["fwd", "inv"])
    ap.add_argument("--format", default="YUYV")
    ap.add_argument("--out-format", default=None, choices=["YUYV", "YU64", "V210", "B64A", "RG48", "RG30", "PLANAR16"])
    ap.add_argument("--interlaced", action="store_true", help="level 1 is the field transform (4:2:2 sources)")
    ap.add_argument("--alpha", action="store_true", help="B64A / RG64 sources: keep alpha as a fourth channel")
    ap.add_argument("--tag", default="")
    a = ap.parse_args()
    pkg = importlib.import_module("cineform-sdk_b200")
    sys.path.insert(0, ROOT)
    import bench
    torch.cuda.init()
    ctx = pkg.Context(0)
    fmt = getattr(pkg, "PIXEL_" + a.format)
    desc = pkg.FrameDesc(a.width, a.height, fmt, pkg.FRAME_ALPHA if a.alpha else 0)
    quant = pkg.quant_for_quality(desc, 4, interlaced=a.interlaced)
    codec = pkg.Codec(ctx, desc, 1)
    if a.interlaced:
        codec.set_interlaced(pkg.INTERLACED)
    lay = codec.layout
    stream = torch.cuda.ExternalStream(ctx.stream)
    n = a.batch
    rng = np.random.default_rng(0)
    if a.format == "YUYV":
        frames = bench.synthetic_frames(n, a.width, a.height)
    else:
        base = rng.integers(0, 65536, (lay.frame_bytes // 2,), dtype=np.uint16)
        base = (base & 0xfff0).astype(np.uint16)
        frames = [np.roll(base, 1024 * i).view(np.uint8) for i in range(n)]
    with torch.cuda.stream(stream):
        d_frames = [torch.from_numpy(np.ascontiguousarray(f).reshape(-1).view(np.uint8)).cuda() for f in frames]
        d_pyr = [torch.zeros(lay.total_bytes, dtype=torch.uint8, device="cuda") for _ in range(n)]
        # B64A from three channels writes 8 bytes per pixel: more than the source frame and the planes
        d_out = [torch.zeros(max(lay.frame_bytes, lay.num_channels * a.width * a.height * 2, a.width * a.height * 8), dtype=torch.uint8,
                             device="cuda") for _ in range(n)]
    fp, pp, op = [t.data_ptr() for t in d_frames], [t.data_ptr() for t in d_pyr], [t.data_ptr() for t in d_out]
    # a full forward first so that every level has real input
    codec.forward_device(fp, lay.frame_pitch, quant, pp)
    ctx.synchronize()
    levels = [int(x) for x in a.levels.split(",")] if a.levels else [a.level]
    bit = sum(1 << (lv - 1) for lv in levels)
    out_fmt = pkg.PIXEL_YUYV if a.format == "YUYV" else pkg.PIXEL_PLANAR16
    out_pitch = lay.frame_pitch if a.format == "YUYV" else a.width * 2
    out_bytes = lay.frame_bytes
    if a.out_format:
        out_fmt = getattr(pkg, "PIXEL_" + a.out_format)
        out_pitch = {"YUYV": a.width * 2, "YU64": a.width * 4, "V210": (a.width + 47) // 48 * 128, "B64A": a.width * 8,
                     "RG48": a.width * 6, "RG30": a.width * 4, "PLANAR16": a.width * 2}[a.out_format]
        out_bytes = out_pitch * a.height
        if a.out_format == "PLANAR16":      # the channels' planes stacked: 2 bytes per sample of every channel
            out_bytes = sum(lay.band[c][0][0].width * lay.band[c][0][0].height * 8 for c in range(lay.num_channels))
    if a.dir == "fwd":
        codec.set_level_mask(bit, 0)
        run = lambda: codec.forward_device(fp, lay.frame_pitch, quant, pp)
    else:
        codec.set_level_mask(0, bit)
        run = lambda: codec.inverse_device(pp, quant, out_fmt, op, out_pitch)
    for _ in range(5):
        run()
    ctx.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(a.iters):
        run()
    e1.record(stream)
    ctx.synchronize()
    ms = e0.elapsed_time(e1) / a.iters
    # algorithmic bytes of this level (SURVEY 8d): level 1 = input frame + 2P, level k = 2P / 4^(k-1) read+write ... all channels
    P = sum(lay.band[c][0][0].width * lay.band[c][0][0].height * 4 for c in range(lay.num_channels))     # samples of all channels
    algo = sum((out_bytes + 2 * P) if lv == 1 else (4 * P // (4 ** (lv - 1))) for lv in levels)
    if a.dir == "fwd" and a.format == "YUYV" and {1, 2} <= set(levels) and a.width % 32 == 0:
        algo -= P
    if a.dir == "inv" and {2, 3} <= set(levels) and all(lay.band[c][1][0].width % 4 == 0 for c in range(lay.num_channels)):
        algo -= P // 4
    gbs = algo * n / (ms * 1e-3) / 1e9
    env = {k: v for k, v in os.environ.items() if k.startswith("CFB_")}
    fmts = a.format + (" +alpha" if a.alpha else "") + (" interlaced" if a.interlaced else "") + (" -> " + a.out_format if a.out_format else "")
    print(f"{a.tag or a.dir + '+'.join(map(str, levels))} {fmts} {env}: {ms * 1000:.1f} us per {n}-frame launch, {gbs:.0f} GB/s algorithmic "
          f"({gbs / 3350.0:.3f} of the 3350 GB/s HBM3 data-sheet peak of an H100 SXM)", flush=True)


if __name__ == "__main__":
    main()
