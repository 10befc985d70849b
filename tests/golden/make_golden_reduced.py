"""Generates golden/reduced_<output>_<resolution>_<W>x<H>.npz: the reference decoder's reduced-resolution frames of the deep
outputs, one file per (output, resolution) this library decodes:
  yu64_half       a 4:2:2 sample (YUYV source, 0 / 255 noise) decoded to YU64 at half resolution;
  rgb10_quarter   an RGB 4:4:4 sample (RG48 source, 0 / 65535 blocks) decoded to RG30, AB10, AR10, R210 and DPX0 at quarter
                  resolution.
Each file holds, per output format <fmt>, the dequantised coded bands the reduced decode read (LL3 and the highpass of the
levels it inverts, keys d_<fmt>_<c>_<level>_<band>; LL3 carries a format-dependent offset, decoder.c:12270-12316), the
lowpass images the decoder converted (ll_<fmt>_<c>) and the frame as the decoder wrote it (frame_<fmt>); and prescale,
width, height.  Needs oracle/_ref (the reference built by oracle/Makefile)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import formats as fm  # noqa: E402
import oracle_lib as ol  # noqa: E402
import parity_util as pu  # noqa: E402


def _save(name, w, h, prescale, res, decodes):
    """decodes: {fmt: (frame, bands)}"""
    arrays = {"prescale": np.array(prescale, np.int32), "width": np.array(w), "height": np.array(h)}
    for fmt, (frame, bands) in decodes.items():
        for (c, lvl, b), a in fm.reduced_coded_bands(bands, res).items():
            arrays[f"d_{fmt}_{c}_{lvl}_{b}"] = a
        for c, ll in enumerate(fm.lowpass_images(bands, res)):
            arrays[f"ll_{fmt}_{c}"] = ll
        arrays[f"frame_{fmt}"] = frame
    path = os.path.join(HERE, f"reduced_{name}_{w}x{h}.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


def main():
    ref_lib = ol.load_ref()
    # YU64, half resolution
    w, h = 336, 48
    frame = pu.synthetic_yuyv(np.random.default_rng(w + h), w, h, "extreme")
    _, _, prescale, sample = pu.ref_encode_frame(ref_lib, frame, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, 4)
    out, _, _, bands = fm.ref_decode_reduced(ref_lib, sample, w, h, fm.OUTPUTS["YU64"].decoded_format, 3, fm.HALF, 4)
    _save("yu64_half", w, h, prescale[0], fm.HALF, {"YU64": (out.view(np.uint16), bands)})
    # the 10-bit RGB words, quarter resolution
    w, h = 328, 48
    frame = fm.block_rg48(w, h, 2, w)
    _, _, prescale, sample = pu.ref_encode_frame(ref_lib, frame.view(np.uint8), w, h, pu.COLOR_FORMAT_RG48, 1, 3, 1)
    decodes = {}
    for fmt in fm.RGB30_FORMATS:
        out, _, _, bands = fm.ref_decode_reduced(ref_lib, sample, w, h, fm.OUTPUTS[fmt].decoded_format, 3, fm.QUARTER, 4)
        decodes[fmt] = (out.view(np.uint32), bands)
    _save("rgb10_quarter", w, h, prescale[0], fm.QUARTER, decodes)


if __name__ == "__main__":
    main()
