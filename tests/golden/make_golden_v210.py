"""Generates golden/decoded_v210_<W>x<H>_q4.npz: the reference decoder's V210 frames of Qbist 4:2:2 samples (FILMSCAN1,
frame 2) at three widths, one per W % 6 in {0, 2, 4}.  Each file holds the dequantised bands the decoder held (the coded
region: LL3 + highpass, keys d_<c>_<level>_<band>), prescale, width, height, and the frame itself (h x natural pitch
bytes as parity_util.ref_decode returns it), not a hash, so that tests can mask the field X the reference
does not determine.  Needs oracle/_ref (the reference built by oracle/Makefile)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import formats as fm  # noqa: E402
import oracle_lib as ol  # noqa: E402
import parity_util as pu  # noqa: E402

SIZES = [(192, 48), (224, 48), (208, 48)]       # W % 6 = 0, 2, 4


def main():
    ref_lib = ol.load_ref()
    for w, h in SIZES:
        frame = pu.qbist_yuy2(ref_lib, w, h, 2)
        _, _, prescale, sample = pu.ref_encode_frame(ref_lib, frame, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, 4)
        pitch = fm.v210_natural_pitch(w)
        out, bands = pu.ref_decode(ref_lib, sample, w, h, fm.OUTPUTS["V210"].decoded_format, 3, pitch, agree=fm.v210_agree(w, pitch))
        arrays = {"prescale": np.array(prescale[0], np.int32), "width": np.array(w), "height": np.array(h), "frame": out}
        for (c, lvl, b), a in bands.items():
            if not (b == "LL" and lvl != 3):
                arrays[f"d_{c}_{lvl}_{b}"] = a
        path = os.path.join(HERE, f"decoded_v210_{w}x{h}_q4.npz")
        np.savez_compressed(path, **arrays)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
