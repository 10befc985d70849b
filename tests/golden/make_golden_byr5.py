"""Generates the BYR5 (12-bit packed Bayer) fixtures in this directory FROM THE REFERENCE ITSELF (oracle/_ref = the
unmodified reference compiled in place).  Run where the reference tree is present:

    python tests/golden/make_golden_byr5.py

  byr5_512x128_p1_q4.npz           a seeded smooth BYR5 frame (planes 256 x 64), Bayer phase 1: the packed frame, the
                                   coded region (LL3 + highpass) of the four channels the reference's EncodeSample produced
                                   for it (b_<c>_<level>_<band>), its divisors and prescale.
  byr5_208x100_p2_extreme_q4.npz   the same for 0 / 4095 noise in every component at planes 104 x 50 (W % 64 != 0, pw % 32
                                   != 0), phase 2.  The encoder pads the plane height to 56 by repeating the last packed row;
                                   `coded_height` holds it.

tests/test_byr5_gpu.py reads them, so the GPU machine needs neither the reference tree nor oracle/_ref for those tests."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import formats as fm  # noqa: E402
import byr4_out_util as b4  # noqa: E402
import oracle_lib as ol  # noqa: E402


def fixture(w, h, phase, kind):
    pw, ph = w // 2, h // 2
    frame = fm.byr5_pack(fm.byr5_random_components(np.random.default_rng(w + h + phase), pw, ph, kind))
    bands, div, prescale, _ = b4.ref_encode_byr5(ol.load_ref(), frame, pw, ph, phase)
    arrays = {"frame": frame, "phase": np.array(phase, np.int32), "divisors": np.array(div, np.int32),
              "prescale": np.array(prescale, np.int32), "coded_height": np.array(bands[(0, 1, "LL")].shape[0] * 2, np.int32)}
    for (c, lvl, b), a in bands.items():
        if b != "LL" or lvl == 3:
            arrays[f"b_{c}_{lvl}_{b}"] = a
    path = os.path.join(HERE, f"byr5_{w}x{h}_p{phase}{'' if kind == 'natural' else '_' + kind}_q4.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    fixture(512, 128, 1, "natural")
    fixture(208, 100, 2, "extreme")
