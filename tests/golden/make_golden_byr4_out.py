"""Generates the BYR4-output fixtures in this directory FROM THE REFERENCE ITSELF (oracle/_ref = the unmodified reference
compiled in place).  Run where the reference tree is present:

    python tests/golden/make_golden_byr4_out.py

Each decoded_byr4_<W>x<H>_p<phase>_<lin|app>[_extreme][_byr5].npz holds a seeded mosaic encoded by the reference's
EncodeSample and decoded by its DecodeSample to DECODED_FORMAT_BYR4 at full resolution:

  d_<c>_<level>_<band>   the coded-region bands (LL3 + highpass) of the four channels as the decoder held them (dequantised)
  prescale               the level prescales; phase, preset: cfhddata.bayer_format / encode_curve_preset AS THE DECODER USED
                         THEM (read back after the decode)
  restore                decoder->BYR4LinearRestore (16384 uint16), in the `lin` fixtures (preset 0: linear restore)
  frame                  the decoded mosaic, height x width uint16; coded_height: the mosaic rows of the coded planes

The encoder's bayer.format and encode_curve_preset do NOT travel in a sample EncodeSample wrote (they are metadata the SDK
attaches), and the decoder resets both to 0 on its first sample, so a decode would silently use phase 0 and the linear
restore.  The probe therefore sets both on the decoder (oracle/ref_probe_bayer.cpp ref_decode_bayer_bands) and reads back what it held.
`lin`: the encoder applied its log-90 curve (BYR4 source, preset 0) or none (BYR5) and the decoder restores through its
table; `app`: curve applied by the application, `& 0xfffe`.  `_byr5`: the sample was encoded from a BYR5 frame (208 x 100:
plane height 50 padded to 56 by the encoder).

tests/test_output_byr4_gpu.py reads them, so the GPU machine needs neither the reference tree nor oracle/_ref for those tests."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import byr4_out_util as b4  # noqa: E402
import formats as fm  # noqa: E402
import oracle_lib as ol  # noqa: E402


def fixture(w, h, phase, preset, kind, byr5=False):
    ref = ol.load_ref()
    rng = np.random.default_rng(w + h + 10 * phase + preset)
    if byr5:
        packed = fm.byr5_pack(fm.byr5_random_components(rng, w // 2, h // 2, kind))
        _, _, prescale, sample = b4.ref_encode_byr5(ref, packed, w // 2, h // 2, phase)
    else:
        _, _, prescale, sample = b4.ref_encode_byr4(ref, fm.synthetic_mosaic(rng, w, h, kind, phase), phase, preset)
    frame, bands, used, table = b4.ref_decode_byr4(sample, w, h, phase, preset)
    assert used == (phase, preset), f"the decoder used {used}, not {(phase, preset)}"
    arrays = {"frame": frame, "width": np.array(w, np.int32), "height": np.array(h, np.int32),
              "coded_height": np.array(bands[(0, 1, "LL")].shape[0] * 4, np.int32), "phase": np.array(used[0], np.int32),
              "preset": np.array(used[1], np.int32), "prescale": np.array(prescale[0], np.int32)}
    if preset == 0:
        arrays["restore"] = table
    for (c, lvl, b), a in bands.items():
        if b != "LL" or lvl == 3:
            arrays[f"d_{c}_{lvl}_{b}"] = a
    name = f"decoded_byr4_{w}x{h}_p{phase}_{'app' if preset else 'lin'}{'' if kind == 'natural' else '_' + kind}{'_byr5' if byr5 else ''}.npz"
    path = os.path.join(HERE, name)
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    fixture(512, 128, 0, 1, "natural")
    fixture(512, 128, 1, 0, "natural")
    fixture(208, 100, 2, 0, "extreme", byr5=True)
    fixture(208, 96, 3, 1, "extreme")
