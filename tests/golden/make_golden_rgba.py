"""Generates the 16-bit RGBA fixtures in this directory FROM THE REFERENCE ITSELF (oracle/_ref = the unmodified reference
compiled in place).  Run where the reference tree is present:

    python tests/golden/make_golden_rgba.py

  rgba_b64a_256x64_q4.npz          a seeded B64A frame with synthetic alpha (every part of the encoder's alpha curve), the
                                   coded region (LL3 + highpass) of the four channels the reference's EncodeSample produced
                                   for it as RGBA 4:4:4:4 (b_<c>_<level>_<band>), its divisors and prescale.
  decoded_rgba_b64a_328x48_q4.npz  the dequantised bands the reference decoder held for the RGBA 4:4:4:4 sample of a seeded
                                   B64A frame (d_<c>_<level>_<band>), its prescale and the SHA-256 of the B64A and RG48
                                   frames it wrote.  328 pixels: band width 164, so the RG48 rule's scalar tail starts inside
                                   the last 8-column group.
  decoded_rgba_b64a_200x48_extreme_q4.npz  the same for 0 / 65535 noise in every word at band width 100 (the tail starts
                                   at column 91): colours and alpha reach both limits of every rule.

tests/test_rgba64_gpu.py reads them, so the GPU machine needs neither the reference tree nor oracle/_ref for those tests."""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import formats as fm  # noqa: E402
import oracle_lib as ol  # noqa: E402
import rgba_util as ru  # noqa: E402


def encoded():
    ref_lib = ol.load_ref()
    w, h = 256, 64
    frame = fm.synthetic_rgba64(np.random.default_rng(64), w, h, "natural", "B64A")
    bands, div, prescale, _ = ru.ref_encode(ref_lib, frame, w, h, "B64A", True)
    arrays = {"frame": frame, "divisors": np.array(div, np.int32), "prescale": np.array(prescale, np.int32)}
    for (c, lvl, b), a in fm.coded_region(bands).items():
        arrays[f"b_{c}_{lvl}_{b}"] = a
    path = os.path.join(HERE, f"rgba_b64a_{w}x{h}_q4.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


def decoded(w, h, kind):
    ref_lib = ol.load_ref()
    frame = fm.synthetic_rgba64(np.random.default_rng(w), w, h, kind, "B64A")
    _, _, prescale, sample = ru.ref_encode(ref_lib, frame, w, h, "B64A", True)
    arrays = {"prescale": np.array(prescale, np.int32)}
    base = None
    for name in ("B64A", "RG48"):
        out, bands = ru.ref_decode_fresh(sample, w, h, fm.OUTPUTS[name].decoded_format, 4, fm.OUTPUTS[name].row_bytes(w), decodes=5)
        bands = fm.coded_region(bands)
        if base is None:
            base = bands
            for (c, lvl, b), a in bands.items():
                arrays[f"d_{c}_{lvl}_{b}"] = a
        for key, a in bands.items():        # no per-format offset on LL3 for these two outputs
            assert np.array_equal(a, base[key]), (name, key)
        arrays[f"sha256_{name}"] = np.array(hashlib.sha256(np.ascontiguousarray(out).tobytes()).hexdigest())
    path = os.path.join(HERE, f"decoded_rgba_b64a_{w}x{h}{'' if kind == 'natural' else '_' + kind}_q4.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    encoded()
    decoded(328, 48, "natural")
    decoded(200, 48, "extreme")
