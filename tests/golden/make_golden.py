"""Generates the golden fixtures in this directory FROM THE REFERENCE ITSELF (oracle/_ref =
the unmodified reference compiled in place).  Run in the build container (needs /root/reference):

    python tests/golden/make_golden.py

Each .npz holds a Qbist input frame (TestCFHD's generator, seed 50) and every wavelet band the
reference's own EncodeSample produced for it (transform[c]->wavelet[k]->band[b]), the quantisation
tables it used, the DEQUANTISED bands the reference's decoder holds after entropy-decoding that sample
(d_*), the lowpass images LL1/LL2 its inverse transform rebuilds (r_*), the 8-bit YUY2 frame its DecodeSample
reconstructs from them, and the half- and quarter-resolution decodes of the same sample (decoded_half/quarter_yuy2).  tests/test_golden.py (CPU, oracle) and tests/test_forward_gpu.py
(GPU, CUDA path) compare against these files, so the GPU box needs neither the reference tree
nor oracle/_ref."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import formats as fm  # noqa: E402
import oracle_lib as ol  # noqa: E402
import parity_util as pu  # noqa: E402


def main(only=None):
    """only: restrict to one width (the 8-bit decoded frames are dithered with rand(), so regenerating a fixture changes
    its decoded_yuy2 array; tests treat it through the dither envelope)."""
    ref_lib = ol.load_ref()
    for (w, h, frame_no, quality) in [(256, 64, 1, 4), (512, 128, 2, 4), (704, 96, 1, 3), (208, 48, 1, 4)]:    # 208: ragged band widths (13 at level 3)
        if only is not None and w != only:
            continue
        frame = pu.qbist_yuy2(ref_lib, w, h, frame_no)
        bands, div, prescale, sample = pu.ref_encode_frame(ref_lib, frame, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, quality)
        import ctypes as C
        _, dec_bands = pu.ref_decode_sample_bands(ref_lib, sample, w, h)      # Codec-level: band dump
        decoded = np.zeros_like(frame)                                      # public API: the decoded picture
        rc = ref_lib.ref_decode_sample(sample.ctypes.data_as(C.c_void_p), C.c_int64(sample.size), w, h,
                                       ol.CFHD_PIXEL_FORMAT_YUY2, decoded.ctypes.data_as(C.c_void_p), w * 2)
        assert rc == 0
        reduced = {}
        for res, name in ((2, "half"), (3, "quarter")):                     # public API, reduced resolution
            buf = np.zeros_like(frame)
            dims = np.zeros(2, np.int32)
            rc = ref_lib.ref_decode_sample_res(sample.ctypes.data_as(C.c_void_p), C.c_int64(sample.size), w, h,
                                               ol.CFHD_PIXEL_FORMAT_YUY2, res, buf.ctypes.data_as(C.c_void_p), w * 2,
                                               dims.ctypes.data_as(C.c_void_p))
            assert rc == 0
            reduced[f"decoded_{name}_yuy2"] = buf[:int(dims[1]), :int(dims[0]) * 2].copy()
        arrays = {"frame": frame, "decoded_yuy2": decoded, **reduced, "divisors": np.array(div, np.int32), "prescale": np.array(prescale[0], np.int32),
                  "quality": np.array(quality), "sample_size": np.array(sample.size)}
        for (c, lvl, name), a in bands.items():
            arrays[f"b_{c}_{lvl}_{name}"] = a
        for (c, lvl, name), a in dec_bands.items():      # decoder side: dequantised, as the FSM decoder leaves them
            if name != "LL" or lvl == 3:
                arrays[f"d_{c}_{lvl}_{name}"] = a
            else:                                       # the decoder's reconstructed lowpass images LL1, LL2
                arrays[f"r_{c}_{lvl}_LL"] = a
        path = os.path.join(HERE, f"qbist_yuy2_{w}x{h}_f{frame_no}_q{quality}.npz")
        np.savez_compressed(path, **arrays)
        print(path, os.path.getsize(path))


def interlaced():
    """Interlaced source (CFHD_ENCODING_FLAGS_YUV_INTERLACED): level 1 is the field transform.  The odd field is
    shifted horizontally so the two fields really differ (motion between fields)."""
    import ctypes as C
    ref_lib = ol.load_ref()
    for (w, h, frame_no, quality, shift) in [(512, 128, 1, 4, 6), (448, 96, 2, 3, 10)]:
        frame = pu.qbist_yuy2(ref_lib, w, h, frame_no).copy()
        frame[1::2] = np.roll(frame[1::2], 2 * shift, axis=1)
        ref_lib.ref_set_interlaced(1)
        try:
            bands, div, prescale, sample = pu.ref_encode_frame(ref_lib, frame, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, quality)
        finally:
            ref_lib.ref_set_interlaced(0)
        decoded, dec_bands = pu.ref_decode_sample_bands(ref_lib, sample, w, h)
        api = np.zeros_like(frame)
        rc = ref_lib.ref_decode_sample(sample.ctypes.data_as(C.c_void_p), C.c_int64(sample.size), w, h,
                                       ol.CFHD_PIXEL_FORMAT_YUY2, api.ctypes.data_as(C.c_void_p), w * 2)
        assert rc == 0
        arrays = {"frame": frame, "decoded_yuy2": api, "divisors": np.array(div, np.int32),
                  "prescale": np.array(prescale[0], np.int32), "quality": np.array(quality), "sample_size": np.array(sample.size)}
        for (c, lvl, name), a in bands.items():
            arrays[f"b_{c}_{lvl}_{name}"] = a
        for (c, lvl, name), a in dec_bands.items():      # decoder side: dequantised, level-1 HL integrated along rows
            if name != "LL" or lvl == 3:
                arrays[f"d_{c}_{lvl}_{name}"] = a
        path = os.path.join(HERE, f"interlaced_yuy2_{w}x{h}_f{frame_no}_q{quality}.npz")
        np.savez_compressed(path, **arrays)
        print(path, os.path.getsize(path))


def yu64():
    """16-bit packed 4:2:2 source (CFHD_PIXEL_FORMAT_YU64): frame + every band of the reference's EncodeSample."""
    ref_lib = ol.load_ref()
    w, h, quality = 448, 96, 4
    frame16 = fm.yu64_from_yuyv(pu.qbist_yuy2(ref_lib, w, h, 2), np.random.default_rng(7))
    bands, div, prescale, sample = pu.ref_encode_frame(ref_lib, frame16.view(np.uint8).reshape(h, w * 4), w, h,
                                                       pu.COLOR_FORMAT_YU64, 0, 3, quality)
    arrays = {"frame16": frame16, "divisors": np.array(div, np.int32), "prescale": np.array(prescale[0], np.int32),
              "quality": np.array(quality), "sample_size": np.array(sample.size)}
    for (c, lvl, name), a in bands.items():
        arrays[f"b_{c}_{lvl}_{name}"] = a
    path = os.path.join(HERE, f"yu64_{w}x{h}_f2_q{quality}.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


def gop2():
    """Two-frame GOP (CFHD_ENCODING_FLAGS_YUV_2FRAME_GOP): both frames and all six wavelets of every channel."""
    ref_lib = ol.load_ref()
    w, h, quality = 512, 128, 4
    fa, fb = pu.qbist_yuy2(ref_lib, w, h, 1), pu.qbist_yuy2(ref_lib, w, h, 2)
    bands, quant, prescale = pu.ref_encode_gop2(ref_lib, fa, fb, w, h, quality)
    arrays = {"frame_a": fa, "frame_b": fb, "quant": np.array(quant, np.int32), "prescale": np.array(prescale, np.int32),
              "quality": np.array(quality)}
    for (c, k, b), a in bands.items():
        if not (b == 0 and k in (0, 1, 4)):              # lowpass images that only feed the next wavelet
            arrays[f"g_{c}_{k}_{b}"] = a
    path = os.path.join(HERE, f"gop2_yuy2_{w}x{h}_q{quality}.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


def v210():
    """10-bit packed 4:2:2 source (CFHD_PIXEL_FORMAT_V210): packed words + every band of the reference's EncodeSample."""
    ref_lib = ol.load_ref()
    w, h, quality = 480, 96, 4
    words, _ = fm.v210_from_yuyv(pu.qbist_yuy2(ref_lib, w, h, 1), np.random.default_rng(11))
    bands, div, prescale, sample = pu.ref_encode_frame(ref_lib, words.view(np.uint8).reshape(h, -1), w, h,
                                                       pu.COLOR_FORMAT_V210, 0, 3, quality)
    arrays = {"words": words, "width": np.array(w), "divisors": np.array(div, np.int32), "prescale": np.array(prescale[0], np.int32),
              "quality": np.array(quality), "sample_size": np.array(sample.size)}
    for (c, lvl, name), a in bands.items():
        arrays[f"b_{c}_{lvl}_{name}"] = a
    path = os.path.join(HERE, f"v210_{w}x{h}_f1_q{quality}.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


def decoded_outputs():
    """The reference decoder's packed outputs of two Qbist samples at 640x96, FILMSCAN1: a 4:2:2 sample (frame 2) decoded
    to YU64 and an RGB 4:4:4 sample (frame 1) decoded to RG48, B64A and the five 10-bit RGB formats.  Each file holds the
    dequantised bands the decoder held (the coded region: LL3 + highpass; the 10-bit formats add a per-format constant to
    LL3, stored as ll3_<format>_<c>) and the SHA-256 of every frame it wrote."""
    import hashlib
    ref_lib = ol.load_ref()
    w, h = 640, 96
    for kind, frame, color_format, chroma, outs in (
            ("yuy2", pu.qbist_yuy2(ref_lib, w, h, 2), pu.COLOR_FORMAT_YUYV, 0, ["YU64"]),
            ("rg48", pu.qbist_rg48(ref_lib, w, h, 1).view(np.uint8), pu.COLOR_FORMAT_RG48, 1,
             ["RG48", "B64A", "RG30", "AB10", "AR10", "R210", "DPX0"])):
        _, _, prescale, sample = pu.ref_encode_frame(ref_lib, frame, w, h, color_format, chroma, 3, 4)
        arrays = {"prescale": np.array(prescale[0], np.int32)}
        base = None
        for name in outs:
            out, bands = pu.ref_decode(ref_lib, sample, w, h, fm.OUTPUTS[name].decoded_format, 3, fm.OUTPUTS[name].row_bytes(w))
            bands = {k: v for k, v in bands.items() if not (k[2] == "LL" and k[1] != 3)}
            if base is None:
                base = bands
                for (c, lvl, b), a in bands.items():
                    arrays[f"d_{c}_{lvl}_{b}"] = a
            for (c, lvl, b), a in bands.items():
                if not np.array_equal(a, base[(c, lvl, b)]):
                    assert (lvl, b) == (3, "LL"), (name, c, lvl, b)
                    arrays[f"ll3_{name}_{c}"] = a
            arrays[f"sha256_{name}"] = np.array(hashlib.sha256(np.ascontiguousarray(out).tobytes()).hexdigest())
        path = os.path.join(HERE, f"decoded_{kind}_{w}x{h}_q4.npz")
        np.savez_compressed(path, **arrays)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    decoded_outputs()
    v210()
    interlaced()
    yu64()
    gop2()
    main()
