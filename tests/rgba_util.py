"""The reference encoder and decoder on 16-bit RGBA (B64A, RG64) frames and their fixtures (test infrastructure); the
formats themselves are described in formats.py."""
import ctypes as C
import os

import numpy as np

import formats as fm
import parity_util as pu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def ref_encode(ref_lib, frame16, width, height, name, alpha, quality=4):
    """The reference's EncodeSample on a B64A / RG64 frame (RGB 4:4:4, or RGBA 4:4:4:4 with alpha); returns (bands,
    divisors[c][k][b], prescale of channel 0, sample).  Its sample buffer is sized for 0/65535 noise in four channels."""
    fn = ref_lib.ref_encode_frame_bands
    fn.restype = C.c_int
    nc = 4 if alpha else 3
    frame = np.ascontiguousarray(frame16).view(np.uint8)
    dims = np.zeros(nc * 9, np.int32)
    quant = np.zeros(nc * 12, np.int32)
    prescale = np.zeros(nc * 3, np.int32)
    cap = width * height * 4 * nc
    bands = np.zeros(cap, np.int16)
    sample = np.zeros(width * height * 16 + 65536, np.uint8)
    cf = fm.COLOR_FORMAT_B64A if name == "B64A" else fm.COLOR_FORMAT_RG64
    vp = C.c_void_p
    size = fn(vp(frame.ctypes.data), width, height, frame.strides[0], cf, 1, nc, quality, vp(dims.ctypes.data),
              vp(quant.ctypes.data), vp(prescale.ctypes.data), vp(bands.ctypes.data), C.c_int64(cap),
              vp(sample.ctypes.data), C.c_int64(sample.size))
    assert size > 0, "reference EncodeSample failed"
    out, pos = {}, 0
    for c in range(nc):
        for k in range(3):
            w, h = int(dims[(c * 3 + k) * 3]), int(dims[(c * 3 + k) * 3 + 1])
            for b in range(4):
                out[(c, k + 1, pu.BAND_NAMES[b])] = bands[pos:pos + w * h].reshape(h, w).copy()
                pos += w * h
    return out, quant.reshape(nc, 3, 4).tolist(), prescale.reshape(nc, 3).tolist()[0], sample[:size].copy()


def _decode_worker(args):
    import oracle_lib as ol
    # one CPU: the reference's row workers of this path de-compand alpha in place and, racing on a many-core host, can
    # convert a row twice
    cpus = sorted(os.sched_getaffinity(0))
    os.sched_setaffinity(0, {cpus[0]})
    return pu.ref_decode(ol.load_ref(), *args)


def ref_decode_fresh(sample, width, height, decoded_format, num_channels, pitch, decodes=1):
    """parity_util.ref_decode in fresh processes bound to one CPU.  The reference's active-metadata output path,
    which RGBA 4:4:4:4 samples take, is not deterministic: its row workers race with the transform workers and with each
    other, and a whole row of the frame can come out wrong in one decode and right in the next.  decodes > 1: every row of
    the returned frame is the one a strict majority of `decodes` independent decodes agree on (bands of the first)."""
    import multiprocessing as mp
    args = (sample, width, height, decoded_format, num_channels, pitch)
    with mp.get_context("spawn").Pool(1, maxtasksperchild=1) as pool:
        runs = [pool.apply(_decode_worker, (args,)) for _ in range(decodes)]
    out = runs[0][0].copy()
    for r in range(height):
        rows = [bytes(run[0][r]) for run in runs]
        best = max(set(rows), key=rows.count)
        assert rows.count(best) * 2 > decodes, f"row {r}: no majority over {decodes} decodes"
        out[r] = np.frombuffer(best, np.uint8)
    return out, runs[0][1]


def load_fixture(name):
    return np.load(os.path.join(GOLDEN, name))


def fixture_bands(z, prefix):
    """{(c, level, band): array} from the keys <prefix>_<c>_<level>_<band> of a fixture."""
    out = {}
    for key in z.files:
        if key.startswith(prefix + "_"):
            c, lvl, b = key[len(prefix) + 1:].split("_")
            out[(int(c), int(lvl), b)] = z[key]
    return out
