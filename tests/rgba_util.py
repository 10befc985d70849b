"""Helpers for the 16-bit RGBA sources (B64A, RG64) and the four-channel B64A output (test infrastructure)."""
import ctypes as C
import os

import numpy as np

import parity_util as pu

COLOR_FORMAT_B64A, COLOR_FORMAT_RG64 = 30, 121          # Codec/color.h:96 / :161
DECODED_FORMAT_B64A, DECODED_FORMAT_RG48 = 30, 120
ALPHA_DC_OFFSET, ALPHA_GAIN = 256, 9400                 # Codec/codec.h:164-165
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# word of each plane (G, R, B, A) inside a pixel of four 16-bit words
WORDS = {"B64A": (2, 1, 3, 0), "RG64": (1, 0, 2, 3)}


def alpha_curve(a16):
    """The encoder's alpha curve on 16-bit samples (Codec/frame.c:6697-6706, :5942-5951): a = A >> 4, and 0 < a < 4095
    -> ((a * 223 + 128) >> 8) + 256; 0 and 4095 pass through."""
    a = (a16.astype(np.int32) >> 4)
    mid = (a > 0) & (a < 4095)
    return np.where(mid, ((a * 223 + 128) >> 8) + 256, a).astype(np.int16)


def unpack_rgba64(frame16, name, alpha):
    """(height, 4 * width) uint16 -> planes G, R, B (+ A) at 12 bits, as ConvertBGRA64ToFrame_4444_16s (B64A, frame.c:6569)
    and ConvertRGBA64ToFrame16s (RG64, frame.c:5737, default branch) produce them."""
    g, r, b, a = WORDS[name]
    planes = [np.ascontiguousarray((frame16[:, k::4] >> 4).astype(np.int16)) for k in (g, r, b)]
    if alpha:
        planes.append(np.ascontiguousarray(alpha_curve(frame16[:, a::4])))
    return planes


def unpack_b64a(frame16, alpha=True):
    return unpack_rgba64(frame16, "B64A", alpha)


def unpack_rg64(frame16, alpha=True):
    return unpack_rgba64(frame16, "RG64", alpha)


def synthetic_alpha(rng, width, height):
    """16-bit alpha that covers the curve: 8 x 8 blocks of raw 0-15 (a = 0), 16-31 (a = 1, the lowest curved input),
    65504-65519 (a = 4094, the highest), 65520-65535 (a = 4095), a ramp over the whole range and uniform noise."""
    kind = np.repeat(np.repeat(rng.integers(0, 6, ((height + 7) // 8, (width + 7) // 8)), 8, 0), 8, 1)[:height, :width]
    lo = rng.integers(0, 16, (height, width))
    yy, xx = np.mgrid[0:height, 0:width]
    ramp = ((xx * 97 + yy * 61) * 16) % 65536
    choices = [lo, 16 + lo, 65504 + lo, 65520 + lo, ramp, rng.integers(0, 65536, (height, width))]
    out = np.zeros((height, width), np.int64)
    for k, v in enumerate(choices):
        out = np.where(kind == k, v, out)
    return out.astype(np.uint16)


def synthetic_rgba64(rng, width, height, kind, name):
    """(height, 4 * width) uint16 frame in the word order of `name` (B64A / RG64): colours as parity_util.synthetic_rg48,
    alpha from synthetic_alpha."""
    rgb = pu.synthetic_rg48(rng, width, height, kind)
    g, r, b, a = WORDS[name]
    f = np.empty((height, 4 * width), np.uint16)
    f[:, r::4], f[:, g::4], f[:, b::4] = rgb[:, 0::3], rgb[:, 1::3], rgb[:, 2::3]
    f[:, a::4] = synthetic_alpha(rng, width, height)
    return f


def alpha_out(plane):
    """B64A alpha word of an RGBA 4:4:4:4 sample from the reconstructed channel-3 plane.  The reference decoder takes such a
    sample with an alpha output through its active-metadata path (Codec/bayer.c:7144-7147): the ...ToRow16u sample >> 4,
    i.e. the 12-bit sample limited to [0, 4095] in every column, then ((a - 256) << 3) * 9400 >> 12 limited to [0, 65535]
    (bayer.c:16215-16224 Convert4444LinesToOutput)."""
    a = np.clip(plane.astype(np.int64), 0, 4095)
    return np.clip(((a - ALPHA_DC_OFFSET) * (8 * ALPHA_GAIN)) >> 12, 0, 65535).astype(np.uint16)


def pack_b64a_alpha(planes, precision=12):
    """[G, R, B, A] int16 planes -> the reference decoder's B64A frame of an RGBA 4:4:4:4 sample: the colour samples of its
    RG48 frame (parity_util.pack_rg48, the ...ToRow16u rule) and the de-companded alpha (alpha_out), A R G B per pixel."""
    rg = pu.pack_rg48(planes[:3], precision)
    h, w = planes[0].shape
    out = np.empty((h, 4 * w), np.uint16)
    out[:, 0::4] = alpha_out(planes[3])
    out[:, 1::4], out[:, 2::4], out[:, 3::4] = rg[:, 0::3], rg[:, 1::3], rg[:, 2::3]
    return out


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
    cf = COLOR_FORMAT_B64A if name == "B64A" else COLOR_FORMAT_RG64
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
    return pu.ref_decode_sample_raw(ol.load_ref(), *args)


def ref_decode_fresh(sample, width, height, decoded_format, num_channels, pitch, decodes=1):
    """parity_util.ref_decode_sample_raw in fresh processes bound to one CPU.  The reference's active-metadata output path,
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


def coded_region(pyr):
    return {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}


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
