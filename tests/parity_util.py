"""Shared helpers for the parity tests (test infrastructure)."""
import ctypes as C

import numpy as np

import oracle_lib as ol

COLOR_FORMAT_UYVY, COLOR_FORMAT_YUYV, COLOR_FORMAT_RG48, COLOR_FORMAT_BYR4 = 1, 2, 120, 104  # Codec/color.h:64-131
BAND_NAMES = ("LL", "LH", "HL", "HH")


# ---------------------------------------------------------------- synthetic frames
def synthetic_yuyv(rng, width, height, kind="natural"):
    """Packed 8-bit 4:2:2 frame (height x 2*width bytes)."""
    if kind == "random":
        return rng.integers(0, 256, (height, width * 2)).astype(np.uint8)
    if kind == "extreme":
        return np.where(rng.integers(0, 2, (height, width * 2)) == 0, 0, 255).astype(np.uint8)
    if kind == "constant":
        return np.full((height, width * 2), 128, np.uint8)
    # smooth gradients + texture + mild noise: natural-image-like statistics
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float32)
    luma = 110 + 70 * np.sin(xx / 37.0) * np.cos(yy / 23.0) + 30 * np.sin((xx + 2 * yy) / 5.0) * (xx > width / 2)
    luma += rng.normal(0, 2.0, luma.shape)
    cb = 128 + 40 * np.sin(xx[:, ::2] / 91.0 + yy[:, ::2] / 57.0)
    cr = 128 + 40 * np.cos(xx[:, ::2] / 71.0 - yy[:, ::2] / 43.0)
    f = np.empty((height, width * 2), np.uint8)
    f[:, 0::2] = np.clip(luma, 0, 255).astype(np.uint8)
    f[:, 1::4] = np.clip(cb, 0, 255).astype(np.uint8)
    f[:, 3::4] = np.clip(cr, 0, 255).astype(np.uint8)
    return f


def reference_decoded(kind, name):
    """A fixture of golden/make_golden.py decoded_outputs(): (dequantised bands the reference decoder held for output
    `name`, prescale, SHA-256 of the frame it wrote).  kind: "yuy2" (4:2:2 sample) or "rg48" (RGB 4:4:4 sample)."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"decoded_{kind}_640x96_q4.npz"))
    bands = {}
    for key in z.files:
        if key.startswith("d_"):
            c, lvl, b = key.split("_")[1:]
            ll3 = f"ll3_{name}_{c}"
            bands[(int(c), int(lvl), b)] = z[ll3] if (lvl, b) == ("3", "LL") and ll3 in z.files else z[key]
    return bands, [int(v) for v in z["prescale"]], str(z[f"sha256_{name}"])


def yuyv_to_uyvy(frame):
    out = np.empty_like(frame)
    out[:, 0::2] = frame[:, 1::2]
    out[:, 1::2] = frame[:, 0::2]
    return out


def qbist_yuy2(ref_lib, width, height, frame_number=1, seed=50):
    """Frame `frame_number` (1-based) of the TestCFHD Qbist sequence (Example/TestCFHD.cpp:1149-1219)."""
    pitch = width * 2
    out = np.zeros((height, pitch), np.uint8)
    ref_lib.ref_qbist_frames(seed, width, height, pitch, ol.CFHD_PIXEL_FORMAT_YUY2, frame_number, out.reshape(-1))
    return out


def qbist_yuy2_sequence(ref_lib, width, height, nframes, seed=50):
    """Frames 1 .. nframes of the TestCFHD Qbist sequence (seed 50, Example/TestCFHD.cpp:41), generated in one pass."""
    pitch = width * 2
    out = np.zeros((nframes, height, pitch), np.uint8)
    fn = ref_lib.ref_qbist_sequence
    fn.argtypes = [C.c_uint, C.c_int, C.c_int, C.c_int, C.c_uint, C.c_int, C.c_void_p]
    fn.restype = None
    fn(seed, width, height, pitch, ol.CFHD_PIXEL_FORMAT_YUY2, nframes, out.ctypes.data_as(C.c_void_p))
    return [out[i] for i in range(nframes)]


# ---------------------------------------------------------------- oracle pyramids
def quant_table(quant, nchan=3):
    return [[[quant.divisor[c][k][b] for b in range(4)] for k in range(3)] for c in range(nchan)]


def forward_pyramid_422(impl, frame, divisors, prescale=(0, 2, 0), fmt=0, midpoint=2, interlaced=False):
    """3-level pyramid of a packed 4:2:2 frame with `impl` (oracle or reference building blocks).
    Returns {(c, level, band_name): array}, LL only for level 3 plus ('LL', level) intermediates under key
    (c, level, 'LL').  interlaced: level 1 is the field transform (encoder.c:2949-2993)."""
    out = {}
    for c in range(3):
        level1 = impl.fwd_fields_422 if interlaced else impl.fwd_level_422
        ll, lh, hl, hh = level1(frame, c, fmt, divisors[c][0], precision=10, midpoint=midpoint)
        out[(c, 1, "LL")], out[(c, 1, "LH")], out[(c, 1, "HL")], out[(c, 1, "HH")] = ll, lh, hl, hh
        for k in (1, 2):
            variant = 1 if prescale[k] == 2 else 0
            ll, lh, hl, hh = impl.fwd_level(ll, variant, divisors[c][k], midpoint)
            out[(c, k + 1, "LL")], out[(c, k + 1, "LH")], out[(c, k + 1, "HL")], out[(c, k + 1, "HH")] = ll, lh, hl, hh
    return out


def oracle_forward_422(orc, frame, quant, fmt=0, interlaced=False):
    """Coded-region bands (LL3 + all highpass) the CUDA path must reproduce."""
    pyr = forward_pyramid_422(orc, frame, quant_table(quant), tuple(quant.prescale), fmt, quant.midpoint_prequant,
                              interlaced=interlaced)
    return {k: v for k, v in pyr.items() if not (k[2] == "LL" and k[1] != 3)}


# ---------------------------------------------------------------- whole-frame reference probe
def ref_encode_frame(ref_lib, frame, width, height, color_format, sampling_444, num_channels, quality):
    """Run the reference's real EncodeSample; returns (bands dict, divisors[c][k][b], prescale[c][k], sample bytes)."""
    fn = ref_lib.ref_encode_frame_bands
    fn.restype = C.c_int
    frame = np.ascontiguousarray(frame)
    pitch = frame.strides[0]
    dims = np.zeros(num_channels * 9, np.int32)
    quant = np.zeros(num_channels * 12, np.int32)
    prescale = np.zeros(num_channels * 3, np.int32)
    cap = width * height * 4 * num_channels
    bands = np.zeros(cap, np.int16)
    sample = np.zeros(width * height * 4 + 65536, np.uint8)
    size = fn(frame.ctypes.data_as(C.c_void_p), width, height, pitch, color_format, sampling_444, num_channels, quality,
              dims.ctypes.data_as(C.c_void_p), quant.ctypes.data_as(C.c_void_p), prescale.ctypes.data_as(C.c_void_p),
              bands.ctypes.data_as(C.c_void_p), C.c_int64(cap), sample.ctypes.data_as(C.c_void_p), C.c_int64(sample.size))
    assert size > 0, "reference EncodeSample failed"
    out, pos = {}, 0
    for c in range(num_channels):
        for k in range(3):
            w, h = int(dims[(c * 3 + k) * 3]), int(dims[(c * 3 + k) * 3 + 1])
            for b in range(4):
                out[(c, k + 1, BAND_NAMES[b])] = bands[pos:pos + w * h].reshape(h, w).copy()
                pos += w * h
    div = quant.reshape(num_channels, 3, 4).tolist()
    return out, div, prescale.reshape(num_channels, 3).tolist(), sample[:size].copy()


# ---------------------------------------------------------------- inverse composition
def dequantize(band, divisor):
    """Codec/decoder.c:20551 DeQuantFSM semantics on a dense band: (int16)(v * quant)."""
    if divisor <= 1:
        return band.copy()
    return (band.astype(np.int32) * divisor).astype(np.int16)


def integrate_hl(hl):
    """The decoder's row integration of the field transform's difference-coded HL band: `line[x] += line[x-1]` in int16
    with wrap-around (Codec/decoder.c:20822-20836)."""
    return np.cumsum(hl, axis=1, dtype=np.int16)


def inverse_pyramid(impl, bands, divisors, prescale, nchan=3, stop_level=0, interlaced=False, hl_integrated=False):
    """bands: {(c, level, name)} QUANTISED coded-region bands (LL3 + highpass of levels 1..3).
    Returns the reconstructed int16 plane of every channel at codec precision (list); stop_level = 1 / 2 stops at
    the lowpass image LL1 / LL2 (half / quarter resolution decode).  hl_integrated (interlaced only): the level-1 HL band
    is already integrated along its rows, as the reference's decoder hands it over, and is not integrated again."""
    planes = []
    for c in range(nchan):
        ll = bands[(c, 3, "LL")]
        for k in (2, 1, 0)[:3 - stop_level]:
            lh = dequantize(bands[(c, k + 1, "LH")], divisors[c][k][1])
            hl = dequantize(bands[(c, k + 1, "HL")], divisors[c][k][2])
            hh = dequantize(bands[(c, k + 1, "HH")], divisors[c][k][3])
            if k == 0 and interlaced:
                # the coded HL band of the field transform is difference coded along each row; the decoder
                # integrates it after dequantisation
                if not hl_integrated:
                    hl = integrate_hl(hl)
                ll = impl.inv_fields(ll, lh, hl, hh)
            else:
                ll = impl.inv_level(ll, lh, hl, hh, 2 if prescale[k] == 2 else 0)
        planes.append(ll)
    return planes


def lowpass_to_422(planes, unsigned_shift, uyvy=False, shift=4):
    """oracle/cfhd_oracle.c orc_lowpass_to_422 on [y, v, u] lowpass planes -> packed 8-bit frame."""
    import ctypes as C
    import oracle_lib as ol
    y, v, u = [np.ascontiguousarray(p, np.int16) for p in planes]
    h, w = y.shape
    out = np.zeros((h, w * 2), np.uint8)
    lib = ol.load_oracle()
    lib.orc_lowpass_to_422.restype = None
    vp = C.c_void_p
    lib.orc_lowpass_to_422(vp(y.ctypes.data), C.c_int(y.strides[0]), vp(v.ctypes.data), C.c_int(v.strides[0]),
                           vp(u.ctypes.data), C.c_int(u.strides[0]), C.c_int(w), C.c_int(h), C.c_int(shift),
                           C.c_int(int(unsigned_shift)), C.c_int(int(uyvy)), vp(out.ctypes.data), C.c_int(w * 2))
    return out


def yuyv_envelope(planes, shift=2, uyvy=False):
    """The two 8-bit values the reference's dithered reduction can produce at every byte of the packed frame:
    out = sat_u8((max(v,0) + d) >> shift), d in {0,1}  (InvertHorizontalStrip16s.c:3807-3892)."""
    y, v, u = planes
    h, w = y.shape
    lo = np.zeros((h, w * 2), np.int32)
    yo, co = (1, 0) if uyvy else (0, 1)
    lo[:, yo::2] = y
    lo[:, co::4] = u
    lo[:, co + 2::4] = v
    lo = np.maximum(lo, 0)
    a = np.clip(lo >> shift, 0, 255).astype(np.uint8)
    b = np.clip((lo + 1) >> shift, 0, 255).astype(np.uint8)
    return a, b


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


# ---------------------------------------------------------------- comparisons of GPU results
def assert_bands(got, want, what=""):
    """Every coded band of `want` ({(c, level, name): array}; the LL of levels 1 and 2 is not coded and is skipped) equals
    the one in `got` bit for bit."""
    for key in sorted(want):
        if key[2] == "LL" and key[1] != 3:
            continue
        g, w_ = got[key], want[key]
        assert g.shape == w_.shape, f"{what} band {key}: shape {g.shape}, want {w_.shape}"
        if not np.array_equal(g, w_):
            bad = np.argwhere(g != w_)
            raise AssertionError(f"{what} band {key} {w_.shape}: {bad.shape[0]} mismatches, first {bad[:4].tolist()}, "
                                 f"rows {sorted(set(bad[:, 0].tolist()))[:12]}, columns {sorted(set(bad[:, 1].tolist()))[:12]}, "
                                 f"got {g[tuple(bad[0])]} want {w_[tuple(bad[0])]}")


def check_planes(got, want, what=""):
    """Lists of int16 planes, equal channel by channel."""
    assert len(got) == len(want)
    for c, (g, w_) in enumerate(zip(got, want)):
        assert g.shape == w_.shape, f"{what} channel {c}: shape {g.shape}, want {w_.shape}"
        if not np.array_equal(g, w_):
            bad = np.argwhere(g != w_)
            raise AssertionError(f"{what} channel {c}: {bad.shape[0]} mismatches, first {bad[:5].tolist()}, "
                                 f"rows {sorted(set(bad[:, 0].tolist()))[:12]}, got {g[tuple(bad[0])]} want {w_[tuple(bad[0])]}")


def planar16(codec, pkg, coded, quant, w, h):
    """Decode one 4:2:2 coefficient buffer to PLANAR16; returns the [Y, V, U] int16 planes."""
    out = np.zeros((3 * h, w), np.int16)
    codec.inverse_host([coded], quant, pkg.PIXEL_PLANAR16, [out])
    return [out[0:h, :w], out[h:2 * h, :w // 2], out[2 * h:3 * h, :w // 2]]


def ref_decode_sample_bands(ref_lib, sample, width, height, decoded_format=COLOR_FORMAT_YUYV, num_channels=3):
    """Reference Codec-level decode; returns (decoded packed frame, {(c, level, name): DEQUANTISED band})."""
    out = np.zeros((height, width * 2), np.uint8)
    dims = np.zeros(num_channels * 9, np.int32)
    quant = np.zeros(num_channels * 12, np.int32)
    cap = width * height * 4 * num_channels
    b = np.zeros(cap, np.int16)
    sample = np.ascontiguousarray(sample)
    rc = ref_lib.ref_decode_sample_bands(sample.ctypes.data_as(C.c_void_p), C.c_int64(sample.size), width, height,
                                         decoded_format, num_channels, out.ctypes.data_as(C.c_void_p), width * 2,
                                         dims.ctypes.data_as(C.c_void_p), quant.ctypes.data_as(C.c_void_p),
                                         b.ctypes.data_as(C.c_void_p), C.c_int64(cap))
    assert rc == 0, f"reference decode failed ({rc})"
    bands, pos = {}, 0
    for c in range(num_channels):
        for k in range(3):
            w, h = int(dims[(c * 3 + k) * 3]), int(dims[(c * 3 + k) * 3 + 1])
            for bi in range(4):
                bands[(c, k + 1, BAND_NAMES[bi])] = b[pos:pos + w * h].reshape(h, w).copy()
                pos += w * h
    return out, bands


UNIT_DIVISORS = [[[1, 1, 1, 1]] * 3] * 3


# ---------------------------------------------------------------- RG48 (packed 16-bit RGB -> 4:4:4, 12 bit)
CFHD_PIXEL_FORMAT_RG48 = (ord("R") << 24) | (ord("G") << 16) | (ord("4") << 8) | ord("8")


def qbist_rg48(ref_lib, width, height, frame_number=1, seed=50):
    pitch = width * 6
    out = np.zeros((height, pitch), np.uint8)
    ref_lib.ref_qbist_frames(seed, width, height, pitch, CFHD_PIXEL_FORMAT_RG48, frame_number, out.reshape(-1))
    return out.view(np.uint16)          # (height, 3*width)


def unpack_rg48(frame16, precision=12):
    """Codec/frame.c:5968 ConvertRGB48ToFrame16s, default branch (:6130-6164): plane0 = G, plane1 = R, plane2 = B,
    each `>> (16 - precision)`."""
    sh = 16 - precision
    r, g, b = frame16[:, 0::3], frame16[:, 1::3], frame16[:, 2::3]
    return [np.ascontiguousarray((x >> sh).astype(np.int16)) for x in (g, r, b)]


def forward_pyramid_planes(impl, planes, divisors, prescale, midpoint=2):
    """3-level pyramid of already unpacked int16 planes (level 1 uses the plain / V210 variant by prescale[0])."""
    out = {}
    for c, ll in enumerate(planes):
        for k in range(3):
            variant = 1 if prescale[k] == 2 else 0
            ll, lh, hl, hh = impl.fwd_level(ll, variant, divisors[c][k], midpoint)
            out[(c, k + 1, "LL")], out[(c, k + 1, "LH")], out[(c, k + 1, "HL")], out[(c, k + 1, "HH")] = ll, lh, hl, hh
    return out


def synthetic_rg48(rng, width, height, kind="natural"):
    if kind == "random":
        return rng.integers(0, 65536, (height, width * 3)).astype(np.uint16)
    if kind == "extreme":
        return np.where(rng.integers(0, 2, (height, width * 3)) == 0, 0, 65535).astype(np.uint16)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float32)
    f = np.empty((height, width * 3), np.uint16)
    for c, (a, b) in enumerate(((37.0, 23.0), (51.0, 31.0), (29.0, 47.0))):
        v = 30000 + 20000 * np.sin(xx / a) * np.cos(yy / b) + 6000 * np.sin((xx + 2 * yy) / 5.0) * (xx > width / 2)
        v += rng.normal(0, 300.0, v.shape)
        f[:, c::3] = np.clip(v, 0, 65535).astype(np.uint16)
    return f


# ---------------------------------------------------------------- BYR4 (16-bit Bayer, curve applied -> 4 planes, 12 bit)
def mosaic_from_rg48(frame16, fmt=0):
    """Bayer mosaic (height x width uint16) sampled from a packed RGB frame; fmt = BAYER_FORMAT_* phase."""
    r, g, b = frame16[:, 0::3], frame16[:, 1::3], frame16[:, 2::3]
    h, w = r.shape
    m = np.empty((h, w), np.uint16)
    # quad positions (line, col): RED_GRN: r g / g b ; GRN_RED: g r / b g ; GRN_BLU: g b / r g ; BLU_GRN: b g / g r
    lay = {0: ("r", "g", "g", "b"), 1: ("g", "r", "b", "g"), 2: ("g", "b", "r", "g"), 3: ("b", "g", "g", "r")}[fmt]
    src = {"r": r, "g": g, "b": b}
    m[0::2, 0::2] = src[lay[0]][0::2, 0::2]; m[0::2, 1::2] = src[lay[1]][0::2, 1::2]
    m[1::2, 0::2] = src[lay[2]][1::2, 0::2]; m[1::2, 1::2] = src[lay[3]][1::2, 1::2]
    return m


def bayer_log90_curve(precision=12):
    """The default encode curve of Codec/frame.c:5208-5245: curve[i] = (int)(lin2log((float)i / 16384, 90) * 4095) with
    lin2log (Common/AVIExtendedHeader.h:153) evaluated in double and rounded to float, 1 << 14 entries, curve[0] = 0."""
    i = np.arange(1 << 14, dtype=np.float32) / np.float32(1 << 14)
    v = (np.log10(i.astype(np.float64) * (np.float64(np.float32(90.0)) - 1.0) + 1.0) / np.log10(np.float64(np.float32(90.0)))).astype(np.float32)
    curve = (v * np.float32((1 << precision) - 1)).astype(np.int32)
    curve[0] = 0
    return curve.astype(np.uint16)


def unpack_byr4(bayer16, fmt=0, precision=12, curve=None):
    """Codec/frame.c:4993 ConvertBYR4ToFrame16s: planes G, R-G, B-G, dG.  curve=None: encode_curve_preset branch
    (:5040-5200, samples >> 4); else the table branch (:5206-5420): sample -> curve[sample >> 2]."""
    sh = 16 - precision
    if curve is None:
        conv = lambda a: (a >> sh).astype(np.int32)
    else:
        conv = lambda a: curve[(a >> 2).astype(np.int64)].astype(np.int32)
    q0 = conv(bayer16[0::2, 0::2]); q1 = conv(bayer16[0::2, 1::2])
    q2 = conv(bayer16[1::2, 0::2]); q3 = conv(bayer16[1::2, 1::2])
    r, g1, g2, b = {0: (q0, q1, q2, q3), 1: (q1, q0, q3, q2), 2: (q2, q0, q3, q1), 3: (q3, q1, q2, q0)}[fmt]
    mid = 1 << 12
    gg = (g1 + g2) >> 1
    planes = [gg, (r - gg + mid) >> 1, (b - gg + mid) >> 1, (g1 - g2 + mid) >> 1]
    return [np.ascontiguousarray(p.astype(np.int16)) for p in planes]


# ---------------------------------------------------------------- YU64 (16-bit packed 4:2:2 -> 10-bit planes)
COLOR_FORMAT_YU64 = 12


def yu64_from_yuyv(frame8, rng):
    """16-bit packed Y0 C1 Y1 C3 frame whose top 8 bits are the given 8-bit frame and whose low bits are random."""
    f16 = (frame8.astype(np.uint16) << 8) | rng.integers(0, 256, frame8.shape).astype(np.uint16)
    return f16                                   # (height, 2 * width) uint16


def unpack_yu64(frame16, precision=10):
    """Codec/frame.c:1556 ConvertYU64ToFrame16s: sample >> (16 - precision); position 1 -> channel 1, position 3 -> channel 2."""
    s = (frame16 >> (16 - precision)).astype(np.int16)
    return [np.ascontiguousarray(s[:, 0::2]), np.ascontiguousarray(s[:, 1::4]), np.ascontiguousarray(s[:, 3::4])]


# ---------------------------------------------------------------- two-frame GOP (FIELDPLUS pyramid)
def ref_encode_gop2(ref_lib, frame_a, frame_b, width, height, quality, num_channels=3, color_format=COLOR_FORMAT_YUYV):
    """The reference's EncodeSample on frame A then frame B with gop_length = 2; returns
    ({(c, wavelet 0..5, band): array}, quant[c][k][b], prescale[c][k])  (oracle/ref_probe.cpp ref_encode_gop2_bands)."""
    fn = ref_lib.ref_encode_gop2_bands
    fn.restype = C.c_int64
    fa, fb = np.ascontiguousarray(frame_a), np.ascontiguousarray(frame_b)
    dims = np.zeros(num_channels * 24, np.int32)
    quant = np.zeros(num_channels * 24, np.int32)
    prescale = np.zeros(num_channels * 8, np.int32)
    cap = width * height * 8 * num_channels
    bands = np.zeros(cap, np.int16)
    vp = C.c_void_p
    n = fn(vp(fa.ctypes.data), vp(fb.ctypes.data), width, height, fa.strides[0], color_format, num_channels, quality,
           vp(dims.ctypes.data), vp(quant.ctypes.data), vp(prescale.ctypes.data), vp(bands.ctypes.data), C.c_int64(cap))
    assert n > 0, "reference two-frame-GOP encode failed"
    d = dims.reshape(num_channels, 6, 4)
    out, pos = {}, 0
    for c in range(num_channels):
        for k in range(6):
            w, h, _, nb = (int(v) for v in d[c, k])
            for b in range(nb):
                out[(c, k, b)] = bands[pos:pos + w * h].reshape(h, w).copy()
                pos += w * h
    return out, quant.reshape(num_channels, 6, 4).tolist(), prescale.reshape(num_channels, 8).tolist()


def gop2_inverse_planes(orc, bands, quant, prescale, nchan=3):
    """Inverse FIELDPLUS composition with the oracle (decoder.c:13109-13170): {(c, wavelet, band)} QUANTISED bands ->
    the two frames' reconstructed planes ([c] lists for frame A and frame B)."""
    lib = ol.load_oracle()
    vp = C.c_void_p
    planes_a, planes_b = [], []
    for c in range(nchan):
        def inv(bands4, k):
            deq = [bands4[0]] + [dequantize(bands4[b], quant[c][k][b]) for b in (1, 2, 3)]
            return orc.inv_level(*deq, 2 if prescale[c][k] == 2 else 0)

        ll4 = inv([bands[(c, 5, b)] for b in range(4)], 5)
        tl = inv([ll4] + [bands[(c, 4, b)] for b in (1, 2, 3)], 4)
        th = inv([bands[(c, 3, b)] for b in range(4)], 3)
        la, lb = np.zeros_like(tl), np.zeros_like(tl)
        hh, ww = tl.shape
        lib.orc_temporal_inv(vp(tl.ctypes.data), vp(th.ctypes.data), ww * 2, ww, hh, 10, vp(la.ctypes.data), vp(lb.ctypes.data), ww * 2)
        planes_a.append(inv([la] + [bands[(c, 0, b)] for b in (1, 2, 3)], 0))
        planes_b.append(inv([lb] + [bands[(c, 1, b)] for b in (1, 2, 3)], 1))
    return planes_a, planes_b


def gop2_pyramid(level1, temporal, level, frame_a, frame_b, quant, prescale, nchan=3, midpoint=2):
    """FIELDPLUS composition (Codec/encoder.c:8431 FinishFieldPlusTransformQuant) from three callables:
    level1(frame, c, divisors) -> 4 bands, temporal(a, b) -> (low, high), level(plane, prescale, divisors) -> 4 bands.
    Returns {(c, wavelet, band)} with the same keys the reference dump has (LL of wavelets 0, 1, 4 omitted)."""
    out = {}
    for c in range(nchan):
        a = level1(frame_a, c, quant[c][0])
        b = level1(frame_b, c, quant[c][1])
        for i in range(1, 4):
            out[(c, 0, i)], out[(c, 1, i)] = a[i], b[i]
        low, high = temporal(a[0], b[0])
        out[(c, 2, 0)], out[(c, 2, 1)] = low, high
        w3 = level(high, prescale[c][3], quant[c][3])
        w4 = level(low, prescale[c][4], quant[c][4])
        w5 = level(w4[0], prescale[c][5], quant[c][5])
        for i in range(4):
            out[(c, 3, i)], out[(c, 5, i)] = w3[i], w5[i]
        for i in range(1, 4):
            out[(c, 4, i)] = w4[i]
    return out


# ---------------------------------------------------------------- V210 (10-bit packed 4:2:2)
COLOR_FORMAT_V210 = 10


def pack_v210(y, cb, cr):
    """y (h, w), cb / cr (h, w/2) 10-bit -> (h, pitch/4) uint32: component stream Cb Y Cr Y ..., three per word at bits
    0, 10, 20 (Codec/convert.c:3365), rows padded to a multiple of 128 bytes (48 pixels)."""
    h, w = y.shape
    comp = np.zeros((h, 2 * w), np.uint32)
    comp[:, 0::4], comp[:, 1::4], comp[:, 2::4], comp[:, 3::4] = cb, y[:, 0::2], cr, y[:, 1::2]
    nwords = ((w + 47) // 48) * 32
    padded = np.zeros((h, nwords * 3), np.uint32)
    padded[:, :2 * w] = comp
    return (padded[:, 0::3] | (padded[:, 1::3] << 10) | (padded[:, 2::3] << 20)).astype(np.uint32)


def v210_from_yuyv(frame8, rng):
    """10-bit planes whose top 8 bits are the given 8-bit YUYV frame (random low bits) and their V210 packing.
    Returns (words, [Y, ch1, ch2]) with ch1 = Cr (second chroma), ch2 = Cb as ConvertV210ToFrame16s assigns them."""
    h, w2 = frame8.shape
    w = w2 // 2
    y = (frame8[:, 0::2].astype(np.uint32) << 2) | rng.integers(0, 4, (h, w)).astype(np.uint32)
    cb = (frame8[:, 1::4].astype(np.uint32) << 2) | rng.integers(0, 4, (h, w // 2)).astype(np.uint32)
    cr = (frame8[:, 3::4].astype(np.uint32) << 2) | rng.integers(0, 4, (h, w // 2)).astype(np.uint32)
    return pack_v210(y, cb, cr), [y.astype(np.int16), cr.astype(np.int16), cb.astype(np.int16)]


# ---------------------------------------------------------------- 10-bit packed RGB (one 32-bit word per pixel)
RGB30_FORMATS = {          # name: (COLOR_FORMAT_* of Codec/color.h, byte swapped, bit position of R, G, B)
    "RG30": (122, False, (0, 10, 20)),
    "R210": (123, True, (20, 10, 0)),
    "AR10": (124, False, (20, 10, 0)),
    "AB10": (125, False, (0, 10, 20)),
    "DPX0": (128, True, (22, 12, 2)),
}


def pack_rgb30(name, r, g, b):
    """10-bit r, g, b planes (h, w) -> (h, w) uint32 words in the layout of Codec/spatial.c:2118-2268."""
    _, swap, (pr, pg, pb) = RGB30_FORMATS[name]
    words = ((r.astype(np.uint32) << pr) | (g.astype(np.uint32) << pg) | (b.astype(np.uint32) << pb)).astype(np.uint32)
    return words.byteswap() if swap else words


def rgb30_planes(r, g, b, precision=12):
    """planes the reference transforms: G, R, B at `precision` bits (value << (precision - 10))."""
    sh = precision - 10
    return [(g.astype(np.int32) << sh).astype(np.int16), (r.astype(np.int32) << sh).astype(np.int16), (b.astype(np.int32) << sh).astype(np.int16)]


# ---------------------------------------------------------------- 16-bit packed outputs of the final inverse level
def row16u_tail_col(band_width):
    """First band column produced by the scalar tail of Codec/InvertHorizontalStrip16s.c:16571 InvertHorizontalStrip16sToRow16u
    (8-column SSE2 loop up to post_column = width - width % 8 - 16, one more group of 7 columns with the SIMD rule)."""
    return (band_width - band_width % 8 - 16) + 7


def row16u(plane, precision):
    """The reference's unsigned 16-bit row output of one reconstructed channel: max(v, 0) << (16 - precision), limited to
    ((1 << precision) - 1) << shift where its SSE2 loop runs (the `protection` clamp) and to 65535 in the scalar tail and
    at the right border (SATURATE_16U)."""
    s = 16 - precision
    v = np.maximum(plane.astype(np.int64), 0) << s
    hi = np.full(plane.shape[1], ((1 << precision) - 1) << s, np.int64)
    hi[2 * row16u_tail_col(plane.shape[1] // 2):] = 65535
    return np.minimum(v, hi[None, :]).astype(np.uint16)


def pack_yu64(planes, precision=10):
    """[Y, ch1, ch2] int16 planes -> packed Y0 C1 Y1 C3 (height x 2*width uint16), Codec/decoder.c:26351-26366."""
    y, c1, c3 = [row16u(p, precision) for p in planes]
    h, w = y.shape
    out = np.zeros((h, 2 * w), np.uint16)
    out[:, 0::2] = y
    out[:, 1::4] = c1
    out[:, 3::4] = c3
    return out


def pack_rg48(planes, precision=12):
    """[G, R, B] int16 planes -> packed R G B (height x 3*width uint16), Codec/wavelet.c:4947 TransformInverseRGB444ToRGB48."""
    g, r, b = [row16u(p, precision) for p in planes]
    h, w = g.shape
    out = np.zeros((h, 3 * w), np.uint16)
    out[:, 0::3], out[:, 1::3], out[:, 2::3] = r, g, b
    return out


def b64a_tail_col(band_width):
    """First band column produced by the scalar code of Codec/InvertHorizontalStrip16s.c:13298 InvertHorizontalStrip16sRGB2B64A:
    its 8-column SSE2 loop runs up to post_column = width - width % 8 (:13319) and always leaves the right border column."""
    return band_width - band_width % 8 if band_width % 8 else band_width - 1


def pack_b64a(planes, precision=12):
    """[G, R, B] int16 planes -> 16-bit A R G B words (height x 4*width uint16) as the reference's decoder writes them for
    DECODED_FORMAT_B64A (Codec/decoder.c:26862 -> InvertHorizontalStrip16s.c:13298 InvertHorizontalStrip16sRGB2B64A): alpha is
    0xfff << 4 (:13385); colour samples are limited to the 12-bit maximum where its SSE2 loop runs (:13387 limiterRGB) and to
    65535 in the scalar tail and at the right border (SATURATE_16U)."""
    s = 16 - precision
    top = ((1 << precision) - 1) << s
    h, w = planes[0].shape
    hi = np.full(w, top, np.int64)
    hi[2 * b64a_tail_col(w // 2):] = 65535
    g, r, b = [np.minimum(np.maximum(p.astype(np.int64), 0) << s, hi[None, :]).astype(np.uint16) for p in planes]
    out = np.full((h, 4 * w), top, np.uint16)
    out[:, 1::4], out[:, 2::4], out[:, 3::4] = r, g, b
    return out


def pack_rgb30_output(name, planes, precision=12):
    """[G, R, B] int16 planes -> the reference decoder's 10-bit packed RGB words (height x width uint32) for
    DECODED_FORMAT_RG30 / R210 / DPX0 / AR10 / AB10 (Codec/decoder.c:26893 -> InvertHorizontalStrip16s.c:14812
    InvertHorizontalStrip16sRGB2RG30): every sample limited to [0, 2^precision - 1] (:14892 limiterRGB; its scalar code
    clamps alike), >> 2 (:15552), packed as on the encode side.  NOTE the reference's lowpass decode adds a format-dependent
    offset to LL3 (decoder.c:12270-12316: 6 for these formats, 0 for RG48 / B64A), so its bands differ between output
    formats; that offset is applied by the host's band decode, upstream of the transform."""
    top = (1 << precision) - 1
    g, r, b = [(np.clip(p.astype(np.int64), 0, top) >> (precision - 10)).astype(np.uint32) for p in planes]
    return pack_rgb30(name, r, g, b)


def ref_decode_sample_raw(ref_lib, sample, width, height, decoded_format, num_channels, pitch):
    """Codec-level reference decode into an arbitrary DECODED_FORMAT_*; returns (bytes (height x pitch), dequantised bands).

    The reference's threaded decoder races when the host is oversubscribed (its output conversion can overtake a
    transform worker: a whole channel of the returned frame then disagrees with the bands the decoder holds; seen about
    once in 40 decodes under `pytest -n 8`, never on an idle host).  That is the reference's defect, not part of the
    transform under test, so the decode is repeated until two consecutive runs return the same frame and bands."""
    prev = None
    for _ in range(8):
        cur = _ref_decode_sample_raw_once(ref_lib, sample, width, height, decoded_format, num_channels, pitch)
        if prev is not None and np.array_equal(prev[0], cur[0]) and all(np.array_equal(prev[1][k], cur[1][k]) for k in cur[1]):
            return cur
        prev = cur
    return prev


def _ref_decode_sample_raw_once(ref_lib, sample, width, height, decoded_format, num_channels, pitch):
    out = np.zeros((height, pitch), np.uint8)
    dims = np.zeros(num_channels * 9, np.int32)
    quant = np.zeros(num_channels * 12, np.int32)
    cap = width * height * 4 * num_channels
    b = np.zeros(cap, np.int16)
    sample = np.ascontiguousarray(sample)
    rc = ref_lib.ref_decode_sample_bands(sample.ctypes.data_as(C.c_void_p), C.c_int64(sample.size), width, height,
                                         decoded_format, num_channels, out.ctypes.data_as(C.c_void_p), pitch,
                                         dims.ctypes.data_as(C.c_void_p), quant.ctypes.data_as(C.c_void_p),
                                         b.ctypes.data_as(C.c_void_p), C.c_int64(cap))
    assert rc == 0, f"reference decode failed ({rc})"
    bands, pos = {}, 0
    for c in range(num_channels):
        for k in range(3):
            w, h = int(dims[(c * 3 + k) * 3]), int(dims[(c * 3 + k) * 3 + 1])
            for bi in range(4):
                bands[(c, k + 1, BAND_NAMES[bi])] = b[pos:pos + w * h].reshape(h, w).copy()
                pos += w * h
    return out, bands
