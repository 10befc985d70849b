"""Shared helpers for the parity tests (test infrastructure)."""
import ctypes as C

import numpy as np

import oracle_lib as ol

COLOR_FORMAT_UYVY, COLOR_FORMAT_YUYV, COLOR_FORMAT_RG48, COLOR_FORMAT_BYR4 = 1, 2, 120, 104  # Codec/color.h:64-131
COLOR_FORMAT_V210, COLOR_FORMAT_YU64, COLOR_FORMAT_BYR5 = 10, 12, 105
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


def ref_decode_sample_bands(ref_lib, sample, width, height, decoded_format=COLOR_FORMAT_YUYV, num_channels=3):
    """One Codec-level reference decode; returns (decoded packed frame, {(c, level, name): DEQUANTISED band})."""
    return _ref_decode_once(ref_lib, sample, width, height, decoded_format, num_channels, width * 2)


def ref_decode(ref_lib, sample, w, h, decoded_format, nchan, pitch, *, resolution=None, bayer=None, agree=None):
    """Codec-level reference decode of `sample` into DECODED_FORMAT_* `decoded_format`; returns (bytes (h x pitch),
    {(c, level, name): DEQUANTISED band the decoder held}).  The probe decodes into a zero-filled buffer of its own and
    copies all of it, so bytes the decoder leaves alone come back as 0.
    resolution: DECODED_RESOLUTION_* for the decode (ref_set_decode_resolution), full resolution again afterwards.
    bayer: (phase, encode_curve_preset) set on the decoder of a Bayer sample (the sample does not carry them), through
    oracle/ref_probe_bayer.cpp (`ref_lib` is its library); also returns ((phase, preset) the decoder held after the decode,
    its linear-restore table or None).
    agree: a byte mask broadcast over the frame; only the bytes it selects are compared between runs (below).

    The reference's threaded decoder races when the host is oversubscribed (its output conversion can overtake a
    transform worker: a whole channel of the returned frame then disagrees with the bands the decoder holds; seen about
    once in 40 decodes under `pytest -n 8`, never on an idle host).  That is the reference's defect, not part of the
    transform under test, so the decode is repeated, up to 8 times, until two consecutive runs return the same frame and
    bands."""
    if resolution is not None:
        set_res = ref_lib.ref_set_decode_resolution
        set_res.argtypes, set_res.restype = [C.c_int], None
        set_res(resolution)
    try:
        prev = None
        for _ in range(8):
            cur = _ref_decode_once(ref_lib, sample, w, h, decoded_format, nchan, pitch, bayer)
            if prev is not None and all(np.array_equal(prev[1][k], cur[1][k]) for k in cur[1]) and \
                    (np.array_equal(prev[0], cur[0]) if agree is None else np.array_equal(prev[0] & agree, cur[0] & agree)):
                return cur
            prev = cur
        return prev
    finally:
        if resolution is not None:
            set_res(1)


def _ref_decode_once(ref_lib, sample, w, h, decoded_format, nchan, pitch, bayer=None):
    out = np.zeros((h, pitch), np.uint8)
    dims = np.zeros(nchan * 9, np.int32)
    quant = np.zeros(nchan * 12, np.int32)
    cap = w * h * 4 * nchan
    b = np.zeros(cap, np.int16)
    sample = np.ascontiguousarray(sample)
    vp = C.c_void_p
    if bayer is None:
        rc = ref_lib.ref_decode_sample_bands(vp(sample.ctypes.data), C.c_int64(sample.size), w, h, decoded_format, nchan,
                                             vp(out.ctypes.data), pitch, vp(dims.ctypes.data), vp(quant.ctypes.data),
                                             vp(b.ctypes.data), C.c_int64(cap))
    else:
        state, table = np.zeros(3, np.int32), np.zeros(16384, np.uint16)
        rc = ref_lib.ref_decode_bayer_bands(vp(sample.ctypes.data), C.c_int64(sample.size), w, h, decoded_format, nchan,
                                            bayer[0], bayer[1], vp(out.ctypes.data), pitch, vp(dims.ctypes.data),
                                            vp(quant.ctypes.data), vp(b.ctypes.data), C.c_int64(cap), vp(state.ctypes.data),
                                            vp(table.ctypes.data))
    assert rc == 0, f"reference decode failed ({rc})"
    bands, pos = {}, 0
    for c in range(nchan):
        for k in range(3):
            bw, bh = int(dims[(c * 3 + k) * 3]), int(dims[(c * 3 + k) * 3 + 1])
            for bi in range(4):
                bands[(c, k + 1, BAND_NAMES[bi])] = b[pos:pos + bw * bh].reshape(bh, bw).copy()
                pos += bw * bh
    if bayer is None:
        return out, bands
    return out, bands, (int(state[0]), int(state[1])), table if state[2] else None


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


UNIT_DIVISORS = [[[1, 1, 1, 1]] * 3] * 3


# ---------------------------------------------------------------- RG48 (packed 16-bit RGB -> 4:4:4, 12 bit)
CFHD_PIXEL_FORMAT_RG48 = (ord("R") << 24) | (ord("G") << 16) | (ord("4") << 8) | ord("8")


def qbist_rg48(ref_lib, width, height, frame_number=1, seed=50):
    pitch = width * 6
    out = np.zeros((height, pitch), np.uint8)
    ref_lib.ref_qbist_frames(seed, width, height, pitch, CFHD_PIXEL_FORMAT_RG48, frame_number, out.reshape(-1))
    return out.view(np.uint16)          # (height, 3*width)


def forward_pyramid_planes(impl, planes, divisors, prescale, midpoint=2):
    """3-level pyramid of already unpacked int16 planes (level 1 uses the plain / V210 variant by prescale[0])."""
    out = {}
    for c, ll in enumerate(planes):
        for k in range(3):
            variant = 1 if prescale[k] == 2 else 0
            ll, lh, hl, hh = impl.fwd_level(ll, variant, divisors[c][k], midpoint)
            out[(c, k + 1, "LL")], out[(c, k + 1, "LH")], out[(c, k + 1, "HL")], out[(c, k + 1, "HH")] = ll, lh, hl, hh
    return out


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


