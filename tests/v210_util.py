"""V210 output of the final 4:2:2 inverse level: a numpy restatement of the frame the reference decoder writes for
DECODED_FORMAT_V210, and the helpers the V210 output tests share (test infrastructure)."""
import ctypes as C

import numpy as np

import parity_util as pu

DECODED_FORMAT_V210, DECODED_FORMAT_YU64 = 10, 12        # Codec/decoder.h DECODED_FORMAT_*
CANARY = 0xA5                                             # fill of output buffers: bytes nobody writes keep it


def row_bytes(w):
    """Bytes of one V210 row: ceil(W / 6) groups of 16 bytes (the last one partial when W % 6 != 0)."""
    return (w + 5) // 6 * 16


def natural_pitch(w):
    """cfb_layout.frame_pitch of a V210 codec: rows padded to 48 pixels = 128 bytes."""
    return (w + 47) // 48 * 128


def pack_v210_components(y, cr, cb):
    """10-bit components y (h, w), cr / cb (h, w/2) -> V210 words (h, 4 * ceil(W / 6)) uint32 as
    Codec/convert.c:13526 ConvertPlanarYUVToV210 writes them: Cb0 Y0 Cr0 | Y1 Cb1 Y2 | Cr1 Y3 Cb2 | Y4 Cr2 Y5 at bits 0 / 10 / 20.
    The partial last group of W % 6 != 0 follows its scalar loop (:13889-13965), which keeps the previous components
    where a column is past the width.  At W % 6 == 4 that loop reads one Cb sample past the row (X, not reproducible);
    this restatement puts Cb1 there, as the library does."""
    y, cr, cb = [np.asarray(a, np.uint32) for a in (y, cr, cb)]
    h, w = y.shape
    full, rem = w // 6, w % 6
    ng = full + (rem > 0)
    comp = np.zeros((h, ng, 12), np.uint32)
    for p in range(3):
        comp[:, :full, 4 * p] = cb[:, p:3 * full:3]
        comp[:, :full, 4 * p + 1] = y[:, 2 * p:6 * full:6]
        comp[:, :full, 4 * p + 2] = cr[:, p:3 * full:3]
        comp[:, :full, 4 * p + 3] = y[:, 2 * p + 1:6 * full:6]
    if rem:
        c = 6 * full
        cb0, y0, cr0, y1 = cb[:, c // 2], y[:, c], cr[:, c // 2], y[:, c + 1]
        if rem == 2:
            tail = [cb0, y0, cr0, y1, cb0, y0, cr0, y1, cb0, y1, cr0, y0]
        else:
            cb1, y2, cr1, y3 = cb[:, c // 2 + 1], y[:, c + 2], cr[:, c // 2 + 1], y[:, c + 3]
            tail = [cb0, y0, cr0, y1, cb1, y2, cr1, y3, cb1, y3, cr1, y2]
        comp[:, full, :] = np.stack(tail, axis=1)
    words = comp[:, :, 0::3] | (comp[:, :, 1::3] << 10) | (comp[:, :, 2::3] << 20)
    return words.reshape(h, 4 * ng).astype(np.uint32)


def pack_v210_output(planes, precision=10):
    """[Y, ch1, ch2] int16 planes of a 4:2:2 decode -> the reference decoder's V210 words (decoder.c:26303 ->
    InvertHorizontalStrip16s.c:6490 -> convert.c:16126 ConvertYUVStripPlanarToV210 with precision 16): every component is
    the ...ToRow16u sample of YU64 (parity_util.row16u) >> 6; Cb = channel 2, Cr = channel 1."""
    y, cr, cb = [pu.row16u(p, precision) >> 6 for p in planes]
    return pack_v210_components(y, cr, cb)


def x_mask(w):
    """Per-word mask (4 * ceil(W / 6),) that clears the one field the reference does not determine: X, bits 20-29 of word 2
    of the last group when W % 6 == 4."""
    m = np.full(4 * ((w + 5) // 6), 0xFFFFFFFF, np.uint32)
    if w % 6 == 4:
        m[-2] = ~np.uint32(0x3FF << 20)
    return m


def frame_words(buf, w, h):
    """The V210 words of a frame buffer (h rows of `pitch` bytes, any dtype) -> (h, 4 * ceil(W / 6)) uint32."""
    b = np.ascontiguousarray(buf).view(np.uint8).reshape(h, -1)
    return np.ascontiguousarray(b[:, :row_bytes(w)]).view("<u4")


def ref_decode_v210(ref_lib, sample, w, h, pitch):
    """The reference decoder's V210 frame of `sample` as (h, pitch) bytes, and the dequantised bands it held.  The probe
    decodes into a zero-filled buffer of its own and copies all of it, so bytes the decoder leaves alone come back as 0.
    As parity_util.ref_decode_sample_raw, the decode is repeated until two runs agree (its threaded decoder can race on an
    oversubscribed host); X is left out of that comparison because it is whatever the decoder's buffer held."""
    mask = x_mask(w)
    prev = None
    for _ in range(8):
        cur = _ref_decode_v210_once(ref_lib, sample, w, h, pitch)
        if prev is not None and np.array_equal(frame_words(prev[0], w, h) & mask, frame_words(cur[0], w, h) & mask) and \
                all(np.array_equal(prev[1][k], cur[1][k]) for k in cur[1]):
            return cur
        prev = cur
    return prev


def _ref_decode_v210_once(ref_lib, sample, w, h, pitch):
    nchan = 3
    out = np.zeros((h, pitch), np.uint8)
    dims = np.zeros(nchan * 9, np.int32)
    quant = np.zeros(nchan * 12, np.int32)
    cap = w * h * 4 * nchan
    b = np.zeros(cap, np.int16)
    sample = np.ascontiguousarray(sample)
    rc = ref_lib.ref_decode_sample_bands(sample.ctypes.data_as(C.c_void_p), C.c_int64(sample.size), w, h, DECODED_FORMAT_V210,
                                         nchan, out.ctypes.data_as(C.c_void_p), pitch, dims.ctypes.data_as(C.c_void_p),
                                         quant.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), C.c_int64(cap))
    assert rc == 0, f"reference decode failed ({rc})"
    bands, pos = {}, 0
    for c in range(nchan):
        for k in range(3):
            bw, bh = int(dims[(c * 3 + k) * 3]), int(dims[(c * 3 + k) * 3 + 1])
            for bi in range(4):
                bands[(c, k + 1, pu.BAND_NAMES[bi])] = b[pos:pos + bw * bh].reshape(bh, bw).copy()
                pos += bw * bh
    return out, bands
