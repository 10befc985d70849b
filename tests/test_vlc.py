"""Host run-length / VLC packing straight from the sparse transfer format (SURVEY 8f rank 1, host side).

The product entry point cfb_sparse_vlc_band must write, bit for bit, what the reference's EncodeQuantLongRuns
(Codec/encoder.c:5386) writes for the same band with the same code tables -- including the state it leaves in the 32-bit
bit buffer -- while reading only the sparse format.  The reference's coder and its tables come from oracle/_ref
(ref_probe.cpp ref_vlc_*); nothing here needs a GPU."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
import parity_util as pu
from gpu_fixtures import pkg  # noqa: F401

needs_ref = pytest.mark.skipif(not ol.ref_available(), reason="oracle/_ref not built (reference absent)")


def ref_tables(ref_lib, codebook):
    rl, vl = C.c_int32(), C.c_int32()
    assert ref_lib.ref_vlc_table_lengths(codebook, C.byref(rl), C.byref(vl)) == 1
    rb, rs, rc = np.zeros(rl.value, np.uint32), np.zeros(rl.value, np.uint8), np.zeros(rl.value, np.uint32)
    vb, vs = np.zeros(vl.value, np.uint32), np.zeros(vl.value, np.uint8)
    assert ref_lib.ref_vlc_tables(codebook, rb.ctypes.data_as(C.c_void_p), rs.ctypes.data_as(C.c_void_p), rc.ctypes.data_as(C.c_void_p),
                                  vb.ctypes.data_as(C.c_void_p), vs.ctypes.data_as(C.c_void_p)) == 1
    return rb, rs, rc, vb, vs


def ref_encode_band(ref_lib, band_padded, width, codebook, lead_bits):
    """The reference's EncodeQuantLongRuns on a (height x pitch/2) int16 array whose first `width` columns are the band."""
    h, pitch = band_padded.shape[0], band_padded.strides[0]
    cap = 4 * band_padded.size + 4096
    out = np.zeros(cap, np.uint8)
    buf, free = C.c_uint32(), C.c_int32()
    fn = ref_lib.ref_vlc_encode_band
    fn.restype = C.c_int64
    n = fn(band_padded.ctypes.data_as(C.c_void_p), width, h, pitch, codebook, lead_bits, out.ctypes.data_as(C.c_void_p),
           C.c_int64(cap), C.byref(buf), C.byref(free))
    assert n >= 0
    return out[:n].copy(), int(buf.value), int(free.value)


def all_bands(lay):
    for c in range(lay.num_channels):
        for k in (2, 1, 0):
            for b in range(4):
                if b == 0 and k != 2:
                    continue
                yield c, k, b


def check_frame(pkg, ref_lib, lay, coded, book, codebook, lead_bits):
    sparse = pkg.sparse_compact(lay, coded)
    assert np.array_equal(pkg.sparse_expand(lay, sparse), coded)
    total_bits = 0
    for c, k, b in all_bands(lay):
        bl = lay.band[c][k][b]
        padded = coded[bl.offset: bl.offset + bl.pitch * bl.height].view(np.int16).reshape(bl.height, bl.pitch // 2)
        want = ref_encode_band(ref_lib, padded, bl.width, codebook, lead_bits)
        cap = want[0].size + 64
        got = pkg.sparse_vlc_band(lay, sparse, c, k, b, book, cap, lead_bits)
        assert np.array_equal(got[0], want[0]), f"band ({c},{k},{b}): stream differs"
        assert got[1:] == want[1:], f"band ({c},{k},{b}): bit-buffer state differs {got[1:]} vs {want[1:]}"
        dense = pkg.dense_vlc_band(padded, bl.pitch, bl.width, book, cap, lead_bits)
        assert np.array_equal(dense[0], want[0]) and dense[1:] == want[1:]
        assert pkg.sparse_band_nonzeros(lay, sparse, c, k, b) == int(np.count_nonzero(padded[:, :bl.width]))
        assert np.array_equal(pkg.sparse_expand_band(lay, sparse, c, k, b), padded[:, :bl.width])
        total_bits += want[0].size * 8
    return total_bits, sparse.size


@needs_ref
@pytest.mark.parametrize("size,lead", [((256, 64), 0), ((704, 96), 5), ((720, 480), 31), ((1920, 1080), 13)])
def test_vlc_from_sparse_matches_reference_coder_on_qbist(pkg, size, lead):
    """TestCFHD's Qbist frames through the reference's real encoder; every coded band of every channel."""
    w, h = size
    ref_lib = ol.load_ref()
    frame = pu.qbist_yuy2(ref_lib, w, h, 3)
    bands, _, _, sample = pu.ref_encode_frame(ref_lib, frame, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, 4)
    lay = pkg.layout_for(pkg.FrameDesc(w, h, pkg.PIXEL_YUYV))
    coded = pkg.pack_coded(lay, bands)
    book = pkg.VlcCodebook.from_arrays(*ref_tables(ref_lib, 1))
    bits, sparse_bytes = check_frame(pkg, ref_lib, lay, coded, book, 1, lead)
    # the highpass payload is the bulk of the reference's sample: the per-band streams add up to (almost) its size
    assert 0.5 * sample.size < bits / 8 < 1.5 * sample.size
    if w >= 1920:
        assert sparse_bytes < lay.coded_bytes // 8


@needs_ref
@pytest.mark.parametrize("codebook", [0, 1, 2])
@pytest.mark.parametrize("kind", ["dense-small", "sparse-large", "extreme", "empty", "single"])
def test_vlc_from_sparse_matches_reference_coder_adversarial(pkg, codebook, kind):
    """Every code set; values beyond the table (clamp), beyond a byte (escapes), runs longer than any run code and across
    block / band boundaries, an all-zero frame, a single coefficient at the very end."""
    ref_lib = ol.load_ref()
    lay = pkg.layout_for(pkg.FrameDesc(704, 96, pkg.PIXEL_YUYV))
    rng = np.random.default_rng(len(kind) + codebook)
    words = lay.coded_bytes // 2
    dense = np.zeros(words, np.int16)
    if kind == "dense-small":
        dense[:] = rng.integers(-3, 4, words)
    elif kind == "sparse-large":
        nz = rng.random(words) < 0.01
        dense[nz] = rng.integers(-2000, 2000, int(nz.sum()))
    elif kind == "extreme":
        nz = rng.random(words) < 0.2
        dense[nz] = rng.choice(np.array([-32768, -32767, -1025, -1024, -1023, -512, -129, -128, -127, -1, 1, 127, 128, 129, 511, 512, 1023, 1024, 32767], np.int16), int(nz.sum()))
    elif kind == "single":
        dense[-1] = -5
    coded = dense.view(np.uint8).copy()
    # the pitch gap and the band alignment are zero in a real coded region
    clean = np.zeros_like(coded)
    for c, k, b in all_bands(lay):
        pkg.band_view(lay, clean, c, k, b)[:] = pkg.band_view(lay, coded, c, k, b)
    book = pkg.VlcCodebook.from_arrays(*ref_tables(ref_lib, codebook))
    check_frame(pkg, ref_lib, lay, clean, book, codebook, 7)


def test_vlc_rejects_bad_arguments(pkg):
    lay = pkg.layout_for(pkg.FrameDesc(256, 64, pkg.PIXEL_YUYV))
    sparse = pkg.sparse_compact(lay, np.zeros(lay.coded_bytes, np.uint8))
    book = pkg.VlcCodebook.from_arrays(np.array([0, 1, 2], np.uint32), np.array([1, 2, 3], np.uint8), np.array([1, 1, 2], np.uint32),
                                       np.arange(8, dtype=np.uint32), np.full(8, 4, np.uint8))
    with pytest.raises(pkg.CfbError):
        pkg.sparse_vlc_band(lay, sparse, 0, 0, 0, book, 4096)          # LL1 is not in the coded region
    with pytest.raises(pkg.CfbError):
        pkg.sparse_vlc_band(lay, sparse, 3, 2, 1, book, 4096)          # no such channel
    with pytest.raises(pkg.CfbError):
        pkg.sparse_vlc_band(lay, sparse, 0, 0, 1, book, 0)             # no room: all-zero band still needs run codes
    bad = sparse.copy(); bad[0] ^= 1
    with pytest.raises(pkg.CfbError):
        pkg.sparse_vlc_band(lay, bad, 0, 0, 1, book, 4096)
    # a run table whose entry covers more zeros than the run it is chosen for would never terminate in the reference
    worse = pkg.VlcCodebook.from_arrays(np.array([0, 1, 2], np.uint32), np.array([1, 2, 3], np.uint8), np.array([1, 2, 2], np.uint32),
                                        np.arange(8, dtype=np.uint32), np.full(8, 4, np.uint8))
    with pytest.raises(pkg.CfbError):
        pkg.sparse_vlc_band(lay, sparse, 0, 0, 1, worse, 4096)


# ---------------------------------------------------------------------------------------------------- decoder side
def ref_encode_band_finished(ref_lib, band_padded, width, codebook):
    h, pitch = band_padded.shape[0], band_padded.strides[0]
    cap = 4 * band_padded.size + 4096
    out = np.zeros(cap, np.uint8)
    fn = ref_lib.ref_vlc_encode_band_finished
    fn.restype = C.c_int64
    n = fn(band_padded.ctypes.data_as(C.c_void_p), width, h, pitch, codebook, out.ctypes.data_as(C.c_void_p), C.c_int64(cap))
    assert n > 0
    return out[:n].copy()


def ref_decode_band(ref_lib, stream, width, height, pitch, codebook, quant):
    out = np.zeros((height, pitch // 2), np.int16)
    rc = ref_lib.ref_vlc_decode_band(stream.ctypes.data_as(C.c_void_p), C.c_int64(stream.size), width, height, pitch, codebook, quant,
                                     out.ctypes.data_as(C.c_void_p))
    assert rc == 0, rc
    return out


def decode_book(pkg, ref_lib, codebook):
    """Every code word of code set `codebook` once.  Run codes and the end-of-band code come from the encoder's tables; the
    value a coefficient code DECODES to (the codec compands magnitudes above 27 inside its entropy coder, codebooks.c:932)
    is learnt from the reference's own FSM decoder: one band holding every table value once, through its coder and back."""
    rb, rs, rc, vb, vs = ref_tables(ref_lib, codebook)
    n = vb.size
    values = np.concatenate([np.arange(1, n // 2), np.arange(-(n // 2) + 1, 0)]).astype(np.int16)
    width, height, pitch = 64, (values.size + 31) // 32, 128
    band = np.zeros((height, pitch // 2), np.int16)
    band[:, 0:64:2].reshape(-1)[:values.size] = values                  # every second column: no two codes adjacent to a run boundary issue
    decoded = ref_decode_band(ref_lib, ref_encode_band_finished(ref_lib, band, width, codebook), width, height, pitch, codebook, 1)
    dec_values = decoded[:, 0:64:2].reshape(-1)[:values.size]
    codes = {}
    for v, dv in zip(values.tolist(), dec_values.tolist()):
        idx = v if v >= 0 else n + v
        key = (int(vb[idx]), int(vs[idx]))
        assert codes.setdefault(key, (0, dv)) == (0, dv), "one code, two decoded values"
    # The run table is indexed by run LENGTH: entry i holds the best single PutBits for a run of at least i zeros, and many
    # entries are concatenations of shorter run codes (codebooks.c ComputeRunLengthCodeTable packs up to 32 bits).  Only the
    # atomic code words belong in a decode book: a concatenation starts with a code word that is already in the set.
    as_string = lambda bits, size: format(bits, "b").zfill(size)[-size:]
    atoms = {as_string(*k) for k in codes}
    for i in range(1, rb.size):
        key = (int(rb[i]), int(rs[i]))
        text = as_string(*key)
        if key in codes or any(text.startswith(a) for a in atoms if len(a) < len(text)):
            continue
        codes[key] = (1, int(rc[i]))
        atoms.add(text)
    eb, es = C.c_uint32(), C.c_int32()
    assert ref_lib.ref_vlc_band_end(codebook, C.byref(eb), C.byref(es)) == 1
    codes[(int(eb.value), int(es.value))] = (2, 0)
    keys = list(codes)
    return pkg.VlcDecodebook.from_arrays([k[0] for k in keys], [k[1] for k in keys], [codes[k][0] for k in keys], [codes[k][1] for k in keys])


@needs_ref
@pytest.mark.parametrize("size", [(256, 64), (704, 96), (720, 480), (1920, 1080)])
def test_band_streams_to_sparse_match_reference_fsm_decoder(pkg, size):
    """Decoder side of the hand-over: the band bit streams of a Qbist frame (the reference's coder, end-of-band code and
    padding included) are parsed straight into the sparse format; expanded, it equals band for band what the reference's
    FSM decoder (DecodeBandFSM16sNoGap, tables scaled by the band's quantiser) writes into its dense bands."""
    w, h = size
    ref_lib = ol.load_ref()
    frame = pu.qbist_yuy2(ref_lib, w, h, 2)
    bands, div, _, _ = pu.ref_encode_frame(ref_lib, frame, w, h, pu.COLOR_FORMAT_YUYV, 0, 3, 4)
    lay = pkg.layout_for(pkg.FrameDesc(w, h, pkg.PIXEL_YUYV))
    coded = pkg.pack_coded(lay, bands)
    dec = pkg.VlcDecoder(lay, decode_book(pkg, ref_lib, 1))
    dec.begin()
    want = np.zeros(lay.coded_bytes, np.uint8)
    for c, k, b in all_bands(lay):
        bl = lay.band[c][k][b]
        padded = coded[bl.offset: bl.offset + bl.pitch * bl.height].view(np.int16).reshape(bl.height, bl.pitch // 2)
        if b == 0:                      # LL3 travels as plain 16-bit values
            dec.dense_band(c, k, b, padded[:, :bl.width])
            pkg.band_view(lay, want, c, k, b)[:] = padded[:, :bl.width]
            continue
        quant = div[c][k][b]
        stream = ref_encode_band_finished(ref_lib, padded, bl.width, 1)
        used = dec.band(c, k, b, stream, quant)
        assert stream.size - 4 <= used <= stream.size
        pkg.band_view(lay, want, c, k, b)[:] = ref_decode_band(ref_lib, stream, bl.width, bl.height, bl.pitch, 1, quant)[:, :bl.width]
    sparse = dec.end()
    assert np.array_equal(pkg.sparse_expand(lay, sparse), want)
    assert np.array_equal(sparse, pkg.sparse_compact(lay, want))            # and byte for byte the canonical packing
    dec.close()


def test_sparse_writer_rejects_misuse(pkg):
    lay = pkg.layout_for(pkg.FrameDesc(256, 64, pkg.PIXEL_YUYV))
    book = pkg.VlcDecodebook.from_arrays([0b0, 0b10, 0b11], [1, 2, 2], [1, 0, 2], [1, 5, 0])
    dec = pkg.VlcDecoder(lay, book)
    dec.begin()
    with pytest.raises(pkg.CfbError):
        dec.band(0, 0, 1, np.array([0x00, 0x00], np.uint8), 1)            # zero runs only, never an end-of-band code
    dec.begin()
    dec.band(0, 2, 1, np.array([0b10110000], np.uint8), 3)                 # value 5 * 3, end of band
    with pytest.raises(pkg.CfbError):
        dec.band(0, 2, 1, np.array([0b11000000], np.uint8), 1)             # the same band again: not the next one
    with pytest.raises(pkg.CfbError):
        pkg.VlcDecoder(lay, pkg.VlcDecodebook.from_arrays([0b0, 0b01], [1, 2], [1, 2], [1, 0]))      # 0 is a prefix of 01
    dec.close()


# ---------------------------------------------------------------------------------------------------- robustness
def test_host_parsers_survive_damaged_input(pkg):
    """Host entry points that take buffers from outside (a sparse buffer from the wire, a band bit stream) must answer a
    damaged one with an error or with a well-formed result -- never read or write out of bounds (the process would die)."""
    lay = pkg.layout_for(pkg.FrameDesc(704, 96, pkg.PIXEL_YUYV))
    rng = np.random.default_rng(11)
    words = lay.coded_bytes // 2
    dense = np.where(rng.random(words) < 0.1, rng.integers(-900, 900, words), 0).astype(np.int16)
    good = pkg.sparse_compact(lay, dense.view(np.uint8))
    book = pkg.VlcCodebook.from_arrays(np.arange(40, dtype=np.uint32) | 0x100, np.full(40, 9, np.uint8), np.minimum(np.arange(40), 7).clip(1).astype(np.uint32),
                                       np.arange(64, dtype=np.uint32), np.full(64, 7, np.uint8))
    outcomes = {"ok": 0, "error": 0}
    for trial in range(300):
        bad = np.zeros(pkg.sparse_max_bytes(lay), np.uint8)        # buffers on the wire have the worst-case size (header)
        bad[:good.size] = good
        n = int(rng.integers(1, 6))
        pos = rng.integers(0, good.size, n) if trial % 3 else rng.integers(0, 32 + 16 * ((words + 8191) // 8192), n)   # often hit header / table
        bad[pos] = rng.integers(0, 256, n).astype(np.uint8)
        for call in (lambda: pkg.sparse_expand(lay, bad),
                     lambda: pkg.sparse_vlc_band(lay, bad, 0, 0, 1, book, 1 << 20),
                     lambda: pkg.sparse_expand_band(lay, bad, 2, 1, 3),
                     lambda: pkg.sparse_band_nonzeros(lay, bad, 1, 0, 2)):
            try:
                call()
                outcomes["ok"] += 1
            except pkg.CfbError:
                outcomes["error"] += 1
    assert outcomes["error"] > 50 and outcomes["ok"] > 50           # both kinds of damage occurred
    # random band streams through the table-driven parser
    dbook = pkg.VlcDecodebook.from_arrays([0b0, 0b10, 0b110, 0b1110, 0b1111], [1, 2, 3, 4, 4], [1, 0, 0, 1, 2], [1, 3, -3, 40, 0])
    dec = pkg.VlcDecoder(lay, dbook)
    for trial in range(200):
        dec.begin()
        stream = rng.integers(0, 256, int(rng.integers(1, 400))).astype(np.uint8)
        try:
            dec.band(0, 2, 1, stream, int(rng.integers(1, 50)))
            back = pkg.sparse_expand(lay, dec.end())                # whatever was accepted is a well-formed buffer
            assert back.size == lay.coded_bytes
        except pkg.CfbError:
            pass
    dec.close()


def _toy_books(pkg):
    """A small prefix-free code set (value table of 8 entries, i.e. shorter than the coder's fast-pair range)."""
    run_bits, run_size, run_count = [0, 0b10, 0b110, 0b1110], [0, 2, 3, 4], [0, 1, 2, 3]
    vcode = {1: "00", -1: "010", 2: "0110", -2: "01110", 3: "011110", -3: "0111110"}
    vb, vs = np.zeros(8, np.uint32), np.zeros(8, np.uint8)
    for v, text in vcode.items():
        vb[v if v >= 0 else 8 + v], vs[v if v >= 0 else 8 + v] = int(text, 2), len(text)
    vb[0], vs[0] = 0b0111111, 7            # never used by the coder (zeros are runs); keeps the table free of zero-length codes
    vb[4], vs[4] = 0b0111111, 7
    enc = pkg.VlcCodebook.from_arrays(np.array(run_bits, np.uint32), np.array(run_size, np.uint8), np.array(run_count, np.uint32), vb, vs)
    bits = [0b10, 0b110, 0b1110, 0b1111] + [int(t, 2) for t in vcode.values()]
    size = [2, 3, 4, 4] + [len(t) for t in vcode.values()]
    kind = [1, 1, 1, 2] + [0] * len(vcode)
    arg = [1, 2, 3, 0] + list(vcode.keys())
    return enc, pkg.VlcDecodebook.from_arrays(bits, size, kind, arg)


def test_toy_code_set_round_trip_through_coder_and_parser(pkg):
    """Property test without the reference: any prefix-free code set, coder -> band stream -> parser -> the same sparse
    buffer.  The value table has 8 entries (shorter than the pre-joined pair range: regression for an out-of-bounds read
    found with AddressSanitizer), runs are longer than the longest run code, values beyond the table are clamped."""
    lay = pkg.layout_for(pkg.FrameDesc(256, 64, pkg.PIXEL_YUYV))
    enc, dec_book = _toy_books(pkg)
    rng = np.random.default_rng(11)
    coded = np.zeros(lay.coded_bytes, np.uint8)
    for c, k, b in all_bands(lay):
        view = pkg.band_view(lay, coded, c, k, b)
        nz = rng.random(view.shape) < (0.3 if k == 2 else 0.02)
        view[nz] = rng.choice(np.array([-3, -2, -1, 1, 2, 3], np.int16), int(nz.sum()))
    sparse = pkg.sparse_compact(lay, coded)
    dec = pkg.VlcDecoder(lay, dec_book)
    dec.begin()
    for c, k, b in all_bands(lay):
        bl = lay.band[c][k][b]
        words, pending, free = pkg.sparse_vlc_band(lay, sparse, c, k, b, enc, 8 * bl.pitch * bl.height + 64, 0)
        padded = coded[bl.offset: bl.offset + bl.pitch * bl.height].view(np.int16).reshape(bl.height, bl.pitch // 2)
        dense = pkg.dense_vlc_band(padded, bl.pitch, bl.width, enc, 8 * bl.pitch * bl.height + 64, 0)
        assert np.array_equal(dense[0], words) and dense[1:] == (pending, free)
        # finish the stream the way the host coder does: pending bits, end-of-band code, zero padding to a word
        text = "".join(format(int(x), "08b") for x in words) + (format(pending, "b").zfill(32 - free)[-(32 - free):] if free < 32 else "") + "1111"
        text += "0" * (-len(text) % 32)
        stream = np.array([int(text[i:i + 8], 2) for i in range(0, len(text), 8)], np.uint8)
        dec.band(c, k, b, stream, 1)
    out = dec.end()
    assert np.array_equal(out, sparse)
    # a value outside the table is clamped to the largest code (vlc.c:188): 100 decodes as 3
    one = np.zeros(lay.coded_bytes, np.uint8)
    pkg.band_view(lay, one, 0, 2, 1)[0, 0] = 100
    words, pending, free = pkg.sparse_vlc_band(lay, pkg.sparse_compact(lay, one), 0, 2, 1, enc, 4096, 0)
    head = ("".join(format(int(x), "08b") for x in words) + format(pending, "b").zfill(32 - free))[:6]
    assert head == "011110"
    dec.close()
