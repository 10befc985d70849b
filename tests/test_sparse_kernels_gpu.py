"""k_sparse_pack / k_sparse_unpack alone, on arbitrary coded regions, against the numpy restatement of 'CFS2' (sparse_ref.py).

With both level masks at 0 the codec runs no transform: inverse_host only uploads a coded region into the slots,
forward_host only downloads it, forward_host_sparse runs k_sparse_pack on the slots and nothing else, and
inverse_host_sparse runs k_sparse_unpack and nothing else.  Every such call is checked to launch exactly the kernels it
should, so each comparison below is one kernel against the reference."""
import numpy as np
import pytest

import formats as fm
import parity_util as pu
import sparse_ref as sr
from gpu_fixtures import pkg  # noqa: F401

pytestmark = pytest.mark.gpu

BADFORMAT = 3

# (source, width, height, frames per launch); the last block of the coded region holds 32 / 8160 / 8192 words
LAYOUTS = [("YUYV", 288, 208, 16), ("YUYV", 224, 304, 16), ("YUYV", 256, 48, 16), ("RG48", 232, 56, 16),
           ("RG48", 600, 152, 16), ("BYR4", 240, 96, 16), ("YUYV", 3840, 2160, 16), ("BYR4", 8192, 4320, 4)]
PARTIAL = [lay for lay in LAYOUTS if lay[1:3] in ((288, 208), (224, 304), (232, 56), (600, 152))]
SMALL = LAYOUTS[:6]
OUT_FORMAT = {"YUYV": "YUYV", "RG48": "RG48", "BYR4": "BYR4"}


def _ids(layouts):
    return [f"{s}-{w}x{h}" for s, w, h, _ in layouts]


class Slots:
    """The coded regions of a codec's slots, moved and converted with the transforms switched off."""

    def __init__(self, pkg, ctx, codec, src):
        self.pkg, self.ctx, self.codec = pkg, ctx, codec
        lay = codec.layout
        self.nwords = lay.coded_bytes // 2
        self.quant = pkg.quant_for_quality(codec.desc, 4)          # read by no kernel: both masks are 0
        self.frame = np.zeros((lay.frame_bytes // lay.frame_pitch, lay.frame_pitch), np.uint8)
        self.out_format = getattr(pkg, "PIXEL_" + OUT_FORMAT[src])
        w, h = codec.desc.width, codec.desc.height
        self.out = np.zeros((h, fm.OUTPUTS[OUT_FORMAT[src]].row_bytes(w)), np.uint8)
        codec.set_level_mask(0, 0)

    def launches(self):
        return self.ctx.stats()["kernel_launches"]

    def _call(self, kernels, fn, *args):
        before = self.launches()
        r = fn(*args)
        assert self.launches() == before + kernels
        return r

    def load(self, dense):
        """int16 regions -> slots 0 .. n-1 (no kernel)."""
        self._call(0, self.codec.inverse_host, [d.view(np.uint8) for d in dense], self.quant, self.out_format, [self.out] * len(dense))

    def read(self, n):
        """slots 0 .. n-1 -> int16 regions (no kernel)."""
        return [d.view(np.int16) for d in self._call(0, self.codec.forward_host, [self.frame] * n, self.quant)]

    def pack(self, n, out=None):
        """k_sparse_pack on slots 0 .. n-1 -> (sparse buffers, sizes)."""
        return self._call(1, self.codec.forward_host_sparse, [self.frame] * n, self.quant, out)

    def unpack(self, sparse):
        """k_sparse_unpack of the buffers into slots 0 .. n-1."""
        self._call(1, self.codec.inverse_host_sparse, sparse, self.quant, self.out_format, [self.out] * len(sparse))


def _same_bytes(got, want, what):
    got, want = np.frombuffer(got, np.uint8), np.frombuffer(want, np.uint8)
    if got.size == want.size and np.array_equal(got, want):
        return
    n = min(got.size, want.size)
    diff = np.flatnonzero(got[:n] != want[:n])
    first = int(diff[0]) if diff.size else n
    pytest.fail(f"{what}: {got.size} bytes, reference {want.size}; {diff.size} differ, the first at byte {first}")


def _same_words(got, want, what):
    if np.array_equal(got, want):
        return
    diff = np.flatnonzero(got != want)
    w = int(diff[0])
    pytest.fail(f"{what}: {diff.size} words differ, the first at word {w} (block {w // sr.BLOCK_WORDS}): {got[w]} != {want[w]}")


def _regions(nwords, n, rng):
    """n distinct adversarial regions: the catalogue first, then the block kinds in shuffled orders."""
    if n < 8:           # the 8K batch: four regions of 4320 blocks
        out = [("blocks", sr.region(nwords, sr.BLOCK_KINDS, rng)), ("empty_runs", sr.empty_runs(nwords, rng)),
               ("escaped", sr.region(nwords, ["escaped"], rng)), ("random", sr.region(nwords, ["random"], rng))]
        return out[:n]
    out = sr.catalogue(nwords, rng)
    while len(out) < n:
        out.append((f"shuffled{len(out)}", sr.region(nwords, list(rng.permutation(sr.BLOCK_KINDS)), rng)))
    return out[:n]


def _check_pack(s, regions, out=None):
    s.load([r for _, r in regions])
    sparse, sizes = s.pack(len(regions), out)
    for (name, r), sp, size in zip(regions, sparse, sizes):
        want = sr.compact(s.nwords, r)
        total = int(sp[:16].view("<u4")[2])
        assert size == total == len(want), name
        _same_bytes(sp[:total], want, f"frame {name}: k_sparse_pack")
    return sparse


def _bands(pkg, lay, dense):
    """The region as one buffer per band (a view with the layout's pitch); the pitch gaps are not part of any band."""
    buf = dense.view(np.uint8)
    out = {}
    for c in range(lay.num_channels):
        for k in range(3):
            for b in range(4):
                if b == 0 and k != 2:
                    continue
                out[(c, k + 1, pkg.BAND_NAMES[b])] = pkg.band_view(lay, buf, c, k, b)
    return out


@pytest.mark.parametrize("src,w,h,n", LAYOUTS, ids=_ids(LAYOUTS))
def test_pack_and_unpack_match_reference(pkg, src, w, h, n):
    """1. k_sparse_pack gives the reference's bytes for n different regions in one launch (per-frame tickets and
    look-back state).  2. k_sparse_unpack restores every word of a slot that held a different region, from the
    reference's buffers and from cfb_sparse_compact_bands' (pitch gaps zero there)."""
    desc = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + src))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, n) as codec:
        s = Slots(pkg, ctx, codec, src)
        lay = codec.layout
        rng = np.random.default_rng(w * 7919 + h)
        regions = _regions(s.nwords, n, rng)
        _check_pack(s, regions)
        for source in ("reference", "bands"):
            sparse, wants = [], []
            for name, r in regions:
                if source == "reference":
                    sparse.append(np.frombuffer(sr.compact(s.nwords, r), np.uint8))
                    wants.append(r)
                else:
                    bands = _bands(pkg, lay, r)
                    sparse.append(pkg.sparse_compact_bands(lay, bands))
                    wants.append(pkg.pack_coded(lay, bands).view(np.int16))
            s.load([~want for want in wants])           # every word of every slot differs from what the unpack must give
            s.unpack(sparse)
            for (name, _), got, want in zip(regions, s.read(n), wants):
                _same_words(got, want, f"frame {name} from the {source} buffer: k_sparse_unpack")


def _natural(src, rng, w, h):
    return pu.synthetic_yuyv(rng, w, h) if src == "YUYV" else fm.synthetic_rg48(rng, w, h)


@pytest.mark.parametrize("src,w,h,n", PARTIAL, ids=_ids(PARTIAL))
def test_kernels_stay_inside_coded_region(pkg, src, w, h, n):
    """The pyramid's scratch region (LL1, LL2) starts right after the coded region, inside the last block when that
    block is partial.  Reads: with LL data there, the packer's bytes are still those of the coded region alone.
    Writes: level 1 of frame B over LL1 of frame A gives the same bytes whether B's coded region arrives dense or
    through the unpacker, which therefore left LL1 alone."""
    desc = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + src))
    fmt = getattr(pkg, "PIXEL_" + OUT_FORMAT[src])
    rng = np.random.default_rng(w + h)
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        quant = pkg.quant_for_quality(desc, 4)
        coded_a, coded_b = (codec.forward_host([_natural(src, rng, w, h)], quant)[0] for _ in range(2))
        out = np.zeros((h, 2 * w if src == "YUYV" else 6 * w), np.uint8)

        def decode_a():                                 # full decode: LL1 of A in the scratch region
            codec.set_level_mask(7, 7)
            codec.inverse_host([coded_a], quant, fmt, [out])

        decode_a()
        s = Slots(pkg, ctx, codec, src)
        nwords = s.nwords
        for name, r in sr.catalogue(nwords, rng):
            _check_pack(s, [(name, r)])

        # level 1 over A's LL1: coded regions whose last words are non-zero, so that a whole-block store would land
        full_b = np.zeros_like(out)
        codec.set_level_mask(7, 7)
        codec.inverse_host([coded_b], quant, fmt, [full_b])
        cases = [("natural", coded_b.view(np.int16))] + [(nm, r) for nm, r in sr.catalogue(nwords, rng)
                                                          if nm in ("escaped", "last_word", "last_group_first_word", "blocks0")]
        for name, r in cases:
            decode_a()
            codec.set_level_mask(0, 1)
            via_dense = np.zeros_like(out)
            codec.inverse_host([r.view(np.uint8)], quant, fmt, [via_dense])
            if name == "natural":
                assert not np.array_equal(via_dense, full_b)        # level 1 really reads A's LL1
            decode_a()
            codec.set_level_mask(0, 1)
            via_sparse = np.zeros_like(out)
            before = ctx.stats()["kernel_launches"]
            codec.inverse_host_sparse([np.frombuffer(sr.compact(nwords, r), np.uint8)], quant, fmt, [via_sparse])
            assert ctx.stats()["kernel_launches"] == before + 2     # unpack + level 1
            _same_bytes(via_sparse, via_dense, f"{name}: level 1 after the sparse hand-over")


SPECULATIVE = SMALL + [("YUYV", 3840, 2160, 1)]


@pytest.mark.parametrize("src,w,h,n", SPECULATIVE, ids=_ids(SPECULATIVE))
def test_speculative_download(pkg, src, w, h, n):
    """The download guesses the size from the previous call: an empty region (header and table only) leaves the guess
    low, a fully escaped one then takes the tail copy and pushes the guess to its clamp at sparse_max_bytes, a sparse one
    shrinks it, and the fully escaped one takes the tail copy again.  The host buffer is reused, filled with a canary."""
    desc = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + src))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 1) as codec:
        s = Slots(pkg, ctx, codec, src)
        rng = np.random.default_rng(h)
        escaped = sr.region(s.nwords, ["escaped"], rng)
        sparse = sr.region(s.nwords, ["single31", "empty", "random"], rng)
        out = [np.zeros(pkg.sparse_max_bytes(codec.layout), np.uint8)]
        sizes = []
        for name, r in (("empty", np.zeros(s.nwords, np.int16)), ("escaped", escaped), ("sparse", sparse),
                        ("escaped again", escaped), ("empty again", np.zeros(s.nwords, np.int16))):
            out[0][:] = fm.CANARY
            s.load([r])
            _, (size,) = s.pack(1, out)
            want = sr.compact(s.nwords, r)
            assert size == len(want), name
            _same_bytes(out[0][:size], want, f"{name}: speculative download")
            sizes.append(size)
        assert sizes[0] == sr.chunks_offset(sr.nblocks(s.nwords))
        assert sizes[1] > sizes[2] > sizes[0]


def _mutations(sp, nwords):
    """(name, buffer) pairs that the host must reject before anything is uploaded."""
    nb = sr.nblocks(nwords)
    lo = sr.chunks_offset(nb)
    base = np.zeros(sr.max_bytes(nwords) + 64, np.uint8)
    base[:len(sp)] = np.frombuffer(sp, np.uint8)
    table = base[32:32 + 16 * nb].view("<u4").reshape(nb, 4)
    full = [b for b in range(nb) if table[b, 1]]
    empty = [b for b in range(nb) if not table[b, 1]]
    b = full[len(full) // 2]
    total = int(base[8:12].view("<u4")[0])

    def mut(name, fn):
        buf = base.copy()
        fn(buf[:32].view("<u4"), buf[32:32 + 16 * nb].view("<u4").reshape(nb, 4))
        return name, buf

    out = [
        mut("magic", lambda h, t: h.__setitem__(0, h[0] ^ 1)),
        mut("nwords + 32", lambda h, t: h.__setitem__(1, h[1] + 32)),
        mut("nwords - 32", lambda h, t: h.__setitem__(1, h[1] - 32)),
        mut("nblocks + 1", lambda h, t: h.__setitem__(3, h[3] + 1)),
        mut("total not a multiple of 16", lambda h, t: h.__setitem__(2, h[2] + 8)),
        mut("total below the chunks", lambda h, t: h.__setitem__(2, lo - 16)),
        mut("total above the largest buffer", lambda h, t: h.__setitem__(2, sr.max_bytes(nwords) + 16)),
        mut("G > 256", lambda h, t: t.__setitem__((b, 1), 257)),
        mut("V > 8192", lambda h, t: t.__setitem__((b, 2), 8193)),
        mut("E > V", lambda h, t: t.__setitem__((b, 3), t[b, 2] + 1)),
        mut("G == 0, V != 0", lambda h, t: t.__setitem__((b, 1), 0)),
        mut("misaligned offset", lambda h, t: t.__setitem__((b, 0), t[b, 0] + 4)),
        mut("offset inside the table", lambda h, t: t.__setitem__((b, 0), lo - 16)),
        mut("chunk past the total", lambda h, t: h.__setitem__(2, h[2] - 16)),
        mut("chunk moved past the total", lambda h, t: t.__setitem__((b, 0), total - 16)),
    ]
    if empty:
        out.append(mut("G != 0, V == 0", lambda h, t: t.__setitem__((empty[0], 1), 1)))
    return base, out


@pytest.mark.parametrize("src,w,h,n", [LAYOUTS[1]], ids=_ids([LAYOUTS[1]]))
def test_malformed_buffers_rejected_before_launch(pkg, src, w, h, n):
    """inverse_host_sparse validates the header and the table on the host: a malformed buffer gives BADFORMAT, launches
    nothing, and leaves the codec working.  Only buffers the host check must refuse are used here."""
    desc = pkg.FrameDesc(w, h, getattr(pkg, "PIXEL_" + src))
    with pkg.Context(0) as ctx, pkg.Codec(ctx, desc, 2) as codec:
        s = Slots(pkg, ctx, codec, src)
        rng = np.random.default_rng(3)
        r = sr.region(s.nwords, sr.BLOCK_KINDS, rng)
        good, bad = _mutations(sr.compact(s.nwords, r), s.nwords)
        for name, buf in bad:
            with pytest.raises(sr.FormatError):
                sr.expand(s.nwords, buf)                # the reference refuses it too
            for batch in ([buf], [good, buf]):
                before = s.launches()
                with pytest.raises(pkg.CfbError) as e:
                    codec.inverse_host_sparse(batch, s.quant, s.out_format, [s.out] * len(batch))
                assert e.value.code == BADFORMAT, name
                assert s.launches() == before, name
        s.load([~r])
        s.unpack([good])
        _same_words(s.read(1)[0], r, "unpack after the rejections")
