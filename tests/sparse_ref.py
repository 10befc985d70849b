"""numpy restatement of the 'CFS2' sparse transfer format of the coded region, and a generator of adversarial coded regions.

Written from the format description at the top of cineform-sdk_b200/csrc/cfb_sparse.cu, not from the C code, so that the
host packer (cfb_sparse_compact) and the GPU kernels (k_sparse_pack / k_sparse_unpack) are checked against an independent
statement of the format:

  header   32 B : u32 'CFS2', u32 nwords, u32 total bytes, u32 nblocks, 4 x u32 0
  table    one 16-B entry per block of 8192 words: {u32 chunk offset, u32 groups, u32 values, u32 escapes}
  chunks   from align16(32 + 16 nblocks), one per block, 0 bytes for an all-zero block, otherwise
             l1     32 B   bit g <=> group g (32 consecutive words) holds a non-zero word
             masks  4 B per non-empty group: bit i <=> word i of the group is non-zero
             bytes  1 B per non-zero word in raster order: the value if -127 <= v <= 127, else -128 (escape)
             wide   2 B per escape, in order: the int16 value
           bytes and wide each zero-padded to 4 B, the chunk zero-padded to 16 B.

The coded region is packed flat: the words between a band's width and its pitch are words like any other.
"""
import numpy as np

MAGIC = 0x32534643          # 'CFS2'
HEADER_BYTES = 32
ENTRY_BYTES = 16
BLOCK_WORDS = 8192
GROUP_WORDS = 32
BLOCK_GROUPS = BLOCK_WORDS // GROUP_WORDS
L1_BYTES = BLOCK_GROUPS // 8
MAX_CHUNK = L1_BYTES + 4 * BLOCK_GROUPS + BLOCK_WORDS + 2 * BLOCK_WORDS     # every word non-zero and escaped: 25 632


def _align(n, a):
    return (n + a - 1) // a * a


def nblocks(nwords):
    return -(-nwords // BLOCK_WORDS)


def chunks_offset(nb):
    return _align(HEADER_BYTES + ENTRY_BYTES * nb, 16)


def chunk_bytes(groups, values, escapes):
    if groups == 0:
        return 0
    return _align(L1_BYTES + 4 * groups + _align(values, 4) + _align(2 * escapes, 4), 16)


def max_bytes(nwords):
    """Largest buffer a region of `nwords` words can need: every block a maximal chunk."""
    nb = nblocks(nwords)
    return chunks_offset(nb) + nb * MAX_CHUNK


def _padded(b, a):
    return b + bytes(_align(len(b), a) - len(b))


def _block_chunk(words):
    """One block of 8192 int16 words (zero beyond the region) -> (chunk bytes, groups, values, escapes)."""
    nz = words != 0
    grp = nz.reshape(BLOCK_GROUPS, GROUP_WORDS)
    occupied = grp.any(axis=1)
    G = int(occupied.sum())
    if G == 0:
        return b"", 0, 0, 0
    l1 = np.packbits(occupied, bitorder="little")                                       # bit g of byte g / 8
    masks = np.packbits(grp[occupied], axis=1, bitorder="little")                       # (G, 4) = little-endian u32
    vals = words[nz]                                                                    # raster order
    esc = (vals < -127) | (vals > 127)
    vbytes = np.where(esc, -128, vals).astype(np.int8)
    wide = vals[esc].astype("<i2")
    chunk = l1.tobytes() + masks.tobytes() + _padded(vbytes.tobytes(), 4) + _padded(wide.tobytes(), 4)
    chunk = _padded(chunk, 16)
    assert len(chunk) == chunk_bytes(G, vals.size, wide.size)
    return chunk, G, int(vals.size), int(wide.size)


def _as_words(nwords, dense):
    dense = np.ascontiguousarray(dense)
    words = dense.view(np.int16) if dense.dtype != np.int16 else dense
    words = words.ravel()
    assert words.size == nwords, (words.size, nwords)
    return words


def compact(nwords, dense):
    """Dense coded region (int16 words, or its bytes) -> the 'CFS2' buffer, as bytes."""
    words = _as_words(nwords, dense)
    nb = nblocks(nwords)
    full = np.zeros(nb * BLOCK_WORDS, np.int16)
    full[:nwords] = words
    blocks = full.reshape(nb, BLOCK_WORDS)
    occupied = blocks.any(axis=1)
    table = np.zeros((nb, 4), "<u4")
    sizes = np.zeros(nb, np.int64)
    chunks = []
    for b in np.flatnonzero(occupied):
        chunk, G, V, E = _block_chunk(blocks[b])
        table[b, 1:] = (G, V, E)
        sizes[b] = len(chunk)
        chunks.append(chunk)
    # the chunks follow each other in block order; an empty block's 0-byte chunk sits where the next chunk starts
    ends = chunks_offset(nb) + np.cumsum(sizes)
    table[:, 0] = ends - sizes
    total = chunks_offset(nb) + int(sizes.sum())
    header = np.array([MAGIC, nwords, total, nb, 0, 0, 0, 0], "<u4")
    head = _padded(header.tobytes() + table.tobytes(), 16)
    return head + b"".join(chunks)


class FormatError(ValueError):
    pass


def _check(cond, msg):
    if not cond:
        raise FormatError(msg)


def expand(nwords, sparse):
    """'CFS2' buffer (bytes or uint8 array) -> the dense coded region (int16 words).  Raises FormatError for anything
    the format does not allow, including non-canonical encodings (a plain byte of 0, an escape that fits a byte, non-zero
    padding), so that a packer which emits them does not pass as equal."""
    buf = np.frombuffer(bytes(sparse), np.uint8)
    _check(buf.size >= HEADER_BYTES, "shorter than the header")
    h = buf[:HEADER_BYTES].view("<u4")
    nb = nblocks(nwords)
    _check(h[0] == MAGIC, "magic")
    _check(h[1] == nwords and h[3] == nb, "nwords / nblocks")
    _check(not h[4:].any(), "reserved header words")
    total = int(h[2])
    lo = chunks_offset(nb)
    _check(lo <= total <= min(buf.size, max_bytes(nwords)) and total % 16 == 0, "total bytes")
    _check(not buf[HEADER_BYTES + ENTRY_BYTES * nb:lo].any(), "padding after the table")
    table = buf[HEADER_BYTES:HEADER_BYTES + ENTRY_BYTES * nb].view("<u4").reshape(nb, 4).astype(np.int64)
    out = np.zeros(nb * BLOCK_WORDS, np.int16)
    for b in range(nb):
        off, G, V, E = (int(x) for x in table[b])
        _check(G <= BLOCK_GROUPS and V <= BLOCK_WORDS and E <= V and (G == 0) == (V == 0), f"block {b}: counts")
        if G == 0:
            _check(E == 0, f"block {b}: escapes in an empty block")
            continue
        cb = chunk_bytes(G, V, E)
        _check(off % 16 == 0 and off >= lo and off + cb <= total, f"block {b}: chunk outside the buffer")
        c = buf[off:off + cb]
        l1 = np.unpackbits(c[:L1_BYTES], bitorder="little").astype(bool)
        _check(int(l1.sum()) == G, f"block {b}: l1 bits != groups")
        mo = L1_BYTES
        bits = np.unpackbits(c[mo:mo + 4 * G].reshape(G, 4), axis=1, bitorder="little").astype(bool)     # (G, 32)
        _check(bits.any(axis=1).all(), f"block {b}: an empty group mask")
        _check(int(bits.sum()) == V, f"block {b}: mask bits != values")
        pos = (np.flatnonzero(l1)[:, None] * GROUP_WORDS + np.arange(GROUP_WORDS))[bits]       # raster order
        bo = mo + 4 * G
        vb = c[bo:bo + V].view(np.int8).astype(np.int16)
        esc = vb == -128
        _check(int(esc.sum()) == E, f"block {b}: escape bytes != escapes")
        _check((vb != 0).all(), f"block {b}: a plain byte of 0")
        wo = bo + _align(V, 4)
        wide = c[wo:wo + 2 * E].view("<i2")
        _check(((wide < -127) | (wide > 127)).all(), f"block {b}: an escape that fits a byte")
        _check(not c[bo + V:wo].any() and not c[wo + 2 * E:].any(), f"block {b}: padding")
        vals = vb.copy()
        vals[esc] = wide
        out[b * BLOCK_WORDS + pos] = vals
    _check(not out[nwords:].any(), "values past the region")
    return out[:nwords].copy()


# ---------------------------------------------------------------------------------------------------------------------
# Adversarial coded regions, built block by block from a catalogue.

ESCAPE_CYCLE = np.array([-32768, 32767, -128, 128, -129], np.int16)     # every word escaped: a maximal chunk
BOUNDARY = np.array([-128, -127, 127, 128], np.int16)                   # -128 is the escape byte itself: it must be escaped
SINGLE_VALUES = np.array([1, -1, 127, -127, 128, -128, 32767, -32768], np.int16)
# first / last word of a group (32), a warp piece (256), a thread piece (2048) and the block
SINGLE_POSITIONS = (0, 31, 32, 255, 256, 2047, 2048, 8191)
BLOCK_KINDS = ("empty",) + tuple(f"single{p}" for p in SINGLE_POSITIONS) + ("per_group", "plain", "escaped", "boundary", "random")


def _values(rng, n, escape_share):
    """n non-zero int16 values, a share of them outside [-127, 127]."""
    sign = rng.choice(np.array([-1, 1], np.int32), n)
    plain = rng.integers(1, 128, n) * sign
    esc = rng.integers(128, 32769, n) * sign
    esc[esc > 32767] = 32767
    return np.where(rng.random(n) < escape_share, esc, plain).astype(np.int16)


def block(kind, rng):
    """One block of 8192 words of the given kind."""
    w = np.zeros(BLOCK_WORDS, np.int16)
    if kind == "empty":
        pass
    elif kind.startswith("single"):
        w[int(kind[6:])] = rng.choice(SINGLE_VALUES)
    elif kind == "per_group":             # one value per group, at a random word of it
        pos = np.arange(BLOCK_GROUPS) * GROUP_WORDS + rng.integers(0, GROUP_WORDS, BLOCK_GROUPS)
        w[pos] = _values(rng, BLOCK_GROUPS, 0.5)
    elif kind == "plain":                 # every word non-zero, none escaped
        w[:] = _values(rng, BLOCK_WORDS, 0.0)
    elif kind == "escaped":
        w[:] = np.roll(np.resize(ESCAPE_CYCLE, BLOCK_WORDS), int(rng.integers(0, ESCAPE_CYCLE.size)))
    elif kind == "boundary":
        nz = rng.random(BLOCK_WORDS) < 0.5
        w[nz] = rng.choice(BOUNDARY, int(nz.sum()))
    elif kind == "random":
        density = 10.0 ** rng.uniform(-3.0, 0.0)
        nz = rng.random(BLOCK_WORDS) < density
        w[nz] = _values(rng, int(nz.sum()), rng.random())
    else:
        raise ValueError(kind)
    return w


def region(nwords, kinds, rng):
    """Block b holds block(kinds[b % len(kinds)]); the region is cut at `nwords` (a partial last block)."""
    nb = nblocks(nwords)
    out = np.empty(nb * BLOCK_WORDS, np.int16)
    for b in range(nb):
        out[b * BLOCK_WORDS:(b + 1) * BLOCK_WORDS] = block(kinds[b % len(kinds)], rng)
    return out[:nwords].copy()


def empty_runs(nwords, rng, runs=(0, 1, 31, 32, 33, 100, 300)):
    """Runs of empty blocks (0-byte chunks), each ending in a dense block; the look-back of the dense block has to sum
    up to hundreds of aggregate-only predecessors.  The last block is dense too."""
    nb = nblocks(nwords)
    kinds = []
    i = 0
    while len(kinds) < nb - 1:
        kinds += ["empty"] * runs[i % len(runs)] + ["escaped" if i % 2 else "plain"]
        i += 1
    kinds = kinds[:nb - 1] + ["escaped"]
    return region(nwords, kinds, rng)


def catalogue(nwords, rng):
    """[(name, region)]: every block kind at least once, in block positions that vary between regions, plus the
    whole-region patterns."""
    nb = nblocks(nwords)
    k = len(BLOCK_KINDS)
    out = [("empty", np.zeros(nwords, np.int16)),
           ("escaped", region(nwords, ["escaped"], rng)),
           ("plain", region(nwords, ["plain"], rng))]
    # rotations of the catalogue: with nb blocks, ceil(k / nb) of them put every kind in some block, and at least two
    # put different kinds in the (possibly partial) last block
    for r in range(max(2, -(-k // nb))):
        out.append((f"blocks{r}", region(nwords, BLOCK_KINDS[r * nb % k:] + BLOCK_KINDS[:r * nb % k], rng)))
    last = np.zeros(nwords, np.int16)
    last[-1] = -128
    out.append(("last_word", last))
    last_group = np.zeros(nwords, np.int16)
    last_group[-GROUP_WORDS] = 32767
    out.append(("last_group_first_word", last_group))
    out.append(("empty_runs", empty_runs(nwords, rng)))
    out.append(("random", region(nwords, ["random"], rng)))
    return out
