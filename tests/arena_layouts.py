"""Re-lay the blocks of any fixture in a new blob: other fillers between blocks, other alignments, other orders, shortened blocks and
offsets past 2^31 and 2^32.

Every result of the engine must depend only on the bytes blob[offsets[i] .. offsets[i] + lengths[i]) of the blocks it reads (DESIGN.md
§2). The fixtures all put zeros (or nothing) between blocks; the layouts here put there whatever an over-reading decoder would like to
see least: 0xff, random bytes, a copy of the block in front of the gap (`echo`) or the next block (`next`).

    lay_out(cids, offsets, lengths, blob, filler="echo", order="shuffled") → Layout (cids, offsets, lengths, blob, n_blocks)

The arrays keep their order (block i is still block i); only where the bytes sit changes. `Layout.over(ts)` gives a tipset-like view
over the new arrays (api.BlockStore.from_tipset, oracle.Store.from_tipset and A.make_tipset_desc accept it)."""
import hashlib

import numpy as np

from tests.util import EditedTipset

FILLERS = ("zero", "ff", "random", "echo", "next")
B2B_PREFIX = bytes([0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20])
B2B_RAW_PREFIX = bytes([0x01, 0x55, 0xa0, 0xe4, 0x02, 0x20])
B2S_PREFIX = bytes([0x01, 0x71, 0xe0, 0xe4, 0x02, 0x20])   # Blake2s-256: a class the CID check skips
FAR_SIZE = (1 << 32) + (64 << 20)


class Layout:
    def __init__(self, cids, offsets, lengths, blob):
        self.cids = np.ascontiguousarray(cids, dtype=np.uint8)
        self.offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        self.lengths = np.ascontiguousarray(lengths, dtype=np.uint32)
        self.blob = blob
        self.n_blocks = len(self.lengths)

    def block(self, i):
        o = int(self.offsets[i])
        return bytes(self.blob[o:o + int(self.lengths[i])])

    def arrays(self):
        return dict(cids=self.cids, offsets=self.offsets, lengths=self.lengths, blob=self.blob, n_blocks=self.n_blocks)

    def over(self, ts):
        return EditedTipset(ts, **self.arrays())


def blocks_of(src):
    """The block bytes of a fixture (anything with cids / offsets / lengths / blob)."""
    blob = np.asarray(src.blob, dtype=np.uint8)
    return [bytes(blob[int(o):int(o) + int(n)]) for o, n in zip(src.offsets, src.lengths)]


def _fill(kind, n, prev, rng):
    if n <= 0:
        return b""
    if kind == "zero":
        return bytes(n)
    if kind == "ff":
        return b"\xff" * n
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind == "echo":   # the block in front again (and again), so what is read past it looks like its own CBOR
        src = prev or b"\0"
        return (src * (n // len(src) + 1))[:n]
    raise ValueError(kind)


def lay_out(cids, offsets, lengths, blob, filler="zero", order="index", seed=0, residues=False, tail=64):
    """New offsets and blob for the same blocks. filler: one of FILLERS (`next`: no gaps at all). order: "index" (monotonic offsets)
    or "shuffled". residues: the k-th placed block starts at an offset ≡ k (mod 16), so every residue 0–15 occurs across the store.
    tail: filler bytes after the last placed block (0: the last block ends exactly at blob_size; only the arena's pad follows it)."""
    src = Layout(cids, offsets, lengths, blob)
    blocks = blocks_of(src)
    rng = np.random.default_rng(seed)
    n = len(blocks)
    perm = np.arange(n) if order == "index" else rng.permutation(n)
    parts, offs, pos, prev = [], np.zeros(n, dtype=np.uint64), 0, b""
    for k, i in enumerate(perm):
        b = blocks[int(i)]
        if filler == "next":
            gap = (k - pos) % 16 if residues else 0
            g = _fill("echo", gap, prev, rng)
        else:
            gap = len(prev) if filler == "echo" else int(rng.integers(1, 48))
            if residues:
                gap += (k - (pos + gap)) % 16
            g = _fill(filler, gap, prev, rng)
        parts.append(g)
        pos += len(g)
        offs[int(i)] = pos
        parts.append(b)
        pos += len(b)
        prev = b
    if tail:
        parts.append(_fill("echo" if filler == "next" else filler, tail, prev, rng))
    return Layout(src.cids, offs, src.lengths, np.frombuffer(b"".join(parts), dtype=np.uint8))


def shortened(layout, i, k):
    """Block i's length becomes k < len; its bytes stay where they are, so the arena continues with the block's own removed suffix.
    The CID is unchanged: a store of these arrays is created without verify_cids."""
    assert 0 <= k < int(layout.lengths[i])
    lengths = layout.lengths.copy()
    lengths[i] = k
    return Layout(layout.cids, layout.offsets, lengths, layout.blob)


SHORTEN = (1, 2, 8, 16, 24, 25, 43, 44)   # k = len − d; plus ⌊len/2⌋, 1 and 0


def shorten_lengths(n):
    ks = {n - d for d in SHORTEN if n - d >= 0} | {n // 2, 1, 0}
    return sorted(k for k in ks if 0 <= k < n)


def far(cids, offsets, lengths, blob, low, order="index", seed=0, straddle32=False):
    """A blob of 2^32 + 64 MiB (np.zeros: untouched pages cost nothing until the copy). The arrays are reordered to low + the rest (the
    engine does not depend on block order). Block low[0] straddles 2^31; low[1] ends exactly at 2^32 and low[2] starts exactly there —
    or, straddle32=True, low[1] straddles 2^32 — and every other block lies above 2^32, echo filled: placed in array order (monotonic
    offsets) or shuffled. Between 2^31 and 2^32 and below 2^31 the blob is zero: gaps of ≈ 2 GiB."""
    src = Layout(cids, offsets, lengths, blob)
    blocks = blocks_of(src)
    low = list(low)
    idx = low + [i for i in range(len(blocks)) if i not in low]
    blocks = [blocks[i] for i in idx]
    n = len(blocks)
    big = np.zeros(FAR_SIZE, dtype=np.uint8)
    offs = np.zeros(n, dtype=np.uint64)

    def put(k, at):
        b = blocks[k]
        big[at:at + len(b)] = np.frombuffer(b, dtype=np.uint8)
        offs[k] = at

    put(0, (1 << 31) - len(blocks[0]) // 2)
    if straddle32:
        put(1, (1 << 32) - len(blocks[1]) // 2)
        pos, first = (1 << 32) + len(blocks[1]), 2
    else:
        put(1, (1 << 32) - len(blocks[1]))
        put(2, 1 << 32)
        pos, first = (1 << 32) + len(blocks[2]), 3
    rest = list(range(first, n))
    if order != "index":
        rest = [rest[j] for j in np.random.default_rng(seed).permutation(len(rest))]
    prev = b""
    for k in rest:
        g = _fill("echo", len(prev) % 61 + 1, prev, None)
        big[pos:pos + len(g)] = np.frombuffer(g, dtype=np.uint8)
        pos += len(g)
        put(k, pos)
        pos += len(blocks[k])
        prev = blocks[k]
    assert pos < FAR_SIZE
    return Layout(src.cids[idx], offs, src.lengths[idx], big)


def chunked(cids, offsets, lengths, blob, chunk=64 << 20):
    """Blocks in index order over more than 2 chunks (the chunked CID check of ipcfp_store_create: a chunk is cut at block i when
    end_i − byte0 ≥ chunk, the next one starts at offsets[i + 1]), with two zero-length blocks and one block under a Blake2s-256 CID
    added. Chunk 0 = blocks [0, 129): block 128 ends exactly at byte0 + chunk (129 ≡ 1 mod 128: the last block of chunk 0 is the first
    of a second 128-thread CTA). Chunk 1 starts with a zero-length block, and is cut at a block straddling its byte0 + chunk. The last
    block is zero-length at offset == blob_size. → (Layout, info) with info = dict(first_of_chunk1, straddle, last, b2s)."""
    src = Layout(cids, offsets, lengths, blob)
    blocks = blocks_of(src)
    cid_list = [bytes(c) for c in src.cids]
    assert len(blocks) > 140, "needs more than 140 blocks (config 2 has 12 873)"
    nz = [i for i in range(len(blocks)) if blocks[i]]
    e1 = B2B_RAW_PREFIX + hashlib.blake2b(b"", digest_size=32).digest()
    e2 = B2B_PREFIX + hashlib.blake2b(b"", digest_size=32).digest()
    b2s_data = blocks[nz[-1]]
    b2s = B2S_PREFIX + hashlib.blake2s(b2s_data, digest_size=32).digest()
    order = list(range(129)) + ["z1"] + list(range(129, len(blocks))) + ["b2s", "z2"]
    out_cids, out_offs, out_lens, parts = [], [], [], []
    pos = 0

    def place(cid, data, at):
        nonlocal pos
        assert at >= pos
        parts.append(bytes(at - pos))
        parts.append(data)
        out_cids.append(cid)
        out_offs.append(at)
        out_lens.append(len(data))
        pos = at + len(data)

    info = {}
    straddle_at = None
    straddle = next(i for i in range(139, len(blocks)) if len(blocks[i]) > 1)
    for k, i in enumerate(order):
        if i == "z1":
            byte0 = chunk + 4096
            place(e1, b"", byte0)
            info["first_of_chunk1"] = k + 1
            straddle_at = byte0 + chunk
            continue
        if i == "b2s":
            place(b2s, b2s_data, pos + 32)
            info["b2s"] = k
            continue
        if i == "z2":
            size = pos + 4096
            parts.append(bytes(size - pos))
            out_cids.append(e2)
            out_offs.append(size)
            out_lens.append(0)
            pos = size
            continue
        data = blocks[i]
        if i == 128:
            at = chunk - len(data)                       # ends exactly at byte0 + chunk
        elif i == straddle:
            at = straddle_at - len(data) // 2            # straddles byte0 + chunk of chunk 1: chunk 1 is cut here
            info["straddle"] = k
        else:
            at = pos + (16 - pos % 16) % 16
        place(cid_list[i], data, at)
    info["last"] = max(j for j in range(len(out_lens)) if out_lens[j] > 0 and out_cids[j][:6] != B2S_PREFIX)
    lay = Layout(np.frombuffer(b"".join(out_cids), dtype=np.uint8).reshape(-1, 38), np.array(out_offs, dtype=np.uint64),
                 np.array(out_lens, dtype=np.uint32), np.frombuffer(b"".join(parts), dtype=np.uint8))
    return lay, info


def first_bad_b2b(layout):
    """Smallest i whose block does not hash (Blake2b-256) to its CID's digest, among the Blake2b-256 CIDs; None if all do."""
    for i in range(layout.n_blocks):
        c = bytes(layout.cids[i])
        if c[2:4] == b"\xa0\xe4" and hashlib.blake2b(layout.block(i), digest_size=32).digest() != c[6:]:
            return i
    return None
