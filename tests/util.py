"""Helpers shared by the parity tests."""
import re

import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A


def spec_of(ts):
    return A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter)


def assert_event_results_equal(got, exp, check_witness_bytes=True):
    assert got.matching.tolist() == exp.matching.tolist()
    assert got.n_exec == exp.n_exec
    assert [p.key() for p in got.proofs] == [p.key() for p in exp.proofs]
    assert got.witness.n_blocks == exp.witness.n_blocks
    assert np.array_equal(got.witness.cids, exp.witness.cids)
    if check_witness_bytes:
        assert np.array_equal(got.witness.lengths, exp.witness.lengths)
        assert got.witness.blocks() == exp.witness.blocks()
    assert np.array_equal(got.data_blob, exp.data_blob)


def assert_witness_equal(a, b):
    assert np.array_equal(a.cids, b.cids)
    assert np.array_equal(a.lengths, b.lengths)
    assert a.blocks() == b.blocks()


# Tipsets of the varied event-shape mode of the synthetic builder (event_shapes = 1), used as extra inputs next to the BASELINE
# configs: emitters with 1- to 8-byte heads, 0-4 topics, data up to 955 bytes, odd codecs and flags, duplicate and unknown keys,
# near misses, 0..events_per_receipt events per receipt (bit width 5: single-node roots, many over 4 KB, and roots with links).
SHAPES = {
    "shapes": dict(seed=41, n_receipts=600, events_per_receipt=40, match_ppm=300000),
    "shapes-nofilter": dict(seed=42, n_receipts=600, events_per_receipt=12, match_ppm=300000, has_actor_filter=0, bw3_permille=300,
                            null_root_permille=50),
}


def synth_tipset(synth_mod, cfg):
    """The BASELINE config `cfg` (an int) or the varied-shape tipset SHAPES[cfg]."""
    if cfg in SHAPES:
        return synth_mod.Tipset(synth_mod.default_params(event_shapes=1, **SHAPES[cfg]))
    return synth_mod.Tipset(synth_mod.config_params(cfg))


class ShuffledTipset:
    """Same tipset with the flat block arrays permuted (the engine must not depend on block order).
    misalign: blocks start 0-6 bytes after the previous one. roots_mod128: the k-th events-root block starts at an offset ≡ k
    (mod 128) and an events root is the last block of the blob (the other blocks 16-byte aligned)."""

    def __init__(self, ts, seed=7, misalign=False, roots_mod128=False):
        rng = np.random.default_rng(seed)
        perm = rng.permutation(ts.n_blocks)
        roots = set()
        if roots_mod128:
            roots = {bytes(ts.events_roots[i]) for i in range(int(ts.n_receipts)) if ts.has_events_root[i]}
            last = max(k for k, i in enumerate(perm) if bytes(ts.cids[i]) in roots)
            perm = np.concatenate([perm[:last], perm[last + 1:], perm[last:last + 1]])
        self._ts = ts
        lens = ts.lengths[perm]
        offs = np.zeros(ts.n_blocks, dtype=np.uint64)
        pos = 0
        chunks = []
        kroot = 0
        for k, i in enumerate(perm):
            if roots_mod128 and bytes(ts.cids[i]) in roots:
                pad = (kroot - pos) % 128
                kroot += 1
            else:
                pad = int(rng.integers(0, 7)) if misalign else (16 - pos % 16) % 16
            chunks.append(bytes(pad))
            pos += pad
            offs[k] = pos
            b = ts.block(int(i))
            chunks.append(b)
            pos += len(b)
        self.blob = np.frombuffer(b"".join(chunks) + bytes(16), dtype=np.uint8)
        self.cids = ts.cids[perm].copy()
        self.offsets = offs
        self.lengths = lens.copy()
        self.n_blocks = ts.n_blocks

    def __getattr__(self, name):
        return getattr(self._ts, name)


class EditedTipset:
    """Tipset view with replaced arrays (for fault injection)."""

    def __init__(self, ts, **over):
        self._ts = ts
        for k in ("cids", "offsets", "lengths", "blob", "n_blocks"):
            setattr(self, k, over.get(k, getattr(ts, k)))
        for k, v in over.items():
            setattr(self, k, v)

    def __getattr__(self, name):
        return getattr(self._ts, name)


def dict_of(ts):
    """cid -> bytes of any tipset-like object, from its flat arrays (first occurrence wins)."""
    d = {}
    for i in range(int(ts.n_blocks)):
        o = int(ts.offsets[i])
        d.setdefault(bytes(ts.cids[i]), bytes(ts.blob[o:o + int(ts.lengths[i])]))
    return d


# ------------------------------------------------------------------ adversarial CID sets
# A tipset rewritten through a bijection on CIDs keeps every block length, so offsets stay valid; the digests no longer hash to their
# blocks, so stores of such tipsets are created without IPCFP_STORE_VERIFY_CIDS.
LINK_HEAD = b"\xd8\x2a\x58\x27\x00"                        # tag 42, bytes(39), multibase 0x00
CID_LINK = re.compile(re.escape(LINK_HEAD) + b"(.{38})", re.S)
FILECOIN_PREFIX = bytes.fromhex("0171a0e40220")            # CIDv1, dag-cbor, blake2b-256, 32 bytes
# Eight valid CIDv1 prefixes (1-byte codec, 3-byte multihash code varint, size 0x20), listed in `Cid` order. Their raw byte order is
# different: the code is a little-endian varint, so 0x407f (ff 80 01) sorts after 0xb220 (a0 e4 02) bytewise.
MIXED_PREFIXES = [bytes.fromhex(h) for h in (
    "0155ffff0120",   # raw,      0x7fff
    "0155a0e40220",   # raw,      0xb220
    "017081800220",   # dag-pb,   0x8001
    "0171ff800120",   # dag-cbor, 0x407f
    "017180800220",   # dag-cbor, 0x8000
    "017192e40220",   # dag-cbor, 0xb212
    "0171a0e40220",   # dag-cbor, 0xb220
    "0171ffff0320",   # dag-cbor, 0xffff
)]
DESC_CID_FIELDS = ("child_cid", "receipts_root", "parent_state_root", "storage_root")
DESC_CID_LISTS = ("parent_cids", "parent_txmeta_cids")


def cid_universe(ts):
    """Every CID a tipset names: the flat cids, every tag-42 link target in the blob (message CIDs included), the descriptor fields."""
    u = {bytes(c) for c in ts.cids}
    u.update(CID_LINK.findall(bytes(ts.blob)))
    for f in DESC_CID_FIELDS:
        u.add(bytes(getattr(ts, f)))
    for f in DESC_CID_LISTS:
        u.update(bytes(c) for c in getattr(ts, f))
    u.update(bytes(ts.events_roots[i]) for i in range(int(ts.n_receipts)) if ts.has_events_root[i])
    return sorted(u)


def clustered_digests(n, rng):
    """n distinct digests in groups that share bytes 0-7 and 16-23 (one hash slot, fingerprint and radix key per group); bytes 8-15
    and 24-31 tell the members apart. Between neighbours in sorted order the first differing byte takes every position 4..31: one
    group per position 8-15 / 24-31 whose members differ only there (31: only the last byte), and for 4-7 / 16-23 pairs of groups
    whose shared bytes first differ there. Then a 512 and a 300 group (runs longer than 256), then groups of 2..64."""
    out = []

    def group(t, size, at):
        for k in range(size):
            d = bytearray(t)
            if size > 256:
                d[at:at + 2] = k.to_bytes(2, "big")
            else:
                d[at] = k
            out.append(bytes(d))

    def template():
        return bytearray(rng.bytes(32))

    for p in list(range(8, 16)) + list(range(24, 32)):
        group(template(), 6, p)
    for p in list(range(4, 8)) + list(range(16, 24)):
        t = template()
        t[p] &= 0x7F
        t2 = bytearray(t)
        t2[p] += 1
        group(t, 5, 8)
        group(t2, 5, 8)
    group(template(), 512, 8)
    group(template(), 300, 24)
    places = list(range(8, 16)) + list(range(24, 32))
    while len(out) < n:
        group(template(), int(rng.integers(2, 65)), places[int(rng.integers(0, len(places)))])
    out = out[:n]
    assert len(set(out)) == len(out)
    return out


def first_difference(a, b):
    return next(k for k in range(len(a)) if a[k] != b[k])


class CidMap:
    """A bijection on CIDs (identity outside `m`) and its image of blocks, witnesses and results."""

    def __init__(self, m=None):
        self.m = dict(m or {})

    def cid(self, c):
        c = bytes(c)
        return self.m.get(c, c)

    def block(self, b):
        return CID_LINK.sub(lambda mo: LINK_HEAD + self.cid(mo.group(1)), bytes(b))

    def witness(self, w):
        """(cids, blocks) of a WitnessPy's image, re-sorted in `Cid` order."""
        from oracle import pyoracle as P
        pairs = sorted(((self.cid(w.cids[i]), self.block(w.block(i))) for i in range(w.n_blocks)), key=lambda cb: P.cid_sort_key(cb[0]))
        return [c for c, _ in pairs], [b for _, b in pairs]

    def proof_keys(self, proofs):
        return [(p.exec_index, p.event_index, p.emitter, tuple(p.topics), p.data, self.cid(p.message_cid)) for p in proofs]

    def storage_proofs(self, proofs):
        out = []
        for p in proofs:
            d = dict(vars(p))
            d["actor_state_cid"], d["storage_root"] = self.cid(p.actor_state_cid), self.cid(p.storage_root)
            out.append(d)
        return out

    def spec_witness(self, res):
        """per-spec witness index lists (ascending) of a StorageResultPy, renumbered into its image's witness order."""
        cids, _ = self.witness(res.witness)
        where = {c: i for i, c in enumerate(cids)}
        return [sorted(where[self.cid(res.witness.cids[i])] for i in lst) for lst in res.spec_witness]


def assert_event_image(got, exp, cm, check_witness_bytes=True):
    """`got` (a result on the rewritten tipset) equals the image under `cm` of `exp` (a result on the original tipset)."""
    assert got.matching.tolist() == exp.matching.tolist()
    assert got.n_exec == exp.n_exec
    assert [p.key() for p in got.proofs] == cm.proof_keys(exp.proofs)
    cids, blocks = cm.witness(exp.witness)
    assert [bytes(c) for c in got.witness.cids] == cids
    assert got.witness.lengths.tolist() == [len(b) for b in blocks]
    if check_witness_bytes:
        assert got.witness.blocks() == blocks


def cid_map(ts, family, seed=0):
    """The bijection of one adversarial family over cid_universe(ts):
    A  clustered digests (clustered_digests) under the Filecoin prefix;
    B  random digests under the eight MIXED_PREFIXES; the first flat CID gets the highest-ranked one (class 0 is not rank 0), and
       some pairs of distinct CIDs (store blocks with store blocks, the rest, message CIDs mostly, with the rest) share one digest
       under two prefixes;
    C  A's digests with B's prefixes and pairs."""
    rng = np.random.default_rng(seed)
    u = cid_universe(ts)
    order = [u[i] for i in rng.permutation(len(u))]
    n = len(u)
    digests = clustered_digests(n, rng) if family in ("A", "C") else [rng.bytes(32) for _ in range(n)]
    m = {}
    for k, c in enumerate(order):
        pre = FILECOIN_PREFIX if family == "A" else MIXED_PREFIXES[(k // 61) % len(MIXED_PREFIXES)]
        m[c] = pre + digests[k]
    if family in ("B", "C"):
        first = bytes(ts.cids[0])
        m[first] = MIXED_PREFIXES[-1] + m[first][6:]
        flat = {bytes(c) for c in ts.cids}
        for lst in ([c for c in order if c in flat and c != first], [c for c in order if c not in flat]):
            for j in range(0, len(lst) - 1, 7):
                a, b = lst[j], lst[j + 1]
                pa, pb = m[a][:6], m[b][:6]
                if pa == pb:
                    pb = MIXED_PREFIXES[(MIXED_PREFIXES.index(pa) + 1) % len(MIXED_PREFIXES)]
                m[b] = pb + m[a][6:]
    assert len(set(m.values())) == len(m)
    return CidMap(m)


def remap_tipset(ts, cm):
    """The tipset rewritten through `cm`: flat cids, every link in the blob, the descriptor's CIDs."""
    def arr(cs):
        return np.frombuffer(b"".join(cm.cid(c) for c in cs), dtype=np.uint8).reshape(-1, 38).copy()

    over = dict(cids=arr(ts.cids), blob=np.frombuffer(cm.block(ts.blob), dtype=np.uint8))
    for f in DESC_CID_FIELDS:
        over[f] = arr([getattr(ts, f)])[0]
    for f in DESC_CID_LISTS:
        over[f] = arr(getattr(ts, f))
    ev = np.array(ts.events_roots, copy=True)
    for i in range(int(ts.n_receipts)):
        if ts.has_events_root[i]:
            ev[i] = np.frombuffer(cm.cid(ts.events_roots[i]), dtype=np.uint8)
    over["events_roots"] = ev
    return EditedTipset(ts, **over)


def with_duplicates(ts, seed=0, n_before=40, n_after=40, n_repeat=1000):
    """Family D: the tipset with extra flat entries that repeat existing CIDs — identical bytes (a fresh copy in the blob) placed
    BEFORE the original, different bytes placed AFTER it, and the receipts root repeated n_repeat times after it with different
    bytes (racing the index build's atomicMin). The returned view's `first_offset` maps every CID to the blob offset of its first
    flat entry (the block a by-reference witness must name)."""
    rng = np.random.default_rng(seed)
    n = int(ts.n_blocks)
    first = {}
    for i in range(n):
        first.setdefault(bytes(ts.cids[i]), i)
    uniq = sorted(first.values())
    hot = first[bytes(ts.receipts_root)]
    pick = rng.permutation([i for i in uniq if i != hot])
    before, after = [hot] + pick[:n_before].tolist(), pick[n_before:n_before + n_after].tolist()
    blob = bytearray(bytes(ts.blob))

    def put(b):
        while len(blob) % 16:
            blob.append(0)
        o = len(blob)
        blob.extend(b)
        return o

    cids, offs, lens = [], [], []
    for i in before:
        cids.append(ts.cids[i]); offs.append(put(ts.block(i))); lens.append(int(ts.lengths[i]))
    cids += list(ts.cids); offs += [int(o) for o in ts.offsets]; lens += [int(x) for x in ts.lengths]
    for i in after:
        b = rng.bytes(int(rng.integers(1, 300)))
        cids.append(ts.cids[i]); offs.append(put(b)); lens.append(len(b))
    junk = put(rng.bytes(97))
    for _ in range(n_repeat):
        cids.append(ts.cids[hot]); offs.append(junk); lens.append(97)
    blob.extend(bytes(32))
    e = EditedTipset(ts, cids=np.array(cids, dtype=np.uint8).reshape(-1, 38), offsets=np.array(offs, dtype=np.uint64),
                     lengths=np.array(lens, dtype=np.uint32), blob=np.frombuffer(bytes(blob), dtype=np.uint8), n_blocks=len(lens))
    e.first_offset = {}
    for c, o in zip(cids, offs):
        e.first_offset.setdefault(bytes(c), o)
    return e


def adversarial_tipset(ts, family, seed=0):
    """(rewritten tipset, CidMap) of family A, B, C or D (D: the identity map plus duplicate flat entries)."""
    if family == "D":
        return with_duplicates(ts, seed), CidMap()
    cm = cid_map(ts, family, seed)
    return remap_tipset(ts, cm), cm


# ------------------------------------------------------------------ the store index's hash (csrc/common.cuh), restated
_M64 = (1 << 64) - 1


def mix64(x):
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & _M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & _M64
    x ^= x >> 33
    return x


def digest_hash(digest, cls):
    """digest_hash(Digest, class) of the device: words 0 and 2 (little-endian loads of bytes 0-7 and 16-23) and the class."""
    w0 = int.from_bytes(digest[0:8], "little")
    w2 = int.from_bytes(digest[16:24], "little")
    return mix64(w0 ^ ((w2 * 0x9E3779B97F4A7C15) & _M64) ^ cls)


def table_slots(n):
    """Slots of a store's hash table: the smallest power of two >= 2n, at least 64."""
    s = 64
    while s < 2 * n:
        s <<= 1
    return s
