"""Hand-built state trees for the storage-path tests (cbor2 + hashlib only; a helper module, not a fixture file).

Blocks are kept as a dict cid -> bytes (`Blocks`); `Blocks.flat()` gives the cids / offsets / lengths / blob arrays every store takes.
The layouts are the ones DESIGN.md §3 states:
  HAMT node      [bitfield: big-endian bytes, [pointer…]], pointer = link | bucket [[key: bytes, value]…], SHA-256 of the key,
                 `bw` bits per level MSB first, at most 256 bits in all (⌊256/bw⌋ levels);
  storage value  Vec<u8> = a CBOR array of u8;
  contract state A1 [params, [SmallMap…]], A2 [params, SmallMap], A3 SmallMap, B1 [root, bitwidth], B2 {root, bitwidth, …},
                 C a bare HAMT read at bit width 5;
  EVM state      6-tuple [bytecode, bytecode_hash, contract_state, transient, nonce, tombstone] or the 5-tuple without transient;
  ActorState     [code, state, sequence, balance, delegated|null];  StateRoot [version, actors, info];  actors HAMT at width 5.
`world_slots()` and `world_proofs(ts)` are the catalogues the GPU tests (tests/test_gpu_storage_tries.py) run and the CPU self-check
(tests/test_storage_trees.py) pins: every success case carries its ground truth, the value the builder put under the key."""
import functools
import hashlib
import random

import cbor2
import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A
from tests.util import EditedTipset

PREFIX = bytes.fromhex("0171a0e40220")      # CIDv1, dag-cbor, blake2b-256
LINK_HEAD = b"\xd8\x2a\x58\x27\x00"


def cid_of(block):
    return PREFIX + hashlib.blake2b(block, digest_size=32).digest()


# ------------------------------------------------------------------ CBOR items, hand encoded where the tests need exact bytes
def head(major, n):
    """Minimal CBOR head."""
    if n < 24:
        return bytes([major << 5 | n])
    for ai, size in ((24, 1), (25, 2), (26, 4), (27, 8)):
        if n < 1 << (8 * size):
            return bytes([major << 5 | ai]) + n.to_bytes(size, "big")
    raise ValueError(n)


def cbytes(b):
    return head(2, len(b)) + bytes(b)


def ctext(s):
    return head(3, len(s)) + s.encode()


def clink(cid):
    assert len(cid) == 38
    return LINK_HEAD + bytes(cid)


def u8vec(v):
    """serde Vec<u8>: a CBOR array of minimal uints."""
    return head(4, len(v)) + b"".join(head(0, x) for x in v)


def id_address(actor_id):
    """Address::new_id(actor_id).to_bytes(): protocol 0 + LEB128 (the actors HAMT key, up to 11 bytes)."""
    out = bytearray([0])
    while actor_id >= 0x80:
        out.append((actor_id & 0x7F) | 0x80)
        actor_id >>= 7
    out.append(actor_id)
    return bytes(out)


def left_pad_32(v):
    return bytes(v[-32:]) if len(v) >= 32 else bytes(32 - len(v)) + bytes(v)


def max_levels(bw):
    """Levels a HAMT of bit width bw can have: level k reads hash bits [k·bw, (k+1)·bw), which must stay ≤ 256."""
    return 256 // bw


def hash_index(key, level, bw):
    assert (level + 1) * bw <= 256
    h = int.from_bytes(hashlib.sha256(key).digest(), "big")
    return (h >> (256 - (level + 1) * bw)) & ((1 << bw) - 1)


class Blocks(dict):
    def put(self, block):
        c = cid_of(block)
        self[c] = bytes(block)
        return c

    def flat(self):
        """cids (n, 38) / offsets / lengths / blob, blocks 16-byte aligned in insertion order."""
        cids, offs, lens, parts, pos = [], [], [], [], 0
        for c, b in self.items():
            pad = (16 - pos % 16) % 16
            parts.append(bytes(pad))
            pos += pad
            cids.append(c)
            offs.append(pos)
            lens.append(len(b))
            parts.append(b)
            pos += len(b)
        parts.append(bytes(32))
        return (np.frombuffer(b"".join(cids), dtype=np.uint8).reshape(-1, 38).copy(), np.array(offs, dtype=np.uint64),
                np.array(lens, dtype=np.uint32), np.frombuffer(b"".join(parts), dtype=np.uint8).copy())


# ------------------------------------------------------------------ HAMT nodes
def hamt_node(pointers, bitfield_len=None):
    """pointers: {index: child CID (38 bytes) | bucket [(key, encoded value)…]}, emitted in index order. The bitfield is the minimal
    big-endian byte string of the set indices, or left-padded with zero bytes to `bitfield_len`."""
    bf = 0
    for i in pointers:
        bf |= 1 << i
    bfb = bf.to_bytes((bf.bit_length() + 7) // 8, "big")
    if bitfield_len is not None:
        bfb = bfb.rjust(bitfield_len, b"\0")
    out = [b"\x82", cbytes(bfb), head(4, len(pointers))]
    for i in sorted(pointers):
        p = pointers[i]
        if isinstance(p, bytes):
            out.append(clink(p))
        else:
            out.append(head(4, len(p)) + b"".join(b"\x82" + cbytes(k) + v for k, v in p))
    return b"".join(out)


def build_hamt(blocks, entries, bw, level=0, bitfield_len=None):
    """Canonical fvm_ipld_hamt trie of entries {key: encoded value} (as insertions build it): the keys that share a slot form a bucket
    (sorted by key) while they are at most 3, else a child node one level down. → root CID."""
    groups = {}
    for k in entries:
        groups.setdefault(hash_index(k, level, bw), []).append(k)
    ptrs = {}
    for i, ks in groups.items():
        if len(ks) <= 3:
            ptrs[i] = [(k, entries[k]) for k in sorted(ks)]
        else:
            ptrs[i] = build_hamt(blocks, {k: entries[k] for k in ks}, bw, level + 1, bitfield_len)
    return blocks.put(hamt_node(ptrs, bitfield_len))


def chain_siblings(key, bw, rng, max_bits=8, per_level=2):
    """Sibling entries for build_chain: at every level k with k·bw < max_bits, up to `per_level` random 32-byte keys that follow
    `key`'s path down to level k and leave it there (so they are reachable). → {level: [key…]}."""
    out = {}
    for level in range(max_levels(bw)):
        if level * bw >= max_bits:
            break
        ks = []
        while len(ks) < per_level:
            k = rng.randbytes(32)
            if all(hash_index(k, j, bw) == hash_index(key, j, bw) for j in range(level)) and hash_index(k, level, bw) != hash_index(key, level, bw):
                ks.append(k)
        out[level] = ks
    return out


def build_chain(blocks, key, value, bw, n_nodes, present=True, siblings=None):
    """n_nodes nodes along key's hash bits: node k holds one link at key's level-k index to node k+1. The last node holds the
    bucket [[key, value]] at key's index (present) or the same bucket one slot off (index ^ 1: the key is there but its bit is clear).
    Levels past the depth limit use index 0. siblings {level: [(key, encoded value)…]} add buckets beside the link. → root CID."""
    def idx(level):
        return hash_index(key, level, bw) if (level + 1) * bw <= 256 else 0

    siblings = siblings or {}
    last = n_nodes - 1
    c = None
    for level in range(last, -1, -1):
        ptrs = {}
        for sk, sv in siblings.get(level, []):
            ptrs.setdefault(hash_index(sk, level, bw), []).append((sk, sv))
        for b in ptrs.values():
            b.sort()
        if level == last:
            ptrs[idx(level) if present else idx(level) ^ 1] = [(key, value)]
        else:
            ptrs[idx(level)] = c
        c = blocks.put(hamt_node(ptrs))
    return c


# ------------------------------------------------------------------ contract-state wrappers and the rest of a state tree
def small_map(pairs, extra=()):
    """SmallMap { v: Vec<(ByteBuf, ByteBuf)> } as a CBOR map (unknown fields `extra` are ignored by the decoder)."""
    d = {"v": [[bytes(k), bytes(v)] for k, v in pairs]}
    for k, v in extra:
        d[k] = v
    return d


def wrap_a1(maps):
    return cbor2.dumps([b"params", maps])


def wrap_a2(m):
    return cbor2.dumps([b"params", m])


def wrap_a3(m):
    return cbor2.dumps(m)


def wrap_b1(root, bw):
    return b"\x82" + clink(root) + head(0, bw)


def wrap_b2(root, bw, fields=None):
    """B2 map. fields: [(name, encoded item)…] in order (duplicates allowed); default {root, bitwidth}."""
    if fields is None:
        fields = [("root", clink(root)), ("bitwidth", head(0, bw))]
    return head(5, len(fields)) + b"".join(ctext(k) + v for k, v in fields)


def evm_state(contract_state, six=True, nonce=1):
    bytecode = cid_of(b"bytecode")
    items = [clink(bytecode), cbytes(hashlib.sha256(b"bytecode").digest()), clink(contract_state)]
    if six:
        items.append(b"\xf6")                 # transient_data: None
    items += [head(0, nonce), b"\xf6"]        # nonce, tombstone: None
    return head(4, len(items)) + b"".join(items)


def actor_state(state_cid, sequence=0):
    code = cid_of(b"fil/16/evm")
    return b"\x85" + clink(code) + clink(state_cid) + head(0, sequence) + cbytes(b"\x01\x00") + b"\xf6"


def state_root(actors_root, version=5):
    return b"\x83" + head(0, version) + clink(actors_root) + clink(cid_of(b"state-info"))


def child_header(ts, new_state_root):
    """ts's child header with its parent_state_root replaced → (header bytes, header CID)."""
    i = next(i for i in range(int(ts.n_blocks)) if bytes(ts.cids[i]) == bytes(ts.child_cid))
    hdr = ts.block(i)
    old = clink(bytes(ts.parent_state_root))
    assert hdr.count(old) == 1
    hdr = hdr.replace(old, clink(new_state_root))
    return hdr, cid_of(hdr)


class Flat:
    """The flat arrays of a Blocks, with fault helpers: replace a block's bytes under the same CID (same length: stores of such arrays
    are created without verify_cids) or drop a block."""

    def __init__(self, blocks):
        self.blocks = blocks
        self.cids, self.offsets, self.lengths, self.blob = blocks.flat()
        self.n_blocks = len(self.lengths)
        self.index = {bytes(c): i for i, c in enumerate(self.cids)}

    def arrays(self):
        return dict(cids=self.cids, offsets=self.offsets, lengths=self.lengths, blob=self.blob, n_blocks=self.n_blocks)

    def replaced(self, cid, new):
        i = self.index[bytes(cid)]
        assert len(new) == int(self.lengths[i])
        blob = self.blob.copy()
        o = int(self.offsets[i])
        blob[o:o + len(new)] = np.frombuffer(new, dtype=np.uint8)
        return dict(self.arrays(), blob=blob)

    def dropped(self, cid):
        keep = [i for i in range(self.n_blocks) if i != self.index[bytes(cid)]]
        return dict(self.arrays(), cids=self.cids[keep], offsets=self.offsets[keep], lengths=self.lengths[keep], n_blocks=len(keep))


def tipset(ts, arrays, child_cid, state_root_cid):
    """A tipset-like object over the given flat arrays (A.make_tipset_desc, api.BlockStore.from_tipset and oracle.Store.from_tipset
    accept it): ts's descriptor with this child header and parent_state_root."""
    return EditedTipset(ts, child_cid=np.frombuffer(child_cid, dtype=np.uint8), parent_state_root=np.frombuffer(state_root_cid, dtype=np.uint8),
                        **arrays)


# ------------------------------------------------------------------ the catalogue of read_storage_slot cases
class SlotCase:
    """One read_storage_slots call: `root` (contract-state CID) and `slots`. truth: per slot the Vec<u8> the builder put under it (as
    bytes) or None; None for a case that must fail (`status`: the failure the decode contract prescribes)."""

    def __init__(self, name, root, slots, truth=None, status=None, bw=None):
        self.name, self.root, self.slots, self.truth, self.status, self.bw = name, root, slots, truth, status, bw

    def slots_np(self):
        return np.frombuffer(b"".join(self.slots), dtype=np.uint8).reshape(-1, 32)

    def root_np(self):
        return np.frombuffer(self.root, dtype=np.uint8)


WIDTHS = range(1, 9)
SIZES = (1, 3, 4, 200, 5000)
VALUE_LENGTHS = (0, 1, 23, 24, 31, 32, 33, 255, 256, 300)


def _value(rng, n=None):
    if n is None:
        n = rng.choice((0, 1, 5, 20, 31, 32, 32, 32, 33, 40))
    return bytes(rng.randrange(256) for _ in range(n))


def _mix(rng, truth, n_present=120, n_absent=40, n_dup=10):
    """Present (a sample of truth's keys), duplicate and absent slots in shuffled order → (slots, their truth values)."""
    keys = list(truth)
    pick = keys if len(keys) <= n_present else rng.sample(keys, n_present)
    pick = pick + [rng.choice(pick) for _ in range(n_dup)] + [rng.randbytes(32) for _ in range(n_absent)]
    rng.shuffle(pick)
    return pick, [truth.get(k) for k in pick]


@functools.lru_cache(maxsize=None)
def width_trees():
    """Canonical tries at every bit width 1–8 and size of SIZES: {(bw, size): (root, truth {slot: value bytes})}, and their blocks."""
    blocks = Blocks()
    out = {}
    for bw in WIDTHS:
        for size in SIZES:
            rng = random.Random(1000 * bw + size)
            truth = {rng.randbytes(32): _value(rng) for _ in range(size)}
            out[(bw, size)] = build_hamt(blocks, {k: u8vec(v) for k, v in truth.items()}, bw), truth
    return blocks, out


@functools.lru_cache(maxsize=None)
def world_slots():
    """Every read_storage_slot case of the GPU tests over ONE block set → (Blocks, [SlotCase])."""
    tblocks, trees = width_trees()
    blocks = Blocks(tblocks)
    cases = []
    rng = random.Random(7)

    # B1 / B2 over every width and size; C (width 5)
    for (bw, size), (root, truth) in trees.items():
        slots, want = _mix(random.Random(bw * 31 + size), truth)
        cases.append(SlotCase(f"B1-w{bw}-n{size}", blocks.put(wrap_b1(root, bw)), slots, want, bw=bw))
        cases.append(SlotCase(f"B2-w{bw}-n{size}", blocks.put(wrap_b2(root, bw)), slots, want, bw=bw))
        if bw == 5:
            cases.append(SlotCase(f"C-n{size}", root, slots, want, bw=5))

    # inline shapes A1–A3: byte-string values of every length, values longer than 32 bytes keep their last 32
    pairs = [(rng.randbytes(32), _value(rng, n)) for n in (0, 1, 31, 32, 33, 40, 64, 100)]
    truth = dict(pairs)
    other = [(rng.randbytes(32), _value(rng, 40))]
    short_key = [(pairs[0][0][:31], b"short key"), (pairs[1][0] + b"\0", b"long key")]
    slots, want = _mix(rng, truth, n_absent=6, n_dup=3)
    slots += [k for k, _ in other]                 # only in the second map of A1: not searched
    want += [None]
    cases.append(SlotCase("A1", blocks.put(wrap_a1([small_map(pairs + short_key), small_map(other)])), slots, want))
    cases.append(SlotCase("A2", blocks.put(wrap_a2(small_map(short_key + pairs, extra=[("x", 7)]))), slots, want))
    cases.append(SlotCase("A3", blocks.put(wrap_a3(small_map(pairs))), slots, want))
    cases.append(SlotCase("A1-first-pair-wins", blocks.put(wrap_a1([small_map([(pairs[2][0], b"first"), (pairs[2][0], b"second")])])),
                          [pairs[2][0]], [b"first"]))

    # value shapes: Vec<u8> of every head size (8x, 98 xx, 99 xxxx), elements in one-byte and `18 xx` form
    vt = {rng.randbytes(32): _value(rng, n) for n in VALUE_LENGTHS}
    vt[rng.randbytes(32)] = bytes(range(24))                     # 1-byte elements only
    vt[rng.randbytes(32)] = bytes(range(24, 256)) + bytes(range(24))
    for bw in (1, 5, 8):
        root = build_hamt(blocks, {k: u8vec(v) for k, v in vt.items()}, bw)
        slots, want = _mix(rng, vt, n_absent=4, n_dup=2)
        cases.append(SlotCase(f"values-w{bw}", blocks.put(wrap_b1(root, bw)), slots, want, bw=bw))
    # elements that must fail: 256, a non-minimal element, a non-minimal array head
    for name, enc in (("elem-256", b"\x82\x01\x19\x01\x00"), ("elem-nonminimal", b"\x82\x01\x18\x05"),
                      ("array-head-nonminimal", b"\x98\x02\x01\x02")):
        k = rng.randbytes(32)
        root = blocks.put(hamt_node({hash_index(k, 0, 5): [(k, enc)]}))
        cases.append(SlotCase(f"value-{name}", root, [k, rng.randbytes(32)], status=A.ERR_DECODE))

    # node shapes
    nt = {rng.randbytes(32): _value(rng) for _ in range(300)}
    root = build_hamt(blocks, {k: u8vec(v) for k, v in nt.items()}, 5, bitfield_len=32)          # leading zero bytes
    slots, want = _mix(rng, nt)
    cases.append(SlotCase("bitfield-leading-zeros", root, slots, want, bw=5))
    root = build_hamt(blocks, {k: u8vec(v) for k, v in nt.items()}, 3, bitfield_len=5)
    cases.append(SlotCase("bitfield-leading-zeros-w3", blocks.put(wrap_b1(root, 3)), slots, want, bw=3))
    # bits above 2^bw (width 3 root with a pointer at index 200): the rank of every real index is unchanged
    small = {rng.randbytes(32): _value(rng) for _ in range(12)}
    ptrs = {}
    for k, v in sorted(small.items()):
        ptrs.setdefault(hash_index(k, 0, 3), []).append((k, u8vec(v)))
    ptrs = {i: b if len(b) <= 3 else b[:3] for i, b in ptrs.items()}
    tr = {k: small[k] for b in ptrs.values() for k, _ in b}
    ptrs[200] = [(rng.randbytes(32), u8vec(b"x"))]
    ptrs[9] = [(rng.randbytes(32), u8vec(b"y"))]
    root = blocks.put(hamt_node(ptrs))
    slots, want = _mix(rng, tr, n_absent=10, n_dup=2)
    cases.append(SlotCase("bits-above-width", blocks.put(wrap_b1(root, 3)), slots, want, bw=3))
    # buckets of 4–30 entries (non-canonical; a `98` head from 24 on), keys of other lengths, a key twice in one bucket
    for n in (4, 23, 24, 30):
        ks = []
        while len(ks) < n:
            k = rng.randbytes(32)
            if hash_index(k, 0, 5) == 17:
                ks.append(k)
        bt = {k: _value(rng) for k in ks}
        other_k = rng.randbytes(32)
        ptrs = {17: [(k, u8vec(v)) for k, v in sorted(bt.items())]}
        ptrs.setdefault(hash_index(other_k, 0, 5), []).append((other_k, u8vec(b"o")))
        bt[other_k] = b"o"
        root = blocks.put(hamt_node(ptrs))
        slots, want = _mix(rng, bt, n_absent=5, n_dup=2)
        cases.append(SlotCase(f"bucket-{n}", root, slots, want, bw=5))
    k = rng.randbytes(32)
    i = hash_index(k, 0, 5)
    bucket = [(k[:31], u8vec(b"31")), (k + b"\0", u8vec(b"33")), (b"", u8vec(b"0")), (k, u8vec(b"first")), (k, u8vec(b"second"))]
    k2 = k[:31] + bytes([k[31] ^ 1])
    root = blocks.put(hamt_node({i: bucket}))
    cases.append(SlotCase("bucket-odd-keys", root, [k, k2, k], [b"first", None, b"first"], bw=5))

    # wrapper bit widths: the `bw as u32` truncation; out-of-range widths; B2 variants; a non-minimal bitwidth integer
    root3, t3 = trees[(3, 200)]
    slots3, want3 = _mix(random.Random(3), t3, n_present=40, n_absent=10, n_dup=2)
    cases.append(SlotCase("B1-bw-2^32+3", blocks.put(wrap_b1(root3, 2 ** 32 + 3)), slots3, want3, bw=3))
    cases.append(SlotCase("B2-bw-2^32+3", blocks.put(wrap_b2(root3, 2 ** 32 + 3)), slots3, want3, bw=3))
    for bw in (0, 9, 2 ** 32, 2 ** 64 - 1):
        cases.append(SlotCase(f"B1-bw-{bw}", blocks.put(wrap_b1(root3, bw)), slots3[:3], status=A.ERR_DECODE))
        cases.append(SlotCase(f"B2-bw-{bw}", blocks.put(wrap_b2(root3, bw)), slots3[:3], status=A.ERR_DECODE))
    cases.append(SlotCase("B2-reordered-unknown", blocks.put(wrap_b2(root3, 3, [("zz", b"\x80"), ("bitwidth", head(0, 3)), ("x", cbytes(b"?")),
                                                                                  ("root", clink(root3))])), slots3, want3, bw=3))
    cases.append(SlotCase("B2-dup-root", blocks.put(wrap_b2(root3, 3, [("root", clink(root3)), ("bitwidth", head(0, 3)), ("root", clink(root3))])),
                          slots3[:3], status=A.ERR_DECODE))
    cases.append(SlotCase("B1-bw-nonminimal", blocks.put(b"\x82" + clink(root3) + b"\x18\x03"), slots3[:3], status=A.ERR_DECODE))

    # depth boundaries at every width: ⌊256/bw⌋ nodes (present; key's bit clear) succeed, one node more is a decode error
    for bw in WIDTHS:
        key = rng.randbytes(32)
        val = _value(rng, 40)
        sib = {lvl: [(k, u8vec(_value(rng))) for k in ks] for lvl, ks in chain_siblings(key, bw, rng).items()}
        truth = {k: _decode_u8vec(v) for lvl in sib for k, v in sib[lvl]}
        n = max_levels(bw)
        top = build_chain(blocks, key, u8vec(val), bw, n, siblings=sib)
        sl = [key] + list(truth) + [rng.randbytes(32)]
        cases.append(SlotCase(f"depth-w{bw}-{n}", blocks.put(wrap_b1(top, bw)), sl, [val] + list(truth.values()) + [None], bw=bw))
        top = build_chain(blocks, key, u8vec(val), bw, n, present=False, siblings=sib)
        cases.append(SlotCase(f"depth-w{bw}-{n}-absent", blocks.put(wrap_b1(top, bw)), sl, [None] + list(truth.values()) + [None], bw=bw))
        top = build_chain(blocks, key, u8vec(val), bw, n + 1)
        cases.append(SlotCase(f"depth-w{bw}-{n + 1}", blocks.put(wrap_b1(top, bw)), [key], status=A.ERR_DECODE, bw=bw))
    return blocks, cases


def _decode_u8vec(enc):
    return bytes(cbor2.loads(enc))


# ------------------------------------------------------------------ full state trees for generate_storage_proofs
ACTOR_IDS = (0, 1000, 2 ** 63, 2 ** 64 - 1)


class ProofWorld:
    """State trees over one block set, each behind its own child header (`tips[name]`): "main" (a canonical actors HAMT), "deep" (the
    deepest accepted path) and "deep52" (an actors chain one level too deep). `actors` maps every actor of main to (ActorState bytes,
    {slot: value} or None where its proofs must fail); `faults` {actor: (slot, node on its path, trie root)} names the nodes the fault
    tests drop or mutate."""


@functools.lru_cache(maxsize=None)
def _world_proofs_blocks():
    tblocks, trees = width_trees()
    blocks = Blocks(tblocks)
    rng = random.Random(11)
    w = ProofWorld()
    actors = {}            # actor id -> (ActorState bytes, {slot: value | None})
    storage = {}           # actor id -> contract-state root

    def add_actor(aid, contract_root, truth, six=True):
        st = blocks.put(evm_state(contract_root, six=six))
        actors[aid] = (actor_state(st, sequence=aid % 7), truth)
        storage[aid] = contract_root

    root3, t3 = trees[(3, 200)]
    root7, t7 = trees[(7, 200)]
    root5, t5 = trees[(5, 200)]
    add_actor(0, blocks.put(wrap_b1(root3, 3)), t3)
    add_actor(1000, blocks.put(wrap_b2(root7, 7)), t7, six=False)
    pairs = [(rng.randbytes(32), _value(rng, n)) for n in (0, 20, 32, 45)]
    add_actor(2 ** 63, blocks.put(wrap_a2(small_map(pairs))), dict(pairs))
    add_actor(2 ** 64 - 1, root5, t5, six=False)
    # depth boundaries through the proof path: B1 chains of ⌊256/bw⌋ nodes (present / key's bit clear) and one more
    w.chain = {}
    for bw in WIDTHS:
        key, val = rng.randbytes(32), _value(rng, 33)
        n = max_levels(bw)
        add_actor(1000 + bw, blocks.put(wrap_b1(build_chain(blocks, key, u8vec(val), bw, n), bw)), {key: val})
        add_actor(1010 + bw, blocks.put(wrap_b1(build_chain(blocks, key, u8vec(val), bw, n, present=False), bw)), {key: None})
        add_actor(1020 + bw, blocks.put(wrap_b1(build_chain(blocks, key, u8vec(val), bw, n + 1), bw)), None)
        w.chain[bw] = key
    # fault carriers: their own small tries, faulted in a copy of the store by the tests
    w.faults = {}
    for aid, bw in ((2001, 2), (2002, 6)):
        tr = {rng.randbytes(32): _value(rng) for _ in range(60)}
        root = build_hamt(blocks, {k: u8vec(v) for k, v in tr.items()}, bw)
        add_actor(aid, blocks.put(wrap_b1(root, bw)), tr)
        # a node at depth 1 on some key's path
        k = next(k for k in tr if _child_on_path(blocks, root, k, bw) is not None)
        w.faults[aid] = (k, _child_on_path(blocks, root, k, bw), root)
    add_actor(2003, blocks.put(wrap_b1(build_chain(blocks, w.chain[4], u8vec(b"x"), 4, 65), 4)), None)    # max depth
    add_actor(2004, blocks.put(wrap_b1(root3, 0)), None)                                                   # broken wrapper
    # fillers sharing one A3 contract state
    shared = dict((rng.randbytes(32), _value(rng)) for _ in range(5))
    shared_root = blocks.put(wrap_a3(small_map(list(shared.items()))))
    w.fillers = []
    while len(w.fillers) < 300:
        aid = rng.randrange(1, 2 ** rng.choice((12, 20, 40, 64)))
        if aid not in actors:
            add_actor(aid, shared_root, shared, six=bool(aid & 1))
            w.fillers.append(aid)
    actors_root = build_hamt(blocks, {id_address(a): s for a, (s, _) in actors.items()}, 5)
    w.main_root = blocks.put(state_root(actors_root))
    w.actors, w.storage = actors, storage

    # the deepest path: actors chain of 51 nodes (width 5) + B1 width-1 chain of 256 nodes = 311 recorded blocks
    w.deep_actor = 2 ** 64 - 1
    w.deep_slot = rng.randbytes(32)
    w.deep_value = _value(rng, 40)
    sib = {lvl: [(k, u8vec(_value(rng))) for k in ks] for lvl, ks in chain_siblings(w.deep_slot, 1, rng).items()}
    w.deep_siblings = {k: _decode_u8vec(v) for lvl in sib for k, v in sib[lvl]}
    deep_storage = blocks.put(wrap_b1(build_chain(blocks, w.deep_slot, u8vec(w.deep_value), 1, 256, siblings=sib), 1))
    deep_state = blocks.put(evm_state(deep_storage))
    akey = id_address(w.deep_actor)
    w.deep_sib_actors = _actor_siblings(akey, actors)
    asib = {0: [(id_address(a), actors[a][0]) for a in w.deep_sib_actors]}
    w.deep_root = blocks.put(state_root(build_chain(blocks, akey, actor_state(deep_state), 5, 51, siblings=asib)))
    w.deep_storage = deep_storage
    w.deep52_root = blocks.put(state_root(build_chain(blocks, akey, actor_state(deep_state), 5, 52)))
    return blocks, w


def _child_on_path(blocks, root, key, bw):
    """CID of the child node key's lookup visits right below the root, or None."""
    node = cbor2.loads(blocks[root])
    i = hash_index(key, 0, bw)
    bf = int.from_bytes(node[0], "big")
    if not (bf >> i) & 1:
        return None
    p = node[1][bin(bf & ((1 << i) - 1)).count("1")]
    return bytes(p.value[1:]) if isinstance(p, cbor2.CBORTag) else None


def _actor_siblings(akey, actors):
    """Actors of the main tree whose width-5 index at level 0 differs from akey's (siblings of the deep chain's root)."""
    i = hash_index(akey, 0, 5)
    return [a for a in sorted(actors) if a != 2 ** 64 - 1 and hash_index(id_address(a), 0, 5) != i][:3]


def world_proofs(ts):
    """(ProofWorld, Flat) with tips {main, deep, deep52} over ts's child header (ts: the ts3_small tipset)."""
    blocks, w = _world_proofs_blocks()
    blocks = Blocks(blocks)
    heads = {}
    for name, root in (("main", w.main_root), ("deep", w.deep_root), ("deep52", w.deep52_root)):
        hdr, c = child_header(ts, root)
        blocks[c] = hdr
        heads[name] = (c, root)
    flat = Flat(blocks)
    w.heads = heads
    w.tips = {name: tipset(ts, flat.arrays(), c, root) for name, (c, root) in heads.items()}
    return w, flat


def proof_truth(w, tip, actor, slot):
    """Ground truth of a proof against tip "main" or "deep": the value bytes or None; KeyError where the proof must fail."""
    if tip == "deep" and actor == w.deep_actor:
        return w.deep_value if slot == w.deep_slot else w.deep_siblings.get(slot)
    if tip == "deep" and actor not in w.deep_sib_actors:
        raise KeyError(actor)
    truth = w.actors[actor][1]
    if truth is None:
        raise KeyError(actor)
    return truth.get(slot)


def proof_batches(w, rng=None):
    """Spec batches over world_proofs' tips → (ok, bad): ok = [(tip, specs)] that must succeed with proof_truth's values, bad =
    [(tip, specs)] whose last spec must fail (depth limit, broken wrapper, actor not found, the 52-node actors chain)."""
    rng = rng or random.Random(5)
    main = []
    for a in ACTOR_IDS + (2001, 2002):
        truth = w.actors[a][1]
        main += [(a, s) for s in sorted(truth)[:4]] + [(a, rng.randbytes(32))]
    for bw in WIDTHS:
        main += [(1000 + bw, w.chain[bw]), (1010 + bw, w.chain[bw]), (1000 + bw, rng.randbytes(32))]
    for a in w.fillers[::15]:
        main.append((a, sorted(w.actors[a][1])[0]))
    deep = [(w.deep_actor, w.deep_slot), (w.deep_actor, rng.randbytes(32))] + [(w.deep_actor, s) for s in w.deep_siblings]
    deep += [(a, sorted(w.actors[a][1])[0]) for a in w.deep_sib_actors]
    good = main[0]
    missing = next(a for a in range(7, 100) if a not in w.actors)
    bad = [("main", [good, (1020 + bw, w.chain[bw])]) for bw in WIDTHS]
    bad += [("main", [good, (2003, w.chain[4])]), ("main", [good, (2004, main[1][1])]), ("main", [good, (missing, main[0][1])]),
            ("deep52", [(w.deep_actor, w.deep_slot)])]
    return [("main", main), ("deep", deep)], bad
