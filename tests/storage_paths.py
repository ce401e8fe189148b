"""Solidity's storage-layout rules restated in Python (a helper module, not a fixture file), and one contract laid out by them in a
hand-built state tree (tests/storage_trees.py) for the storage-path tests.

The rules (docs.soliditylang.org, "Layout of State Variables in Storage"), all arithmetic mod 2^256:
  mapping        value of key k at keccak256(h(k) ‖ p): h(k) is the 32-byte padded form of a value type, the raw bytes of bytes / string
  dynamic array  length word at p, element i at keccak256(p) + (i / per_slot) * elem_slots
  static array   element i at p + (i / per_slot) * elem_slots
  struct member  at p + its slot offset
  bytes / string a header word at p: length*2 with the bytes in the high-order end (short, <= 31), or length*2 + 1 with the bytes in
                 ceil(length / 32) slots from keccak256(p) (long, >= 32)
keccak256 is oracle/pyoracle.py's, pinned by the forge-std known answers (tests/test_oracle_cpu.py)."""
import random

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200.api import StoragePath
from oracle.pyoracle import keccak256
from tests import storage_trees as T

M = 1 << 256
ZERO = bytes(32)


def u256(b):
    return int.from_bytes(b, "big")


def b32(x):
    return (x % M).to_bytes(32, "big")


def derive(path):
    """A StoragePath's slots: (length-word slots of its ARRAY steps, value or header slots, final slot, packed byte offset)."""
    slot, lengths, off = path.base_slot, [], 0
    for op, key, index, elem_slots, elem_bytes in path.steps:
        off = 0
        if op == A.PATH_MAPPING:
            slot = keccak256(key + slot)
        elif op == A.PATH_FIELD:
            slot = b32(u256(slot) + index)
        else:
            per = 32 // elem_bytes if elem_slots == 1 and elem_bytes >= 1 else 1
            if op == A.PATH_ARRAY:
                lengths.append(slot)
                slot = keccak256(slot)
            slot = b32(u256(slot) + (index // per) * elem_slots)
            if per > 1:
                off = (index % per) * elem_bytes
    values = [b32(u256(slot) + w) for w in range(path.n_words)] if path.kind == A.PATH_WORDS else [slot]
    return lengths, values, slot, off


def expand(path, read):
    """The path against storage, read(slot) → its 32-byte word (zero when absent) → (expanded specs [(actor, slot)], status, value,
    final slot, byte offset), as include/ipcfp.h states them."""
    lengths, values, slot, off = derive(path)
    status = A.PATH_OK
    arrays = [s for s in path.steps if s[0] == A.PATH_ARRAY]
    for ls, st in zip(lengths, arrays):
        if status == A.PATH_OK and u256(read(ls)) <= st[2]:
            status = A.PATH_INDEX_OUT_OF_RANGE
    specs, value = lengths + values, b""
    if path.kind == A.PATH_WORDS:
        value = b"".join(read(s) for s in values)
    else:
        h = read(slot)
        hv, bstat = u256(h), A.PATH_OK
        if hv & 1 == 0:
            n = (hv & 0xff) >> 1
            if n > 31:
                bstat = A.PATH_BAD_BYTES
            else:
                value = h[:n]
        else:
            n = hv >> 1
            if n > A.PATH_MAX_BYTES:
                bstat = A.PATH_TOO_LONG
            elif n < 32:
                bstat = A.PATH_BAD_BYTES
            else:
                base = u256(keccak256(slot))
                data = [b32(base + j) for j in range((n + 31) // 32)]
                specs += data
                value = b"".join(read(d) for d in data)[:n]
        if status == A.PATH_OK:
            status = bstat
    return [(path.actor_id, s) for s in specs], status, value, slot, off


# ------------------------------------------------------------------ random paths and hand-picked edges (the host campaign and the GPU worlds)
KEY_EDGES = (0, 1, 31, 32, 33, 103, 104, 105, 135, 136, 137, 239, 240, 241, 375, 376, 377, A.PATH_MAX_KEY - 1, A.PATH_MAX_KEY)
U64_EDGES = (0, 1, 2, 31, 32, 33, 2 ** 32 - 1, 2 ** 32, 2 ** 63, 2 ** 64 - 1)


def random_u256(rng):
    return rng.choice([rng.randrange(16), M - 1 - rng.randrange(16), rng.randrange(M), (1 << rng.randrange(256)) - rng.randrange(3)]) % M


def step(rng):
    op = rng.choice((A.PATH_MAPPING, A.PATH_MAPPING, A.PATH_ARRAY, A.PATH_STATIC, A.PATH_FIELD))
    if op == A.PATH_MAPPING:
        n = rng.choice(KEY_EDGES + (32, 32, 20, rng.randrange(A.PATH_MAX_KEY + 1)))
        return (op, rng.randbytes(n), 0, 0, 0)
    index = rng.choice(U64_EDGES + (rng.randrange(100), rng.randrange(2 ** 64)))
    if op == A.PATH_FIELD:
        return (op, b"", index, 0, 0)
    es = rng.choice((1, 1, 1, 2, 3, 7, 2 ** 32 - 1))
    eb = rng.choice((0, 0, 1, 2, 3, 8, 16, 20, 31, 32))
    return (op, b"", index, es, eb)


def header(rng):
    """a bytes / string header word of every form"""
    kind = rng.randrange(7)
    if kind == 0:
        return bytes(31) + bytes([2 * rng.randrange(32)])                        # short
    if kind == 1:
        return rng.randbytes(31) + bytes([2 * rng.randrange(32, 128)])           # short, BAD_BYTES
    if kind == 2:
        return b32(2 * rng.choice((32, 33, 63, 64, 65, rng.randrange(32, A.PATH_MAX_BYTES + 1), A.PATH_MAX_BYTES)) + 1)   # long
    if kind == 3:
        return b32(2 * rng.randrange(32) + 1)                                    # long, BAD_BYTES
    if kind == 4:
        return b32(2 * rng.choice((A.PATH_MAX_BYTES + 1, rng.randrange(A.PATH_MAX_BYTES + 1, 2 ** 64), rng.randrange(M // 2))) + 1)   # TOO_LONG
    if kind == 5:
        return rng.randbytes(32)
    return bytes(32)


def case(rng, storage, actors=None):
    """One random path; its words go into storage. Without actors the path's actor ID is random and storage is one {slot: word};
    with actors (a sequence of IDs) the actor is drawn from them and storage is {actor: {slot: word}}. The random-number calls
    without actors are those of the host campaign's seeds, so a seed always gives the same paths."""
    steps = tuple(step(rng) for _ in range(rng.choice((0, 1, 2, 3, 4, 6, A.PATH_MAX_STEPS))))
    is_bytes = rng.random() < 0.5
    actor = rng.randrange(2 ** 64) if actors is None else rng.choice(actors)
    if is_bytes:
        p = StoragePath(actor, random_u256(rng), steps, A.PATH_BYTES, 0)
    else:
        p = StoragePath(actor, random_u256(rng), steps, A.PATH_WORDS, rng.choice((1, 1, 2, 3, A.PATH_MAX_WORDS)))
    st = storage if actors is None else storage[actor]
    lengths, values, slot, _ = derive(p)
    arrays = [s for s in steps if s[0] == A.PATH_ARRAY]
    for ls, s in zip(lengths, arrays):
        if rng.random() < 0.8:
            st[ls] = rng.choice((b32(s[2] + 1 + rng.randrange(5)), b32(s[2]), b32(max(s[2] - 1, 0)), rng.randbytes(32)))
    if p.kind == A.PATH_WORDS:
        for v in values:
            if rng.random() < 0.7:
                st[v] = rng.randbytes(32)
    else:
        st[slot] = header(rng)
        base = u256(keccak256(slot))
        for j in range(A.PATH_MAX_BYTES // 32 + 1):
            if rng.random() < 0.9:
                st[b32(base + j)] = rng.randbytes(32)
    return p


EDGE_ACTOR = 7


def edges():
    """hand-picked paths: carries out of the top byte, the caps, every header form on one slot each (actor EDGE_ACTOR)"""
    top = M - 1
    P = lambda base, *steps, kind=A.PATH_WORDS, n=1: StoragePath(EDGE_ACTOR, base, steps, kind, n)
    paths = [P(top, (A.PATH_FIELD, b"", 1, 0, 0)), P(top, (A.PATH_FIELD, b"", 2 ** 64 - 1, 0, 0), n=A.PATH_MAX_WORDS),
             P(top - 5, (A.PATH_STATIC, b"", 2 ** 64 - 1, 2 ** 32 - 1, 0)), P(0, (A.PATH_STATIC, b"", 2 ** 64 - 1, 1, 1)),
             P(3, (A.PATH_ARRAY, b"", 2 ** 64 - 1, 2 ** 32 - 1, 0), (A.PATH_FIELD, b"", 2 ** 64 - 1, 0, 0))]
    paths += [P(5, (A.PATH_MAPPING, (bytes(range(256)) * 4)[:n], 0, 0, 0)) for n in KEY_EDGES]
    paths += [P(k, (A.PATH_ARRAY, b"", i, 1, eb)) for k, (i, eb) in enumerate((i, eb) for eb in range(1, 33) for i in (0, 31, 32, 63))]
    paths += [P(9000 + k, kind=A.PATH_BYTES) for k in range(12)]
    return paths


def edge_storage(paths):
    """{slot: word} for edges(): the twelve header forms with every data slot written, every array length 2^64 - 1"""
    storage = {}
    hdr = [bytes(32), bytes(31) + b"\x3e", bytes(31) + b"\x40", b32(2 * 32 + 1), b32(2 * 31 + 1), b32(1),
           b32(2 * A.PATH_MAX_BYTES + 1), b32(2 * (A.PATH_MAX_BYTES + 1) + 1), b"\xff" * 32, b32(2 * 33 + 1),
           b32(2 * 65 + 1), b"\xff" * 31 + b"\xfe"]
    for k, p in enumerate(paths[-12:]):
        storage[p.base_slot] = hdr[k]
        base = u256(keccak256(p.base_slot))
        for j in range(A.PATH_MAX_BYTES // 32 + 1):
            storage[b32(base + j)] = bytes([j % 256]) * 32
    for p in paths[:-12]:
        for ls in derive(p)[0]:
            storage[ls] = b32(2 ** 64 - 1)
    return storage


def encode_string(slot, s):
    """{slot: word} of a bytes / string value stored at slot"""
    s = bytes(s)
    if len(s) <= 31:
        return {slot: s.ljust(31, b"\0") + bytes([2 * len(s)])}
    out = {slot: b32(2 * len(s) + 1)}
    base = u256(keccak256(slot))
    for j in range(0, len(s), 32):
        out[b32(base + j // 32)] = s[j:j + 32].ljust(32, b"\0")
    return out


# ------------------------------------------------------------------ one contract
ACTOR = 4242
STRING_LENGTHS = (0, 31, 32, 33, 64, 65, A.PATH_MAX_BYTES, A.PATH_MAX_BYTES + 1)


class Contract:
    """Storage of one contract, {slot: word}, with the state variables
        0  mapping(bytes32 => Subnet) subnets        Subnet { uint256 stake; address owner; uint64 topDownNonce; string name }
                                                     (slot offsets 0, 1, 1 packed at byte 20, 2)
        1  mapping(address => mapping(uint256 => uint256)) allowance
        2  mapping(string => uint256) byName
        3  uint256[] nums          4  uint8[] small (packed)     5  address[] owners      6  Triple[] triples (3 slots each)
        7  uint256[3] fixed3       10 Pair pair { uint256 x; uint256 y }
        12 mapping(uint256 => string) texts: the lengths of STRING_LENGTHS at keys 0.., and two encodings Solidity refuses at 100, 101
        13 mapping(uint256 => uint256) empty (never written)
    and `paths`: (name, StoragePath) over all of it, in-range and out of range, present and absent."""

    def __init__(self, seed=7):
        rng = random.Random(seed)
        st = {}
        p = lambda n: b32(n)
        self.subnet_ids = [rng.randbytes(32) for _ in range(3)]
        for i, sid in enumerate(self.subnet_ids):
            base = keccak256(sid + p(0))
            st[base] = b32(10 ** 18 * (i + 1))
            owner, nonce = rng.randbytes(20), 1000 + i
            st[b32(u256(base) + 1)] = bytes(4) + nonce.to_bytes(8, "big") + owner
            st.update(encode_string(b32(u256(base) + 2), f"calib-subnet-{i}".encode() * (i * 3 + 1)))
        self.owners = [rng.randbytes(20) for _ in range(3)]
        for a in self.owners:
            inner = keccak256(bytes(12) + a + p(1))
            for k in (0, 1, 2 ** 200):
                st[keccak256(b32(k) + inner)] = b32(rng.randrange(1, M))
        for name in ("alpha", "a" * 40, ""):
            st[keccak256(name.encode() + p(2))] = b32(rng.randrange(M))
        nums = [rng.randrange(M) for _ in range(5)]
        st[p(3)] = b32(len(nums))
        for i, v in enumerate(nums):
            st[b32(u256(keccak256(p(3))) + i)] = b32(v)
        small = [rng.randrange(256) for _ in range(70)]
        st[p(4)] = b32(len(small))
        for i in range(0, len(small), 32):
            st[b32(u256(keccak256(p(4))) + i // 32)] = bytes(reversed(bytes(small[i:i + 32]).ljust(32, b"\0")))
        st[p(5)] = b32(len(self.owners))
        for i, a in enumerate(self.owners):
            st[b32(u256(keccak256(p(5))) + i)] = bytes(12) + a
        st[p(6)] = b32(2)
        for i in range(2):
            for f in range(3):
                st[b32(u256(keccak256(p(6))) + 3 * i + f)] = b32(100 * i + f + 1)
        for i in range(3):
            st[p(7 + i)] = b32(7 + i)
        st[p(10)], st[p(11)] = b32(11), b32(12)
        self.texts = {}
        for k, n in enumerate(STRING_LENGTHS):
            s = bytes(rng.randrange(32, 127) for _ in range(n))
            self.texts[k] = s
            st.update(encode_string(keccak256(b32(k) + p(12)), s))
        st[keccak256(b32(100) + p(12))] = b32(80)    # short form with length 40
        st[keccak256(b32(101) + p(12))] = b32(11)    # long form with length 5
        self.storage = st
        self.small, self.nums = small, nums

        P = lambda slot: StoragePath(ACTOR, slot)
        paths = []
        for i, sid in enumerate(self.subnet_ids):
            s = P(0).mapping(sid, "bytes32")
            paths += [(f"subnet{i}.stake", s.field(0)), (f"subnet{i}.owner+nonce", s.field(1)), (f"subnet{i}.name", s.field(2).bytes()),
                      (f"subnet{i}.whole", s.words(2))]
        paths.append(("subnet.absent", P(0).mapping(rng.randbytes(32), "bytes32").field(1)))
        for a in self.owners:
            for k in (0, 2 ** 200, 5):
                paths.append((f"allowance.{k}", P(1).mapping(a, "address").mapping(k, "uint256")))
        for name in ("alpha", "a" * 40, "", "missing"):
            paths.append((f"byName.{name[:8]}", P(2).mapping(name, "string")))
        for i in (0, 4, 5, 2 ** 40):
            paths.append((f"nums[{i}]", P(3).array(i)))
        for i in (0, 31, 32, 69, 70):
            paths.append((f"small[{i}]", P(4).array(i, 1, 1)))
        for i in (0, 2, 3):
            paths.append((f"owners[{i}]", P(5).array(i, 1, 20)))
        for i in (0, 1, 2):
            paths += [(f"triples[{i}].2", P(6).array(i, 3).field(2)), (f"triples[{i}]", P(6).array(i, 3).words(3))]
        paths += [("fixed3[2]", P(7).static(2)), ("fixed3", P(7).words(3)), ("pair.y", P(10).field(1)), ("pair", P(10).words(2))]
        for k in list(self.texts) + [100, 101]:
            paths.append((f"texts[{k}]", P(12).mapping(k, "uint256").bytes()))
        paths += [("empty[3]", P(13).mapping(3, "uint256")), ("empty.bytes", P(13).mapping(3, "uint256").bytes())]
        self.paths = paths

    def read(self, slot):
        return self.storage.get(bytes(slot), ZERO)

    def expected(self, path):
        return expand(path, self.read)

    def world(self, ts, bw=5, drop=()):
        """(Flat, tipset) of a state tree with this contract as actor ACTOR (B1 wrapper at bit width bw) behind ts's child header.
        drop: slots whose HAMT entries are left out (their proofs then prove absence)."""
        blocks = T.Blocks()
        entries = {s: T.u8vec(w) for s, w in self.storage.items() if s not in drop}
        root = T.build_hamt(blocks, entries, bw)
        state = blocks.put(T.evm_state(blocks.put(T.wrap_b1(root, bw))))
        actors = {ACTOR: T.actor_state(state), 1: T.actor_state(state, 1)}
        sroot = blocks.put(T.state_root(T.build_hamt(blocks, {T.id_address(a): v for a, v in actors.items()}, 5)))
        hdr, c = T.child_header(ts, sroot)
        blocks[c] = hdr
        flat = T.Flat(blocks)
        return flat, T.tipset(ts, flat.arrays(), c, sroot)
