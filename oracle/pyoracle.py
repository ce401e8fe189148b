"""Independent Python restatement of the hot path (cbor2 + hashlib) — TEST INFRASTRUCTURE.

Second, independently written implementation used to pin the C++ oracle (oracle/oracle.cpp):
decoding is done by cbor2 (a third-party CBOR codec), Blake2b/SHA-256 by hashlib, Keccak by the
small pure-Python permutation below (checked against published vectors in tests). It follows the
same reference lines as the C++ oracle (events/generator.rs:60-307, common/evm.rs:13-59,
storage/decode.rs:36-97, storage/generator.rs:29-178) on WELL-FORMED inputs; strictness on
malformed inputs is the C++ oracle's job.
"""
import hashlib

import cbor2

CID_PREFIX = bytes([0x01, 0x71, 0xA0, 0xE4, 0x02, 0x20])

# ----------------------------------------------------------------------------- keccak-256
_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
       0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
       0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
       0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
_M = (1 << 64) - 1


def _rol(x, n):
    n %= 64
    return ((x << n) | (x >> (64 - n))) & _M if n else x


_ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]  # [x][y]


def _f1600(a):
    """Keccak-f[1600] on lanes a[x][y] (textbook theta / rho+pi / chi / iota)."""
    for rnd in range(24):
        c = [a[x][0] ^ a[x][1] ^ a[x][2] ^ a[x][3] ^ a[x][4] for x in range(5)]
        d = [c[(x - 1) % 5] ^ _rol(c[(x + 1) % 5], 1) for x in range(5)]
        a = [[a[x][y] ^ d[x] for y in range(5)] for x in range(5)]
        b = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                b[y][(2 * x + 3 * y) % 5] = _rol(a[x][y], _ROT[x][y])
        a = [[(b[x][y] ^ ((~b[(x + 1) % 5][y]) & b[(x + 2) % 5][y])) & _M for y in range(5)] for x in range(5)]
        a[0][0] ^= _RC[rnd]
    return a


def keccak256(data: bytes) -> bytes:
    rate = 136
    p = bytearray(data)
    p.append(0x01)
    while len(p) % rate:
        p.append(0)
    p[-1] |= 0x80
    a = [[0] * 5 for _ in range(5)]
    for off in range(0, len(p), rate):
        for i in range(rate // 8):
            a[i % 5][i // 5] ^= int.from_bytes(p[off + 8 * i: off + 8 * i + 8], "little")
        a = _f1600(a)
    out = b"".join(a[i % 5][i // 5].to_bytes(8, "little") for i in range(4))
    return out


def blake2b256(data: bytes) -> bytes:
    return hashlib.blake2b(data, digest_size=32).digest()


def cid_of(block: bytes) -> bytes:
    return CID_PREFIX + blake2b256(block)


def _varint(b, pos):
    v = 0
    shift = 0
    while True:
        c = b[pos]
        pos += 1
        v |= (c & 0x7F) << shift
        shift += 7
        if not c & 0x80:
            return v, pos


def cid_sort_key(cid: bytes):
    """`Ord` of cid::Cid: (version, codec, (mh code, mh size, digest))."""
    pos = 0
    ver, pos = _varint(cid, pos)
    codec, pos = _varint(cid, pos)
    code, pos = _varint(cid, pos)
    size, pos = _varint(cid, pos)
    return (ver, codec, code, size, cid[pos:])


def _link(tag):
    assert isinstance(tag, cbor2.CBORTag) and tag.tag == 42 and tag.value[0] == 0
    return bytes(tag.value[1:])


class Recorder:
    """RecordingBlockStore (common/blockstore.rs:8-39) over a dict store."""

    def __init__(self, store):
        self.store = store
        self.seen = set()

    def get(self, cid):
        self.seen.add(cid)
        return self.store.get(cid)


class MissingBlock(Exception):
    pass


# ----------------------------------------------------------------------------- AMT
class Amt:
    def __init__(self, root_cid, rec, version):
        raw = rec.get(root_cid)
        if raw is None:
            raise MissingBlock(root_cid)
        r = cbor2.loads(raw)
        if version == 0:
            self.bw = 3
            self.height, self.count, self.root = r
        else:
            self.bw, self.height, self.count, self.root = r
        if not 1 <= self.bw <= 8 or self.height * self.bw > 64:
            raise ValueError("amt: bit width %d, height %d" % (self.bw, self.height))
        self.rec = rec

    def _expand(self, node):
        bmap, links, values = node
        width = 1 << self.bw
        out = [None] * width
        items = links if links else values
        k = 0
        for i in range(width):
            if bmap[i // 8] & (1 << (i % 8)):
                out[i] = items[k]
                k += 1
        assert k == len(items)
        return bool(links), out

    def _load(self, link):
        raw = self.rec.get(_link(link))
        if raw is None:
            raise MissingBlock(_link(link))
        return cbor2.loads(raw)

    def get(self, i):
        width = 1 << self.bw
        if i >= width ** (self.height + 1):
            return None
        node = self.root
        for h in range(self.height, -1, -1):
            is_link, slots = self._expand(node)
            idx = (i // (width ** h)) % width
            if slots[idx] is None:
                return None
            if not is_link:
                return slots[idx] if h == 0 else None
            node = self._load(slots[idx])
        return None

    def for_each(self, f):
        width = 1 << self.bw

        def walk(node, h, base):
            is_link, slots = self._expand(node)
            for i, s in enumerate(slots):
                if s is None:
                    continue
                if is_link:
                    walk(self._load(s), h - 1, base + i * width ** h)
                else:
                    f(base + i, s)

        walk(self.root, self.height, 0)


# ----------------------------------------------------------------------------- evm.rs
def extract_evm_log(entries):
    m = {}
    for flags, key, codec, value in entries:
        m[key] = value
    if "topics" in m:
        tb = m["topics"]
        if len(tb) % 32:
            return None
        return [tb[i:i + 32] for i in range(0, len(tb), 32)], m.get("data", b"")
    topics = []
    for k in ("t1", "t2", "t3", "t4"):
        if k not in m:
            break
        if len(m[k]) != 32:
            return None
        topics.append(m[k])
    if not topics:
        return None
    return topics, m.get("d", b"")


def ascii_to_bytes32(s):
    b = s.encode()[:32]
    return b + bytes(32 - len(b))


def left_pad_32(v):
    return v[-32:] if len(v) >= 32 else bytes(32 - len(v)) + v


def compute_mapping_slot(key32, slot_index):
    return keccak256(key32 + slot_index.to_bytes(32, "big"))


# ----------------------------------------------------------------------------- events path
def collect_exec_list(store_get, txmeta_cids):
    out, seen = [], set()
    rec = Recorder({})
    rec.get = store_get
    for tx in txmeta_cids:
        raw = store_get(tx)
        if raw is None:
            raise MissingBlock(tx)
        bls, secp = cbor2.loads(raw)
        for root in (bls, secp):
            amt = Amt(_link(root), rec, 0)

            def f(_, c):
                c = _link(c)
                if c not in seen:
                    seen.add(c)
                    out.append(c)

            amt.for_each(f)
    return out


def generate_event_proof(store, ts, event_signature, topic_1, actor_id_filter=None):
    """store: dict cid->bytes; ts: object with the synth.Tipset descriptor attributes."""
    topic0 = keccak256(event_signature.encode())
    topic1 = ascii_to_bytes32(topic_1)

    def matches(log):
        topics, _ = log
        return len(topics) >= 2 and topics[0] == topic0 and topics[1] == topic1

    needed = set()
    for c in ts.parent_cids:
        needed.add(bytes(c))
    needed.add(bytes(ts.child_cid))
    needed.add(bytes(ts.receipts_root))
    txmeta = [bytes(c) for c in ts.parent_txmeta_cids]
    needed.update(txmeta)
    for tx in txmeta:
        rec = Recorder(store)
        raw = rec.get(tx)
        if raw is None:
            raise MissingBlock(tx)
        bls, secp = cbor2.loads(raw)
        for root in (bls, secp):
            Amt(_link(root), rec, 0).for_each(lambda i, v: None)
        needed |= rec.seen
    exec_order = collect_exec_list(store.get, txmeta)

    rec_receipts = Recorder(store)
    r_amt = Amt(bytes(ts.receipts_root), rec_receipts, 0)
    matching = []
    for i in range(int(ts.n_receipts)):
        if not ts.has_events_root[i]:
            continue
        amt = Amt(bytes(ts.events_roots[i]), Recorder(store), 3)
        hit = []

        def f(j, se):
            emitter, entries = se
            if actor_id_filter is not None and emitter != actor_id_filter:
                return
            log = extract_evm_log(entries)
            if log and matches(log):
                hit.append(j)

        amt.for_each(f)
        if hit:
            matching.append(i)
    proofs = []
    for i in matching:
        if i >= len(exec_order):
            raise IndexError("Missing message at index %d" % i)
        msg = exec_order[i]
        if r_amt.get(i) is None:
            continue
        rec_e = Recorder(store)
        amt = Amt(bytes(ts.events_roots[i]), rec_e, 3)

        def g(j, se, i=i, msg=msg):
            emitter, entries = se
            if actor_id_filter is not None and emitter != actor_id_filter:
                return
            log = extract_evm_log(entries)
            if log and matches(log):
                proofs.append((i, j, emitter, tuple(log[0]), log[1], msg))

        amt.for_each(g)
        needed |= rec_e.seen
    needed |= rec_receipts.seen
    witness = sorted(needed, key=cid_sort_key)
    for c in witness:
        if c not in store:
            raise MissingBlock(c)
    return dict(matching=matching, proofs=proofs, witness=witness, exec_order=exec_order)


# ----------------------------------------------------------------------------- HAMT / storage path
def hamt_get(rec, root, bw, key):
    raw = rec.get(root)
    if raw is None:
        raise MissingBlock(root)
    node = cbor2.loads(raw)
    h = int.from_bytes(hashlib.sha256(key).digest(), "big")
    consumed = 0
    while True:
        idx = (h >> (256 - consumed - bw)) & ((1 << bw) - 1)
        consumed += bw
        bf = int.from_bytes(node[0], "big")
        if not (bf >> idx) & 1:
            return None
        pos = bin(bf & ((1 << idx) - 1)).count("1")
        p = node[1][pos]
        if isinstance(p, cbor2.CBORTag):
            raw = rec.get(_link(p))
            if raw is None:
                raise MissingBlock(_link(p))
            node = cbor2.loads(raw)
            continue
        for k, v in p:
            if k == key:
                return v
        return None


def _is_small_map(x):
    return isinstance(x, dict) and "v" in x and isinstance(x["v"], list) and all(
        isinstance(p, list) and len(p) == 2 and isinstance(p[0], bytes) and isinstance(p[1], bytes) for p in x["v"])


def read_storage_slot(rec, root, slot):
    raw = rec.get(root)
    if raw is None:
        raise MissingBlock(root)
    x = cbor2.loads(raw)

    def find(sm):
        for k, v in sm["v"]:
            if k == slot:
                return v
        return None

    if isinstance(x, list) and len(x) == 2 and isinstance(x[0], bytes) and isinstance(x[1], list) and all(_is_small_map(e) for e in x[1]):
        if x[1]:
            return find(x[1][0])
    if isinstance(x, list) and len(x) == 2 and isinstance(x[0], bytes) and _is_small_map(x[1]):
        return find(x[1])
    if _is_small_map(x):
        return find(x)
    val = None
    if isinstance(x, list) and len(x) == 2 and isinstance(x[0], cbor2.CBORTag) and isinstance(x[1], int) and x[1] >= 0:
        val = hamt_get(rec, _link(x[0]), x[1] & 0xffffffff, slot)   # `bw as u32` (storage/decode.rs:79)
    elif isinstance(x, dict) and isinstance(x.get("root"), cbor2.CBORTag) and isinstance(x.get("bitwidth"), int):
        val = hamt_get(rec, _link(x["root"]), x["bitwidth"] & 0xffffffff, slot)   # `bitwidth as u32` (:86)
    else:
        val = hamt_get(rec, root, 5, slot)
    return None if val is None else bytes(val)  # Vec<u8> arrives as a list of ints


def _id_address(actor_id):
    out = bytearray([0])
    while actor_id >= 0x80:
        out.append((actor_id & 0x7F) | 0x80)
        actor_id >>= 7
    out.append(actor_id)
    return bytes(out)


def generate_storage_proof(store, ts, actor_id, slot):
    needed = set()
    child = bytes(ts.child_cid)
    hdr = cbor2.loads(store[child])
    psr = _link(hdr[8])
    assert psr == bytes(ts.parent_state_root)
    needed.update([child, psr])
    rec = Recorder(store)
    sr = cbor2.loads(rec.get(psr))
    actor = hamt_get(rec, _link(sr[1]), 5, _id_address(actor_id))
    if actor is None:
        raise KeyError("actor not found")
    state_cid = _link(actor[1])
    evm = cbor2.loads(rec.get(state_cid))
    storage_root = _link(evm[2])
    needed.update([state_cid, storage_root])
    needed |= rec.seen
    rec2 = Recorder(store)
    raw = read_storage_slot(rec2, storage_root, slot)
    needed |= rec2.seen
    return dict(actor_state_cid=state_cid, storage_root=storage_root, found=raw is not None, raw=raw or b"",
                value=left_pad_32(raw or b""), witness=sorted(needed, key=cid_sort_key))
