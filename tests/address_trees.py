"""Hand-built state trees with an Init actor for the address-resolution tests (cbor2 + hashlib only; a helper module, not a fixture
file), and a restatement of ipcfp_resolve_addresses in Python.

Layouts (DESIGN.md §3), on top of tests/storage_trees.py's HAMT, ActorState and StateRoot builders:
  InitState      [address_map: link, next_id: uint, network_name: text], exactly these three items;
  address_map    HAMT at width 5, key Address::to_bytes(), value the ActorID as one CBOR unsigned integer;
  Init actor     ID 1 in the actors HAMT (key 00 01).
Address bytes follow fvm_shared: protocol 0 = minimal LEB128 u64; 1 and 2 = 20 bytes; 3 = 48 bytes; 4 = minimal LEB128 namespace followed
by at most 54 bytes.

`resolve(blocks, state_root, addresses)` states the call's rules independently of the library: the Init path once, then one walk per
non-ID address, with the decode contract's strictness (minimal heads, exact tuples, no trailing bytes, the 256-bit depth limit). It
returns the same five things the call does: actor IDs, per-address status, init status, the missing CIDs and the read set."""
import functools
import hashlib
import io
import random

import cbor2

from ipc_filecoin_proofs_b200 import _abi as A
from oracle.pyoracle import cid_sort_key
from tests import storage_trees as T

HAMT_BW = 5
INIT_KEY = b"\x00\x01"
VALUES = (0, 23, 24, 255, 256, 65535, 2 ** 32, 2 ** 64 - 1)   # every CBOR head size of an ActorID


# ------------------------------------------------------------------ addresses
def leb(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def id_addr(v):
    return b"\x00" + leb(v)


def delegated(ns, sub):
    return b"\x04" + leb(ns) + bytes(sub)


def eth_masked_id(v):
    return b"\xff" + bytes(11) + v.to_bytes(8, "big")


def address_valid(a):
    """fvm_shared Address::from_bytes accepts a."""
    if not a or len(a) > A.ADDRESS_MAX:
        return False
    p, rest = a[0], a[1:]
    if p == 0:
        r = _leb_read(rest)
        return r is not None and r[1] == len(rest)
    if p in (1, 2):
        return len(rest) == 20
    if p == 3:
        return len(rest) == 48
    if p == 4:
        r = _leb_read(rest)
        return r is not None and len(rest) - r[1] <= 54
    return False


def _leb_read(b):
    v = 0
    for i, c in enumerate(b[:10]):
        if i == 9 and (c & 0x7F) > 1:
            return None
        v |= (c & 0x7F) << (7 * i)
        if not c & 0x80:
            if i > 0 and c == 0:
                return None
            return v, i + 1
    return None


B32 = "abcdefghijklmnopqrstuvwxyz234567"


def b32(data):
    bits = "".join(f"{x:08b}" for x in data)
    bits += "0" * (-len(bits) % 5)
    return "".join(B32[int(bits[i:i + 5], 2)] for i in range(0, len(bits), 5))


def address_text(a, net="f"):
    """The text form of Address bytes a (the inverse of ipcfp_address_parse)."""
    p = a[0]
    if p == 0:
        return f"{net}0{_leb_read(a[1:])[0]}"
    ck = hashlib.blake2b(a, digest_size=4).digest()
    if p == 4:
        ns, used = _leb_read(a[1:])
        return f"{net}4{ns}f{b32(a[1 + used:] + ck)}"
    return f"{net}{p}{b32(a[1:] + ck)}"


def random_address(rng, kind):
    if kind in (1, 2):
        return bytes([kind]) + rng.randbytes(20)
    if kind == 3:
        return b"\x03" + rng.randbytes(48)
    if kind == "f410":
        return delegated(10, rng.randbytes(20))
    ns = rng.choice((0, 1, 9, 11, 127, 128, 2 ** 32, 2 ** 63, 2 ** 64 - 1))
    return delegated(ns, rng.randbytes(rng.randrange(55)))


KINDS = (1, 2, 3, "f410", "f4")


# ------------------------------------------------------------------ builders
def init_state(address_map, next_id=1000, name="testnet"):
    return b"\x83" + T.clink(address_map) + T.head(0, next_id) + T.ctext(name)


def state_tree(blocks, entries, init=None, others=(), version=5):
    """A StateRoot whose actors HAMT holds the Init actor (ActorState over the InitState `init`, or a canonical one over the address_map
    of `entries` {address bytes: actor id}) and `others` {actor id: ActorState bytes}. init=False: no Init actor. → StateRoot CID."""
    actors = dict(others)
    if init is not False:
        if init is None:
            init = init_state(T.build_hamt(blocks, {k: T.head(0, v) for k, v in entries.items()}, HAMT_BW))
        actors[1] = T.actor_state(blocks.put(init))
    aroot = T.build_hamt(blocks, {T.id_address(a): s for a, s in actors.items()}, HAMT_BW)
    return blocks.put(T.state_root(aroot, version))


# ------------------------------------------------------------------ the restatement
class Fault(Exception):
    def __init__(self, status, cid=None):
        super().__init__(status)
        self.status, self.cid = status, cid


def _strict(raw):
    """A DAG-CBOR item in its one accepted encoding (minimal heads, definite lengths, nothing after it), else a decode fault."""
    try:
        fp = io.BytesIO(raw)
        x = cbor2.CBORDecoder(fp).decode()
        if fp.tell() != len(raw) or cbor2.dumps(x) != raw:
            raise ValueError
    except Exception:
        raise Fault(A.ERR_DECODE)
    return x


def _link(x):
    if not (isinstance(x, cbor2.CBORTag) and x.tag == 42 and isinstance(x.value, bytes) and len(x.value) == 39 and x.value[:2] == b"\x00\x01"):
        raise Fault(A.ERR_DECODE)
    return x.value[1:]


def _uint(x):
    if type(x) is not int or not 0 <= x < 2 ** 64:
        raise Fault(A.ERR_DECODE)
    return x


def _actor_state(v):
    if not (isinstance(v, list) and len(v) == 5):
        raise Fault(A.ERR_DECODE)
    _link(v[0])
    st = _link(v[1])
    _uint(v[2])
    if not isinstance(v[3], bytes) or not (v[4] is None or isinstance(v[4], bytes)):
        raise Fault(A.ERR_DECODE)
    return st


class Reader:
    def __init__(self, blocks):
        self.blocks, self.read = blocks, set()

    def get(self, cid):
        cid = bytes(cid)
        if cid not in self.blocks:
            raise Fault(A.ERR_MISSING_BLOCK, cid)
        self.read.add(cid)
        return self.blocks[cid]


def hamt_get(rd, root, key, value):
    """fvm_ipld_hamt Hamt::get at width 5 with every node decoded whole (each value through `value`, which raises on a bad one)."""
    h = int.from_bytes(hashlib.sha256(key).digest(), "big")
    raw = rd.get(root)
    consumed = 0
    while True:
        node = _strict(raw)
        if not (isinstance(node, list) and len(node) == 2 and isinstance(node[0], bytes) and len(node[0]) <= 32 and isinstance(node[1], list)):
            raise Fault(A.ERR_DECODE)
        bf = int.from_bytes(node[0], "big")
        hit = None
        for p in node[1]:
            if isinstance(p, cbor2.CBORTag):
                _link(p)
            elif isinstance(p, list):
                for e in p:
                    if not (isinstance(e, list) and len(e) == 2 and isinstance(e[0], bytes)):
                        raise Fault(A.ERR_DECODE)
                    value(e[1])
            else:
                raise Fault(A.ERR_DECODE)
        if bin(bf).count("1") != len(node[1]):
            raise Fault(A.ERR_DECODE)
        if consumed + HAMT_BW > 256:
            raise Fault(A.ERR_DECODE)
        idx = (h >> (256 - consumed - HAMT_BW)) & 31
        consumed += HAMT_BW
        if not (bf >> idx) & 1:
            return None
        p = node[1][bin(bf & ((1 << idx) - 1)).count("1")]
        if isinstance(p, cbor2.CBORTag):
            raw = rd.get(_link(p))
            continue
        for k, v in p:
            if k == key:
                hit = v
                break
        return hit


def init_path(rd, state_root):
    sr = _strict(rd.get(state_root))
    if not (isinstance(sr, list) and len(sr) == 3) or _uint(sr[0]) > 5:
        raise Fault(A.ERR_DECODE)
    actors = _link(sr[1])
    _link(sr[2])
    actor = hamt_get(rd, actors, INIT_KEY, _actor_state)
    if actor is None:
        raise Fault(A.ERR_ACTOR_NOT_FOUND)
    st = _strict(rd.get(_actor_state(actor)))
    if not (isinstance(st, list) and len(st) == 3 and isinstance(st[2], str)):
        raise Fault(A.ERR_DECODE)
    _uint(st[1])
    return _link(st[0])


def resolve(blocks, state_root, addresses):
    """→ (ids, status, init_status, missing (sorted unique CIDs), read set (sorted CIDs))."""
    rd = Reader(blocks)
    missing = set()
    try:
        amap, init_status = init_path(rd, bytes(state_root)), A.OK
    except Fault as f:
        amap, init_status = None, f.status
        if f.cid:
            missing.add(f.cid)
    ids, status = [], []
    for a in addresses:
        a = bytes(a)
        if not address_valid(a):
            ids.append(0), status.append(A.ERR_INVALID_ARG)
        elif a[0] == 0:
            ids.append(_leb_read(a[1:])[0]), status.append(A.OK)
        elif init_status != A.OK:
            ids.append(0), status.append(init_status)
        else:
            try:
                v = hamt_get(rd, amap, a, _uint)
                ids.append(0 if v is None else v), status.append(A.ERR_ACTOR_NOT_FOUND if v is None else A.OK)
            except Fault as f:
                ids.append(0), status.append(f.status)
                if f.cid:
                    missing.add(f.cid)
    return ids, status, init_status, sorted(missing, key=cid_sort_key), sorted(rd.read, key=cid_sort_key)


# ------------------------------------------------------------------ the catalogue
class Case:
    """One ipcfp_resolve_addresses call: `root` (StateRoot CID), `addrs` (bytes each) and `truth` ({address: id} the builder put in the
    map; None where the case's outcome comes from the restatement alone)."""

    def __init__(self, name, root, addrs, truth=None):
        self.name, self.root, self.addrs, self.truth = name, root, addrs, truth


SIZES = (1, 3, 200, 5000, 100000)


def _entries(rng, n):
    out = {}
    while len(out) < n:
        a = random_address(rng, KINDS[len(out) % len(KINDS)])
        out[a] = VALUES[len(out) % len(VALUES)] if len(out) < 4 * len(VALUES) else rng.randrange(2 ** rng.choice((10, 20, 40, 64)))
    return out


def _absent(rng, entries, k):
    return [random_address(rng, KINDS[i % len(KINDS)]) for i in range(k)]


def _mix(rng, entries, n_present=120, n_absent=30, n_dup=10):
    keys = list(entries)
    pick = keys if len(keys) <= n_present else rng.sample(keys, n_present)
    pick = pick + [rng.choice(pick) for _ in range(n_dup)] + _absent(rng, entries, n_absent)
    pick += [id_addr(v) for v in VALUES[:4]]
    rng.shuffle(pick)
    return pick


def _hidx(key, level=0):
    return T.hash_index(key, level, HAMT_BW)


@functools.lru_cache(maxsize=None)
def world():
    """Every GPU case over ONE block set → (Blocks, [Case], {size: (root, entries)})."""
    blocks = T.Blocks()
    cases = []
    maps = {}
    rng = random.Random(2024)
    others = {1000 + i: T.actor_state(T.cid_of(b"evm-%d" % i)) for i in range(20)}
    for n in SIZES:
        ent = _entries(random.Random(n), n)
        root = state_tree(blocks, ent, others=others)
        maps[n] = (root, ent)
        cases.append(Case(f"map-{n}", root, _mix(random.Random(n + 1), ent), ent))

    # buckets of 1-3 entries at one slot, absent keys in that bucket's slot, and a key that differs from one in the bucket only in length
    for size in (1, 2, 3):
        while True:
            base = delegated(10, rng.randbytes(20))
            short = base[:-1]
            if _hidx(short) == _hidx(base):
                break
        ks = [base]
        while len(ks) < size:
            k = delegated(10, rng.randbytes(20))
            if _hidx(k) == _hidx(base):
                ks.append(k)
        absent_same_slot = next(k for k in (delegated(10, rng.randbytes(20)) for _ in range(10 ** 5)) if _hidx(k) == _hidx(base))
        ent = {k: VALUES[i + 5] for i, k in enumerate(ks)}
        node = T.hamt_node({_hidx(base): [(k, T.head(0, ent[k])) for k in sorted(ks)]})
        root = state_tree(blocks, {}, init=init_state(blocks.put(node)))
        clear = next(k for k in (delegated(10, rng.randbytes(20)) for _ in range(10 ** 5)) if _hidx(k) != _hidx(base))
        cases.append(Case(f"bucket-{size}", root, ks + [short, base + b"\x00", absent_same_slot, clear], ent))

    # a width-5 chain to the depth limit (51 levels: present, key's bit clear) and one level past it
    key = delegated(10, rng.randbytes(20))
    for n, present, name in ((51, True, "chain-51"), (51, False, "chain-51-absent"), (52, True, "chain-52")):
        top = T.build_chain(blocks, key, T.head(0, 2 ** 64 - 1), HAMT_BW, n, present=present)
        root = state_tree(blocks, {}, init=init_state(top))
        cases.append(Case(name, root, [key, delegated(10, rng.randbytes(20))], {key: 2 ** 64 - 1} if n == 51 and present else None))

    # ID addresses, masked-ID eth addresses and invalid bytes: settled without a read of the map
    small_root, small = maps[3]
    ids = [id_addr(v) for v in VALUES] + [id_addr(1), id_addr(1000)]
    invalid = [b"", b"\x05" + bytes(20), b"\x01" + bytes(19), b"\x02" + bytes(21), b"\x03" + bytes(47), b"\x00\x80\x00", b"\x00\x80",
               b"\x00" + b"\xff" * 9 + b"\x02", delegated(10, bytes(55)), b"\x04\x80\x00" + bytes(20), b"\x04"]
    cases.append(Case("ids-and-invalid", small_root, ids + invalid + list(small), small))

    # faults of the Init path and of the map
    good_map = T.build_hamt(blocks, {k: T.head(0, v) for k, v in small.items()}, HAMT_BW)
    amap_link = T.clink(good_map)
    for name, init in (("init-4-tuple", b"\x84" + amap_link + T.head(0, 1) + T.ctext("n") + b"\x00"),
                       ("init-2-tuple", b"\x82" + amap_link + T.head(0, 1)),
                       ("init-trailing", init_state(good_map) + b"\x00"),
                       ("init-map-not-link", b"\x83" + T.cbytes(good_map) + T.head(0, 1) + T.ctext("n")),
                       ("init-next-id-negative", b"\x83" + amap_link + b"\x20" + T.ctext("n")),
                       ("init-name-bytes", b"\x83" + amap_link + T.head(0, 1) + T.cbytes(b"n")),
                       ("init-not-array", T.cbytes(b"init"))):
        cases.append(Case(name, state_tree(blocks, {}, init=init), list(small) + [id_addr(7)]))
    cases.append(Case("init-absent", state_tree(blocks, {}, init=False, others=others), list(small) + [id_addr(7)]))
    cases.append(Case("state-root-version-6", state_tree(blocks, small, version=6), list(small)))
    sr_bad = blocks.put(b"\x84" + T.head(0, 5) + T.clink(good_map) + T.clink(good_map) + b"\x00")
    cases.append(Case("state-root-4-tuple", sr_bad, list(small)))
    k = delegated(10, rng.randbytes(20))
    for name, enc in (("value-negative", b"\x20"), ("value-bytes", T.cbytes(b"\x01")), ("value-nonminimal", b"\x18\x05"),
                      ("value-u64-nonminimal", b"\x1b" + (7).to_bytes(8, "big")), ("value-text", T.ctext("7")), ("value-null", b"\xf6")):
        node = T.hamt_node({_hidx(k): [(k, enc)]})
        cases.append(Case(name, state_tree(blocks, {}, init=init_state(blocks.put(node))), [k, delegated(10, rng.randbytes(20))]))
    return blocks, cases, maps


def mutations(blocks, root, rng, n):
    """n seeded truncations and bit flips of the blocks on root's read set → [(name, {cid: new bytes})] (same CIDs: stores of such
    sets are made without CID checks)."""
    _, _, _, _, read = resolve(blocks, root, [])
    out = []
    for i in range(n):
        c = read[i % len(read)]
        b = bytearray(blocks[c])
        if i % 2:
            b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            out.append((f"flip-{i}", {c: bytes(b)}))
        else:
            out.append((f"trunc-{i}", {c: bytes(b[:rng.randrange(len(b))])}))
    return out
