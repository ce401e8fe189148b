"""Hand-built state trees for the actor-proof tests (cbor2 + hashlib only; a helper module, not a fixture file), and a restatement of
ipcfp_generate_actor_proofs_resident in Python.

Layouts (DESIGN.md §3), on top of tests/storage_trees.py (HAMTs, StateRoot, child headers) and tests/address_trees.py (InitState,
address_map, the Init path and the HAMT walk of the restatement):
  ActorState   [code, head, sequence, balance, delegated | null], balance in fvm's bigint_ser (empty = 0, else sign byte 0 / 1 and the
               big-endian magnitude), delegated an Address's bytes;
  EVM state    EvmStateV6 [bytecode, bytecode_hash, contract_state, transient, nonce, tombstone] or the V5 5-tuple without transient;
  bytecode     a raw block (CIDv1, codec 0x55, Blake2b-256), whose keccak256 is bytecode_hash.

`prove(...)` states the call's rules independently of the library: the refusals, then per request the header and its ParentStateRoot,
the Init path (once, for non-ID addresses) and the address_map, the actors HAMT, every field, the EVM state of an actor whose code is in
the EVM code set and, with code, the bytecode block and its hash. It returns the proofs (as the fields of api's ActorProof), the
per-proof read sets and their union, or the call's failure (status, index)."""
import functools
import hashlib
import random

import cbor2

from ipc_filecoin_proofs_b200 import _abi as A
from oracle.pyoracle import cid_sort_key, keccak256
from tests import address_trees as R
from tests import storage_trees as T

RAW_PREFIX = bytes.fromhex("0155a0e40220")   # CIDv1, raw, blake2b-256: the bytecode block
ACCOUNT = T.cid_of(b"fil/16/account")
EVM_A = T.cid_of(b"fil/16/evm")              # the code of tests/storage_trees.py's actors
EVM_B = T.cid_of(b"fil/15/evm")
MINER = T.cid_of(b"fil/16/storageminer")
EVM_SETS = {"none": [], "one": [EVM_A], "several": [T.cid_of(b"fil/14/evm"), EVM_B, EVM_A]}


# ------------------------------------------------------------------ builders
def bigint(v):
    """fvm bigint_ser bytes of v."""
    if v == 0:
        return b""
    m = abs(v)
    return (b"\x01" if v < 0 else b"\x00") + m.to_bytes((m.bit_length() + 7) // 8, "big")


def actor_state(code, head, sequence=0, balance=b"", delegated=None):
    return (b"\x85" + T.clink(code) + T.clink(head) + T.head(0, sequence) + T.cbytes(balance) +
            (b"\xf6" if delegated is None else T.cbytes(delegated)))


def evm_state(bytecode_cid, bytecode_hash, contract_state, six=True, nonce=1):
    items = [T.clink(bytecode_cid), T.cbytes(bytecode_hash), T.clink(contract_state)]
    if six:
        items.append(b"\xf6")
    items += [T.head(0, nonce), b"\xf6"]
    return T.head(4, len(items)) + b"".join(items)


def evm_actor(blocks, code, seed, six=True, nonce=3, balance=b"", delegated=None, put_code=True, hash_of=None):
    """An EVM actor with its own bytecode block (kept out of the store when put_code is false; hash_of: the bytes its bytecode_hash is
    taken from, the bytecode itself by default) → ActorState bytes."""
    bytecode = hashlib.sha256(b"code-%d" % seed).digest() * (1 + seed % 40)
    bc = RAW_PREFIX + hashlib.blake2b(bytecode, digest_size=32).digest()
    if put_code:
        blocks[bc] = bytecode
    cs = blocks.put(T.wrap_a3(T.small_map([(bytes(32), b"\x01")])))
    st = blocks.put(evm_state(bc, keccak256(bytecode if hash_of is None else hash_of), cs, six, nonce))
    return actor_state(code, st, seed % 17, balance, delegated)


def account(blocks, seed, balance=b"", delegated=None):
    return actor_state(ACCOUNT, blocks.put(b"\x82\x00" + T.cbytes(b"acct-%d" % seed)), seed % 11, balance, delegated)


def state_tree(blocks, actors, amap=None):
    """A StateRoot whose actors HAMT holds `actors` {id: ActorState bytes} and, when amap {address bytes: id} is given, an Init actor over
    that address_map → StateRoot CID."""
    actors = dict(actors)
    if amap is not None:
        init = R.init_state(T.build_hamt(blocks, {k: T.head(0, v) for k, v in amap.items()}, 5))
        actors[1] = actor_state(T.cid_of(b"fil/16/init"), blocks.put(init))
    return blocks.put(T.state_root(T.build_hamt(blocks, {T.id_address(a): s for a, s in actors.items()}, 5)))


# ------------------------------------------------------------------ the restatement
class Failure(Exception):
    def __init__(self, status, index):
        super().__init__(status, index)
        self.status, self.index = status, index

    def __eq__(self, o):
        return isinstance(o, Failure) and (self.status, self.index) == (o.status, o.index)


def empty_proof(address, status, actor_id=0):
    return dict(address=bytes(address), status=status, actor_id=actor_id, code=bytes(38), head=bytes(38), sequence=0, balance=0,
                delegated=None, is_evm=False, bytecode_cid=bytes(38), bytecode_hash=bytes(32), evm_nonce=0, contract_state=bytes(38),
                bytecode=None)


def _balance(b):
    if not b:
        return 0
    if b[0] > 1 or len(b) - 1 > 32:
        raise R.Fault(A.ERR_DECODE)
    m = int.from_bytes(b[1:], "big")
    return -m if b[0] == 1 else m


def _evm(raw):
    x = _canonical(raw)
    for n in (6, 5):
        if isinstance(x, list) and len(x) == n and isinstance(x[1], bytes) and len(x[1]) == 32 and type(x[n - 2]) is int and 0 <= x[n - 2] < 2 ** 64:
            try:
                return R._link(x[0]), x[1], R._link(x[2]), x[n - 2]
            except R.Fault:
                pass
    raise R.Fault(A.ERR_DECODE)


def _canonical(raw):
    """A DAG-CBOR item in its one accepted encoding (minimal heads, definite lengths, links as the only tag, float64 the only float (the device decoder's rules), nothing after it), else a
    decode fault; checked head by head, without re-encoding. → the decoded item."""
    pos, todo, link = 0, 1, False
    while todo:
        if pos >= len(raw):
            raise R.Fault(A.ERR_DECODE)
        b = raw[pos]
        major, ai = b >> 5, b & 31
        pos += 1
        todo -= 1
        if ai < 24:
            arg = ai
        elif ai < 28:
            k = 1 << (ai - 24)
            if pos + k > len(raw):
                raise R.Fault(A.ERR_DECODE)
            arg = int.from_bytes(raw[pos:pos + k], "big")
            pos += k
            if arg < (24 if k == 1 else 1 << (4 * k)):
                raise R.Fault(A.ERR_DECODE)
        else:
            raise R.Fault(A.ERR_DECODE)
        if link and not (major == 2 and 1 <= arg <= len(raw) - pos and raw[pos] == 0):
            raise R.Fault(A.ERR_DECODE)
        link = False
        if major in (2, 3):
            if arg > len(raw) - pos:
                raise R.Fault(A.ERR_DECODE)
            pos += arg
        elif major == 4:
            todo += arg
        elif major == 5:
            todo += 2 * arg
        elif major == 6:   # a link: tag 42 over bytes that start with the identity multibase 0x00
            if arg != 42:
                raise R.Fault(A.ERR_DECODE)
            todo += 1
            link = True
            continue
        elif major == 7 and not (20 <= ai <= 22 or ai == 27):   # false, true, null, or a float64 with a minimal head
            raise R.Fault(A.ERR_DECODE)
    if pos != len(raw):
        raise R.Fault(A.ERR_DECODE)
    try:
        return cbor2.loads(raw)
    except Exception:   # invalid UTF-8 in a text string
        raise R.Fault(A.ERR_DECODE)


def _hamt_get(rd, root, key, value):
    """address_trees.hamt_get (width 5, every node decoded whole) with _canonical as the strictness check."""
    h = int.from_bytes(hashlib.sha256(key).digest(), "big")
    raw = rd.get(root)
    consumed = 0
    while True:
        node = _canonical(raw)
        if not (isinstance(node, list) and len(node) == 2 and isinstance(node[0], bytes) and len(node[0]) <= 32 and isinstance(node[1], list)):
            raise R.Fault(A.ERR_DECODE)
        bf = int.from_bytes(node[0], "big")
        for p in node[1]:
            if isinstance(p, cbor2.CBORTag):
                R._link(p)
            elif isinstance(p, list):
                for e in p:
                    if not (isinstance(e, list) and len(e) == 2 and isinstance(e[0], bytes)):
                        raise R.Fault(A.ERR_DECODE)
                    value(e[1])
            else:
                raise R.Fault(A.ERR_DECODE)
        if bin(bf).count("1") != len(node[1]) or consumed + 5 > 256:
            raise R.Fault(A.ERR_DECODE)
        idx = (h >> (256 - consumed - 5)) & 31
        consumed += 5
        if not (bf >> idx) & 1:
            return None
        p = node[1][bin(bf & ((1 << idx) - 1)).count("1")]
        if isinstance(p, cbor2.CBORTag):
            raw = rd.get(R._link(p))
            continue
        return next((v for k, v in p if k == key), None)


def _init_path(rd, sroot):
    """address_trees.init_path with _canonical and _hamt_get: the address_map root."""
    sr = _canonical(rd.get(sroot))
    if not (isinstance(sr, list) and len(sr) == 3) or R._uint(sr[0]) > 5:
        raise R.Fault(A.ERR_DECODE)
    actors = R._link(sr[1])
    R._link(sr[2])
    actor = _hamt_get(rd, actors, R.INIT_KEY, R._actor_state)
    if actor is None:
        raise R.Fault(A.ERR_ACTOR_NOT_FOUND)
    st = _canonical(rd.get(R._actor_state(actor)))
    if not (isinstance(st, list) and len(st) == 3 and isinstance(st[2], str)):
        raise R.Fault(A.ERR_DECODE)
    R._uint(st[1])
    return R._link(st[0])


def _one(rd, child, sroot, a, amap, init_fault, evm, with_code):
    hdr = cbor2.loads(rd.get(child))
    if bytes(hdr[8].value[1:]) != sroot:
        raise R.Fault(A.ERR_STATE_ROOT_MISMATCH)
    if a[0] == 0:
        aid = R._leb_read(a[1:])[0]
    else:
        if init_fault is not None:
            raise init_fault
        aid = _hamt_get(rd, amap, a, R._uint)
        if aid is None:
            return empty_proof(a, A.ACTOR_NO_ADDRESS)
    sr = _canonical(rd.get(sroot))
    if not (isinstance(sr, list) and len(sr) == 3) or R._uint(sr[0]) > 5:
        raise R.Fault(A.ERR_DECODE)
    actors = R._link(sr[1])
    R._link(sr[2])
    st = _hamt_get(rd, actors, T.id_address(aid), R._actor_state)
    if st is None:
        return empty_proof(a, A.ACTOR_NO_ACTOR, aid)
    p = empty_proof(a, A.ACTOR_FOUND, aid)
    p.update(code=R._link(st[0]), head=R._link(st[1]), sequence=st[2], balance=_balance(st[3]))
    if st[4] is not None:
        if not R.address_valid(st[4]):
            raise R.Fault(A.ERR_DECODE)
        p["delegated"] = bytes(st[4])
    if p["code"] in evm:
        bc, h, cs, nonce = _evm(rd.get(p["head"]))
        p.update(is_evm=True, bytecode_cid=bc, bytecode_hash=h, contract_state=cs, evm_nonce=nonce)
        if with_code:
            code = rd.get(bc)
            if keccak256(code) != h:
                raise R.Fault(A.ERR_DECODE)
            p["bytecode"] = code
    return p


def prove(blocks, child, sroot, addrs, evm=(), with_code=False):
    """→ (proofs, per-proof read sets (sorted CIDs), union (sorted CIDs)), or raises Failure(status, index)."""
    child, sroot, evm = bytes(child), bytes(sroot), [bytes(c) for c in evm]
    addrs = [bytes(a) for a in addrs]
    if len(addrs) > A.ACTOR_MAX:
        raise Failure(A.ERR_INVALID_ARG, None)
    for i, a in enumerate(addrs):
        if not R.address_valid(a):
            raise Failure(A.ERR_INVALID_ARG, i)
    amap, init_fault, init_read = None, None, set()
    if any(a[0] != 0 for a in addrs):
        rd = R.Reader(blocks)
        try:
            amap = _init_path(rd, sroot)
        except R.Fault as f:
            init_fault = R.Fault(f.status)
        init_read = rd.read
    proofs, lists, union = [], [], set()
    for i, a in enumerate(addrs):
        rd = R.Reader(blocks)
        try:
            proofs.append(_one(rd, child, sroot, a, amap, init_fault, evm, with_code))
        except R.Fault as f:
            raise Failure(f.status, i)
        read = set(rd.read) | (init_read if a[0] != 0 else set())
        lists.append(sorted(read, key=cid_sort_key))
        union |= read
    return proofs, lists, sorted(union, key=cid_sort_key)


def read_set(blocks, child, sroot, addrs, evm=(), with_code=False):
    """The blocks the call reads, as far as the blocks present go: what a fetch loop from an empty store ends up holding."""
    return prove(blocks, child, sroot, addrs, evm, with_code)[2]


# ------------------------------------------------------------------ the world
class Tree:
    """One state tree behind its own child header: `root`, `addrs` (the requests of its GPU case) and `status` (the call's failure
    status, or None)."""

    def __init__(self, name, root, addrs, status=None, with_code=False, evm="several"):
        self.name, self.root, self.addrs, self.status, self.with_code, self.evm = name, root, addrs, status, with_code, evm


SIZES = (1, 1000, 100000)
BALANCES = {"zero": b"", "one-byte": bigint(5), "twelve-bytes": bigint(2 ** 95 - 7), "thirty-two-bytes": b"\x00" + b"\xff" * 32,
            "negative": bigint(-(2 ** 90 + 3)), "plus-zero": b"\x00", "minus-zero": b"\x01\x00\x00", "leading-zeros": b"\x00\x00\x00\x07"}


@functools.lru_cache(maxsize=None)
def blocks_and_trees():
    """Every tree over ONE block set → (Blocks, [Tree], main) with main = {"actors": {id: kind}, "amap": {address: id}}."""
    blocks = T.Blocks()
    rng = random.Random(77)
    trees = []
    actors, kinds = {}, {}

    def add(aid, st, kind):
        actors[aid] = st
        kinds[aid] = kind

    for i, (name, b) in enumerate(BALANCES.items()):
        add(100 + i, account(blocks, i, b), "balance-" + name)
    f410 = R.delegated(10, rng.randbytes(20))
    add(120, account(blocks, 20, bigint(7), delegated=f410), "delegated")
    add(121, evm_actor(blocks, EVM_A, 21, six=True, balance=bigint(10 ** 18), delegated=R.delegated(10, rng.randbytes(20))), "evm-v6")
    add(122, evm_actor(blocks, EVM_A, 22, six=False, nonce=0), "evm-v5")
    add(123, evm_actor(blocks, EVM_B, 23, six=True, nonce=2 ** 64 - 1), "evm-b")
    add(124, actor_state(MINER, blocks.put(b"\x80"), 4, bigint(1)), "miner")
    add(0, account(blocks, 30), "id-0")
    add(2 ** 64 - 1, account(blocks, 31, bigint(1)), "id-max")
    amap = {}
    for kind, aid in zip(R.KINDS, (100, 120, 121, 122, 123)):
        amap[R.random_address(rng, kind)] = aid
    amap[R.delegated(10, rng.randbytes(20))] = 5555           # in the map, not an actor
    amap[R.delegated(32, b"")] = 2 ** 64 - 1
    main = dict(actors=dict(kinds), amap=dict(amap))
    absent_addrs = [R.random_address(rng, k) for k in R.KINDS]
    ids = [R.id_addr(a) for a in actors] + [R.id_addr(a) for a in (1, 2, 999, 2 ** 63)]
    main_root = state_tree(blocks, actors, amap)
    main["root"] = main_root
    trees.append(Tree("main", main_root, ids + list(amap) + absent_addrs))
    trees.append(Tree("main-code", main_root, ids + list(amap), with_code=True))
    # forgeries of main: well-formed trees whose every block hashes to its CID, each differing from main in one claim (a false absence of
    # an actor or an address, another balance, another EVM nonce and storage root)
    forged = {"forged-no-actor": {k: v for k, v in actors.items() if k != 121},
              "forged-balance": {**actors, 100: account(blocks, 0, bigint(10 ** 30))},
              "forged-evm": {**actors, 122: evm_actor(blocks, EVM_A, 22, six=False, nonce=9)}}
    for name, acts in forged.items():
        trees.append(Tree(name, state_tree(blocks, acts, amap), ids + list(amap), with_code=True))
    trees.append(Tree("forged-no-address", state_tree(blocks, actors, {k: v for k, v in amap.items() if v != 122}), ids + list(amap), with_code=True))
    # size worlds: 1 actor (no Init actor, ID requests only) and fillers around the main actors
    for n in SIZES:
        if n == 1:
            root = state_tree(blocks, {0: account(blocks, 30)})
            trees.append(Tree("actors-1", root, [R.id_addr(0), R.id_addr(7)]))
            continue
        big = dict(actors)
        frng = random.Random(n)
        while len(big) < n:   # (heads are never read: an account's head is not EVM state)
            big[frng.randrange(2, 2 ** frng.choice((16, 32, 64)))] = actor_state(ACCOUNT, T.cid_of(b"filler-%d" % len(big)), len(big) % 5)
        root = state_tree(blocks, big, amap)
        pick = frng.sample(sorted(big), 200)
        trees.append(Tree(f"actors-{n}", root, [R.id_addr(a) for a in pick] + ids + list(amap) + absent_addrs))
    # faults: each in its own tree, requested after a good actor so that the failure's index is 1
    good = {100: actors[100]}
    for name, st, status, with_code in (
            ("sign-byte-2", account(blocks, 50, b"\x02\x01"), A.ERR_DECODE, False),
            ("magnitude-33-bytes", account(blocks, 51, b"\x00" + b"\x01" * 33), A.ERR_DECODE, False),
            ("delegated-not-an-address", account(blocks, 52, delegated=b"\x05" + bytes(20)), A.ERR_DECODE, False),
            ("evm-head-not-evm-state", actor_state(EVM_A, blocks.put(b"\x82\x00\x00"), 1), A.ERR_DECODE, False),
            ("evm-head-missing", actor_state(EVM_A, T.cid_of(b"never stored"), 1), A.ERR_MISSING_BLOCK, False),
            ("bytecode-missing", evm_actor(blocks, EVM_A, 53, put_code=False), A.ERR_MISSING_BLOCK, True),
            ("bytecode-hash-mismatch", evm_actor(blocks, EVM_A, 54, hash_of=b"other"), A.ERR_DECODE, True)):
        root = state_tree(blocks, {**good, 200: st})
        trees.append(Tree(name, root, [R.id_addr(100), R.id_addr(200)], status, with_code))
    for name, st in (("bytecode-missing-without-code", evm_actor(blocks, EVM_A, 55, put_code=False)),
                     ("bytecode-hash-mismatch-without-code", evm_actor(blocks, EVM_A, 56, hash_of=b"other"))):
        trees.append(Tree(name, state_tree(blocks, {**good, 200: st}), [R.id_addr(100), R.id_addr(200)]))
    no_init = state_tree(blocks, good)
    trees.append(Tree("no-init-actor", no_init, [R.id_addr(100), next(iter(amap))], A.ERR_ACTOR_NOT_FOUND))
    trees.append(Tree("no-init-actor-ids-only", no_init, [R.id_addr(100), R.id_addr(3)]))
    # the deepest two-HAMT path: address_map and actors HAMT chains at the depth limit (51 nodes each)
    key = R.delegated(10, rng.randbytes(20))
    deep_id = 2 ** 64 - 2
    amap_top = T.build_chain(blocks, key, T.head(0, deep_id), 5, 51)
    init_st = actor_state(T.cid_of(b"fil/16/init"), blocks.put(R.init_state(amap_top)))
    akey = T.id_address(deep_id)
    chain = T.build_chain(blocks, akey, evm_actor(blocks, EVM_A, 57), 5, 51, siblings={0: [(T.id_address(1), init_st)]})
    deep_root = blocks.put(T.state_root(chain))
    trees.append(Tree("deep", deep_root, [key, R.id_addr(deep_id)], with_code=True))
    # … and the Init actor at the bottom of a 51-node actors-HAMT chain, the actor a sibling at its top: the Init path's own list at the
    # depth limit, joined with the address_map chain's
    ikey = T.id_address(1)
    actor_st = evm_actor(blocks, EVM_A, 58)
    assert T.hash_index(akey, 0, 5) != T.hash_index(ikey, 0, 5)
    chain = T.build_chain(blocks, ikey, init_st, 5, 51, siblings={0: [(akey, actor_st)]})
    trees.append(Tree("deep-init", blocks.put(T.state_root(chain)), [key, R.id_addr(deep_id)], with_code=True))
    return blocks, trees, main


def world(ts):
    """(Blocks with every tree's child header, {name: Tree} with .child and .tip set, main, Flat)."""
    blocks, trees, main = blocks_and_trees()
    blocks = T.Blocks(blocks)
    for t in trees:
        hdr, c = T.child_header(ts, t.root)
        blocks[c] = hdr
        t.child = c
    flat = T.Flat(blocks)
    for t in trees:
        t.tip = T.tipset(ts, flat.arrays(), t.child, t.root)
    return blocks, {t.name: t for t in trees}, main, flat
