"""State trees for the storage-path campaign on the GPU (a helper module, not a fixture file; tests/storage_trees.py's builders, cbor2
and hashlib only), the fault variants, and the hostile proof lists of the path verifier with their expected verdicts.

One state tree holds:
  * the seeded random campaign (storage_paths.case) over actors 0, 1 000, 2^63 and 2^64 - 1, whose storage HAMTs have bit widths 1, 5,
    8 and 5; actor SHARER has actor 1 000's EVM state, so it reads the same storage trie;
  * storage_paths.edges() over edge_storage() as actor EDGE (width 3), with deep_path() beside them: 32 ARRAY steps and 256 words, the
    largest number of fixed specs a path can have (288);
  * HAND (width 2): a hand-laid contract for the fault and verifier cases, among 400 filler slots, so that a lookup visits three to
    six nodes:
        0 uint256[] arr (6)     1 string s33     2 string s65     3 string s100     4 bytes[] list (a 40-byte and a short element)
        5 string short          6 Pair pair {uint256 x; uint256 y}
A second tree (variant 1) differs only in HAND: s33 holds 65 bytes and arr one element more.

The fault variants drop one HAMT node of HAND's trie and replace another with 0xff bytes (a node that does not decode), placed so
that one path meets both faults, once with the missing node first in expanded order and once with the undecodable one first."""
import functools
import random

import cbor2

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200.api import StoragePath
from tests import storage_paths as SP
from tests import storage_trees as T

ACTORS = (0, 1000, 2 ** 63, 2 ** 64 - 1)
WIDTH = {0: 1, 1000: 5, 2 ** 63: 8, 2 ** 64 - 1: 5, SP.EDGE_ACTOR: 3, 5000: 2}
SHARER = 1001
EDGE = SP.EDGE_ACTOR
HAND = 5000
ABSENT = 999                 # no such actor in the tree
CAMPAIGN_SEED, CAMPAIGN_N = 20261019, 600
ZERO = SP.ZERO


def _p(n):
    return SP.b32(n)


def _elem(base, i):
    return SP.b32(SP.u256(SP.keccak256(_p(base))) + i)


def deep_path():
    """32 ARRAY steps (index 1 of 2 each) and 256 words: 32 length words + 256 value words = 288 fixed specs"""
    return StoragePath(EDGE, 77, [(A.PATH_ARRAY, b"", 1, 1, 0)] * A.PATH_MAX_STEPS, A.PATH_WORDS, A.PATH_MAX_WORDS)


def _hand_storage(variant):
    rng = random.Random(5000 + variant)
    st = {rng.randbytes(32): rng.randbytes(32) for _ in range(400)}
    arr = [rng.randrange(SP.M) for _ in range(6 + variant)]
    st[_p(0)] = SP.b32(len(arr))
    for i, v in enumerate(arr):
        st[_elem(0, i)] = SP.b32(v)
    text = lambda n: bytes(rng.randrange(32, 127) for _ in range(n))
    for slot, n in ((1, 65 if variant else 33), (2, 65), (3, 100)):
        st.update(SP.encode_string(_p(slot), text(n)))
    st[_p(4)] = SP.b32(2)
    st.update(SP.encode_string(_elem(4, 0), text(40)))
    st.update(SP.encode_string(_elem(4, 1), b"el"))
    st.update(SP.encode_string(_p(5), b"short"))
    st[_p(6)], st[_p(7)] = SP.b32(6), SP.b32(7)
    return st


def hand_paths():
    """{name: StoragePath} over HAND"""
    P = lambda slot: StoragePath(HAND, slot)
    out = {f"arr[{i}]": P(0).array(i) for i in range(8)}
    out.update({"s33": P(1).bytes(), "s65": P(2).bytes(), "s100": P(3).bytes(), "list[0]": P(4).array(0).bytes(),
                "list[1]": P(4).array(1).bytes(), "list[2]": P(4).array(2).bytes(), "short": P(5).bytes(), "pair": P(6).words(2),
                "pair.y": P(6).field(1), "absent": P(123456).words(3)})
    return out


class World:
    """storage {actor: {slot: word}} (SHARER's dict is actor 1 000's), campaign [StoragePath], edges [StoragePath], hand {name:
    StoragePath}, blocks (T.Blocks, no child header), roots {actor: storage HAMT root}."""

    def read(self, actor):
        st = self.storage.get(actor, {})
        return lambda slot: st.get(bytes(slot), ZERO)

    def expected(self, path):
        """(specs, status, value, slot, byte offset) of storage_paths.expand over the path's actor's dict"""
        return SP.expand(path, self.read(path.actor_id))

    def tip(self, ts):
        """(Flat, tipset) of this tree behind ts's child header"""
        blocks = T.Blocks(self.blocks)
        hdr, c = T.child_header(ts, self.state_root)
        blocks[c] = hdr
        flat = T.Flat(blocks)
        return flat, T.tipset(ts, flat.arrays(), c, self.state_root)


@functools.lru_cache(maxsize=None)
def build(variant=0):
    """The campaign tree (variant 0) or its second version (variant 1: HAND's s33 at 65 bytes, arr one element longer)."""
    w = World()
    rng = random.Random(CAMPAIGN_SEED)
    storage = {a: {} for a in ACTORS}
    storage[SHARER] = storage[1000]
    w.campaign = [SP.case(rng, storage, ACTORS + (SHARER,)) for _ in range(CAMPAIGN_N)]
    w.edges = SP.edges()
    storage[EDGE] = SP.edge_storage(w.edges)
    deep = deep_path()
    lengths, values, _, _ = SP.derive(deep)
    for s in lengths:
        storage[EDGE][s] = SP.b32(2)
    for k, s in enumerate(values):
        storage[EDGE][s] = SP.b32(k * 0x0101 + 1)
    storage[HAND] = _hand_storage(variant)
    w.storage, w.hand = storage, hand_paths()
    w.blocks = blocks = T.Blocks()
    w.roots, w.contract_states, states = {}, {}, {}
    for a in ACTORS + (EDGE, HAND):
        bw = WIDTH[a]
        w.roots[a] = T.build_hamt(blocks, {s: T.u8vec(v) for s, v in storage[a].items()}, bw)
        w.contract_states[a] = blocks.put(T.wrap_b1(w.roots[a], bw))
        states[a] = blocks.put(T.evm_state(w.contract_states[a]))
    states[SHARER] = states[1000]
    actors = {T.id_address(a): T.actor_state(s, a % 5) for a, s in states.items()}
    w.state_root = blocks.put(T.state_root(T.build_hamt(blocks, actors, 5)))
    return w


def lookup_nodes(blocks, root, key, bw):
    """CIDs of the HAMT nodes a lookup of key visits from root"""
    out, node, level = [root], cbor2.loads(blocks[root]), 0
    while True:
        i = T.hash_index(key, level, bw)
        bf = int.from_bytes(node[0], "big")
        if not (bf >> i) & 1:
            return out
        p = node[1][bin(bf & ((1 << i) - 1)).count("1")]
        if not isinstance(p, cbor2.CBORTag):
            return out
        cid = bytes(p.value[1:])
        out.append(cid)
        node, level = cbor2.loads(blocks[cid]), level + 1


# ------------------------------------------------------------------ fault variants
# (name, path name in hand_paths(), a, b): the path meets a fault at expanded spec a and another at spec b > a
FAULT_PAIRS = (("len+value", "arr[2]", 0, 1),      # both in wave 1
               ("data+data", "s100", 1, 3),        # both in wave 2
               ("len+data", "list[0]", 0, 2))      # wave 1, then wave 2
FAULT_NAMES = tuple(f"{name}:{first}-first" for name, _, _, _ in FAULT_PAIRS for first in ("missing", "decode"))
ABSENT_NAMES = ("wave2-missing-then-absent", "absent-then-wave2-missing")
# the hostile proof lists of the path verifier, in hostile_lists' order
HOSTILE_NAMES = ("honest-shuffled", "honest+world", "empty", "tampered-header-before", "tampered-header-after", "tampered-header-only",
                 "tampered-length-before", "tampered-length-after", "tampered-length-only", "tampered-data-before",
                 "tampered-data-after", "tampered-data-only", "other-actor-only", "found-false-zero", "found-false-same-value",
                 "swapped-data", "second-world")


class Fault:
    """One fault variant: drop (a node CID) and corrupt (a node CID replaced by 0xff bytes of its length) in HAND's trie; path: the path
    that meets both; first: 'missing' or 'decode', the fault at the earlier spec."""

    def __init__(self, name, path, drop, corrupt, first):
        self.name, self.path, self.drop, self.corrupt, self.first = name, path, drop, corrupt, first

    def arrays(self, flat):
        arr = flat.replaced(self.corrupt, b"\xff" * int(flat.lengths[flat.index[self.corrupt]]))
        keep = [i for i in range(flat.n_blocks) if i != flat.index[self.drop]]
        return dict(arr, cids=arr["cids"][keep], offsets=arr["offsets"][keep], lengths=arr["lengths"][keep], n_blocks=len(keep))


@functools.lru_cache(maxsize=None)
def faults():
    """Both orders of every FAULT_PAIRS entry → [Fault], named as FAULT_NAMES. Each node is the deepest one on its spec's lookup that no earlier spec of the
    fault batch (fault_batch) visits."""
    w = build()
    bw, root = WIDTH[HAND], w.roots[HAND]
    out = []
    for name, pname, a, b in FAULT_PAIRS:
        path = w.hand[pname]
        specs = w.expected(path)[0]
        before = [s for p in fault_batch(path)[:2] for _, s in w.expected(p)[0] if p.actor_id == HAND]
        visited = lambda slots: {n for s in slots for n in lookup_nodes(w.blocks, root, s, bw)}
        na = lookup_nodes(w.blocks, root, specs[a][1], bw)[-1]
        nb = lookup_nodes(w.blocks, root, specs[b][1], bw)[-1]
        assert na not in visited(before + [s for _, s in specs[:a]]), name
        assert nb not in visited(before + [s for _, s in specs[:b]]), name
        out.append(Fault(f"{name}:missing-first", path, na, nb, "missing"))
        out.append(Fault(f"{name}:decode-first", path, nb, na, "decode"))
    return out


def fault_batch(path):
    """The batch a fault path runs in: two good paths in front (another actor and HAND), the path, and the path again"""
    w = build()
    return [w.edges[0], w.hand["pair"], path, path]


def absent_batches():
    """(name, batch, Fault) of the ACTOR_NOT_FOUND cases: a path to an absent actor behind a path whose first fault is a missing data
    slot node (wave 2), and in front of it"""
    f = next(f for f in faults() if f.name == "data+data:missing-first")
    absent = StoragePath(ABSENT, 0)
    return [(ABSENT_NAMES[0], [f.path, absent], f), (ABSENT_NAMES[1], [absent, f.path], f)]


def oracle_outcomes(ostore, tip, batch):
    """Per path of batch, per expanded spec (storage_paths.expand over the tree's dicts): None where the C++ oracle proves the spec
    alone, else its status"""
    w = build()
    out = []
    for p in batch:
        row = []
        for spec in w.expected(p)[0]:
            try:
                ostore.generate_storage_proofs(tip, [spec])
                row.append(None)
            except A.IpcfpError as e:
                row.append(e.status)
        out.append(row)
    return out


def first_failure(outcomes):
    """(status, path index) the header's rule gives: the first failing path, its first failing spec in expanded order"""
    for i, row in enumerate(outcomes):
        for s in row:
            if s is not None:
                return s, i
    return None


def union_witness(*flats):
    """A WitnessPy over every block of the given Flats"""
    blocks = T.Blocks()
    for f in flats:
        blocks.update(f.blocks)
    cids, offsets, lengths, blob = blocks.flat()
    return A.WitnessPy(cids, offsets, lengths, blob)


def world_specs():
    """(actor, slot) of every slot the tree holds, SHARER's included"""
    w = build()
    return [(a, s) for a in sorted(w.storage) for s in sorted(w.storage[a])]


def verifier_inputs(oracle_mod, ts):
    """(paths, witness over both trees, tip of the first, {name: proof list}) of the verifier cases, every proof made by the C++
    oracle"""
    w0, w1 = build(0), build(1)
    flat0, tip0 = w0.tip(ts)
    flat1, tip1 = w1.tip(ts)
    paths = verifier_paths()
    gen = lambda flat, tip, specs: oracle_mod.Store(flat.cids, flat.offsets, flat.lengths, flat.blob).generate_storage_proofs(tip, specs).proofs
    honest = gen(flat0, tip0, [s for p in paths for s in w0.expected(p)[0]])
    second = gen(flat1, tip1, [s for p in paths for s in w1.expected(p)[0]])
    lists = hostile_lists(honest, gen(flat0, tip0, world_specs()), second)
    return paths, union_witness(flat0, flat1), tip0, lists


# ------------------------------------------------------------------ the path verifier
def verifier_paths():
    """The paths the verifier cases check: every HAND path, a word SHARER and actor 1 000 both hold, 60 campaign paths, the edges'
    header forms"""
    w = build()
    shared = sorted(w.storage[1000])[0]
    return (list(w.hand.values()) + [StoragePath(SHARER, shared), StoragePath(1000, shared)] + w.campaign[:60] + w.edges[-12:])


def _with(q, **kw):
    d = dict(actor_id=q.actor_id, actor_state_cid=q.actor_state_cid, storage_root=q.storage_root, slot=q.slot, value=q.value,
             found=q.found, raw_len=q.raw_len)
    d.update(kw)
    return A.StorageProofPy(**d)


def _flip(q):
    return _with(q, value=bytes([q.value[0] ^ 1]) + q.value[1:])


def hostile_lists(honest, world_proofs, second):
    """{name: [StorageProofPy]} from the honest proofs of verifier_paths() (spec order), proofs of every slot of the tree and the
    second tree's proofs of the same paths"""
    w = build()
    H = w.hand
    rng = random.Random(24)
    by_key = {(q.actor_id, q.slot): q for q in honest}

    def key(pname, k):
        return w.expected(H[pname])[0][k]

    out = {}
    shuffled = list(honest)
    rng.shuffle(shuffled)
    out["honest-shuffled"] = shuffled
    out["honest+world"] = honest + world_proofs
    out["empty"] = []
    for role, (pname, k) in (("header", ("s65", 0)), ("length", ("arr[3]", 0)), ("data", ("s65", 2))):
        kk = key(pname, k)
        bad = _flip(by_key[kk])
        out[f"tampered-{role}-before"] = [bad] + honest
        out[f"tampered-{role}-after"] = honest + [bad]
        out[f"tampered-{role}-only"] = [bad if (q.actor_id, q.slot) == kk else q for q in honest]
    shared = sorted(w.storage[1000])[0]
    out["other-actor-only"] = [q for q in honest if (q.actor_id, q.slot) != (SHARER, shared)]
    kk = key("pair", 1)
    out["found-false-zero"] = [_with(q, found=False, value=ZERO, raw_len=0) if (q.actor_id, q.slot) == kk else q for q in honest]
    out["found-false-same-value"] = [_with(q, found=False) if (q.actor_id, q.slot) == kk else q for q in honest]
    a = [key("s65", j) for j in (1, 2, 3)]
    b = [key("s100", j) for j in (1, 2, 3)]
    swap = {x: by_key[y].value for x, y in zip(a, b)}
    swap.update({y: by_key[x].value for x, y in zip(a, b)})
    out["swapped-data"] = [_with(q, value=swap[(q.actor_id, q.slot)]) if (q.actor_id, q.slot) in swap else q for q in honest]
    out["second-world"] = list(second)
    assert tuple(out) == HOSTILE_NAMES
    return out


def expected_verdicts(paths, proofs, verdicts):
    """The path verifier's result over proofs (list, in list order) whose per-proof verdicts are `verdicts`: per path (valid, status,
    value, specs). A spec's word is that of the first proof in the list that verifies for its (actor_id, slot); storage_paths.expand
    gives the status, value and specs from those words; valid = every expanded spec has one. A spec with no verifying proof reads
    as follows: a length word does not make the index out of range, a BYTES header reads as zero (no data slots, empty value), any
    other word is that of the first listed proof for the key (what the path's value then shows), or zero when the list has none."""
    good, listed = {}, {}
    for q, v in zip(proofs, verdicts):
        k = (q.actor_id, bytes(q.slot))
        listed.setdefault(k, q.value)
        if v:
            good.setdefault(k, q.value)
    out = []
    for p in paths:
        lengths, _, final, _ = SP.derive(p)
        lengths = set(lengths)

        def read_status(slot, p=p, lengths=lengths):
            k = (p.actor_id, bytes(slot))
            if k in good:
                return good[k]
            return SP.b32(SP.M - 1) if bytes(slot) in lengths else ZERO

        def read_value(slot, p=p, final=final):
            k = (p.actor_id, bytes(slot))
            if k in good:
                return good[k]
            if p.kind == A.PATH_BYTES and bytes(slot) == final:
                return ZERO
            return listed.get(k, ZERO)

        specs, status, _, _, _ = SP.expand(p, read_status)
        _, _, value, _, _ = SP.expand(p, read_value)
        out.append((all(k in good for k in specs), status, value, specs))
    return out
