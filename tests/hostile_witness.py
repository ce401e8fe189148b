"""Hostile witnesses whose every block hashes to its CID (cbor2 + hashlib only; a helper module, not a fixture file).

A party that hands over a proof bundle can write any block, give it its true CID, and re-encode and re-hash every block above it up
to the child header. The store's Blake2b check then admits every block: what stands between such a witness and a wrong verdict is
the verifier's decoders, its order of checks, and the caller's trust in the child header. `Forge` does this to a block set: a block
replaced (under any CID prefix) or dropped, and every block that links a changed CID re-encoded with the new link and re-hashed,
repeatedly, up to the roots. The catalogues plant one fault per case on a proof path of a witness the generator recorded:

  event_cases()    child header, parent headers, TxMeta blocks, message AMTs, receipts AMT, events AMTs, decoys (tests/event_amts.py's
                   synthetic tipset with a second parent block whose TxMeta and message AMTs are its own)
  storage_cases()  header / StateRoot / actors HAMT / ActorState / EVM state / storage value (tests/storage_trees.py's world_proofs)

Each case states what the restated verifier (the C++ oracle, which follows the reference's order) returns: the verdict list, or
(status, index of the first failing proof). `event_claim_holds` / `storage_claim_holds` follow the links the descriptor's child CID
commits to, so every accepted claim can be checked against the chain it was accepted for. `event_batches` / `storage_batches` plant
faults in different proofs of one call. tests/test_hostile_witness.py pins the catalogues on the CPU; tests/test_gpu_hostile_witness.py
runs them through the GPU verifiers."""
import copy
import functools
import hashlib
import random
import struct
from types import SimpleNamespace

import cbor2
import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A
from oracle import pyoracle as P
from tests import event_amts as E
from tests import message_amts as MA
from tests import storage_trees as S
from tests.storage_trees import Blocks, cbytes, clink, ctext, head
from tests.util import CID_LINK, EditedTipset, LINK_HEAD

RAW_PREFIX = bytes.fromhex("0155a0e40220")        # CIDv1, raw, blake2b-256: hashed by the store, not DAG-CBOR
BLAKE2S_PREFIX = bytes.fromhex("0171e0e40220")    # CIDv1, dag-cbor, blake2s-256: a class the store does not hash
HASHED_CODE = bytes.fromhex("a0e40220")           # multihash blake2b-256, 32 bytes


def b2b(data):
    return hashlib.blake2b(data, digest_size=32).digest()


def hashes_to_cid(cid, data):
    """The check the store makes: for a Blake2b-256 CID, the digest is Blake2b(data); other classes are not hashed (None)."""
    if cid[2:6] != HASHED_CODE:
        return None
    return cid[6:] == b2b(data)


# ------------------------------------------------------------------ re-anchoring
class Forge:
    """A block set {cid: bytes} under edits. `replace` and `drop` change blocks; after a replacement every block linking a changed CID
    is re-encoded with the new link (its own prefix kept) and re-hashed, until no block links a replaced CID. `cid(c)` follows c to its
    current CID; `created` holds every CID written here."""

    def __init__(self, blocks):
        self.blocks = dict(blocks)
        self.m = {}
        self.created = set()

    def cid(self, c):
        c = bytes(c)
        while c in self.m:
            c = self.m[c]
        return c

    def _put(self, old, data, prefix):
        new = prefix + b2b(data)
        self.blocks.pop(old, None)
        self.blocks[new] = data
        self.created.add(new)
        if new != old:
            self.m[old] = new
        return new

    def _propagate(self):
        while True:
            changed = False
            for c in list(self.blocks):
                b = self.blocks[c]
                b2 = CID_LINK.sub(lambda mo: LINK_HEAD + self.cid(mo.group(1)), b)
                if b2 != b:
                    self._put(c, b2, c[:6])
                    changed = True
            if not changed:
                return

    def replace(self, old, data, prefix=None):
        """Block `old` (an original or current CID) becomes `data` under `prefix` (default: its own). → the new CID."""
        cur = self.cid(old)
        new = self._put(cur, bytes(data), prefix or cur[:6])
        self._propagate()
        return self.cid(new)

    def relink(self, old, prefix):
        """The same bytes under another CID prefix (every link to it follows)."""
        return self.replace(old, self.blocks[self.cid(old)], prefix)

    def add(self, blocks):
        for c, b in blocks.items():
            self.blocks[bytes(c)] = bytes(b)
            self.created.add(bytes(c))

    def drop(self, c):
        self.blocks.pop(self.cid(c))

    def get(self, c):
        return self.blocks[self.cid(c)]


def witness_py(entries):
    """[(cid, bytes)] in the order given (duplicates kept) → WitnessPy."""
    cids = np.frombuffer(b"".join(c for c, _ in entries), dtype=np.uint8).reshape(-1, A.CID_LEN).copy() if entries else np.zeros((0, 38), np.uint8)
    offs, lens, blob = [], [], bytearray()
    for _, b in entries:
        offs.append(len(blob))
        lens.append(len(b))
        blob += b
    return A.WitnessPy(cids, np.array(offs, dtype=np.uint64), np.array(lens, dtype=np.uint32), np.frombuffer(bytes(blob) + bytes(16), dtype=np.uint8))


def sorted_entries(blocks):
    return sorted(blocks.items(), key=lambda cb: P.cid_sort_key(cb[0]))


def _arr(cs):
    return np.frombuffer(b"".join(bytes(c) for c in cs), dtype=np.uint8).reshape(-1, 38).copy() if cs else np.zeros((0, 38), np.uint8)


class Case:
    """One verifier call on a hostile witness. entries: the witness [(cid, bytes)] (decoys and duplicates included); ts: the tipset
    descriptor (the re-anchored child and parent CIDs); proofs: EventProofPy or StorageProofPy; expect: [bool] per proof, or (status,
    index of the first failing proof); unchecked: CIDs of decoys under a class the store does not hash; chain: {cid: bytes} the child
    CID commits to (for the ground truth of accepted claims)."""

    def __init__(self, name, kind, entries, ts, proofs, expect, unchecked=(), chain=None):
        self.name, self.kind, self.entries, self.ts, self.proofs, self.expect = name, kind, entries, ts, list(proofs), expect
        self.unchecked = set(unchecked)
        self.chain = chain if chain is not None else dict(entries)

    @property
    def fails(self):
        return isinstance(self.expect, tuple)

    def witness(self):
        return witness_py(self.entries)

    def result(self):
        """The result-like object the verifiers and the bundle renderers take."""
        if self.kind == "event":
            raw, blob = A.pack_event_proofs(self.proofs)
            return SimpleNamespace(proofs=self.proofs, raw_proofs=raw, data_blob=blob[:len(blob) - 16], witness=self.witness())
        return SimpleNamespace(proofs=self.proofs, raw_proofs=A.pack_storage_proofs(self.proofs), witness=self.witness())


# ------------------------------------------------------------------ the event side
HDR_PARENTS, HDR_HEIGHT, HDR_RECEIPTS, HDR_MESSAGES = 5, 7, 9, 10
IGNORED_FIELDS = (0, 1, 2, 3, 4, 6, 11, 13, 15)    # header fields the decoder skips (IgnoredAny)


def hdr_items(raw):
    """The 16 fields of a header block as their canonical encodings."""
    h = cbor2.loads(raw)
    assert cbor2.dumps(h) == raw and len(h) == 16
    return [cbor2.dumps(x) for x in h]


def hdr_bytes(items):
    return head(4, len(items)) + b"".join(items)


def _link(c):
    return cbor2.CBORTag(42, b"\0" + bytes(c))


def _unlink(tag):
    return bytes(tag.value[1:])


# CBOR items an IgnoredAny field may hold (DESIGN.md §3) and items the decoder refuses there
ACCEPTED_KINDS = {
    "f64": b"\xfb" + struct.pack(">d", -2.5),
    "false": b"\xf4", "true": b"\xf5", "null": b"\xf6",
    "link": clink(S.cid_of(b"elsewhere")),
    "nested": head(4, 3) + head(4, 1) + head(5, 1) + ctext("k") + head(4, 0) + head(5, 0) + head(4, 2) + head(1, 7) + cbytes(b"\x00\x01"),
    "utf8": head(3, len("héllö ✓ \U0001f600".encode())) + "héllö ✓ \U0001f600".encode(),
}
REFUSED_KINDS = {
    "f16": b"\xf9\x3c\x00",
    "f32": b"\xfa\x3f\xc0\x00\x00",
    "undefined": b"\xf7",
    "simple-f8": b"\xf8\x20",
    "tag-1": b"\xc1\x00",
    "tag-43-link": b"\xd8\x2b\x58\x27\x00" + S.cid_of(b"elsewhere"),
    "indef-array": b"\x9f\xff",
    "indef-map": b"\xbf\xff",
    "indef-bytes": b"\x5f\xff",
    "indef-text": b"\x7f\xff",
    "nonminimal-uint": b"\x18\x05",
    "nonminimal-bytes": b"\x58\x01\xaa",
    "bad-utf8": b"\x62\xc3\x28",
}


@functools.lru_cache(maxsize=None)
def event_world():
    """The honest tipset the event catalogue forges: tests/event_amts.py's synthetic tipset (600 receipts, one parent block) with a
    second parent block whose own message AMTs (a BLS AMT of height 1, a SECP AMT) repeat messages of the first, so the execution order
    is the first parent's. → SimpleNamespace(ts, blocks {cid: bytes} of the whole tipset, proofs, witness {cid: bytes}, tx, amts)."""
    import oracle
    ts0 = E.base_tipset()
    blocks, u, roots = MA.base_blocks(ts0)
    bls1 = MA.build_amt(blocks, {i: u[19 - i] for i in range(20)})   # no node in common with the first parent's AMTs
    secp1 = MA.build_amt(blocks, {0: u[30], 9: u[31]})
    tm1 = MA.txmeta(blocks, bls1.root, secp1.root)
    ts = MA.edit_tipset(ts0, blocks, [bytes(ts0.parent_txmeta_cids[0]), tm1])
    spec = A.make_event_spec(ts.event_signature, ts.topic1, None)
    r = oracle.Store.from_tipset(ts).generate_event_proof(ts, spec)
    assert len(r.proofs) >= 40, len(r.proofs)
    wit = {bytes(r.witness.cids[i]): r.witness.block(i) for i in range(r.witness.n_blocks)}
    bls0 = MA.Amt(roots[0], {}, {}, None)
    return SimpleNamespace(ts=ts, blocks=dict(blocks), proofs=list(r.proofs), witness=wit, spec=spec, u=u,
                           tx=[bytes(ts.parent_txmeta_cids[0]), tm1], bls=[roots[0], bls1.root], secp=[roots[1], secp1.root],
                           bls1=bls1, bls0=bls0)


def _amt_nodes(blocks, root):
    """Non-root node CIDs of a (well-formed) AMT in `blocks`, top down."""
    raw = cbor2.loads(blocks[root])
    node = raw[-1]
    out, todo = [], [node]
    while todo:
        n = todo.pop(0)
        for ln in n[1]:
            c = _unlink(ln)
            out.append(c)
            todo.append(cbor2.loads(blocks[c]))
    return out


def retarget(ts, f, parents=None, **over):
    """ts's descriptor after forging: child, parents and TxMeta CIDs followed through `f` (parents: an explicit list)."""
    pc = [f.cid(c) for c in ts.parent_cids] if parents is None else parents
    tx = [f.cid(c) for c in ts.parent_txmeta_cids][:len(pc)]
    tx += [bytes(38)] * (len(pc) - len(tx))
    return EditedTipset(ts, child_cid=np.frombuffer(f.cid(ts.child_cid), dtype=np.uint8).copy(),
                        parent_cids=_arr(pc), parent_txmeta_cids=_arr(tx), n_parents=len(pc),
                        receipts_root=np.frombuffer(f.cid(ts.receipts_root), dtype=np.uint8).copy(), **over)


def event_entries(w, f, decoys=False):
    """The forged witness: the generator's witness followed through `f` (dropped blocks stay out) plus every block `f` wrote, in `Cid`
    order; decoys: the honest originals that are no longer in it, after them."""
    out = {}
    for c in w.witness:
        cur = f.cid(c)
        if cur in f.blocks:
            out[cur] = f.blocks[cur]
    for c in f.created:
        if c in f.blocks:
            out[c] = f.blocks[c]
    entries = sorted_entries(out)
    if decoys:
        entries += [(c, b) for c, b in sorted_entries(w.witness) if c not in out]
    return entries


def event_claim_holds(chain, ts, p):
    """Ground truth of one event claim in the chain `ts.child_cid` commits to (blocks from `chain`): the child header lists the
    descriptor's parents at its epoch, parent 0 is at the parent epoch, exec[exec_index] is the claimed message, and the receipt at
    exec_index carries, at event_index, the claimed emitter, topics and data."""
    try:
        child = cbor2.loads(chain[bytes(ts.child_cid)])
        parents = [bytes(c) for c in np.asarray(ts.parent_cids, dtype=np.uint8).reshape(-1, 38)]
        if [_unlink(x) for x in child[HDR_PARENTS]] != parents or child[HDR_HEIGHT] != int(ts.child_epoch) or not parents:
            return False
        if cbor2.loads(chain[parents[0]])[HDR_HEIGHT] != int(ts.parent_epoch):
            return False
        txm = [_unlink(cbor2.loads(chain[c])[HDR_MESSAGES]) for c in parents]
        for t in txm:
            if t[:6] != S.PREFIX or t[6:] != b2b(chain[t]):
                return False
        exec_order = P.collect_exec_list(chain.get, txm)
        if p.exec_index >= len(exec_order) or exec_order[p.exec_index] != bytes(p.message_cid):
            return False
        rec = P.Recorder(chain)
        rc = P.Amt(_unlink(child[HDR_RECEIPTS]), rec, 0).get(p.exec_index)
        if rc is None or rc[3] is None:
            return False
        se = P.Amt(_unlink(rc[3]), rec, 3).get(p.event_index)
        if se is None or se[0] != p.emitter:
            return False
        log = P.extract_evm_log(se[1])
        return log is not None and [bytes(t) for t in log[0]] == [bytes(t) for t in p.topics] and bytes(log[1]) == bytes(p.data)
    except (KeyError, P.MissingBlock):
        return False


def _ev(ts, f):
    return retarget(ts, f)


def _receipts(w, f):
    """{index: receipt bytes} of the current receipts AMT (the whole tipset's blocks are in f)."""
    return E.chain_receipts(f.blocks, SimpleNamespace(receipts_root=f.cid(w.ts.receipts_root)))


def _new_receipts(w, f, recs, height=None):
    nb = Blocks()
    amt = E.build_receipts_amt(nb, recs, height)
    f.add(nb)
    f.replace(w.ts.receipts_root, nb[amt.root])
    return amt


def _events_root(f, w, i):
    recs = _receipts(w, f)
    return _unlink(cbor2.loads(recs[i])[3])


def _event_values(f, root):
    """(bw, height, {index: event bytes}) of an events AMT."""
    bw, h, _, _ = E.read_root(f.blocks[root], 3)
    vals = {}
    for j, item in E.walk(f.blocks, root, 3):
        enc = cbor2.dumps(item)
        vals[j] = enc
    return bw, h, vals


def _new_events(w, f, i, vals, bw, height=None, root_bytes=None, nb=None):
    """Receipt i's events root replaced by an AMT of `vals` (or by `root_bytes` with the blocks `nb`)."""
    old = _events_root(f, w, i)
    if root_bytes is None:
        nb = Blocks()
        a = E.build_events_amt(nb, vals, bw, height)
        root_bytes = nb[a.root]
    f.add(nb or {})
    f.replace(old, root_bytes)


def _entry_kv(entries, key):
    for e in entries:
        if e[1] == key:
            return e
    return None


def event_cases():
    """The event catalogue → [Case]."""
    w = event_world()
    ts, proofs = w.ts, w.proofs
    D, M, X = A.ERR_DECODE, A.ERR_MISSING_BLOCK, A.ERR_CID_MISMATCH
    n = len(proofs)
    T, F = [True] * n, [False] * n
    cases = []

    def forge():
        return Forge(w.blocks)

    def add(name, f, expect, decoys=False, desc=None, prf=None, extra=(), unchecked=()):
        entries = event_entries(w, f, decoys) + list(extra)
        cases.append(Case(name, "event", entries, desc if desc is not None else _ev(ts, f), prf if prf is not None else proofs, expect,
                          unchecked, chain=dict(f.blocks)))

    add("honest", forge(), T)

    # ---- child header
    child_items = hdr_items(w.blocks[bytes(ts.child_cid)])
    p01 = [bytes(c) for c in ts.parent_cids]
    for name, parents in (("reordered", p01[::-1]), ("shortened", p01[:1])):
        it = list(child_items)
        it[HDR_PARENTS] = cbor2.dumps([_link(c) for c in parents])
        f = forge()
        f.replace(ts.child_cid, hdr_bytes(it))
        add(f"child-parents-{name}", f, F)
    for d in (1, -1):
        it = list(child_items)
        it[HDR_HEIGHT] = cbor2.dumps(int(ts.child_epoch) + d)
        f = forge()
        f.replace(ts.child_cid, hdr_bytes(it))
        add(f"child-height{d:+d}", f, F)
    for nf in (15, 17):
        f = forge()
        f.replace(ts.child_cid, hdr_bytes(child_items[:15] if nf == 15 else child_items + [b"\x00"]))
        add(f"child-{nf}-fields", f, (D, 0))
    for kinds, ok in ((ACCEPTED_KINDS, True), (REFUSED_KINDS, False)):
        for kname, enc in kinds.items():
            for fld in IGNORED_FIELDS:
                it = list(child_items)
                it[fld] = enc
                f = forge()
                f.replace(ts.child_cid, hdr_bytes(it))
                add(f"child-field{fld}-{kname}", f, T if ok else (D, 0))
    it = list(child_items)
    it[HDR_PARENTS] = b"\x80"
    f = forge()
    f.replace(ts.child_cid, hdr_bytes(it))
    add("child-no-parents", f, (D, 0), desc=retarget(ts, f, parents=[]))

    # ---- parent headers: every one is decoded, only parent 0's height is compared
    p1_items = hdr_items(w.blocks[p01[1]])
    for name, items, expect in (("15-fields", p1_items[:15], (D, 0)), ("f32", [REFUSED_KINDS["f32"]] + p1_items[1:], (D, 0)),
                                ("height-other", p1_items[:HDR_HEIGHT] + [cbor2.dumps(int(ts.parent_epoch) + 7)] + p1_items[HDR_HEIGHT + 1:], T)):
        f = forge()
        f.replace(p01[1], hdr_bytes(items))
        add(f"parent1-{name}", f, expect)
    p0_items = hdr_items(w.blocks[p01[0]])
    f = forge()
    f.replace(p01[0], hdr_bytes(p0_items[:HDR_HEIGHT] + [cbor2.dumps(int(ts.parent_epoch) + 1)] + p0_items[HDR_HEIGHT + 1:]))
    add("parent0-height+1", f, F)

    # ---- TxMeta: linked under the raw codec (hashed, so admitted; the DAG-CBOR recompute differs), alone and with walk faults
    bls0_nodes = _amt_nodes(w.blocks, w.bls[0])
    bls1_nodes = _amt_nodes(w.blocks, w.bls[1])
    assert bls0_nodes and bls1_nodes and not set(bls0_nodes) & set(bls1_nodes)

    def walk_fault(f, where):
        if where == "missing0":
            f.drop(bls0_nodes[-1])
        elif where == "undecodable0":
            f.replace(bls0_nodes[-1], f.get(bls0_nodes[-1]) + b"\x00")
        elif where == "missing1":
            f.drop(bls1_nodes[0])
        elif where == "undecodable1":
            f.replace(bls1_nodes[0], f.get(bls1_nodes[0]) + b"\x00")
        elif where == "txmeta1-undecodable":
            f.replace(w.tx[1], f.get(w.tx[1]) + b"\x00")
        elif where == "txmeta1-missing":
            f.drop(w.tx[1])

    for raw_at in (0, 1):
        f = forge()
        f.relink(w.tx[raw_at], RAW_PREFIX)
        add(f"txmeta{raw_at}-raw", f, (X, 0))
    # the reference meets parent k's TxMeta mismatch before any fault in parent k's AMTs or in a later parent
    for where in ("missing0", "undecodable0", "missing1", "undecodable1", "txmeta1-undecodable", "txmeta1-missing"):
        f = forge()
        walk_fault(f, where)
        f.relink(w.tx[0], RAW_PREFIX)
        add(f"txmeta0-raw+{where}", f, (X, 0))
    for where in ("missing1", "undecodable1"):
        f = forge()
        walk_fault(f, where)
        f.relink(w.tx[1], RAW_PREFIX)
        add(f"txmeta1-raw+{where}", f, (X, 0))
    # ... and a fault in an earlier parent before a later parent's mismatch
    for where, st in (("missing0", M), ("undecodable0", D)):
        f = forge()
        walk_fault(f, where)
        f.relink(w.tx[1], RAW_PREFIX)
        add(f"txmeta1-raw+{where}", f, (st, 0))
    f = forge()
    f.relink(w.tx[0], RAW_PREFIX)
    add("txmeta0-raw-decoys", f, (X, 0), decoys=True)

    # ---- message AMTs: a message moved or duplicated, execution positions shift
    bls_vals = MA.amt_values(w.blocks, w.bls[0])
    secp_vals = MA.amt_values(w.blocks, w.secp[0])
    shift_at = proofs[n // 2].exec_index
    assert shift_at < len(bls_vals) - 3
    for name, seq in (("moved", bls_vals[:shift_at] + bls_vals[shift_at + 1:shift_at + 3] + [bls_vals[shift_at]] + bls_vals[shift_at + 3:]),
                      ("duplicated", bls_vals[:shift_at] + [bls_vals[shift_at + 2]] + bls_vals[shift_at:]),
                      ("inserted", bls_vals[:shift_at] + [S.cid_of(b"not a message of this chain")] + bls_vals[shift_at:])):
        nb = Blocks()
        a = MA.build_amt(nb, dict(enumerate(seq)))
        f = forge()
        f.add(nb)
        f.replace(w.tx[0], b"\x82" + clink(a.root) + clink(w.secp[0]))
        order = MA.exec_order([(seq, secp_vals)])
        add(f"messages-{name}", f, [order[p.exec_index] == p.message_cid for p in proofs])

    # ---- receipts AMT
    r0 = proofs[0].exec_index
    at_r0 = [p.exec_index != r0 for p in proofs]
    base_recs = E.chain_receipts(w.blocks, ts)
    f = forge()
    _new_receipts(w, f, {i: b for i, b in base_recs.items() if i != r0})
    add("receipts-hole", f, at_r0)
    f = forge()
    _new_receipts(w, f, {i: b for i, b in base_recs.items() if i != r0})
    add("receipts-hole-decoys", f, at_r0, decoys=True)
    f = forge()
    recs = dict(base_recs)
    ec, ret, gas, _ = cbor2.loads(recs[r0])
    recs[r0] = E.receipt(ec, ret, gas, None)
    _new_receipts(w, f, recs)
    add("receipts-events-root-null", f, at_r0)
    for r in sorted({p.exec_index for p in proofs})[1:4]:
        sib = r ^ 1
        recs = dict(base_recs)
        ec, ret, gas, er = cbor2.loads(recs[sib])
        recs[sib] = E.receipt(2 ** 32, ret, gas, _unlink(er) if er is not None else None)
        f = forge()
        _new_receipts(w, f, recs)
        first = next(k for k, p in enumerate(proofs) if p.exec_index // 8 == r // 8)
        add(f"receipts-sibling-exit-2^32-r{r}", f, (D, first))
    h = E.read_root(w.blocks[bytes(ts.receipts_root)], 0)[1]
    f = forge()
    _new_receipts(w, f, base_recs, height=h + 1)
    add("receipts-taller-root", f, T)
    rr = cbor2.loads(w.blocks[bytes(ts.receipts_root)])
    rr[2][2] = [cbor2.loads(base_recs[r0])]
    f = forge()
    f.replace(ts.receipts_root, cbor2.dumps(rr))
    add("receipts-root-links-and-values", f, (D, 0))

    # ---- events AMT of the receipt of one proof
    pk = next(k for k, p in enumerate(proofs) if k > 0 and _entry_kv(cbor2.loads(_ev_bytes(w, p))[1], "t2") is not None)
    pe = proofs[pk]
    R, J = pe.exec_index, pe.event_index
    root = _events_root(Forge(w.blocks), w, R)
    bw, eh, vals = _event_values(Forge(w.blocks), root)
    nb = Blocks()
    assert E.build_events_amt(nb, vals, bw, eh).root == root       # the rebuild is the chain's own AMT
    same = [not (p.exec_index == R and p.event_index == J) for p in proofs]
    em, ents = cbor2.loads(vals[J])

    def ev_case(name, new_vals, expect, bw2=None, h2=None, decoys=False):
        f = forge()
        _new_events(w, f, R, new_vals, bw2 or bw, h2 if h2 is not None else eh)
        add(f"events-{name}", f, expect, decoys=decoys)

    def with_event(em2, ents2):
        v = dict(vals)
        v[J] = cbor2.dumps([em2, ents2])
        return v

    ev_case("emitter", with_event(em ^ 1, ents), same)
    t2 = _entry_kv(ents, "t2")
    ev_case("topic-byte", with_event(em, [[a, k, c, (bytes([v[0] ^ 1]) + v[1:]) if k == "t2" else v] for a, k, c, v in ents]), same)
    ev_case("topic-byte-decoys", with_event(em, [[a, k, c, (bytes([v[0] ^ 1]) + v[1:]) if k == "t2" else v] for a, k, c, v in ents]), same,
            decoys=True)
    dk = "d"
    ev_case("data", with_event(em, [[a, k, c, v + b"\x01" if k == dk else v] for a, k, c, v in ents] +
                               ([] if _entry_kv(ents, dk) else [[3, dk, 0x55, b"\x01"]])), same)
    tks = [e[3] for e in ents if e[1] in ("t1", "t2", "t3", "t4")]
    dat = _entry_kv(ents, "d")
    ev_case("case-b-to-a", with_event(em, [[t2[0], "topics", t2[2], b"".join(tks)], [t2[0], "data", t2[2], dat[3] if dat else b""]]), T)
    ev_case("t2-31-bytes", with_event(em, [[a, k, c, v[:31] if k == "t2" else v] for a, k, c, v in ents]), same)
    v = dict(vals)
    del v[J]
    ev_case("removed", v, same)
    width = 1 << bw
    leaf_lo = J - J % width
    sib = J + 1
    assert sib < leaf_lo + width
    v = dict(vals)
    v[sib] = b"\x83\x01\x80\x00"      # a StampedEvent of three fields, after the claimed one in its leaf
    first = next(k for k, p in enumerate(proofs) if p.exec_index == R and (eh == 0 or p.event_index // width == J // width))
    ev_case("sibling-undecodable", v, (D, first))
    for bw2 in sorted({1, 2, 8} - {bw}):
        ev_case(f"relaid-bw{bw2}", vals, T, bw2=bw2, h2=E.min_height(list(vals), bw2))
    ev_case(f"relaid-bw{bw}-taller", vals, T, h2=eh + 2)
    first_r = next(k for k, p in enumerate(proofs) if p.exec_index == R)
    for wbw in (3, 5):
        wh = E.overflow_heights(wbw)[0]
        nb = Blocks()
        wroot = E.chain_root(nb, wbw, wh, 3, vals[J])
        f = forge()
        _new_events(w, f, R, None, None, root_bytes=nb[wroot], nb=nb)
        add(f"events-root-height-wraps-bw{wbw}", f, (D, first_r))

    # ---- decoys
    hon = sorted_entries(w.witness)
    cases.append(Case("duplicate-entries", "event", hon + hon[::-1], ts, proofs, T, chain=dict(w.blocks)))
    for name, target in (("child", bytes(ts.child_cid)), ("receipts-root", bytes(ts.receipts_root)), ("txmeta0", w.tx[0]),
                         ("events-root", root)):
        d = BLAKE2S_PREFIX + target[6:]
        # listed before the block whose digest it carries, with the bytes of another header
        cases.append(Case(f"blake2s-decoy-{name}", "event", [(d, w.blocks[p01[1]])] + hon, ts, proofs, T, unchecked=[d], chain=dict(w.blocks)))
    return cases


def _ev_bytes(w, p):
    f = Forge(w.blocks)
    root = _events_root(f, w, p.exec_index)
    return cbor2.dumps(dict(E.walk(f.blocks, root, 3))[p.event_index])


# ------------------------------------------------------------------ the storage side
@functools.lru_cache(maxsize=None)
def storage_world(ts):
    """world_proofs(ts) with honest proofs of tip "main": → SimpleNamespace(w, blocks, ts, specs, proofs, witness)."""
    import oracle
    w, flat = S.world_proofs(ts)
    tip = w.tips["main"]
    specs = []
    for a in (0, 1000, 2 ** 63, 2 ** 64 - 1, 2001):
        specs += [(a, s) for s in sorted(w.actors[a][1])[:3]]
    specs.append((0, b"\x01" * 32))
    r = oracle.Store(flat.cids, flat.offsets, flat.lengths, flat.blob).generate_storage_proofs(tip, specs)
    wit = {bytes(r.witness.cids[i]): r.witness.block(i) for i in range(r.witness.n_blocks)}
    return SimpleNamespace(w=w, blocks=wit, ts=tip, specs=specs, proofs=list(r.proofs), witness=wit,
                           child=bytes(tip.child_cid), psr=w.main_root)


def storage_claim_holds(chain, ts, p):
    """Ground truth of one storage claim in the chain `ts.child_cid` commits to: the header's state root is the descriptor's, and the
    actor's state, its storage root and the slot's value are the claimed ones."""
    try:
        t = P.generate_storage_proof(chain, ts, p.actor_id, bytes(p.slot))
    except (AssertionError, KeyError, P.MissingBlock):
        return False
    return t["actor_state_cid"] == bytes(p.actor_state_cid) and t["storage_root"] == bytes(p.storage_root) and t["value"] == bytes(p.value)


def _sdesc(sw, f, psr=None):
    return EditedTipset(sw.ts, child_cid=np.frombuffer(f.cid(sw.child), dtype=np.uint8).copy(),
                        parent_state_root=np.frombuffer(psr if psr is not None else f.cid(sw.psr), dtype=np.uint8).copy())


def storage_entries(sw, f):
    out = {}
    for c in sw.witness:
        cur = f.cid(c)
        if cur in f.blocks:
            out[cur] = f.blocks[cur]
    for c in f.created:
        if c in f.blocks:
            out[c] = f.blocks[c]
    return sorted_entries(out)


def _actors_root(sw, f):
    return _unlink(cbor2.loads(f.get(sw.psr))[1])


def _new_actors(sw, f, actors):
    nb = Blocks()
    root = S.build_hamt(nb, {S.id_address(a): s for a, s in actors.items()}, 5)
    f.add(nb)
    f.replace(sw.psr, S.state_root(root))


def _evm_of(sw, aid):
    return _unlink(cbor2.loads(sw.w.actors[aid][0])[1])


def evm_variant(contract_root, six, transient, tombstone):
    """EVM state with the nullable fields null or present: transient [state link, [origin, nonce]], tombstone [origin, nonce]."""
    bytecode = S.cid_of(b"bytecode")
    items = [clink(bytecode), cbytes(hashlib.sha256(b"bytecode").digest()), clink(contract_root)]
    if six:
        items.append(b"\x82" + clink(S.cid_of(b"transient")) + b"\x82\x19\x03\xe8\x07" if transient else b"\xf6")
    items += [head(0, 3), b"\x82\x19\x03\xe9\x02" if tombstone else b"\xf6"]
    return head(4, len(items)) + b"".join(items)


def storage_cases(ts):
    """The storage catalogue over world_proofs(ts) → [Case]."""
    sw = storage_world(ts)
    proofs = sw.proofs
    D = A.ERR_DECODE
    n = len(proofs)
    T, F = [True] * n, [False] * n
    cases = []

    def forge():
        return Forge(sw.blocks)

    def add(name, f, expect, desc=None, prf=None):
        cases.append(Case(name, "storage", storage_entries(sw, f), desc if desc is not None else _sdesc(sw, f), prf if prf is not None else proofs,
                          expect, chain=dict(f.blocks)))

    add("storage-honest", forge(), T)
    f = forge()
    add("state-root-differs", f, F, desc=_sdesc(sw, f, psr=sw.w.deep_root))
    f = forge()
    f.replace(sw.psr, S.state_root(_actors_root(sw, f), version=6))
    add("state-root-version-6", f, (D, 0))
    f = forge()
    ar = _actors_root(sw, f)
    f.replace(ar, f.get(ar) + b"\x00")
    add("actors-root-undecodable", f, (D, 0))
    for aid in (1000, 2001):
        f = forge()
        _new_actors(sw, f, {a: s for a, (s, _) in sw.w.actors.items() if a != aid})
        first = next(k for k, p in enumerate(proofs) if p.actor_id == aid)
        add(f"actor-{aid}-removed", f, (A.ERR_ACTOR_NOT_FOUND, first))
    # a re-hashed EVM state naming another storage trie: only the trust anchor on the child header stops the forged claims
    victim, other = 0, 1000
    for six in (True, False):
        for transient in ((False, True) if six else (False,)):
            for tomb in (False, True):
                f = forge()
                evm = evm_variant(sw.w.storage[other], six, transient, tomb)
                f.replace(_evm_of(sw, victim), evm)
                desc = _sdesc(sw, f)
                chain = dict(f.blocks)
                slot = sorted(sw.w.actors[other][1])[0]
                t = P.generate_storage_proof(chain, desc, victim, slot)
                forged = A.StorageProofPy(victim, t["actor_state_cid"], t["storage_root"], slot, t["value"], True, 32)
                need = {f.cid(c) for c in sw.witness if f.cid(c) in f.blocks} | set(t["witness"])
                entries = sorted_entries({c: chain[c] for c in need})
                prf = proofs + [forged]
                cases.append(Case(f"evm-retarget-v{6 if six else 5}{'-transient' if transient else ''}{'-tombstone' if tomb else ''}",
                                  "storage", entries, desc, prf, [p.actor_id != victim for p in proofs] + [True], chain=chain))
    # a storage value element of 256 under a re-hashed contract state
    k = b"\x42" * 32
    nb = Blocks()
    sroot = nb.put(S.hamt_node({S.hash_index(k, 0, 5): [(k, b"\x82\x01\x19\x01\x00")]}))
    f = forge()
    f.add(nb)
    evm_cid = f.replace(_evm_of(sw, victim), S.evm_state(sroot))
    bad = A.StorageProofPy(victim, evm_cid, sroot, k, bytes(32), True, 32)
    add("value-element-256", f, (D, 3), prf=proofs[:3] + [bad])
    return cases


# ------------------------------------------------------------------ batches: faults in different proofs of one call
BATCH_SIZES = (1, 4, 5, 128, 129, 16385)


def _cycle(seq, n, rng, order):
    idx = list(range(len(seq)))
    if order == "reversed":
        idx = idx[::-1]
    elif order == "shuffled":
        rng.shuffle(idx)
    return [seq[idx[k % len(idx)]] for k in range(n)]


def event_batch_world():
    """One forged witness with two fault sites (a sibling receipt of receipt r1 with exit code 2^32: DECODE for the proofs of its
    leaf; the events root of receipt r2 dropped: MISSING_BLOCK for its proofs), proofs that verify, and proofs whose emitter lies."""
    w = event_world()
    proofs = w.proofs
    execs = sorted({p.exec_index for p in proofs})
    r1 = execs[len(execs) // 3]
    r2 = next(r for r in execs[::-1] if r // 8 != r1 // 8)
    recs = E.chain_receipts(w.blocks, w.ts)
    ec, ret, gas, er = cbor2.loads(recs[r1 ^ 1])
    recs[r1 ^ 1] = E.receipt(2 ** 32, ret, gas, _unlink(er) if er is not None else None)
    f = Forge(w.blocks)
    _new_receipts(w, f, recs)
    ev2 = _events_root(f, w, r2)
    entries = [(c, b) for c, b in event_entries(w, f) if c != ev2]
    ok = [p for p in proofs if p.exec_index // 8 != r1 // 8 and p.exec_index != r2]
    lied = [copy.copy(p) for p in ok[::5]]
    for p in lied:
        p.emitter ^= 1
    bad = [(p, A.ERR_DECODE) for p in proofs if p.exec_index // 8 == r1 // 8][:2] + [(p, A.ERR_MISSING_BLOCK) for p in proofs if p.exec_index == r2][:2]
    return SimpleNamespace(entries=entries, ts=_ev(w.ts, f), ok=ok, lied=lied, bad=bad, chain=dict(f.blocks))


def storage_batch_world(ts):
    """One forged witness with two fault sites (actor 2001 removed: ACTOR_NOT_FOUND; actor 0's contract state re-hashed to a value
    element of 256: DECODE), proofs that verify, and proofs whose value lies."""
    sw = storage_world(ts)
    f = Forge(sw.blocks)
    gone = 2001
    _new_actors(sw, f, {a: s for a, (s, _) in sw.w.actors.items() if a != gone})
    k = b"\x42" * 32
    nb = Blocks()
    sroot = nb.put(S.hamt_node({S.hash_index(k, 0, 5): [(k, b"\x82\x01\x19\x01\x00")]}))
    f.add(nb)
    evm_cid = f.replace(_evm_of(sw, 0), S.evm_state(sroot))
    ok = [p for p in sw.proofs if p.actor_id not in (gone, 0)]
    lied = [copy.copy(p) for p in ok[::3]]
    for p in lied:
        p.value = bytes([p.value[0] ^ 1]) + p.value[1:]
    bad = [(p, A.ERR_ACTOR_NOT_FOUND) for p in sw.proofs if p.actor_id == gone][:1] + \
        [(A.StorageProofPy(0, evm_cid, sroot, k, bytes(32), True, 32), A.ERR_DECODE)]
    return SimpleNamespace(entries=storage_entries(sw, f), ts=_sdesc(sw, f), ok=ok, lied=lied, bad=bad, chain=dict(f.blocks))


def _batches(prefix, kind, bw, rng, sizes):
    """Per size and order (generated, reversed, shuffled): a batch without fault (false exactly for the lying claims), and the same
    batch with a faulty proof planted at the first, middle or last position and another at the end: (its status, that position)."""
    out = []
    lied = {id(p) for p in bw.lied}
    for n in sizes:
        for order in ("generated", "reversed", "shuffled"):
            clean = _cycle(bw.ok + bw.lied, n, rng, order)
            out.append(Case(f"{prefix}clean-n{n}-{order}", kind, bw.entries, bw.ts, clean, [id(p) not in lied for p in clean], chain=bw.chain))
            for pos in sorted({0, n // 2, n - 1}):
                prf = list(clean)
                first = bw.bad[rng.randrange(len(bw.bad))]
                prf[pos] = first[0]
                if pos + 1 < n:
                    prf[n - 1] = bw.bad[rng.randrange(len(bw.bad))][0]
                out.append(Case(f"{prefix}fault-n{n}-{order}-at{pos}", kind, bw.entries, bw.ts, prf, (first[1], pos), chain=bw.chain))
    return out


def event_batches(sizes=BATCH_SIZES):
    return _batches("", "event", event_batch_world(), random.Random(17), sizes)


def storage_batches(ts, sizes=BATCH_SIZES):
    return _batches("storage-", "storage", storage_batch_world(ts), random.Random(19), sizes)
