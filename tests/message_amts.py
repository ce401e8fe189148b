"""Hand-built message AMTs and tipsets whose parent blocks share their messages (cbor2 + hashlib only; a helper module, not a fixture file).

`build_amt` writes an AMT v0 (bit width 3) from an explicit {index: message CID} map at any height 0–21: minimal or taller roots, holes,
indices up to 8^(height+1) − 1 (beyond 2^64 at height 21) and nodes that are dropped or do not decode. `edit_tipset` turns a synthetic
tipset with one parent block into a tipset of P parent blocks, each with its own BLS and SECP message lists (or a shared TxMeta), with
honest CIDs throughout. `exec_order` is the ground truth: the first-seen union over the parents, each parent's BLS values in index order,
then its SECP values (events/utils.rs:48-94). Receipts do not name messages, so any arrangement keeps the receipts and events valid; only
`n_exec` and each proof's `message_cid` move. `catalogue(ts)` lists the cases tests/test_message_amts.py (CPU) and
tests/test_gpu_message_amts.py run."""
import functools
import random

import cbor2
import numpy as np

from tests.storage_trees import Blocks, cid_of, clink, head
from tests.util import EditedTipset

MAX_HEIGHT = 21        # height · 3 ≤ 64
KEY_BASE_BITS = 44     # the subtree-base field of the engine's message-AMT fault key (tx_err_key, csrc/common.cuh)


def min_height(indices):
    h = 0
    while indices and max(indices) >= 8 ** (h + 1):
        h += 1
    return h


class Amt:
    """A built message AMT: `root` (CID), `nodes` {(level, base): CID} of every non-root node, `values` {index: CID}."""

    def __init__(self, root, nodes, values, height):
        self.root, self.nodes, self.values, self.height = root, nodes, values, height

    def in_order(self):
        return [self.values[i] for i in sorted(self.values)]


def _node(blocks, level, base, items, nodes, bad):
    """Encoded node at `level` covering [base, base + 8^(level+1)) holding `items` [(index, cid)] (sorted). Children are written to
    `blocks`; a node whose (level, base) is in `bad` is written without its last byte (it does not decode)."""
    bm, links, vals = 0, [], []
    if level == 0:
        for i, c in items:
            bm |= 1 << (i - base)
            vals.append(clink(c))
    else:
        span = 8 ** level
        groups = {}
        for i, c in items:
            groups.setdefault((i - base) // span, []).append((i, c))
        for slot in sorted(groups):
            cb = base + slot * span
            enc = _node(blocks, level - 1, cb, groups[slot], nodes, bad)
            if (level - 1, cb) in bad:
                enc = enc[:-1]
            nodes[(level - 1, cb)] = blocks.put(enc)
            bm |= 1 << slot
            links.append(clink(nodes[(level - 1, cb)]))
    return b"\x83" + head(2, 1) + bytes([bm]) + head(4, len(links)) + b"".join(links) + head(4, len(vals)) + b"".join(vals)


def build_amt(blocks, values, height=None, bad=()):
    """AMT v0 of `values` {index: message CID} at `height` (default: the minimal one) → Amt. Nodes with no value below them are absent.
    bad: {(level, base)} of non-root nodes to write undecodable."""
    h = min_height(list(values)) if height is None else height
    assert 0 <= h <= MAX_HEIGHT and all(0 <= i < 8 ** (h + 1) for i in values)
    nodes = {}
    node = _node(blocks, h, 0, sorted(values.items()), nodes, set(bad))
    root = blocks.put(b"\x83" + head(0, h) + head(0, len(values)) + node)
    return Amt(root, nodes, dict(values), h)


def amt_values(blocks, root):
    """In-order values of a (well-formed) message AMT in `blocks` → [CID]."""
    height, _, node = cbor2.loads(blocks[root])
    out = []

    def walk(n, h):
        bm, links, vals = n
        if h == 0:
            out.extend(bytes(v.value[1:]) for v in vals)
        for ln in links:
            walk(cbor2.loads(blocks[bytes(ln.value[1:])]), h - 1)

    walk(node, height)
    return out


def txmeta(blocks, bls_root, secp_root):
    return blocks.put(b"\x82" + clink(bls_root) + clink(secp_root))


def base_blocks(ts):
    """The blocks of a synthetic tipset, its universe U (messages in execution order) and its one parent's (bls, secp) roots."""
    assert int(ts.n_parents) == 1
    blocks = Blocks()
    for i in range(int(ts.n_blocks)):
        blocks.setdefault(bytes(ts.cids[i]), ts.block(i))
    tm = cbor2.loads(blocks[bytes(ts.parent_txmeta_cids[0])])
    roots = tuple(bytes(r.value[1:]) for r in tm)
    u = amt_values(blocks, roots[0]) + amt_values(blocks, roots[1])
    assert len(u) == len(set(u)) == int(ts.n_receipts)
    return blocks, u, roots


def _link(cid):
    return cbor2.CBORTag(42, b"\0" + bytes(cid))


def edit_tipset(ts, blocks, txmetas):
    """ts (one parent block) with the parent blocks replaced: parent k is a copy of ts's parent header with `[10] messages` = txmetas[k]
    and `[12] timestamp` + k (so the headers differ), and the child header lists them in `[5] parents`. `blocks` must hold ts's blocks
    and every TxMeta and AMT named; it gains the headers. → EditedTipset with honest CIDs."""
    old = blocks[bytes(ts.parent_cids[0])]
    hdr = cbor2.loads(old)
    assert cbor2.dumps(hdr) == old and len(hdr) == 16
    pcids = []
    for k, tm in enumerate(txmetas):
        h = list(hdr)
        h[10] = _link(tm)
        h[12] = hdr[12] + k
        pcids.append(blocks.put(cbor2.dumps(h)))
    child_old = blocks[bytes(ts.child_cid)]
    child = cbor2.loads(child_old)
    assert cbor2.dumps(child) == child_old
    child[5] = [_link(c) for c in pcids]
    child_cid = blocks.put(cbor2.dumps(child))
    cids, offs, lens, blob = blocks.flat()

    def arr(cs):
        return np.frombuffer(b"".join(cs), dtype=np.uint8).reshape(-1, 38).copy()

    return EditedTipset(ts, cids=cids, offsets=offs, lengths=lens, blob=blob, n_blocks=len(lens), n_parents=len(pcids),
                        parent_cids=arr(pcids), parent_txmeta_cids=arr(txmetas),
                        child_cid=np.frombuffer(child_cid, dtype=np.uint8).copy())


def exec_order(lists):
    """First-seen union of [(bls values in index order, secp values in index order)] per parent → [CID]."""
    out, seen = [], set()
    for bls, secp in lists:
        for c in list(bls) + list(secp):
            if c not in seen:
                seen.add(c)
                out.append(c)
    return out


class Case:
    """One tipset of the catalogue. `truth`: the execution order, or None where the call fails with `status`. `lists`: per parent the
    (bls, secp) value lists. `blocks` {cid: bytes} (dropped blocks are gone). `large`: skipped by the Python oracle."""

    def __init__(self, name, ts, blocks, lists, truth, status=None, large=False, amts=None):
        self.name, self.ts, self.blocks, self.lists, self.truth, self.status, self.large = name, ts, blocks, lists, truth, status, large
        self.amts = amts or []


def _seq_amt(blocks, seq):
    return build_amt(blocks, dict(enumerate(seq)))


def shared_case(name, ts, parents):
    """parents: per parent (bls sequence, secp sequence) over U, or the literal 'base' for the synthetic parent's own TxMeta. Equal
    sequences share their AMT (and equal pairs their TxMeta)."""
    blocks, u, roots = base_blocks(ts)
    made, tms, lists = {}, [], []
    for p in parents:
        if p == "base":
            tms.append(bytes(ts.parent_txmeta_cids[0]))
            lists.append((u[:len(amt_values(blocks, roots[0]))], u[len(amt_values(blocks, roots[0])):]))
            continue
        rs = []
        for seq in p:
            key = tuple(seq)
            if key not in made:
                made[key] = _seq_amt(blocks, seq).root
            rs.append(made[key])
        tms.append(txmeta(blocks, *rs))
        lists.append((list(p[0]), list(p[1])))
    return Case(name, edit_tipset(ts, blocks, tms), blocks, lists, exec_order(lists))


def shared_cases(ts):
    """Parents that share their messages, over the universe U of ts (one parent, n_receipts messages)."""
    _, u, _ = base_blocks(ts)
    n = len(u)
    rng = random.Random(3)
    cases = []
    for p in (2, 5, 64):
        cases.append(shared_case(f"same-txmeta-P{p}", ts, ["base"] * p))
    a = 3 * n // 4
    m = (n - a) // 4 + 1
    cases.append(shared_case("same-bls-other-secp", ts, [(u[:a], u[a + k * m:a + (k + 1) * m]) for k in range(4)]))
    perm = u[:]
    rng.shuffle(perm)
    cases.append(shared_case("permutation-later", ts, [(u[:n // 2], u[n // 2:]), (perm, perm[::-1][:37])]))
    q = n // 4
    inter = []
    for k in range(4):
        lo, hi = max(0, k * q - 40), min(n, (k + 1) * q + 40)
        part = u[lo:hi]
        inter.append((part[::2] + u[(k * 97) % n:(k * 97) % n + 5], part[1::2]))
    cases.append(shared_case("interleaved-overlaps", ts, inter))
    cases.append(shared_case("secp-then-bls", ts, [(u[:n // 2], u[n // 2:n // 2 + 30]), (u[n // 2 + 10:], u[:8] + u[n // 2:n // 2 + 3])]))
    cases.append(shared_case("cid-twice-in-one-amt", ts, [(u[:100] + u[40:60] + u[100:n // 2] + u[5:6], u[n // 2:] + u[n - 3:]),
                                                           (u[:3], u[:3])]))
    short = shared_case("union-shorter", ts, [(u[:n // 3], u[n // 3:n // 3 + 7]), (u[:n // 3], u[:2])])
    assert len(short.truth) < n
    short.truth_short = True
    cases.append(short)
    return cases


def shape_values(height, rng, u):
    """A few values for a hand-built AMT of `height`: index 0, the first index of root slot 1, the top index 8^(h+1) − 1, sparse
    random ones, and — where the height reaches them — indices beyond 2^44 and 2^64. Message CIDs are drawn from U."""
    top = 8 ** (height + 1)
    idx = {0, top - 1, 8 ** height if height else 1}
    for _ in range(3):
        idx.add(rng.randrange(top))
    for b in (KEY_BASE_BITS, 50, 64):
        if 2 ** b + 5 < top:
            idx.add(2 ** b + 5)
    picks = rng.sample(u, len(idx))
    return dict(zip(sorted(idx), picks))


def hand_tipset(name, ts, amts, n_copies=1, blocks=None, drop=(), status=None):
    """Parents 0 .. n_copies−1 carry the hand-built (bls, secp) Amt pair, the last parent the synthetic TxMeta (so the union covers U
    and every receipt keeps its message). drop: CIDs removed from the store afterwards."""
    if blocks is None:
        blocks, u, roots = base_blocks(ts)
    else:
        _, u, roots = base_blocks(ts)
    bls, secp = amts
    tm = txmeta(blocks, bls.root, secp.root)
    na = len(amt_values(blocks, roots[0])) if status is None else None
    lists = [(bls.in_order(), secp.in_order())] * n_copies
    e = edit_tipset(ts, blocks, [tm] * n_copies + [bytes(ts.parent_txmeta_cids[0])])
    if status is None:
        lists = lists + [(u[:na], u[na:])]
    if drop:
        keep = {c: b for c, b in blocks.items() if c not in set(drop)}
        blocks = Blocks(keep)
        cids, offs, lens, blob = blocks.flat()
        e = EditedTipset(e, cids=cids, offsets=offs, lengths=lens, blob=blob, n_blocks=len(lens))
    return Case(name, e, blocks, lists, exec_order(lists) if status is None else None, status=status, amts=[bls, secp])


def shape_cases(ts, copies=(1,)):
    """Hand-built message AMTs of every height 0–21 holding a few values (minimal and taller roots, sparse and top indices, indices
    beyond 2^44), at 1 and at 63 copies beside the synthetic parent (64 parents: frontiers past k_amt_top's fused rounds)."""
    _, u, _ = base_blocks(ts)
    cases = []
    for n_copies in copies:
        for h in range(MAX_HEIGHT + 1):
            rng = random.Random(100 * h + n_copies)
            blocks = base_blocks(ts)[0]
            bls = build_amt(blocks, shape_values(h, rng, u), h)
            small = {0: u[0], 5: u[1]} if h == 0 else {8 ** h - 1: u[2]}
            secp = build_amt(blocks, small, h)                 # taller than it needs to be
            cases.append(hand_tipset(f"shape-h{h}-x{n_copies}", ts, (bls, secp), n_copies, blocks))
        # an empty AMT, a height-0 AMT with 8 values
        blocks = base_blocks(ts)[0]
        cases.append(hand_tipset(f"shape-empty-full-x{n_copies}", ts, (build_amt(blocks, {}), build_amt(blocks, dict(enumerate(u[:8])))),
                                 n_copies, blocks))
    return cases


def _path_nodes(amt, index):
    """(level, base) of the non-root nodes on the path to `index`, top down."""
    out = []
    for level in range(amt.height - 1, -1, -1):
        span = 8 ** (level + 1)
        out.append((level, index // span * span))
    return out


def fault_cases(ts):
    """Single faults (a missing child, an undecodable node) at every height 1–21, and two faults in one AMT in both orders, with their
    subtree bases below 2^44 (height 5) and beyond it (height 15). Each case's status is what the in-order walk meets first."""
    from ipc_filecoin_proofs_b200 import _abi as A
    _, u, _ = base_blocks(ts)
    cases = []
    for h in range(1, MAX_HEIGHT + 1):
        rng = random.Random(7 * h)
        vals = shape_values(h, rng, u)
        target = sorted(vals)[len(vals) // 2]
        lvl, base = _path_nodes(build_amt(Blocks(), vals, h), target)[rng.randrange(h)]
        blocks = base_blocks(ts)[0]
        bls = build_amt(blocks, vals, h)
        secp = build_amt(blocks, {0: u[3]})
        cases.append(hand_tipset(f"missing-h{h}-l{lvl}", ts, (bls, secp), 1, blocks, drop=[bls.nodes[(lvl, base)]],
                                 status=A.ERR_MISSING_BLOCK))
        blocks = base_blocks(ts)[0]
        bls = build_amt(blocks, vals, h, bad={(lvl, base)})
        cases.append(hand_tipset(f"decode-h{h}-l{lvl}", ts, (bls, secp), 1, blocks, status=A.ERR_DECODE))
    for h in (5, 15):
        for decode_first in (True, False):
            rng = random.Random(h)
            # values under root slots 1 and 2; in slot 1 a node at level 3 (level 0 at height 5 would also do; 3 keeps it mid-tree)
            s1, s2 = 8 ** h, 2 * 8 ** h
            vals = {s1 + 12345: u[10], s1 + 8 ** 4 * 3 + 7: u[11], s2 + 99: u[12], s2 + 8 ** 5: u[13]}
            fault_lvl = min(3, h - 1)
            a_node = (fault_lvl, (s1 + 12345) // 8 ** (fault_lvl + 1) * 8 ** (fault_lvl + 1))
            b_node = (h - 1, s2)
            if not decode_first:
                a_node, b_node = (fault_lvl, (s2 + 99) // 8 ** (fault_lvl + 1) * 8 ** (fault_lvl + 1)), (h - 1, s1)
            blocks = base_blocks(ts)[0]
            bls = build_amt(blocks, vals, h, bad={a_node})
            secp = build_amt(blocks, {})
            tag = "decode-then-missing" if decode_first else "missing-then-decode"
            cases.append(hand_tipset(f"two-faults-h{h}-{tag}", ts, (bls, secp), 1, blocks, drop=[bls.nodes[b_node]],
                                     status=A.ERR_DECODE if decode_first else A.ERR_MISSING_BLOCK))
    return cases


@functools.lru_cache(maxsize=None)
def base_tipset(n_receipts=600, seed=77):
    """The synthetic tipset the catalogue starts from: one parent, events on most receipts, matches spread over the receipts."""
    import synth
    return synth.Tipset(synth.default_params(seed=seed, n_receipts=n_receipts, n_parents=1, events_per_receipt=4, match_ppm=150000,
                                             has_actor_filter=0, bw3_permille=0))


@functools.lru_cache(maxsize=None)
def capacity_tipset():
    """20 000 receipts, 10 % of them with an events root, one parent with 15 000 BLS + 5 000 SECP messages."""
    import synth
    return synth.Tipset(synth.default_params(seed=91, n_receipts=20000, n_parents=1, events_per_receipt=2, match_ppm=2000,
                                             null_root_permille=900, has_actor_filter=0, bw3_permille=0))


def capacity_case(p):
    """Every one of p parents carries the synthetic parent's TxMeta (one 20 000-message list)."""
    c = shared_case(f"capacity-P{p}", capacity_tipset(), ["base"] * p)
    c.large = True
    return c


def leaf_frontier(case):
    """Message-AMT nodes at the leaf level summed over every parent block's two AMTs: what a walk that takes each AMT on its own holds
    in its last round's frontier (shared AMT nodes counted once per parent)."""
    total = 0
    for bls, secp in case.lists:
        total += (len(bls) + 7) // 8 + (len(secp) + 7) // 8
    return total


def catalogue(ts):
    return shared_cases(ts) + shape_cases(ts) + fault_cases(ts)
