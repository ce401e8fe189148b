"""Hand-built events AMTs and receipts AMTs (cbor2 + hashlib only; a helper module, not a fixture file).

`build_events_amt` writes an AMT v3 (`[bit_width, height, count, node]`) at any bit width 1–8 and any height up to 64 // bw from an
explicit {index: event} map: holes, top indices, a `count` field that lies (so its encoded width can be chosen), empty nodes, and
nodes that are dropped or do not decode. `chain_root` writes the roots the decode contract refuses for their height alone (height·bw
above 64, including heights whose product wraps modulo 2^64) over a chain of one-link nodes. `build_receipts_amt` writes an AMT v0
of receipts at any height up to 21, with holes. `edit_tipset` rewrites a synthetic tipset with honest CIDs around them.

`walk` is a strict restatement of the AMT part of DESIGN.md §3 in Python integers; `truth` gives from it the expected result of a
valid case (matching receipts, proofs, witness CID set). `catalogue(ts)` lists the cases tests/test_event_amts.py (CPU) and
tests/test_gpu_event_amts.py run."""
import functools
import random

import cbor2
import numpy as np

from oracle import pyoracle as P
from tests.message_amts import base_blocks
from tests.storage_trees import Blocks, cbytes, clink, ctext, head
from tests.util import EditedTipset

U64 = 1 << 64
RECEIPTS_MAX_HEIGHT = 21


def width(bw):
    return 1 << bw


def bmap_len(bw):
    return 1 if bw <= 3 else 1 << (bw - 3)


def max_height(bw):
    return 64 // bw


def min_height(indices, bw):
    h = 0
    while indices and max(indices) >= width(bw) ** (h + 1):
        h += 1
    return h


# ------------------------------------------------------------------ events
def _entry(key, value, flags=3, codec=0x55):
    return b"\x84" + head(0, flags) + ctext(key) + head(0, codec) + cbytes(value)


def stamped(emitter, entries):
    return b"\x82" + head(0, emitter) + head(4, len(entries)) + b"".join(entries)


def ev_case_b(t0, t1, emitter=1001, data=b"", extra=()):
    """Case B: t1 = topic0, t2 = topic1 (then t3…), d."""
    ents = [_entry("t1", t0), _entry("t2", t1)] + [_entry("t%d" % (3 + k), t) for k, t in enumerate(extra)]
    return stamped(emitter, ents + [_entry("d", data)])


def ev_case_a(t0, t1, emitter=1002, data=b"", extra=()):
    """Case A: `topics` = the concatenated topics, `data`."""
    return stamped(emitter, [_entry("topics", t0 + t1 + b"".join(extra)), _entry("data", data)])


class Events:
    """Event encoders for one matcher (keccak256(signature), ascii_to_bytes32(topic1))."""

    def __init__(self, signature, topic1):
        self.t0 = P.keccak256(signature.encode())
        self.t1 = P.ascii_to_bytes32(topic1)

    def match_b(self, k):
        return ev_case_b(self.t0, self.t1, emitter=1000 + k, data=bytes([k % 251]) * (k % 7), extra=[bytes([k % 256]) * 32][:k % 2])

    def match_a(self, k):
        return ev_case_a(self.t0, self.t1, emitter=2000 + k, data=bytes([k % 253]) * (k % 5 + 1))

    def other(self, k):
        return ev_case_b(bytes([0x5A]) + k.to_bytes(31, "big"), self.t1, emitter=3000 + k)

    def near_topic1(self, k):
        return ev_case_b(self.t0, self.t1[:31] + bytes([self.t1[31] ^ 1]), emitter=4000 + k)

    def near_short(self, k):
        return ev_case_b(self.t0, self.t1[:31], emitter=5000 + k)

    def mixed(self, k):
        """Matching and non-matching events interleaved, so that an event's AMT index and its ordinal among matches differ."""
        return (self.match_b, self.other, self.match_a, self.near_topic1, self.near_short)[k % 5](k)


# ------------------------------------------------------------------ AMT writers
class EvAmt:
    """A built AMT: `root` (CID), `nodes` {(level, base): CID} of every non-root node, `values` {index: bytes}, `bw`, `height`."""

    def __init__(self, root, nodes, values, bw, height):
        self.root, self.nodes, self.values, self.bw, self.height = root, nodes, values, bw, height


def _node(blocks, bw, level, base, items, nodes, bad):
    """Encoded node at `level` covering [base, base + W^(level+1)) holding `items` [(index, value bytes)] (sorted); children are
    written to `blocks`. A child whose (level, base) is in `bad` is written without its last byte."""
    w = width(bw)
    bm, links, vals = 0, [], []
    if level == 0:
        for i, v in items:
            bm |= 1 << (i - base)
            vals.append(v)
    else:
        span = w ** level
        groups = {}
        for i, v in items:
            groups.setdefault((i - base) // span, []).append((i, v))
        for slot in sorted(groups):
            cb = base + slot * span
            enc = _node(blocks, bw, level - 1, cb, groups[slot], nodes, bad)
            if (level - 1, cb) in bad:
                enc = enc[:-1]
            nodes[(level - 1, cb)] = blocks.put(enc)
            bm |= 1 << slot
            links.append(clink(nodes[(level - 1, cb)]))
    n = bmap_len(bw)
    return b"\x83" + head(2, n) + bm.to_bytes(n, "little") + head(4, len(links)) + b"".join(links) + head(4, len(vals)) + b"".join(vals)


def build_events_amt(blocks, values, bw, height=None, count=None, bad=()):
    """AMT v3 of `values` {index: StampedEvent bytes} → EvAmt. height: default the minimal one; count: the root's count field (default
    the number of values; any value, so its encoded width can be chosen). bad: {(level, base)} of non-root nodes written undecodable."""
    h = min_height(list(values), bw) if height is None else height
    assert 1 <= bw <= 8 and 0 <= h <= max_height(bw) and all(0 <= i < width(bw) ** (h + 1) for i in values)
    nodes = {}
    node = _node(blocks, bw, h, 0, sorted(values.items()), nodes, set(bad))
    c = len(values) if count is None else count
    root = blocks.put(b"\x84" + head(0, bw) + head(0, h) + head(0, c) + node)
    return EvAmt(root, nodes, dict(values), bw, h)


def chain_root(blocks, bw, height, depth, leaf=None, version=3):
    """A root with bit width bw (version 0: bw 3, no bw field) and `height` written as is, over a chain of `depth` one-link nodes
    (slot 0) ending in a node that holds `leaf` at slot 0, or nothing. → root CID."""
    n = bmap_len(bw)
    last = b"\x83" + head(2, n) + (1 if leaf else 0).to_bytes(n, "little") + b"\x80" + (b"\x81" + leaf if leaf else b"\x80")
    for _ in range(depth):
        c = blocks.put(last)
        last = b"\x83" + head(2, n) + (1).to_bytes(n, "little") + b"\x81" + clink(c) + b"\x80"
    if version == 0:
        return blocks.put(b"\x83" + head(0, height) + head(0, 1 if leaf else 0) + last)
    return blocks.put(b"\x84" + head(0, bw) + head(0, height) + head(0, 1 if leaf else 0) + last)


def overflow_heights(bw):
    """Heights h < 2^64 whose product h·bw wraps to at most 64 (h·bw mod 2^64 ≤ 64 while h·bw > 64)."""
    out = []
    for k in range(1, bw):
        for m in range(65):
            if (k * U64 + m) % bw == 0:
                out.append((k * U64 + m) // bw)
    return out


def build_receipts_amt(blocks, receipts, height=None, bad=()):
    """AMT v0 of `receipts` {index: receipt bytes} → EvAmt (bw 3). height: default the minimal one, at most 21."""
    h = min_height(list(receipts), 3) if height is None else height
    assert 0 <= h <= RECEIPTS_MAX_HEIGHT and all(0 <= i < 8 ** (h + 1) for i in receipts)
    nodes = {}
    node = _node(blocks, 3, h, 0, sorted(receipts.items()), nodes, set(bad))
    root = blocks.put(b"\x83" + head(0, h) + head(0, len(receipts)) + node)
    return EvAmt(root, nodes, dict(receipts), 3, h)


def receipt(exit_code, ret, gas, events_root):
    return b"\x84" + head(0, exit_code) + cbytes(ret) + head(0, gas) + (clink(events_root) if events_root else b"\xf6")


# ------------------------------------------------------------------ the strict restatement (DESIGN.md §3, AMT part)
class Fault(Exception):
    def __init__(self, status):
        super().__init__(status)
        self.status = status


def _status(name):
    from ipc_filecoin_proofs_b200 import _abi as A
    return getattr(A, name)


def _strict(raw):
    """One CBOR item that must span the whole block in minimal heads: its canonical re-encoding is the block (a trailing byte fails)."""
    try:
        x = cbor2.loads(raw)
    except Exception:
        raise Fault(_status("ERR_DECODE"))
    if cbor2.dumps(x) != raw:
        raise Fault(_status("ERR_DECODE"))
    return x


def _cid(link):
    if not isinstance(link, cbor2.CBORTag) or link.tag != 42 or not isinstance(link.value, bytes) or len(link.value) != 39:
        raise Fault(_status("ERR_DECODE"))
    return bytes(link.value[1:])


def _node_items(node, bw, level):
    """(is_link, [(slot, item)]) of a decoded node, or Fault."""
    bad = Fault(_status("ERR_DECODE"))
    if not isinstance(node, list) or len(node) != 3:
        raise bad
    bm, links, vals = node
    if not isinstance(bm, bytes) or len(bm) != bmap_len(bw) or not isinstance(links, list) or not isinstance(vals, list):
        raise bad
    bits = int.from_bytes(bm, "little")
    if bits >> width(bw):
        raise bad
    slots = [s for s in range(width(bw)) if bits >> s & 1]
    if links and vals:
        raise bad
    if links:
        if level == 0 or len(slots) != len(links):
            raise bad
        return True, list(zip(slots, [_cid(x) for x in links]))
    if (vals and level != 0) or len(slots) != len(vals):
        raise bad
    return False, list(zip(slots, vals))


def read_root(raw, version):
    """(bw, height, count, node) of a root block, or Fault: 1 ≤ bw ≤ 8 and height·bw ≤ 64, in integers that do not wrap."""
    r = _strict(raw)
    bad = Fault(_status("ERR_DECODE"))
    if not isinstance(r, list) or len(r) != (3 if version == 0 else 4):
        raise bad
    if version == 0:
        bw, (h, count, node) = 3, r
    else:
        bw, h, count, node = r
    if not all(isinstance(x, int) and 0 <= x < U64 for x in (bw, h, count)) or not 1 <= bw <= 8 or h * bw > 64:
        raise bad
    return bw, h, count, node


def walk(blocks, root, version=3, seen=None):
    """Amt::for_each in order → [(index, value item)], every node recorded in `seen`; Fault(status) at the first fault met."""
    raw = blocks.get(root)
    if raw is None:
        raise Fault(_status("ERR_MISSING_BLOCK"))
    if seen is not None:
        seen.add(root)
    bw, h, _, node = read_root(raw, version)
    out = []

    def rec(n, level, base):
        is_link, items = _node_items(n, bw, level)
        for slot, it in items:
            if not is_link:
                out.append((base + slot, it))
                continue
            b = blocks.get(it)
            if b is None:
                raise Fault(_status("ERR_MISSING_BLOCK"))
            if seen is not None:
                seen.add(it)
            rec(_strict(b), level - 1, base + slot * width(bw) ** level)

    rec(node, h, 0)
    return out


def get(blocks, root, i, seen):
    """Amtv0::get(i) with recording → the value item or None."""
    bw, h, _, node = read_root(blocks[root], 0)
    seen.add(root)
    if i >= 8 ** (h + 1):
        return None
    for level in range(h, -1, -1):
        is_link, items = _node_items(node, bw, level)
        slot = i // 8 ** level % 8
        hit = dict(items).get(slot)
        if hit is None or (not is_link and level != 0):
            return None
        if not is_link:
            return hit
        seen.add(hit)
        node = _strict(blocks[hit])
    return None


def honest_verdicts(case, result):
    """What the verifier says of a valid case's own proofs: true, except for an event at index 2^64 − 1 of an AMT with height·bw = 64.
    `get` finds the child slot as i / nodes_for_height with nodes_for_height saturated to 2^64 − 1 (fvm_ipld_amt), which sends
    2^64 − 1 to slot 1 while `for_each` found it in slot 0: such a proof does not verify, in the reference as here."""
    out = []
    for p in result.proofs:
        a = case.amts.get(p.exec_index)
        out.append(not (a is not None and a.bw * a.height == 64 and p.event_index == U64 - 1))
    return out


def _matches(ev, events):
    emitter, entries = ev
    log = P.extract_evm_log(entries)
    return log is not None and len(log[0]) >= 2 and log[0][0] == events.t0 and log[0][1] == events.t1, log, emitter


def truth(case):
    """Expected result of a valid case from the restatement: {matching, proofs [(exec, event, emitter, topics, data, msg)], witness}
    (witness: the set of CIDs), or Fault."""
    ts, blocks, events = case.ts, case.blocks, case.events
    seen = set(bytes(c) for c in ts.parent_cids) | {bytes(ts.child_cid), bytes(ts.receipts_root)}
    seen |= {bytes(c) for c in ts.parent_txmeta_cids}
    exec_order = []
    for tm in ts.parent_txmeta_cids:
        for root in cbor2.loads(blocks[bytes(tm)]):
            for _, c in walk(blocks, _cid(root), 0, seen):
                c = _cid(c)
                if c not in exec_order:
                    exec_order.append(c)
    hits = {}
    for i in range(int(ts.n_receipts)):
        if ts.has_events_root[i]:
            evs = walk(blocks, bytes(ts.events_roots[i]))
            h = [(j, log, em) for j, ev in evs for ok, log, em in [_matches(ev, events)] if ok]
            if h:
                hits[i] = h
    proofs = []
    for i in sorted(hits):
        if i >= len(exec_order):
            raise Fault(_status("ERR_MISSING_EXEC"))
        if get(blocks, bytes(ts.receipts_root), i, seen) is None:
            continue
        walk(blocks, bytes(ts.events_roots[i]), 3, seen)
        for j, log, em in hits[i]:
            proofs.append((i, j, em, tuple(log[0]), log[1], exec_order[i]))
    return dict(matching=sorted(hits), proofs=proofs, witness=seen, n_exec=len(exec_order))


# ------------------------------------------------------------------ tipsets
def chain_receipts(blocks, ts):
    """{index: receipt bytes} of ts's receipts AMT."""
    return {i: cbor2.dumps(v) for i, v in walk(blocks, bytes(ts.receipts_root), 0)}


def _link(cid):
    return cbor2.CBORTag(42, b"\0" + bytes(cid))


def edit_tipset(ts, blocks, roots, receipts_height=None, holes=(), rpc_roots=None, receipts_root=None):
    """ts with receipt i's events root set to roots[i] (a CID or None) in the receipts AMT and in the descriptor, the receipts AMT
    rewritten at `receipts_height` without the receipts in `holes`, and the child header's [9] receipts root and CID updated.
    rpc_roots {i: CID}: the descriptor's events root of receipt i differs from the chain's. receipts_root: a ready receipts-AMT root
    CID (the receipts are then not rewritten). `blocks` gains the blocks written. → EditedTipset."""
    n = int(ts.n_receipts)
    ev = np.array(ts.events_roots, copy=True)
    has = np.array(ts.has_events_root, copy=True)
    if receipts_root is None:
        recs = {}
        for i, raw in chain_receipts(blocks, ts).items():
            ec, ret, gas, er = cbor2.loads(raw)
            if i in roots:
                er = roots[i]
            elif er is not None:
                er = _cid(er)
            if i not in holes:
                recs[i] = receipt(ec, ret, gas, er)
        receipts_root = build_receipts_amt(blocks, recs, receipts_height).root
    for i, r in roots.items():
        has[i] = r is not None
        ev[i] = np.frombuffer(r, dtype=np.uint8) if r is not None else 0
    for i, r in (rpc_roots or {}).items():
        has[i] = 1
        ev[i] = np.frombuffer(r, dtype=np.uint8)
    child = cbor2.loads(blocks[bytes(ts.child_cid)])
    assert cbor2.dumps(child) == blocks[bytes(ts.child_cid)]
    child[9] = _link(receipts_root)
    child_cid = blocks.put(cbor2.dumps(child))
    cids, offs, lens, blob = blocks.flat()
    assert len(ev) == n
    return EditedTipset(ts, cids=cids, offsets=offs, lengths=lens, blob=blob, n_blocks=len(lens), events_roots=ev, has_events_root=has,
                        receipts_root=np.frombuffer(receipts_root, dtype=np.uint8).copy(),
                        child_cid=np.frombuffer(child_cid, dtype=np.uint8).copy())


class Case:
    """One tipset of the catalogue. status: None for a valid case, else the expected status (index: the receipt it names, or None
    where it is not pinned). big: event indices at or above 2^64 (compared with the C++ oracle only). amts {receipt: EvAmt}."""

    def __init__(self, name, ts, blocks, events, status=None, index=None, big=False, amts=None, holes=()):
        self.name, self.ts, self.blocks, self.events, self.status, self.index, self.big = name, ts, blocks, events, status, index, big
        self.amts, self.holes = amts or {}, set(holes)


@functools.lru_cache(maxsize=None)
def base_tipset(n_receipts=600, seed=83):
    """The synthetic tipset the catalogue starts from: one parent, a few events per receipt, no actor filter."""
    import synth
    return synth.Tipset(synth.default_params(seed=seed, n_receipts=n_receipts, n_parents=1, events_per_receipt=3, match_ppm=100000,
                                             has_actor_filter=0, bw3_permille=0))


def _events(ts):
    return Events(ts.event_signature, ts.topic1)


def _path_sets(bw, h, rng, cap):
    """First and last index of every subtree on the path to one random index (those below `cap`)."""
    w = width(bw)
    x = rng.randrange(min(w ** (h + 1), cap))
    out = set()
    for level in range(h + 1):
        span = w ** (level + 1)
        lo = x - x % span
        out |= {lo, lo + span - 1}
    return {i for i in out if i < cap}


def valid_amts(blocks, ev, big):
    """(name, EvAmt) of the valid hand-built events AMTs. big=False: every index below 2^64; big=True: AMTs holding indices ≥ 2^64."""
    out = []
    for bw in range(1, 9):
        w = width(bw)
        rng = random.Random(bw)
        for h in sorted({0, 1, 2, max_height(bw)}):
            top = w ** (h + 1)
            if big:
                if top <= U64:
                    continue
                idx = {U64, U64 + 5, top - 1, top - w, U64 - 1, 0} | {rng.randrange(U64, top) for _ in range(4)}
                out.append((f"bw{bw}-h{h}-beyond-2^64", build_events_amt(blocks, {i: ev.mixed(k) for k, i in enumerate(sorted(idx))}, bw, h)))
                continue
            cap = min(top, U64)
            sets = {"zero": {0}, "width-1": {w - 1}, "path": _path_sets(bw, h, rng, cap),
                    "sparse": {rng.randrange(cap) for _ in range(9)} | {cap - 1 if cap < U64 else cap - 2}}
            for sname, idx in sets.items():
                vals = {i: (ev.mixed(k) if sname in ("path", "sparse") else ev.match_b(k)) for k, i in enumerate(sorted(idx))}
                out.append((f"bw{bw}-h{h}-{sname}", build_events_amt(blocks, vals, bw, h)))
                if sname == "sparse" and min_height(list(idx), bw) != h:
                    out.append((f"bw{bw}-hmin-{sname}", build_events_amt(blocks, vals, bw)))
    if big:
        return out
    # the deepest legal walk: bit width 1, height 64, one value at 2^64 − 2 (65 frames)
    out.append(("bw1-h64-deepest", build_events_amt(blocks, {U64 - 2: ev.match_a(7)}, 1, 64)))
    # single-node roots around pass 1's staged header limit: count fields of 1, 2, 3, 5 and 9 bytes
    for bw in (6, 7, 8):
        for nv in (0, 1, 23, 24, 256):
            nv = min(nv, width(bw))
            for count in (nv, 200, 1000, 1 << 20, 1 << 40):
                vals = {i: ev.mixed(i) for i in range(nv)}
                out.append((f"bw{bw}-single-nv{nv}-count{count}", build_events_amt(blocks, vals, bw, 0, count=count)))
    # empty roots above height 0
    for bw in range(1, 9):
        for h in sorted({1, 2, max_height(bw)}):
            out.append((f"bw{bw}-h{h}-empty", build_events_amt(blocks, {}, bw, h)))
    return out


def valid_case(ts, big=False):
    """Every valid hand-built events AMT under a receipt of its own (receipts 0, 1, 2, …) in one tipset."""
    blocks, _, _ = base_blocks(ts)
    ev = _events(ts)
    amts = valid_amts(blocks, ev, big)
    assert len(amts) <= int(ts.n_receipts)
    roots = {i: a.root for i, (_, a) in enumerate(amts)}
    e = edit_tipset(ts, blocks, roots)
    c = Case("valid-big" if big else "valid", e, blocks, ev, big=big, amts={i: a for i, (_, a) in enumerate(amts)})
    c.names = {i: n for i, (n, _) in enumerate(amts)}
    return c


FAULT_RECEIPT = 77


def _fault(ts, name, make, status, index=FAULT_RECEIPT, drop=()):
    """A tipset whose receipt `index` carries the root `make(blocks, ev)` writes; `drop`: a callable giving CIDs removed afterwards."""
    blocks, _, _ = base_blocks(ts)
    ev = _events(ts)
    made = make(blocks, ev)
    root = made.root if isinstance(made, EvAmt) else made
    gone = set(drop(made)) if drop else set()
    e = edit_tipset(ts, blocks, {index: root})
    if gone:
        blocks = Blocks({c: b for c, b in blocks.items() if c not in gone})
        cids, offs, lens, blob = blocks.flat()
        e = EditedTipset(e, cids=cids, offsets=offs, lengths=lens, blob=blob, n_blocks=len(lens))
    return Case(name, e, blocks, ev, status=status, index=index, amts={index: made} if isinstance(made, EvAmt) else {})


def _node_bytes(bw, bm, links=(), vals=(), blen=None):
    n = bmap_len(bw) if blen is None else blen
    return b"\x83" + head(2, n) + (bm % (1 << 8 * n)).to_bytes(n, "little") + head(4, len(links)) + b"".join(clink(c) for c in links) + \
        head(4, len(vals)) + b"".join(vals)


def _root_bytes(bw, h, count, node):
    return b"\x84" + head(0, bw) + head(0, h) + head(0, count) + node


def fault_cases(ts):
    """Events-AMT roots and nodes the decode contract refuses, each under receipt FAULT_RECEIPT of a tipset of its own."""
    D, M = _status("ERR_DECODE"), _status("ERR_MISSING_BLOCK")
    cases = []

    def leaf(ev, bw, bm, n):
        return _node_bytes(bw, bm, vals=[ev.match_b(k) for k in range(n)])

    for bw in (1, 2, 3, 5, 8):   # a bitmap of the wrong length (one byte short, one byte long)
        for d in (-1, 1):
            blen = bmap_len(bw) + d
            if blen >= 0:
                cases.append(_fault(ts, f"bitmap-len-bw{bw}-{blen}", lambda b, ev, bw=bw, blen=blen: b.put(_root_bytes(bw, 0, 1, _node_bytes(
                    bw, 1, vals=[ev.match_b(0)], blen=blen))), D))
    for bw in (1, 2):            # a bit beyond the node width
        cases.append(_fault(ts, f"bit-beyond-width-bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 0, 2, leaf(ev, bw, 1 | 1 << width(bw), 2))), D))
    for bw in (3, 8):            # popcount ≠ number of values / links
        cases.append(_fault(ts, f"popcount-values-bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 0, 2, leaf(ev, bw, 0b101, 1))), D))
        cases.append(_fault(ts, f"popcount-links-bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 1, 1, _node_bytes(
            bw, 0b11, links=[b.put(leaf(ev, bw, 1, 1))]))), D))
        cases.append(_fault(ts, f"links-and-values-bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 1, 1, _node_bytes(
            bw, 1, links=[b.put(leaf(ev, bw, 1, 1))], vals=[ev.match_b(1)]))), D))
        cases.append(_fault(ts, f"values-above-0-bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 1, 1, leaf(ev, bw, 1, 1))), D))
        cases.append(_fault(ts, f"links-at-0-bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 0, 1, _node_bytes(
            bw, 1, links=[b.put(leaf(ev, bw, 1, 1))]))), D))
        cases.append(_fault(ts, f"trailing-byte-root-bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 0, 1, leaf(ev, bw, 1, 1)) + b"\x00"), D))
        cases.append(_fault(ts, f"trailing-byte-node-bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 1, 1, _node_bytes(
            bw, 1, links=[b.put(leaf(ev, bw, 1, 1) + b"\x00")]))), D))
    for bw in (0, 9):
        cases.append(_fault(ts, f"bw{bw}", lambda b, ev, bw=bw: b.put(_root_bytes(bw, 0, 1, _node_bytes(3, 1, vals=[ev.match_b(0)]))), D))
    for bw in range(1, 9):       # one level too tall
        cases.append(_fault(ts, f"height-bw{bw}-{max_height(bw) + 1}", lambda b, ev, bw=bw: chain_root(b, bw, max_height(bw) + 1,
                                                                                                    max_height(bw) + 1, ev.match_b(0)), D))
    for bw in range(2, 9):       # heights whose product with bw wraps to ≤ 64
        for h in overflow_heights(bw):
            h32 = h & 0xFFFFFFFF
            depth = h32 if h32 <= 70 else 70
            # a chain as deep as the truncated height (1 proof if the height were taken mod 2^32), else 70 levels under it
            cases.append(_fault(ts, f"wrap-bw{bw}-h{h:#x}", lambda b, ev, bw=bw, h=h, depth=depth, h32=h32: chain_root(
                b, bw, h, depth, ev.match_b(1) if h32 <= 70 else None), D))
    for bw in (1, 3, 8):         # a missing child and an undecodable node at every level of a full-height AMT
        h = max_height(bw)
        rng = random.Random(50 + bw)
        x = rng.randrange(min(width(bw) ** (h + 1), U64))
        vals_idx = [0, x]
        for level in range(h):
            span = width(bw) ** (level + 1)
            base = x - x % span
            mk = lambda b, ev, bw=bw, h=h, bad=(): build_events_amt(b, {i: ev.mixed(k) for k, i in enumerate(sorted(set(vals_idx)))}, bw, h, bad=bad)
            cases.append(_fault(ts, f"missing-bw{bw}-l{level}", mk, M, drop=lambda a, level=level, base=base: [a.nodes[(level, base)]]))
            if level % 4 == 0 or level == h - 1:
                cases.append(_fault(ts, f"undecodable-bw{bw}-l{level}", lambda b, ev, mk=mk, level=level, base=base: mk(b, ev, bad={(level, base)}), D))
    return cases


# receipts at the edges of a warp (32) and of a pass-1 CTA (128)
HOLES = (0, 31, 32, 63, 127, 128, 255, 256)


def receipts_cases(ts):
    """The receipts AMT at every height from the minimal one up to 21, without the matching receipts HOLES (their proofs are dropped);
    an RPC events root that differs from the chain's."""
    ev = _events(ts)
    cases = []
    n = int(ts.n_receipts)
    for h in range(min_height([n - 1], 3), RECEIPTS_MAX_HEIGHT + 1):
        blocks, _, _ = base_blocks(ts)
        roots = {i: build_events_amt(blocks, {3 * i: ev.match_b(i), 3 * i + 1: ev.other(i)}, 5).root for i in HOLES}
        e = edit_tipset(ts, blocks, roots, receipts_height=h, holes=HOLES)
        cases.append(Case(f"receipts-h{h}-holes", e, blocks, ev, holes=HOLES))
    blocks, _, _ = base_blocks(ts)
    chain = {i: build_events_amt(blocks, {0: ev.match_b(i)}, 3).root for i in (5, 130)}
    rpc = {5: build_events_amt(blocks, {9: ev.match_a(5), 2: ev.match_b(5)}, 4).root, 130: build_events_amt(blocks, {}, 2).root}
    e = edit_tipset(ts, blocks, chain, rpc_roots=rpc)
    cases.append(Case("rpc-root-differs", e, blocks, ev))
    return cases


def receipts_overflow_cases(ts):
    """Receipts-AMT roots (v0, bw 3) whose height wraps: (k·2^64 + m) / 3 with m ≤ 64, over a chain of one-link nodes."""
    cases = []
    ev = _events(ts)
    for h in overflow_heights(3):
        blocks, _, _ = base_blocks(ts)
        root = chain_root(blocks, 3, h, 3, None, version=0)
        e = edit_tipset(ts, blocks, {}, receipts_root=root)
        cases.append(Case(f"receipts-wrap-h{h:#x}", e, blocks, ev, status=_status("ERR_DECODE")))
    return cases


def message_overflow_cases(ts):
    """Message-AMT roots (v0) whose height wraps, as the BLS AMT of a parent block (tests/message_amts.py's tipsets)."""
    from tests import message_amts as MA
    cases = []
    for h in overflow_heights(3):
        blocks, u, _ = base_blocks(ts)
        bls = MA.Amt(chain_root(blocks, 3, h, 3, clink(u[0]), version=0), {}, {}, h)
        secp = MA.build_amt(blocks, {0: u[1]})
        c = MA.hand_tipset(f"message-wrap-h{h:#x}", ts, (bls, secp), 1, blocks, status=_status("ERR_DECODE"))
        cases.append(Case(c.name, c.ts, c.blocks, _events(ts), status=c.status))
    return cases


def catalogue(ts):
    return [valid_case(ts), valid_case(ts, big=True)] + receipts_cases(ts) + fault_cases(ts) + receipts_overflow_cases(ts) + \
        message_overflow_cases(ts)
