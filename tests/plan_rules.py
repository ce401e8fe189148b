"""The fetch planner's rules (DESIGN.md §2, "Fetch planning") restated in Python on cbor2 and the Python oracle's decoders, independent
of the library: restate_plan(held, ts, sspecs, especs) gives N(S) \\ S in `Cid` order and |N(S) ∩ S| for the blocks held (test
infrastructure: tests/test_gpu_plan_fetch.py checks the device against it, tests/test_plan_fetch_host.py the per-item code on the CPU)."""
import cbor2
import numpy as np

from oracle import pyoracle as P


# ------------------------------------------------------------------------------------------ the rules, restated
def _link(x):
    if not (isinstance(x, cbor2.CBORTag) and x.tag == 42 and isinstance(x.value, bytes) and len(x.value) == 39 and x.value[0] == 0):
        raise ValueError("not a 38-byte CID link")
    return bytes(x.value[1:])


def _children(kind, raw, bw, tree):
    """The children of one held block under its rule (plan_children): [] when it does not decode."""
    try:
        x = cbor2.loads(raw)
        if kind == "tx":
            if not (isinstance(x, list) and len(x) == 2):
                return []
            return [("msgroot", _link(x[0]), 3, 0), ("msgroot", _link(x[1]), 3, 0)]
        if kind in ("msgroot", "evroot"):
            if kind == "msgroot":
                h, _, node = x
            else:
                bw, h, _, node = x
                if not 1 <= bw <= 8:
                    return []
            if h > 64 or h * bw > 64:
                return []
        else:
            node = x
        bmap, links = node[0], node[1]
        if len(bmap) != (1 if bw <= 3 else 1 << (bw - 3)) or (bw < 3 and bmap[0] >> (1 << bw)):
            return []
        return [("node", _link(c), bw, tree) for c in links]
    except Exception:
        return []


class _Held:
    """get() over the held blocks that records what is needed and what is missing."""

    def __init__(self, held):
        self.held, self.need, self.miss = held, set(), set()

    def get(self, c):
        b = self.held.get(c)
        (self.need if b is not None else self.miss).add(c)
        return b


def _matches(held, root, especs):
    rec = P.Recorder(held)
    try:
        amt = P.Amt(root, rec, 3)
        hit = []

        def f(_, se):
            emitter, entries = se
            for t0, t1, actor in especs:
                if actor is not None and emitter != actor:
                    continue
                log = P.extract_evm_log(entries)
                if log and len(log[0]) >= 2 and log[0][0] == t0 and log[0][1] == t1:
                    hit.append(1)
        amt.for_each(f)
        return bool(hit)
    except Exception:
        return False


def _receipt_path(g, root, i):
    raw = g.held.get(root)
    if raw is None:
        return
    try:
        h, _, node = cbor2.loads(raw)
        if i >= 8 ** (h + 1):
            return
        for lvl in range(h, -1, -1):
            bmap, links = node[0], node[1]
            idx = (i // 8 ** lvl) % 8
            if not links or not (bmap[0] >> idx) & 1:
                return
            c = _link(links[bin(bmap[0] & ((1 << idx) - 1)).count("1")])
            raw = g.get(c)
            if raw is None:
                return
            node = cbor2.loads(raw)
    except Exception:
        return


def _storage_path(g, ts, actor_id, slot):
    raw = g.held.get(bytes(ts.child_cid))
    try:
        if raw is None or _link(cbor2.loads(raw)[8]) != bytes(ts.parent_state_root):
            return
        sr = g.get(bytes(ts.parent_state_root))
        if sr is None:
            return
        actor = P.hamt_get(g, _link(cbor2.loads(sr)[1]), 5, P._id_address(actor_id))
        if actor is None:
            return
        evm = g.get(_link(actor[1]))
        if evm is None:
            return
        P.read_storage_slot(g, _link(cbor2.loads(evm)[2]), slot)
    except P.MissingBlock:
        pass
    except Exception:
        return


def restate_plan(held, ts, sspecs, especs):
    """(M(S) in `Cid` order, |N(S) ∩ S|) for held = {cid: bytes}; especs: [(signature, topic_1, actor or None)]."""
    g = _Held(held)
    front = []
    if especs:
        for c in list(np.asarray(ts.parent_cids).reshape(-1, 38)) + [ts.child_cid, ts.receipts_root]:
            g.get(bytes(c))
        front += [("tx", bytes(c), 3, 0) for c in np.asarray(ts.parent_txmeta_cids).reshape(-1, 38)]
        roots = np.asarray(ts.events_roots).reshape(-1, 38)
        front += [("evroot", bytes(roots[i]), 0, 1) for i in range(int(ts.n_receipts)) if ts.has_events_root[i]]
    if sspecs:
        g.get(bytes(ts.child_cid))
        g.get(bytes(ts.parent_state_root))
    seen, ev_missing = set(), False
    while front:
        nxt = []
        for kind, c, bw, tree in front:
            raw = g.get(c)
            if raw is None:
                ev_missing |= bool(tree)
                continue
            key = (kind, bw if kind == "node" else 0, tree, c)
            if key not in seen:
                seen.add(key)
                nxt += _children(kind, raw, bw, tree)
        front = nxt
    if especs and not ev_missing:
        keys = [(P.keccak256(sig.encode()), P.ascii_to_bytes32(t1), actor) for sig, t1, actor in especs]
        roots = np.asarray(ts.events_roots).reshape(-1, 38)
        for i in range(int(ts.n_receipts)):
            if ts.has_events_root[i] and _matches(held, bytes(roots[i]), keys):
                _receipt_path(g, bytes(ts.receipts_root), i)
    for actor_id, slot in sspecs:
        _storage_path(g, ts, actor_id, bytes(slot))
    return sorted(g.miss, key=P.cid_sort_key), len(g.need)
