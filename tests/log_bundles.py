"""Proof bundles of log filters (ipcfp_generate_log_bundle*) composed from the two restated generators, as generate_proof_bundle composes
its generators: the storage specs, then every filter in order, then the BTreeSet union of the witnesses. The Python composition uses
pyoracle.generate_storage_proof and tests/oracle_logs.generate_log_proof; the C++ one the C++ oracle's storage generator and
tests/oracle_logs.cpp. Also the filter sets the bundle tests run on."""
import numpy as np

import oracle
from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import api
from oracle import pyoracle as P
from tests import oracle_logs as OL

EVM_ACTORS = (1001, 1002, 1003, 1004, 1005, 1006)   # the six contract_state shapes of the synthetic state tree


def spec_filter(event_signature, topic_1, actor=None):
    """LogFilter.from_spec with the CPU keccak (no device needed)."""
    t1 = topic_1.encode()[:32]
    return api.LogFilter(None if actor is None else [int(actor)], [bytes(oracle.keccak256(event_signature.encode())), t1 + bytes(32 - len(t1))])


def filter_of_cspec(cs):
    """The filter an A.EventSpec stands for."""
    return spec_filter(cs.event_signature.decode(), cs.topic_1.decode(), cs.actor_id_filter if cs.has_actor_id_filter else None)


def storage_specs(ts, n):
    """n storage specs over the six contract shapes: present and absent slots."""
    m = int(ts.params.hamt_entries)
    keys = [ts.storage_entry(min(k, m))[0] for k in (0, 1, 3, m // 2)] + [ts.storage_absent_key(k) for k in (0, 1)]
    slots = [bytes(oracle.compute_mapping_slot(k, 0)) for k in keys]
    return [(EVM_ACTORS[j % 6], slots[(5 * j) % len(slots)]) for j in range(n)]


def _rand32(rng, n):
    return [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(n)]


def filter_sets(ts, logs, seed=0):
    """Named lists of 0 to 8 filters: wildcards, n_positions 0-4, value and emitter sets of 1, 4, 5 and 65 536 (both sides of the inline
    switch and the bitmap step), a filter that matches nothing, duplicates and the all-wildcard filter."""
    rng = np.random.default_rng(seed)
    F = api.LogFilter
    spec = spec_filter(ts.event_signature, ts.topic1, ts.actor_filter)
    emitters = sorted({e for e, _ in logs})
    vals = [sorted({t[k] for _, t in logs if len(t) > k}) for k in range(4)]

    def pick(k, n):
        have = vals[k][:max(0, n - 1)] if vals[k] else []
        return have + _rand32(rng, n - len(have))

    nothing = F(topics=_rand32(rng, 1))
    mixed = [spec, F(topics=[None] * 3), F(topics=[pick(0, 4)]), F(topics=[None, pick(1, 5)]), F(emitters=emitters[:5], topics=[]),
             F(topics=[None, None, pick(2, 1), pick(3, 4)]), spec, nothing]
    return {
        "none": [],
        "spec": [spec],
        "wildcard": [F()],
        "nothing": [nothing],
        "positions": [F(topics=[None] * k) for k in range(5)],
        "mixed8": mixed,
        "big": [F(topics=[pick(0, A.LOG_FILTER_MAX_VALUES)]), F(emitters=emitters[:1] + [int(x) for x in rng.integers(1 << 40, 1 << 62, A.LOG_FILTER_MAX_EMITTERS - 1)])],
        "dup_wild": [F(), spec, F()],
    }


def py_bundle(d, ts, sspecs, filters):
    """→ ('ok', dict(storage, events, union)) or ('err', exception name): the first generator that fails, storage first."""
    try:
        st = [P.generate_storage_proof(d, ts, a, bytes(s)) for a, s in sspecs]
        ev = [OL.generate_log_proof(d, ts, *OL.filter_of(f)) for f in filters]
    except Exception as e:   # MissingBlock, KeyError (actor not found), decode errors, IndexError
        return ("err", type(e).__name__)
    union = sorted({c for x in st + ev for c in x["witness"]}, key=P.cid_sort_key)
    return ("ok", dict(storage=st, events=ev, union=union))


def cpp_bundle(ts, sspecs, filters, ostore=None, cpp=None, threads=1):
    """→ ('ok', dict(storage: StorageResultPy or None, events: [EventResultPy], union)) or ('err', status, index)."""
    ostore = ostore or oracle.Store.from_tipset(ts)
    cpp = cpp or OL.CppOracle(ts)
    storage = None
    if sspecs:
        try:
            storage = ostore.generate_storage_proofs(ts, sspecs)
        except A.IpcfpError as e:
            return ("err", e.status, int(e.index))
    events = []
    for f in filters:
        r = cpp.generate(ts, f, threads=threads)
        if r[0] != "ok":
            return r
        events.append(r[1])
    lists = ([storage.witness] if storage else []) + [e.witness for e in events]
    union = sorted({bytes(c) for w in lists for c in w.cids}, key=P.cid_sort_key)
    return ("ok", dict(storage=storage, events=events, union=union))


def assert_compositions_agree(py, cpp):
    assert py[0] == cpp[0], (py, cpp[:1])
    if py[0] != "ok":
        return
    py, cpp = py[1], cpp[1]
    st = cpp["storage"].proofs if cpp["storage"] else []
    assert len(st) == len(py["storage"])
    for p, q in zip(st, py["storage"]):
        assert (p.actor_state_cid, p.storage_root, p.value, p.found) == (q["actor_state_cid"], q["storage_root"], q["value"], q["found"])
    assert len(cpp["events"]) == len(py["events"])
    for r, e in zip(cpp["events"], py["events"]):
        keys = [(i, j, em, tuple(bytes(t) for t in tp), bytes(dt), bytes(m)) for i, j, em, tp, dt, m in e["proofs"]]
        assert r.matching.tolist() == e["matching"] and [p.key() for p in r.proofs] == keys
        assert [bytes(c) for c in r.witness.cids] == e["witness"]
    assert cpp["union"] == py["union"]


def log_matches_any(filters, emitter, topics):
    return any(f.matches(emitter, topics) for f in filters)
