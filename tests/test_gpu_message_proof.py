"""Event proofs for the logs of given messages (ipcfp_generate_message_log_proof*, ipcfp_plan_fetch_message_log_resident) on the GPU.

Two yardsticks: the merged log-filter call (the whole execution order as the message list gives it byte for byte, and any list gives its
result restricted to the selected receipts), and tests/oracle_messages.py, the call restated in Python. Beside them: a store without the
unselected receipts' events AMTs, or with other bytes under their CIDs, gives the same result; faults in selected receipts carry the
log-filter call's status and index; every proof verifies; the fetch planner converges to the restated read set; refusals launch nothing."""
import ctypes as C

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import oracle_logs as OL
from tests import oracle_messages as OM
from tests.test_gpu_log_filter import _digest, _json_sha, _pack, _same_result
from tests.util import assert_event_results_equal, dict_of

pytestmark = pytest.mark.gpu

U64 = 2 ** 64 - 1


def _spec_filter(api, ts):
    spec = api.EventProofSpec(ts.event_signature, ts.topic1, None if ts.actor_filter is None else int(ts.actor_filter))
    return api.LogFilter.from_spec(spec)


def _run(fn):
    try:
        return ("ok", fn())
    except A.IpcfpError as e:
        return ("err", e.status, e.index)


def _cids(lst):
    return np.frombuffer(b"".join(lst), np.uint8).reshape(-1, 38) if lst else np.zeros((0, 38), np.uint8)


def _filters(api, ts, d, rng):
    """None (every log), the spec's filter and a few random filters over the tipset's logs."""
    out = [None, _spec_filter(api, ts)]
    logs = OL.candidate_logs(d, ts)
    for _ in range(3):
        if not logs:
            break
        e, t = logs[int(rng.integers(len(logs)))]
        npos = int(rng.integers(0, min(len(t), 3) + 1))
        topics = [t[k] if rng.random() < 0.5 else None for k in range(npos)]
        out.append(api.LogFilter([e] if rng.random() < 0.5 else None, topics))
    return out


class _Masked:
    """The tipset with the events roots of every receipt outside `keep` taken away: the log-filter call on it runs the restricted loop
    (pass 1 over the kept receipts, pass 2 over those that match), so its result and its first fault are the message call's."""

    def __init__(self, ts, keep):
        self._ts = ts
        h = np.zeros(int(ts.n_receipts), np.uint8)
        for i in keep:
            h[i] = 1 if ts.has_events_root[i] else 0
        self.has_events_root = h

    def __getattr__(self, name):
        return getattr(self._ts, name)


def _restricted(full, keep):
    """The log-filter result restricted to the receipts in keep: (matching, proof keys)."""
    return [i for i in full.matching.tolist() if i in keep], [p.key() for p in full.proofs if p.exec_index in keep]


def _check_subset(api, ts, store, tip, d, msgs, flt):
    """The call against the Python restatement and against the log-filter result restricted to the selection."""
    got, idx = store.generate_message_log_proof_resident(tip, _cids(msgs), flt)
    ef, pos = (set(), []) if flt is None else OL.filter_of(flt)
    exp = OM.generate_message_log_proof(d, ts, msgs, ef, pos)
    assert idx.tolist() == exp["exec_indices"]
    assert got.matching.tolist() == exp["matching"]
    keys = [(i, j, e, tuple(bytes(t) for t in tp), bytes(dt), bytes(m)) for i, j, e, tp, dt, m in exp["proofs"]]
    assert [p.key() for p in got.proofs] == keys
    assert [bytes(c) for c in got.witness.cids] == exp["witness"]
    full = store.generate_log_proof_resident(tip, flt if flt is not None else api.LogFilter())
    sel = {i for i in exp["exec_indices"] if i != U64 and i < int(ts.n_receipts)}
    m, k = _restricted(full, sel)
    assert got.matching.tolist() == m and [p.key() for p in got.proofs] == k
    masked = store.generate_log_proof(_Masked(ts, sel), flt if flt is not None else api.LogFilter())
    _same_result(masked, got)
    ref = OM.CppOracle(ts).generate(ts, msgs, flt)
    assert ref[0] == "ok" and ref[2] == idx.tolist()
    assert_event_results_equal(got, ref[1])
    return got, idx


# ------------------------------------------------------------------ 1. the whole execution order gives the log-filter call
@pytest.mark.parametrize("which", ["ts1", "ts2", "ts3_small"])
@pytest.mark.parametrize("flags", [0, A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE, A.SCAN_SKIP_TX_AMTS])
def test_whole_execution_order_is_the_log_filter_call(api, request, which, flags):
    ts = request.getfixturevalue(which)
    d = dict_of(ts)
    store = api.BlockStore.from_tipset(ts, verify_cids=True)
    tip = store.upload_tipset(ts)
    order = OM.execution_order(d, ts)
    for flt in _filters(api, ts, d, np.random.default_rng(len(order))):
        a = store.generate_log_proof_resident(tip, flt if flt is not None else api.LogFilter(), flags)
        b, idx = store.generate_message_log_proof_resident(tip, _cids(order), flt, flags)
        c, _ = store.generate_message_log_proof(ts, _cids(order), flt, flags)
        _same_result(a, b, flags & A.WITNESS_BY_REFERENCE)
        _same_result(a, c, flags & A.WITNESS_BY_REFERENCE)
        assert idx.tolist() == list(range(len(order)))


def test_whole_execution_order_on_hand_built_amts(api):
    """Every case of tests/event_amts.py and the message-AMT cases whose parents share messages: the call with the whole execution
    order equals the log-filter call, or fails with its status and index."""
    from tests import event_amts as E
    from tests import message_amts as MA
    cases = [(c.name, c.ts) for c in E.catalogue(E.base_tipset())]
    cases += [(c.name, c.ts) for c in MA.shared_cases(MA.base_tipset())]
    n = 0
    for name, ts in cases:
        store = api.BlockStore.from_tipset(ts)
        tip = store.upload_tipset(ts)
        try:
            order = OM.execution_order(dict_of(ts), ts)
        except Exception:
            order = []
        a = _run(lambda: store.generate_log_proof_resident(tip, api.LogFilter(), A.RESULT_JSON))
        b = _run(lambda: store.generate_message_log_proof_resident(tip, _cids(order), None, A.RESULT_JSON))
        if a[0] == "err" and a[1] == A.ERR_MISSING_EXEC:
            # a matching receipt past the execution order fails the log-filter call; no message selects it, so the message call is the
            # log-filter call on the receipts the order covers
            a = _run(lambda: store.generate_log_proof(_Masked(ts, range(min(len(order), int(ts.n_receipts)))), api.LogFilter(), A.RESULT_JSON))
        if a[0] != "ok":
            if order:   # a tipset whose message AMTs fail gives no order to ask for; the call then fails alike with an empty list
                assert a == b, name
            continue
        assert b[0] == "ok", (name, b)
        # the data blob through the proofs that index it: the slots of receipts missing from the receipts AMT are never written
        a, b = a[1], b[1][0]
        assert a.matching.tolist() == b.matching.tolist() and a.n_exec == b.n_exec, name
        assert [p.key() for p in a.proofs] == [p.key() for p in b.proofs] and np.array_equal(a.raw_proofs, b.raw_proofs), name
        assert np.array_equal(a.witness.cids, b.witness.cids) and a.witness.blocks() == b.witness.blocks() and a.json == b.json, name
        n += 1
    assert n > 10


# ------------------------------------------------------------------ 2. subsets
@pytest.mark.parametrize("which", ["ts1", "ts2", "ts3_small"])
def test_subsets(api, synth_mod, request, which):
    ts = request.getfixturevalue(which)
    d = dict_of(ts)
    store = api.BlockStore.from_tipset(ts, verify_cids=True)
    tip = store.upload_tipset(ts)
    order = OM.execution_order(d, ts)
    rng = np.random.default_rng(11)
    nr = int(ts.n_receipts)
    no_root = [order[i] for i in range(min(nr, len(order))) if not ts.has_events_root[i]]
    past = order[nr:]
    stranger = [bytes(c) for c in rng.integers(0, 256, (3, 38), dtype=np.uint8)]
    stranger = [order[0][:6] + s[6:] for s in stranger] if order else stranger
    full = store.generate_log_proof_resident(tip, api.LogFilter())
    some = [order[i] for i in full.matching.tolist()[:5]]
    lists = {
        "empty": [],
        "one": some[:1],
        "many": [order[int(i)] for i in rng.choice(len(order), size=min(len(order), 200), replace=False)],
        "duplicates": some[:3] * 3 + some[:1],
        "not executed": stranger + some[:2],
    }
    if no_root:
        lists["no events root"] = no_root[:4] + some[:1]
    if past:
        lists["past n_receipts"] = past[:3] + some[:1]
    for name, msgs in lists.items():
        for flt in _filters(api, ts, d, rng)[:3]:
            got, idx = _check_subset(api, ts, store, tip, d, msgs, flt)
            if name == "empty":
                assert len(got.proofs) == 0 and len(idx) == 0
            if name == "not executed":
                assert idx.tolist()[:3] == [U64] * 3


class _Truncated:
    """The tipset described with only its first m receipts: the messages executed at positions >= m have no receipt."""

    def __init__(self, ts, m):
        self._ts = ts
        self.n_receipts = m
        self.events_roots = np.ascontiguousarray(np.asarray(ts.events_roots)[:m])
        self.has_events_root = np.ascontiguousarray(np.asarray(ts.has_events_root)[:m])

    def __getattr__(self, name):
        return getattr(self._ts, name)


def _compare_hand_built(api, name, ts, msgs):
    """The call against the C++ restatement (result and exec indices, or status and index) and, when it succeeds, against the
    log-filter call on the tipset with the other receipts' events roots taken away. → 'ok' or 'err'."""
    nr = int(ts.n_receipts)
    store = api.BlockStore.from_tipset(ts)
    got = _run(lambda: store.generate_message_log_proof(ts, _cids(msgs), None, A.RESULT_JSON))
    ref = OM.CppOracle(ts).generate(ts, msgs)
    if ref[0] == "err":
        assert got == ref, name
        return "err"
    assert got[0] == "ok", (name, got)
    res, idx = got[1]
    assert idx.tolist() == ref[2], name
    # the data blob through the proofs that index it: the slots of receipts missing from the receipts AMT are never written
    assert res.matching.tolist() == ref[1].matching.tolist() and [p.key() for p in res.proofs] == [p.key() for p in ref[1].proofs], name
    assert np.array_equal(res.witness.cids, ref[1].witness.cids) and res.witness.blocks() == ref[1].witness.blocks(), name
    sel = {i for i in ref[2] if i != U64 and i < nr}
    masked = store.generate_log_proof(_Masked(ts, sel), api.LogFilter(), A.RESULT_JSON)
    assert masked.matching.tolist() == res.matching.tolist() and np.array_equal(masked.raw_proofs, res.raw_proofs), name
    assert np.array_equal(masked.witness.cids, res.witness.cids) and masked.json == res.json, name
    return "ok"


def test_rootless_receipts_and_positions_past_the_receipts(api, synth_mod):
    """Receipts without an events root (a synthetic tipset with null roots), messages executed at positions >= n_receipts (the same
    tipset described with fewer receipts, and message_amts' parents that share messages), together with receipts that match."""
    ts = synth_mod.Tipset(synth_mod.default_params(seed=0x3E55, n_receipts=3000, events_per_receipt=6, match_ppm=100000, null_root_permille=150))
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    nr = int(ts.n_receipts)
    rootless = [order[i] for i in range(min(nr, len(order))) if not ts.has_events_root[i]]
    with_root = [order[i] for i in range(min(nr, len(order))) if ts.has_events_root[i]]
    assert len(rootless) > 100 and len(with_root) > 100
    assert _compare_hand_built(api, "rootless", ts, rootless[:40] + with_root[::50]) == "ok"
    short = _Truncated(ts, nr // 2)
    past = order[nr // 2:]
    assert len(past) > 100
    assert _compare_hand_built(api, "past n_receipts", short, past[::20] + order[:nr // 2:25] + rootless[:3]) == "ok"
    from tests import message_amts as MA
    for c in MA.shared_cases(MA.base_tipset()):
        o = OM.execution_order(dict_of(c.ts), c.ts)
        m = min(len(o), int(c.ts.n_receipts)) * 2 // 3
        assert len(o) > m
        assert _compare_hand_built(api, c.name, _Truncated(c.ts, m), o[m:][:10] + o[:m:17]) == "ok"


def test_subsets_on_hand_built_events_amts(api):
    """Every case of tests/event_amts.py (events AMTs at every bit width and height, receipts-AMT holes, refused roots and nodes, missing
    blocks), with a selection that holds the faulty receipt: the C++ restatement's result or status and index."""
    from tests import event_amts as E
    n_fail = 0
    for c in E.catalogue(E.base_tipset()):
        if c.big:
            continue
        ts = c.ts
        try:
            order = OM.execution_order(dict_of(ts), ts)
        except Exception:
            continue
        rng = np.random.default_rng(len(c.name))
        msgs = [order[int(i)] for i in rng.choice(len(order), size=min(len(order), 30), replace=False)] + [order[E.FAULT_RECEIPT]]
        n_fail += _compare_hand_built(api, c.name, ts, msgs) == "err"
    assert n_fail > 3


# ------------------------------------------------------------------ 3. only its blocks are read
def _stores_without_unselected(ts, d, selected):
    """(store without the unselected receipts' events-AMT blocks, store holding other bytes under their CIDs), neither CID-checked."""
    keep = OM.events_blocks(d, ts, selected) | set(OM.read_set(d, ts, []))
    drop = OM.events_blocks(d, ts, range(int(ts.n_receipts))) - keep
    assert drop
    held = {c: b for c, b in d.items() if c not in drop}
    rng = np.random.default_rng(5)
    bent = {c: (bytes(rng.integers(0, 256, len(b), dtype=np.uint8)) if c in drop else b) for c, b in d.items()}
    return held, bent


@pytest.mark.parametrize("which", ["ts1", "ts2"])
def test_only_selected_events_amts_are_read(api, request, which):
    ts = request.getfixturevalue(which)
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    complete = api.BlockStore.from_tipset(ts)
    ctip = complete.upload_tipset(ts)
    full = complete.generate_log_proof_resident(ctip, api.LogFilter())
    msgs = [order[i] for i in full.matching.tolist()[::7][:20]]
    selected, _ = OM.select(order, int(ts.n_receipts), msgs)
    held, bent = _stores_without_unselected(ts, d, selected)
    want, widx = complete.generate_message_log_proof_resident(ctip, _cids(msgs), None, A.RESULT_JSON)
    for blocks in (held, bent):
        store = api.BlockStore(*_pack(blocks))
        tip = store.upload_tipset(ts)
        got, idx = store.generate_message_log_proof_resident(tip, _cids(msgs), None, A.RESULT_JSON)
        assert idx.tolist() == widx.tolist()
        _same_result(want, got)
        assert _run(lambda: store.generate_log_proof_resident(tip, api.LogFilter()))[0] == "err"


# ------------------------------------------------------------------ 4. faults
def _damage(d, cid, how):
    out = dict(d)
    if how == "missing":
        del out[cid]
    elif how == "truncated":
        out[cid] = d[cid][:max(1, len(d[cid]) // 2)]
    else:
        b = bytearray(d[cid])
        b[len(b) // 3] ^= 0x40
        out[cid] = bytes(b)
    return out


@pytest.mark.parametrize("how", ["missing", "truncated", "flipped"])
def test_faults_in_selected_receipts_and_message_amts(api, ts1, how):
    ts = ts1
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    complete = api.BlockStore.from_tipset(ts)
    full = complete.generate_log_proof_resident(complete.upload_tipset(ts), api.LogFilter())
    m = full.matching.tolist()
    i = m[len(m) // 2]
    msgs = [order[j] for j in m[::5]] + [order[i]]
    rec = OM.P.Recorder(d)
    OM.P.Amt(bytes(ts.receipts_root), rec, 0).get(i)
    receipt_path = sorted(rec.seen - {bytes(ts.receipts_root)})
    tx = [bytes(c) for c in ts.parent_txmeta_cids]
    msg_blocks = sorted(OM.read_set(d, ts, []) - set(bytes(c) for c in ts.parent_cids) - {bytes(ts.child_cid), bytes(ts.receipts_root)} - set(tx))
    targets = [bytes(ts.events_roots[i])] + receipt_path[-1:] + msg_blocks[:1]
    selected, _ = OM.select(order, int(ts.n_receipts), msgs)
    n_fail = 0
    for cid in targets:
        bad = _damage(d, cid, how)
        store = api.BlockStore(*_pack(bad))
        tip = store.upload_tipset(ts)
        got = _run(lambda: store.generate_message_log_proof_resident(tip, _cids(msgs)))
        ref = _run(lambda: store.generate_log_proof(_Masked(ts, selected), api.LogFilter()))
        if got[0] == "ok":
            got = ("ok",)
        if ref[0] == "ok":
            ref = ("ok",)
        try:
            OM.generate_message_log_proof(bad, ts, msgs)
            py_ok = True
        except Exception:
            py_ok = False
        assert got == ref, (cid.hex(), got, ref)
        cpp = OM.CppOracle(arrays=_pack(bad)).generate(ts, msgs)
        assert (("ok",) if cpp[0] == "ok" else cpp) == got, (cid.hex(), got, cpp)
        assert py_ok == (got[0] == "ok"), cid.hex()
        n_fail += got[0] != "ok"
    assert n_fail >= (2 if how != "flipped" else 0)   # a flipped byte inside a digest or a data field still decodes


# ------------------------------------------------------------------ 5. verification
def test_proofs_verify(api, ts2):
    ts = ts2
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    flt = _spec_filter(api, ts)
    msgs = order[::3]
    for f in (None, flt):
        got, _ = store.generate_message_log_proof_resident(tip, _cids(msgs), f, A.RESULT_JSON)
        assert len(got.proofs) > 0
        assert all(api.verify_event_proofs(got.witness, ts, got))
        assert all(api.verify_event_proofs(got.witness, ts, got, filter_spec=f if f is not None else api.LogFilter()))
        v = api.verify_bundle_json(got.json)
        assert len(v.event_results) == len(got.proofs) and all(v.event_results)


# ------------------------------------------------------------------ 6. planning
def _plan_loop(api, ts, d, plan):
    held, fetched, rounds = {}, set(), 0
    while True:
        store = api.BlockStore(*_pack(held))
        tip = store.upload_tipset(ts)
        want = [bytes(c) for c in plan(store, tip).cids]
        if not want:
            return store, tip, fetched, rounds
        assert all(c in d and c not in held for c in want)
        held.update((c, d[c]) for c in want)
        fetched |= set(want)
        rounds += 1
        assert rounds < 200


@pytest.mark.parametrize("which", ["ts1", "ts2"])
def test_fetch_planning(api, request, which):
    ts = request.getfixturevalue(which)
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    complete = api.BlockStore.from_tipset(ts)
    full = complete.generate_log_proof_resident(complete.upload_tipset(ts), api.LogFilter())
    msgs = [order[i] for i in full.matching.tolist()[::9][:12]] + [order[-1]]
    flt = None
    # round 1 on an empty store: the base roots only (no message-AMT block is held yet)
    empty = api.BlockStore(*_pack({}))
    p1 = {bytes(c) for c in empty.plan_fetch_messages(empty.upload_tipset(ts), _cids(msgs)).cids}
    base = {bytes(c) for c in ts.parent_cids} | {bytes(ts.child_cid), bytes(ts.receipts_root)} | {bytes(c) for c in ts.parent_txmeta_cids}
    assert p1 == base
    # a store holding every message-AMT block: the selected receipts' events AMTs, and nothing of the unselected ones
    msg_only = {c: d[c] for c in OM.read_set(d, ts, [])}
    s2 = api.BlockStore(*_pack(msg_only))
    p2 = {bytes(c) for c in s2.plan_fetch_messages(s2.upload_tipset(ts), _cids(msgs)).cids}
    selected, _ = OM.select(order, int(ts.n_receipts), msgs)
    roots = {bytes(ts.events_roots[i]) for i in selected if ts.has_events_root[i]}
    assert p2 == roots - set(msg_only)
    # the loop converges to the restated read set, the call's result, and fewer blocks than the log-filter loop
    store, tip, fetched, rounds = _plan_loop(api, ts, d, lambda s, t: s.plan_fetch_messages(t, _cids(msgs), flt))
    assert fetched == OM.read_set(d, ts, msgs) and rounds > 1
    got, _ = store.generate_message_log_proof_resident(tip, _cids(msgs), flt, A.RESULT_JSON)
    want, _ = complete.generate_message_log_proof(ts, _cids(msgs), flt, A.RESULT_JSON)
    assert got.json == want.json
    _, _, fetched_logs, _ = _plan_loop(api, ts, d, lambda s, t: s.plan_fetch_logs(t, api.LogFilter()))
    assert fetched < fetched_logs


# ------------------------------------------------------------------ 7. scale
@pytest.fixture(scope="module")
def ts1m(synth_mod):
    return synth_mod.Tipset(synth_mod.config_params(4, n_receipts=1_000_000))


def _records(r):
    """The EventProof fields of a raw result as a structured array (see test_gpu_log_filter._digest)."""
    n = int(r.n_proofs)
    return np.frombuffer(A._arr(C.cast(r.proofs, C.c_void_p).value, n * C.sizeof(A.EventProofC), np.uint8).tobytes(), dtype=np.dtype({
        "names": ["exec_index", "event_index", "emitter", "message_cid"],
        "formats": [np.uint64, np.uint64, np.uint64, (np.uint8, 38)],
        "offsets": [getattr(A.EventProofC, f).offset for f in ("exec_index", "event_index", "emitter", "message_cid")],
        "itemsize": C.sizeof(A.EventProofC)}))


def test_one_million_receipts(api, ts1m):
    """|M| = 1, 1 000 and IPCFP_MESSAGE_MAX (a call's cap): the all-wildcard log-filter result restricted to M, and the same tipset
    with the events roots outside M taken away by SHA-256 (JSON included). Every receipt of this tipset has a matching event, so the
    full result's proofs name the whole execution order."""
    ts = ts1m
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    f, fkeep = api.LogFilter().as_c()
    L = api.lib()
    out = C.POINTER(A.EventResultC)()
    assert L.ipcfp_generate_log_proof_resident(store._h, tip._h, C.byref(f), 0, C.byref(out)) == A.OK
    try:
        n_exec = int(out.contents.n_exec)
        assert int(out.contents.n_matching) == int(ts.n_receipts) == n_exec
        recs = _records(out.contents).copy()
    finally:
        L.ipcfp_event_result_free(out)
    _, first = np.unique(recs["exec_index"], return_index=True)
    cids = np.ascontiguousarray(recs["message_cid"][first])
    assert len(cids) == n_exec
    rng = np.random.default_rng(1)
    for k in (1, 1000, A.MESSAGE_MAX):
        pick = np.sort(rng.choice(n_exec, size=k, replace=False)).astype(np.uint64)
        sub = np.ascontiguousarray(cids[pick])
        idx = np.zeros(k, np.uint64)
        out = C.POINTER(A.EventResultC)()
        assert L.ipcfp_generate_message_log_proof_resident(store._h, tip._h, sub.ctypes.data, k, None, A.RESULT_JSON, idx.ctypes.data,
                                                           C.byref(out)) == A.OK
        try:
            assert np.array_equal(idx, pick)
            assert A._arr(out.contents.matching_indices, int(out.contents.n_matching), np.uint64).tolist() == pick.tolist()
            exp = recs[np.isin(recs["exec_index"], pick)]
            mine = _records(out.contents)
            for fld in ("exec_index", "event_index", "emitter", "message_cid"):
                assert np.array_equal(mine[fld], exp[fld]), fld
            got = (_digest(out.contents), _json_sha(out.contents.json, int(out.contents.json_len)))
        finally:
            L.ipcfp_event_result_free(out)
        if k == A.MESSAGE_MAX:
            masked = _Masked(ts, set(pick.tolist()))
            d, keep = A.make_tipset_desc(masked)
            out = C.POINTER(A.EventResultC)()
            assert L.ipcfp_generate_log_proof(store._h, C.byref(d), C.byref(f), A.RESULT_JSON, C.byref(out)) == A.OK
            try:
                assert got == (_digest(out.contents), _json_sha(out.contents.json, int(out.contents.json_len)))
            finally:
                L.ipcfp_event_result_free(out)


# ------------------------------------------------------------------ 8. refusals
def test_refusals_launch_nothing(api, ts1):
    store = api.BlockStore.from_tipset(ts1)
    tip = store.upload_tipset(ts1)
    L = api.lib()
    cids = np.zeros((A.MESSAGE_MAX + 1, 38), np.uint8)
    idx = np.zeros(len(cids), np.uint64)
    d, keep = A.make_tipset_desc(ts1)
    bad = A.LogFilterC()
    bad.n_positions = 5
    out = C.POINTER(A.EventResultC)()
    plan = C.POINTER(A.FetchPlanC)()
    cases = [(None, 1, idx.ctypes.data, None), (cids.ctypes.data, 1, None, None), (cids.ctypes.data, A.MESSAGE_MAX + 1, idx.ctypes.data, None),
             (cids.ctypes.data, 1, idx.ctypes.data, C.byref(bad))]
    before = api.kernel_launch_count()
    for ptr, n, ip, fp in cases:
        assert L.ipcfp_generate_message_log_proof_resident(store._h, tip._h, ptr, n, fp, 0, ip, C.byref(out)) == A.ERR_INVALID_ARG
        assert L.ipcfp_generate_message_log_proof(store._h, C.byref(d), ptr, n, fp, 0, ip, C.byref(out)) == A.ERR_INVALID_ARG
        if ip is not None:
            assert L.ipcfp_plan_fetch_message_log_resident(store._h, tip._h, ptr, n, fp, 0, C.byref(plan)) == A.ERR_INVALID_ARG
    assert api.kernel_launch_count() == before
    # the cap itself is accepted
    got, gidx = store.generate_message_log_proof_resident(tip, cids[:A.MESSAGE_MAX])
    assert len(got.proofs) == 0 and (gidx == U64).all()
    with pytest.raises(A.IpcfpError):
        store.plan_fetch_messages(tip, cids[:1], flags=1)
