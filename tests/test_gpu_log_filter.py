"""Event proofs for log filters (ipcfp_generate_log_proof*, ipcfp_plan_fetch_log_resident, ipcfp_verify_event_proofs_log) on the GPU.

Two oracles: the spec path itself (a spec and its equivalent filter give the same bytes: matching receipts, proofs, data blob, witness
in both modes, the device JSON, and the same status and index on faulty tipsets), and tests/oracle_logs.py, the generator restated in
Python with the filter as its predicate. Every bundle also passes three verifiers: ipcfp_verify_event_proofs with no filter, the new
call with the same filter, and the C++ oracle's verifier with check_event = None."""
import ctypes as C
import os

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import oracle_logs as OL
from tests.test_gpu_event_shapes import faulted
from tests.util import SHAPES, assert_event_results_equal, dict_of

pytestmark = pytest.mark.gpu

LF_INLINE = 4   # values per position / emitters carried inside the kernel argument (csrc/log_filter.cuh)


def _spec(api, ts):
    return api.EventProofSpec(ts.event_signature, ts.topic1, None if ts.actor_filter is None else int(ts.actor_filter))


def _run(fn):
    try:
        return ("ok", fn())
    except A.IpcfpError as e:
        return ("err", e.status, e.index)


def _same_result(a, b, by_ref=False):
    assert a.matching.tolist() == b.matching.tolist()
    assert a.n_exec == b.n_exec
    assert [p.key() for p in a.proofs] == [p.key() for p in b.proofs]
    assert np.array_equal(a.raw_proofs, b.raw_proofs)
    assert np.array_equal(a.data_blob, b.data_blob)
    assert np.array_equal(a.witness.cids, b.witness.cids)
    assert np.array_equal(a.witness.lengths, b.witness.lengths)
    assert np.array_equal(a.witness.offsets, b.witness.offsets) if by_ref else a.witness.blocks() == b.witness.blocks()
    assert a.json == b.json


@pytest.fixture(scope="module")
def shapes(synth_mod):
    return synth_mod.Tipset(synth_mod.default_params(event_shapes=1, **SHAPES["shapes-nofilter"]))


# ------------------------------------------------------------------ the spec and its filter
@pytest.mark.parametrize("which", ["ts1", "ts2", "ts3_small", "shapes"])
@pytest.mark.parametrize("flags", [0, A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE, A.SCAN_SKIP_TX_AMTS])
def test_spec_and_equivalent_filter_give_the_same_bytes(api, request, which, flags):
    ts = request.getfixturevalue(which)
    store = api.BlockStore.from_tipset(ts, verify_cids=True)
    spec = _spec(api, ts)
    flt = api.LogFilter.from_spec(spec)
    tip = store.upload_tipset(ts)
    a = store.generate_event_proof(ts, spec, flags)
    b = store.generate_log_proof_resident(tip, flt, flags)
    c = store.generate_log_proof(ts, flt, flags)
    _same_result(a, b, flags & A.WITNESS_BY_REFERENCE)
    _same_result(a, c, flags & A.WITNESS_BY_REFERENCE)
    assert len(a.proofs) > 0 or which in ("ts3_small", "shapes")   # config 3's spec matches nothing


@pytest.mark.parametrize("seed", range(4))
def test_spec_and_filter_fail_alike_on_faulty_tipsets(api, synth_mod, seed):
    ts = synth_mod.Tipset(synth_mod.default_params(event_shapes=1, seed=0x5A1 + seed, n_receipts=4000, events_per_receipt=12, match_ppm=80000))
    d = dict_of(ts)
    index_of = {bytes(ts.cids[k]): k for k in range(int(ts.n_blocks))}
    rng = np.random.default_rng(seed)
    bad, _ = faulted(ts, index_of, d, rng, drop_leaf=bool(seed & 1))
    store = api.BlockStore.from_tipset(bad)
    spec = _spec(api, ts)
    a = _run(lambda: store.generate_event_proof(bad, spec))
    b = _run(lambda: store.generate_log_proof(bad, api.LogFilter.from_spec(spec)))
    if a[0] == "ok":
        assert b[0] == "ok"
        _same_result(a[1], b[1])
    else:
        assert a == b


def test_spec_and_filter_on_hand_built_events_amts(api, synth_mod):
    """Every case of tests/event_amts.py (events AMTs at every bit width and height, receipts AMTs, refused roots and nodes): the spec and
    its filter give the same result, or the same status and index. The data blob is compared through the proofs that index it: the
    slots of receipts missing from the receipts AMT are never written."""
    from tests import event_amts as E
    from tests.test_event_amts import COUNTS
    n = nf = 0
    for c in E.catalogue(E.base_tipset()):
        ts = c.ts
        store = api.BlockStore.from_tipset(ts, verify_cids=True)
        spec = _spec(api, ts)
        a = _run(lambda: store.generate_event_proof(ts, spec, A.RESULT_JSON))
        b = _run(lambda: store.generate_log_proof(ts, api.LogFilter.from_spec(spec), A.RESULT_JSON))
        if a[0] != "ok":
            assert a == b, c.name
            nf += 1
            continue
        a, b = a[1], b[1]
        assert a.matching.tolist() == b.matching.tolist() and a.n_exec == b.n_exec, c.name
        assert [p.key() for p in a.proofs] == [p.key() for p in b.proofs] and np.array_equal(a.raw_proofs, b.raw_proofs), c.name
        assert np.array_equal(a.witness.cids, b.witness.cids) and a.witness.blocks() == b.witness.blocks() and a.json == b.json, c.name
        n += 1
    assert n == COUNTS["valid"] + COUNTS["receipts"] + COUNTS["rpc"] and n + nf == sum(COUNTS.values())


# ------------------------------------------------------------------ filters against the restated generator
def _check_filter(api, oracle_mod, ts, store, flt, d=None, cpp=None):
    """The engine against both restated generators, which are compared with each other: results field by field, or on failure the
    same status and index (the C++ oracle's) and a failure of the Python one."""
    d = d if d is not None else dict_of(ts)
    cpp = cpp or OL.CppOracle(ts)
    try:
        exp = ("ok", OL.generate_log_proof(d, ts, *OL.filter_of(flt)))
    except Exception as e:   # the Python oracle raises MissingBlock / decode errors / IndexError, without the engine's status
        exp = ("err", type(e).__name__)
    ref = cpp.generate(ts, flt)
    got = _run(lambda: store.generate_log_proof(ts, flt))
    if ref[0] == "err":
        assert exp[0] == "err" and got == ref
        return None
    assert exp[0] == "ok" and got[0] == "ok"
    exp, ref, got = exp[1], ref[1], got[1]
    keys = [(i, j, e, tuple(bytes(t) for t in tp), bytes(dt), bytes(m)) for i, j, e, tp, dt, m in exp["proofs"]]
    assert ref.matching.tolist() == exp["matching"] and [p.key() for p in ref.proofs] == keys
    assert [bytes(c) for c in ref.witness.cids] == exp["witness"]
    assert_event_results_equal(got, ref)
    if got.proofs:
        assert all(api.verify_event_proofs(got.witness, ts, got))
        assert all(api.verify_event_proofs(got.witness, ts, got, filter_spec=flt))
        assert all(oracle_mod.verify_event_proofs(got.witness, ts, got))
    return got


def _values_of(logs, k, n, rng, miss=0):
    vals = sorted({t[k] for _, t in logs if len(t) > k})
    pick = [vals[int(i)] for i in rng.choice(len(vals), size=min(n, len(vals)), replace=False)] if vals else []
    return pick + [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(max(0, n - len(pick)) + miss)]


def test_wildcards_positions_and_topic_counts(api, oracle_mod, shapes):
    store = api.BlockStore.from_tipset(shapes, verify_cids=True)
    d = dict_of(shapes)
    logs = OL.candidate_logs(d, shapes)
    assert {len(t) for _, t in logs} >= {1, 2, 3, 4}
    rng = np.random.default_rng(7)
    for npos in range(5):
        _check_filter(api, oracle_mod, shapes, store, api.LogFilter(topics=[None] * npos), d)   # trailing wildcards only
    for k in range(4):   # one constrained position at a time, every other a wildcard, the constraint last or not
        vals = _values_of(logs, k, 2, rng)
        _check_filter(api, oracle_mod, shapes, store, api.LogFilter(topics=[None] * k + [vals]), d)
        _check_filter(api, oracle_mod, shapes, store, api.LogFilter(topics=[None] * k + [vals] + [None] * (3 - k)), d)
    # topic 2 and topic 3 together, duplicates, and an emitter set
    t2, t3 = _values_of(logs, 2, 3, rng), _values_of(logs, 3, 3, rng)
    _check_filter(api, oracle_mod, shapes, store, api.LogFilter(topics=[None, None, t2 + t2, t3]), d)
    emitters = sorted({e for e, _ in logs})[:3]
    _check_filter(api, oracle_mod, shapes, store, api.LogFilter(emitters=emitters + emitters[:1], topics=[None, None]), d)


# 64 values are the largest set whose bitmap has the minimum 4 096 bits; 65 take 8 192
@pytest.mark.parametrize("n", [1, 2, LF_INLINE - 1, LF_INLINE, LF_INLINE + 1, 64, 65, 4096, A.LOG_FILTER_MAX_VALUES])
def test_value_sets_either_side_of_the_inline_switch(api, oracle_mod, shapes, n):
    store = api.BlockStore.from_tipset(shapes)
    d = dict_of(shapes)
    logs = OL.candidate_logs(d, shapes)
    rng = np.random.default_rng(n)
    v0 = _values_of(logs, 0, min(n, 6), rng)
    v0 += [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(n - len(v0))]
    _check_filter(api, oracle_mod, shapes, store, api.LogFilter(topics=[v0[:n]]), d)
    v1 = _values_of(logs, 1, min(n, 6), rng)
    v1 += [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(n - len(v1))]
    _check_filter(api, oracle_mod, shapes, store, api.LogFilter(topics=[None, v1[:n]]), d)


@pytest.mark.parametrize("n", [1, 2, LF_INLINE - 1, LF_INLINE, LF_INLINE + 1, 64, 65, 1024, A.LOG_FILTER_MAX_EMITTERS])
def test_emitter_sets(api, oracle_mod, shapes, n):
    store = api.BlockStore.from_tipset(shapes)
    d = dict_of(shapes)
    logs = OL.candidate_logs(d, shapes)
    have = sorted({e for e, _ in logs})
    rng = np.random.default_rng(n)
    pick = [have[int(i)] for i in rng.choice(len(have), size=min(len(have), max(1, n // 2)), replace=False)]
    em = (pick + [int(x) for x in rng.integers(0, 2**63, n, dtype=np.uint64)])[:n]
    _check_filter(api, oracle_mod, shapes, store, api.LogFilter(emitters=em), d)


def _custom(synth_mod, events):
    from tests.test_oracle_cpu import _custom_events_tipset
    return _custom_events_tipset(synth_mod, events)


def test_binary_values_case_a_shapes_and_short_logs(api, oracle_mod, synth_mod):
    E = lambda k, v, fl=3, codec=0x55: [fl, k, codec, v]  # noqa: E731
    addr = bytes(12) + bytes(range(0xEC, 0x100))            # an indexed address: twelve leading zero bytes
    binv = bytes([0xFF, 0xFE, 0x00, 0x80] * 8)               # not UTF-8, zero byte inside
    other = bytes(31) + b"\x01"
    events = [
        [1001, [E("t1", addr), E("t2", binv), E("t3", other)]],
        [1001, [E("topics", b"")]],                                         # Case A, zero topics
        [1002, [E("topics", addr + binv + other + addr + binv + other)]],   # Case A, six topics
        [1002, [E("topics", binv + addr), E("data", b"x")]],
        [1003, [E("t1", binv)]],                                            # one topic
        [1003, [E("t1", addr), E("t2", other), E("t3", binv), E("t4", addr), E("d", b"yz")]],
        [1004, [E("t1", addr), E("t2", b"short")]],                         # void: extract_evm_log refuses it
        [1001, [E("topics", addr[:31])]],                                   # void: not a multiple of 32
    ]
    ts = _custom(synth_mod, events)
    store = api.BlockStore.from_tipset(ts, verify_cids=True)
    d = dict_of(ts)
    F = api.LogFilter
    cases = [
        F(topics=[]), F(topics=[None]), F(topics=[None] * 4), F(topics=[addr]), F(topics=[[addr, binv]]), F(topics=[None, binv]),
        F(topics=[None, None, [other, binv]]), F(topics=[None, None, None, addr]), F(topics=[binv, addr]), F(topics=[addr, None, None, None]),
        F(emitters=[1002], topics=[]), F(emitters=[1002, 1003], topics=[None, [addr, binv]]), F(topics=["0x" + addr.hex()]),
    ]
    n_hits = 0
    for f in cases:
        got = _check_filter(api, oracle_mod, ts, store, f, d)
        n_hits += len(got.proofs) if got else 0
    assert n_hits > 0


def test_narrower_filter_marks_exactly_the_excluded_proofs_false(api, shapes):
    store = api.BlockStore.from_tipset(shapes)
    d = dict_of(shapes)
    wide = api.LogFilter(topics=[None])
    got = store.generate_log_proof(shapes, wide)
    logs = OL.candidate_logs(d, shapes)
    rng = np.random.default_rng(3)
    narrow = api.LogFilter(emitters=sorted({e for e, _ in logs})[:5], topics=[None, _values_of(logs, 1, 40, rng)])
    res = api.verify_event_proofs(got.witness, shapes, got, filter_spec=narrow)
    assert res == [narrow.matches(p.emitter, p.topics) for p in got.proofs]
    assert 0 < sum(res) < len(res)


def test_json_bundle_verifies(api, shapes):
    store = api.BlockStore.from_tipset(shapes)
    got = store.generate_log_proof(shapes, api.LogFilter(topics=[None, None]), A.RESULT_JSON)
    v = api.verify_bundle_json(got.json)
    assert len(v.event_results) == len(got.proofs) > 0 and all(v.event_results)


def test_refused_filters(api, ts1):
    store = api.BlockStore.from_tipset(ts1)
    tip = store.upload_tipset(ts1)
    L = api.lib()
    v = np.zeros(32 * (A.LOG_FILTER_MAX_VALUES + 1), np.uint8)
    e = np.arange(A.LOG_FILTER_MAX_EMITTERS + 1, dtype=np.uint64)

    def call(**kw):
        f = A.LogFilterC()
        f.n_positions = kw.get("npos", 1)
        for k, n in kw.get("values", {}).items():
            f.n_values[k] = n
            f.values[k] = None if kw.get("null") else v.ctypes.data
        f.n_emitters = kw.get("ne", 0)
        f.emitters = None if kw.get("null") else e.ctypes.data
        out = C.POINTER(A.EventResultC)()
        st = L.ipcfp_generate_log_proof_resident(store._h, tip._h, C.byref(f), 0, C.byref(out))
        if st == A.OK:
            L.ipcfp_event_result_free(out)
        return st

    assert call(npos=5) == A.ERR_INVALID_ARG
    assert call(npos=1, values={1: 1}) == A.ERR_INVALID_ARG
    assert call(npos=4, values={3: 1}, null=True) == A.ERR_INVALID_ARG
    assert call(ne=1, null=True) == A.ERR_INVALID_ARG
    assert call(values={0: A.LOG_FILTER_MAX_VALUES + 1}) == A.ERR_INVALID_ARG
    assert call(values={0: A.LOG_FILTER_MAX_VALUES}) == A.OK
    assert call(ne=A.LOG_FILTER_MAX_EMITTERS + 1) == A.ERR_INVALID_ARG
    assert call(ne=A.LOG_FILTER_MAX_EMITTERS) == A.OK
    assert call(npos=4) == A.OK
    with pytest.raises(A.IpcfpError):
        store.plan_fetch_logs(tip, api.LogFilter(topics=[None]), flags=1)


# ------------------------------------------------------------------ the fetch loop
def _pack(held):
    cids = list(held)
    blocks = [held[c] for c in cids]
    lens = np.array([len(b) for b in blocks], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens, dtype=np.uint64)[:-1]]).astype(np.uint64) if blocks else np.zeros(0, np.uint64)
    blob = np.frombuffer(b"".join(blocks), np.uint8) if blocks else np.zeros(0, np.uint8)
    cid_arr = np.frombuffer(b"".join(cids), np.uint8).reshape(-1, 38) if cids else np.zeros((0, 38), np.uint8)
    return cid_arr, offs, lens, blob


@pytest.mark.parametrize("which", ["ts1", "shapes"])
def test_fetch_loop_from_an_empty_store_converges_to_the_same_bundle(api, request, which):
    ts = request.getfixturevalue(which)
    full = dict_of(ts)
    flt = api.LogFilter(topics=[None, None]) if which == "shapes" else api.LogFilter.from_spec(_spec(api, ts))
    held = {}
    for rounds in range(1, 200):
        store = api.BlockStore(*_pack(held))
        tip = store.upload_tipset(ts)
        want = [bytes(c) for c in store.plan_fetch_logs(tip, flt).cids]
        if not want:
            break
        assert all(c in full and c not in held for c in want)
        held.update((c, full[c]) for c in want)
    assert not want and rounds > 1
    got = store.generate_log_proof_resident(tip, flt, A.RESULT_JSON)
    ref = api.BlockStore.from_tipset(ts).generate_log_proof(ts, flt, A.RESULT_JSON)
    assert got.json == ref.json and len(ref.proofs) > 0


# ------------------------------------------------------------------ the 1 M-receipt tipset of bench.py, sparse and dense
def _gather_hash(h, buf, offs, lens, chunk=1 << 17):
    """SHA-256 update with buf[offs[k] : offs[k] + lens[k]] for every k in order, in bounded memory."""
    offs, lens = np.asarray(offs, np.int64), np.asarray(lens, np.int64)
    for a in range(0, len(lens), chunk):
        o, n = offs[a:a + chunk], lens[a:a + chunk]
        if not n.sum():
            continue
        start = np.repeat(o - np.concatenate([[0], np.cumsum(n)[:-1]]), n)
        h.update(buf[start + np.arange(int(n.sum()))].tobytes())


def _digest(r, store_blob=None):
    """SHA-256 over a raw ipcfp_event_result: matching indices, every EventProof field (topics and data by their offsets, so the blob's
    layout does not enter), n_exec, witness CIDs and block bytes (from the store's blob when the witness came by reference)."""
    import hashlib
    h = hashlib.sha256()
    n = int(r.n_proofs)
    h.update(A._arr(r.matching_indices, int(r.n_matching), np.uint64).tobytes())
    recs = np.frombuffer(A._arr(C.cast(r.proofs, C.c_void_p).value, n * C.sizeof(A.EventProofC), np.uint8).tobytes(), dtype=np.dtype({
        "names": ["exec_index", "event_index", "emitter", "n_topics", "data_len", "data_off", "topics_off", "message_cid"],
        "formats": [np.uint64, np.uint64, np.uint64, np.uint32, np.uint32, np.uint64, np.uint64, (np.uint8, 38)],
        "offsets": [getattr(A.EventProofC, f).offset for f in ("exec_index", "event_index", "emitter", "n_topics", "data_len", "data_off",
                                                               "topics_off", "message_cid")],
        "itemsize": C.sizeof(A.EventProofC)}))
    for f in ("exec_index", "event_index", "emitter", "n_topics", "data_len", "message_cid"):
        h.update(np.ascontiguousarray(recs[f]).tobytes())
    blob = A._arr(r.data_blob, int(r.data_blob_size), np.uint8)
    _gather_hash(h, blob, recs["topics_off"], 32 * recs["n_topics"].astype(np.int64))
    _gather_hash(h, blob, recs["data_off"], recs["data_len"])
    h.update(int(r.n_exec).to_bytes(8, "little"))
    m = int(r.witness.n_blocks)
    h.update(A._arr(r.witness.cids, 38 * m, np.uint8).tobytes())
    offs, lens = A._arr(r.witness.offsets, m, np.uint64), A._arr(r.witness.lengths, m, np.uint32)
    wblob = store_blob if store_blob is not None else A._arr(r.witness.blob, int(r.witness.blob_size), np.uint8)
    _gather_hash(h, wblob, offs, lens)
    return h.hexdigest()


def _json_sha(ptr, n):
    import hashlib
    return hashlib.sha256(memoryview((C.c_char * n).from_address(ptr))).hexdigest()


@pytest.fixture(scope="module")
def ts1m(synth_mod):
    return synth_mod.Tipset(synth_mod.config_params(4, n_receipts=1_000_000))


def _engine(api, store, tip, flt, flags):
    out = C.POINTER(A.EventResultC)()
    f, keep = flt.as_c()
    assert api.lib().ipcfp_generate_log_proof_resident(store._h, tip._h, C.byref(f), flags, C.byref(out)) == A.OK, api.lib().ipcfp_last_error()
    return out


def test_one_million_receipts_spec_and_filter(api, ts1m):
    store = api.BlockStore.from_tipset(ts1m)
    tip = store.upload_tipset(ts1m)
    spec = _spec(api, ts1m)
    cs = spec.as_c()
    out = C.POINTER(A.EventResultC)()
    assert api.lib().ipcfp_generate_event_proof_resident(store._h, tip._h, C.byref(cs), A.RESULT_JSON, C.byref(out)) == A.OK
    b = _engine(api, store, tip, api.LogFilter.from_spec(spec), A.RESULT_JSON)
    try:
        assert _digest(out.contents) == _digest(b.contents) and out.contents.n_proofs > 0
        assert _json_sha(out.contents.json, int(out.contents.json_len)) == _json_sha(b.contents.json, int(b.contents.json_len))
    finally:
        api.lib().ipcfp_event_result_free(out)
        api.lib().ipcfp_event_result_free(b)


def test_one_million_receipts_every_event(api, ts1m):
    """The all-wildcard filter: every receipt matches (about 8 M proofs, pass 2 one receipt per thread). The result with flags 0, with
    IPCFP_RESULT_JSON and with IPCFP_RESULT_JSON | IPCFP_WITNESS_BY_REFERENCE against the C++ restated generator (oracle_logs.cpp) by
    SHA-256; the device JSON against the host rendering (ipcfp_event_result_to_json) of the oracle's result."""
    flt = api.LogFilter()
    cpp = OL.CppOracle(ts1m)
    st = cpp.raw(ts1m, flt, threads=os.cpu_count() or 1)
    assert st[0] == "ok"
    ref = st[1]
    try:
        want = _digest(ref.contents)
        assert int(ref.contents.n_matching) == int(ts1m.n_receipts) and int(ref.contents.n_proofs) > 4 * int(ts1m.n_receipts)
        d, keep = A.make_tipset_desc(ts1m)
        txt, tlen = C.c_void_p(), C.c_uint64()
        assert api.lib().ipcfp_event_result_to_json(C.cast(ref, C.c_void_p), C.byref(d), C.byref(txt), C.byref(tlen)) == A.OK
        want_json = _json_sha(txt.value, tlen.value)
        api.lib().ipcfp_json_free(txt)
    finally:
        OL.CppOracle.free(ref)
    store = api.BlockStore.from_tipset(ts1m)
    tip = store.upload_tipset(ts1m)
    blob = np.ascontiguousarray(ts1m.blob, dtype=np.uint8)
    for flags in (0, A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE):
        out = _engine(api, store, tip, flt, flags)
        try:
            r = out.contents
            assert _digest(r, blob if flags & A.WITNESS_BY_REFERENCE else None) == want, flags
            if flags & A.RESULT_JSON:
                assert _json_sha(r.json, int(r.json_len)) == want_json, flags
        finally:
            api.lib().ipcfp_event_result_free(out)
