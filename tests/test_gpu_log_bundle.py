"""Proof bundles of log filters on the GPU: ipcfp_generate_log_bundle[_resident], ipcfp_plan_fetch_log_bundle_resident,
ipcfp_verify_event_proofs_any and ipcfp_verify_bundle_json_any.

Oracles: the spec bundle itself (the filters the specs stand for give the same bytes, and the same status and index on failure), and the
Python and C++ compositions of tests/log_bundles.py, which must agree with each other and with the engine."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import oracle
from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import bundle_json as J
from oracle import pyoracle as P
from tests import hostile_witness as H
from tests import log_bundles as LB
from tests import oracle_logs as OL
from tests import rpc_blocks as B
from tests import util as U
from tests.test_gpu_event_shapes import faulted
from tests.test_gpu_log_filter import _digest, _json_sha
from tests.test_zz_proof_bundle_resident import (CASES, JSON_FLAGS, SYNTH_STATE, _assert_bundles_equal, _assert_by_reference, _case, _plain,
                                                 _synth_specs, _synth_state)
from tests.util import EditedTipset, ShuffledTipset, dict_of

pytestmark = pytest.mark.gpu

ALL_FLAGS = (0, A.WITNESS_BY_REFERENCE) + JSON_FLAGS


def _status(fn):
    try:
        fn()
    except A.IpcfpError as e:
        return e.status, int(e.index)
    return A.OK, None


def _plain_log(api, store, ts, sspecs, filters):
    """ipcfp_generate_log_bundle → (BundlePy, ipcfp_bundle_to_json of it)."""
    L = api.lib()
    sarr, ns, _, _ = store._bundle_specs(sspecs, [])
    farr, nf, keep = api._log_filters_c(filters)
    d, dkeep = A.make_tipset_desc(ts)
    out = C.POINTER(A.BundleC)()
    api._check(L.ipcfp_generate_log_bundle(store._h, C.byref(d), sarr, ns, farr, nf, 0, C.byref(out)))
    try:
        return A.bundle_from_c(out.contents), api.bundle_to_json(out, ts)
    finally:
        L.ipcfp_bundle_free(out)


# ------------------------------------------------------------------ 1. a spec and its filter, byte for byte
def _spec_vs_filter(api, ts, sspecs, especs, store=None):
    store = store or api.BlockStore.from_tipset(ts)
    filters = [api.LogFilter.from_spec(api.EventProofSpec(s.event_signature.decode(), s.topic_1.decode(),
                                                          s.actor_id_filter if s.has_actor_id_filter else None)) for s in especs]
    base, want = _plain(api, store, ts, sspecs, especs)
    got, text = _plain_log(api, store, ts, sspecs, filters)
    _assert_bundles_equal(got, base)
    assert text == want
    tip = store.upload_tipset(ts)
    try:
        for flags in ALL_FLAGS:
            a = store.generate_proof_bundle_resident(tip, sspecs, especs, flags)
            b = store.generate_log_bundle_resident(tip, sspecs, filters, flags)
            by_ref = bool(flags & A.WITNESS_BY_REFERENCE)
            _assert_bundles_equal(b, a, witness_bytes=not by_ref)
            assert b.json == a.json and (b.json == want) == bool(flags & A.RESULT_JSON), flags
            if by_ref:
                _assert_by_reference(ts, b, base)
    finally:
        tip.close()
    return base


@pytest.mark.parametrize("name", CASES)
def test_spec_and_filter_bundles_equal(api, ts3_small, name):
    _spec_vs_filter(api, ts3_small, *_case(api, ts3_small, name))


@pytest.mark.parametrize("which", ["ts1", "ts2", "ts3_small"])
@pytest.mark.parametrize("n", [0, 1, 3])
def test_spec_and_filter_bundles_equal_configs(api, request, which, n):
    from tests.test_zz_proof_bundle_resident import _event_specs
    ts = request.getfixturevalue(which)
    sspecs = _case(api, ts, "s2e1")[0] if which == "ts3_small" else []
    _spec_vs_filter(api, ts, sspecs, _event_specs(ts, n))


@pytest.mark.parametrize("k", range(len(SYNTH_STATE)))
def test_spec_and_filter_bundles_synthetic_state(api, synth_mod, k):
    ts = _synth_state(synth_mod, k)
    base = _spec_vs_filter(api, ts, *_synth_specs(api, ts))
    assert base.events[0].proofs and base.storage.proofs


def test_spec_and_filter_bundles_shuffled_and_adversarial(api, ts3_small):
    sspecs, especs = _case(api, ts3_small, "s6e3")
    _spec_vs_filter(api, ShuffledTipset(ts3_small, seed=11, misalign=True), sspecs, especs)
    for family in ("B", "D"):
        rt, _ = U.adversarial_tipset(ts3_small, family)
        _spec_vs_filter(api, rt, sspecs, especs, store=api.BlockStore.from_tipset(rt))


@pytest.mark.parametrize("seed", range(4))
def test_spec_and_filter_bundles_fail_alike(api, synth_mod, seed):
    ts = synth_mod.Tipset(synth_mod.default_params(event_shapes=1, seed=0x5A1 + seed, n_receipts=4000, events_per_receipt=12, match_ppm=80000))
    d = dict_of(ts)
    index_of = {bytes(ts.cids[k]): k for k in range(int(ts.n_blocks))}
    bad, _ = faulted(ts, index_of, d, np.random.default_rng(seed), drop_leaf=bool(seed & 1))
    store = api.BlockStore.from_tipset(bad)
    especs = [A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter), A.make_event_spec(ts.event_signature, "calib-subnet-2", None)]
    filters = [LB.filter_of_cspec(s) for s in especs]
    a = _status(lambda: store.generate_proof_bundle(bad, [], especs))
    b = _status(lambda: store.generate_log_bundle(bad, [], filters))
    assert a == b
    if a[0] == A.OK:
        _assert_bundles_equal(store.generate_log_bundle(bad, [], filters), store.generate_proof_bundle(bad, [], especs))


# ------------------------------------------------------------------ 2. against the two compositions
def _assert_engine_equals(got, cc, d):
    """The engine's flagless bundle against the C++ composition's dict."""
    assert (got.storage is None) == (cc["storage"] is None)
    if got.storage is not None:
        assert [vars(p) for p in got.storage.proofs] == [vars(p) for p in cc["storage"].proofs]
        U.assert_witness_equal(got.storage.witness, cc["storage"].witness)
    assert len(got.events) == len(cc["events"])
    for g, e in zip(got.events, cc["events"]):
        U.assert_event_results_equal(g, e)
    assert [bytes(c) for c in got.witness.cids] == cc["union"]
    assert got.witness.blocks() == [d[c] for c in cc["union"]]


@pytest.fixture(scope="module")
def state_ts(synth_mod):
    return _synth_state(synth_mod, 1)


@pytest.mark.parametrize("n_sspecs", [0, 2, 12])
def test_bundles_against_both_compositions(api, state_ts, n_sspecs):
    ts = state_ts
    d = dict_of(ts)
    sspecs = LB.storage_specs(ts, n_sspecs)
    ostore, cpp = oracle.Store.from_tipset(ts), OL.CppOracle(ts)
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    try:
        for name, filters in LB.filter_sets(ts, OL.candidate_logs(d, ts)).items():
            cc = LB.cpp_bundle(ts, sspecs, filters, ostore, cpp)
            LB.assert_compositions_agree(LB.py_bundle(d, ts, sspecs, filters), cc)
            assert cc[0] == "ok", name
            got = store.generate_log_bundle_resident(tip, sspecs, filters)
            _assert_engine_equals(got, cc[1], d)
            assert got.storage is None or len(got.storage.proofs) == n_sspecs
            # 3. the device text equals the host renderings of the flagless bundle
            base, want = _plain_log(api, store, ts, sspecs, filters)
            _assert_bundles_equal(base, got)
            assert want == J.dumps(J.unified_bundle(ts, base))
            for flags in JSON_FLAGS:
                assert store.generate_log_bundle_resident(tip, sspecs, filters, flags).json == want, (name, flags)
    finally:
        tip.close()


def test_one_filter_is_the_log_proof(api, state_ts):
    ts = state_ts
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    try:
        for f in LB.filter_sets(ts, OL.candidate_logs(dict_of(ts), ts))["mixed8"]:
            for flags in ALL_FLAGS:
                a = store.generate_log_proof_resident(tip, f, flags & A.WITNESS_BY_REFERENCE)
                b = store.generate_log_bundle_resident(tip, [], [f], flags)
                by_ref = bool(flags & A.WITNESS_BY_REFERENCE)
                U.assert_event_results_equal(b.events[0], a, check_witness_bytes=not by_ref)
                assert np.array_equal(b.witness.cids, a.witness.cids) and np.array_equal(b.witness.lengths, a.witness.lengths)
                if not by_ref:
                    assert b.witness.blocks() == a.witness.blocks()
    finally:
        tip.close()


# ------------------------------------------------------------------ 4. verification with a set
def _verify_sets(api, ts, bundle, filters):
    for r in bundle.events:
        if not r.proofs:
            continue
        w = bundle.witness
        per = [api.verify_event_proofs(w, ts, r, filter_spec=f) for f in filters]
        anyv = api.verify_event_proofs_any(w, ts, r, filters)
        assert anyv == [any(x) for x in zip(*per)] if per else anyv == api.verify_event_proofs(w, ts, r)
        assert anyv == [LB.log_matches_any(filters, p.emitter, p.topics) for p in r.proofs] if filters else all(anyv)
        for f, one in zip(filters, per):
            assert api.verify_event_proofs_any(w, ts, r, [f]) == one
        for j in range(len(filters) if len(filters) > 1 else 0):   # dropping filter j marks exactly the proofs only it matched false
            # (the set of one is left out: without its filter it is the empty set, which is no check_event)
            rest = filters[:j] + filters[j + 1:]
            got = api.verify_event_proofs_any(w, ts, r, rest)
            only = [filters[j].matches(p.emitter, p.topics) and not LB.log_matches_any(rest, p.emitter, p.topics) for p in r.proofs]
            assert got == [a and not o for a, o in zip(anyv, only)]


def test_verify_any_equals_the_or_of_single_filters(api, state_ts):
    ts = state_ts
    store = api.BlockStore.from_tipset(ts)
    sets = LB.filter_sets(ts, OL.candidate_logs(dict_of(ts), ts))
    wide = store.generate_log_bundle(ts, LB.storage_specs(ts, 2), [api.LogFilter()])
    for name in ("spec", "nothing", "positions", "mixed8", "big", "dup_wild", "none"):
        _verify_sets(api, ts, wide, sets[name])
        _verify_sets(api, ts, store.generate_log_bundle(ts, [], sets[name]), sets[name])


def test_verify_any_fails_as_the_unfiltered_call(api):
    filters = [api.LogFilter(), api.LogFilter(topics=[bytes(32)]), api.LogFilter(emitters=[1, 2, 3, 4, 5], topics=[None, None])]
    n = 0
    for c in H.event_cases() + H.event_batches():
        plain = _status(lambda: api.verify_event_proofs(c.witness(), c.ts, c.result()))
        for fs in (filters, filters[1:2], []):
            got = _status(lambda: api.verify_event_proofs_any(c.witness(), c.ts, c.result(), fs))
            assert got[0] == plain[0] and got[1] == plain[1], (c.name, got, plain)
        if plain[0] == A.OK:
            assert api.verify_event_proofs_any(c.witness(), c.ts, c.result(), filters[:1]) == api.verify_event_proofs(c.witness(), c.ts, c.result())
        n += plain[0] != A.OK
    assert n > 0


def test_verify_bundle_json_any(api, state_ts):
    ts = state_ts
    store = api.BlockStore.from_tipset(ts)
    sets = LB.filter_sets(ts, OL.candidate_logs(dict_of(ts), ts))
    made = sets["mixed8"][:5]
    tip = store.upload_tipset(ts)
    try:
        b = store.generate_log_bundle_resident(tip, LB.storage_specs(ts, 12), made, A.RESULT_JSON)
    finally:
        tip.close()
    child, parents = bytes(ts.child_cid), bytes(np.ascontiguousarray(ts.parent_cids, np.uint8))
    texts = (b.json, json.dumps(json.loads(b.json), indent=1))
    for check in (made, made[:1], made[2:4], [], sets["nothing"]):
        want_s = api.verify_storage_proofs(b.witness, ts, b.storage)
        want_e = [x for r in b.events for x in (api.verify_event_proofs_any(b.witness, ts, r, check) if r.proofs else [])]
        for text, dev in zip(texts, (True, False)):
            v = api.verify_bundle_json_any(text, log_filters=check)
            assert v.parsed_on_device == dev
            assert v.storage_results == want_s and v.event_results == want_e
            assert all(want_s) and (all(want_e) if check is made or not check else True)
            v = api.verify_bundle_json_any(text, trusted_parent=lambda e, p: p == parents, trusted_child=lambda e, c: c == child, log_filters=check)
            assert v.storage_results == want_s and v.event_results == want_e
            v = api.verify_bundle_json_any(text, trusted_parent=lambda e, p: False, log_filters=check)
            assert v.storage_results == want_s and v.event_results == [False] * len(want_e)
            v = api.verify_bundle_json_any(text, trusted_child=lambda e, c: False, log_filters=check)
            assert v.storage_results == [False] * len(want_s) and v.event_results == [False] * len(want_e)
    assert api.verify_bundle_json_any(b.json).event_results == api.verify_bundle_json(b.json).event_results


# ------------------------------------------------------------------ 5. fetch planning
def _full(ts):
    cids, blocks = B.blocks_of(ts)
    return {bytes(c): b for c, b in zip(cids, blocks)}


def _rounds(api, ts, full, plan_a, plan_b):
    """Both planners from the empty store, round for round, until the plan is empty."""
    held = {}
    for rounds in range(1, 500):
        cids = list(held)
        store = api.BlockStore(*_pack(held, cids))
        tip = store.upload_tipset(ts)
        a, b = plan_a(store, tip), plan_b(store, tip)
        assert [bytes(c) for c in a.cids] == [bytes(c) for c in b.cids] and a.n_needed == b.n_needed
        tip.close()
        if not len(a.cids):
            return rounds
        held.update((bytes(c), full[bytes(c)]) for c in a.cids)
    raise AssertionError("no fixed point")


def _pack(held, cids):
    blocks = [held[c] for c in cids]
    lens = np.array([len(b) for b in blocks], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens, dtype=np.uint64)[:-1]]).astype(np.uint64) if blocks else np.zeros(0, np.uint64)
    blob = np.frombuffer(b"".join(blocks), np.uint8) if blocks else np.zeros(0, np.uint8)
    return (np.frombuffer(b"".join(cids), np.uint8).reshape(-1, 38) if cids else np.zeros((0, 38), np.uint8)), offs, lens, blob


def test_plan_one_filter_equals_plan_fetch_logs(api, synth_mod):
    ts = synth_mod.Tipset(synth_mod.default_params(event_shapes=1, seed=7, n_receipts=600, events_per_receipt=6, match_ppm=60000))
    for f in (api.LogFilter(topics=[None, None]), LB.spec_filter(ts.event_signature, ts.topic1, ts.actor_filter)):
        assert _rounds(api, ts, _full(ts), lambda s, t: s.plan_fetch_log_bundle(t, [], [f]), lambda s, t: s.plan_fetch_logs(t, f)) > 1


def test_plan_spec_filters_equals_plan_fetch(api, state_ts):
    ts = state_ts
    sspecs, especs = _synth_specs(api, ts)
    filters = [LB.filter_of_cspec(s) for s in especs]
    assert _rounds(api, ts, _full(ts), lambda s, t: s.plan_fetch_log_bundle(t, sspecs, filters), lambda s, t: s.plan_fetch(t, sspecs, especs)) > 1


def _loop(api, ts, sspecs, filters):
    full = _full(ts)

    def fetch(cids, first_id):
        return B.render([], elements=[B.element(first_id + k, full[bytes(c)]) for k, c in enumerate(cids)])

    store, tip, rounds, _, _ = api.fetch_log_bundle_until_complete(fetch, lambda s: s.upload_tipset(ts), sspecs, filters, verify_cids=False)
    try:
        ref = api.BlockStore.from_tipset(ts)
        rtip = ref.upload_tipset(ts)
        a = store.generate_log_bundle_resident(tip, sspecs, filters, A.RESULT_JSON)
        b = ref.generate_log_bundle_resident(rtip, sspecs, filters, A.RESULT_JSON)
        assert a.json == b.json and len(rounds) > 1
        rtip.close()
    finally:
        tip.close()


@pytest.mark.parametrize("which", ["ts1", "ts2", "ts3_small"])
def test_fetch_loop_converges(api, request, which):
    ts = request.getfixturevalue(which)
    _loop(api, ts, [], [LB.spec_filter(ts.event_signature, ts.topic1, ts.actor_filter), api.LogFilter(topics=[None, None, None])])


def test_fetch_loop_converges_unified(api, state_ts):
    ts = state_ts
    _loop(api, ts, LB.storage_specs(ts, 12), LB.filter_sets(ts, OL.candidate_logs(dict_of(ts), ts))["mixed8"])


# ------------------------------------------------------------------ 6. refusals
def test_refusals_carry_the_filter_position(api, state_ts):
    ts = state_ts
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    sspecs = LB.storage_specs(ts, 2)
    good = [api.LogFilter(topics=[None]), LB.spec_filter(ts.event_signature, ts.topic1), api.LogFilter(), api.LogFilter(topics=[None] * 2)]
    ref = store.generate_log_bundle_resident(tip, sspecs, good, A.RESULT_JSON)
    v = np.zeros(32 * (A.LOG_FILTER_MAX_VALUES + 1), np.uint8)
    e = np.arange(A.LOG_FILTER_MAX_EMITTERS + 1, dtype=np.uint64)

    class Raw:   # a refused ipcfp_log_filter, which api.LogFilter cannot express
        def __init__(self, **kw):
            self.kw = kw

        def as_c(self):
            f = A.LogFilterC()
            f.n_positions = self.kw.get("npos", 1)
            for k, n in self.kw.get("values", {}).items():
                f.n_values[k] = n
                f.values[k] = None if self.kw.get("null") else v.ctypes.data
            f.n_emitters = self.kw.get("ne", 0)
            f.emitters = None if self.kw.get("null") else e.ctypes.data
            return f, None

    bad = [Raw(npos=5), Raw(values={1: 1}), Raw(npos=4, values={3: 1}, null=True), Raw(ne=1, null=True),
           Raw(values={0: A.LOG_FILTER_MAX_VALUES + 1}), Raw(ne=A.LOG_FILTER_MAX_EMITTERS + 1)]
    wit = ref.witness
    calls = [lambda fs: store.generate_log_bundle_resident(tip, sspecs, fs, A.RESULT_JSON), lambda fs: store.generate_log_bundle(ts, sspecs, fs),
             lambda fs: store.plan_fetch_log_bundle(tip, sspecs, fs), lambda fs: api.verify_event_proofs_any(wit, ts, ref.events[1], fs),
             lambda fs: api.verify_bundle_json_any(ref.json, log_filters=fs)]
    try:
        for b in bad:
            for pos in (0, 1, 3):
                fs = good[:pos] + [b] + good[pos + 1:]
                for call in calls:
                    assert _status(lambda: call(fs)) == (A.ERR_INVALID_ARG, pos)
                got = store.generate_log_bundle_resident(tip, sspecs, good, A.RESULT_JSON)
                assert got.json == ref.json
        # the single-filter calls keep their index-free refusal
        assert _status(lambda: store.plan_fetch_logs(tip, bad[0]))[0] == A.ERR_INVALID_ARG
        # flags, storage specs without a state root, by reference on a store without a caller blob
        for flags in (A.SCAN_SKIP_TX_AMTS, 0x20, A.RESULT_JSON | 0x40):
            assert _status(lambda: store.generate_log_bundle_resident(tip, sspecs, good, flags))[0] == A.ERR_INVALID_ARG
        assert _status(lambda: store.plan_fetch_log_bundle(tip, sspecs, good, flags=1))[0] == A.ERR_INVALID_ARG
        nosr = EditedTipset(ts, parent_state_root=np.zeros(0, dtype=np.uint8))
        tip2 = store.upload_tipset(nosr)
        assert _status(lambda: store.generate_log_bundle_resident(tip2, sspecs, good))[0] == A.ERR_INVALID_ARG
        assert _status(lambda: store.plan_fetch_log_bundle(tip2, sspecs, good))[0] == A.ERR_INVALID_ARG
        assert store.generate_log_bundle_resident(tip2, [], good, A.RESULT_JSON).json == store.generate_log_bundle_resident(tip, [], good, A.RESULT_JSON).json
        tip2.close()
        cids, blocks = B.blocks_of(ts)
        rpc = api.BlockStore.from_rpc_json(cids, B.render(blocks))
        rtip = rpc.upload_tipset(ts)
        assert _status(lambda: rpc.generate_log_bundle_resident(rtip, sspecs, good, A.WITNESS_BY_REFERENCE)) == \
            _status(lambda: rpc.generate_proof_bundle_resident(rtip, sspecs, [], A.WITNESS_BY_REFERENCE))
        assert rpc.generate_log_bundle_resident(rtip, sspecs, good, A.RESULT_JSON).json == ref.json
        rtip.close()
        # a generator failure: the first failing generator's status and index, storage first
        missing = sspecs + [(1000 + int(ts.params.n_actors) + 7, sspecs[0][1])]
        assert _status(lambda: store.generate_log_bundle_resident(tip, missing, good)) == (A.ERR_ACTOR_NOT_FOUND, len(sspecs))
        assert store.generate_log_bundle_resident(tip, sspecs, good, A.RESULT_JSON).json == ref.json
    finally:
        tip.close()


# ------------------------------------------------------------------ 7. scale: the 1 M-receipt tipset
def test_one_million_receipts_bundle(api, synth_mod):
    """65 536 storage lookups and the filters {the tipset's spec, the all-wildcard filter}: every proof field and the witness against
    the C++ composition by SHA-256, with flags 0, IPCFP_RESULT_JSON and IPCFP_RESULT_JSON | IPCFP_WITNESS_BY_REFERENCE; the text (the same
    in both modes) verifies against the set. It is longer than the device parser's 4 GiB, so the host parser reads it."""
    ts = synth_mod.Tipset(synth_mod.config_params(4, with_state_tree=1, hamt_entries=20000))
    m = int(ts.params.hamt_entries)
    keys = [ts.storage_entry(k % m)[0] for k in range(60000)] + [ts.storage_absent_key(k) for k in range(5536)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    sspecs = [(LB.EVM_ACTORS[k % 6], bytes(slots[k])) for k in range(len(keys))]
    assert len(sspecs) == 65536
    filters = [LB.spec_filter(ts.event_signature, ts.topic1, ts.actor_filter), api.LogFilter()]
    threads = os.cpu_count() or 1
    cpp = OL.CppOracle(ts)
    want_ev = []
    for f in filters:
        r = cpp.raw(ts, f, threads=threads)
        assert r[0] == "ok"
        try:
            want_ev.append(_digest(r[1].contents))
        finally:
            OL.CppOracle.free(r[1])
    want_st = oracle.Store.from_tipset(ts).generate_storage_proofs(ts, sspecs)
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    blob = np.ascontiguousarray(ts.blob, dtype=np.uint8)
    L = api.lib()
    sarr, ns, _, _ = store._bundle_specs(sspecs, [])
    farr, nf, keep = api._log_filters_c(filters)
    try:
        for flags in (0, A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE):
            out = C.POINTER(A.BundleC)()
            api._check(L.ipcfp_generate_log_bundle_resident(store._h, tip._h, sarr, ns, farr, nf, flags, C.byref(out)))
            try:
                b = out.contents
                by_ref = bool(flags & A.WITNESS_BY_REFERENCE)
                assert [_digest(b.events[k].contents, blob if by_ref else None) for k in range(2)] == want_ev, flags
                st = A.storage_result_from_c(b.storage.contents)
                assert [vars(p) for p in st.proofs] == [vars(p) for p in want_st.proofs]
                assert np.array_equal(st.witness.cids, want_st.witness.cids)
                w = b.witness
                union = sorted({bytes(c) for c in want_st.witness.cids} | {bytes(c) for k in range(2)
                                for c in A._arr(b.events[k].contents.witness.cids, 38 * int(b.events[k].contents.witness.n_blocks), np.uint8).reshape(-1, 38)},
                               key=P.cid_sort_key)
                assert A._arr(w.cids, 38 * int(w.n_blocks), np.uint8).tobytes() == b"".join(union)
                if flags & A.WITNESS_BY_REFERENCE:
                    assert _json_sha(b.json, int(b.json_len)) == text_sha
                elif flags & A.RESULT_JSON:
                    text_sha = _json_sha(b.json, int(b.json_len))
                    vout = C.POINTER(A.BundleVerdictC)()
                    api._check(L.ipcfp_verify_bundle_json_any(C.cast(C.c_void_p(b.json), C.c_char_p), int(b.json_len), 0, A.TrustedParentFn(), A.TrustedChildFn(),
                                                               None, farr, nf, C.byref(vout)))
                    try:
                        v = vout.contents
                        assert int(v.n_storage_proofs) == 65536
                        ne = int(v.n_event_proofs)
                        assert ne == sum(int(b.events[k].contents.n_proofs) for k in range(2))
                        assert A._arr(v.event_results, ne, np.uint8).all()
                        sres = A._arr(v.storage_results, 65536, np.uint8)
                        assert sres.all()
                    finally:
                        L.ipcfp_bundle_verdict_free(vout)
            finally:
                L.ipcfp_bundle_free(out)
    finally:
        tip.close()
