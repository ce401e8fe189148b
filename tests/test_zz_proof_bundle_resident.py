"""ipcfp_generate_proof_bundle_resident (include/ipcfp.h): generate_proof_bundle against an uploaded tipset, with the witness union built on
the device and, with IPCFP_RESULT_JSON, the UnifiedProofBundle text rendered on the device. Without flags it must equal
ipcfp_generate_proof_bundle on the same store and the oracle's generate_proof_bundle; its text must be byte for byte what
ipcfp_bundle_to_json and bundle_json.py render from the flagless bundle. (An opt-in mode: last in the suite, with the other ones.)"""
import ctypes as C
import json

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import bundle_json as J
from tests import util as U
from tests.util import EditedTipset, ShuffledTipset, assert_event_results_equal, assert_witness_equal

pytestmark = pytest.mark.gpu

JSON_FLAGS = (A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE)
EVM_ACTORS = (1001, 1002, 1003, 1004, 1005, 1006)   # the six contract_state shapes of the synthetic state tree


def _slots(api, ts, present=(0, 1, 77), absent=(1,)):
    n = int(ts.params.hamt_entries)
    keys = [ts.storage_entry(min(k, n))[0] for k in present] + [ts.storage_absent_key(k) for k in absent]
    return api.compute_mapping_slots(keys, [0] * len(keys))


def _event_specs(ts, k):
    """0, 1 or 3 event specs: the tipset's own, one without an actor filter, one that matches nothing."""
    all3 = [A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter), A.make_event_spec(ts.event_signature, "calib-subnet-2", None),
            A.make_event_spec("NoSuchEvent(bytes32)", "no-such-topic", None)]
    return all3[:k]


def _case(api, ts, name):
    slots = _slots(api, ts)
    if name == "s6e3":
        return [(a, s) for a in EVM_ACTORS for s in slots], _event_specs(ts, 3)
    if name == "s2e1":
        return [(1001, slots[0]), (1003, slots[-1])], _event_specs(ts, 1)
    if name == "s0e3":
        return [], _event_specs(ts, 3)
    if name == "s3e0":
        return [(1006, slots[1]), (1002, slots[-1]), (1001, slots[2])], []
    assert name == "s0e0"
    return [], []


CASES = ["s6e3", "s2e1", "s0e3", "s3e0", "s0e0"]


def _status(fn):
    try:
        fn()
    except A.IpcfpError as e:
        return e.status, e.index
    return A.OK, None


def _plain(api, store, ts, sspecs, especs):
    """ipcfp_generate_proof_bundle → (BundlePy, ipcfp_bundle_to_json of it)."""
    L = api.lib()
    sarr, ns, earr, ne = store._bundle_specs(sspecs, especs)
    d, keep = A.make_tipset_desc(ts)
    out = C.POINTER(A.BundleC)()
    api._check(L.ipcfp_generate_proof_bundle(store._h, C.byref(d), sarr, ns, earr, ne, C.byref(out)))
    try:
        assert not out.contents.json and out.contents.json_len == 0 and out.contents.ms_json == 0
        return A.bundle_from_c(out.contents), api.bundle_to_json(out, ts)
    finally:
        L.ipcfp_bundle_free(out)


def _assert_bundles_equal(got, exp, witness_bytes=True):
    assert (got.storage is None) == (exp.storage is None)
    if got.storage is not None:
        assert [vars(p) for p in got.storage.proofs] == [vars(p) for p in exp.storage.proofs]
        assert got.storage.spec_witness == exp.storage.spec_witness
        assert np.array_equal(got.storage.witness.cids, exp.storage.witness.cids)
        if witness_bytes:
            assert_witness_equal(got.storage.witness, exp.storage.witness)
    assert len(got.events) == len(exp.events)
    for g, e in zip(got.events, exp.events):
        assert_event_results_equal(g, e, check_witness_bytes=witness_bytes)
    assert np.array_equal(got.witness.cids, exp.witness.cids) and np.array_equal(got.witness.lengths, exp.witness.lengths)
    if witness_bytes:
        assert_witness_equal(got.witness, exp.witness)


def _assert_by_reference(ts, got, base):
    """Every witness of `got` (by reference) names, in the blob the store was created from, the bytes of `base`'s (flagless) witness."""
    blob = bytes(ts.blob)
    pairs = [(got.witness, base.witness)] + [(g.witness, b.witness) for g, b in zip(got.events, base.events)]
    if base.storage is not None:
        pairs.append((got.storage.witness, base.storage.witness))
    for w, b in pairs:
        assert len(w.blob) == 0 and np.array_equal(w.cids, b.cids) and np.array_equal(w.lengths, b.lengths)
        assert [blob[int(o):int(o) + int(n)] for o, n in zip(w.offsets, w.lengths)] == b.blocks()


def _check_store(api, oracle_mod, ts, sspecs, especs, store=None, oracle_too=True):
    """Every flag combination of the resident call against the plain call (and the oracle) on one store → (flagless bundle, its text)."""
    store = store or api.BlockStore.from_tipset(ts)
    base, want = _plain(api, store, ts, sspecs, especs)
    if oracle_too:
        _assert_bundles_equal(base, oracle_mod.Store.from_tipset(ts).generate_proof_bundle(ts, sspecs, especs))
    assert want == J.dumps(J.unified_bundle(ts, base))
    tip = store.upload_tipset(ts)
    try:
        got = store.generate_proof_bundle_resident(tip, sspecs, especs)
        assert got.json is None and got.timings["total"] > 0
        _assert_bundles_equal(got, base)
        got = store.generate_proof_bundle_resident(tip, sspecs, especs, A.WITNESS_BY_REFERENCE)
        assert got.json is None
        _assert_bundles_equal(got, base, witness_bytes=False)
        _assert_by_reference(ts, got, base)
        for flags in JSON_FLAGS:
            got = store.generate_proof_bundle_resident(tip, sspecs, especs, flags)
            assert len(got.json) == len(want) and got.json == want, flags
            assert got.timings["json"] > 0 and got.timings["total"] >= got.timings["json"]
            _assert_bundles_equal(got, base, witness_bytes=not flags & A.WITNESS_BY_REFERENCE)
            if flags & A.WITNESS_BY_REFERENCE:
                _assert_by_reference(ts, got, base)
    finally:
        tip.close()
    doc = json.loads(want)
    assert list(doc) == ["storage_proofs", "event_proofs", "blocks"]
    assert len(doc["storage_proofs"]) == len(sspecs) and len(doc["blocks"]) == base.witness.n_blocks
    assert len(doc["event_proofs"]) == sum(len(r.proofs) for r in base.events)
    return base, want


@pytest.mark.parametrize("name", CASES)
def test_resident_bundle_equals_plain_and_oracle(api, oracle_mod, ts3_small, name):
    sspecs, especs = _case(api, ts3_small, name)
    base, text = _check_store(api, oracle_mod, ts3_small, sspecs, especs)
    if name == "s0e0":
        assert text == '{"storage_proofs":[],"event_proofs":[],"blocks":[]}'
    if name == "s6e3":
        assert not base.events[2].proofs
        assert any(p.found for p in base.storage.proofs) and not all(p.found for p in base.storage.proofs)


SYNTH_STATE = [
    dict(n_receipts=2000, events_per_receipt=8, match_ppm=20000, n_actors=64, hamt_entries=5000),
    dict(n_receipts=300, events_per_receipt=3, match_ppm=200000, has_actor_filter=0, n_actors=16, hamt_entries=300, null_root_permille=100),
]


def _synth_state(synth_mod, k):
    return synth_mod.Tipset(synth_mod.config_params(2, with_state_tree=1, **SYNTH_STATE[k]))


def _synth_specs(api, ts):
    slots = _slots(api, ts, present=(0, 3, 299), absent=(0, 5))
    return [(a, s) for a in EVM_ACTORS[::-1] for s in slots[::2]] + [(1001, s) for s in slots], _event_specs(ts, 3)


@pytest.mark.parametrize("k", range(len(SYNTH_STATE)))
def test_resident_bundle_synthetic_state_trees(api, oracle_mod, synth_mod, k):
    ts = _synth_state(synth_mod, k)
    base, _ = _check_store(api, oracle_mod, ts, *_synth_specs(api, ts))
    assert base.events[0].proofs and not base.events[2].proofs


def test_resident_bundle_json_extreme_epochs(api, oracle_mod, synth_mod):
    ts = _synth_state(synth_mod, 1)
    sspecs, especs = _synth_specs(api, ts)
    for pe, ce in ((-(2 ** 63), 2 ** 63 - 1), (-1, 0), (2 ** 63 - 1, -(2 ** 63))):
        e = EditedTipset(ts, parent_epoch=pe, child_epoch=ce)
        _, text = _check_store(api, oracle_mod, e, sspecs, especs, oracle_too=False)
        assert text.startswith(f'{{"storage_proofs":[{{"child_epoch":{ce},') and f'"parent_epoch":{pe},"child_epoch":{ce},' in text


def test_resident_bundle_shuffled_misaligned_store(api, oracle_mod, ts3_small):
    sspecs, especs = _case(api, ts3_small, "s6e3")
    _check_store(api, oracle_mod, ShuffledTipset(ts3_small, seed=11, misalign=True), sspecs, especs)


@pytest.mark.parametrize("family", ["B", "D"])
def test_resident_bundle_adversarial_cids(api, oracle_mod, ts3_small, family):
    """B: eight CID prefixes (the union's order is `Cid` order, not byte order); D: the store holds duplicate CIDs with other bytes."""
    rt, _ = U.adversarial_tipset(ts3_small, family)
    sspecs, especs = _case(api, ts3_small, "s6e3")
    base, _ = _check_store(api, oracle_mod, rt, sspecs, especs, store=api.BlockStore.from_tipset(rt))
    if family == "B":
        assert len({bytes(c[:6]) for c in base.witness.cids}) > 1


@pytest.mark.parametrize("name", ["s6e3", "s0e3", "s3e0", "synthetic"])
def test_resident_bundle_json_round_trip(api, synth_mod, ts3_small, name):
    ts = _synth_state(synth_mod, 0) if name == "synthetic" else ts3_small
    sspecs, especs = _synth_specs(api, ts) if name == "synthetic" else _case(api, ts, name)
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    try:
        for flags in JSON_FLAGS:
            got = store.generate_proof_bundle_resident(tip, sspecs, especs, flags)
            v = api.verify_bundle_json(got.json)
            assert v.parsed_on_device
            assert v.storage_results == [True] * len(sspecs)
            assert v.event_results == [True] * sum(len(r.proofs) for r in got.events)
            assert v.n_blocks == got.witness.n_blocks
    finally:
        tip.close()


def test_resident_bundle_failures_leave_the_store_serving(api, ts3_small):
    ts = ts3_small
    sspecs, especs = _case(api, ts, "s2e1")
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    first = store.generate_proof_bundle_resident(tip, sspecs, especs, A.RESULT_JSON)

    def again():
        got = store.generate_proof_bundle_resident(tip, sspecs, especs, A.RESULT_JSON)
        _assert_bundles_equal(got, first)
        assert got.json == first.json

    try:
        # a storage spec for an actor the state tree does not hold: the same status and index from both bundle calls
        missing = sspecs + [(1000 + int(ts.params.n_actors) + 7, sspecs[0][1])]
        for flags in (0,) + JSON_FLAGS:
            st = _status(lambda: store.generate_proof_bundle_resident(tip, missing, especs, flags))
            assert st == (A.ERR_ACTOR_NOT_FOUND, len(sspecs))
            assert st == _status(lambda: store.generate_proof_bundle(ts, missing, especs))
            again()
        # flag bits the bundle call does not know
        for flags in (A.SCAN_SKIP_TX_AMTS, A.SHARDED_UNION_FULL, 0x20, 0x80000000, A.RESULT_JSON | 0x40):
            assert _status(lambda: store.generate_proof_bundle_resident(tip, sspecs, especs, flags))[0] == A.ERR_INVALID_ARG
            again()
        # storage specs against a tipset uploaded without the child's parent_state_root (event specs alone are fine)
        nosr = EditedTipset(ts, parent_state_root=np.zeros(0, dtype=np.uint8))
        tip2 = store.upload_tipset(nosr)
        try:
            for flags in (0, A.RESULT_JSON):
                assert _status(lambda: store.generate_proof_bundle_resident(tip2, sspecs, especs, flags))[0] == A.ERR_INVALID_ARG
                assert _status(lambda: store.generate_proof_bundle(nosr, sspecs, especs))[0] == A.ERR_INVALID_ARG
                again()
            ev_only = store.generate_proof_bundle_resident(tip2, [], especs, A.RESULT_JSON)
            assert ev_only.json == store.generate_proof_bundle_resident(tip, [], especs, A.RESULT_JSON).json
        finally:
            tip2.close()
    finally:
        tip.close()


def test_resident_bundle_full_tipset(api, synth_mod):
    """The 1 M-receipt tipset (BASELINE.json configs[3]) with a state tree, 16 storage specs and 2 event specs: the device text equals the
    host renderer byte for byte."""
    ts = synth_mod.Tipset(synth_mod.config_params(4, with_state_tree=1, hamt_entries=20000))
    slots = _slots(api, ts, present=(0, 1, 2, 77, 500, 19999), absent=(1, 2))
    sspecs = [(EVM_ACTORS[k % 6], slots[k % len(slots)]) for k in range(16)]
    especs = _event_specs(ts, 2)
    store = api.BlockStore.from_tipset(ts)
    base, want = _plain(api, store, ts, sspecs, especs)
    assert len(want) > 50_000_000
    tip = store.upload_tipset(ts)
    try:
        for flags in JSON_FLAGS:
            got = store.generate_proof_bundle_resident(tip, sspecs, especs, flags)
            assert got.json == want, flags
            assert np.array_equal(got.witness.cids, base.witness.cids)
    finally:
        tip.close()
