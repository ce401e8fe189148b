"""ipcfp_tipset_upload_json (include/ipcfp.h) on the GPU: a resident tipset straight from the Lotus JSON-RPC texts (tests/rpc_json.py) must
be the tipset ipcfp_tipset_upload makes from the synthetic descriptor — read back with ipcfp_tipset_describe, events roots included — and
every resident call against it must give byte-equal results. Canonical receipt lists are parsed on the device, every other text through
the host parser with the same results, and every failure gives the status and index the rules of tests/rpc_json.py give."""
import ctypes as C

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import rpc_json as R
from tests.util import spec_of

pytestmark = pytest.mark.gpu


def _event(api, store, tip, spec, flags=0):
    L = api.lib()
    out = C.POINTER(A.EventResultC)()
    api._check(L.ipcfp_generate_event_proof_resident(store._h, tip._h, C.byref(spec), flags, C.byref(out)))
    try:
        return A.event_result_from_c(out.contents)
    finally:
        L.ipcfp_event_result_free(out)


def _shard(api, store, tip, spec, lo, hi):
    L = api.lib()
    out = C.POINTER(A.EventResultC)()
    api._check(L.ipcfp_generate_event_proof_shard_resident(store._h, tip._h, C.byref(spec), lo, hi, 1, 0, 0, C.byref(out)))
    try:
        return A.event_result_from_c(out.contents)
    finally:
        L.ipcfp_event_result_free(out)


def _assert_same_event(got, exp):
    assert got.matching.tolist() == exp.matching.tolist() and got.n_exec == exp.n_exec
    assert [p.key() for p in got.proofs] == [p.key() for p in exp.proofs]
    assert np.array_equal(got.witness.cids, exp.witness.cids) and np.array_equal(got.witness.lengths, exp.witness.lengths)
    assert np.array_equal(got.witness.offsets, exp.witness.offsets) and np.array_equal(got.witness.blob, exp.witness.blob)
    assert got.json == exp.json


def _assert_same_tipset(tip_json, tip_ref, ts):
    got, ref = tip_json.describe(), tip_ref.describe()
    assert not ref.parsed_on_device and ref.ms_parse == 0
    R.assert_desc_equal(got, ref)
    R.assert_desc_equal(got, ts)
    return got


def _assert_same_results(api, store, tip_json, tip_ref, ts, flag_sets=(0, A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE)):
    spec = spec_of(ts)
    for flags in flag_sets:
        _assert_same_event(_event(api, store, tip_json, spec, flags), _event(api, store, tip_ref, spec, flags))


@pytest.mark.parametrize("config", [1, 2])
def test_canonical_text_is_parsed_on_the_device(api, synth_mod, config):
    ts = synth_mod.Tipset(synth_mod.config_params(config, null_root_permille=100))
    store = api.BlockStore.from_tipset(ts)
    tip_ref = store.upload_tipset(ts)
    tip_json = store.upload_tipset_json(*R.texts(ts))
    info = _assert_same_tipset(tip_json, tip_ref, ts)
    assert info.parsed_on_device and info.ms_parse > 0
    _assert_same_results(api, store, tip_json, tip_ref, ts)
    n = int(ts.n_receipts)
    spec = spec_of(ts)
    a, b = _shard(api, store, tip_json, spec, n // 3, n), _shard(api, store, tip_ref, spec, n // 3, n)
    assert a.matching.tolist() == b.matching.tolist() and [p.key() for p in a.proofs] == [p.key() for p in b.proofs]
    assert np.array_equal(a.witness.cids, b.witness.cids)
    # describe() without the events roots leaves them on the device
    short = tip_json.describe(with_events_roots=False)
    assert short.n_receipts == n and short.events_roots is None and short.has_events_root is None


def test_million_receipt_text(api, synth_mod):
    """The 1 M-receipt tipset: about 130 MB of canonical text, parsed on the device, events roots equal to the descriptor's."""
    ts = synth_mod.Tipset(synth_mod.config_params(4))
    p, c, r = R.texts(ts)
    assert len(r) > 100_000_000
    store = api.BlockStore.from_tipset(ts)
    tip_ref = store.upload_tipset(ts)
    tip_json = store.upload_tipset_json(p, c, r)
    info = _assert_same_tipset(tip_json, tip_ref, ts)
    assert info.parsed_on_device
    _assert_same_results(api, store, tip_json, tip_ref, ts, flag_sets=(A.RESULT_JSON | A.WITNESS_BY_REFERENCE,))
    # one receipt deep inside in another key order: the whole list goes through the host parser, with the same tipset
    recs = R.receipt_records(ts)
    k = len(recs) * 7 // 9
    recs[k] = R.dump(R._pairs(R.receipt_pairs(ts, k), lambda l: l[::-1]))
    tip_host = store.upload_tipset_json(p, c, "[" + ",".join(recs) + "]")
    info = _assert_same_tipset(tip_host, tip_ref, ts)
    assert not info.parsed_on_device and info.ms_parse > 0


def test_proof_bundle_with_storage_specs(api, synth_mod, ts3_small):
    """generate_proof_bundle_resident with storage specs: the child's ParentStateRoot comes from the JSON text."""
    ts = ts3_small
    store = api.BlockStore.from_tipset(ts)
    tip_ref = store.upload_tipset(ts)
    tip_json = store.upload_tipset_json(*R.texts(ts))
    assert _assert_same_tipset(tip_json, tip_ref, ts).parsed_on_device
    keys = [ts.storage_entry(k)[0] for k in (0, 1, 77)] + [ts.storage_absent_key(1)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    sspecs = [(a, s) for a in (1001, 1003, 1006) for s in slots]
    especs = [spec_of(ts), A.make_event_spec(ts.event_signature, "calib-subnet-2", None)]
    for flags in (0, A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE):
        a = store.generate_proof_bundle_resident(tip_json, sspecs, especs, flags)
        b = store.generate_proof_bundle_resident(tip_ref, sspecs, especs, flags)
        assert [vars(x) for x in a.storage.proofs] == [vars(x) for x in b.storage.proofs]
        assert a.storage.spec_witness == b.storage.spec_witness
        for x, y in zip(a.events, b.events):
            _assert_same_event(x, y)
        assert np.array_equal(a.witness.cids, b.witness.cids) and np.array_equal(a.witness.blob, b.witness.blob)
        assert a.json == b.json


FORCED_HOST = ["pretty", "trailing_space", "key_order_one", "unknown_field", "escaped_key", "events_root_missing", "return_escaped_record",
               "return_any_string", "escaped_cid", "space_around"]


@pytest.fixture(scope="module")
def nulls(synth_mod, api):
    ts = synth_mod.Tipset(synth_mod.config_params(1, null_root_permille=250))
    store = api.BlockStore.from_tipset(ts)
    return ts, store, store.upload_tipset(ts)


@pytest.mark.parametrize("name", FORCED_HOST)
def test_non_canonical_text_goes_through_the_host_parser(api, nulls, name):
    ts, store, tip_ref = nulls
    fn, outcome = next((f, o) for n, f, o in R.MUTATORS if n == name)
    assert outcome == A.OK
    texts = fn(ts, int(ts.n_receipts) * 2 // 3)
    tip = store.upload_tipset_json(*texts)
    info = tip.describe()
    assert not info.parsed_on_device, name
    R.assert_desc_equal(info, R.read(*texts))
    R.assert_desc_equal(info, ts)
    _assert_same_results(api, store, tip, tip_ref, ts, flag_sets=(A.RESULT_JSON,))


def test_other_accepted_mutators(api, nulls):
    """Every other accepted mutator: the descriptor the rules give, through whichever path."""
    ts, store, _ = nulls
    for name, fn, outcome in R.MUTATORS:
        if outcome != A.OK:
            continue
        texts = fn(ts, int(ts.n_receipts) * 2 // 3)
        info = store.upload_tipset_json(*texts).describe()
        R.assert_desc_equal(info, R.read(*texts))
        if name in ("canonical", "empty_list", "exit_code_u32_max", "gas_u64_max", "height_negative", "unknown_in_tipset"):
            assert info.parsed_on_device, name


@pytest.mark.parametrize("name", [n for n, f, o in R.MUTATORS if o != A.OK])
def test_failures_give_the_rules_status_and_index(api, nulls, name):
    ts, store, _ = nulls
    fn = next(f for n, f, o in R.MUTATORS if n == name)
    texts = fn(ts, int(ts.n_receipts) * 2 // 3)
    want = R.expected(*texts)
    assert isinstance(want, tuple)
    with pytest.raises(A.IpcfpError) as e:
        store.upload_tipset_json(*texts)
    assert (e.value.status, e.value.index) == want


def test_upload_checks_follow_the_parse(api, synth_mod):
    """A parse that succeeds is followed by ipcfp_tipset_upload's own checks: 65 parent blocks are unsupported there."""
    ts = synth_mod.Tipset(synth_mod.config_params(1))
    store = api.BlockStore.from_tipset(ts)
    parent, child = R.tipsets(ts)
    one_cid, one_block = parent.pairs[0][1][0], parent.pairs[1][1][0]
    parent = R._set(R._set(parent, "Cids", [one_cid] * 65), "Blocks", [one_block] * 65)
    texts = (R.dump(parent), R.dump(child), "[" + ",".join(R.receipt_records(ts)) + "]")
    assert isinstance(R.expected(*texts), dict)
    with pytest.raises(A.IpcfpError) as e:
        store.upload_tipset_json(*texts)
    assert e.value.status == A.ERR_UNSUPPORTED
    # … and a receipt-list failure comes before them
    bad = (texts[0], texts[1], texts[2][:-1])
    with pytest.raises(A.IpcfpError) as e:
        store.upload_tipset_json(*bad)
    assert (e.value.status, e.value.index) == R.expected(*bad)
