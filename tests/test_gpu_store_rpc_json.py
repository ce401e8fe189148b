"""ipcfp_store_create_rpc_json (include/ipcfp.h) on the GPU: a block store straight from Filecoin.ChainReadObj responses
(tests/rpc_blocks.py) must be the store ipcfp_store_create makes from the same blocks — its size, get / has of every CID, and byte-equal
results of every generator run on it. Canonical texts are parsed on the device however they are split, every other input through the host
parser with the same store, and every failure gives the status and index the rules of tests/rpc_blocks.py give."""
import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import rpc_blocks as B
from tests.util import spec_of

pytestmark = pytest.mark.gpu


def _assert_same_witness(a, b):
    assert np.array_equal(a.cids, b.cids) and np.array_equal(a.lengths, b.lengths) and a.blocks() == b.blocks()


def _assert_same_event(a, b):
    assert a.matching.tolist() == b.matching.tolist() and a.n_exec == b.n_exec
    assert [p.key() for p in a.proofs] == [p.key() for p in b.proofs]
    _assert_same_witness(a.witness, b.witness)
    assert a.json == b.json


def _assert_same_store(got, ref, cids, sample=None):
    L = got._h and __import__("ipc_filecoin_proofs_b200.api", fromlist=["lib"]).lib()
    assert L.ipcfp_store_n_blocks(got._h) == L.ipcfp_store_n_blocks(ref._h) == len(cids)
    idx = range(len(cids)) if sample is None else np.random.default_rng(7).choice(len(cids), sample, replace=False)
    for i in idx:
        c = cids[i]
        assert got.has(c) and got.get(c) == ref.get(c)
    missing = cids[0].copy()
    missing[-1] ^= 0x5a
    assert got.has(missing) == ref.has(missing)


def _assert_same_results(got, ref, ts, storage=False):
    spec = spec_of(ts)
    tg, tr = got.upload_tipset(ts), ref.upload_tipset(ts)
    for flags in (0, A.RESULT_JSON):
        a = got.generate_event_proof(ts, spec, flags)
        b = ref.generate_event_proof(ts, spec, flags)
        _assert_same_event(a, b)
        x = got.generate_proof_bundle_resident(tg, _sspecs(got, ts) if storage else [], [spec], flags)
        y = ref.generate_proof_bundle_resident(tr, _sspecs(ref, ts) if storage else [], [spec], flags)
        _assert_same_witness(x.witness, y.witness)
        for e, f in zip(x.events, y.events):
            _assert_same_event(e, f)
        assert x.json == y.json
        if storage:
            assert [vars(p) for p in x.storage.proofs] == [vars(p) for p in y.storage.proofs]
    if storage:
        a, b = got.generate_storage_proofs(ts, _sspecs(got, ts)), ref.generate_storage_proofs(ts, _sspecs(ref, ts))
        assert [vars(p) for p in a.proofs] == [vars(p) for p in b.proofs] and a.spec_witness == b.spec_witness
        _assert_same_witness(a.witness, b.witness)


def _sspecs(store, ts):
    import ipc_filecoin_proofs_b200.api as api
    keys = [ts.storage_entry(k)[0] for k in (0, 1, 77)] + [ts.storage_absent_key(1)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    return [(a, s) for a in (1001, 1003, 1006) for s in slots]


@pytest.mark.parametrize("config", [1, 2, 3])
def test_canonical_texts_are_parsed_on_the_device(api, synth_mod, ts3_small, config):
    ts = ts3_small if config == 3 else synth_mod.Tipset(synth_mod.config_params(config))
    cids, blocks = B.blocks_of(ts)
    ref = api.BlockStore.from_tipset(ts, verify_cids=True)
    for k, texts in enumerate((B.render(blocks), B.render(blocks, 5, seed=config), B.render(blocks, single=True, seed=2),
                               [b"[]"] + B.render(blocks, 2, seed=3) + [b"[]"])):
        got = api.BlockStore.from_rpc_json(cids, texts, verify_cids=k % 2 == 0)
        assert got.json_info.parsed_on_device and got.json_info.ms_parse > 0 and got.json_info.ms_kernels > 0
        _assert_same_store(got, ref, cids, sample=None if len(cids) <= 3000 else 3000)
        if k == 1:
            _assert_same_results(got, ref, ts, storage=config == 3)
        got.close()


def test_million_receipt_blocks(api, synth_mod):
    """The 1 M-receipt tipset's ≈ 1.3 M blocks as one batch, as batches of 10 000 and as one object per text: parsed on the device."""
    ts = synth_mod.Tipset(synth_mod.config_params(4))
    cids, blocks = B.blocks_of(ts)
    ref = api.BlockStore.from_tipset(ts)
    els = [B.element(i, d) for i, d in enumerate(blocks)]
    order = np.random.default_rng(4).permutation(len(els))
    shuffled = [els[k] for k in order]
    n = len(els)
    for k, texts in enumerate(([b"[" + b",".join(els) + b"]"],
                               [b"[" + b",".join(shuffled[a:a + 10000]) + b"]" for a in range(0, n, 10000)],
                               shuffled)):
        got = api.BlockStore.from_rpc_json(cids, texts, verify_cids=k == 0)
        assert got.json_info.parsed_on_device, k
        _assert_same_store(got, ref, cids, sample=2000)
        if k == 1:
            spec = spec_of(ts)
            _assert_same_event(got.generate_event_proof(ts, spec, A.RESULT_JSON), ref.generate_event_proof(ts, spec, A.RESULT_JSON))
        got.close()


@pytest.fixture(scope="module")
def small(api, synth_mod):
    ts = synth_mod.Tipset(synth_mod.config_params(1))
    cids, blocks = B.blocks_of(ts)
    return ts, cids, blocks, api.BlockStore.from_tipset(ts)


def test_non_canonical_texts_take_the_host_path(api, small):
    ts, cids, blocks, ref = small
    els = [B.pretty(i, d) if i % 3 == 0 else B.element(i, d) for i, d in enumerate(blocks)]
    for texts in (B.render(blocks, elements=els), [b" " + t for t in B.render(blocks, 3, seed=1)], B.render(blocks)):
        got = api.BlockStore.from_rpc_json(cids, texts)
        assert got.json_info.parsed_on_device == (texts == B.render(blocks))
        _assert_same_store(got, ref, cids)
    got = api.BlockStore.from_rpc_json(cids, B.render(blocks, elements=els))
    assert not got.json_info.parsed_on_device and got.json_info.ms_kernels == 0
    _assert_same_results(got, ref, ts)


@pytest.mark.parametrize("case", range(36))
def test_cases_give_the_rules_outcome(api, small, case):
    ts, cids, blocks, ref = small
    cids, blocks = cids[:40].copy(), blocks[:40]
    blocks[7] = b""
    name, texts, outcome = B.cases(blocks)[case]
    want = B.expected(len(cids), texts)
    if outcome == A.OK:
        got = api.BlockStore.from_rpc_json(cids, texts, verify_cids=False)
        for i in range(len(cids)):
            assert got.get(cids[i]) is not None
        assert got.n_blocks == 40
        return
    with pytest.raises(A.IpcfpError) as e:
        api.BlockStore.from_rpc_json(cids, texts)
    assert (e.value.status, e.value.index) == want, name


def test_tampered_block_gives_the_binary_routes_mismatch(api, small):
    ts, cids, blocks, _ = small
    k = next(i for i in range(len(blocks) * 2 // 3, len(blocks)) if bytes(cids[i][2:6]) == b"\xa0\xe4\x02\x20" and blocks[i])
    bad = list(blocks)
    bad[k] = bytes([bad[k][0] ^ 1]) + bad[k][1:]
    offs, lens, blob = B.arrays(bad)
    with pytest.raises(A.IpcfpError) as want:
        api.BlockStore(cids, offs, lens, blob, verify_cids=True)
    for texts in (B.render(bad, 3, seed=8), B.render(bad, elements=[B.pretty(i, d) for i, d in enumerate(bad)])):
        with pytest.raises(A.IpcfpError) as got:
            api.BlockStore.from_rpc_json(cids, texts, verify_cids=True)
        assert got.value.status == want.value.status == A.ERR_CID_MISMATCH
        assert got.value.index == want.value.index == got.value.first_bad_block == want.value.first_bad_block == k
    # without the check the store is made
    assert api.BlockStore.from_rpc_json(cids, B.render(bad)).n_blocks == len(bad)


def test_witness_by_reference_is_unsupported(api, small):
    ts, cids, blocks, ref = small
    spec = spec_of(ts)
    for texts in (B.render(blocks), B.render(blocks, elements=[B.pretty(i, d) for i, d in enumerate(blocks)])):
        got = api.BlockStore.from_rpc_json(cids, texts)
        tip = got.upload_tipset(ts)
        for call in (lambda: got.generate_event_proof(ts, spec, A.WITNESS_BY_REFERENCE),
                     lambda: got.generate_proof_bundle_resident(tip, [], [spec], A.WITNESS_BY_REFERENCE | A.RESULT_JSON)):
            with pytest.raises(A.IpcfpError) as e:
                call()
            assert e.value.status == A.ERR_UNSUPPORTED
        # … while the store made by ipcfp_store_create still gives by-reference witnesses
        assert ref.generate_event_proof(ts, spec, A.WITNESS_BY_REFERENCE).witness.n_blocks > 0


def test_empty_store(api):
    got = api.BlockStore.from_rpc_json(np.zeros((0, 38), np.uint8), [b"[]"], verify_cids=True)
    assert got.n_blocks == 0 and got.json_info.parsed_on_device
