"""IPCFP_RESULT_JSON (include/ipcfp.h): the EventProofBundle text rendered on the device (csrc/json.cu) must be byte for byte what
ipcfp_event_result_to_json renders on the host from the flagless result of the same store, and what bundle_json.py renders; everything
else of the result is unchanged. (An opt-in mode: last in the suite, with the other one.)"""
import ctypes as C
import json

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import bundle_json as J
from tests.util import EditedTipset, ShuffledTipset, spec_of, synth_tipset

pytestmark = pytest.mark.gpu


def _call(api, store, ts, spec, flags, resident=False):
    """One generate_event_proof call through the C ABI → (EventResultPy, host rendering of the C result or None)."""
    L = api.lib()
    d, keep = A.make_tipset_desc(ts)
    out = C.POINTER(A.EventResultC)()
    if resident:
        th = C.c_void_p()
        api._check(L.ipcfp_tipset_upload(store._h, C.byref(d), C.byref(th)))
        try:
            st = L.ipcfp_generate_event_proof_resident(store._h, th, C.byref(spec), flags, C.byref(out))
        finally:
            L.ipcfp_tipset_free(th)
    else:
        st = L.ipcfp_generate_event_proof(store._h, C.byref(d), C.byref(spec), flags, C.byref(out))
    api._check(st)
    try:
        host = None if flags & (A.RESULT_JSON | A.WITNESS_BY_REFERENCE) else api.event_result_to_json(out, ts)
        if not flags & A.RESULT_JSON:
            assert not out.contents.json and out.contents.json_len == 0
        return A.event_result_from_c(out.contents), host
    finally:
        L.ipcfp_event_result_free(out)


def _check(api, ts, flags=0, resident_too=True, store=None):
    spec = spec_of(ts)
    store = store or api.BlockStore.from_tipset(ts)
    base, want = _call(api, store, ts, spec, flags)
    assert base.json is None
    assert want == J.dumps(J.event_bundle(ts, base))
    for resident in ((False, True) if resident_too else (False,)):
        for extra in (A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE):
            got, _ = _call(api, store, ts, spec, flags | extra, resident)
            assert len(got.json) == len(want)
            assert got.json == want, (resident, extra)
            assert got.matching.tolist() == base.matching.tolist() and got.n_exec == base.n_exec
            assert [p.key() for p in got.proofs] == [p.key() for p in base.proofs]   # topics and data included (the blob bytes of
            # skipped slots are never written, so the blobs are compared through the proofs)
            assert len(got.data_blob) == len(base.data_blob)
            assert np.array_equal(got.witness.cids, base.witness.cids) and np.array_equal(got.witness.lengths, base.witness.lengths)
            if extra & A.WITNESS_BY_REFERENCE:
                assert len(got.witness.blob) == 0
            else:
                assert got.witness.blocks() == base.witness.blocks()
            assert got.timings["json"] > 0
    doc = json.loads(want)
    assert list(doc) == ["proofs", "blocks"] and len(doc["proofs"]) == len(base.proofs) and len(doc["blocks"]) == base.witness.n_blocks
    return base, want


@pytest.mark.parametrize("cfg", [1, 2, "shapes", "shapes-nofilter"])
def test_json_equals_host_renderers(api, synth_mod, cfg):
    base, _ = _check(api, synth_tipset(synth_mod, cfg))
    assert base.proofs


@pytest.mark.parametrize("kw", [
    dict(n_receipts=300, events_per_receipt=40, match_ppm=100000),
    dict(n_receipts=500, events_per_receipt=3, null_root_permille=200, match_ppm=200000),
    dict(n_receipts=257, events_per_receipt=8, bw3_permille=1000, match_ppm=50000, has_actor_filter=0),
    dict(n_receipts=1000, events_per_receipt=8, case_a_permille=500, malformed_permille=100, match_ppm=30000),
    dict(n_receipts=1, events_per_receipt=1, match_ppm=1000000, dup_msgs=0, n_parents=1),
    dict(n_receipts=9, events_per_receipt=8, match_ppm=0, n_parents=3, dup_msgs=2),
    dict(n_receipts=700, events_per_receipt=300, match_ppm=20000, n_parents=1),
])
def test_json_event_proof_shapes(api, synth_mod, kw):
    base, text = _check(api, synth_mod.Tipset(synth_mod.default_params(seed=99, **kw)), resident_too=False)
    if kw.get("match_ppm") == 0:
        assert text.startswith('{"proofs":[],"blocks":[')


def test_json_skips_receipts_missing_from_the_amt(api, synth_mod):
    """Proof slots pass 2 reserved for receipts the receipts AMT does not hold (the host compacts them away) are not rendered."""
    import cbor2
    from oracle import pyoracle as P
    ts = synth_mod.Tipset(synth_mod.default_params(seed=21, n_receipts=40, events_per_receipt=4, match_ppm=400000, n_parents=1, dup_msgs=0))
    d = ts.as_dict()
    height, count, node = cbor2.loads(d[bytes(ts.receipts_root)])
    bmap, links, vals = node
    root_b = cbor2.dumps([height, count, [bytes([bmap[0] & 0x0f]), links[:4], vals]])
    new_root = P.cid_of(root_b)
    hdr = cbor2.loads(d[bytes(ts.child_cid)])
    hdr[9] = cbor2.CBORTag(42, b"\x00" + new_root)
    hdr_b = cbor2.dumps(hdr)
    blob = bytearray(ts.blob.tobytes())
    offs, lens, cids = list(ts.offsets), list(ts.lengths), [ts.cids]
    for c, b in ((new_root, root_b), (P.cid_of(hdr_b), hdr_b)):
        while len(blob) % 16:
            blob.append(0)
        offs.append(len(blob)); lens.append(len(b)); blob += b
        cids.append(np.frombuffer(c, dtype=np.uint8).reshape(1, 38))
    blob += bytes(32)
    e = EditedTipset(ts, cids=np.concatenate(cids), offsets=np.array(offs, dtype=np.uint64), lengths=np.array(lens, dtype=np.uint32),
                     blob=np.frombuffer(bytes(blob), dtype=np.uint8), n_blocks=len(lens), receipts_root=np.frombuffer(new_root, dtype=np.uint8),
                     child_cid=np.frombuffer(P.cid_of(hdr_b), dtype=np.uint8))
    base, _ = _check(api, e)
    assert any(i >= 32 for i in base.matching.tolist()) and base.proofs and all(p.exec_index < 32 for p in base.proofs)


def test_json_shuffled_misaligned_store(api, ts2):
    _check(api, ShuffledTipset(ts2, seed=5, misalign=True))


def test_json_general_walk(api, synth_mod, monkeypatch):
    monkeypatch.setenv("IPCFP_BFS_GENERAL", "1")
    _check(api, synth_mod.Tipset(synth_mod.default_params(seed=7, n_receipts=700, events_per_receipt=5, match_ppm=50000, n_parents=3, dup_msgs=4)))


def test_json_skip_tx_amts(api, ts2):
    _check(api, ts2, flags=A.SCAN_SKIP_TX_AMTS, resident_too=False)


def test_json_extreme_epochs(api, ts1):
    for pe, ce in ((-(2 ** 63), 2 ** 63 - 1), (-1, 0), (-123456789, 10 ** 18)):
        text = _check(api, EditedTipset(ts1, parent_epoch=pe, child_epoch=ce), resident_too=False)[1]
        assert f'"parent_epoch":{pe},"child_epoch":{ce},' in text


def test_json_full_tipset(api, synth_mod):
    """The 1 M-receipt tipset (BASELINE.json configs[3]): ≈ 92 MB of text, equal byte for byte."""
    ts = synth_mod.Tipset(synth_mod.config_params(4))
    _, want = _check(api, ts, resident_too=False)
    assert len(want) > 50_000_000


def test_json_refused_by_shard_calls_and_launch_count(api, ts2):
    """Shard calls refuse the flag and leave the store serving; a flagless call launches as many kernels before and after JSON calls."""
    spec = spec_of(ts2)
    store = api.BlockStore.from_tipset(ts2)

    def flagless_launches():
        k0 = api.kernel_launch_count()
        r, _ = _call(api, store, ts2, spec, 0)
        return api.kernel_launch_count() - k0, r

    n0, r0 = flagless_launches()
    with pytest.raises(A.IpcfpError) as ei:
        store.generate_event_proof_shard(ts2, spec, 0, int(ts2.n_receipts), 1, 0, flags=A.RESULT_JSON)
    assert ei.value.status == A.ERR_UNSUPPORTED
    L = api.lib()
    d, keep = A.make_tipset_desc(ts2)
    th, out = C.c_void_p(), C.POINTER(A.EventResultC)()
    api._check(L.ipcfp_tipset_upload(store._h, C.byref(d), C.byref(th)))
    try:
        st = L.ipcfp_generate_event_proof_shard_resident(store._h, th, C.byref(spec), 0, int(ts2.n_receipts), 1, 0, A.RESULT_JSON, C.byref(out))
        assert st == A.ERR_UNSUPPORTED and not out
    finally:
        L.ipcfp_tipset_free(th)
    for flags in (A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE):
        assert _call(api, store, ts2, spec, flags)[0].json
    n1, r1 = flagless_launches()
    assert n1 == n0
    assert [p.key() for p in r1.proofs] == [p.key() for p in r0.proofs] and r1.witness.blocks() == r0.witness.blocks()
