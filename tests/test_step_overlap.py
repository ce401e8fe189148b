"""Guards for any change to the order or the streams of generate_event_proof's phases (message-AMT walk, pass 1, pass 2, witness
copy): which fault is reported when the message AMTs and pass 1 both fail, a store reused after failed calls (per-call buffers
are freed in stream order), and the dense walk's fallback with matches present."""
import cbor2
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests.test_oracle_cpu import _patched
from tests.util import EditedTipset, assert_event_results_equal, spec_of

pytestmark = pytest.mark.gpu


def _without(ts, cids):
    gone = {bytes(c) for c in cids}
    keep = [i for i in range(ts.n_blocks) if bytes(ts.cids[i]) not in gone]
    return EditedTipset(ts, cids=ts.cids[keep], offsets=ts.offsets[keep], lengths=ts.lengths[keep], n_blocks=len(keep))


def _outcome(make_store, ts, spec):
    try:
        return ("ok", make_store().generate_event_proof(ts, spec))
    except A.IpcfpError as e:
        return ("err", e.status, e.index)


def test_message_amt_fault_wins_over_pass1_fault(api, oracle_mod, ts2):
    """A message-AMT node and the events root of receipt 0 are both missing: the walk's fault is reported, as by the reference."""
    spec = spec_of(ts2)
    assert ts2.has_events_root[0]
    d = ts2.as_dict()
    tm = cbor2.loads(d[bytes(ts2.parent_txmeta_cids[0])])
    msg_node = cbor2.loads(d[tm[0].value[1:]])[2][1][0].value[1:]   # first child of the BLS message AMT
    pass1_only = _without(ts2, [ts2.events_roots[0]])
    both = _without(ts2, [msg_node, ts2.events_roots[0]])
    o1 = _outcome(lambda: oracle_mod.Store.from_tipset(pass1_only), pass1_only, spec)
    o = _outcome(lambda: oracle_mod.Store.from_tipset(both), both, spec)
    g = _outcome(lambda: api.BlockStore.from_tipset(both), both, spec)
    assert o1[0] == o[0] == g[0] == "err"
    assert o1[2] == 0 and o != o1            # the two faults are told apart by the reference
    assert g[1:] == o[1:], (o, g)


def test_failed_calls_leave_the_store_healthy(api, oracle_mod, ts2):
    """One store: a call that fails in the message AMTs, a call that fails in pass 1, then a healthy call whose results must be
    those of the reference, three times over."""
    spec = spec_of(ts2)
    exp = oracle_mod.Store.from_tipset(ts2).generate_event_proof(ts2, spec)
    store = api.BlockStore.from_tipset(ts2)
    bad_txmeta = ts2.parent_txmeta_cids.copy()
    bad_txmeta[1, -1] ^= 0xFF
    bad_root = ts2.events_roots.copy()
    bad_root[7, -1] ^= 0xFF
    faulting = [EditedTipset(ts2, parent_txmeta_cids=bad_txmeta), EditedTipset(ts2, events_roots=bad_root)]
    for _ in range(3):
        for ts in faulting:
            o = _outcome(lambda: oracle_mod.Store.from_tipset(ts), ts, spec)
            g = _outcome(lambda: store, ts, spec)
            assert o[0] == g[0] == "err"
            assert g[1:] == o[1:], (o, g)
        assert_event_results_equal(store.generate_event_proof(ts2, spec), exp)


def test_dense_walk_fallback_with_matches(api, oracle_mod, ts2):
    """A message-AMT leaf with a hole makes the dense walk give up and redo the walk with the general kernels; with matches
    present, pass 2 must pair pass 1's matches with the execution order of the second walk, as the reference does."""
    spec = spec_of(ts2)
    d = ts2.as_dict()
    tm = cbor2.loads(d[bytes(ts2.parent_txmeta_cids[0])])
    root_cid = tm[0].value[1:]
    height, count, node = cbor2.loads(d[root_cid])
    cur_cid, cur = root_cid, node
    while cur[1]:
        cur_cid = cur[1][0].value[1:]
        cur = cbor2.loads(d[cur_cid])
    bmap, _, vals = cur
    assert height > 0 and len(vals) >= 2
    last = max(b for b in range(8) if bmap[0] >> b & 1)
    ts = _patched(ts2, cur_cid, cbor2.dumps([bytes([bmap[0] & ~(1 << last)]), [], vals[:-1]]))
    exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec)
    assert len(exp.matching) > 0
    assert_event_results_equal(api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec), exp)
