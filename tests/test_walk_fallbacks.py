"""The message-AMT walk of an unsharded generate_event_proof is planned on the device (k_setup) and learns only at the synchronisation
after the witness snapshot whether the plan held. Each way it can give up must end in the reference's results: a plan that is not
taken (more messages than the receipts allow), a level above the leaves that is not what the plan expects, and a leaf that does not
decode while pass 1 fails too (the walk's fault outranks pass 1's)."""
import cbor2
import numpy as np
import pytest

from tests.test_oracle_cpu import _patched
from tests.test_step_overlap import _outcome, _without
from tests.util import EditedTipset, assert_event_results_equal, spec_of

pytestmark = pytest.mark.gpu


def _first_path(d, root_cid, depth):
    """CIDs and decoded nodes along the first-child path of a message AMT, `depth` links below its root."""
    height, count, node = cbor2.loads(d[root_cid])
    path = [(root_cid, node)]
    for _ in range(depth):
        cid = path[-1][1][1][0].value[1:]
        path.append((cid, cbor2.loads(d[cid])))
    return height, count, path


def _bls_root(ts):
    tm = cbor2.loads(ts.as_dict()[bytes(ts.parent_txmeta_cids[0])])
    return tm[0].value[1:]


def test_hole_above_the_leaves(api, oracle_mod, ts2):
    """A level-1 node of a message AMT lacks its last child: the dense walk gives up before its last round, and the general walk's
    execution order (shorter by that child's messages) pairs with pass 1's matches as in the reference."""
    spec = spec_of(ts2)
    d = ts2.as_dict()
    height, _, path = _first_path(d, _bls_root(ts2), 0)
    assert height >= 2
    height, _, path = _first_path(d, _bls_root(ts2), height - 1)
    cid, (bmap, links, vals) = path[-1]
    assert not vals and len(links) >= 2
    last = max(b for b in range(8) if bmap[0] >> b & 1)
    ts = _patched(ts2, cid, cbor2.dumps([bytes([bmap[0] & ~(1 << last)]), links[:-1], []]))
    exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec)
    assert exp.n_exec < oracle_mod.Store.from_tipset(ts2).generate_event_proof(ts2, spec).n_exec
    assert_event_results_equal(api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec), exp)


def test_leaf_decode_fault_wins_over_pass1_fault(api, oracle_mod, ts2):
    """A message-AMT leaf that does not decode and a missing events root of receipt 0: the dense walk's last round gives up and
    pass 1 fails too; the message-AMT fault is reported, as by the reference."""
    spec = spec_of(ts2)
    d = ts2.as_dict()
    height, _, _ = _first_path(d, _bls_root(ts2), 0)
    _, _, path = _first_path(d, _bls_root(ts2), height)
    leaf_cid, (_, links, vals) = path[-1]
    assert not links and vals
    pass1_only = _without(ts2, [ts2.events_roots[0]])
    both = _patched(pass1_only, leaf_cid, d[leaf_cid][:-7])   # cut inside the last value's CID
    o1 = _outcome(lambda: oracle_mod.Store.from_tipset(pass1_only), pass1_only, spec)
    o = _outcome(lambda: oracle_mod.Store.from_tipset(both), both, spec)
    g = _outcome(lambda: api.BlockStore.from_tipset(both), both, spec)
    assert o1[0] == o[0] == g[0] == "err"
    assert o1[2] == 0 and o != o1            # the two faults are told apart by the reference
    assert g[1:] == o[1:], (o, g)


def test_message_count_above_the_receipts_bound(api, oracle_mod, ts2):
    """The message AMTs hold more values than n_parents × n_receipts + 1024, the dense walk's bound on the list it writes: the
    general walk takes the tipset and gives the reference's results."""
    d = ts2.as_dict()
    total = 0
    for t in ts2.parent_txmeta_cids:
        tm = cbor2.loads(d[bytes(t)])
        total += sum(cbor2.loads(d[tm[k].value[1:]])[1] for k in range(2))
    n = 4000
    assert total > int(ts2.n_parents) * n + 1024
    ts = EditedTipset(ts2, n_receipts=n, events_roots=np.ascontiguousarray(ts2.events_roots[:n]),
                      has_events_root=np.ascontiguousarray(ts2.has_events_root[:n]))
    spec = spec_of(ts)
    exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec)
    assert exp.n_exec == oracle_mod.Store.from_tipset(ts2).generate_event_proof(ts2, spec).n_exec
    assert_event_results_equal(api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec), exp)
