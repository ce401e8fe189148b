"""The hand-built message AMTs and shared-message tipsets of tests/message_amts.py are what the GPU tests (tests/test_gpu_message_amts.py)
take them for (no GPU): on every case the builder's ground truth (the first-seen execution order), the C++ oracle (oracle/oracle.cpp) and
the Python oracle (oracle/pyoracle.py) agree — `n_exec` and every proof's `message_cid` on success, the same failure otherwise — and the
oracle's proofs pass its own verifier. The shapes the cases are named after are checked on the blocks themselves."""
import cbor2
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from oracle import pyoracle as P
from tests import message_amts as M
from tests.util import spec_of


@pytest.fixture(scope="module")
def base(synth_mod):
    return M.base_tipset()


@pytest.fixture(scope="module")
def cases(base):
    return M.catalogue(base)


def _oracle(oracle_mod, c):
    ts = c.ts
    try:
        return oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts)), None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _first_match_at_or_after(oracle_mod, base, n):
    full = oracle_mod.Store.from_tipset(base).generate_event_proof(base, spec_of(base))
    return next(i for i in full.matching.tolist() if i >= n)


def test_catalogue_agrees_with_both_oracles(oracle_mod, base, cases):
    assert len(cases) > 60
    n_fail = 0
    for c in cases:
        r, err = _oracle(oracle_mod, c)
        if getattr(c, "truth_short", False):
            # the union is shorter than the receipts: exec.get(i) fails at the first matching receipt past it
            assert err == (A.ERR_MISSING_EXEC, _first_match_at_or_after(oracle_mod, base, len(c.truth))), c.name
            with pytest.raises(IndexError):
                P.generate_event_proof(c.blocks, c.ts, c.ts.event_signature, c.ts.topic1, c.ts.actor_filter)
            continue
        if c.truth is None:
            assert err is not None and err[0] == c.status, (c.name, err)
            with pytest.raises(Exception):
                P.generate_event_proof(c.blocks, c.ts, c.ts.event_signature, c.ts.topic1, c.ts.actor_filter)
            n_fail += 1
            continue
        assert err is None, (c.name, err)
        assert r.n_exec == len(c.truth), c.name
        assert len(r.proofs) > 0, c.name
        for p in r.proofs:
            assert p.message_cid == c.truth[p.exec_index], c.name
        assert all(oracle_mod.verify_event_proofs(r.witness, c.ts, r)), c.name
        py = P.generate_event_proof(c.blocks, c.ts, c.ts.event_signature, c.ts.topic1, c.ts.actor_filter)
        assert py["exec_order"] == c.truth, c.name
        assert [pr[5] for pr in py["proofs"]] == [p.message_cid for p in r.proofs], c.name
    assert n_fail >= 40


def test_capacity_cases_agree_with_the_oracle(oracle_mod, synth_mod):
    """The capacity cases (too large for the Python oracle): the C++ oracle's execution order is the builder's."""
    for p in (8, 16):
        c = M.capacity_case(p)
        r, err = _oracle(oracle_mod, c)
        assert err is None and r.n_exec == len(c.truth) == 20000
        assert all(pr.message_cid == c.truth[pr.exec_index] for pr in r.proofs) and len(r.proofs) > 0
        assert M.leaf_frontier(c) == p * (15000 // 8 + 5000 // 8)


def test_cases_have_their_shapes(base, cases):
    by = {c.name: c for c in cases}
    # shared TxMeta: one TxMeta CID in every parent, P distinct headers
    c = by["same-txmeta-P64"]
    assert len({bytes(x) for x in c.ts.parent_txmeta_cids}) == 1 and len({bytes(x) for x in c.ts.parent_cids}) == 64
    assert int(c.ts.n_parents) == 64
    child = cbor2.loads(c.blocks[bytes(c.ts.child_cid)])
    assert [bytes(x.value[1:]) for x in child[5]] == [bytes(x) for x in c.ts.parent_cids]
    # hand-built heights 0..21, roots one level taller than needed, values beyond 2^44 and 2^64
    for h in range(M.MAX_HEIGHT + 1):
        bls, secp = by[f"shape-h{h}-x1"].amts
        assert cbor2.loads(c.blocks.get(bls.root) or by[f"shape-h{h}-x1"].blocks[bls.root])[0] == h
        assert max(bls.values) == 8 ** (h + 1) - 1
        assert secp.height == h and M.min_height(list(secp.values)) == max(h - 1, 0)
        if h >= 14:
            assert any(i >= 2 ** 44 for i in bls.values)
    assert any(i >= 2 ** 64 for i in by["shape-h21-x1"].amts[0].values)
    # a CID twice inside one AMT; a CID in one parent's SECP list and in another's BLS list
    bls0 = by["cid-twice-in-one-amt"].lists[0][0]
    assert len(bls0) > len(set(bls0))
    l2 = by["secp-then-bls"].lists
    assert set(l2[0][1]) & set(l2[1][0]) and set(l2[1][1]) & set(l2[0][0])
    # the two-fault pairs lie in root slots 1 and 2: bases beyond 2^44 at height 15, below it at height 5
    assert 8 ** 15 > 2 ** 44 > 2 * 8 ** 5
