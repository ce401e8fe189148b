"""The message-AMT walk on the GPU on hand-built message AMTs and on parent blocks that share their messages (tests/message_amts.py),
against the C++ oracle field by field and against the builder's ground truth (the first-seen execution order), with the default walk
(dense plan, general walk behind it) and with the general walk forced (IPCFP_BFS_GENERAL). Covered: every parent on one TxMeta (2, 5 and
64 parents), shared BLS roots, permutations, interleaved overlaps, CIDs in a BLS and a SECP list, a CID twice in one AMT, a union
shorter than the receipts; AMTs of every height 0–21 with sparse, top and > 2^44 / > 2^64 indices at 1 and 64 parents; single faults
at every height and two faults in one AMT in both orders, below and beyond 2^44; the GPU verifier on the same tipsets; and inputs whose
walk holds more nodes than the store has blocks (the capacity cases), for generate_event_proof and for the verifier."""
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import message_amts as M
from tests.util import assert_event_results_equal, spec_of

pytestmark = pytest.mark.gpu

WALKS = [None, "1"]   # IPCFP_BFS_GENERAL unset / set


@pytest.fixture(scope="module")
def base(synth_mod):
    return M.base_tipset()


@pytest.fixture(scope="module")
def catalogue(base):
    return M.catalogue(base)


@pytest.fixture(scope="module")
def shapes64(base):
    return M.shape_cases(base, copies=(63,))


def _walk(monkeypatch, general):
    if general is None:
        monkeypatch.delenv("IPCFP_BFS_GENERAL", raising=False)
    else:
        monkeypatch.setenv("IPCFP_BFS_GENERAL", general)


def _outcome(fn):
    try:
        return fn(), None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _check(api, oracle_mod, c, verify=True):
    """Engine == oracle (every field, or the same (status, index)); on success == the ground truth, and the GPU verifier == the
    restated verifier on the oracle's proofs. → the oracle's failure or None."""
    ts, spec = c.ts, spec_of(c.ts)
    exp, eerr = _outcome(lambda: oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec))
    got, gerr = _outcome(lambda: api.BlockStore.from_tipset(ts, verify_cids=True).generate_event_proof(ts, spec))
    assert gerr == eerr, (c.name, gerr, eerr)
    if eerr:
        return eerr
    assert (got.n_exec, [p.key() for p in got.proofs]) == (exp.n_exec, [p.key() for p in exp.proofs]), c.name
    assert_event_results_equal(got, exp)
    assert got.n_exec == len(c.truth), c.name
    assert [p.message_cid for p in got.proofs] == [c.truth[p.exec_index] for p in got.proofs], c.name
    if verify:
        want = oracle_mod.verify_event_proofs(exp.witness, ts, exp)
        assert all(want) and api.verify_event_proofs(exp.witness, ts, exp) == want, c.name
    return None


@pytest.mark.parametrize("general", WALKS)
def test_shared_messages(api, oracle_mod, catalogue, monkeypatch, general):
    _walk(monkeypatch, general)
    for c in catalogue:
        if c.name.startswith(("shape-", "missing-", "decode-", "two-faults-")):
            continue
        err = _check(api, oracle_mod, c)
        if getattr(c, "truth_short", False):
            assert err is not None and err[0] == A.ERR_MISSING_EXEC, c.name
        else:
            assert err is None, (c.name, err)


@pytest.mark.parametrize("general", WALKS)
@pytest.mark.parametrize("parents", [1, 64])
def test_hand_built_heights(api, oracle_mod, catalogue, shapes64, monkeypatch, general, parents):
    """Heights 0–21 (20 is the deepest dense plan), roots taller than needed, holes, index 0, the first index of root slot 1, the top
    index, indices beyond 2^44 and 2^64; with 2 message AMTs beside the synthetic parent's the frontier stays in k_amt_top's fused
    rounds up to round 3, with 128 it leaves them after round 1."""
    _walk(monkeypatch, general)
    cases = [c for c in catalogue if c.name.startswith("shape-")] if parents == 1 else shapes64
    assert len(cases) == M.MAX_HEIGHT + 2
    for c in cases:
        assert _check(api, oracle_mod, c, verify=parents == 1) is None, c.name


@pytest.mark.parametrize("general", WALKS)
def test_faults_at_every_height(api, oracle_mod, catalogue, monkeypatch, general):
    """A missing child or an undecodable node at every height 1–21, and two faults in one AMT (root slots 1 and 2) in both orders, with
    subtree bases below 2^44 (height 5) and beyond it (height 15): the failure the in-order walk meets first, as (status, index)."""
    _walk(monkeypatch, general)
    n = 0
    for c in catalogue:
        if c.name.startswith(("missing-", "decode-", "two-faults-")):
            err = _check(api, oracle_mod, c)
            assert err is not None and err[0] == c.status, (c.name, err)
            n += 1
    assert n == 2 * M.MAX_HEIGHT + 4


def _old_bound(n_blocks):
    """The frontier capacity the walk had before it was sized by what it walks: 4 · blocks in the store + 1024."""
    return 4 * int(n_blocks) + 1024


@pytest.mark.parametrize("general", WALKS)
@pytest.mark.parametrize("p", [16, 64])
def test_capacity_generate(api, oracle_mod, synth_mod, monkeypatch, general, p):
    """p parent blocks on one TxMeta of 20 000 messages: each parent's AMTs are walked on their own, so the leaf frontier is p × 2 500
    nodes while the store holds them once."""
    _walk(monkeypatch, general)
    c = M.capacity_case(p)
    assert M.leaf_frontier(c) > _old_bound(c.ts.n_blocks)
    assert _check(api, oracle_mod, c, verify=False) is None


@pytest.mark.parametrize("general", WALKS)
def test_capacity_verify(api, oracle_mod, synth_mod, monkeypatch, general):
    """The GPU verifier walks the message AMTs on the WITNESS store, which holds each shared node once: 8 parents with one 20 000-message
    list give a leaf frontier of 20 000 against about 3 000 witness blocks."""
    _walk(monkeypatch, general)
    c = M.capacity_case(8)
    ts = c.ts
    exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
    assert len(exp.proofs) > 0
    assert M.leaf_frontier(c) > _old_bound(exp.witness.n_blocks)
    want = oracle_mod.verify_event_proofs(exp.witness, ts, exp)
    assert all(want)
    assert api.verify_event_proofs(exp.witness, ts, exp) == want
