"""The storage-path worlds (tests/storage_path_worlds.py) pinned without a GPU: every slot of both trees reads back through the C++
oracle as its dict says, the campaign holds every path status, the per-spec oracle outcomes behind each fault case, the expected
verdict of every hostile proof list against the oracle's verifier, and the case counts, so that no case can go missing from
tests/test_gpu_storage_path_worlds.py."""
import collections

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import storage_path_worlds as W
from tests import storage_paths as SP
from tests import storage_trees as T


@pytest.mark.parametrize("variant", [0, 1])
def test_every_slot_reads_back_through_the_oracle(oracle_mod, ts3_small, variant):
    w = W.build(variant)
    flat, tip = w.tip(ts3_small)
    ostore = oracle_mod.Store(flat.cids, flat.offsets, flat.lengths, flat.blob)
    for a, cstate in w.contract_states.items():
        slots = sorted(w.storage[a]) + [SP.b32(2 ** 255 + a)]
        r = ostore.read_storage_slots(np.frombuffer(cstate, np.uint8), np.frombuffer(b"".join(slots), np.uint8))
        assert r.found.tolist() == [1] * (len(slots) - 1) + [0], a
        assert [bytes(v) for v in r.values[:-1]] == [w.storage[a][s] for s in slots[:-1]], a


def test_campaign_shape():
    w = W.build()
    assert len(w.campaign) == W.CAMPAIGN_N
    statuses = collections.Counter(w.expected(p)[1] for p in w.campaign)
    assert set(statuses) == {A.PATH_OK, A.PATH_INDEX_OUT_OF_RANGE, A.PATH_BAD_BYTES, A.PATH_TOO_LONG}, statuses
    assert {p.actor_id for p in w.campaign} == set(W.ACTORS) | {W.SHARER}
    assert {p.kind for p in w.campaign} == {A.PATH_WORDS, A.PATH_BYTES}
    assert max(len(p.steps) for p in w.campaign) == A.PATH_MAX_STEPS
    deep = W.deep_path()
    specs, status, value, _, _ = w.expected(deep)
    assert (len(specs), status, len(value)) == (A.PATH_MAX_STEPS + A.PATH_MAX_WORDS, A.PATH_OK, 32 * A.PATH_MAX_WORDS)
    assert W.build(1).storage[W.HAND] != w.storage[W.HAND] and W.build(1).storage[1000] == w.storage[1000]


def test_fault_cases_have_two_faults_of_different_status(oracle_mod, ts3_small):
    w = W.build()
    flat, tip = w.tip(ts3_small)
    fs = W.faults()
    assert len(fs) == 2 * len(W.FAULT_PAIRS) == 6
    for f, (name, pname, a, b) in zip(fs, [p for p in W.FAULT_PAIRS for _ in (0, 1)]):
        arrays = f.arrays(flat)
        t2 = T.tipset(ts3_small, arrays, bytes(tip.child_cid), bytes(tip.parent_state_root))
        ostore = oracle_mod.Store(arrays["cids"], arrays["offsets"], arrays["lengths"], arrays["blob"])
        out = W.oracle_outcomes(ostore, t2, W.fault_batch(f.path))
        first, second = (A.ERR_MISSING_BLOCK, A.ERR_DECODE) if f.first == "missing" else (A.ERR_DECODE, A.ERR_MISSING_BLOCK)
        assert out[0] == [None] * len(out[0]) and out[1] == [None] * len(out[1]), f.name
        row = out[2]
        assert row[:a] == [None] * a and row[a] == first and row[b] == second, (f.name, row)
        assert W.first_failure(out) == (first, 2), f.name
    for name, batch, f in W.absent_batches():
        arrays = f.arrays(flat)
        t2 = T.tipset(ts3_small, arrays, bytes(tip.child_cid), bytes(tip.parent_state_root))
        ostore = oracle_mod.Store(arrays["cids"], arrays["offsets"], arrays["lengths"], arrays["blob"])
        want = (A.ERR_MISSING_BLOCK, 0) if name.startswith("wave2") else (A.ERR_ACTOR_NOT_FOUND, 0)
        assert W.first_failure(W.oracle_outcomes(ostore, t2, batch)) == want, name


@pytest.fixture(scope="module")
def verifier_cases(oracle_mod, ts3_small):
    paths, witness, tip, lists = W.verifier_inputs(oracle_mod, ts3_small)
    verdicts = {name: oracle_mod.verify_storage_proofs(witness, tip, _packed(ps)) for name, ps in lists.items()}
    return paths, lists, verdicts


class _packed:
    def __init__(self, proofs):
        self.proofs, self.raw_proofs = proofs, A.pack_storage_proofs(proofs)


def test_hostile_lists_expected_verdicts(verifier_cases):
    paths, lists, verdicts = verifier_cases
    assert tuple(lists) == W.HOSTILE_NAMES
    w = W.build()
    names = {id(p): n for n, p in w.hand.items()}
    honest = W.expected_verdicts(paths, lists["honest-shuffled"], verdicts["honest-shuffled"])
    assert all(v[0] for v in honest)
    assert [v[1:] for v in honest] == [(s, val, specs) for specs, s, val, _, _ in map(w.expected, paths)]

    def by_name(name):
        got = W.expected_verdicts(paths, lists[name], verdicts[name])
        return {names.get(id(p), i): v for i, (p, v) in enumerate(zip(paths, got))}

    def invalid(name):
        return {k for k, v in by_name(name).items() if not v[0]}

    assert invalid("honest+world") == set()
    empty = W.expected_verdicts(paths, [], [])
    assert not any(v[0] for v in empty)
    assert [len(v[3]) for v in empty] == [len(SP.derive(p)[0]) + len(SP.derive(p)[1]) for p in paths]
    for role, pname in (("header", "s65"), ("length", "arr[3]"), ("data", "s65")):
        assert invalid(f"tampered-{role}-before") == set() and invalid(f"tampered-{role}-after") == set(), role
        assert by_name(f"tampered-{role}-before")[pname] == by_name("honest-shuffled")[pname], role
        assert sum(1 for v in verdicts[f"tampered-{role}-before"] if not v) == 1, role
        assert pname in invalid(f"tampered-{role}-only"), role
    # arr[0..7] share the length word: every arr path falls with it
    assert invalid("tampered-length-only") == {f"arr[{i}]" for i in range(8)}
    sharer = next(i for i, p in enumerate(paths) if p.actor_id == W.SHARER)
    assert invalid("other-actor-only") == {sharer}
    assert invalid("found-false-zero") == {"pair", "pair.y"}
    assert invalid("found-false-same-value") == set()    # the verifier compares values; found is not part of the claim
    assert invalid("swapped-data") == {"s65", "s100"}
    assert invalid("second-world") == set(w.hand)       # HAND's state differs; the other actors' proofs still verify
    second = by_name("second-world")
    assert second["s33"][3] == w.expected(w.hand["s33"])[0][:1]    # the header that does not verify adds no data slots


def test_case_counts(verifier_cases):
    paths, lists, verdicts = verifier_cases
    assert len(paths) == len(W.hand_paths()) + 2 + 60 + 12
    assert len(lists) == len(W.HOSTILE_NAMES) == 17
    assert tuple(n for n, _, _ in W.absent_batches()) == W.ABSENT_NAMES
    assert tuple(f.name for f in W.faults()) == W.FAULT_NAMES and len(W.FAULT_NAMES) == 6
    assert len(lists["honest+world"]) == len(lists["honest-shuffled"]) + len(W.world_specs())
