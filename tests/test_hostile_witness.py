"""The hostile-witness catalogues (tests/hostile_witness.py) pinned on the CPU: how many cases each has, that every witness block hashes
to its CID (bar the declared decoys under a class the store does not hash), that the C++ oracle's restated verifier returns each
case's stated verdicts or (status, first failing proof), and that every claim it accepts holds in the chain the child CID commits to."""
import ctypes as C

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import hostile_witness as H

COUNTS = dict(event=235, storage=13, event_batches=66, storage_batches=66)
SMALL = (1, 4, 5, 128, 129)


def oracle_outcome(oracle_mod, c):
    """The oracle's verdicts, or (status, index of the first failing proof): the restated verifier clears results[i] when it starts proof
    i and stops at the first Err, so with the array preset to 2 the failing proof is the last one that is no longer 2."""
    L = oracle_mod.lib()
    r = c.result()
    d, keep = A.make_tipset_desc(c.ts)
    w, keep2 = c.witness().as_c()
    n = len(c.proofs)
    res = np.full(max(n, 1), 2, dtype=np.uint8)
    raw = np.ascontiguousarray(r.raw_proofs)
    if c.kind == "event":
        blob = np.concatenate([np.ascontiguousarray(r.data_blob), np.zeros(16, np.uint8)])
        st = L.oracle_verify_event_proofs(C.byref(w), C.byref(d), raw.ctypes.data, n, blob.ctypes.data, None, res.ctypes.data)
    else:
        st = L.oracle_verify_storage_proofs(C.byref(w), C.byref(d), raw.ctypes.data, n, res.ctypes.data)
    if st != A.OK:
        k = 0
        while k < n and res[k] != 2:
            k += 1
        return (st, max(k - 1, 0))
    return [bool(x) for x in res[:n]]


@pytest.fixture(scope="module")
def event_cases(oracle_mod):
    return H.event_cases()


@pytest.fixture(scope="module")
def storage_cases(ts3_small):
    return H.storage_cases(ts3_small)


def test_case_counts(event_cases, storage_cases, ts3_small):
    assert len(event_cases) == COUNTS["event"] and len(storage_cases) == COUNTS["storage"]
    assert len({c.name for c in event_cases + storage_cases}) == len(event_cases) + len(storage_cases)
    assert len(H.event_batches(SMALL)) == COUNTS["event_batches"] - 12
    assert len(H.storage_batches(ts3_small, SMALL)) == COUNTS["storage_batches"] - 12
    kinds = {c.name.split("-")[0] for c in event_cases}
    assert {"child", "parent1", "parent0", "txmeta0", "txmeta1", "messages", "receipts", "events", "blake2s", "duplicate"} <= kinds


def test_every_block_hashes_to_its_cid(event_cases, storage_cases):
    decoys = 0
    for c in event_cases + storage_cases:
        for cid, b in c.entries:
            h = H.hashes_to_cid(cid, b)
            if h is None:
                assert cid in c.unchecked, c.name
                decoys += 1
            else:
                assert h, (c.name, cid.hex())
    assert decoys == 4


def _check(oracle_mod, c):
    got = oracle_outcome(oracle_mod, c)
    assert got == c.expect, (c.name, got if isinstance(got, tuple) else sum(got), c.expect if c.fails else sum(c.expect))
    if not c.fails:
        holds = H.event_claim_holds if c.kind == "event" else H.storage_claim_holds
        for p, v in zip(c.proofs, got):
            if v:
                assert holds(c.chain, c.ts, p), c.name


def test_oracle_event_verdicts(oracle_mod, event_cases):
    for c in event_cases:
        _check(oracle_mod, c)
    # the suspected-defect shape: a raw-codec TxMeta hides nothing behind a later walk fault
    assert [c.expect for c in event_cases if c.name.startswith("txmeta0-raw+")] == [(A.ERR_CID_MISMATCH, 0)] * 6


def test_oracle_storage_verdicts(oracle_mod, storage_cases):
    for c in storage_cases:
        _check(oracle_mod, c)
    # the trust anchor is the only thing that stops these: the forged claim verifies under the re-anchored child
    forged = [c for c in storage_cases if c.name.startswith("evm-retarget")]
    assert len(forged) == 6 and all(c.expect[-1] and not any(c.expect[k] for k, p in enumerate(c.proofs[:-1]) if p.actor_id == 0) for c in forged)


def test_oracle_batches(oracle_mod, ts3_small):
    for c in H.event_batches(SMALL) + H.storage_batches(ts3_small, SMALL):
        _check(oracle_mod, c)
