"""The hand-built state trees of tests/storage_trees.py are what the GPU storage tests take them for (no GPU): on every success case the
builder's ground truth, the C++ oracle (oracle/oracle.cpp) and the Python oracle (oracle/pyoracle.py, cbor2 + hashlib) give the same
answer; on every case meant to fail the C++ oracle fails with the status the decode contract (DESIGN.md §3) prescribes. The shapes the
cases are named after are checked on the blocks themselves (depths, bitfield sizes, recorded block counts)."""
import cbor2
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from oracle import pyoracle as P
from tests import storage_trees as T


@pytest.fixture(scope="module")
def slot_world(oracle_mod):
    blocks, cases = T.world_slots()
    f = T.Flat(blocks)
    return blocks, cases, oracle_mod.Store(f.cids, f.offsets, f.lengths, f.blob)


@pytest.fixture(scope="module")
def proof_world(oracle_mod, ts3_small):
    w, f = T.world_proofs(ts3_small)
    return w, f, oracle_mod.Store(f.cids, f.offsets, f.lengths, f.blob)


def test_slot_cases_agree_with_both_oracles(slot_world):
    blocks, cases, store = slot_world
    assert len(cases) > 100
    for c in cases:
        if c.truth is None:
            with pytest.raises(A.IpcfpError) as ei:
                store.read_storage_slots(c.root_np(), c.slots_np())
            assert ei.value.status == c.status, c.name
            continue
        r = store.read_storage_slots(c.root_np(), c.slots_np())
        assert r.found.tolist() == [int(v is not None) for v in c.truth], c.name
        assert r.raw_len.tolist() == [len(v or b"") for v in c.truth], c.name
        assert [bytes(v) for v in r.values] == [T.left_pad_32(v or b"") for v in c.truth], c.name
        assert r.witness.n_blocks > 0 and all(T.cid_of(r.witness.block(i)) == bytes(r.witness.cids[i]) for i in range(r.witness.n_blocks))
        for s, v in list(zip(c.slots, c.truth))[:40]:
            rec = P.Recorder(blocks)
            assert P.read_storage_slot(rec, c.root, s) == v, c.name
        # the mixed batches hold present and absent slots alike
        assert c.truth.count(None) not in (0, len(c.truth)) or len(c.slots) <= 3 or c.name.startswith("depth"), c.name


def test_slot_cases_have_their_shapes(slot_world):
    blocks, cases, store = slot_world
    by = {c.name: c for c in cases}
    for bw in T.WIDTHS:
        n = T.max_levels(bw)
        # wrapper + n chain nodes, every one visited by the present key
        for name in (f"depth-w{bw}-{n}", f"depth-w{bw}-{n}-absent"):
            r = store.read_storage_slots(by[name].root_np(), by[name].slots_np()[:1])
            assert r.witness.n_blocks == 1 + n, name
    # width 8: a root bitfield of 32 bytes, and lookups whose root index is ≥ 128
    c = by["B1-w8-n5000"]
    root = bytes(cbor2.loads(blocks[c.root])[0].value[1:])
    assert len(cbor2.loads(blocks[root])[0]) == 32
    assert sum(T.hash_index(s, 0, 8) >= 128 for s, v in zip(c.slots, c.truth) if v is not None) > 20
    # the value heads: 8x, 98 xx, 99 xxxx; values longer than 32 bytes
    lens = {len(v) for v in by["values-w5"].truth if v is not None}
    assert {0, 23, 24, 255, 256, 300} <= lens
    # bucket sizes past 23 (a `98` head) and bitfields with leading zero bytes
    assert any(len(b) == 24 for b in cbor2.loads(blocks[by["bucket-24"].root])[1] if isinstance(b, list))
    assert blocks[by["bitfield-leading-zeros"].root][1:3] == b"\x58\x20"


def test_proof_cases_agree_with_both_oracles(oracle_mod, proof_world):
    w, f, store = proof_world
    ok, bad = T.proof_batches(w)
    for tip, specs in ok:
        ts = w.tips[tip]
        r = store.generate_storage_proofs(ts, specs)
        for (actor, slot), p, sw in zip(specs, r.proofs, r.spec_witness):
            v = T.proof_truth(w, tip, actor, slot)
            assert (p.found, p.raw_len, bytes(p.value)) == (v is not None, len(v or b""), T.left_pad_32(v or b"")), (tip, actor)
            py = P.generate_storage_proof(f.blocks, ts, actor, slot)
            assert (py["found"], py["raw"], py["value"]) == (v is not None, v or b"", T.left_pad_32(v or b""))
            assert bytes(p.actor_state_cid) == py["actor_state_cid"] and bytes(p.storage_root) == py["storage_root"]
            assert sorted(bytes(r.witness.cids[i]) for i in sw) == sorted(py["witness"]), (tip, actor)
        assert all(oracle_mod.verify_storage_proofs(r.witness, ts, r))
    # the deepest path: header, StateRoot, 51 actors nodes, EVM state, B1 wrapper, 256 storage nodes
    r = store.generate_storage_proofs(w.tips["deep"], [(w.deep_actor, w.deep_slot)])
    assert len(r.spec_witness[0]) == 311 and r.proofs[0].found
    for tip, specs in bad:
        with pytest.raises(A.IpcfpError) as ei:
            store.generate_storage_proofs(w.tips[tip], specs)
        assert (ei.value.index, ei.value.status) == (len(specs) - 1, A.ERR_ACTOR_NOT_FOUND if specs[-1][0] not in w.actors and tip == "main"
                                                     else A.ERR_DECODE), (tip, specs[-1][0])


def test_actor_keys_and_faults(proof_world):
    w, f, store = proof_world
    assert [len(T.id_address(a)) for a in T.ACTOR_IDS] == [2, 3, 11, 11]
    for aid, (key, child, root) in w.faults.items():
        # the faulted node is a child of the root on `key`'s path, and only that actor's trie holds it
        assert child in f.blocks and T._child_on_path(f.blocks, root, key, {2001: 2, 2002: 6}[aid]) == child
