"""ipcfp_generate_actor_proofs_resident, ipcfp_plan_fetch_actor_proofs_resident and ipcfp_verify_actor_proofs on the GPU (include/ipcfp.h,
DESIGN.md §2 "Actor proofs") on the hand-built state trees of tests/actor_trees.py, against its Python restatement: every field of every
proof, the statuses, the per-proof witness lists and the union, in both witness modes, with the fast HAMT node decoder and with
IPCFP_HAMT_STRICT=1. Also: failures by (status, index), refusals, batches of 0, 1 and IPCFP_ACTOR_MAX, the verifier on every generated
proof and on changed claims, the fetch loop from an empty store, and the cross-checks against storage proofs and address resolution."""
import ctypes as C
import random

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from oracle.pyoracle import keccak256
from tests import actor_trees as AT
from tests import address_trees as R
from tests import rpc_blocks as B
from tests import storage_trees as T

pytestmark = pytest.mark.gpu

NAMES = [t.name for t in AT.blocks_and_trees()[1]]


@pytest.fixture(scope="module")
def world(api, ts3_small):
    blocks, trees, main, flat = AT.world(ts3_small)
    store = api.BlockStore(flat.cids, flat.offsets, flat.lengths, flat.blob, verify_cids=True)
    yield blocks, trees, main, flat, store
    store.close()


@pytest.fixture(params=[None, "1"], ids=["fast", "strict"])
def mode(request, monkeypatch):
    if request.param:
        monkeypatch.setenv("IPCFP_HAMT_STRICT", request.param)
    else:
        monkeypatch.delenv("IPCFP_HAMT_STRICT", raising=False)


def _generate(store, t, addrs=None, evm=None, with_code=None, flags=0):
    tip = store.upload_tipset(t.tip)
    try:
        return store.generate_actor_proofs_resident(tip, t.addrs if addrs is None else addrs, AT.EVM_SETS[t.evm] if evm is None else evm,
                                                    t.with_code if with_code is None else with_code, flags)
    finally:
        tip.close()


def _check(blocks, store, t, addrs=None, evm=None, with_code=None, flags=0):
    """The call == the restatement: proofs, per-proof lists, union (bytes too), or the same (status, index). → the result or None."""
    addrs = t.addrs if addrs is None else addrs
    evm = AT.EVM_SETS[t.evm] if evm is None else evm
    with_code = t.with_code if with_code is None else with_code
    try:
        exp = AT.prove(blocks, t.child, t.root, addrs, evm, with_code)
    except AT.Failure as f:
        with pytest.raises(A.IpcfpError) as e:
            _generate(store, t, addrs, evm, with_code, flags)
        assert (e.value.status, e.value.index) == (f.status, f.index), t.name
        return None
    got = _generate(store, t, addrs, evm, with_code, flags)
    proofs, lists, union = exp
    assert [vars(p) for p in got.proofs] == proofs, t.name
    cids = [bytes(c) for c in got.witness.cids]
    assert cids == union, t.name
    assert [[cids[k] for k in w] for w in got.proof_witness] == lists, t.name
    if flags & A.WITNESS_BY_REFERENCE:
        assert len(got.witness.blob) == 0
    else:
        assert got.witness.blocks() == [blocks[c] for c in union], t.name
    return got


@pytest.mark.parametrize("name", NAMES)
def test_trees(world, mode, name):
    blocks, trees, _, _, store = world
    t = trees[name]
    got = _check(blocks, store, t)
    assert (got is None) == (t.status is not None), name
    if got is not None and t.name == "main":
        assert {p.status for p in got.proofs} == {A.ACTOR_FOUND, A.ACTOR_NO_ADDRESS, A.ACTOR_NO_ACTOR}


@pytest.mark.parametrize("name", ["main", "main-code", "actors-100000", "deep"])
def test_witness_by_reference(world, name):
    blocks, trees, _, _, store = world
    _check(blocks, store, trees[name], flags=A.WITNESS_BY_REFERENCE)


@pytest.mark.parametrize("evm", list(AT.EVM_SETS))
def test_evm_code_sets(world, evm):
    blocks, trees, _, _, store = world
    got = _check(blocks, store, trees["main"], evm=AT.EVM_SETS[evm])
    assert sum(p.is_evm for p in got.proofs) == {"none": 0, "one": 4, "several": 6}[evm]


def test_ground_truth(world, api):
    blocks, trees, main, _, store = world
    t = trees["main-code"]
    got = _generate(store, t)
    by_id = {p.actor_id: p for p in got.proofs if p.address[0] == 0}
    mags = {"zero": 0, "one-byte": 5, "twelve-bytes": 2 ** 95 - 7, "thirty-two-bytes": 2 ** 256 - 1, "negative": -(2 ** 90 + 3),
            "plus-zero": 0, "minus-zero": 0, "leading-zeros": 7}
    for aid, kind in main["actors"].items():
        if kind.startswith("balance-"):
            assert by_id[aid].balance == mags[kind[8:]], kind
    assert by_id[120].delegated is not None and by_id[100].delegated is None
    v6, v5 = by_id[121], by_id[122]
    assert v6.is_evm and v5.is_evm and v5.evm_nonce == 0 and by_id[123].evm_nonce == 2 ** 64 - 1
    for p in (v6, v5):
        assert keccak256(p.bytecode) == p.bytecode_hash
    for a, aid in main["amap"].items():
        p = next(p for p in got.proofs if p.address == a)
        assert p.actor_id == aid and p.status == (A.ACTOR_FOUND if aid != 5555 else A.ACTOR_NO_ACTOR)


@pytest.mark.parametrize("n", [0, 1, A.ACTOR_MAX])
def test_batches(world, n):
    """Requests drawn with repeats from the 100 000-actor tree's: every proof and list is its address's, the union theirs."""
    blocks, trees, _, _, store = world
    t = trees["actors-100000"]
    rng = random.Random(n)
    addrs = [rng.choice(t.addrs) for _ in range(n)]
    uniq = sorted(set(addrs))
    proofs, lists, union = AT.prove(blocks, t.child, t.root, uniq, AT.EVM_SETS[t.evm])
    by = {a: (p, l) for a, p, l in zip(uniq, proofs, lists)}
    got = _generate(store, t, addrs=addrs)
    cids = [bytes(c) for c in got.witness.cids]
    assert cids == union and got.host_syncs == 4 and len(got.proofs) == n
    for a, p, w in zip(addrs, got.proofs, got.proof_witness):
        assert (vars(p), [cids[k] for k in w]) == by[a]


def test_refusals(world, api):
    blocks, trees, _, _, store = world
    t = trees["main"]
    for addrs, index in (([R.id_addr(1), b"\x05" + bytes(20)], 1), ([b"\x00\x80"], 0), ([b"\x01" + bytes(19)], 0)):
        with pytest.raises(A.IpcfpError) as e:
            _generate(store, t, addrs=addrs)
        assert (e.value.status, e.value.index) == (A.ERR_INVALID_ARG, index)
    with pytest.raises(A.IpcfpError) as e:
        _generate(store, t, addrs=[R.id_addr(0)] * (A.ACTOR_MAX + 1))
    assert e.value.status == A.ERR_INVALID_ARG
    with pytest.raises(A.IpcfpError) as e:
        _generate(store, t, flags=0x40)
    assert e.value.status == A.ERR_INVALID_ARG
    L = api.lib()
    tip = store.upload_tipset(t.tip)
    try:
        out = C.POINTER(A.ActorResultC)()
        assert L.ipcfp_generate_actor_proofs_resident(store._h, tip._h, None, 3, None, 0, 0, C.byref(out)) == A.ERR_INVALID_ARG
        addrs = A.make_addresses([R.id_addr(0)])
        assert L.ipcfp_generate_actor_proofs_resident(store._h, tip._h, addrs, 1, None, 2, 0, C.byref(out)) == A.ERR_INVALID_ARG
    finally:
        tip.close()


def test_state_root_mismatch(world, ts3_small):
    blocks, trees, _, flat, store = world
    t, other = trees["main"], trees["actors-1000"]
    bad = T.tipset(ts3_small, flat.arrays(), t.child, other.root)
    with pytest.raises(A.IpcfpError) as e:
        tip = store.upload_tipset(bad)
        try:
            store.generate_actor_proofs_resident(tip, [R.id_addr(0)])
        finally:
            tip.close()
    assert (e.value.status, e.value.index) == (A.ERR_STATE_ROOT_MISMATCH, 0)


def test_descriptor_form_equals_resident(world, api):
    blocks, trees, _, _, store = world
    t = trees["main-code"]
    got = _generate(store, t)
    d, keep = A.make_tipset_desc(t.tip)
    addrs = A.make_addresses(t.addrs)
    ev = np.frombuffer(b"".join(AT.EVM_SETS[t.evm]), np.uint8).copy()
    again = api._result("ipcfp_generate_actor_proofs", A.ActorResultC, A.actor_result_from_c, "ipcfp_actor_result_free", store._h, C.byref(d),
                        addrs, len(t.addrs), ev.ctypes.data, len(AT.EVM_SETS[t.evm]), A.ACTOR_WITH_CODE)
    assert np.array_equal(again.raw_proofs, got.raw_proofs) and np.array_equal(again.witness.cids, got.witness.cids)


# ------------------------------------------------------------------ the verifier
def _claims(raw):
    return (A.ActorProofC * (len(raw) // C.sizeof(A.ActorProofC))).from_buffer_copy(raw.tobytes())


@pytest.mark.parametrize("name", ["main", "main-code", "actors-100000", "deep", "no-init-actor-ids-only"])
def test_verifier_accepts_and_rejects(world, api, name):
    """Every generated proof verifies; each proof with one claim changed (field, absence or presence) does not. The replay follows the
    address alone, so every changed claim is replayed on the same blocks and all of them go into one call."""
    blocks, trees, _, _, store = world
    t = trees[name]
    got = _generate(store, t)
    evm = AT.EVM_SETS[t.evm]
    assert api.verify_actor_proofs(got.witness, t.tip, got, evm, t.with_code) == [True] * len(got.proofs)
    recs = _claims(got.raw_proofs)
    edits = {
        "balance": lambda p: p.balance.__setitem__(31, p.balance[31] ^ 1),
        "sign": lambda p: setattr(p, "balance_negative", 1 - p.balance_negative),
        "nonce": lambda p: setattr(p, "sequence", p.sequence + 1),
        "code": lambda p: p.code.__setitem__(37, p.code[37] ^ 1),
        "head": lambda p: p.head.__setitem__(37, p.head[37] ^ 1),
        "delegated": lambda p: (setattr(p, "has_delegated", 1), setattr(p.delegated, "len", 21), p.delegated.bytes.__setitem__(1, 0x77)),
        "evm-nonce": lambda p: setattr(p, "evm_nonce", p.evm_nonce ^ 1),
        "contract-state": lambda p: p.contract_state.__setitem__(37, p.contract_state[37] ^ 1),
        "bytecode-cid": lambda p: p.bytecode_cid.__setitem__(37, p.bytecode_cid[37] ^ 1),
        "bytecode-hash": lambda p: p.bytecode_hash.__setitem__(0, p.bytecode_hash[0] ^ 1),
        "is-evm": lambda p: setattr(p, "is_evm", 1 - p.is_evm),
        "absent": lambda p: setattr(p, "status", A.ACTOR_NO_ACTOR if p.status == A.ACTOR_FOUND else A.ACTOR_FOUND),
        "no-address": lambda p: setattr(p, "status", A.ACTOR_NO_ADDRESS if p.status != A.ACTOR_NO_ADDRESS else A.ACTOR_FOUND),
        "actor-id": lambda p: setattr(p, "actor_id", p.actor_id ^ 1),
    }
    if t.with_code:
        edits["bytecode"] = lambda p: setattr(p, "code_len", p.code_len + 1)
    changed = []
    for k in range(len(recs)):
        for what, edit in edits.items():
            one = (A.ActorProofC * 1).from_buffer_copy(bytes(recs[k]))
            edit(one[0])
            if bytes(one[0]) != bytes(recs[k]):
                changed.append(bytes(one[0]))
    assert len(changed) >= 10 * len(recs)
    raw = np.frombuffer(b"".join(changed), np.uint8).copy()
    assert api.verify_actor_proofs(got.witness, t.tip, raw, evm, t.with_code) == [False] * len(changed)


def test_verifier_witness_faults(world, api):
    blocks, trees, _, _, store = world
    t = trees["main-code"]
    got = _generate(store, t)
    w = got.witness
    # every block of the union left out in turn: each call fails or rejects, never accepts a claim it cannot replay
    for drop in range(w.n_blocks):
        keep = [i for i in range(w.n_blocks) if i != drop]
        part = A.WitnessPy(w.cids[keep], w.offsets[keep], w.lengths[keep], w.blob)
        needs = [k for k, lst in enumerate(got.proof_witness) if drop in lst]
        try:
            verdict = api.verify_actor_proofs(part, t.tip, got, AT.EVM_SETS[t.evm], True)
        except A.IpcfpError as e:
            assert e.status in (A.ERR_MISSING_BLOCK, A.ERR_DECODE, A.ERR_ACTOR_NOT_FOUND)
            continue
        assert not needs, drop


# ------------------------------------------------------------------ the fetch loop
def _fetcher(full, held):
    def fetch(cids, first_id):
        els = []
        for k, c in enumerate(cids):
            c = bytes(c)
            assert c not in held, "a CID was requested twice"
            held[c] = full[c]
            els.append(B.element(first_id + k, full[c]))
        return B.render([], elements=els)
    return fetch


@pytest.mark.parametrize("name", ["main-code", "actors-1000", "deep", "no-init-actor-ids-only"])
def test_fetch_loop_fetches_exactly_the_read_set(world, api, name):
    blocks, trees, _, _, store = world
    t = trees[name]
    full = _generate(store, t)
    held = {}
    st, tip, rounds, _, _ = api.fetch_actor_proofs_until_complete(_fetcher(blocks, held), lambda s: s.upload_tipset(t.tip), t.addrs,
                                                                  AT.EVM_SETS[t.evm], t.with_code)
    try:
        assert set(held) == {bytes(c) for c in full.witness.cids} and len(rounds) >= 1
        again = st.generate_actor_proofs_resident(tip, t.addrs, AT.EVM_SETS[t.evm], t.with_code)
        assert np.array_equal(again.raw_proofs, full.raw_proofs) and np.array_equal(again.witness.cids, full.witness.cids)
    finally:
        tip.close()
        st.close()


# ------------------------------------------------------------------ cross-checks
def test_storage_world_cross_check(api, ts3_small):
    w, f = T.world_proofs(ts3_small)
    store = api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True)
    try:
        tipset = w.tips["main"]
        specs = [(a, s) for a in T.ACTOR_IDS + tuple(w.fillers[:20]) for s in list(w.actors[a][1])[:1]]
        sp = store.generate_storage_proofs(tipset, specs)
        tip = store.upload_tipset(tipset)
        try:
            got = store.generate_actor_proofs_resident(tip, [a for a, _ in specs], [AT.EVM_A])
        finally:
            tip.close()
        cids = [bytes(c) for c in got.witness.cids]
        scids = [bytes(c) for c in sp.witness.cids]
        for p, q, lst, slst in zip(got.proofs, sp.proofs, got.proof_witness, sp.spec_witness):
            assert p.status == A.ACTOR_FOUND and p.head == q.actor_state_cid and p.contract_state == q.storage_root
            assert {cids[k] for k in lst} <= {scids[k] for k in slst}
    finally:
        store.close()


def test_non_id_actor_id_equals_resolution(world):
    blocks, trees, main, _, store = world
    t = trees["actors-100000"]
    others = [a for a in t.addrs if a[0] != 0]
    got = _generate(store, t, addrs=others)
    r = store.resolve_addresses(t.root, others)
    for p, s, i in zip(got.proofs, r.status.tolist(), r.actor_ids.tolist()):
        assert (p.status == A.ACTOR_NO_ADDRESS) == (s == A.ERR_ACTOR_NOT_FOUND)
        if s == A.OK:
            assert p.actor_id == i


@pytest.mark.parametrize("forgery", ["forged-no-actor", "forged-balance", "forged-evm", "forged-no-address"])
def test_verifier_never_accepts_a_forged_claim(world, api, forgery):
    """Hostile witnesses whose every block hashes to its CID (the approach of tests/hostile_witness.py): the forgery is a well-formed state
    tree that differs from main in one claim (a false absence of an actor or an address, another balance, another EVM state). Its proofs,
    verified against main's tipset over main's witness with the forged blocks added, or over the forged blocks alone, are never accepted
    where they differ from main's proof; against the forged tree's own tipset they verify (they are true there)."""
    blocks, trees, _, _, store = world
    t, f = trees["main-code"], trees[forgery]
    evm = AT.EVM_SETS[t.evm]
    true = _generate(store, t)
    lie = _generate(store, f)
    assert api.verify_actor_proofs(lie.witness, f.tip, lie, evm, True) == [True] * len(lie.proofs)
    differs = [vars(p) != vars(q) for p, q in zip(lie.proofs, true.proofs)]
    assert any(differs)
    merged = {**true.witness.as_dict(), **lie.witness.as_dict()}
    both = A.WitnessPy(*T.Blocks(merged).flat())
    for w in (both, lie.witness):
        try:
            verdict = api.verify_actor_proofs(w, t.tip, lie, evm, True)
        except A.IpcfpError as e:
            assert e.status in (A.ERR_MISSING_BLOCK, A.ERR_DECODE)
            continue
        for d, v in zip(differs, verdict):
            assert not (d and v)
