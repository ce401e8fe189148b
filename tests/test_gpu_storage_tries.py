"""The storage path on the GPU on hand-built state trees (tests/storage_trees.py), against the C++ oracle bit for bit: HAMTs of every bit
width 1–8 behind B1 / B2 wrappers (and C, A1–A3), tries at the depth limit of every width and one level past it, Vec<u8> values of every
head size, odd node shapes, out-of-range wrapper bit widths, full state trees with 11-byte actor keys, the deepest path the decode contract
accepts (311 recorded blocks), several faults in one k_storage_proofs launch, and the unified bundle of the deepest tree. Found flags,
raw lengths, values and witnesses are compared; for proofs also every field and the per-spec witness lists; failures by (status, index).
Success cases also match the builder's ground truth. The same cases are pinned against both oracles on the CPU by test_storage_trees.py."""
import copy
import ctypes as C
import json
import random

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import bundle_json as J
from tests import storage_trees as T
from tests.util import assert_witness_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def slot_world(api, oracle_mod):
    blocks, cases = T.world_slots()
    f = T.Flat(blocks)
    return ({c.name: c for c in cases}, api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True),
            oracle_mod.Store(f.cids, f.offsets, f.lengths, f.blob))


@pytest.fixture(scope="module")
def proof_world(api, oracle_mod, ts3_small):
    w, f = T.world_proofs(ts3_small)
    return w, f, api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True), oracle_mod.Store(f.cids, f.offsets, f.lengths, f.blob)


def _outcome(fn):
    try:
        return fn(), None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _check_slots(gstore, ostore, root, slots, truth=None, name=""):
    """Engine == oracle (values, found flags, raw lengths, witness, or the same failure) and, on success, == truth. → failure or None."""
    exp, eerr = _outcome(lambda: ostore.read_storage_slots(root, slots))
    got, gerr = _outcome(lambda: gstore.read_storage_slots(root, slots))
    assert gerr == eerr, name
    if eerr:
        return eerr
    assert np.array_equal(got.found, exp.found) and np.array_equal(got.raw_len, exp.raw_len) and np.array_equal(got.values, exp.values), name
    assert_witness_equal(got.witness, exp.witness)
    if truth is not None:
        assert got.found.tolist() == [int(v is not None) for v in truth], name
        assert got.raw_len.tolist() == [len(v or b"") for v in truth], name
        assert [bytes(v) for v in got.values] == [T.left_pad_32(v or b"") for v in truth], name
    return None


@pytest.mark.parametrize("strict", [None, "1"])
def test_read_slots_every_width_and_shape(slot_world, monkeypatch, strict):
    """Every case of the catalogue: B1 / B2 at widths 1–8 over tries of 1, 3, 4, 200 and 5 000 entries, C, A1–A3, value and node
    shapes, wrapper bit widths, depth boundaries; with the fast node decoder and with IPCFP_HAMT_STRICT."""
    if strict is None:
        monkeypatch.delenv("IPCFP_HAMT_STRICT", raising=False)
    else:
        monkeypatch.setenv("IPCFP_HAMT_STRICT", strict)
    cases, gstore, ostore = slot_world
    n_fail = 0
    for c in cases.values():
        err = _check_slots(gstore, ostore, c.root_np(), c.slots_np(), c.truth, c.name)
        assert (err is None) == (c.status is None), c.name
        if err:
            assert err[0] == c.status, c.name
            n_fail += 1
    assert n_fail >= 20


@pytest.mark.parametrize("strict", [None, "1"])
@pytest.mark.parametrize("k", [1000, 16385])   # one lookup per warp up to 16 384, one per thread (strict decoder) above
@pytest.mark.parametrize("bw", [1, 3, 8])
def test_read_slots_lookup_counts(slot_world, monkeypatch, bw, k, strict):
    if strict is None:
        monkeypatch.delenv("IPCFP_HAMT_STRICT", raising=False)
    else:
        monkeypatch.setenv("IPCFP_HAMT_STRICT", strict)
    cases, gstore, ostore = slot_world
    c = cases[f"B{1 + k % 2}-w{bw}-n5000"]
    truth = T.width_trees()[1][(bw, 5000)][1]
    rng = random.Random(k * 10 + bw)
    keys = list(truth)
    slots = [rng.choice(keys) for _ in range(k - k // 10)] + [rng.randbytes(32) for _ in range(k // 10)]
    rng.shuffle(slots)
    want = [truth.get(s) for s in slots]
    assert _check_slots(gstore, ostore, c.root_np(), np.frombuffer(b"".join(slots), dtype=np.uint8).reshape(-1, 32), want, c.name) is None


def _check_proofs(gstore, ostore, ts, specs):
    """generate_storage_proofs: engine == oracle (every field, witness, per-spec witness lists) or the same failure."""
    exp, eerr = _outcome(lambda: ostore.generate_storage_proofs(ts, specs))
    got, gerr = _outcome(lambda: gstore.generate_storage_proofs(ts, specs))
    assert gerr == eerr
    if eerr:
        return None, eerr
    assert [vars(p) for p in got.proofs] == [vars(p) for p in exp.proofs]
    assert_witness_equal(got.witness, exp.witness)
    assert got.spec_witness == exp.spec_witness
    return got, None


def test_storage_proofs_full_state_trees(api, oracle_mod, proof_world):
    """Actor IDs 0, 1000, 2^63, 2^64 − 1 (11-byte keys), depth-limit chains of every width behind the proof path, the deepest path."""
    w, f, gstore, ostore = proof_world
    ok, _ = T.proof_batches(w)
    for tip, specs in ok:
        got, err = _check_proofs(gstore, ostore, w.tips[tip], specs)
        assert err is None, tip
        for (actor, slot), p in zip(specs, got.proofs):
            v = T.proof_truth(w, tip, actor, slot)
            assert (p.found, p.raw_len, bytes(p.value)) == (v is not None, len(v or b""), T.left_pad_32(v or b"")), (tip, actor)
        assert oracle_mod.verify_storage_proofs(got.witness, w.tips[tip], got) == api.verify_storage_proofs(got.witness, w.tips[tip], got)
    # header + StateRoot + 51 actors nodes + EVM state + B1 wrapper + 256 storage nodes, in one recorder
    got, _ = _check_proofs(gstore, ostore, w.tips["deep"], [(w.deep_actor, w.deep_slot)])
    assert len(got.spec_witness[0]) == 311 and got.proofs[0].found
    assert bytes(got.proofs[0].value) == w.deep_value[-32:]


def test_storage_proofs_depth_and_decode_failures(proof_world):
    """One more level than a width allows (actors chain of 52 at width 5, storage chains of ⌊256/bw⌋ + 1), a broken wrapper, an actor
    that is not there: the oracle's (status, index)."""
    w, f, gstore, ostore = proof_world
    _, bad = T.proof_batches(w)
    for tip, specs in bad:
        _, err = _check_proofs(gstore, ostore, w.tips[tip], specs)
        assert err is not None and err[1] == len(specs) - 1 and err[0] in (A.ERR_DECODE, A.ERR_ACTOR_NOT_FOUND), (tip, specs[-1][0])


def test_verify_storage_proofs_deepest(api, oracle_mod, proof_world):
    w, f, gstore, ostore = proof_world
    ok, _ = T.proof_batches(w)
    ts = w.tips["deep"]
    r = gstore.generate_storage_proofs(ts, ok[1][1])
    exp = oracle_mod.verify_storage_proofs(r.witness, ts, r)
    assert api.verify_storage_proofs(r.witness, ts, r) == exp and all(exp)
    sz = r.raw_proofs.size // len(r.proofs)
    for k in (0, 1, 2):                       # the deep value, an absent slot, a sibling's value: the last value byte flipped
        r2 = copy.copy(r)
        r2.raw_proofs = r.raw_proofs.copy()
        r2.raw_proofs[sz * k + 8 + 38 + 38 + 32 + 31] ^= 1
        exp2 = oracle_mod.verify_storage_proofs(r.witness, ts, r2)
        assert api.verify_storage_proofs(r.witness, ts, r2) == exp2
        assert not exp2[k] and sum(exp2) == len(exp2) - 1


def test_fault_ordering_across_one_launch(api, oracle_mod, proof_world):
    """A missing node at depth 1, a node mutated under its CID (same length), a chain past the depth limit and a broken wrapper, planted
    in specs of one ≥ 64-spec launch (one spec per warp, four per CTA) in several orders: the reported (status, index) is the oracle's,
    the first failing spec; the store keeps answering correctly afterwards."""
    w, f, _, _ = proof_world
    ok, _ = T.proof_batches(w)
    good = [s for s in ok[0][1] if s[0] not in (2001, 2002)]
    (k1, drop, _), (k2, mut, _) = w.faults[2001], w.faults[2002]
    arrays = f.dropped(drop)
    i = int(np.nonzero((arrays["cids"] == np.frombuffer(mut, dtype=np.uint8)).all(axis=1))[0][0])
    blob = arrays["blob"].copy()
    assert blob[int(arrays["offsets"][i])] == 0x82
    blob[int(arrays["offsets"][i])] = 0x83                      # [bitfield, pointers] → an array of 3: decode error, same length
    arrays["blob"] = blob
    ts = T.tipset(w.tips["main"], arrays, *w.heads["main"])
    gstore = api.BlockStore.from_tipset(ts)
    ostore = oracle_mod.Store.from_tipset(ts)
    faults = [(2001, k1), (2002, k2), (2003, w.chain[4]), (2004, good[0][1])]
    status = {2001: A.ERR_MISSING_BLOCK, 2002: A.ERR_DECODE, 2003: A.ERR_DECODE, 2004: A.ERR_DECODE}
    for seed in range(8):
        rng = random.Random(seed)
        specs = list(good)
        rng.shuffle(specs)
        specs = specs[:60]
        order = faults[seed % 4:] + faults[:seed % 4]
        if seed >= 4:
            order = [order[0]] + order[:0:-1]
        first = 5 + 7 * seed                                    # the first fault in CTA first // 4, the others in later CTAs
        for j, fs in enumerate(order):
            specs.insert(first + 5 * j * (1 + seed % 3), fs)
        assert len(specs) >= 64 and specs.index(order[0]) == first
        _, err = _check_proofs(gstore, ostore, ts, specs)
        assert err == (status[order[0][0]], first), seed
        got, err = _check_proofs(gstore, ostore, ts, good)
        assert err is None


# ------------------------------------------------------------------ the unified bundle of the deepest tree (as in test_zz_proof_bundle_resident)
def _plain(api, store, ts, sspecs):
    """ipcfp_generate_proof_bundle → (BundlePy, ipcfp_bundle_to_json of it)."""
    L = api.lib()
    sarr, ns, earr, ne = store._bundle_specs(sspecs, [])
    d, keep = A.make_tipset_desc(ts)
    out = C.POINTER(A.BundleC)()
    api._check(L.ipcfp_generate_proof_bundle(store._h, C.byref(d), sarr, ns, earr, ne, C.byref(out)))
    try:
        return A.bundle_from_c(out.contents), api.bundle_to_json(out, ts)
    finally:
        L.ipcfp_bundle_free(out)


def test_unified_bundle_of_the_deepest_tree(api, oracle_mod, proof_world):
    w, f, gstore, ostore = proof_world
    ok, _ = T.proof_batches(w)
    ts = w.tips["deep"]
    sspecs = ok[1][1]
    base, want = _plain(api, gstore, ts, sspecs)
    exp = ostore.generate_proof_bundle(ts, sspecs, [])
    assert [vars(p) for p in base.storage.proofs] == [vars(p) for p in exp.storage.proofs]
    assert base.storage.spec_witness == exp.storage.spec_witness
    assert_witness_equal(base.witness, exp.witness)
    assert want == J.dumps(J.unified_bundle(ts, base))
    tip = gstore.upload_tipset(ts)
    try:
        got = gstore.generate_proof_bundle_resident(tip, sspecs, [], A.RESULT_JSON)
    finally:
        tip.close()
    assert got.json == want
    assert [vars(p) for p in got.storage.proofs] == [vars(p) for p in base.storage.proofs]
    doc = json.loads(want)
    assert len(doc["storage_proofs"]) == len(sspecs) and len(doc["blocks"]) == base.witness.n_blocks > 311
    v = api.verify_bundle_json(want)
    assert v.storage_results == [True] * len(sspecs)
