"""Storage paths on the GPU over the multi-actor campaign tree (tests/storage_path_worlds.py): ipcfp_generate_storage_path_proofs_resident
on the seeded campaign and at the kernels' launch edges, its failure ordering on trees with two faults in one path,
ipcfp_verify_storage_paths against hostile proof lists, and the fetch loop from an empty store.

Every batch is checked three ways: each path's status, slot, byte offset, first_spec, n_specs, value and specs equal
storage_paths.expand over its actor's dict; result.storage is byte for byte ipcfp_generate_storage_proofs of result.specs (by value) and
the resident bundle's storage (IPCFP_WITNESS_BY_REFERENCE); the raw proofs equal the C++ oracle's."""
import random
import types

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200.api import StoragePath
from tests import storage_path_worlds as W
from tests import storage_paths as SP
from tests import storage_trees as T

pytestmark = pytest.mark.gpu
ROW = 160    # sizeof(ipcfp_storage_proof)


class _Ctx:
    def __init__(self, api, oracle_mod, ts):
        self.w = W.build()
        self.flat, self.tip = self.w.tip(ts)
        self.store = api.BlockStore.from_tipset(self.tip, verify_cids=True)
        self.rt = self.store.upload_tipset(self.tip)
        self.ostore = oracle_mod.Store(self.flat.cids, self.flat.offsets, self.flat.lengths, self.flat.blob)
        self.rows, self._exp = {}, {}

    def expected(self, p):
        """w.expected(p), cached by the path's value (an object's id can be reused once it is freed)"""
        key = (p.actor_id, p.base_slot, p.steps, p.kind, p.n_words)
        e = self._exp.get(key)
        if e is None:
            e = self._exp[key] = self.w.expected(p)
        return e

    def oracle_rows(self, specs):
        """the C++ oracle's raw proof of every spec, (n, 160) uint8"""
        todo = list(dict.fromkeys(s for s in specs if s not in self.rows))
        if todo:
            raw = self.ostore.generate_storage_proofs(self.tip, todo).raw_proofs.reshape(-1, ROW)
            self.rows.update(zip(todo, raw))
        return np.stack([self.rows[s] for s in specs]) if specs else np.zeros((0, ROW), np.uint8)


@pytest.fixture(scope="module")
def ctx(api, oracle_mod, ts3_small):
    c = _Ctx(api, oracle_mod, ts3_small)
    yield c
    c.rt.close()
    c.store.close()


def _assert_storage_equal(a, b):
    assert np.array_equal(a.raw_proofs, b.raw_proofs)
    for f in ("cids", "offsets", "lengths", "blob"):
        assert np.array_equal(getattr(a.witness, f), getattr(b.witness, f)), f
    assert a.spec_witness == b.spec_witness


def _run(ctx, paths):
    """the batch through the generator, checked three ways → its result"""
    r = ctx.store.generate_storage_path_proofs_resident(ctx.rt, paths)
    assert len(r.paths) == len(paths)
    k = 0
    for i, (p, got) in enumerate(zip(paths, r.paths)):
        specs, status, value, slot, off = ctx.expected(p)
        assert (got.status, got.slot, got.byte_offset, got.valid, got.first_spec, got.n_specs) == (status, slot, off, True, k, len(specs)), i
        assert got.value == value, i
        assert r.specs[k:k + len(specs)] == specs, i
        k += len(specs)
    assert len(r.specs) == k
    _assert_storage_equal(r.storage, ctx.store.generate_storage_proofs(ctx.tip, r.specs))
    rb = ctx.store.generate_storage_path_proofs_resident(ctx.rt, paths, A.WITNESS_BY_REFERENCE)
    assert rb.paths == r.paths and rb.specs == r.specs
    ref = ctx.store.generate_proof_bundle_resident(ctx.rt, r.specs, [], A.WITNESS_BY_REFERENCE).storage
    if r.specs:
        _assert_storage_equal(rb.storage, ref)
    else:    # a bundle without storage specs has no storage result
        assert ref is None and rb.storage.raw_proofs.size == 0 and rb.storage.witness.n_blocks == 0 and rb.storage.spec_witness == []
    assert np.array_equal(r.storage.raw_proofs.reshape(-1, ROW), ctx.oracle_rows(r.specs))
    return r


def test_whole_campaign_in_seed_order_and_shuffled(ctx):
    w = ctx.w
    r = _run(ctx, w.campaign)
    assert {g.status for g in r.paths} == {A.PATH_OK, A.PATH_INDEX_OUT_OF_RANGE, A.PATH_BAD_BYTES, A.PATH_TOO_LONG}
    exp = ctx.ostore.generate_storage_proofs(ctx.tip, r.specs)
    assert np.array_equal(r.storage.witness.cids, exp.witness.cids) and r.storage.spec_witness == exp.spec_witness
    shuffled = list(w.campaign)
    random.Random(3).shuffle(shuffled)
    _run(ctx, shuffled)


def test_edges_and_the_largest_path(ctx):
    r = _run(ctx, ctx.w.edges)
    assert {g.status for g in r.paths} == {A.PATH_OK, A.PATH_INDEX_OUT_OF_RANGE, A.PATH_BAD_BYTES, A.PATH_TOO_LONG}
    r = _run(ctx, [W.deep_path()])
    assert (r.paths[0].status, r.paths[0].n_specs) == (A.PATH_OK, A.PATH_MAX_STEPS + A.PATH_MAX_WORDS)
    _run(ctx, [W.deep_path(), ctx.w.hand["s100"], W.deep_path()])


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 127, 128, 129, 4097])
def test_path_counts(ctx, n):
    _run(ctx, random.Random(n).choices(ctx.w.campaign, k=n))


def _n_fixed(p):
    lengths, values, _, _ = SP.derive(p)
    return len(lengths) + len(values)


@pytest.mark.parametrize("residue", [0, 1, 3])
def test_fixed_spec_totals_mod_4(ctx, residue):
    """k_path_proofs and k_path_place run four warps per block: the last block full, with one warp, with three"""
    paths = list(ctx.w.campaign[:50])
    while sum(map(_n_fixed, paths)) % 4 != residue:
        paths.append(ctx.w.hand["pair.y"])
    r = _run(ctx, paths)
    assert sum(map(_n_fixed, paths)) % 4 == residue and len(r.specs) >= sum(map(_n_fixed, paths))


def test_all_words_batch(ctx):
    """wave 2 launches over the final list and skips every spec"""
    paths = [p for p in ctx.w.campaign if p.kind == A.PATH_WORDS]
    r = _run(ctx, paths)
    assert len(r.specs) == sum(map(_n_fixed, paths))


def test_all_empty_string_batch(ctx):
    """every value empty: value_blob_size 0"""
    paths = [StoragePath(a, 7919 * i + 100003).bytes() for a in W.ACTORS + (W.SHARER, W.EDGE, W.HAND) for i in range(6)]
    paths += [ctx.w.edges[-12]] * 3
    r = _run(ctx, paths)
    assert all(g.status == A.PATH_OK and g.value == b"" for g in r.paths) and len(r.specs) == len(paths)


def test_all_too_long_batch(ctx):
    paths = [p for p in ctx.w.campaign + ctx.w.edges if ctx.expected(p)[1] == A.PATH_TOO_LONG]
    assert len(paths) > 40
    r = _run(ctx, paths)
    assert all(g.status == A.PATH_TOO_LONG for g in r.paths) and len(r.specs) == sum(map(_n_fixed, paths))


def test_65537_specs_across_mixed_kinds(ctx):
    rng = random.Random(65537)
    paths, total = [], 0
    while True:
        p = rng.choice(ctx.w.campaign)
        n = len(ctx.expected(p)[0])
        if total + n > 65537:
            break
        paths.append(p)
        total += n
    paths += [ctx.w.hand["pair.y"]] * (65537 - total)
    r = _run(ctx, paths)
    assert len(r.specs) == 65537 and {p.kind for p in paths} == {A.PATH_WORDS, A.PATH_BYTES}


def test_max_paths_drawn_from_the_campaign(ctx):
    paths = random.Random(A.PATH_MAX_PATHS).choices(ctx.w.campaign, k=A.PATH_MAX_PATHS)
    r = _run(ctx, paths)
    assert len(r.paths) == A.PATH_MAX_PATHS


# ------------------------------------------------------------------ failures
def _fault_call(api, ctx, ts, f, batch):
    arrays = f.arrays(ctx.flat)
    t2 = T.tipset(ts, arrays, bytes(ctx.tip.child_cid), bytes(ctx.tip.parent_state_root))
    s2 = api.BlockStore.from_tipset(t2)
    rt2 = s2.upload_tipset(t2)
    try:
        with pytest.raises(A.IpcfpError) as e:
            s2.generate_storage_path_proofs_resident(rt2, batch)
        return (e.value.status, e.value.index), t2, arrays
    finally:
        rt2.close()
        s2.close()


@pytest.mark.parametrize("name", W.FAULT_NAMES)
def test_two_faults_in_one_path(api, oracle_mod, ctx, ts3_small, name):
    f = next(f for f in W.faults() if f.name == name)
    batch = W.fault_batch(f.path)
    got, t2, arrays = _fault_call(api, ctx, ts3_small, f, batch)
    ostore = oracle_mod.Store(arrays["cids"], arrays["offsets"], arrays["lengths"], arrays["blob"])
    want = W.first_failure(W.oracle_outcomes(ostore, t2, batch))
    assert got == want == ((A.ERR_MISSING_BLOCK if f.first == "missing" else A.ERR_DECODE), 2), f.name


@pytest.mark.parametrize("name", W.ABSENT_NAMES)
def test_absent_actor_and_a_wave2_missing_block(api, oracle_mod, ctx, ts3_small, name):
    batch, f = next((b, f) for n, b, f in W.absent_batches() if n == name)
    got, t2, arrays = _fault_call(api, ctx, ts3_small, f, batch)
    ostore = oracle_mod.Store(arrays["cids"], arrays["offsets"], arrays["lengths"], arrays["blob"])
    assert got == W.first_failure(W.oracle_outcomes(ostore, t2, batch)), name


# ------------------------------------------------------------------ the verifier
@pytest.fixture(scope="module")
def verifier_cases(oracle_mod, ts3_small):
    return W.verifier_inputs(oracle_mod, ts3_small)


def _packed(proofs):
    return types.SimpleNamespace(proofs=proofs, raw_proofs=A.pack_storage_proofs(proofs))


@pytest.mark.parametrize("name", W.HOSTILE_NAMES)
def test_verifier_on_hostile_lists(api, oracle_mod, verifier_cases, name):
    paths, witness, tip, lists = verifier_cases
    proofs = lists[name]
    verdicts = oracle_mod.verify_storage_proofs(witness, tip, _packed(proofs))
    assert api.verify_storage_proofs(witness, tip, _packed(proofs)) == verdicts
    want = W.expected_verdicts(paths, proofs, verdicts)
    v = api.verify_storage_paths(witness, tip, proofs, paths)
    assert v.storage is None
    k = 0
    for i, (g, (valid, status, value, specs)) in enumerate(zip(v.paths, want)):
        assert (g.valid, g.status, g.first_spec, g.n_specs) == (valid, status, k, len(specs)), (name, i)
        assert g.value == value, (name, i)
        assert v.specs[k:k + len(specs)] == specs, (name, i)
        k += len(specs)
    assert len(v.paths) == len(paths) and len(v.specs) == k
    if name == "empty":
        assert not any(g.valid for g in v.paths) and [g.n_specs for g in v.paths] == [_n_fixed(p) for p in paths]


# ------------------------------------------------------------------ the planner
def test_fetch_loop_converges_on_the_campaign(api, ctx, ts3_small):
    import base64
    full = ctx.flat.blocks

    def fetch(cids, first_id):
        els = [b'{"jsonrpc":"2.0","result":"' + base64.b64encode(full[bytes(x)]) + b'","id":' + str(first_id + k).encode() + b"}"
               for k, x in enumerate(cids)]
        return b"[" + b",".join(els) + b"]"

    paths = ctx.w.campaign
    store, rt, rounds, cids, _ = api.fetch_storage_paths_until_complete(fetch, lambda s: s.upload_tipset(ctx.tip), paths)
    try:
        got = store.generate_storage_path_proofs_resident(rt, paths)
        want = ctx.store.generate_storage_path_proofs_resident(ctx.rt, paths)
        assert got.paths == want.paths and got.specs == want.specs
        _assert_storage_equal(got.storage, want.storage)
        fetched = {bytes(c) for c in cids}
        assert len(fetched) == len(cids)                           # no block fetched twice
        assert fetched == {bytes(c) for c in want.storage.witness.cids}
        assert len(rounds) >= 2
    finally:
        rt.close()
        store.close()
