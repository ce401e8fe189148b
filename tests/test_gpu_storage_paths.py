"""Storage paths on the GPU (ipcfp_generate_storage_path_proofs_resident, ipcfp_plan_fetch_storage_paths_resident,
ipcfp_verify_storage_paths) over one contract laid out by Solidity's rules in a hand-built state tree (tests/storage_paths.py):
  * specs, statuses, final slots, packed offsets and values equal the Python restatement, and the proofs the oracle's;
  * result.storage is, byte for byte, what ipcfp_generate_storage_proofs gives for the expanded specs (with and without
    IPCFP_WITNESS_BY_REFERENCE);
  * the expanded specs as ordinary storage specs of a log bundle give JSON that ipcfp_verify_bundle_json accepts;
  * the verifier accepts the real proofs and rejects a changed value, a left-out data slot and a lying length word;
  * the fetch loop from an empty store converges to the complete result, a long string taking more rounds;
  * missing blocks in wave 1 and in wave 2 fail at the first failing path; every refusal is IPCFP_ERR_INVALID_ARG;
  * batches at the caps: 65 536 paths, and long strings of IPCFP_PATH_MAX_BYTES."""
import ctypes as C
import random

import cbor2
import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200.api import StoragePath
from tests import storage_paths as SP
from tests import storage_trees as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def world(api, ts3_small):
    c = SP.Contract()
    flat, tip = c.world(ts3_small)
    store = api.BlockStore.from_tipset(tip, verify_cids=True)
    rt = store.upload_tipset(tip)
    yield c, flat, tip, store, rt
    rt.close()
    store.close()


def _check_against_restatement(c, paths, r):
    assert len(r.paths) == len(paths)
    k = 0
    for (name, p), got in zip(paths, r.paths):
        specs, status, value, slot, off = c.expected(p)
        assert (got.status, got.slot, got.byte_offset, got.valid) == (status, slot, off, True), name
        assert got.value == value, name
        assert (got.first_spec, got.n_specs) == (k, len(specs)), name
        assert r.specs[k:k + len(specs)] == specs, name
        k += len(specs)
    assert len(r.specs) == k


def _assert_storage_equal(a, b):
    assert np.array_equal(a.raw_proofs, b.raw_proofs)
    for f in ("cids", "offsets", "lengths", "blob"):
        assert np.array_equal(getattr(a.witness, f), getattr(b.witness, f)), f
    assert a.spec_witness == b.spec_witness


@pytest.mark.parametrize("flags", [0, A.WITNESS_BY_REFERENCE])
def test_paths_match_restatement_and_storage_proofs(api, oracle_mod, world, flags):
    c, flat, tip, store, rt = world
    paths = [p for _, p in c.paths]
    r = store.generate_storage_path_proofs_resident(rt, paths, flags)
    _check_against_restatement(c, c.paths, r)
    ref = store.generate_proof_bundle_resident(rt, r.specs, [], flags).storage
    _assert_storage_equal(r.storage, ref)
    if not flags:
        _assert_storage_equal(r.storage, store.generate_storage_proofs(tip, r.specs))
        exp = oracle_mod.Store(flat.cids, flat.offsets, flat.lengths, flat.blob).generate_storage_proofs(tip, r.specs)
        assert np.array_equal(r.storage.raw_proofs, exp.raw_proofs)
        assert np.array_equal(r.storage.witness.cids, exp.witness.cids)
    for (_, p), got in zip(c.paths, r.paths):   # every value word is the proof's value, as the restatement reads storage
        for (_, slot), q in zip(r.specs[got.first_spec:got.first_spec + got.n_specs], r.storage.proofs[got.first_spec:got.first_spec + got.n_specs]):
            assert q.slot == slot and q.value == c.read(slot)
    assert r.host_syncs == 4 and r.timings["total"] > 0


def test_expanded_specs_in_a_log_bundle_verify_as_json(api, world):
    c, flat, tip, store, rt = world
    r = store.generate_storage_path_proofs_resident(rt, [p for _, p in c.paths])
    b = store.generate_log_bundle_resident(rt, r.specs, [], A.RESULT_JSON)
    v = api.verify_bundle_json(b.json)
    assert len(v.storage_results) == len(r.specs) and all(v.storage_results)


def test_verifier_accepts_real_proofs_and_rejects_tampering(api, world):
    c, flat, tip, store, rt = world
    paths = [p for _, p in c.paths]
    r = store.generate_storage_path_proofs_resident(rt, paths)
    v = api.verify_storage_paths(r.storage.witness, tip, r.storage, paths)
    assert [x.valid for x in v.paths] == [True] * len(paths)
    assert [(x.status, x.value, x.slot) for x in v.paths] == [(x.status, x.value, x.slot) for x in r.paths]
    assert v.specs == r.specs and v.storage is None
    names = [n for n, _ in c.paths]
    i = names.index("texts[5]")      # 65 bytes: header + 3 data slots
    g = r.paths[i]
    proofs = list(r.storage.proofs)

    def verdict(ps):
        return [x.valid for x in api.verify_storage_paths(r.storage.witness, tip, ps, paths).paths]

    bad = list(proofs)   # a data slot that claims another value
    q = bad[g.first_spec + 2]
    bad[g.first_spec + 2] = A.StorageProofPy(q.actor_id, q.actor_state_cid, q.storage_root, q.slot, bytes([q.value[0] ^ 1]) + q.value[1:], q.found, q.raw_len)
    assert verdict(bad) == [k != i for k in range(len(paths))]
    left_out = proofs[:g.first_spec + 1] + proofs[g.first_spec + 2:]   # a data slot left out
    assert verdict(left_out) == [k != i for k in range(len(paths))]
    lie = list(proofs)    # a header word that claims a shorter string: its proof no longer verifies
    q = lie[g.first_spec]
    lie[g.first_spec] = A.StorageProofPy(q.actor_id, q.actor_state_cid, q.storage_root, q.slot, SP.b32(2 * 40 + 1), q.found, q.raw_len)
    assert verdict(lie)[i] is False
    j = names.index("nums[4]")       # an array length word that lies (every copy of it: the nums paths share it)
    key = r.specs[r.paths[j].first_spec]
    lie = [A.StorageProofPy(q.actor_id, q.actor_state_cid, q.storage_root, q.slot, SP.b32(3), q.found, q.raw_len) if (q.actor_id, q.slot) == key else q
           for q in proofs]
    assert verdict(lie)[j] is False


def _rounds(api, flat, tip, paths):
    full = {bytes(flat.cids[i]): bytes(flat.blob[int(flat.offsets[i]):int(flat.offsets[i]) + int(flat.lengths[i])]) for i in range(flat.n_blocks)}

    def fetch(cids, first_id):
        import base64
        els = [b'{"jsonrpc":"2.0","result":"' + base64.b64encode(full[bytes(x)]) + b'","id":' + str(first_id + k).encode() + b"}"
               for k, x in enumerate(cids)]
        return b"[" + b",".join(els) + b"]"

    store, rt, rounds, cids, _ = api.fetch_storage_paths_until_complete(fetch, lambda s: s.upload_tipset(tip), paths)
    return store, rt, rounds


def test_fetch_loop_converges_to_the_complete_result(api, world):
    c, flat, tip, full_store, full_rt = world
    by = dict(c.paths)
    short = [by["subnet0.stake"], by["texts[1]"], by["nums[4]"]]
    long_ = short + [by["texts[4]"]]
    counts = []
    for paths in (short, long_):
        store, rt, rounds = _rounds(api, flat, tip, paths)
        got = store.generate_storage_path_proofs_resident(rt, paths)
        want = full_store.generate_storage_path_proofs_resident(full_rt, paths)
        assert [(x.status, x.value) for x in got.paths] == [(x.status, x.value) for x in want.paths] and got.specs == want.specs
        assert np.array_equal(got.storage.raw_proofs, want.storage.raw_proofs)
        counts.append(len(rounds))
        rt.close()
        store.close()
    assert counts[1] == counts[0] + 1   # the data slots are known once the header word is: one round more


def _hamt_path(blocks, root, key, bw):
    """CIDs of the HAMT nodes Hamt::get(key) visits from root"""
    out, node, level = [root], cbor2.loads(blocks[root]), 0
    while True:
        i = T.hash_index(key, level, bw)
        bf = int.from_bytes(node[0], "big")
        if not (bf >> i) & 1:
            return out
        p = node[1][bin(bf & ((1 << i) - 1)).count("1")]
        if not isinstance(p, cbor2.CBORTag):
            return out
        cid = bytes(p.value[1:])
        out.append(cid)
        node, level = cbor2.loads(blocks[cid]), level + 1


def test_missing_blocks_fail_at_the_first_failing_path(api, world, ts3_small):
    c, flat, tip, store, rt = world
    paths = [p for _, p in c.paths]
    r = store.generate_storage_path_proofs_resident(rt, paths)
    wrapper = cbor2.loads(flat.blocks[bytes(r.storage.proofs[0].storage_root)])
    root = bytes(wrapper[0].value[1:])
    node_paths = {s: _hamt_path(flat.blocks, root, s, 5) for _, s in r.specs}
    fixed_n = [len(SP.derive(p)[0]) + len(SP.derive(p)[1]) for p in paths]
    def first_failure(node):
        for i, g in enumerate(r.paths):
            for k in range(g.n_specs):
                if node in node_paths[r.specs[g.first_spec + k][1]]:
                    return i, k >= fixed_n[i]
        return None

    cands = {n: first_failure(n) for v in node_paths.values() for n in v[1:]}
    wave2 = [n for n, f in sorted(cands.items()) if f and f[1]][:4]
    wave1 = [n for n, f in sorted(cands.items()) if f and not f[1]][:4]
    assert wave1 and wave2, "a fault in wave 1 and one in wave 2"
    for node in wave1 + wave2:
        t2 = T.tipset(ts3_small, flat.dropped(node), bytes(tip.child_cid), bytes(tip.parent_state_root))
        s2 = api.BlockStore.from_tipset(t2)
        rt2 = s2.upload_tipset(t2)
        with pytest.raises(A.IpcfpError) as e:
            s2.generate_storage_path_proofs_resident(rt2, paths)
        assert (e.value.status, e.value.index) == (A.ERR_MISSING_BLOCK, cands[node][0])
        rt2.close()
        s2.close()


EMPTY = A.WitnessPy(np.zeros((0, 38), np.uint8), np.zeros(0, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.uint8))


def test_refusals(api, world):
    c, flat, tip, store, rt = world
    P = StoragePath(SP.ACTOR, 0)
    bad = [P._with((7, b"", 0, 0, 0)), StoragePath(SP.ACTOR, 0, kind=5), P.array(0, 1, 33), P.array(0, 0, 0), P.static(0, 0, 0), P.words(0),
           P.words(A.PATH_MAX_WORDS + 1), P.mapping(b"x" * (A.PATH_MAX_KEY + 1), "bytes"), StoragePath(SP.ACTOR, 0, [(A.PATH_FIELD, b"", 1, 0, 0)] * 33)]
    for p in bad:
        for call in (lambda: store.generate_storage_path_proofs_resident(rt, [P, p]), lambda: store.plan_fetch_storage_paths(rt, [P, p]),
                     lambda: api.verify_storage_paths(EMPTY, tip, [], [P, p])):
            with pytest.raises(A.IpcfpError) as e:
                call()
            assert e.value.status == A.ERR_INVALID_ARG
    # the limits themselves are accepted
    ok = [P.mapping(b"x" * A.PATH_MAX_KEY, "bytes"), P.words(A.PATH_MAX_WORDS), StoragePath(SP.ACTOR, 0, [(A.PATH_FIELD, b"", 1, 0, 0)] * 32)]
    store.generate_storage_path_proofs_resident(rt, ok)
    with pytest.raises(A.IpcfpError) as e:
        store.generate_storage_path_proofs_resident(rt, [P], A.RESULT_JSON)
    assert e.value.status == A.ERR_INVALID_ARG
    with pytest.raises(A.IpcfpError) as e:
        store.plan_fetch_storage_paths(rt, [P], A.WITNESS_BY_REFERENCE)
    assert e.value.status == A.ERR_INVALID_ARG
    with pytest.raises(A.IpcfpError) as e:
        store.generate_storage_path_proofs_resident(rt, [P] * (A.PATH_MAX_PATHS + 1))
    assert e.value.status == A.ERR_INVALID_ARG
    L = api.lib()
    out = C.POINTER(A.PathResultC)()
    assert L.ipcfp_generate_storage_path_proofs_resident(store._h, rt._h, None, 1, 0, C.byref(out)) == A.ERR_INVALID_ARG
    steps_null = A.StoragePathC()
    steps_null.n_steps, steps_null.kind, steps_null.n_words = 1, A.PATH_WORDS, 1
    assert L.ipcfp_generate_storage_path_proofs_resident(store._h, rt._h, C.byref(steps_null), 1, 0, C.byref(out)) == A.ERR_INVALID_ARG


def test_batches_at_the_caps(api, world):
    c, flat, tip, store, rt = world
    rng = random.Random(9)
    P = StoragePath(SP.ACTOR, 1)
    keys = [0, 1, 2 ** 200, 5]
    paths = [P.mapping(c.owners[rng.randrange(3)], "address").mapping(rng.choice(keys), "uint256") for _ in range(A.PATH_MAX_PATHS)]
    r = store.generate_storage_path_proofs_resident(rt, paths)
    assert len(r.paths) == A.PATH_MAX_PATHS and len(r.specs) == A.PATH_MAX_PATHS
    for p, g in zip(paths[::97], r.paths[::97]):
        specs, status, value, slot, _ = c.expected(p)
        assert (g.status, g.value, g.slot) == (status, value, slot)
    assert [x[1] for x in r.specs[:50]] == [SP.derive(p)[2] for p in paths[:50]]
    i = SP.STRING_LENGTHS.index(A.PATH_MAX_BYTES)
    longs = [StoragePath(SP.ACTOR, 12).mapping(i, "uint256").bytes()] * 64
    r = store.generate_storage_path_proofs_resident(rt, longs)
    assert all(g.status == A.PATH_OK and g.value == c.texts[i] and g.n_specs == 1 + A.PATH_MAX_BYTES // 32 for g in r.paths)
    _assert_storage_equal(r.storage, store.generate_storage_proofs(tip, r.specs))
