"""ipcfp_resolve_addresses on the GPU (include/ipcfp.h, DESIGN.md §2 "Address resolution") on the hand-built state trees of
tests/address_trees.py, against the C++ oracle (tests/oracle_resolve.cpp, on oracle/oracle.cpp's decoders and HAMT walk) and against the
Python restatement of tests/address_trees.py: actor IDs, per-address status, the Init path's status, the missing CIDs and the witness,
with the fast HAMT node decoder and with IPCFP_HAMT_STRICT=1. Success cases also match the builder's
ground truth. Also: batches of 0 to 65 536 addresses, every block of a path dropped in turn, truncated and bit-flipped blocks, the fetch
loop from an empty store, and the config-3 tipset end to end (Ethereum address → actor ID → storage proofs → bundle verification)."""
import random

import cbor2
import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import address_trees as T
from tests import oracle_resolve as O
from tests import rpc_blocks as B
from tests import storage_trees as S

pytestmark = pytest.mark.gpu

MODES = [None, "1"]


@pytest.fixture(params=MODES, ids=["fast", "strict"])
def mode(request, monkeypatch):
    if request.param:
        monkeypatch.setenv("IPCFP_HAMT_STRICT", request.param)
    else:
        monkeypatch.delenv("IPCFP_HAMT_STRICT", raising=False)
    return request.param


@pytest.fixture(scope="module")
def world(api):
    blocks, cases, maps = T.world()
    f = S.Flat(blocks)
    return (blocks, {c.name: c for c in cases}, maps, api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True),
            O.Oracle(blocks))


def _check(store, oracle, blocks, root, addrs, truth=None, name=""):
    """The call == the C++ oracle == the restatement, field by field, and == truth where the builder put the address. → the result."""
    got = store.resolve_addresses(root, addrs)
    ids, status, init, missing, read = oracle.resolve(root, addrs)
    assert (ids, status, init, missing, read) == T.resolve(blocks, root, addrs), name
    assert got.init_status == init, name
    assert got.status.tolist() == status, name
    assert got.actor_ids.tolist() == ids, name
    assert [bytes(c) for c in got.missing] == missing, name
    assert [bytes(c) for c in got.witness.cids] == read, name
    assert got.witness.blocks() == [blocks[c] for c in read], name
    if truth:
        for a, i, s in zip(addrs, got.actor_ids.tolist(), got.status.tolist()):
            if a in truth:
                assert (s, i) == (A.OK, truth[a]), name
    return got


@pytest.mark.parametrize("name", [c.name for c in T.world()[1]])
def test_catalogue(world, mode, name):
    blocks, cases, _, store, oracle = world
    c = cases[name]
    _check(store, oracle, blocks, c.root, c.addrs, c.truth, name)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 16384, 65536])
def test_batches_with_duplicates(world, mode, n):
    blocks, _, maps, store, oracle = world
    root, ent = maps[100000]
    rng = random.Random(n)
    keys = list(ent)
    addrs = [rng.choice(keys) for _ in range(n * 3 // 4)]
    addrs += [T.random_address(rng, T.KINDS[i % 5]) for i in range(n // 8)]
    addrs += [T.id_addr(rng.randrange(2 ** 64)) for _ in range(n - len(addrs))]
    rng.shuffle(addrs)
    got = _check(store, oracle, blocks, root, addrs, ent, f"batch-{n}")
    assert (got.status == A.OK).sum() >= n * 3 // 4


def test_masked_id_eth_addresses_read_nothing(api, world):
    blocks, cases, _, store, _ = world
    c = cases["map-3"]
    addrs = [api.address_from_eth(T.eth_masked_id(v)) for v in T.VALUES]
    got = store.resolve_addresses(c.root, addrs)
    assert got.status.tolist() == [A.OK] * len(addrs) and got.actor_ids.tolist() == list(T.VALUES)
    # the witness is the Init path's alone, which every call walks once
    alone = store.resolve_addresses(c.root, [])
    assert [bytes(x) for x in got.witness.cids] == [bytes(x) for x in alone.witness.cids] == T.resolve(blocks, c.root, [])[4]


def _sub_store(api, blocks, drop=None, replace=None):
    part = S.Blocks({k: v for k, v in blocks.items() if k != drop})
    for k, v in (replace or {}).items():
        part[k] = v
    f = S.Flat(part)
    return part, api.BlockStore(f.cids, f.offsets, f.lengths, f.blob), O.Oracle(part)


@pytest.mark.parametrize("name", ["map-200", "chain-51", "bucket-3"])
def test_every_path_block_dropped_in_turn(api, world, mode, name):
    blocks, cases, _, _, _ = world
    c = cases[name]
    read = T.resolve(blocks, c.root, c.addrs)[4]
    for cid in read:
        part, store, oracle = _sub_store(api, blocks, drop=cid)
        try:
            got = _check(store, oracle, part, c.root, c.addrs, name=f"{name} without {cid.hex()}")
            assert [bytes(x) for x in got.missing] == [cid]
        finally:
            store.close()


def test_truncated_and_bit_flipped_blocks(api, world, mode):
    blocks, cases, _, _, _ = world
    c = cases["map-200"]
    for name, repl in T.mutations(blocks, c.root, random.Random(9), 48):
        part, store, oracle = _sub_store(api, blocks, replace=repl)
        try:
            _check(store, oracle, part, c.root, c.addrs, name=name)
        finally:
            store.close()


def test_invalid_state_root_length_is_refused(world):
    store = world[3]
    with pytest.raises(ValueError):
        store.resolve_addresses(b"\x01" * 37, [])


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


@pytest.mark.parametrize("name", ["map-5000", "chain-51", "init-trailing", "value-bytes", "ids-and-invalid"])
def test_fetch_loop_fetches_exactly_the_read_set(api, world, name):
    blocks, cases, _, store, oracle = world
    c = cases[name]
    full = store.resolve_addresses(c.root, c.addrs)
    assert [bytes(x) for x in full.witness.cids] == oracle.resolve(c.root, c.addrs)[4]
    held = {}
    st, got, rounds, cids, texts = api.resolve_until_complete(_fetcher(blocks, held), c.root, c.addrs)
    try:
        assert got.status.tolist() == full.status.tolist() and got.actor_ids.tolist() == full.actor_ids.tolist()
        assert got.init_status == full.init_status
        assert set(held) == {bytes(x) for x in full.witness.cids}
        assert [bytes(x) for x in got.witness.cids] == [bytes(x) for x in full.witness.cids]
        assert len(rounds) >= 1
        # resuming from the blocks already held: nothing more to fetch
        st2, again, rounds2, _, _ = api.resolve_until_complete(_fetcher(blocks, {}), c.root, c.addrs, cids=cids, texts=texts)
        st2.close()
        assert rounds2 == [] and again.status.tolist() == full.status.tolist()
    finally:
        st.close()


# ------------------------------------------------------------------ config 3 end to end
def _actor_entries(blocks, root):
    """{key: encoded value} of every entry of a HAMT (any layout synth writes)."""
    out = {}
    node = cbor2.loads(blocks[root])
    for p in node[1]:
        if isinstance(p, cbor2.CBORTag):
            out.update(_actor_entries(blocks, bytes(p.value[1:])))
        else:
            for k, v in p:
                out[bytes(k)] = cbor2.dumps(v)
    return out


def test_config3_eth_address_to_storage_proof(api, ts3_small):
    ts = ts3_small
    cids, raw = B.blocks_of(ts)
    blocks = S.Blocks({bytes(c): b for c, b in zip(cids, raw)})
    old_root = bytes(ts.parent_state_root)
    sr = cbor2.loads(blocks[old_root])
    actors = _actor_entries(blocks, bytes(sr[1].value[1:]))
    contract = 1001
    eth = bytes(range(0xa0, 0xb4))
    amap = S.build_hamt(blocks, {T.delegated(10, eth): S.head(0, contract), T.delegated(10, bytes(20)): S.head(0, 1003)}, 5)
    actors[S.id_address(1)] = S.actor_state(blocks.put(T.init_state(amap)))
    new_root = blocks.put(b"\x83" + S.head(0, sr[0]) + S.clink(S.build_hamt(blocks, actors, 5)) + S.clink(bytes(sr[2].value[1:])))
    hdr, child = S.child_header(ts, new_root)
    blocks[child] = hdr
    f = S.Flat(blocks)
    tip_ts = S.tipset(ts, f.arrays(), child, new_root)
    store = api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True)
    try:
        aid = api.resolve_eth_address_to_actor_id(store, new_root, "0x" + eth.hex())
        assert aid == contract
        with pytest.raises(A.IpcfpError) as e:
            api.resolve_eth_address_to_actor_id(store, new_root, "0x" + bytes(range(20)).hex())
        assert e.value.status == A.ERR_ACTOR_NOT_FOUND
        keys = [ts.storage_entry(k)[0] for k in (0, 1, 77)] + [ts.storage_absent_key(1)]
        slots = [bytes(s) for s in api.compute_mapping_slots(keys, [0] * len(keys))]
        got = store.generate_storage_proofs(tip_ts, [(aid, s) for s in slots])
        want = store.generate_storage_proofs(tip_ts, [(contract, s) for s in slots])
        assert [vars(p) for p in got.proofs] == [vars(p) for p in want.proofs]
        assert np.array_equal(got.witness.cids, want.witness.cids)
        tip = store.upload_tipset(tip_ts)
        try:
            bundle = store.generate_proof_bundle_resident(tip, [(aid, s) for s in slots], [], A.RESULT_JSON)
        finally:
            tip.close()
        v = api.verify_bundle_json(bundle.json)
        assert v.storage_results == [True] * len(slots)
    finally:
        store.close()
