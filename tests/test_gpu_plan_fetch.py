"""ipcfp_plan_fetch_resident (include/ipcfp.h, DESIGN.md §2 "Fetch planning") on the GPU. Every round's plan must be N(S) \\ S as the
restatement below computes it from the blocks held so far (cbor2 and the Python oracle's decoders, independent of the library); the loop
from an empty store must request every block the Python oracle reads while generating on the full store, each exactly once, and the
bundle generated on the planned store must be byte-equal to the bundle of the full store. The fetcher answers from the synthetic block
map through tests/rpc_blocks.py's canonical rendering."""
import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from oracle import pyoracle as P
from tests import rpc_blocks as B
from tests.plan_rules import restate_plan
from tests.util import spec_of

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------ fixtures
class _LoggedStore(dict):
    """The oracle's dict store, logging every CID it is asked about."""

    def __init__(self, *a):
        super().__init__(*a)
        self.read = set()

    def get(self, c, d=None):
        self.read.add(bytes(c))
        return super().get(c, d)

    def __contains__(self, c):
        self.read.add(bytes(c))
        return super().__contains__(c)

    def __getitem__(self, c):
        self.read.add(bytes(c))
        return super().__getitem__(c)


def _especs(ts):
    return [(ts.event_signature, ts.topic1, None if ts.actor_filter is None or ts.actor_filter < 0 else int(ts.actor_filter))]


def _oracle_reads(full, ts, sspecs, especs):
    st = _LoggedStore(full)
    for sig, t1, actor in especs:
        P.generate_event_proof(st, ts, sig, t1, actor)
    for actor_id, slot in sspecs:
        P.generate_storage_proof(st, ts, actor_id, bytes(slot))
    return st.read


def _sspecs(api, ts):
    keys = [ts.storage_entry(k)[0] for k in (0, 1, 77)] + [ts.storage_absent_key(1)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    return [(a, bytes(s)) for a in (1001, 1003, 1006) for s in slots]


def _run_loop(api, ts, full, sspecs, especs_c, especs_py):
    """The planning loop from an empty store, each round checked against the restatement; returns (store, tipset, rounds)."""
    held = {}

    def fetch(cids, first_id):
        els = []
        for k, c in enumerate(cids):
            c = bytes(c)
            assert c not in held, "a CID was requested twice"
            held[c] = full[c]
            els.append(B.element(first_id + k, full[c]))
        return B.render([], elements=els)

    expected_rounds = []
    probe = {}
    while True:
        exp, _ = restate_plan(probe, ts, sspecs, especs_py)
        expected_rounds.append(exp)
        if not exp:
            break
        probe.update({c: full[c] for c in exp})
    store, tip, rounds, cids, _ = api.fetch_until_complete(fetch, lambda s: s.upload_tipset(ts),
                                                          sspecs, especs_c)
    assert len(rounds) == len(expected_rounds) - 1
    for r, exp in zip(rounds, expected_rounds):
        assert [bytes(c) for c in r.cids] == exp
    return store, tip, rounds


def _check_loop(api, ts, sspecs, especs_c, especs_py):
    cids, blocks = B.blocks_of(ts)
    full = {bytes(c): b for c, b in zip(cids, blocks)}
    store, tip, rounds = _run_loop(api, ts, full, sspecs, especs_c, especs_py)
    union = {bytes(c) for r in rounds for c in r.cids}
    assert union == _oracle_reads(full, ts, sspecs, especs_py)
    ref = api.BlockStore.from_tipset(ts)
    rtip = ref.upload_tipset(ts)
    a = store.generate_proof_bundle_resident(tip, sspecs, especs_c, A.RESULT_JSON)
    b = ref.generate_proof_bundle_resident(rtip, sspecs, especs_c, A.RESULT_JSON)
    assert a.json == b.json
    plan = ref.plan_fetch(rtip, sspecs, especs_c)
    assert len(plan.cids) == 0 and plan.n_needed == len(union)
    return rounds


# ------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("config", [1, 2, 3])
def test_loop_from_an_empty_store_matches_the_restatement(api, synth_mod, ts3_small, config):
    ts = ts3_small if config == 3 else synth_mod.Tipset(synth_mod.config_params(config))
    rounds = _check_loop(api, ts, [], [spec_of(ts)], _especs(ts))
    assert len(rounds) >= 2


def test_unified_bundle_loop(api, ts3_small):
    ts = ts3_small
    _check_loop(api, ts, _sspecs(api, ts), [spec_of(ts)], _especs(ts))


def test_no_specs_and_full_store_plan_nothing(api, ts1):
    empty = api.BlockStore(np.zeros((0, 38), np.uint8), np.zeros(0, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.uint8))
    p = empty.plan_fetch(empty.upload_tipset(ts1), [], [])
    assert len(p.cids) == 0 and p.n_needed == 0
    full = api.BlockStore.from_tipset(ts1)
    p = full.plan_fetch(full.upload_tipset(ts1), [], [spec_of(ts1)])
    assert len(p.cids) == 0 and p.n_needed > 0


def test_flags_and_storage_specs_without_state_root_are_refused(api, ts1, ts3_small):
    full = api.BlockStore.from_tipset(ts1)
    tip = full.upload_tipset(ts1)
    with pytest.raises(A.IpcfpError) as e:
        full.plan_fetch(tip, [], [spec_of(ts1)], flags=A.RESULT_JSON)
    assert e.value.status == A.ERR_INVALID_ARG
    # a tipset uploaded without child_parent_state_root: storage specs are refused as ipcfp_generate_proof_bundle_resident refuses them
    ts = _Edited(ts3_small, parent_state_root=np.zeros(0, np.uint8))
    st = api.BlockStore.from_tipset(ts3_small)
    tip = st.upload_tipset(ts)
    sspecs = _sspecs(api, ts3_small)
    errs = []
    for fn in (st.plan_fetch, st.generate_proof_bundle_resident):
        with pytest.raises(A.IpcfpError) as e:
            fn(tip, sspecs, [spec_of(ts3_small)])
        errs.append(e.value.status)
    assert errs == [A.ERR_INVALID_ARG, A.ERR_INVALID_ARG]
    assert len(st.plan_fetch(tip, [], [spec_of(ts3_small)]).cids) == 0   # event specs alone need no state root


@pytest.mark.parametrize("seed", range(6))
def test_random_subsets_match_the_restatement(api, ts3_small, seed):
    ts = ts3_small
    cids, blocks = B.blocks_of(ts)
    rng = np.random.default_rng(seed)
    keep = rng.random(len(cids)) < [0.2, 0.5, 0.8, 0.9, 0.97, 0.995][seed]
    sub = api.BlockStore(*_pack(cids[keep], [b for b, k in zip(blocks, keep) if k]))
    held = {bytes(c): b for c, b, k in zip(cids, blocks, keep) if k}
    sspecs = _sspecs(api, ts)
    p = sub.plan_fetch(sub.upload_tipset(ts), sspecs, [spec_of(ts)])
    exp, n_needed = restate_plan(held, ts, sspecs, _especs(ts))
    assert [bytes(c) for c in p.cids] == exp
    assert p.n_needed == n_needed


def _pack(cids, blocks):
    lens = np.array([len(b) for b in blocks], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens, dtype=np.uint64)[:-1]]).astype(np.uint64) if len(blocks) else np.zeros(0, np.uint64)
    blob = np.frombuffer(b"".join(blocks), np.uint8) if blocks else np.zeros(0, np.uint8)
    return np.ascontiguousarray(cids, np.uint8), offs, lens, blob


class _Edited:
    """A tipset descriptor with some attributes replaced."""

    def __init__(self, ts, **over):
        self._ts, self._over = ts, over

    def __getattr__(self, k):
        return self._over[k] if k in self._over else getattr(self._ts, k)


def test_foreign_prefix_is_missing_and_sorted_in_cid_order(api, ts1):
    roots = np.asarray(ts1.events_roots).reshape(-1, 38).copy()
    i = int(np.flatnonzero(np.asarray(ts1.has_events_root))[0])
    roots[i, 1] = 0x55   # raw codec: a prefix no block of the store has
    ts = _Edited(ts1, events_roots=roots)
    full = api.BlockStore.from_tipset(ts1)
    p = full.plan_fetch(full.upload_tipset(ts), [], [spec_of(ts1)])
    assert [bytes(c) for c in p.cids] == [bytes(roots[i])]
    held = {bytes(c): b for c, b in zip(*B.blocks_of(ts1))}
    assert restate_plan(held, ts, [], _especs(ts1))[0] == [bytes(roots[i])]
    # with a second missing CID of the chain prefix the host puts the two in `Cid` order (codec 0x55 < 0x71)
    sub_cids, sub_blocks = B.blocks_of(ts1)
    drop = bytes(ts1.receipts_root)
    keep = [k for k in range(len(sub_cids)) if bytes(sub_cids[k]) != drop]
    sub = api.BlockStore(*_pack(sub_cids[keep], [sub_blocks[k] for k in keep]))
    p = sub.plan_fetch(sub.upload_tipset(ts), [], [spec_of(ts1)])
    assert [bytes(c) for c in p.cids] == sorted([bytes(roots[i]), drop], key=P.cid_sort_key) == [bytes(roots[i]), drop]


def _manual_loop(api, ts, blk, especs_c, verify=False):
    """Plan / fetch rounds from an empty store over the blocks `blk` can supply; stops when a plan is empty or names only CIDs `blk`
    lacks. Returns (store, tipset, the CIDs nobody could supply)."""
    cids, texts = [], []
    store = api.BlockStore(np.zeros((0, 38), np.uint8), np.zeros(0, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.uint8))
    tip = store.upload_tipset(ts)
    while True:
        want = [bytes(c) for c in store.plan_fetch(tip, [], especs_c).cids]
        got = [c for c in want if c in blk]
        if not got:
            return store, tip, want
        texts += B.render([], elements=[B.element(len(cids) + k, blk[c]) for k, c in enumerate(got)])
        cids += got
        store = api.BlockStore.from_rpc_json(np.frombuffer(b"".join(cids), np.uint8).reshape(-1, 38), texts, verify_cids=verify)
        tip = store.upload_tipset(ts)


def _outcome(store, tip, especs_c):
    try:
        return store.generate_proof_bundle_resident(tip, [], especs_c, A.RESULT_JSON).json, None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def test_undecodable_and_unavailable_blocks(api, ts1):
    """A fetched block that does not decode: the loop ends and the planned store gives the full store's status and index. A CID no node
    can supply: the store the rounds reach without it gives MISSING_BLOCK at the index the full store without that block gives."""
    cids, blocks = B.blocks_of(ts1)
    full = {bytes(c): b for c, b in zip(cids, blocks)}
    roots = np.asarray(ts1.events_roots).reshape(-1, 38)
    i = int(np.flatnonzero(np.asarray(ts1.has_events_root))[-1])
    bad_cid = bytes(roots[i])
    spec = [spec_of(ts1)]
    for mode in ("undecodable", "unavailable"):
        blk = dict(full)
        if mode == "undecodable":
            blk[bad_cid] = b"\xff"
        else:
            del blk[bad_cid]
        store, tip, unsupplied = _manual_loop(api, ts1, blk, spec)
        assert unsupplied == ([] if mode == "undecodable" else [bad_cid])
        ks = list(blk)
        ref = api.BlockStore(*_pack(np.frombuffer(b"".join(ks), np.uint8).reshape(-1, 38), [blk[c] for c in ks]))
        got, exp = _outcome(store, tip, spec), _outcome(ref, ref.upload_tipset(ts1), spec)
        assert got == exp and got[1][0] == (A.ERR_DECODE if mode == "undecodable" else A.ERR_MISSING_BLOCK)


def test_request_batch_is_accepted_by_the_device_parser(api, ts1):
    cids, blocks = B.blocks_of(ts1)
    full = {bytes(c): b for c, b in zip(cids, blocks)}
    empty = api.BlockStore(np.zeros((0, 38), np.uint8), np.zeros(0, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.uint8))
    p = empty.plan_fetch(empty.upload_tipset(ts1), [], [spec_of(ts1)])
    import json
    req = json.loads(api.fetch_plan_to_rpc_json(p.cids, 5))
    assert [r["id"] for r in req] == list(range(5, 5 + len(p.cids)))
    pad = cids[:5]
    els = [B.element(k, full[bytes(c)]) for k, c in enumerate(pad)]
    els += [B.element(r["id"], full[bytes(c)]) for r, c in zip(req, p.cids)]
    st = api.BlockStore.from_rpc_json(np.concatenate([pad, p.cids]), B.render([], elements=els), verify_cids=True)
    assert st.json_info.parsed_on_device
    assert all(st.has(c) for c in p.cids)


# ------------------------------------------------------------------------------------------ hand-built trees
def _hand_loop(api, ts, blocks, sspecs, especs_c, especs_py):
    """_check_loop over a hand-built block set (a dict that may hold more than the tipset needs)."""
    full = {bytes(c): bytes(b) for c, b in blocks.items()}
    store, tip, rounds = _run_loop(api, ts, full, sspecs, especs_c, especs_py)
    union = {bytes(c) for r in rounds for c in r.cids}
    assert union == _oracle_reads(full, ts, sspecs, especs_py)
    ref = api.BlockStore.from_tipset(ts)
    rtip = ref.upload_tipset(ts)
    assert (store.generate_proof_bundle_resident(tip, sspecs, especs_c, A.RESULT_JSON).json ==
            ref.generate_proof_bundle_resident(rtip, sspecs, especs_c, A.RESULT_JSON).json)
    return rounds


def test_hand_built_events_amts_every_bit_width_and_height():
    """tests/event_amts.py's valid catalogue: events AMTs at bit widths 1–8, heights 0, 1, 2, the minimal one and 64 // bw (bit width 1 at
    height 64 included), sparse and edge indices, empty roots, under the receipts of one tipset."""
    import ipc_filecoin_proofs_b200.api as api
    from tests import event_amts as E
    c = E.valid_case(E.base_tipset())
    rounds = _hand_loop(api, c.ts, c.blocks, [], [spec_of(c.ts)], _especs(c.ts))
    assert len(rounds) >= 66   # the bit-width-1, height-64 AMT is fetched one level per round


@pytest.mark.parametrize("h", list(range(0, 22)) + ["empty"])
def test_hand_built_message_amts_every_height(h):
    """tests/message_amts.py's shape cases: message AMTs of every height 0–21 (and an empty and a full height-0 pair) as a parent's
    TxMeta, beside the synthetic parent."""
    import ipc_filecoin_proofs_b200.api as api
    from tests import message_amts as M
    cases = {c.name: c for c in M.shape_cases(M.base_tipset())}
    c = cases[f"shape-h{h}-x1" if h != "empty" else "shape-empty-full-x1"]
    rounds = _hand_loop(api, c.ts, c.blocks, [], [spec_of(c.ts)], _especs(c.ts))
    assert len(rounds) >= (h if h != "empty" else 0) + 2   # TxMeta, then the AMT roots, then one round per node level


def _shapes_world(ts):
    """One state tree whose actors hold every contract-state shape: A1, A2, A3, B1 at storage-HAMT bit widths 1–8, B2 and C; with the
    slots each spec asks for (present and absent)."""
    import random
    from tests import storage_trees as T
    rng = random.Random(3)
    blocks = T.Blocks()
    pairs = [(rng.randbytes(32), rng.randbytes(n)) for n in (0, 5, 32, 40)]
    trie = {rng.randbytes(32): T.u8vec(rng.randbytes(rng.randrange(1, 40))) for _ in range(150)}
    shapes = {1: blocks.put(T.wrap_a1([T.small_map(pairs), T.small_map(pairs[:1])])), 2: blocks.put(T.wrap_a2(T.small_map(pairs))),
              3: blocks.put(T.wrap_a3(T.small_map(pairs)))}
    for bw in range(1, 9):
        shapes[10 + bw] = blocks.put(T.wrap_b1(T.build_hamt(blocks, trie, bw), bw))
    shapes[20] = blocks.put(T.wrap_b2(T.build_hamt(blocks, trie, 4), 4))
    shapes[21] = T.build_hamt(blocks, trie, 5)   # C: the contract state is the HAMT root itself
    actors = {aid: T.actor_state(blocks.put(T.evm_state(root, six=bool(aid & 1)))) for aid, root in shapes.items()}
    root = blocks.put(T.state_root(T.build_hamt(blocks, {T.id_address(a): s for a, s in actors.items()}, 5)))
    hdr, child = T.child_header(ts, root)
    blocks[child] = hdr
    for i in range(int(ts.n_blocks)):
        blocks.setdefault(bytes(ts.cids[i]), ts.block(i))
    flat = T.Flat(blocks)
    keys = sorted(trie)
    slots = [pairs[0][0], pairs[2][0], keys[0], keys[77], rng.randbytes(32)]
    specs = [(a, s) for a in shapes for s in slots] + [(999, slots[0])]   # actor 999 does not exist
    return T.tipset(ts, flat.arrays(), child, root), blocks, specs


def test_hand_built_state_trees_every_contract_state_shape(api, ts3_small):
    ts, blocks, specs = _shapes_world(ts3_small)
    ok = [s for s in specs if s[0] != 999]
    _hand_loop(api, ts, blocks, ok, [], [])
    # an actor that does not exist: the loop converges and the planned store fails where the complete one fails
    full = {bytes(c): bytes(b) for c, b in blocks.items()}
    store, tip, rounds = _run_loop(api, ts, full, specs, [], [])
    ref = api.BlockStore.from_tipset(ts)
    errs = []
    for s, t in ((store, tip), (ref, ref.upload_tipset(ts))):
        with pytest.raises(A.IpcfpError) as e:
            s.generate_proof_bundle_resident(t, specs, [])
        errs.append((e.value.status, e.value.index))
    assert errs[0] == errs[1] and errs[0][0] == A.ERR_ACTOR_NOT_FOUND


def test_hand_built_deep_state_tree(api, ts3_small):
    """storage_trees.world_proofs: the deepest accepted path (a 51-node actors chain, then a 256-node width-1 storage chain), one block
    fetched per round."""
    from tests import storage_trees as T
    w, flat = T.world_proofs(ts3_small)
    rounds = _hand_loop(api, w.tips["deep"], flat.blocks, [(w.deep_actor, w.deep_slot)], [], [])
    assert len(rounds) == 310   # 311 blocks, the child header and the StateRoot in the first round


def test_one_million_receipts_converge_to_the_same_bundle(api, synth_mod):
    ts = synth_mod.Tipset(synth_mod.config_params(4))
    cids, blocks = B.blocks_of(ts)
    full = {bytes(c): b for c, b in zip(cids, blocks)}
    del cids, blocks
    asked = set()

    def fetch(cs, first_id):
        for c in cs:
            assert bytes(c) not in asked
            asked.add(bytes(c))
        return B.render([], elements=[B.element(first_id + k, full[bytes(c)]) for k, c in enumerate(cs)])

    spec = [spec_of(ts)]
    store, tip, rounds, _, _ = api.fetch_until_complete(fetch, lambda s: s.upload_tipset(ts), [], spec, verify_cids=False)
    ref = api.BlockStore.from_tipset(ts)
    rtip = ref.upload_tipset(ts)
    assert store.generate_proof_bundle_resident(tip, [], spec, A.RESULT_JSON).json == \
        ref.generate_proof_bundle_resident(rtip, [], spec, A.RESULT_JSON).json
    assert ref.plan_fetch(rtip, [], spec).n_needed == len(asked)
