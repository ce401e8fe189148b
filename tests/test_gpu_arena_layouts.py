"""The engine on re-laid arenas (tests/arena_layouts.py): results depend only on [offset, offset + length) of the blocks read.

A. Fillers (zero, ff, random, echo, next) × order (index, shuffled) and every start residue mod 16 with the last block ending at
   blob_size: each layout gives the canonical layout's results, field for field, and the witness block for block (CIDs, and the bytes
   at each (offset, length): the pad bytes between witness blocks are unspecified). By-reference offsets are the new layout's.
B. Shortened in place: each block of a call's read set cut to k < len with its own suffix still behind it → the oracle's (status, index)
   or result on the same arrays (the oracle's Blockstore::get clones exactly len bytes).
C. Far offsets: config 2 in a 2^32 + 64 MiB blob, blocks straddling 2^31 and 2^32, ending and starting at 2^32, the rest above;
   monotonic (chunked CID check) and shuffled (one chunk). By-reference offsets come back ≥ 2^32 unchanged; the verifiers accept a
   by-reference witness into that blob; the batched hashes read messages at offsets 2^31 − 3, 2^32 − 1 and 2^32 + 5.
D. The chunked CID check: one flipped byte in the first block, the last block of chunk 0, the first of chunk 1, the straddling block,
   the last block, two blocks in two chunks, a Blake2s-listed block → the smallest Blake2b mismatch (or none), chunked and not.
E. Non-zero scratch memory: the cudaMallocAsync pool filled with 0xA5 before every call and the library's device pool before every
   store; every result equals the unpoisoned one.
Entry points: generate_event_proof (flags 0, JSON, by reference, both), tipset_upload + generate_log_proof_resident (the spec's filter,
the all-wildcard filter), generate_proof_bundle_resident with JSON, verify_bundle_json on that text, plan_fetch_resident on a store
missing blocks, read_storage_slots (1 000 and 16 385 lookups, fast and IPCFP_HAMT_STRICT), generate_storage_proofs, resolve_addresses
(fast and strict), verify_event_proofs / verify_storage_proofs on witnesses the builder laid out. Not covered: witnesses re-anchored to
honest CIDs after a block is shortened (the hostile-witness tests cover forged witnesses under honest CIDs on the canonical layout)."""
import ctypes as C
import hashlib
import random

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import address_trees as AT
from tests import arena_layouts as L
from tests import event_amts as E
from tests import storage_trees as T
from tests.util import spec_of, synth_tipset

pytestmark = pytest.mark.gpu

EV_FLAGS = (0, A.RESULT_JSON, A.WITNESS_BY_REFERENCE, A.RESULT_JSON | A.WITNESS_BY_REFERENCE)


def _outcome(fn):
    try:
        return fn(), None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _wit_key(w, lay=None, byref=False):
    """CIDs, lengths and block bytes of a witness; by reference: the bytes are read from the layout's blob, and every offset must be the
    layout's offset of that CID."""
    if byref:
        assert len(w.blob) == 0
        offs = {}
        for i in range(lay.n_blocks):
            offs.setdefault(bytes(lay.cids[i]), []).append(int(lay.offsets[i]))
        for i in range(w.n_blocks):
            assert int(w.offsets[i]) in offs[bytes(w.cids[i])], i
        blocks = [bytes(lay.blob[int(o):int(o) + int(n)]) for o, n in zip(w.offsets, w.lengths)]
    else:
        blocks = w.blocks()
    return (w.cids.tobytes(), w.lengths.tobytes(), blocks)


def _ev_key(r, lay=None, flags=0):
    return (r.matching.tolist(), r.n_exec, [p.key() for p in r.proofs], r.data_blob.tobytes(),
            _wit_key(r.witness, lay, bool(flags & A.WITNESS_BY_REFERENCE)), r.json if flags & A.RESULT_JSON else None)


def _none():
    pass


def event_calls(api, store, ts, lay, poison=_none):
    """The event-side entry points on one store → {call: comparable result}. poison() runs before every call."""
    spec = spec_of(ts)
    out = {}
    for fl in EV_FLAGS:
        poison()
        out[("event", fl)] = _ev_key(store.generate_event_proof(ts, spec, flags=fl), lay, fl)
    poison()
    tip = store.upload_tipset(ts)
    try:
        for name, f in (("spec", api.LogFilter.from_spec(api.EventProofSpec(ts.event_signature, ts.topic1, ts.actor_filter))), ("any", api.LogFilter())):
            poison()
            out[("log", name)] = _ev_key(store.generate_log_proof_resident(tip, f), lay, 0)
        poison()
        b = store.generate_proof_bundle_resident(tip, [], [spec], flags=A.RESULT_JSON)
        out["bundle"] = (b.json, _wit_key(b.witness))
        poison()
        v = api.verify_bundle_json(b.json)
        out["verify_bundle_json"] = (v.event_results, v.storage_results, v.n_blocks)
    finally:
        tip.close()
    return out


def plan_calls(api, ts, lay, poison=_none):
    """plan_fetch_resident on a store of the layout missing every fifth block of the event call's read set → the plan's CIDs."""
    full = api.BlockStore.from_tipset(lay.over(ts))
    try:
        read = {bytes(c) for c in full.generate_event_proof(lay.over(ts), spec_of(ts)).witness.cids}
    finally:
        full.close()
    drop = set(sorted(read)[::5])
    keep = [i for i in range(lay.n_blocks) if bytes(lay.cids[i]) not in drop]
    part = L.Layout(lay.cids[keep], lay.offsets[keep], lay.lengths[keep], lay.blob)
    t = part.over(ts)
    store = api.BlockStore.from_tipset(t)
    try:
        poison()
        tip = store.upload_tipset(t)
        try:
            poison()
            p = store.plan_fetch(tip, [], [spec_of(t)])
        finally:
            tip.close()
    finally:
        store.close()
    assert p.cids.shape[0] > 0
    return p.cids.tobytes(), p.n_needed


def resolve_calls(store, aw, poison=_none):
    """resolve_addresses over the 5 000-entry address map, fast and strict HAMT decoder (the HV_U64 fast path of hamt_node_lookup_fast)."""
    out = {}
    for strict in (None, "1"):
        aw.mp.setenv("IPCFP_HAMT_STRICT", "1") if strict else aw.mp.delenv("IPCFP_HAMT_STRICT", raising=False)
        poison()
        r = store.resolve_addresses(aw.root, aw.addrs)
        out[("resolve", strict)] = (r.init_status, r.status.tolist(), r.actor_ids.tolist(), r.missing.tobytes(), _wit_key(r.witness))
    aw.mp.delenv("IPCFP_HAMT_STRICT", raising=False)
    return out


def storage_calls(store, w, slot_case, monkeypatch, poison=_none):
    rng = random.Random(11)
    out = {}
    slots = list(slot_case.slots)
    for n in (1000, 16385):
        batch = [slots[i % len(slots)] if i % 3 else rng.randbytes(32) for i in range(n)]
        arr = np.frombuffer(b"".join(batch), dtype=np.uint8).reshape(-1, 32)
        for strict in (None, "1"):
            if strict:
                monkeypatch.setenv("IPCFP_HAMT_STRICT", "1")
            else:
                monkeypatch.delenv("IPCFP_HAMT_STRICT", raising=False)
            poison()
            r = store.read_storage_slots(slot_case.root_np(), arr)
            out[("slots", n, strict)] = (r.found.tobytes(), r.raw_len.tobytes(), r.values.tobytes(), _wit_key(r.witness))
    monkeypatch.delenv("IPCFP_HAMT_STRICT", raising=False)
    ok, _ = T.proof_batches(w)
    for tip, specs in ok:
        poison()
        r = store.generate_storage_proofs(w.tips[tip], specs)
        out[("proofs", tip)] = ([(p.found, p.raw_len, bytes(p.value)) for p in r.proofs], _wit_key(r.witness), r.raw_proofs.tobytes())
    return out


@pytest.fixture(scope="module")
def storage_world(ts3_small):
    """world_proofs' blocks and the largest slot case of world_slots (its root and slots) in one flat set."""
    w, f = T.world_proofs(ts3_small)
    sblocks, cases = T.world_slots()
    blocks = T.Blocks(f.blocks)
    for c, b in sblocks.items():
        blocks.setdefault(c, b)
    case = max((c for c in cases if c.truth is not None), key=lambda c: len(c.slots))
    flat = T.Flat(blocks)
    w.tips = {name: T.tipset(ts3_small, flat.arrays(), c, root) for name, (c, root) in w.heads.items()}
    return w, flat, case


class AddressWorld:
    """A state tree whose Init actor holds a 5 000-entry address map (tests/address_trees.py), its blocks, and a batch of addresses:
    every 10th key of the map, random absent addresses of every kind and ID addresses."""

    def __init__(self, mp):
        self.mp = mp
        blocks = T.Blocks()
        ent = AT._entries(random.Random(5000), 5000)
        self.root = AT.state_tree(blocks, ent)
        self.blocks = dict(blocks)
        rng = random.Random(7)
        self.addrs = list(ent)[::10] + [AT.random_address(rng, AT.KINDS[i % len(AT.KINDS)]) for i in range(60)] + [AT.id_addr(7)]
        self.flat = T.Flat(blocks)


@pytest.fixture
def address_world(monkeypatch):
    return AddressWorld(monkeypatch)


def _layouts(src, seed=3):
    for filler in L.FILLERS:
        for order in ("index", "shuffled"):
            yield f"{filler}-{order}", L.lay_out(src.cids, src.offsets, src.lengths, src.blob, filler=filler, order=order, seed=seed)
    yield "residues", L.lay_out(src.cids, src.offsets, src.lengths, src.blob, filler="echo", residues=True, tail=0, seed=seed)


# ---------------------------------------------------------------------------------------------------------------- A
@pytest.mark.parametrize("walk", [None, "1"])
@pytest.mark.parametrize("cfg", [1, 2, "shapes", "ts3", "event-amts"])
def test_a_event_paths_on_every_layout(api, synth_mod, ts3_small, monkeypatch, cfg, walk):
    """event-amts: tests/event_amts.py's valid hand-built events AMTs, bit widths 1–8 at heights 0, 1, 2 and the maximum, one per
    receipt of one tipset."""
    if walk:
        monkeypatch.setenv("IPCFP_BFS_GENERAL", "1")
    case = E.valid_case(E.base_tipset()) if cfg == "event-amts" else None
    ts = ts3_small if cfg == "ts3" else (case.ts if case else synth_tipset(synth_mod, cfg))
    canon = L.Layout(ts.cids, ts.offsets, ts.lengths, ts.blob)
    store = api.BlockStore.from_tipset(ts, verify_cids=True)
    exp = event_calls(api, store, ts, canon)
    res = store.generate_event_proof(ts, spec_of(ts))
    store.close()
    # the bundle text verifies as the reference would: every proof, except (event-amts) an event at index 2^64 − 1 of an AMT with
    # height·bw = 64, which the reference's `get` cannot reach (tests/event_amts.py honest_verdicts)
    assert exp["verify_bundle_json"][0] == (E.honest_verdicts(case, res) if case else [True] * len(res.proofs))
    exp_plan = plan_calls(api, ts, canon)
    for name, lay in _layouts(ts):
        t = lay.over(ts)
        store = api.BlockStore.from_tipset(t, verify_cids=True)
        try:
            got = event_calls(api, store, t, lay)
        finally:
            store.close()
        for k in exp:
            assert got[k] == exp[k], (name, k)
        assert plan_calls(api, ts, lay) == exp_plan, name
        # the verifiers on a witness laid out by the builder
        r = api.BlockStore.from_tipset(t).generate_event_proof(t, spec_of(t))
        wl = L.lay_out(r.witness.cids, r.witness.offsets, r.witness.lengths, r.witness.blob, filler="echo", order="shuffled")
        assert api.verify_event_proofs(wl, t, r) == (E.honest_verdicts(case, r) if case else [True] * len(r.proofs)), name


def test_a_storage_paths_on_every_layout(api, storage_world, monkeypatch):
    w, flat, case = storage_world
    store = api.BlockStore(flat.cids, flat.offsets, flat.lengths, flat.blob, verify_cids=True)
    exp = storage_calls(store, w, case, monkeypatch)
    store.close()
    for name, lay in _layouts(flat):
        store = api.BlockStore(lay.cids, lay.offsets, lay.lengths, lay.blob, verify_cids=True)
        try:
            got = storage_calls(store, w, case, monkeypatch)
        finally:
            store.close()
        for k in exp:
            assert got[k] == exp[k], (name, k)
    ok, _ = T.proof_batches(w)
    tip, specs = ok[0]
    r = api.BlockStore(flat.cids, flat.offsets, flat.lengths, flat.blob).generate_storage_proofs(w.tips[tip], specs)
    wl = L.lay_out(r.witness.cids, r.witness.offsets, r.witness.lengths, r.witness.blob, filler="ff", order="shuffled")
    assert all(api.verify_storage_proofs(wl, w.tips[tip], r))


def test_a_resolve_on_every_layout(api, address_world):
    aw = address_world
    f = aw.flat
    store = api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True)
    exp = resolve_calls(store, aw)
    store.close()
    assert exp[("resolve", None)][0] == A.OK and sum(s == A.OK for s in exp[("resolve", None)][1]) >= 500
    for name, lay in _layouts(f):
        store = api.BlockStore(lay.cids, lay.offsets, lay.lengths, lay.blob, verify_cids=True)
        try:
            got = resolve_calls(store, aw)
        finally:
            store.close()
        assert got == exp, name


# ---------------------------------------------------------------------------------------------------------------- B
def test_b_shortened_blocks_of_the_event_path(api, oracle_mod, synth_mod):
    """Parent and child headers, TxMeta, message-, receipts- and events-AMT roots and nodes: each block of the config-1 call's read
    set cut in place to every length of arena_layouts.shorten_lengths → the oracle's outcome on the same arrays."""
    ts = synth_mod.Tipset(synth_mod.config_params(1))
    lay = L.lay_out(ts.cids, ts.offsets, ts.lengths, ts.blob, filler="echo")
    spec = spec_of(ts)
    full = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec)
    index = {bytes(c): i for i, c in enumerate(lay.cids)}
    runs = 0
    for c in full.witness.cids:
        i = index[bytes(c)]
        for k in L.shorten_lengths(int(lay.lengths[i])):
            t = L.shortened(lay, i, k).over(ts)
            exp, eerr = _outcome(lambda: oracle_mod.Store.from_tipset(t).generate_event_proof(t, spec))
            store = api.BlockStore.from_tipset(t)
            try:
                for fl in (0, A.WITNESS_BY_REFERENCE):
                    got, gerr = _outcome(lambda: store.generate_event_proof(t, spec, flags=fl))
                    assert gerr == eerr, (i, k, fl)
                    if eerr is None:
                        assert _ev_key(got, L.shortened(lay, i, k), fl)[:5] == _ev_key(exp)[:5], (i, k, fl)
            finally:
                store.close()
            runs += 1
    assert runs > 200


def test_b_shortened_blocks_of_the_storage_path(api, oracle_mod, storage_world):
    """Actors-HAMT nodes, EVM state, contract state, storage-HAMT nodes (and the header, StateRoot): each block of a storage-proof
    call's read set cut in place → the oracle's (status, index) or proofs."""
    w, flat, case = storage_world
    ok, _ = T.proof_batches(w)
    tip, specs = ok[0]
    specs = specs[:12]                       # actors of every root shape A1–C with present and absent slots: every block kind
    ts = w.tips[tip]
    lay = L.lay_out(flat.cids, flat.offsets, flat.lengths, flat.blob, filler="echo")
    full = oracle_mod.Store(flat.cids, flat.offsets, flat.lengths, flat.blob).generate_storage_proofs(ts, specs)
    index = {bytes(c): i for i, c in enumerate(lay.cids)}
    runs = 0
    for c in full.witness.cids:
        i = index[bytes(c)]
        for k in L.shorten_lengths(int(lay.lengths[i])):
            s = L.shortened(lay, i, k)
            t = s.over(ts)
            exp, eerr = _outcome(lambda: oracle_mod.Store(s.cids, s.offsets, s.lengths, s.blob).generate_storage_proofs(t, specs))
            store = api.BlockStore(s.cids, s.offsets, s.lengths, s.blob)
            try:
                got, gerr = _outcome(lambda: store.generate_storage_proofs(t, specs))
            finally:
                store.close()
            assert gerr == eerr, (i, k)
            if eerr is None:
                assert [(p.found, p.raw_len, bytes(p.value)) for p in got.proofs] == [(p.found, p.raw_len, bytes(p.value)) for p in exp.proofs], (i, k)
                assert _wit_key(got.witness) == _wit_key(exp.witness), (i, k)
            runs += 1
    assert runs > 50


def test_b_shortened_blocks_of_address_resolution(api, address_world):
    """StateRoot, actors-HAMT nodes, the Init ActorState, InitState and address_map nodes: each block of the resolve call's read set cut
    in place to every length of arena_layouts.shorten_lengths → the Python restatement (tests/address_trees.resolve) on a block set
    holding exactly the cut bytes: per-address status and ID, Init status, missing CIDs and read set."""
    aw = address_world
    addrs = aw.addrs[:40] + aw.addrs[-20:]
    lay = L.lay_out(aw.flat.cids, aw.flat.offsets, aw.flat.lengths, aw.flat.blob, filler="echo")
    _, _, _, _, read = AT.resolve(aw.blocks, aw.root, addrs)
    index = {bytes(c): i for i, c in enumerate(lay.cids)}
    runs = 0
    for mode in (None, "1"):
        aw.mp.setenv("IPCFP_HAMT_STRICT", "1") if mode else aw.mp.delenv("IPCFP_HAMT_STRICT", raising=False)
        for c in read:
            i = index[c]
            for k in L.shorten_lengths(int(lay.lengths[i])):
                s = L.shortened(lay, i, k)
                exact = dict(aw.blocks)
                exact[c] = s.block(i)
                ids, status, init, missing, rd = AT.resolve(exact, aw.root, addrs)
                store = api.BlockStore(s.cids, s.offsets, s.lengths, s.blob)
                try:
                    got = store.resolve_addresses(aw.root, addrs)
                finally:
                    store.close()
                assert (got.init_status, got.status.tolist(), got.actor_ids.tolist()) == (init, status, ids), (c.hex(), k, mode)
                assert [bytes(x) for x in got.missing] == missing and [bytes(x) for x in got.witness.cids] == rd, (c.hex(), k, mode)
                runs += 1
    assert runs > 100


# ---------------------------------------------------------------------------------------------------------------- C
def _low_blocks(ts):
    roots = {bytes(ts.events_roots[i]) for i in range(int(ts.n_receipts)) if ts.has_events_root[i]}
    return [i for i in range(ts.n_blocks) if bytes(ts.cids[i]) not in roots and int(ts.lengths[i]) > 8][:3]


@pytest.mark.parametrize("order", ["index", "shuffled"])
def test_c_far_offsets(api, synth_mod, order):
    ts = synth_mod.Tipset(synth_mod.config_params(2))
    canon = L.Layout(ts.cids, ts.offsets, ts.lengths, ts.blob)
    store = api.BlockStore.from_tipset(ts, verify_cids=True)
    exp = event_calls(api, store, ts, canon)
    store.close()
    lay = L.far(ts.cids, ts.offsets, ts.lengths, ts.blob, _low_blocks(ts), order=order, straddle32=order != "index")
    t = lay.over(ts)
    store = api.BlockStore.from_tipset(t, verify_cids=True)
    try:
        got = event_calls(api, store, t, lay)
        for k in exp:
            assert got[k] == exp[k], k
        ref = store.generate_event_proof(t, spec_of(t), flags=A.WITNESS_BY_REFERENCE)
    finally:
        store.close()
    assert int(ref.witness.offsets.max()) >= 1 << 32
    # the verifiers on a by-reference witness into the far blob
    w = L.Layout(ref.witness.cids, ref.witness.offsets, ref.witness.lengths, lay.blob)
    assert all(api.verify_event_proofs(w, t, ref))
    del lay, w, t


@pytest.mark.parametrize("order", ["index", "shuffled"])
def test_c_far_offsets_storage_and_resolve(api, storage_world, address_world, monkeypatch, order):
    """The storage world and the 5 000-entry address map in one block set, laid out far: read_storage_slots, generate_storage_proofs
    and resolve_addresses equal the canonical layout's, and the storage verifier accepts a by-reference-style witness into that blob."""
    w, flat, case = storage_world
    aw = address_world
    blocks = T.Blocks(flat.blocks)
    for c, b in aw.blocks.items():
        blocks.setdefault(c, b)
    f = T.Flat(blocks)
    store = api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True)
    exp = {**storage_calls(store, w, case, monkeypatch), **resolve_calls(store, aw)}
    store.close()
    low = [i for i in range(f.n_blocks) if int(f.lengths[i]) > 8][:3]
    lay = L.far(f.cids, f.offsets, f.lengths, f.blob, low, order=order, straddle32=order != "index")
    store = api.BlockStore(lay.cids, lay.offsets, lay.lengths, lay.blob, verify_cids=True)
    try:
        got = {**storage_calls(store, w, case, monkeypatch), **resolve_calls(store, aw)}
        ok, _ = T.proof_batches(w)
        tip, specs = ok[0]
        r = store.generate_storage_proofs(w.tips[tip], specs)
    finally:
        store.close()
    for k in exp:
        assert got[k] == exp[k], k
    offs = {bytes(lay.cids[i]): int(lay.offsets[i]) for i in range(lay.n_blocks)}
    wl = L.Layout(r.witness.cids, np.array([offs[bytes(c)] for c in r.witness.cids], dtype=np.uint64), r.witness.lengths, lay.blob)
    assert int(wl.offsets.max()) >= 1 << 32
    assert all(api.verify_storage_proofs(wl, w.tips[tip], r))
    del lay, wl


def test_c_hash_batches_past_4_gib(api):
    from oracle import keccak256
    lib = api.lib()
    offs = ((1 << 31) - 3, (1 << 32) - 1, (1 << 32) + 5)
    lens = (0, 1, 127, 128, 135, 136, 137)
    blob = np.zeros((1 << 32) + 4096, dtype=np.uint8)
    rng = np.random.default_rng(9)
    for o in offs:
        blob[o:o + 160] = rng.integers(0, 256, 160, dtype=np.uint8)
    o_arr = np.array([o for o in offs for _ in lens], dtype=np.uint64)
    l_arr = np.array([n for _ in offs for n in lens], dtype=np.uint32)
    msgs = [bytes(blob[int(o):int(o) + int(n)]) for o, n in zip(o_arr, l_arr)]
    refs = {"ipcfp_blake2b256_batch": lambda m: hashlib.blake2b(m, digest_size=32).digest(),
            "ipcfp_sha256_batch": lambda m: hashlib.sha256(m).digest(),
            "ipcfp_keccak256_batch": lambda m: bytes(keccak256(m))}
    for fn, ref in refs.items():
        out = np.zeros((len(msgs), 32), dtype=np.uint8)
        st = getattr(lib, fn)(C.c_void_p(blob.ctypes.data), C.c_uint64(blob.size), C.c_void_p(o_arr.ctypes.data), C.c_void_p(l_arr.ctypes.data),
                              C.c_uint64(len(msgs)), 0, C.c_void_p(out.ctypes.data))
        assert st == A.OK, fn
        assert [bytes(r) for r in out] == [ref(m) for m in msgs], fn
    del blob


# ---------------------------------------------------------------------------------------------------------------- D
def _flip(lay, *idx):
    blob = lay.blob.copy()
    for i in idx:
        o, n = int(lay.offsets[i]), int(lay.lengths[i])
        blob[o + n // 2] ^= 0x40
    return L.Layout(lay.cids, lay.offsets, lay.lengths, blob)


def _shuffled_twin(lay, seed=1):
    """The same arrays, the blocks placed in a shuffled order (non-monotonic: the one-chunk path)."""
    s = L.lay_out(lay.cids, lay.offsets, lay.lengths, lay.blob, filler="zero", order="shuffled", seed=seed)
    return s


def test_d_chunked_cid_check(api, synth_mod):
    ts = synth_mod.Tipset(synth_mod.config_params(2))
    lay, info = L.chunked(ts.cids, ts.offsets, ts.lengths, ts.blob)
    s = info["straddle"]
    cases = {"a-first": (0,), "b-last-of-chunk0": (128,), "c-first-of-chunk1": (info["first_of_chunk1"],), "d-straddle": (s,),
             "e-last": (info["last"],), "f-two-chunks": (s + 5, 128), "g-blake2s": (info["b2s"],)}
    for name, idx in cases.items():
        bad = _flip(lay, *idx)
        expect = L.first_bad_b2b(bad)
        assert (expect is None) == (name == "g-blake2s"), name
        for variant in ("chunked", "one-chunk"):
            v = bad if variant == "chunked" else _shuffled_twin(bad)
            if expect is None:
                api.BlockStore(v.cids, v.offsets, v.lengths, v.blob, verify_cids=True).close()
                continue
            with pytest.raises(A.IpcfpError) as ei:
                api.BlockStore(v.cids, v.offsets, v.lengths, v.blob, verify_cids=True)
            assert ei.value.status == A.ERR_CID_MISMATCH and ei.value.index == expect and ei.value.first_bad_block == expect, (name, variant)
    # untampered: the chunked store gives the unchunked store's proofs
    t = lay.over(ts)
    store = api.BlockStore.from_tipset(t, verify_cids=True)
    try:
        got = store.generate_event_proof(t, spec_of(t))
    finally:
        store.close()
    exp = api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
    assert _ev_key(got) == _ev_key(exp)


# ---------------------------------------------------------------------------------------------------------------- E
def _cu():
    cu = C.CDLL("libcuda.so.1")
    for name, args in (("cuInit", [C.c_uint]), ("cuDeviceGet", [C.POINTER(C.c_int), C.c_int]),
                       ("cuDevicePrimaryCtxRetain", [C.POINTER(C.c_void_p), C.c_int]), ("cuDevicePrimaryCtxRelease_v2", [C.c_int]),
                       ("cuCtxPushCurrent_v2", [C.c_void_p]), ("cuCtxPopCurrent_v2", [C.POINTER(C.c_void_p)]),
                       ("cuDeviceGetDefaultMemPool", [C.POINTER(C.c_void_p), C.c_int]),
                       ("cuMemGetInfo_v2", [C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
                       ("cuMemAllocFromPoolAsync", [C.POINTER(C.c_uint64), C.c_size_t, C.c_void_p, C.c_void_p]),
                       ("cuMemsetD8Async", [C.c_uint64, C.c_ubyte, C.c_size_t, C.c_void_p]), ("cuMemFreeAsync", [C.c_uint64, C.c_void_p]),
                       ("cuStreamSynchronize", [C.c_void_p]), ("cuMemcpyDtoH_v2", [C.c_void_p, C.c_uint64, C.c_size_t])):
        getattr(cu, name).argtypes = args
        getattr(cu, name).restype = C.c_int
    return cu


def poison_async_pool(device=0):
    """Fill min(2 GiB, free / 8) of the device's default cudaMallocAsync pool with 0xA5 and give it back to the pool (the library sets
    the pool's release threshold to ∞, so the memory stays there); then check that a fresh 1 MiB allocation reads 0xA5."""
    cu = _cu()
    ok = lambda r, what: r == 0 or pytest.fail(f"{what}: CUresult {r}")   # noqa: E731
    ok(cu.cuInit(0), "cuInit")
    dev, ctx = C.c_int(), C.c_void_p()
    ok(cu.cuDeviceGet(C.byref(dev), device), "cuDeviceGet")
    ok(cu.cuDevicePrimaryCtxRetain(C.byref(ctx), dev), "cuDevicePrimaryCtxRetain")
    ok(cu.cuCtxPushCurrent_v2(ctx), "cuCtxPushCurrent")
    try:
        pool, free, total = C.c_void_p(), C.c_size_t(), C.c_size_t()
        ok(cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev), "cuDeviceGetDefaultMemPool")
        ok(cu.cuMemGetInfo_v2(C.byref(free), C.byref(total)), "cuMemGetInfo")
        n = min(2 << 30, free.value // 8)
        p = C.c_uint64()
        ok(cu.cuMemAllocFromPoolAsync(C.byref(p), n, pool, None), "cuMemAllocFromPoolAsync")
        ok(cu.cuMemsetD8Async(p.value, 0xA5, n, None), "cuMemsetD8Async")
        ok(cu.cuMemFreeAsync(p.value, None), "cuMemFreeAsync")
        ok(cu.cuStreamSynchronize(None), "cuStreamSynchronize")
        q = C.c_uint64()
        ok(cu.cuMemAllocFromPoolAsync(C.byref(q), 1 << 20, pool, None), "cuMemAllocFromPoolAsync")
        ok(cu.cuStreamSynchronize(None), "cuStreamSynchronize")
        host = np.zeros(1 << 20, dtype=np.uint8)
        ok(cu.cuMemcpyDtoH_v2(host.ctypes.data, q.value, 1 << 20), "cuMemcpyDtoH")
        ok(cu.cuMemFreeAsync(q.value, None), "cuMemFreeAsync")
        ok(cu.cuStreamSynchronize(None), "cuStreamSynchronize")
        if not (host == 0xA5).all():
            pytest.fail("the cudaMallocAsync pool does not hand back the 0xA5-filled memory: the poisoning cannot be observed")
    finally:
        cu.cuCtxPopCurrent_v2(C.byref(C.c_void_p()))
        cu.cuDevicePrimaryCtxRelease_v2(dev)


def poison_device_pool(api, n, blob_size):
    """Create and destroy a store with this n and blob_size, every byte 0xA5 (random digests under the class prefix, no CID check):
    the library's device pool then hands the real store arrays that held 0xA5."""
    rng = np.random.default_rng(n)
    cids = np.zeros((n, 38), dtype=np.uint8)
    cids[:, :6] = np.frombuffer(L.B2B_PREFIX, dtype=np.uint8)
    cids[:, 6:] = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    lens = np.full(n, min(64, blob_size // max(n, 1)), dtype=np.uint32)
    offs = np.arange(n, dtype=np.uint64) * np.uint64(int(lens[0]) if n else 0)
    api.BlockStore(cids, offs, lens, np.full(blob_size, 0xA5, dtype=np.uint8)).close()


def test_e_poisoned_scratch_memory(api, synth_mod, storage_world, address_world, monkeypatch):
    """Both pools poisoned before every entry point (and the device pool before every store): each result equals its unpoisoned one."""
    ts = synth_mod.Tipset(synth_mod.config_params(2))
    w, flat, case = storage_world
    aw = address_world
    canon = L.Layout(ts.cids, ts.offsets, ts.lengths, ts.blob)
    store = api.BlockStore.from_tipset(ts)
    exp_ev = event_calls(api, store, ts, canon)
    store.close()
    exp_plan = plan_calls(api, ts, canon)
    store = api.BlockStore(flat.cids, flat.offsets, flat.lengths, flat.blob)
    exp_st = storage_calls(store, w, case, monkeypatch)
    store.close()
    f = aw.flat
    store = api.BlockStore(f.cids, f.offsets, f.lengths, f.blob)
    exp_rs = resolve_calls(store, aw)
    store.close()
    # the pinned read-back pool comes back dirty: the large all-wildcard log filter first
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    store.generate_log_proof_resident(tip, api.LogFilter())
    tip.close()
    store.close()

    def poison():
        poison_async_pool()

    poison_async_pool()
    poison_device_pool(api, ts.n_blocks, len(ts.blob))
    store = api.BlockStore.from_tipset(ts)
    try:
        got = event_calls(api, store, ts, canon, poison)
    finally:
        store.close()
    for k in exp_ev:
        assert got[k] == exp_ev[k], k
    assert plan_calls(api, ts, canon, poison) == exp_plan
    poison_async_pool()
    poison_device_pool(api, flat.n_blocks, len(flat.blob))
    store = api.BlockStore(flat.cids, flat.offsets, flat.lengths, flat.blob)
    try:
        got = storage_calls(store, w, case, monkeypatch, poison)
    finally:
        store.close()
    for k in exp_st:
        assert got[k] == exp_st[k], k
    poison_async_pool()
    poison_device_pool(api, f.n_blocks, len(f.blob))
    store = api.BlockStore(f.cids, f.offsets, f.lengths, f.blob)
    try:
        got = resolve_calls(store, aw, poison)
    finally:
        store.close()
    assert got == exp_rs
