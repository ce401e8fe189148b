"""CPU tests: the oracle against golden vectors / the independent Python oracle / the restated verifiers,
host logic, and the C-ABI library surface (no GPU compute)."""
import ctypes as C
import hashlib
import os
import re

import cbor2
import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import golden_util
from tests.util import SHAPES, EditedTipset, ShuffledTipset, assert_event_results_equal, dict_of, spec_of, synth_tipset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ hashes
def test_hash_known_answers(oracle_mod, synth_mod):
    from oracle import pyoracle as P
    assert oracle_mod.blake2b256(b"").hex() == "0e5751c026e543b2e8ab2eb06099daa1d1e5df47778f7787faab45cdf12fe3a8"
    assert oracle_mod.keccak256(b"").hex() == "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"
    assert oracle_mod.keccak256(b"Transfer(address,address,uint256)").hex() == "ddf252ad1be2c89b69c2b068fc378daa952ba7f163c4a11628f55a4df523b3ef"
    assert oracle_mod.sha256(b"").hex() == "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"
    rng = np.random.default_rng(0)
    for n in [0, 1, 55, 56, 63, 64, 65, 111, 112, 127, 128, 129, 135, 136, 137, 255, 256, 257, 1028, 4096]:
        m = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert oracle_mod.blake2b256(m) == hashlib.blake2b(m, digest_size=32).digest() == synth_mod.blake2b256(m)
        assert oracle_mod.sha256(m) == hashlib.sha256(m).digest() == synth_mod.sha256(m)
        assert oracle_mod.keccak256(m) == P.keccak256(m) == synth_mod.keccak256(m)


def test_golden_kats(oracle_mod):
    z, _, _ = golden_util.load()
    off = 0
    for k, n in enumerate(z["kat_lens"]):
        m = z["kat_msgs"][off:off + int(n)].tobytes()
        off += int(n)
        assert oracle_mod.blake2b256(m) == z["kat_blake2b"][k].tobytes()
        assert oracle_mod.sha256(m) == z["kat_sha256"][k].tobytes()
        assert oracle_mod.keccak256(m) == z["kat_keccak"][k].tobytes()


def test_topic_constants(oracle_mod):
    # the reference's demo spec (src/main.rs:60-64,38): NewTopDownMessage(bytes32,uint256), "calib-subnet-1", slot index 0
    t0 = oracle_mod.keccak256(b"NewTopDownMessage(bytes32,uint256)")
    assert len(t0) == 32
    key = b"calib-subnet-1" + bytes(18)
    assert oracle_mod.compute_mapping_slot(key, 0) == oracle_mod.keccak256(key + bytes(32))
    assert oracle_mod.compute_mapping_slot(key, 7) == oracle_mod.keccak256(key + (7).to_bytes(32, "big"))


# ------------------------------------------------------------------ synthetic data is well-formed DAG-CBOR with valid CIDs
@pytest.mark.parametrize("cfg", [1, 2, "shapes", "shapes-nofilter"])
def test_synth_blocks_roundtrip_cbor2(synth_mod, cfg):
    ts = synth_tipset(synth_mod, cfg)
    for i in range(ts.n_blocks):
        b = ts.block(i)
        assert cbor2.dumps(cbor2.loads(b)) == b                       # minimal, definite-length encoding
        assert hashlib.blake2b(b, digest_size=32).digest() == bytes(ts.cids[i][6:])
        assert bytes(ts.cids[i][:6]) == bytes([0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20])
        assert int(ts.offsets[i]) % 16 == 0
    import collections
    d = ts.as_dict()
    roots = [d[bytes(ts.events_roots[i])] for i in range(int(ts.n_receipts)) if ts.has_events_root[i]]
    if cfg in SHAPES:
        _check_varied_shapes(ts, roots)
    else:
        # shapes from SURVEY.md §8(a)
        lens = collections.Counter(len(r) for r in roots)
        assert lens.most_common(1)[0][0] == 1028   # events-AMT v3 bw5 root with 8 x 127-byte StampedEvents
    assert oracle_mod_verify(ts)


def _check_varied_shapes(ts, roots):
    """The varied mode covers what it is there for: every emitter head size, Case A with 0-4 topics, Case B with 1-4 topics,
    2-byte data length heads (59 nnnn), odd codecs and flags, duplicate and unknown keys, empty and linked AMTs, and single-node
    roots over 4 KB that hold a forced match."""
    seen = set()
    linked = empty = 0
    for raw in roots:
        bw, height, count, node = cbor2.loads(raw)
        linked += bool(node[1])
        empty += count == 0
        for em, entries in node[2]:
            seen.add(("head", 0 if em < 24 else 1 if em < 256 else 2 if em < 65536 else 4 if em < 2 ** 32 else 8))
            keys = [e[1] for e in entries]
            seen.update(("key", key) for key in keys)
            if len(set(keys)) < len(keys):
                seen.add("duplicate")
            if "topics" in keys:
                seen.add(("case A topics", len(entries[keys.index("topics")][3]) // 32))
            else:
                seen.add(("case B topics", sum(1 for t in ("t1", "t2", "t3", "t4") if t in keys)))
            for flags, key, codec, value in entries:
                if flags != 3 or codec != 0x55:
                    seen.add("odd codec or flags")
                if len(value) >= 256:
                    seen.add("2-byte length")
    d = ts.as_dict()
    big_selected = sum(1 for raw in (d[bytes(ts.events_roots[i])] for i in ts.selected.tolist()) if len(raw) > 4096 and not cbor2.loads(raw)[3][1])
    want = {("head", h) for h in (0, 1, 2, 4, 8)} | {("case A topics", n) for n in range(5)} | {("case B topics", n) for n in range(1, 5)}
    want |= {("key", k) for k in ("t1", "t2", "t3", "t4", "d", "topics", "data", "t5", "dat")} | {"duplicate", "odd codec or flags", "2-byte length"}
    assert want <= seen, want - seen
    assert empty > 0 and big_selected > 0
    if ts.params.events_per_receipt > 32:
        assert linked > 0 and big_selected >= 20


def oracle_mod_verify(ts):
    import oracle
    return oracle.Store.from_tipset(ts).verify_cids(threads=2) is None


# ------------------------------------------------------------------ oracle vs golden (independent Python oracle)
def test_oracle_matches_golden_events(oracle_mod):
    z, ts, _ = golden_util.load()
    st = oracle_mod.Store.from_tipset(ts)
    r = st.generate_event_proof(ts, A.make_event_spec(ts.event_signature, ts.topic1, None))
    golden_util.check_event_result(z, r)


def test_oracle_matches_golden_storage(oracle_mod):
    z, _, s = golden_util.load()
    st = oracle_mod.Store.from_tipset(s)
    specs = [(int(a), z["s_slot"][k].tobytes()) for k, a in enumerate(z["s_actor"])]
    golden_util.check_storage_result(z, st.generate_storage_proofs(s, specs))


@pytest.mark.parametrize("cfg", [1, 2, "shapes", "shapes-nofilter"])
def test_oracle_vs_python_oracle(oracle_mod, synth_mod, cfg):
    from oracle import pyoracle as P
    ts = synth_tipset(synth_mod, cfg)
    r = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
    pr = P.generate_event_proof(ts.as_dict(), ts, ts.event_signature, ts.topic1, ts.actor_filter)
    assert pr["matching"] == r.matching.tolist() == ts.selected.tolist()
    assert [bytes(c) for c in r.witness.cids] == pr["witness"]
    assert [(p.exec_index, p.event_index, p.emitter, tuple(p.topics), p.data, p.message_cid) for p in r.proofs] == pr["proofs"]
    assert r.n_exec == len(pr["exec_order"])


def test_oracle_threads_and_order_independent(oracle_mod, ts2):
    st = oracle_mod.Store.from_tipset(ts2)
    a = st.generate_event_proof(ts2, spec_of(ts2), threads=1)
    b = st.generate_event_proof(ts2, spec_of(ts2), threads=4)
    assert_event_results_equal(a, b)
    sh = ShuffledTipset(ts2, seed=11, misalign=True)
    c = oracle_mod.Store.from_tipset(sh).generate_event_proof(sh, spec_of(sh))
    assert_event_results_equal(a, c)


# ------------------------------------------------------------------ generate → verify closed loop, minimality
def test_verify_and_minimality(oracle_mod, ts1):
    st = oracle_mod.Store.from_tipset(ts1)
    spec = spec_of(ts1)
    r = st.generate_event_proof(ts1, spec)
    assert len(r.proofs) > 0 and all(oracle_mod.verify_event_proofs(r.witness, ts1, r, spec))
    # dropping ANY witness block must break verification of at least one proof (or raise "missing")
    w = r.witness
    for drop in range(w.n_blocks):
        keep = [i for i in range(w.n_blocks) if i != drop]
        w2 = A.WitnessPy(w.cids[keep], w.offsets[keep], w.lengths[keep], w.blob)
        try:
            ok = oracle_mod.verify_event_proofs(w2, ts1, r, spec)
        except A.IpcfpError:
            continue
        assert not all(ok), f"witness block {drop} is not needed"
    # a tampered claim must fail
    r.raw_proofs = r.raw_proofs.copy()
    r.raw_proofs[8] ^= 1  # event_index of proof 0
    assert not oracle_mod.verify_event_proofs(w, ts1, r, spec)[0]


def test_storage_verify(oracle_mod, ts3_small):
    ts = ts3_small
    st = oracle_mod.Store.from_tipset(ts)
    n = int(ts.params.hamt_entries)
    slots = [oracle_mod.compute_mapping_slot(ts.storage_entry(k)[0], 0) for k in (0, 5, n)] + [oracle_mod.compute_mapping_slot(ts.storage_absent_key(3), 0)]
    specs = [(a, s) for a in (1001, 1002, 1003, 1004, 1005, 1006) for s in slots]
    r = st.generate_storage_proofs(ts, specs)
    assert all(oracle_mod.verify_storage_proofs(r.witness, ts, r))
    v = ts.storage_entry(5)[1]
    assert r.proofs[1].found and r.proofs[1].value == bytes(32 - len(v)) + v
    assert not r.proofs[3].found and r.proofs[3].value == bytes(32)
    assert r.proofs[2].value == bytes(31) + b"\x0f"       # the calib-subnet-1 nonce entry
    # inline small maps only hold entries 0..2: entry 5 is absent there
    assert not r.proofs[2 * 4 + 1].found
    with pytest.raises(A.IpcfpError) as ei:
        st.generate_storage_proofs(ts, [(999999, slots[0])])
    assert ei.value.status == A.ERR_ACTOR_NOT_FOUND


# ------------------------------------------------------------------ reference semantics (SURVEY Appendix B traps)
def _patched(ts, cid, new_bytes):
    """Tipset whose block `cid` is replaced by new_bytes (same CID: the engine does not re-hash unless asked)."""
    idx = [i for i in range(ts.n_blocks) if bytes(ts.cids[i]) == bytes(cid)][0]
    blob = np.concatenate([ts.blob, np.frombuffer(bytes(new_bytes) + bytes(32), dtype=np.uint8)])
    offs = ts.offsets.copy()
    lens = ts.lengths.copy()
    offs[idx] = len(ts.blob)
    lens[idx] = len(new_bytes)
    return EditedTipset(ts, blob=blob, offsets=offs, lengths=lens)


def test_error_semantics(oracle_mod, ts1):
    spec = spec_of(ts1)
    base = oracle_mod.Store.from_tipset(ts1).generate_event_proof(ts1, spec)
    # B-1: a receipt without events root is skipped entirely
    has = ts1.has_events_root.copy()
    victim = int(base.matching[0])
    has[victim] = 0
    r = oracle_mod.Store.from_tipset(ts1).generate_event_proof(EditedTipset(ts1, has_events_root=has), spec)
    assert victim not in r.matching.tolist() and len(r.matching) == len(base.matching) - 1
    # missing events-AMT block → MISSING_BLOCK at that receipt
    keep = [i for i in range(ts1.n_blocks) if bytes(ts1.cids[i]) != bytes(ts1.events_roots[5])]
    e = EditedTipset(ts1, cids=ts1.cids[keep], offsets=ts1.offsets[keep], lengths=ts1.lengths[keep], n_blocks=len(keep))
    with pytest.raises(A.IpcfpError) as ei:
        oracle_mod.Store.from_tipset(e).generate_event_proof(e, spec)
    assert (ei.value.status, ei.value.index) == (A.ERR_MISSING_BLOCK, 5)
    # trailing byte after a node → DECODE at that receipt (strict decoder)
    blk = ts1.as_dict()[bytes(ts1.events_roots[9])]
    p = _patched(ts1, ts1.events_roots[9], blk + b"\x00")
    with pytest.raises(A.IpcfpError) as ei:
        oracle_mod.Store.from_tipset(p).generate_event_proof(p, spec)
    assert (ei.value.status, ei.value.index) == (A.ERR_DECODE, 9)
    # B-4: execution order shorter than a matching index → MISSING_EXEC (checked before the receipt get)
    # (drop the last parent block's TxMeta from the descriptor: fewer messages than receipts)
    e2 = EditedTipset(ts1, parent_cids=ts1.parent_cids[:1], parent_txmeta_cids=ts1.parent_txmeta_cids[:1], n_parents=1)
    with pytest.raises(A.IpcfpError) as ei:
        oracle_mod.Store.from_tipset(e2).generate_event_proof(e2, spec)
    assert ei.value.status == A.ERR_MISSING_EXEC and ei.value.index >= 32


def test_extract_evm_log_traps(oracle_mod, synth_mod):
    """Appendix B-6: duplicate keys (last wins), `topics` beats t1, bad tK length voids the log, gaps stop the walk."""
    from oracle import pyoracle as P
    t0 = P.keccak256(b"NewTopDownMessage(bytes32,uint256)")
    t1 = P.ascii_to_bytes32("calib-subnet-1")
    other = bytes(32)
    E = lambda k, v: [3, k, 0x55, v]  # noqa: E731
    events = [
        [1001, [E("t1", other), E("t2", t1), E("t1", t0)]],                 # 0 duplicate t1: last wins → match
        [1001, [E("t1", t0), E("t1", other), E("t2", t1)]],                 # 1 last t1 is wrong → no match
        [1001, [E("topics", t0 + t1), E("t1", other), E("data", b"xy")]],    # 2 Case A wins → match
        [1001, [E("topics", (t0 + t1)[:63]), E("t1", t0), E("t2", t1)]],     # 3 Case A bad length → None
        [1001, [E("t1", t0), E("t2", t1), E("t3", b"short")]],               # 4 bad t3 voids the whole log
        [1001, [E("t1", t0), E("t2", t1), E("t4", b"short")]],               # 5 t3 missing → t4 ignored → match
        [1001, [E("t2", t1), E("d", b"")]],                                   # 6 no t1 → None
        [1001, [E("t1", t0)]],                                                # 7 one topic only → no match
        [1002, [E("t1", t0), E("t2", t1)]],                                   # 8 wrong emitter
        [1001, [E("t1", t0), E("t2", t1), E("t3", other), E("t4", other), E("d", bytes(range(40)))]],  # 9 four topics + data → match
    ]
    ts = _custom_events_tipset(synth_mod, events)
    r = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, A.make_event_spec("NewTopDownMessage(bytes32,uint256)", "calib-subnet-1", 1001))
    assert [p.event_index for p in r.proofs] == [0, 2, 5, 9]
    assert r.proofs[1].data == b"xy" and len(r.proofs[3].topics) == 4 and r.proofs[3].data == bytes(range(40))
    pr = P.generate_event_proof(dict_of(ts), ts, "NewTopDownMessage(bytes32,uint256)", "calib-subnet-1", 1001)
    assert [(p.exec_index, p.event_index, p.emitter, tuple(p.topics), p.data, p.message_cid) for p in r.proofs] == pr["proofs"]


def _custom_events_tipset(synth_mod, events, n_receipts=9, target=4):
    """A small synthetic tipset whose receipt `target` gets a hand-made events AMT (bit width 5, one node)."""
    from oracle import pyoracle as P
    ts = synth_mod.Tipset(synth_mod.default_params(seed=5, n_receipts=n_receipts, events_per_receipt=2, match_ppm=0, n_parents=1, dup_msgs=0))
    n = len(events)
    bmap = bytearray(4)
    for i in range(n):
        bmap[i // 8] |= 1 << (i % 8)
    root = cbor2.dumps([5, 0, n, [bytes(bmap), [], events]])
    cid = P.cid_of(root)
    # new events root for `target` → the receipts AMT leaf must change too; rebuild leaf + root by hand
    d = ts.as_dict()
    rr = cbor2.loads(d[bytes(ts.receipts_root)])
    height, count, node = rr
    assert height == 1 and count == n_receipts
    leaf_links = node[1]
    leaf0 = cbor2.loads(d[P._link(leaf_links[target // 8])])
    leaf0[2][target % 8][3] = cbor2.CBORTag(42, b"\x00" + cid)
    leaf0_b = cbor2.dumps(leaf0)
    leaf_links[target // 8] = cbor2.CBORTag(42, b"\x00" + P.cid_of(leaf0_b))
    root_b = cbor2.dumps([height, count, node])
    new_root_cid = P.cid_of(root_b)
    # child header points at the receipts root: patch field 9 and re-hash the header
    hdr = cbor2.loads(d[bytes(ts.child_cid)])
    hdr[9] = cbor2.CBORTag(42, b"\x00" + new_root_cid)
    hdr_b = cbor2.dumps(hdr)
    extra = [(cid, root), (P.cid_of(leaf0_b), leaf0_b), (new_root_cid, root_b), (P.cid_of(hdr_b), hdr_b)]
    blob = bytearray(ts.blob.tobytes())
    cids, offs, lens = [ts.cids], list(ts.offsets), list(ts.lengths)
    for c, b in extra:
        while len(blob) % 16:
            blob.append(0)
        offs.append(len(blob))
        lens.append(len(b))
        blob += b
        cids.append(np.frombuffer(c, dtype=np.uint8).reshape(1, 38))
    blob += bytes(32)
    roots = ts.events_roots.copy()
    roots[target] = np.frombuffer(cid, dtype=np.uint8)
    return EditedTipset(ts, cids=np.concatenate(cids), offsets=np.array(offs, dtype=np.uint64), lengths=np.array(lens, dtype=np.uint32),
                        blob=np.frombuffer(bytes(blob), dtype=np.uint8), n_blocks=len(lens), events_roots=roots,
                        receipts_root=np.frombuffer(new_root_cid, dtype=np.uint8), child_cid=np.frombuffer(P.cid_of(hdr_b), dtype=np.uint8))


def test_cid_ordering(oracle_mod):
    from oracle import pyoracle as P
    rng = np.random.default_rng(3)
    cids = []
    for k in range(200):
        prefix = [bytes([1, 0x71, 0xa0, 0xe4, 2, 0x20]), bytes([1, 0x55, 0xa0, 0xe4, 2, 0x20]), bytes([1, 0x71, 0x92, 0xe4, 2, 0x20])][k % 3]
        cids.append(prefix + rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
    cids += cids[:10]
    got = oracle_mod.sort_unique_cids(np.frombuffer(b"".join(cids), dtype=np.uint8))
    exp = sorted(set(cids), key=P.cid_sort_key)
    assert [bytes(c) for c in got] == exp


# ------------------------------------------------------------------ the C-ABI library
def test_abi_exports_match_header():
    hdr = open(os.path.join(ROOT, "include", "ipcfp.h")).read()
    declared = set(re.findall(r"\b(ipcfp_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"ipcfp_store", "ipcfp_tipset"}
    from ipc_filecoin_proofs_b200 import api
    L = api.lib()
    missing = [name for name in sorted(declared) if not hasattr(L, name)]
    assert not missing, missing
    assert set(api.EXPORTS) <= declared


def test_no_cpu_fallback(api, ts1):
    """Without a CUDA device every compute entry point fails loudly (IPCFP_ERR_NO_DEVICE)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(A.IpcfpError) as ei:
        api.BlockStore.from_tipset(ts1)
    assert ei.value.status == A.ERR_NO_DEVICE
    with pytest.raises(A.IpcfpError) as ei:
        api.keccak256_batch([b"abc"])
    assert ei.value.status == A.ERR_NO_DEVICE
    assert api.lib().ipcfp_version().decode().startswith("ipcfp-b200")


def test_product_does_not_link_oracle():
    """The product library and package never reference oracle/ or synth/."""
    import subprocess
    from ipc_filecoin_proofs_b200 import api
    out = subprocess.run(["ldd", api.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle" not in out and "synth" not in out
    syms = subprocess.run(["nm", "-D", api.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle_" not in syms and "synth_" not in syms
    pkg = os.path.join(ROOT, "ipc_filecoin_proofs_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "oracle/" not in txt.replace("oracle/__init__.py", ""), f


def test_oracle_vs_python_oracle_config4_shape(oracle_mod, synth_mod):
    """The two independent oracle implementations on a config-4-SHAPED tipset at 100 k receipts (0.1 % match, events-AMT bit widths 3/5
    mixed, duplicate messages, 5-level receipts AMT) — VERDICT r1: the cross-check used to stop at configs 1-2."""
    from oracle import pyoracle as P
    ts = synth_mod.Tipset(synth_mod.config_params(4, n_receipts=100_000))
    r = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts), threads=4)
    pr = P.generate_event_proof(ts.as_dict(), ts, ts.event_signature, ts.topic1, ts.actor_filter)
    assert pr["matching"] == r.matching.tolist() == ts.selected.tolist() and len(pr["matching"]) > 20
    assert [bytes(c) for c in r.witness.cids] == pr["witness"]
    assert [(p.exec_index, p.event_index, p.emitter, tuple(p.topics), p.data, p.message_cid) for p in r.proofs] == pr["proofs"]
    assert r.n_exec == len(pr["exec_order"])


def test_oracle_vs_python_oracle_full_size_hamt(oracle_mod, synth_mod):
    """Both oracles on the FULL-SIZE storage tree of configs[2] (1 M slots): 300 lookups (present, absent, the six root shapes)."""
    from oracle import pyoracle as P
    ts = synth_mod.Tipset(synth_mod.config_params(3))
    st = oracle_mod.Store.from_tipset(ts)
    store = ts.as_dict()
    rng = np.random.default_rng(11)
    keys = [ts.storage_entry(int(k))[0] for k in rng.choice(1_000_000, size=270, replace=False)] + [ts.storage_absent_key(k) for k in range(30)]
    slots = [oracle_mod.compute_mapping_slot(k, 0) for k in keys]
    got = st.read_storage_slots(ts.storage_root, np.frombuffer(b"".join(slots), dtype=np.uint8))
    rec = P.Recorder(store)
    for i, s in enumerate(slots):
        v = P.read_storage_slot(rec, bytes(ts.storage_root), s)
        assert bool(got.found[i]) == (v is not None)
        if v is not None:
            assert bytes(got.values[i]) == bytes(32 - len(v)) + v if len(v) <= 32 else v[-32:]
    assert sorted(rec.seen) == sorted(bytes(c) for c in got.witness.cids)
    specs = [(a, slots[k]) for k, a in enumerate((1001, 1002, 1003, 1004, 1005, 1006))]
    r = st.generate_storage_proofs(ts, specs)
    for (a, s), p in zip(specs, r.proofs):
        pp = P.generate_storage_proof(store, ts, a, s)
        assert (p.actor_state_cid, p.storage_root, p.value) == (pp["actor_state_cid"], pp["storage_root"], pp["value"])


# Constants of the public Filecoin chain — NOT taken from the reference tree (which holds no vectors); any Filecoin node or block explorer
# shows them: the `Messages` CID of every block header without messages (MsgMeta/TxMeta over two empty v0 AMTs), builtin-actors'
# `EMPTY_ARR_CID` (empty AMT v3, bit width 3) and the empty HAMT node (the "empty map" of actor state).
FILECOIN_EMPTY_TXMETA = "bafy2bzacecmda75ovposbdateg7eyhwij65zklgyijgcjwynlklmqazpwlhba"
FILECOIN_EMPTY_ARR = "bafy2bzacedijw74yui7otvo63nfl3hdq2vdzuy7wx2tnptwed6zml4vvz7wee"
FILECOIN_EMPTY_HAMT = "bafy2bzaceamp42wmmgr2g2ymg46euououzfyck7szknvfacqscohrvaikwfay"
EMPTY_AMT_V0 = bytes([0x83, 0x00, 0x00, 0x83, 0x41, 0x00, 0x80, 0x80])            # [height 0, count 0, [bmap h'00', [], []]]
EMPTY_AMT_V3 = bytes([0x84, 0x03, 0x00, 0x00, 0x83, 0x41, 0x00, 0x80, 0x80])      # [bit_width 3, height 0, count 0, node]
EMPTY_HAMT_NODE = bytes([0x82, 0x40, 0x80])                                       # [bitfield h'', []]


def test_public_filecoin_constants_pin_the_encodings(oracle_mod, synth_mod):
    """External known answers for the [UPSTREAM] encodings the whole path rests on (DESIGN.md §3/§7): DAG-CBOR tuples and links,
    AMT v0 / v3 root and node layout, the HAMT node layout, Blake2b-256 CIDv1 (dag-cbor) and its base32 spelling. Three independent
    implementations must land on the chain's own constants: hashlib + the Python helpers, the C++ oracle's hash, and the synthetic
    tipset builder (whose blocks are what every parity test feeds to the engine)."""
    from ipc_filecoin_proofs_b200 import bundle_json as J
    from oracle import pyoracle as P
    import cbor2

    def link(c):
        return bytes([0xd8, 0x2a, 0x58, 0x27, 0x00]) + c

    cid_v0, cid_v3, cid_h = P.cid_of(EMPTY_AMT_V0), P.cid_of(EMPTY_AMT_V3), P.cid_of(EMPTY_HAMT_NODE)
    txmeta = bytes([0x82]) + link(cid_v0) + link(cid_v0)
    assert J.cid_to_string(P.cid_of(txmeta)) == FILECOIN_EMPTY_TXMETA
    assert J.cid_to_string(cid_v3) == FILECOIN_EMPTY_ARR
    assert J.cid_to_string(cid_h) == FILECOIN_EMPTY_HAMT
    assert J.cid_from_string(FILECOIN_EMPTY_TXMETA) == P.cid_of(txmeta)
    # the C++ oracle's Blake2b agrees on the same bytes
    for blk in (EMPTY_AMT_V0, EMPTY_AMT_V3, EMPTY_HAMT_NODE, txmeta):
        assert bytes(oracle_mod.blake2b256(blk)) == P.cid_of(blk)[6:]
    # the decoders read these blocks as what they are: empty AMTs (both versions), an empty HAMT node
    store = {cid_v0: EMPTY_AMT_V0, cid_v3: EMPTY_AMT_V3, cid_h: EMPTY_HAMT_NODE, P.cid_of(txmeta): txmeta}
    for cid, ver in ((cid_v0, 0), (cid_v3, 3)):
        amt = P.Amt(cid, P.Recorder(store), ver)
        seen = []
        amt.for_each(lambda i, v: seen.append(i))
        assert (amt.bw, amt.height, amt.count, seen) == (3, 0, 0, []) and amt.get(0) is None
    assert P.hamt_get(P.Recorder(store), cid_h, 5, bytes(32)) is None
    assert [bytes(t.value) for t in cbor2.loads(txmeta)] == [bytes([0]) + cid_v0] * 2
    # the synthetic tipset builder emits exactly the chain's constant for a parent block without messages …
    ts = synth_mod.Tipset(synth_mod.default_params(seed=1, n_receipts=1, n_parents=3))
    tx = [J.cid_to_string(bytes(t)) for t in np.asarray(ts.parent_txmeta_cids, dtype=np.uint8).reshape(-1, 38)]
    assert tx.count(FILECOIN_EMPTY_TXMETA) == 2
    blocks = ts.as_dict()
    assert blocks[J.cid_from_string(FILECOIN_EMPTY_TXMETA)] == txmeta and blocks[cid_v0] == EMPTY_AMT_V0
    # … and both oracles walk such a tipset to the same answer (the empty AMTs are recorded into the witness like any other block)
    spec = spec_of(ts)
    r = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec)
    wit = {bytes(c) for c in r.witness.cids}
    assert J.cid_from_string(FILECOIN_EMPTY_TXMETA) in wit and cid_v0 in wit


# Public Solidity storage-layout vectors (docs.soliditylang.org "Layout of State Variables in Storage": the value of mapping key k
# at slot p lives at keccak256(h(k) . p); a dynamic array at slot p starts at keccak256(p)) — not from the reference tree, which holds no
# vectors; any EVM toolchain prints them. They pin compute_mapping_slot (storage/utils.rs:5-12: keccak256(key32 ‖ u256_be(slot_index)))
# and the Keccak-256 (not SHA3-256) padding against the real EVM rather than against ourselves.
SOLIDITY_SLOT_VECTORS = [
    # (key32, slot index, keccak256(key32 ‖ u256(slot)))
    (bytes(32), 0, "ad3228b676f7d3cd4284a5443f17f1962b36e491b30a40b2405849e597ba5fb5"),
    (bytes(32), 1, "a6eef7e35abe7026729641147f7915573c7e97b47efa546f5f6e3230263bcb49"),
    (bytes(31) + b"\x01", 0, "ada5013122d395ba3c54772283fb069b10426056ef8ca54750cb9bb552a59e7d"),
]
SOLIDITY_ARRAY_VECTORS = [
    (bytes(32), "290decd9548b62a8d60345a988386fc84ba6bc95484008f6362f93160ef3e563"),              # keccak256(uint256(0))
    (bytes(31) + b"\x01", "b10e2d527612073b26eecdfd717e6a320cf44b4afac2b0732d9fcbe2b7fa0cf6"),    # keccak256(uint256(1))
]


def test_public_solidity_storage_layout_vectors(oracle_mod, synth_mod):
    from oracle import pyoracle as P
    for key, idx, want in SOLIDITY_SLOT_VECTORS:
        assert oracle_mod.compute_mapping_slot(key, idx).hex() == want
        assert P.keccak256(key + idx.to_bytes(32, "big")).hex() == want
    for msg, want in SOLIDITY_ARRAY_VECTORS:
        assert oracle_mod.keccak256(msg).hex() == P.keccak256(msg).hex() == synth_mod.keccak256(msg).hex() == want


def test_public_filecoin_id_address_bytes():
    """ID addresses (protocol 0) are `0x00 ‖ unsigned-LEB128(id)` — Filecoin spec, "Address" appendix; f01000 is 00 e8 07 on any node.
    This is the state-tree HAMT key of get_actor_state (common/decode.rs:34, storage/generator.rs:116)."""
    from oracle import pyoracle as P
    assert P._id_address(0) == bytes.fromhex("0000")
    assert P._id_address(127) == bytes.fromhex("007f")
    assert P._id_address(128) == bytes.fromhex("008001")
    assert P._id_address(1000) == bytes.fromhex("00e807")
    assert P._id_address(2**64 - 1) == bytes.fromhex("00" + "ff" * 9 + "01")


def test_keccak_vectors_held_by_the_reference_tree(oracle_mod, synth_mod):
    """The only known answers in the reference tree that pin something the hot path computes: Keccak-256 constants of the vendored
    forge-std (cheat-code / default-sender addresses, hashInitCode(hex"6080"), CREATE / CREATE2 addresses, a function selector, the
    EIP-55 checksums of its address literals) — tests/golden/reference_keccak_vectors.json, extracted by
    tests/golden/make_reference_keccak_vectors.py. Checked here with the three CPU implementations; the GPU kernel has its own test."""
    from oracle import pyoracle as P
    from tests.golden_util import check_reference_keccak_vectors
    for impl in (oracle_mod.keccak256, P.keccak256, synth_mod.keccak256):
        assert check_reference_keccak_vectors(impl) >= 20
