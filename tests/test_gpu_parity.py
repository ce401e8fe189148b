"""GPU parity tests: the CUDA path through the C ABI vs the CPU oracle (bit-exact)."""
import hashlib

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests.util import ShuffledTipset, assert_event_results_equal, assert_witness_equal, spec_of, synth_tipset

pytestmark = pytest.mark.gpu

LENS = [0, 1, 2, 31, 32, 55, 56, 63, 64, 65, 111, 112, 127, 128, 129, 135, 136, 137, 255, 256, 257, 271, 272, 273, 1027, 1028, 1029, 4096, 5000]


def _msgs():
    rng = np.random.default_rng(1)
    return [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in LENS]


def test_blake2b_batch(api):
    msgs = _msgs()
    got = api.blake2b256_batch(msgs)
    assert got == [hashlib.blake2b(m, digest_size=32).digest() for m in msgs]
    assert got[0].hex() == "0e5751c026e543b2e8ab2eb06099daa1d1e5df47778f7787faab45cdf12fe3a8"


def test_sha256_batch(api):
    msgs = _msgs()
    assert api.sha256_batch(msgs) == [hashlib.sha256(m).digest() for m in msgs]


def test_keccak_batch(api, oracle_mod):
    msgs = _msgs() + [b"Transfer(address,address,uint256)", b"NewTopDownMessage(bytes32,uint256)"]
    got = api.keccak256_batch(msgs)
    assert got == [oracle_mod.keccak256(m) for m in msgs]
    assert got[0].hex() == "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"
    assert got[-2].hex() == "ddf252ad1be2c89b69c2b068fc378daa952ba7f163c4a11628f55a4df523b3ef"


def test_mapping_slots(api, oracle_mod):
    keys = [bytes([i]) * 32 for i in range(5)] + [b"calib-subnet-1" + bytes(18)]
    idx = [0, 1, 2, 2**40, 2**64 - 1, 0]
    got = api.compute_mapping_slots(keys, idx)
    assert got == [oracle_mod.compute_mapping_slot(k, i) for k, i in zip(keys, idx)]
    assert api.calculate_storage_slot("calib-subnet-1", 0) == got[-1]


def test_store_get_has_verify(api, ts1):
    st = api.BlockStore.from_tipset(ts1, verify_cids=True)
    for i in (0, 5, ts1.n_blocks - 1):
        assert st.get(ts1.cids[i]) == ts1.block(i)
        assert st.has(ts1.cids[i])
    assert st.get(np.zeros(38, dtype=np.uint8)) is None
    assert not st.has(bytes([1, 0x71, 0xa0, 0xe4, 2, 0x20]) + bytes(32))
    # corrupt one byte of one block → CID mismatch at that block
    blob = ts1.blob.copy()
    victim = 17
    blob[int(ts1.offsets[victim]) + 3] ^= 0x40
    with pytest.raises(A.IpcfpError) as ei:
        api.BlockStore(ts1.cids, ts1.offsets, ts1.lengths, blob, verify_cids=True)
    assert ei.value.status == A.ERR_CID_MISMATCH and ei.value.index == victim


@pytest.mark.parametrize("cfg", [1, 2])
def test_event_proof_parity(api, oracle_mod, synth_mod, cfg):
    ts = synth_mod.Tipset(synth_mod.config_params(cfg))
    exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
    got = api.BlockStore.from_tipset(ts, verify_cids=True).generate_event_proof(ts, spec_of(ts))
    assert_event_results_equal(got, exp)
    assert got.matching.tolist() == ts.selected.tolist()
    assert all(oracle_mod.verify_event_proofs(got.witness, ts, got, spec_of(ts)))


@pytest.mark.parametrize("kw", [
    dict(n_receipts=300, events_per_receipt=40, match_ppm=100000),                       # two-level events AMTs (bw 5) / three-level (bw 3)
    dict(n_receipts=500, events_per_receipt=3, null_root_permille=200, match_ppm=200000),  # receipts without events root
    dict(n_receipts=257, events_per_receipt=8, bw3_permille=1000, match_ppm=50000, has_actor_filter=0),
    dict(n_receipts=1000, events_per_receipt=8, case_a_permille=500, malformed_permille=100, match_ppm=30000),
    dict(n_receipts=1, events_per_receipt=1, match_ppm=1000000, dup_msgs=0, n_parents=1),
    dict(n_receipts=9, events_per_receipt=8, match_ppm=0, n_parents=3, dup_msgs=2),
    dict(n_receipts=700, events_per_receipt=300, match_ppm=20000, n_parents=1),             # bw-3 AMTs of height 2
    # varied event shapes (synth event_shapes = 1): single-node roots over 4 KB and roots with links, events larger than pass 1's ring
    dict(event_shapes=1, n_receipts=600, events_per_receipt=40, match_ppm=300000),
    dict(event_shapes=1, n_receipts=500, events_per_receipt=12, match_ppm=300000, has_actor_filter=0, bw3_permille=300, null_root_permille=50),
    dict(event_shapes=1, n_receipts=300, events_per_receipt=40, match_ppm=200000, target_actor=65536 + 7, bw3_permille=500),
    # N on either side of the single-CTA scan of pass 1's counts (16 384)
    dict(event_shapes=1, n_receipts=16384, events_per_receipt=6, match_ppm=60000, null_root_permille=20),
    dict(event_shapes=1, n_receipts=16385, events_per_receipt=6, match_ppm=60000, has_actor_filter=0, n_parents=3),
])
def test_event_proof_shapes(api, oracle_mod, synth_mod, kw):
    ts = synth_mod.Tipset(synth_mod.default_params(seed=99, **kw))
    exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
    got = api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
    assert_event_results_equal(got, exp)
    if kw.get("event_shapes"):
        assert got.matching.tolist() == ts.selected.tolist() and len(got.proofs) == len(ts.selected) > 0


def test_event_proof_block_order_and_alignment(api, oracle_mod, synth_mod, ts2):
    for ts in (ts2, synth_tipset(synth_mod, "shapes")):
        exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
        for layout in (dict(misalign=False), dict(misalign=True), dict(roots_mod128=True)):
            sh = ShuffledTipset(ts, seed=3, **layout)
            got = api.BlockStore.from_tipset(sh, verify_cids=True).generate_event_proof(sh, spec_of(sh))
            assert_event_results_equal(got, exp)


def test_skip_tx_flag(api, oracle_mod, ts2):
    exp = oracle_mod.Store.from_tipset(ts2).generate_event_proof(ts2, spec_of(ts2), flags=A.SCAN_SKIP_TX_AMTS)
    got = api.BlockStore.from_tipset(ts2).generate_event_proof(ts2, spec_of(ts2), flags=A.SCAN_SKIP_TX_AMTS)
    assert_event_results_equal(got, exp)


def test_storage_slots_parity(api, oracle_mod, ts3_small):
    ts = ts3_small
    n = int(ts.params.hamt_entries)
    rng = np.random.default_rng(5)
    ks = rng.integers(0, n, 900).tolist() + [n]
    keys = [ts.storage_entry(k)[0] for k in ks] + [ts.storage_absent_key(k) for k in range(100)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    slots_np = np.frombuffer(b"".join(slots), dtype=np.uint8)
    exp = oracle_mod.Store.from_tipset(ts).read_storage_slots(ts.storage_root, slots_np)
    got = api.BlockStore.from_tipset(ts, verify_cids=True).read_storage_slots(ts.storage_root, slots_np)
    assert np.array_equal(got.found, exp.found) and np.array_equal(got.raw_len, exp.raw_len) and np.array_equal(got.values, exp.values)
    assert_witness_equal(got.witness, exp.witness)
    assert got.found[:901].all() and not got.found[901:].any()
    for i, k in enumerate(ks[:50]):
        v = ts.storage_entry(k)[1]
        assert bytes(got.values[i][32 - len(v):]) == v


@pytest.mark.parametrize("strict", [None, "1"])
@pytest.mark.parametrize("k", [1000, 16384, 16385])   # one lookup per warp up to 16 384, one per thread (strict decoder) above
def test_storage_slots_parity_lookup_counts(api, oracle_mod, ts3_small, monkeypatch, k, strict):
    """Present, duplicate and absent keys in shuffled order, on both sides of k_read_slots' per-warp / per-thread switch, with the
    strict HAMT decoder forced or not: found flags, raw lengths, values and witness equal the oracle's."""
    if strict is None:
        monkeypatch.delenv("IPCFP_HAMT_STRICT", raising=False)
    else:
        monkeypatch.setenv("IPCFP_HAMT_STRICT", strict)
    ts = ts3_small
    n = int(ts.params.hamt_entries)
    rng = np.random.default_rng(5 + k)
    n_absent, n_dup = k // 10, k // 20
    ks = rng.integers(0, n, k - n_absent - n_dup - 1).tolist() + [n]
    ks += rng.choice(ks, n_dup).tolist()                                          # duplicate keys
    keys = [ts.storage_entry(e)[0] for e in ks] + [ts.storage_absent_key(e) for e in range(n_absent)]
    present = np.array([True] * len(ks) + [False] * n_absent)
    order = rng.permutation(k)
    keys, present = [keys[i] for i in order], present[order]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    slots_np = np.frombuffer(b"".join(slots), dtype=np.uint8)
    exp = oracle_mod.Store.from_tipset(ts).read_storage_slots(ts.storage_root, slots_np)
    got = api.BlockStore.from_tipset(ts, verify_cids=True).read_storage_slots(ts.storage_root, slots_np)
    assert len(got.found) == k
    assert np.array_equal(got.found, exp.found) and np.array_equal(got.raw_len, exp.raw_len) and np.array_equal(got.values, exp.values)
    assert_witness_equal(got.witness, exp.witness)
    assert np.array_equal(got.found.astype(bool), present)
    for pos in np.nonzero(present)[0][:50]:
        v = ts.storage_entry(ks[order[pos]])[1]
        assert bytes(got.values[pos][32 - len(v):]) == v


def test_storage_proofs_parity(api, oracle_mod, ts3_small):
    ts = ts3_small
    n = int(ts.params.hamt_entries)
    keys = [ts.storage_entry(k)[0] for k in (0, 1, 2, 77, n)] + [ts.storage_absent_key(1)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    specs = [(actor, s) for actor in (1001, 1002, 1003, 1004, 1005, 1006) for s in slots]
    exp = oracle_mod.Store.from_tipset(ts).generate_storage_proofs(ts, specs)
    got = api.BlockStore.from_tipset(ts).generate_storage_proofs(ts, specs)
    assert [vars(p) for p in got.proofs] == [vars(p) for p in exp.proofs]
    assert_witness_equal(got.witness, exp.witness)
    assert got.spec_witness == exp.spec_witness
    assert all(oracle_mod.verify_storage_proofs(got.witness, ts, got))


def test_bundle_parity(api, oracle_mod, ts3_small):
    ts = ts3_small
    slot = api.calculate_storage_slot("calib-subnet-1", 0)
    sspecs = [(1001, slot), (1003, slot)]
    especs = [A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter), A.make_event_spec(ts.event_signature, "calib-subnet-2", None)]
    exp = oracle_mod.Store.from_tipset(ts).generate_proof_bundle(ts, sspecs, especs)
    got = api.BlockStore.from_tipset(ts).generate_proof_bundle(ts, sspecs, especs)
    assert [vars(p) for p in got.storage.proofs] == [vars(p) for p in exp.storage.proofs]
    for g, e in zip(got.events, exp.events):
        assert_event_results_equal(g, e)
    assert_witness_equal(got.witness, exp.witness)


# ------------------------------------------------------------------ golden fixtures (independent Python oracle)
def test_engine_matches_golden(api):
    from tests import golden_util
    z, ts, s = golden_util.load()
    r = api.BlockStore.from_tipset(ts, verify_cids=True).generate_event_proof(ts, A.make_event_spec(ts.event_signature, ts.topic1, None))
    golden_util.check_event_result(z, r)
    specs = [(int(a), z["s_slot"][k].tobytes()) for k, a in enumerate(z["s_actor"])]
    golden_util.check_storage_result(z, api.BlockStore.from_tipset(s, verify_cids=True).generate_storage_proofs(s, specs))
    off = 0
    msgs = []
    for n in z["kat_lens"]:
        msgs.append(z["kat_msgs"][off:off + int(n)].tobytes())
        off += int(n)
    assert api.blake2b256_batch(msgs) == [x.tobytes() for x in z["kat_blake2b"]]
    assert api.sha256_batch(msgs) == [x.tobytes() for x in z["kat_sha256"]]
    assert api.keccak256_batch(msgs) == [x.tobytes() for x in z["kat_keccak"]]


# ------------------------------------------------------------------ reference semantics / error parity
def _both(api, oracle_mod, ts, spec, flags=0):
    """Runs oracle and engine; returns ('ok', result) or ('err', status, index) for each."""
    out = []
    for mk in (lambda: oracle_mod.Store.from_tipset(ts), lambda: api.BlockStore.from_tipset(ts)):
        try:
            out.append(("ok", mk().generate_event_proof(ts, spec, flags)))
        except A.IpcfpError as e:
            out.append(("err", e.status, e.index))
    return out


def test_extract_evm_log_traps_gpu(api, oracle_mod, synth_mod):
    from tests.test_oracle_cpu import _custom_events_tipset
    from oracle import pyoracle as P
    t0 = P.keccak256(b"NewTopDownMessage(bytes32,uint256)")
    t1 = P.ascii_to_bytes32("calib-subnet-1")
    other = bytes(32)
    E = lambda k, v, fl=3, codec=0x55: [fl, k, codec, v]  # noqa: E731
    events = [
        [1001, [E("t1", other), E("t2", t1), E("t1", t0)]],
        [1001, [E("t1", t0), E("t1", other), E("t2", t1)]],
        [1001, [E("topics", t0 + t1), E("t1", other), E("data", b"xy")]],
        [1001, [E("topics", (t0 + t1)[:63]), E("t1", t0), E("t2", t1)]],
        [1001, [E("t1", t0), E("t2", t1), E("t3", b"short")]],
        [1001, [E("t1", t0), E("t2", t1), E("t4", b"short")]],
        [1001, [E("t2", t1), E("d", b"")]],
        [1001, [E("t1", t0)]],
        [1002, [E("t1", t0), E("t2", t1)]],
        [1001, [E("t1", t0), E("t2", t1), E("t3", other), E("t4", other), E("d", bytes(range(40)))]],
        [1001, [E("t1", t0, fl=300), E("t2", t1, codec=0x71), E("d", bytes(300))]],                 # wide flags / other codec / 2-byte length
        [2 ** 40 + 1001, [E("t1", t0), E("t2", t1)]],                                               # 8-byte emitter
        [1001, [E("t1", t0), E("other-key-é", b"zz"), E("t2", t1), E("topic", b""), E("dat", b"")]],  # unknown / non-ASCII keys
        [1001, []],
        [1001, [E("topics", t0 + t1 + other * 5), E("data", bytes(70))]],                           # 7 topics (Case A may exceed 4)
        [1001, [E("topics", b"")]],                                                                  # Case A, zero topics → Some but no match
    ]
    ts = _custom_events_tipset(synth_mod, events)
    spec = A.make_event_spec("NewTopDownMessage(bytes32,uint256)", "calib-subnet-1", 1001)
    o, g = _both(api, oracle_mod, ts, spec)
    assert o[0] == g[0] == "ok"
    assert_event_results_equal(g[1], o[1])
    assert [p.event_index for p in g[1].proofs] == [0, 2, 5, 9, 10, 12, 14]
    assert len(g[1].proofs[6].topics) == 7
    # no actor filter: the wrong-emitter and huge-emitter events match too
    spec2 = A.make_event_spec("NewTopDownMessage(bytes32,uint256)", "calib-subnet-1", None)
    o, g = _both(api, oracle_mod, ts, spec2)
    assert_event_results_equal(g[1], o[1])
    assert [p.event_index for p in g[1].proofs] == [0, 2, 5, 8, 9, 10, 11, 12, 14]
    assert g[1].proofs[6].emitter == 2 ** 40 + 1001


def test_error_parity(api, oracle_mod, synth_mod, ts1):
    import cbor2
    from tests.test_oracle_cpu import _patched
    from tests.util import EditedTipset
    spec = spec_of(ts1)
    d = ts1.as_dict()
    cases = []
    # receipts without events root are skipped
    has = ts1.has_events_root.copy()
    has[::3] = 0
    cases.append(EditedTipset(ts1, has_events_root=has))
    # missing events block / missing receipts-AMT leaf / missing message-AMT node / missing TxMeta / missing parent header
    def without(cid):
        keep = [i for i in range(ts1.n_blocks) if bytes(ts1.cids[i]) != bytes(cid)]
        return EditedTipset(ts1, cids=ts1.cids[keep], offsets=ts1.offsets[keep], lengths=ts1.lengths[keep], n_blocks=len(keep))
    cases.append(without(ts1.events_roots[5]))
    rr = cbor2.loads(d[bytes(ts1.receipts_root)])
    cases.append(without(rr[2][1][1].value[1:]))                      # a receipts-AMT leaf on some matching path or not
    tm = cbor2.loads(d[bytes(ts1.parent_txmeta_cids[0])])
    bls_root = cbor2.loads(d[tm[0].value[1:]])
    cases.append(without(bls_root[2][1][0].value[1:]))                 # first child of the BLS message AMT
    cases.append(without(ts1.parent_txmeta_cids[1]))
    cases.append(without(ts1.parent_cids[0]))                          # base witness block missing → materialize error
    cases.append(without(ts1.receipts_root))
    # malformed blocks (same CID, different bytes: the engine does not re-hash unless IPCFP_STORE_VERIFY_CIDS is set)
    ev = d[bytes(ts1.events_roots[9])]
    for bad in (ev + b"\x00", ev[:-1], ev[:1] + b"\x06" + ev[2:], ev[:5] + b"\x45\xff\x00\x00\x00\x00" + ev[10:], b"\xa0", b"",
                ev.replace(b"\x62t1", b"\x62t\xff", 1), ev.replace(b"\x18\x55\x58\x20", b"\x18\x17\x58\x20", 1),
                ev.replace(b"\x19\x03", b"\x1a\x00\x00\x03", 1)):
        cases.append(_patched(ts1, ts1.events_roots[9], bad))
    leaf_cid = rr[2][1][0].value[1:]
    leaf = d[leaf_cid]
    cases.append(_patched(ts1, leaf_cid, leaf[:-1]))
    cases.append(_patched(ts1, leaf_cid, leaf.replace(b"\x84\x00\x40", b"\x84\x20\x40", 1)))   # negative exit code
    cases.append(_patched(ts1, ts1.parent_txmeta_cids[0], cbor2.dumps([tm[0]])))               # TxMeta with one element
    # execution order shorter than the receipts list
    cases.append(EditedTipset(ts1, parent_cids=ts1.parent_cids[:1], parent_txmeta_cids=ts1.parent_txmeta_cids[:1], n_parents=1))
    seen_err = 0
    for k, ts in enumerate(cases):
        o, g = _both(api, oracle_mod, ts, spec)
        assert o[0] == g[0], (k, o, g)
        if o[0] == "ok":
            assert_event_results_equal(g[1], o[1])
        else:
            seen_err += 1
            assert o[1:] == g[1:], (k, o, g)
    assert seen_err >= 15


def test_sparse_message_amt_takes_general_walk(api, oracle_mod, synth_mod, ts1):
    """The dense message-AMT walk (index arithmetic, one launch per level) must hand over to the general
    count → scan → expand walk when an AMT has holes or its `count` lies; results stay those of the reference."""
    import cbor2
    from tests.test_oracle_cpu import _patched
    d = ts1.as_dict()
    spec = spec_of(ts1)
    tm = cbor2.loads(d[bytes(ts1.parent_txmeta_cids[0])])
    ran = 0
    for which in (0, 1):
        root_cid = tm[which].value[1:]
        height, count, node = cbor2.loads(d[root_cid])
        cur_cid, cur, is_root = root_cid, node, True
        while cur[1]:
            cur_cid = cur[1][0].value[1:]
            cur, is_root = cbor2.loads(d[cur_cid]), False
        bmap, links, vals = cur
        if len(vals) < 2:
            continue
        for drop_first in (True, False):
            slots = [b for b in range(8) if bmap[0] >> b & 1]
            gone = slots[0] if drop_first else slots[-1]
            node2 = [bytes([bmap[0] & ~(1 << gone)]), [], vals[1:] if drop_first else vals[:-1]]
            new = cbor2.dumps([height, count, node2]) if is_root else cbor2.dumps(node2)
            o, g = _both(api, oracle_mod, _patched(ts1, cur_cid, new), spec)
            assert o[0] == g[0], (which, drop_first, o, g)
            if o[0] == "ok":
                assert_event_results_equal(g[1], o[1])
            else:
                assert o[1:] == g[1:], (which, drop_first, o, g)
            ran += 1
    assert ran >= 2


def test_general_walk_forced(api, oracle_mod, synth_mod, monkeypatch):
    """IPCFP_BFS_GENERAL=1 disables the dense walk: the general kernels alone must give the same answers."""
    monkeypatch.setenv("IPCFP_BFS_GENERAL", "1")
    for cfg in (1, 2):
        ts = synth_mod.Tipset(synth_mod.config_params(cfg))
        exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
        got = api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
        assert_event_results_equal(got, exp)


def test_receipt_missing_from_amt_is_skipped(api, oracle_mod, synth_mod):
    """events/generator.rs:249-251: r_amt.get(i) == None ⇒ `continue` (no proof, no events recording)."""
    import cbor2
    from oracle import pyoracle as P
    from tests.util import EditedTipset
    ts = synth_mod.Tipset(synth_mod.default_params(seed=21, n_receipts=40, events_per_receipt=4, match_ppm=400000, n_parents=1, dup_msgs=0))
    d = ts.as_dict()
    height, count, node = cbor2.loads(d[bytes(ts.receipts_root)])
    # drop the last leaf (receipts 32..39) from the receipts AMT root
    bmap, links, vals = node
    node2 = [bytes([bmap[0] & 0x0f]), links[:4], vals]
    root_b = cbor2.dumps([height, count, node2])
    new_root = P.cid_of(root_b)
    hdr = cbor2.loads(d[bytes(ts.child_cid)])
    hdr[9] = cbor2.CBORTag(42, b"\x00" + new_root)
    hdr_b = cbor2.dumps(hdr)
    blob = bytearray(ts.blob.tobytes())
    offs, lens, cids = list(ts.offsets), list(ts.lengths), [ts.cids]
    for c, b in ((new_root, root_b), (P.cid_of(hdr_b), hdr_b)):
        while len(blob) % 16:
            blob.append(0)
        offs.append(len(blob)); lens.append(len(b)); blob += b
        cids.append(np.frombuffer(c, dtype=np.uint8).reshape(1, 38))
    blob += bytes(32)
    e = EditedTipset(ts, cids=np.concatenate(cids), offsets=np.array(offs, dtype=np.uint64), lengths=np.array(lens, dtype=np.uint32),
                     blob=np.frombuffer(bytes(blob), dtype=np.uint8), n_blocks=len(lens), receipts_root=np.frombuffer(new_root, dtype=np.uint8),
                     child_cid=np.frombuffer(P.cid_of(hdr_b), dtype=np.uint8))
    o, g = _both(api, oracle_mod, e, spec_of(ts))
    assert o[0] == g[0] == "ok"
    assert any(i >= 32 for i in o[1].matching.tolist()) and all(p.exec_index < 32 for p in o[1].proofs)
    assert g[1].matching.tolist() == o[1].matching.tolist()
    assert [p.key() for p in g[1].proofs] == [p.key() for p in o[1].proofs]
    assert np.array_equal(g[1].witness.cids, o[1].witness.cids)


def test_storage_error_parity(api, oracle_mod, ts3_small):
    from tests.util import EditedTipset
    ts = ts3_small
    slot = api.calculate_storage_slot("calib-subnet-1", 0)

    def run(t, specs):
        out = []
        for mk in (lambda: oracle_mod.Store.from_tipset(t), lambda: api.BlockStore.from_tipset(t)):
            try:
                r = mk().generate_storage_proofs(t, specs)
                out.append(("ok", [vars(p) for p in r.proofs]))
            except A.IpcfpError as e:
                out.append(("err", e.status, e.index))
        return out
    o, g = run(ts, [(1001, slot), (424242, slot)])
    assert o == g == [("err", A.ERR_ACTOR_NOT_FOUND, 1)] * 2 or (o == g and o[0] == "err")
    wrong = EditedTipset(ts, parent_state_root=ts.child_cid)
    o, g = run(wrong, [(1001, slot)])
    assert o == g and o[0] == "err" and o[1] == A.ERR_STATE_ROOT_MISMATCH
    keep = [i for i in range(ts.n_blocks) if bytes(ts.cids[i]) != bytes(ts.storage_root)]
    e = EditedTipset(ts, cids=ts.cids[keep], offsets=ts.offsets[keep], lengths=ts.lengths[keep], n_blocks=len(keep))
    o, g = run(e, [(1003, slot), (1001, slot)])
    assert o == g and o[0] == "err" and o[1:] == (A.ERR_MISSING_BLOCK, 1)


# ------------------------------------------------------------------ BASELINE.json full sizes
def test_full_size_config4(api, oracle_mod, synth_mod):
    """1 M receipts x 8 events, 0.1 % match, AMT bit widths 3/5: bit-exact vs the oracle + size-independent properties."""
    ts = synth_mod.Tipset(synth_mod.config_params(4))
    spec = spec_of(ts)
    store = api.BlockStore.from_tipset(ts, verify_cids=True)
    d, keep = A.make_tipset_desc(ts)
    got = store.generate_event_proof(ts, spec)
    assert got.matching.tolist() == ts.selected.tolist()                # ground truth by construction
    assert got.n_exec == ts.n_receipts
    # witness: sorted, unique, every block hashes to its CID, union contains every recorded kind of block
    w = got.witness
    digs = [bytes(c[6:]) for c in w.cids]
    assert digs == sorted(set(digs))
    for i in np.random.default_rng(0).integers(0, w.n_blocks, 2000):
        assert hashlib.blake2b(w.block(int(i)), digest_size=32).digest() == digs[int(i)]
    # closed loop: the witness verifies the proofs (restated events/verifier.rs). The reference's verifier
    # rebuilds the 1 M-entry execution order per proof, so only a few proofs are replayed here.
    import copy
    import ctypes
    few = copy.copy(got)
    few.proofs = got.proofs[:3]
    few.raw_proofs = got.raw_proofs[:3 * ctypes.sizeof(A.EventProofC)]
    assert all(oracle_mod.verify_event_proofs(w, ts, few, spec))
    # bit-exact against the CPU oracle (pass 1 on 8 threads)
    exp = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec, threads=8)
    assert got.matching.tolist() == exp.matching.tolist()
    assert [p.key() for p in got.proofs] == [p.key() for p in exp.proofs]
    assert np.array_equal(w.cids, exp.witness.cids) and np.array_equal(w.lengths, exp.witness.lengths)
    sample = np.random.default_rng(1).integers(0, w.n_blocks, 3000)
    assert all(w.block(int(i)) == exp.witness.block(int(i)) for i in sample)
    # idempotence: a second scan of the resident store gives the same answer
    again = store.generate_event_proof(ts, spec)
    assert np.array_equal(again.witness.cids, w.cids) and [p.key() for p in again.proofs] == [p.key() for p in got.proofs]


def test_full_size_config3(api, oracle_mod, synth_mod):
    """1 M-slot storage HAMT, 1 k lookups (900 present + 100 absent)."""
    ts = synth_mod.Tipset(synth_mod.config_params(3))
    n = int(ts.params.hamt_entries)
    ks = np.random.default_rng(9).integers(0, n, 900).tolist()
    keys = [ts.storage_entry(k)[0] for k in ks] + [ts.storage_absent_key(k) for k in range(100)]
    slots = np.frombuffer(b"".join(api.compute_mapping_slots(keys, [0] * len(keys))), dtype=np.uint8)
    got = api.BlockStore.from_tipset(ts, verify_cids=True).read_storage_slots(ts.storage_root, slots)
    exp = oracle_mod.Store.from_tipset(ts).read_storage_slots(ts.storage_root, slots)
    assert np.array_equal(got.found, exp.found) and np.array_equal(got.raw_len, exp.raw_len) and np.array_equal(got.values, exp.values)
    assert_witness_equal(got.witness, exp.witness)
    assert got.found[:900].all() and not got.found[900:].any()
    for i, k in enumerate(ks):
        v = ts.storage_entry(k)[1]
        assert bytes(got.values[i][32 - len(v):]) == v


# ------------------------------------------------------------------ GPU-batched verifiers (events/verifier.rs, storage/verifier.rs)
def _verify_both(api, oracle_mod, w, ts, r, spec):
    """GPU verdicts == oracle verdicts, or both raise the same status."""
    try:
        exp = oracle_mod.verify_event_proofs(w, ts, r, spec)
    except A.IpcfpError as e:
        with pytest.raises(A.IpcfpError) as ei:
            api.verify_event_proofs(w, ts, r, spec)
        assert ei.value.status == e.status, (ei.value.status, ei.value.msg, e.status, e.msg)
        return None
    got = api.verify_event_proofs(w, ts, r, spec)
    assert got == exp
    return got


@pytest.mark.parametrize("cfg", [1, 2, "shapes", "shapes-nofilter"])
def test_verify_event_proofs_gpu(api, oracle_mod, synth_mod, cfg):
    ts = synth_tipset(synth_mod, cfg)
    spec = spec_of(ts)
    r = api.BlockStore.from_tipset(ts, verify_cids=True).generate_event_proof(ts, spec)
    assert len(r.proofs) > 0
    assert all(_verify_both(api, oracle_mod, r.witness, ts, r, spec))
    assert all(_verify_both(api, oracle_mod, r.witness, ts, r, None))
    # a different predicate: nothing satisfies it
    other = A.make_event_spec("SomethingElse(uint256)", ts.topic1, None)
    assert not any(_verify_both(api, oracle_mod, r.witness, ts, r, other))
    w = r.witness
    # drop-one-block minimality probe: same verdicts / same failure as the restated verifier, and every block is needed
    step = 1 if cfg == 1 else max(1, w.n_blocks // 60)
    for drop in range(0, w.n_blocks, step):
        keep = [i for i in range(w.n_blocks) if i != drop]
        w2 = A.WitnessPy(w.cids[keep], w.offsets[keep], w.lengths[keep], w.blob)
        got = _verify_both(api, oracle_mod, w2, ts, r, spec)
        if cfg == 1:
            assert got is None or not all(got), f"witness block {drop} is not needed"
    # tampered claims: event index, exec index, a topic byte, the message CID, the emitter
    import copy
    for off, what in ((8, "event_index"), (0, "exec_index"), (16, "emitter"), (48, "message_cid")):
        r2 = copy.copy(r)
        r2.raw_proofs = r.raw_proofs.copy()
        r2.raw_proofs[off] ^= 1
        got = _verify_both(api, oracle_mod, w, ts, r2, spec)
        assert got is None or not got[0], what
    r3 = copy.copy(r)
    r3.data_blob = r.data_blob.copy()
    r3.data_blob[5] ^= 0x80
    got = _verify_both(api, oracle_mod, w, ts, r3, spec)
    assert not got[0]
    # a witness block whose bytes do not hash to its CID never gets in (the check the reference's load_witness_store lacks)
    blob = w.blob.copy()
    blob[int(w.offsets[3]) + 1] ^= 0x10
    with pytest.raises(A.IpcfpError) as ei:
        api.verify_event_proofs(A.WitnessPy(w.cids, w.offsets, w.lengths, blob), ts, r, spec)
    assert ei.value.status == A.ERR_CID_MISMATCH and ei.value.index == 3


def test_verify_storage_proofs_gpu(api, oracle_mod, ts3_small):
    ts = ts3_small
    n = int(ts.params.hamt_entries)
    slots = [oracle_mod.compute_mapping_slot(ts.storage_entry(k)[0], 0) for k in (0, 5, n)] + [oracle_mod.compute_mapping_slot(ts.storage_absent_key(3), 0)]
    specs = [(a, s) for a in (1001, 1002, 1003, 1004, 1005, 1006) for s in slots]
    r = api.BlockStore.from_tipset(ts, verify_cids=True).generate_storage_proofs(ts, specs)
    exp = oracle_mod.verify_storage_proofs(r.witness, ts, r)
    got = api.verify_storage_proofs(r.witness, ts, r)
    assert got == exp and all(got)
    # tampered claims: value, storage root, actor state CID
    import copy
    sz = r.raw_proofs.size // len(r.proofs)
    for off in (8 + 38 + 38 + 32 + 31, 8 + 38 + 5, 8 + 5):
        r2 = copy.copy(r)
        r2.raw_proofs = r.raw_proofs.copy()
        r2.raw_proofs[sz * 2 + off] ^= 1
        exp2 = oracle_mod.verify_storage_proofs(r.witness, ts, r2)
        got2 = api.verify_storage_proofs(r.witness, ts, r2)
        assert got2 == exp2 and not got2[2] and got2[0]
    # a dropped witness block: same verdicts or the same failure
    w = r.witness
    for drop in range(0, w.n_blocks, max(1, w.n_blocks // 40)):
        keep = [i for i in range(w.n_blocks) if i != drop]
        w2 = A.WitnessPy(w.cids[keep], w.offsets[keep], w.lengths[keep], w.blob)
        try:
            e2 = oracle_mod.verify_storage_proofs(w2, ts, r)
        except A.IpcfpError as e:
            with pytest.raises(A.IpcfpError) as ei:
                api.verify_storage_proofs(w2, ts, r)
            assert ei.value.status == e.status
            continue
        assert api.verify_storage_proofs(w2, ts, r) == e2
