"""The engine on adversarial CID sets (tests/util.py: families A clustered, B mixed prefixes, C both, D duplicate flat entries).

Every witness comes out of a bitmap indexed by the store's `Cid` rank (`sort_by_cid`: radix passes on digest bytes 0-3 and on the
class rank, then `k_tie_fix`), and every block lookup goes through one open-addressing table (`k_build_index`, `store_find`) hashed on
digest words 0 and 2 and the class. Synthetic chains under one prefix with random digests almost never reach the tie fix, the class
pass, a probe past a fingerprint match or the duplicate rule; these tests make every one of them decide the result. Each result is
compared with the CPU oracle on the rewritten tipset and with the image of the oracle's result on the original one."""
import ctypes as C
import re

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import bundle_json as J
from tests import util as U
from tests.util import assert_event_results_equal, assert_witness_equal, spec_of

pytestmark = pytest.mark.gpu

FAMILIES = ["A", "B", "C", "D"]


def _event_call(api, store, ts, spec, flags=0, resident=False, host_json=False):
    """One generate_event_proof call through the C ABI → EventResultPy (and the host renderer's text of the C result)."""
    L = api.lib()
    d, keep = A.make_tipset_desc(ts)
    out = C.POINTER(A.EventResultC)()
    if resident:
        th = C.c_void_p()
        api._check(L.ipcfp_tipset_upload(store._h, C.byref(d), C.byref(th)))
        try:
            st = L.ipcfp_generate_event_proof_resident(store._h, th, C.byref(spec), flags, C.byref(out))
        finally:
            L.ipcfp_tipset_free(th)
    else:
        st = L.ipcfp_generate_event_proof(store._h, C.byref(d), C.byref(spec), flags, C.byref(out))
    api._check(st)
    try:
        r = A.event_result_from_c(out.contents)
        return (r, api.event_result_to_json(out, ts)) if host_json else r
    finally:
        L.ipcfp_event_result_free(out)


def _check_events(api, oracle_mod, ts, family, flags=0, resident_too=False):
    rt, cm = U.adversarial_tipset(ts, family)
    spec = spec_of(ts)
    exp0 = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec, flags=flags)
    exp = oracle_mod.Store.from_tipset(rt).generate_event_proof(rt, spec, flags=flags)
    store = api.BlockStore.from_tipset(rt)
    blob = np.asarray(rt.blob, dtype=np.uint8)
    for resident in ((False, True) if resident_too else (False,)):
        got = _event_call(api, store, rt, spec, flags, resident)
        assert_event_results_equal(got, exp)
        U.assert_event_image(got, exp0, cm)
        ref = _event_call(api, store, rt, spec, flags | A.WITNESS_BY_REFERENCE, resident)
        assert ref.matching.tolist() == got.matching.tolist() and ref.n_exec == got.n_exec
        assert [p.key() for p in ref.proofs] == [p.key() for p in got.proofs]
        assert np.array_equal(ref.witness.cids, got.witness.cids) and np.array_equal(ref.witness.lengths, got.witness.lengths)
        assert len(ref.witness.blob) == 0
        for i in range(got.witness.n_blocks):
            o, n = int(ref.witness.offsets[i]), int(ref.witness.lengths[i])
            assert bytes(blob[o:o + n]) == got.witness.block(i), i
            if family == "D":   # the first flat entry of a repeated CID is the block the index keeps
                assert o == rt.first_offset[bytes(got.witness.cids[i])], i
    assert exp.proofs or not exp0.proofs
    return rt, cm, got


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("cfg", [1, 2])
def test_event_proofs(api, oracle_mod, synth_mod, cfg, family):
    ts = synth_mod.Tipset(synth_mod.config_params(cfg))
    _, _, got = _check_events(api, oracle_mod, ts, family, resident_too=True)
    assert got.proofs


@pytest.mark.parametrize("family", FAMILIES)
def test_event_proofs_with_duplicate_messages(api, oracle_mod, synth_mod, family):
    """A test_event_proof_shapes shape (two- and three-level events AMTs) with 4 duplicate messages per message AMT pair."""
    ts = synth_mod.Tipset(synth_mod.default_params(seed=99, n_receipts=300, events_per_receipt=40, match_ppm=100000, dup_msgs=4))
    _check_events(api, oracle_mod, ts, family)


@pytest.mark.parametrize("family", FAMILIES)
def test_event_proofs_general_walk(api, oracle_mod, synth_mod, monkeypatch, family):
    monkeypatch.setenv("IPCFP_BFS_GENERAL", "1")
    ts = synth_mod.Tipset(synth_mod.default_params(seed=7, n_receipts=700, events_per_receipt=5, match_ppm=50000, n_parents=3, dup_msgs=4))
    _check_events(api, oracle_mod, ts, family, resident_too=True)


@pytest.mark.parametrize("family", FAMILIES)
def test_event_proofs_skip_tx_amts(api, oracle_mod, ts2, family):
    _check_events(api, oracle_mod, ts2, family, flags=A.SCAN_SKIP_TX_AMTS)


@pytest.mark.parametrize("family", FAMILIES)
def test_storage_and_bundle(api, oracle_mod, ts3_small, family):
    ts = ts3_small
    rt, cm = U.adversarial_tipset(ts, family)
    n = int(ts.params.hamt_entries)
    rng = np.random.default_rng(5)
    ks = rng.integers(0, n, 300).tolist() + [n]
    keys = [ts.storage_entry(k)[0] for k in ks] + [ts.storage_absent_key(k) for k in range(40)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    slots_np = np.frombuffer(b"".join(slots), dtype=np.uint8)
    o0, o = oracle_mod.Store.from_tipset(ts), oracle_mod.Store.from_tipset(rt)
    store = api.BlockStore.from_tipset(rt)

    exp0, exp = o0.read_storage_slots(ts.storage_root, slots_np), o.read_storage_slots(rt.storage_root, slots_np)
    got = store.read_storage_slots(rt.storage_root, slots_np)
    for e in (exp0, exp):
        assert np.array_equal(got.found, e.found) and np.array_equal(got.raw_len, e.raw_len) and np.array_equal(got.values, e.values)
    assert got.found[:301].all() and not got.found[301:].any()
    assert_witness_equal(got.witness, exp.witness)
    assert ([bytes(c) for c in got.witness.cids], got.witness.blocks()) == cm.witness(exp0.witness)

    specs = [(actor, s) for actor in (1001, 1002, 1003, 1006) for s in slots[:4] + slots[-2:]]
    exp0, exp = o0.generate_storage_proofs(ts, specs), o.generate_storage_proofs(rt, specs)
    got = store.generate_storage_proofs(rt, specs)
    assert [vars(p) for p in got.proofs] == [vars(p) for p in exp.proofs] == cm.storage_proofs(exp0.proofs)
    assert_witness_equal(got.witness, exp.witness)
    assert ([bytes(c) for c in got.witness.cids], got.witness.blocks()) == cm.witness(exp0.witness)
    assert got.spec_witness == exp.spec_witness == cm.spec_witness(exp0)

    sspecs = [(1001, slots[0]), (1003, slots[1]), (1006, slots[-1])]
    especs = [A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter), A.make_event_spec(ts.event_signature, "calib-subnet-2", None)]
    exp0, exp = o0.generate_proof_bundle(ts, sspecs, especs), o.generate_proof_bundle(rt, sspecs, especs)
    got = store.generate_proof_bundle(rt, sspecs, especs)
    assert [vars(p) for p in got.storage.proofs] == [vars(p) for p in exp.storage.proofs] == cm.storage_proofs(exp0.storage.proofs)
    for g, e, e0 in zip(got.events, exp.events, exp0.events):
        assert_event_results_equal(g, e)
        U.assert_event_image(g, e0, cm)
    assert_witness_equal(got.witness, exp.witness)
    assert ([bytes(c) for c in got.witness.cids], got.witness.blocks()) == cm.witness(exp0.witness)
    assert got.witness.n_blocks > got.storage.witness.n_blocks


@pytest.mark.parametrize("cfg", [1, 2])
def test_result_json_mixed_prefixes(api, oracle_mod, synth_mod, cfg):
    """IPCFP_RESULT_JSON on a family-B store: the device text equals the host renderer and bundle_json.py, and its CID strings carry
    the other prefixes (not the `bafy2bzace` of dag-cbor / blake2b-256)."""
    ts = synth_mod.Tipset(synth_mod.config_params(cfg))
    rt, cm = U.adversarial_tipset(ts, "B")
    spec = spec_of(rt)
    store = api.BlockStore.from_tipset(rt)
    base, want = _event_call(api, store, rt, spec, host_json=True)
    assert want == J.dumps(J.event_bundle(rt, base))
    for resident in (False, True):
        for extra in (A.RESULT_JSON, A.RESULT_JSON | A.WITNESS_BY_REFERENCE):
            got = _event_call(api, store, rt, spec, extra, resident)
            assert got.json == want, (resident, extra)
    strings = re.findall(r'"(?:message_cid|child_block_cid|parent_tipset_cids)":\[?"([a-z2-7]+)"', want)
    assert strings and any(not s.startswith("bafy2bzace") for s in strings)
    assert {J.cid_to_string(cm.cid(p.message_cid)) for p in oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec).proofs} == \
        {J.cid_to_string(p.message_cid) for p in base.proofs}


# ------------------------------------------------------------------ the store index, directly
def _family_cids(family, n, seed=0):
    """n distinct CIDs of a family (A clustered / B mixed prefixes with shared digests / C both) without a tipset."""
    rng = np.random.default_rng(seed)
    digs = U.clustered_digests(n, rng) if family in ("A", "C") else [rng.bytes(32) for _ in range(n)]
    if family == "A":
        pres = [U.FILECOIN_PREFIX] * n
    else:
        pres = [U.MIXED_PREFIXES[(k // 61) % 8] for k in range(n)]
        if n:
            pres[0] = U.MIXED_PREFIXES[-1]
        for j in range(1, n - 1, 7):
            digs[j + 1] = digs[j]
            if pres[j + 1] == pres[j]:
                pres[j + 1] = U.MIXED_PREFIXES[(U.MIXED_PREFIXES.index(pres[j]) + 1) % 8]
    cids = [p + d for p, d in zip(pres, digs)]
    assert len(set(cids)) == n
    return cids


def _flat(cids, blocks):
    offs, blob = [], bytearray()
    for b in blocks:
        while len(blob) % 16:
            blob.append(0)
        offs.append(len(blob))
        blob.extend(b)
    blob.extend(bytes(32))
    return (np.frombuffer(b"".join(cids), dtype=np.uint8).reshape(-1, 38), np.array(offs, dtype=np.uint64),
            np.array([len(b) for b in blocks], dtype=np.uint32), np.frombuffer(bytes(blob), dtype=np.uint8))


def _store(api, cids, blocks):
    return api.BlockStore(*_flat(cids, blocks))


def _store_set(family, n, seed=0):
    """(flat cids, flat blocks, cid -> expected block): family D is family A plus repeats of its CIDs — identical bytes before the
    original, different bytes after it, and one CID 1 000 more times."""
    rng = np.random.default_rng(seed + 1)
    cids = _family_cids("A" if family == "D" else family, n, seed)
    blocks = [rng.bytes(int(rng.integers(0, 200))) for _ in cids]
    if family == "D":
        before = [int(i) for i in rng.choice(n, 60, replace=False)]
        after = [int(i) for i in rng.choice(n, 60, replace=False)]
        hot = 700   # a member of the 512 group
        cids = [cids[i] for i in before] + cids + [cids[i] for i in after] + [cids[hot]] * 1000
        blocks = [blocks[i] for i in before] + blocks + [rng.bytes(int(rng.integers(1, 64))) for _ in after] + [b"x" * 33] * 1000
    want = {}
    for c, b in zip(cids, blocks):
        want.setdefault(c, b)
    return cids, blocks, want


def _near_misses(c, prefixes):
    out = []
    for p in range(6, 38):   # every digest byte flipped
        for x in (0x80, 0x01, 0xFF):
            m = bytearray(c)
            m[p] ^= x
            out.append(bytes(m))
    out += [q + c[6:] for q in prefixes if q != c[:6]]
    out.append(bytes.fromhex("0172a0e40220") + c[6:])   # a prefix no store here holds
    return out


def _expect(store, want, probes):
    for p in probes:
        assert store.get(p) == want.get(p), p.hex()
        assert store.has(p) == (p in want), p.hex()


@pytest.mark.parametrize("family", FAMILIES)
def test_store_index_families(api, family):
    cids, blocks, want = _store_set(family, 1500)
    store = _store(api, cids, blocks)
    _expect(store, want, list(want))
    held = sorted({c[:6] for c in want})
    probes = []
    for c in list(want)[::97] + list(want)[600:606]:
        probes += _near_misses(c, held)
    _expect(store, want, probes)
    if family in ("B", "C"):   # some prefix swaps land on the other CID of a digest shared under two prefixes
        assert any(p in want and p[6:] == c[6:] for c in want for p in _near_misses(c, held)[96:-1])


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025])
def test_store_index_sizes(api, n):
    rng = np.random.default_rng(n)
    cids = _family_cids("C" if n >= 64 else "A", n, seed=n)
    blocks = [rng.bytes(int(rng.integers(0, 100))) for _ in cids]
    store = _store(api, cids, blocks)
    want = dict(zip(cids, blocks))
    _expect(store, want, cids)
    probes = [U.FILECOIN_PREFIX + rng.bytes(32) for _ in range(16)]
    for c in cids[:: max(1, n // 8)]:
        probes += _near_misses(c, sorted({x[:6] for x in cids}))
    _expect(store, want, probes)


def test_store_index_probe_wraps(api):
    """Every CID of the store hashes into the last two slots of the table, so inserts and lookups wrap from slot `mask` to 0; misses
    aimed at the same slots walk the whole wrapped run."""
    n = 40
    mask = U.table_slots(n) - 1
    rng = np.random.default_rng(11)

    def aimed(k):
        out = []
        while len(out) < k:
            d = rng.bytes(32)
            if U.digest_hash(d, 0) & mask >= mask - 1:
                out.append(U.FILECOIN_PREFIX + d)
        return out
    cids = aimed(n)
    assert mask == 127 and all(U.digest_hash(c[6:], 0) & mask >= mask - 1 for c in cids)   # the aim (class 0: one prefix)
    blocks = [rng.bytes(int(rng.integers(1, 80))) for _ in cids]
    store = _store(api, cids, blocks)
    want = dict(zip(cids, blocks))
    _expect(store, want, cids)
    misses = aimed(20)
    for c in cids[::5]:
        m = bytearray(c)
        m[6 + 9] ^= 0x40   # outside digest words 0 and 2: same hash, same fingerprint
        misses.append(bytes(m))
    assert all(U.digest_hash(c[6:], 0) & mask >= mask - 1 for c in misses)
    _expect(store, want, misses)


# ------------------------------------------------------------------ refusals at ingest
def test_store_accepts_eight_prefixes_and_refuses_a_ninth(api):
    rng = np.random.default_rng(2)
    cids = [U.MIXED_PREFIXES[k % 8] + rng.bytes(32) for k in range(40)]
    blocks = [rng.bytes(10) for _ in cids]
    store = _store(api, cids, blocks)
    _expect(store, dict(zip(cids, blocks)), cids)
    ninth = bytes.fromhex("0171a1e40220")   # a valid ninth prefix (multihash code 0xb221)
    bad = list(cids)
    bad[23] = ninth + bad[23][6:]
    bad[31] = ninth + bad[31][6:]
    with pytest.raises(A.IpcfpError) as ei:
        _store(api, bad, blocks)
    assert ei.value.status == A.ERR_UNSUPPORTED and ei.value.index == 23


@pytest.mark.parametrize("at", [0, 17])
def test_store_refuses_an_unparseable_prefix(api, at):
    """A sha2-256 CIDv1 (01 71 12 20 + 32 bytes) padded to 38 bytes has no 6-byte prefix the store can hold."""
    rng = np.random.default_rng(4)
    cids = [U.FILECOIN_PREFIX + rng.bytes(32) for _ in range(30)]
    cids[at] = bytes.fromhex("01711220") + rng.bytes(34)
    with pytest.raises(A.IpcfpError) as ei:
        _store(api, cids, [rng.bytes(8) for _ in cids])
    assert ei.value.status == A.ERR_UNSUPPORTED
