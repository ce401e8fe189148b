"""ipcfp_generate_message_proofs_resident on the GPU (include/ipcfp.h, DESIGN.md §2 "Message proofs") against tests/message_receipts.py,
the call restated in Python: every proof field, status, data-blob byte and the witness union, in both witness modes, with and without
IPCFP_MESSAGE_WITH_BODY, on hand-built worlds of real Message / SignedMessage blocks and receipts AMTs of height 0, 1 and 21. Also:
failures by (status, index) for dropped and truncated blocks, batches of 0, 1 and IPCFP_MESSAGE_MAX, the refusals, a tipset with an
empty receipt list, and the cross-checks against the message-log call (exec_index, the base witness) and the synthetic tipsets'
receipt lists."""
import ctypes as C
import random

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from oracle import pyoracle as P
from tests import message_amts as MA
from tests import message_receipts as MR
from tests.util import EditedTipset, dict_of

pytestmark = pytest.mark.gpu

WORLDS = {
    "min": dict(seed=1),
    "tall": dict(seed=2, height=21),
    "h0": dict(seed=3, short=25, height=0),
    "no_events": dict(seed=4, short=3, empty_events=True),
}


@pytest.fixture(scope="module")
def worlds(api):
    ts = MA.base_tipset()
    out = {}
    for name, kw in WORLDS.items():
        w = MR.world(ts, **kw)
        store = api.BlockStore(w.ts.cids, w.ts.offsets, w.ts.lengths, w.ts.blob, verify_cids=True)
        out[name] = (w, store)
    yield out
    for _, store in out.values():
        store.close()


def _cids(cs):
    return np.frombuffer(b"".join(bytes(c) for c in cs), np.uint8).reshape(-1, 38) if cs else np.zeros((0, 38), np.uint8)


def _generate(store, ts, cids, with_body=False, flags=0):
    tip = store.upload_tipset(ts)
    try:
        return store.generate_message_proofs_resident(tip, _cids(cids), with_body, flags)
    finally:
        tip.close()


def _check(blocks, store, ts, cids, with_body=False, flags=0):
    """The call == the restatement (proofs, data blob, witness CIDs and bytes), or the same (status, index). → the result or None."""
    try:
        proofs, wit = MR.prove(blocks, ts, cids, with_body)
    except MR.Fault as f:
        with pytest.raises(A.IpcfpError) as e:
            _generate(store, ts, cids, with_body, flags)
        assert (e.value.status, e.value.index) == (f.status, f.index)
        return None
    got = _generate(store, ts, cids, with_body, flags)
    assert [MR.proof_dict(p) for p in got.proofs] == proofs
    assert got.data_blob == b"".join(p["return_data"] + p.get("params", b"") for p in proofs)
    union = sorted(wit, key=P.cid_sort_key)
    assert [bytes(c) for c in got.witness.cids] == union
    if flags & A.WITNESS_BY_REFERENCE:
        assert len(got.witness.blob) == 0
    else:
        assert got.witness.blocks() == [blocks[c] for c in union]
    assert got.host_syncs == 5 and got.timings["total"] > 0
    return got


@pytest.mark.parametrize("by_ref", [0, A.WITNESS_BY_REFERENCE], ids=["by_value", "by_reference"])
@pytest.mark.parametrize("with_body", [False, True], ids=["receipt", "body"])
@pytest.mark.parametrize("name", list(WORLDS))
def test_worlds(worlds, name, with_body, by_ref):
    w, store = worlds[name]
    got = _check(w.blocks, store, w.ts, w.requests(), with_body, by_ref)
    st = [p.status for p in got.proofs]
    assert st.count(MR.NOT_EXECUTED) == len(w.never) + 1
    assert MR.NO_RECEIPT in st and MR.EXECUTED in st
    if with_body:
        assert {p.sig_type for p in got.proofs if p.has_body} == {0, 1, 2, 3}
        assert {p.to[0] for p in got.proofs if p.has_body} == set(range(5))


def test_shared_message_takes_its_first_position(worlds):
    w, store = worlds["min"]
    got = _generate(store, w.ts, [w.shared] + w.exec)
    assert got.proofs[0].exec_index == w.exec.index(w.shared) < w.shared_second
    assert [p.exec_index for p in got.proofs[1:]] == list(range(len(w.exec)))


def test_batches_of_0_1_and_max(api, worlds):
    w, store = worlds["min"]
    got = _generate(store, w.ts, [])
    assert got.proofs == [] and got.data_blob == b""
    tip = store.upload_tipset(w.ts)
    try:
        log, idx = store.generate_message_log_proof_resident(tip, _cids([]))
    finally:
        tip.close()
    assert [bytes(c) for c in got.witness.cids] == [bytes(c) for c in log.witness.cids], "n = 0: the base witness"
    _check(w.blocks, store, w.ts, [w.exec[5]], True)
    reqs = w.requests()
    rng = random.Random(5)
    big = [rng.choice(reqs) for _ in range(A.MESSAGE_MAX)]
    _check(w.blocks, store, w.ts, big, False)


def test_refusals(api, worlds):
    w, store = worlds["min"]
    lib = api.lib()
    tip = store.upload_tipset(w.ts)
    try:
        out = C.POINTER(A.MessageResultC)()
        one = _cids(w.exec[:1])
        assert lib.ipcfp_generate_message_proofs_resident(store._h, tip._h, None, 1, 0, C.byref(out)) == A.ERR_INVALID_ARG
        assert lib.ipcfp_generate_message_proofs_resident(store._h, tip._h, one.ctypes.data, 65537, 0, C.byref(out)) == A.ERR_INVALID_ARG
        for bit in (0x1, 0x2, 0x4, 0x10, 0x20, 0x80, 1 << 31):
            assert lib.ipcfp_generate_message_proofs_resident(store._h, tip._h, one.ctypes.data, 1, bit, C.byref(out)) == A.ERR_INVALID_ARG
    finally:
        tip.close()


def test_empty_receipt_list_gives_the_same_result(worlds):
    w, store = worlds["tall"]
    bare = EditedTipset(w.ts, n_receipts=0, events_roots=np.zeros((0, 38), np.uint8), has_events_root=np.zeros(0, np.uint8))
    a = _generate(store, w.ts, w.requests(), True)
    b = _generate(store, bare, w.requests(), True)
    assert a.raw_proofs.tobytes() == b.raw_proofs.tobytes() and a.data_blob == b.data_blob
    assert [bytes(c) for c in a.witness.cids] == [bytes(c) for c in b.witness.cids]


def _fault_cases(w):
    """(name, blocks) with one block dropped or truncated: every receipts-AMT node on two paths, the receipts leaf of a message
    shared by two parents, and message blocks."""
    out = []
    for i in (0, len(w.receipts) - 1):
        for c in MR.receipt_path(w, i):
            out.append((f"drop-path-{i}-{c.hex()[-8:]}", {k: v for k, v in w.blocks.items() if k != c}))
            out.append((f"trunc-path-{i}-{c.hex()[-8:]}", {**w.blocks, c: w.blocks[c][:-1]}))
    for j in (0, 7, len(w.exec) - 1):
        c = w.exec[j]
        out.append((f"drop-msg-{j}", {k: v for k, v in w.blocks.items() if k != c}))
        out.append((f"trunc-msg-{j}", {**w.blocks, c: w.blocks[c][:-1]}))
    return out


@pytest.mark.parametrize("name", ["min", "tall"])
def test_faults_match_the_restatement(api, worlds, name):
    w, _ = worlds[name]
    reqs = list(reversed(w.requests()))
    n_faults = 0
    for case, blocks in _fault_cases(w):
        ts = MR.with_blocks(w, blocks)
        store = api.BlockStore(ts.cids, ts.offsets, ts.lengths, ts.blob, verify_cids=False)
        try:
            for body in (False, True):
                n_faults += _check(blocks, store, w.ts, reqs, body) is None
        finally:
            store.close()
    assert n_faults >= len(_fault_cases(w))


@pytest.mark.parametrize("cfg", [1, 2, 3])
def test_synthetic_tipsets_agree_with_their_receipt_lists(api, synth_mod, cfg):
    ts = synth_mod.Tipset(synth_mod.config_params(cfg, hamt_entries=20000) if cfg == 3 else synth_mod.config_params(cfg))
    blocks = dict_of(ts)
    ex = P.collect_exec_list(blocks.get, [bytes(ts.parent_txmeta_cids[k]) for k in range(int(ts.n_parents))])
    store = api.BlockStore.from_tipset(ts, verify_cids=True)
    try:
        reqs = ex + [P.cid_of(b"not a message")]
        got = _generate(store, ts, reqs)
        tip = store.upload_tipset(ts)
        try:
            _, idx = store.generate_message_log_proof_resident(tip, _cids(reqs))
        finally:
            tip.close()
        assert [MR.U64 if p.exec_index is None else p.exec_index for p in got.proofs] == [int(x) for x in idx]
        n = int(ts.n_receipts)
        for p in got.proofs[:-1]:
            i = p.exec_index
            if i < n:
                assert p.status == MR.EXECUTED
                want = bytes(ts.events_roots[i]) if ts.has_events_root[i] else None
                assert p.events_root == want
        if cfg == 3:
            proofs, wit = MR.prove(blocks, ts, reqs)
            assert [MR.proof_dict(p) for p in got.proofs] == proofs
            assert [bytes(c) for c in got.witness.cids] == sorted(wit, key=P.cid_sort_key)
    finally:
        store.close()


# ------------------------------------------------------------------ the verifier
def _witness_of(blocks):
    from types import SimpleNamespace
    from tests.storage_trees import Blocks
    cids, offs, lens, blob = Blocks(blocks).flat()
    return SimpleNamespace(cids=cids, offsets=offs, lengths=lens, blob=blob)


def _changed(rec, blob, k, body):
    """proof record rec (A.MessageProofC) and the data blob with claim k changed → (record, blob), or None when the claim does not apply"""
    r = A.MessageProofC.from_buffer_copy(bytes(rec))
    b = bytearray(blob)
    executed = r.status == MR.EXECUTED
    if k == "exit_code" and executed:
        r.exit_code ^= 1
    elif k == "gas_used" and executed:
        r.gas_used ^= 1
    elif k == "return_byte" and executed and r.return_len:
        b[r.return_off] ^= 1
    elif k == "return_len" and executed:
        r.return_len += 1
    elif k == "events_root" and executed:
        r.has_events_root ^= 1
        r.events_root[:] = list(bytes(38) if not r.has_events_root else bytes(rec.message_cid))
    elif k == "exec_plus" and r.exec_index != MR.U64:
        r.exec_index += 1
    elif k == "exec_minus" and r.exec_index not in (0, MR.U64):
        r.exec_index -= 1
    elif k == "not_executed" and r.status != MR.NOT_EXECUTED:
        r.status, r.exec_index = MR.NOT_EXECUTED, MR.U64
    elif k == "executed" and r.status == MR.NOT_EXECUTED:
        r.status, r.exec_index = MR.EXECUTED, 0
    elif body and r.has_body and k in ("version", "sequence", "gas_limit", "method_num"):
        setattr(r, k, getattr(r, k) ^ 1)
    elif body and r.has_body and k in ("value", "gas_fee_cap", "gas_premium"):
        getattr(r, k)[31] ^= 1
    elif body and r.has_body and k in ("to", "from_"):
        getattr(r, k).bytes[getattr(r, k).len - 1] ^= 1
    elif body and r.has_body and k == "sig_type":
        r.sig_type = 3 if r.sig_type != 3 else 1
    elif body and r.has_body and k == "params_byte" and r.params_len:
        b[r.params_off] ^= 1
    elif body and r.has_body and k == "params_len":
        r.params_len += 1
    else:
        return None
    return r, bytes(b)


CLAIMS = ["exit_code", "gas_used", "return_byte", "return_len", "events_root", "exec_plus", "exec_minus", "not_executed", "executed", "version",
          "sequence", "gas_limit", "method_num", "value", "gas_fee_cap", "gas_premium", "to", "from_", "sig_type", "params_byte", "params_len"]


@pytest.mark.parametrize("with_body", [False, True], ids=["receipt", "body"])
@pytest.mark.parametrize("name", ["min", "tall", "h0"])
def test_verifier_accepts_every_proof_and_rejects_every_changed_claim(api, worlds, name, with_body):
    w, store = worlds[name]
    got = _generate(store, w.ts, w.requests(), with_body)
    assert all(api.verify_message_proofs(got.witness, w.ts, got, with_body))
    recs = (A.MessageProofC * len(got.proofs)).from_buffer_copy(got.raw_proofs.tobytes())
    applied = set()
    for k in CLAIMS:
        for i in range(len(recs)):
            ch = _changed(recs[i], got.data_blob, k, with_body)
            if ch is None:
                continue
            r, blob = ch
            raw = bytearray(got.raw_proofs.tobytes())
            raw[i * C.sizeof(r):(i + 1) * C.sizeof(r)] = bytes(r)
            v = api.verify_message_proofs(got.witness, w.ts, np.frombuffer(bytes(raw), np.uint8), with_body, data_blob=blob)
            assert not v[i], (k, i)
            if k not in ("return_byte", "params_byte"):
                assert sum(v) == len(v) - 1, (k, i)
            applied.add(k)
            break
    assert applied == set(CLAIMS if with_body else CLAIMS[:9])


def test_verifier_never_accepts_a_forged_receipts_amt(api, worlds):
    w, _ = worlds["min"]
    fts, fblocks = MR.forge(w)
    fstore = api.BlockStore(fts.cids, fts.offsets, fts.lengths, fts.blob, verify_cids=True)
    try:
        forged = _generate(fstore, fts, w.requests())
    finally:
        fstore.close()
    assert any(p.status == MR.EXECUTED for p in forged.proofs)
    assert all(api.verify_message_proofs(forged.witness, fts, forged))   # honest against its own tipset
    with pytest.raises(A.IpcfpError):                                    # the true child header is not in the forged witness
        api.verify_message_proofs(forged.witness, w.ts, forged)
    both = {**w.blocks, **fblocks}
    v = api.verify_message_proofs(_witness_of(both), w.ts, forged)
    for p, ok in zip(forged.proofs, v):
        assert not (ok and p.status == MR.EXECUTED)


# ------------------------------------------------------------------ the fetch loop
def _fetcher(full, held):
    from tests import rpc_blocks as B

    def fetch(cids, first_id):
        els = []
        for k, c in enumerate(cids):
            c = bytes(c)
            assert c not in held, "a CID was requested twice"
            held[c] = full[c]
            els.append(B.element(first_id + k, full[c]))
        return B.render([], elements=els)
    return fetch


@pytest.mark.parametrize("with_body", [False, True], ids=["receipt", "body"])
@pytest.mark.parametrize("name", ["min", "tall"])
def test_fetch_loop_fetches_exactly_the_read_set(api, worlds, name, with_body):
    w, store = worlds[name]
    reqs = w.requests()
    full = _generate(store, w.ts, reqs, with_body)
    held = {}
    st, tip, rounds, _, _ = api.fetch_message_proofs_until_complete(_fetcher(w.blocks, held), lambda s: s.upload_tipset(w.ts), _cids(reqs),
                                                                    with_body)
    try:
        assert set(held) == {bytes(c) for c in full.witness.cids} == MR.read_set(w.blocks, w.ts, reqs, with_body)
        assert not {r[3] for r in w.receipts.values() if r[3]} & set(held)   # no events AMT
        assert len(rounds) >= 2
        again = st.generate_message_proofs_resident(tip, _cids(reqs), with_body)
        assert np.array_equal(again.raw_proofs, full.raw_proofs) and again.data_blob == full.data_blob
    finally:
        tip.close()
        st.close()
