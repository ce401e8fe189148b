"""The event path on the GPU on hand-built events AMTs and receipts AMTs (tests/event_amts.py): events AMTs of every bit width 1–8 at
heights 0, 1, 2, the minimal one and 64 // bw with holes, sparse and top indices (and indices at or above 2^64), the deepest legal walk
(bit width 1, height 64, 65 frames), single-node roots on both sides of pass 1's staged header limit, empty roots above height 0;
receipts AMTs of every height up to 21 missing matching receipts at warp and CTA edges; an RPC events root that is not the chain's;
and, one tipset each, the roots and nodes the decode contract refuses, among them every height whose product with the bit width wraps
modulo 2^64. Checked for each: generate_event_proof == the C++ oracle field by field (witness bytes included) or the same (status,
index), and == the restatement's ground truth below 2^64; the device JSON == the host rendering of the flagless result; the GPU
verifier == the oracle's verifier on honest and tampered proofs; verify_bundle_json on the device text == verify_event_proofs."""
import copy
import ctypes as C

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import event_amts as E
from tests.test_event_amts import COUNTS, kind
from tests.util import assert_event_results_equal, spec_of

pytestmark = pytest.mark.gpu

N_VALID = COUNTS["valid"] + COUNTS["receipts"] + COUNTS["rpc"]
N_FAULT = sum(COUNTS.values()) - N_VALID


@pytest.fixture(scope="module")
def base(synth_mod):
    return E.base_tipset()


@pytest.fixture(scope="module")
def cases(base):
    return E.catalogue(base)


def _outcome(fn):
    try:
        return fn(), None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _pass2(monkeypatch, per_thread):
    if per_thread:
        monkeypatch.setenv("IPCFP_PASS2_PER_THREAD", "1")
    else:
        monkeypatch.delenv("IPCFP_PASS2_PER_THREAD", raising=False)


def _generate(api, oracle_mod, c):
    """GPU == oracle (every field, or the same (status, index)); valid cases == the ground truth. → (gpu result, oracle result) or
    the failure."""
    ts, spec = c.ts, spec_of(c.ts)
    exp, eerr = _outcome(lambda: oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec))
    got, gerr = _outcome(lambda: api.BlockStore.from_tipset(ts, verify_cids=True).generate_event_proof(ts, spec))
    assert gerr == eerr, (c.name, gerr, eerr)
    if eerr:
        return eerr
    if c.holes:
        # the proof slots of receipts missing from the receipts AMT are dropped, and their bytes in the data blob are never written:
        # everything but the blob, whose contents the proofs carry
        assert got.matching.tolist() == exp.matching.tolist() and got.n_exec == exp.n_exec, c.name
        assert [p.key() for p in got.proofs] == [p.key() for p in exp.proofs], c.name
        assert np.array_equal(got.witness.cids, exp.witness.cids) and got.witness.blocks() == exp.witness.blocks(), c.name
    else:
        try:
            assert_event_results_equal(got, exp)
        except AssertionError:
            raise AssertionError(c.name)
    t = E.truth(c)
    assert got.matching.tolist() == t["matching"] and {bytes(x) for x in got.witness.cids} == t["witness"], c.name
    if not c.big:
        assert [p.key() for p in got.proofs] == [(i, j, em, tuple(tp), d, m) for i, j, em, tp, d, m in t["proofs"]], c.name
    return got, exp


@pytest.mark.parametrize("per_thread", [False, True])
def test_generator_on_valid_amts(api, oracle_mod, cases, monkeypatch, per_thread):
    _pass2(monkeypatch, per_thread)
    n = 0
    for c in cases:
        if c.status is None:
            out = _generate(api, oracle_mod, c)
            assert isinstance(out, tuple) and len(out[1].proofs) > 0, c.name
            n += 1
    assert n == N_VALID


def test_generator_on_refused_amts(api, oracle_mod, cases):
    """Every fault case, wrapping heights included: the expected status at the receipt the sequential walk meets it."""
    n, wraps = 0, 0
    for c in cases:
        if c.status is None:
            continue
        err = _generate(api, oracle_mod, c)
        assert err[0] == c.status and (c.index is None or err[1] == c.index), (c.name, err)
        n += 1
        wraps += kind(c) in ("wrap", "receipts-wrap", "message-wrap")
    assert n == N_FAULT and wraps == 352 + 43 + 43


def _c_call(api, store, ts, spec, flags):
    L = api.lib()
    d, keep = A.make_tipset_desc(ts)
    out = C.POINTER(A.EventResultC)()
    api._check(L.ipcfp_generate_event_proof(store._h, C.byref(d), C.byref(spec), flags, C.byref(out)))
    try:
        host = None if flags & A.RESULT_JSON else api.event_result_to_json(out, ts)
        return A.event_result_from_c(out.contents), host
    finally:
        L.ipcfp_event_result_free(out)


def test_json_render(api, cases):
    """IPCFP_RESULT_JSON: the device text is the host rendering of the flagless result, event indices up to 2^64 − 1 included."""
    n = 0
    for c in cases:
        if c.status is not None:
            continue
        spec = spec_of(c.ts)
        store = api.BlockStore.from_tipset(c.ts)
        base, want = _c_call(api, store, c.ts, spec, 0)
        got, _ = _c_call(api, store, c.ts, spec, A.RESULT_JSON)
        assert got.json == want, c.name
        if c.name == "valid":
            assert '"event_index":18446744073709551614' in want
        n += 1
    assert n == N_VALID


def _set_u64(r, k, off, v):
    sz = C.sizeof(A.EventProofC)
    r.raw_proofs[sz * k + off:sz * k + off + 8] = np.frombuffer(int(v).to_bytes(8, "little"), dtype=np.uint8)


def _verify_both(api, oracle_mod, w, ts, r):
    """→ (verdicts, None) or (None, (status, index)). A fault inside the oracle's AMT helpers carries no proof index (2^64 − 1); the
    device names the proof that met it."""
    exp, eerr = _outcome(lambda: oracle_mod.verify_event_proofs(w, ts, r))
    got, gerr = _outcome(lambda: api.verify_event_proofs(w, ts, r))
    assert got == exp and (gerr is None) == (eerr is None)
    if eerr:
        assert gerr[0] == eerr[0] and (eerr[1] == 2 ** 64 - 1 or gerr[1] == eerr[1]), (gerr, eerr)
        return None, gerr
    return exp, eerr


def _tampered(c, r):
    """(kind, result copy, tampered proof numbers): event_index set to its ordinal among the AMT's values, to a hole, to j + width^k;
    exec_index set to a receipt missing from the receipts AMT."""
    out = []
    for what in ("ordinal", "hole", "plus-width-power", "exec-hole"):
        r2 = copy.copy(r)
        r2.raw_proofs = r.raw_proofs.copy()
        hit = []
        for k, p in enumerate(r.proofs):
            a = c.amts.get(p.exec_index)
            j, v, off = p.event_index, None, 8
            if what == "exec-hole":
                v, off = (sorted(c.holes)[k % len(c.holes)] if c.holes else None), 0
            elif a is not None:
                top = min(E.width(a.bw) ** (a.height + 1), E.U64)
                if what == "ordinal":
                    v = sorted(a.values).index(j)
                elif what == "hole":
                    v = next((x for x in (j + 1, j - 1, j + 2, top - 1, 0) if 0 <= x < top and x not in a.values), None)
                else:
                    step = E.width(a.bw) ** (k % (a.height + 1))
                    v = j + step if j + step < E.U64 else None
                if v is not None and v in a.values:
                    v = None
            if v is not None and v != (p.exec_index if off == 0 else j):
                _set_u64(r2, k, off, v)
                hit.append(k)
        if hit:
            out.append((what, r2, hit))
    return out


def test_verifiers(api, oracle_mod, cases):
    """The GPU verifier == the oracle's verifier on honest and tampered proofs; honest proofs verify (except where the reference's
    saturating `get` cannot reach the event, E.honest_verdicts); tampered ones do not; verify_bundle_json on the device text gives
    the verdicts verify_event_proofs gives."""
    n, kinds = 0, set()
    for c in cases:
        if c.status is not None:
            continue
        ts = c.ts
        store = api.BlockStore.from_tipset(ts)
        r, _ = _c_call(api, store, ts, spec_of(ts), 0)
        exp, eerr = _verify_both(api, oracle_mod, r.witness, ts, r)
        if c.name == "rpc-root-differs":
            # the first proof of receipt 5, whose chain events root the witness does not hold
            assert eerr is not None and eerr[0] == A.ERR_MISSING_BLOCK and r.proofs[eerr[1]].exec_index == 5
            assert all(p.exec_index != 5 for p in r.proofs[:eerr[1]])
        elif not c.big:
            assert exp == E.honest_verdicts(c, r), c.name
        if not c.big:
            for what, r2, hit in _tampered(c, r):
                v2, e2 = _verify_both(api, oracle_mod, r.witness, ts, r2)
                if e2 is None:
                    assert not any(v2[k] for k in hit), (c.name, what)
                kinds.add(what)
        doc, _ = _c_call(api, store, ts, spec_of(ts), A.RESULT_JSON)
        vj, ej = _outcome(lambda: api.verify_bundle_json(doc.json))
        if eerr is None:
            assert ej is None and vj.event_results == exp, c.name
        else:
            assert ej is not None and ej[0] == eerr[0], (c.name, ej, eerr)
        n += 1
    assert n == N_VALID and kinds == {"ordinal", "hole", "plus-width-power", "exec-hole"}
