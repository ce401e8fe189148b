"""The hand-built events AMTs and receipts AMTs of tests/event_amts.py are what the GPU tests (tests/test_gpu_event_amts.py) take them
for (no GPU): the builder writes the shapes the cases are named after; on every valid case the strict restatement of DESIGN.md §3
(`truth`), the Python oracle and the C++ oracle agree on the matching receipts, every proof and the witness CID set (event indices at
or above 2^64 are the C++ oracle's saturating arithmetic, so those proofs are compared between the two Python sides only); and every
fault case fails in the restatement and in the C++ oracle with the expected status at the expected receipt. Roots whose height·bw
wraps modulo 2^64 are among the faults: the restatement, both oracles and the device refuse them."""
import cbor2
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from oracle import pyoracle as P
from tests import event_amts as E
from tests.util import spec_of

# case counts per kind; a change of the catalogue has to change these
COUNTS = {"valid": 2, "receipts": 19, "rpc": 1, "wrap": 352, "receipts-wrap": 43, "message-wrap": 43, "missing": 93, "undecodable": 26,
          "other-faults": 36}


def kind(c):
    n = c.name
    for k in ("receipts-wrap", "message-wrap", "valid", "rpc", "wrap", "missing", "undecodable"):
        if n.startswith(k):
            return k
    return "receipts" if n.startswith("receipts-h") else "other-faults"


@pytest.fixture(scope="module")
def base(synth_mod):
    return E.base_tipset()


@pytest.fixture(scope="module")
def cases(base):
    return E.catalogue(base)


def _oracle(oracle_mod, c):
    ts = c.ts
    try:
        return oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts)), None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _python(c):
    return P.generate_event_proof(c.blocks, c.ts, c.ts.event_signature, c.ts.topic1, c.ts.actor_filter)


def test_catalogue_counts(cases):
    got = {}
    for c in cases:
        got[kind(c)] = got.get(kind(c), 0) + 1
    assert got == COUNTS


def test_builder_shapes(cases):
    by = {c.name: c for c in cases}
    valid = by["valid"]
    names = {n: valid.amts[i] for i, n in valid.names.items()}
    for i, a in valid.amts.items():
        bw, h, count, node = cbor2.loads(valid.blocks[a.root])
        assert (bw, h) == (a.bw, a.height) and len(node[0]) == E.bmap_len(bw)
        assert bytes(valid.ts.events_roots[i]) == a.root and valid.ts.has_events_root[i]
    assert set(range(1, 9)) == {a.bw for a in valid.amts.values()}
    for bw in range(1, 9):
        assert {0, 1, 2, E.max_height(bw)} <= {a.height for a in valid.amts.values() if a.bw == bw}
    deep = names["bw1-h64-deepest"]
    assert deep.height == 64 and list(deep.values) == [2 ** 64 - 2] and len(deep.nodes) == 64
    # sparse sets hold matching and non-matching events, so an event's AMT index is not its ordinal among the matches
    sp = names["bw5-h2-sparse"]
    assert len(sp.values) >= 8 and min(sp.values) > 0
    # single-node roots: the header up to the values' first byte on both sides of pass 1's staged limit (48 bytes)
    sizes = set()
    for n, a in names.items():
        if "-single-" in n:
            raw = valid.blocks[a.root]
            hdr = len(raw) - sum(len(v) for v in a.values.values())
            sizes.add(hdr > 48)
            assert raw[1] == a.bw and not a.nodes
    assert sizes == {False, True}
    big = by["valid-big"]
    assert all(any(i >= 2 ** 64 for i in a.values) for a in big.amts.values()) and len(big.amts) == 8
    # overflow heights: h < 2^64, h·bw > 64 and h·bw mod 2^64 ≤ 64; the 70-deep chain of the issue's example is there
    for bw in range(2, 9):
        hs = E.overflow_heights(bw)
        assert hs and all(h < 2 ** 64 and h * bw > 64 and (h * bw) % 2 ** 64 <= 64 for h in hs)
    assert "wrap-bw5-h0x3333333333333334" in by
    assert not E.overflow_heights(1)
    # receipts AMTs: every height from the minimal one to 21, the HOLES absent from the chain but named by the RPC roots
    for h in range(3, 22):
        c = by[f"receipts-h{h}-holes"]
        assert cbor2.loads(c.blocks[bytes(c.ts.receipts_root)])[0] == h
        rec = E.chain_receipts(c.blocks, c.ts)
        assert all(i not in rec and c.ts.has_events_root[i] for i in E.HOLES) and len(rec) == int(c.ts.n_receipts) - len(E.HOLES)
    c = by["rpc-root-differs"]
    rec = E.chain_receipts(c.blocks, c.ts)
    assert bytes(cbor2.loads(rec[5])[3].value[1:]) != bytes(c.ts.events_roots[5])


def _truth_proofs(t):
    return [(i, j, em, tuple(tp), d, m) for i, j, em, tp, d, m in t["proofs"]]


def test_valid_cases_agree_with_both_oracles(oracle_mod, cases):
    n = 0
    for c in cases:
        if c.status is not None:
            continue
        t = E.truth(c)
        r, err = _oracle(oracle_mod, c)
        assert err is None, (c.name, err)
        py = _python(c)
        assert py["matching"] == t["matching"] == r.matching.tolist(), c.name
        assert [tuple(p) for p in py["proofs"]] == _truth_proofs(t), c.name
        assert set(py["witness"]) == t["witness"] == {bytes(x) for x in r.witness.cids}, c.name
        assert r.n_exec == t["n_exec"]
        if not c.big:
            assert [p.key() for p in r.proofs] == _truth_proofs(t), c.name
        else:
            # the C++ oracle's indices are the saturating ones: equal below 2^64, and the same proofs otherwise
            assert len(r.proofs) == len(t["proofs"])
            for p, q in zip(r.proofs, t["proofs"]):
                assert p.key()[:1] + p.key()[2:] == q[:1] + q[2:]
                if q[1] < 2 ** 64:
                    assert p.event_index == q[1]
        if c.name == "rpc-root-differs":
            # proofs come from the RPC's events roots; the verifier follows the chain's, whose blocks the witness does not hold
            with pytest.raises(A.IpcfpError) as e:
                oracle_mod.verify_event_proofs(r.witness, c.ts, r)
            assert e.value.status == A.ERR_MISSING_BLOCK
            n += 1
            continue
        v = oracle_mod.verify_event_proofs(r.witness, c.ts, r)
        if not c.big:
            assert v == E.honest_verdicts(c, r), c.name
        else:   # a wrapped index names another slot or nothing; below 2^64 − 1 the proofs verify
            assert all(ok for ok, q in zip(v, t["proofs"]) if q[1] < 2 ** 64 - 1) and not all(v), c.name
        n += 1
        if c.name == "valid":
            # event indices differ from the ordinal of the event among its AMT's matches
            ordinals = {}
            assert any(p.event_index != ordinals.setdefault(p.exec_index, []).__len__() or ordinals[p.exec_index].append(1)
                       for p in r.proofs)
            assert 2 ** 64 - 2 in {p.event_index for p in r.proofs}
            assert not all(E.honest_verdicts(c, r))
        if c.name.startswith("receipts-h"):
            # the holes match, their proofs are dropped
            assert set(E.HOLES) <= set(t["matching"]) and not {p.exec_index for p in r.proofs} & set(E.HOLES)
    assert n == COUNTS["valid"] + COUNTS["receipts"] + COUNTS["rpc"]


def test_fault_cases_fail_in_the_restatement_and_the_oracle(oracle_mod, cases):
    n = 0
    for c in cases:
        if c.status is None:
            continue
        with pytest.raises(E.Fault) as f:
            E.truth(c)
        assert f.value.status == c.status, c.name
        _, err = _oracle(oracle_mod, c)
        assert err is not None and err[0] == c.status, (c.name, err)
        if c.index is not None:
            assert err[1] == c.index, (c.name, err)
        n += 1
    assert n == sum(v for k, v in COUNTS.items() if k not in ("valid", "receipts", "rpc"))


def test_oracles_refuse_wrapping_heights(oracle_mod, cases):
    """height·bw ≤ 64 checked without the product: every root whose product wraps to ≤ 64 is a decode error in the C++ oracle at the
    receipt (events AMTs) or for the tipset (receipts and message AMTs), and the Python oracle refuses it too."""
    n = 0
    for c in cases:
        if kind(c) in ("wrap", "receipts-wrap", "message-wrap"):
            _, err = _oracle(oracle_mod, c)
            assert err is not None and err[0] == A.ERR_DECODE, (c.name, err)
            with pytest.raises(ValueError):
                _python(c)
            n += 1
    assert n == 352 + 43 + 43
