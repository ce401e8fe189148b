"""The GPU event path on the varied event shapes of the synthetic builder (event_shapes = 1) at sizes where the kernels change
behaviour: several faults at once in different pass-1 CTAs, and pass 2 on either side of its one-match-per-warp / one-per-thread switch.
Pass 1 sizes pass 2's output (per-receipt proof and byte counts → bases), so a count that disagrees with pass 2's walk on some shape would
corrupt results; every case is compared with the CPU oracle."""
import collections

import cbor2
import numpy as np
import pytest

from tests.test_gpu_parity import _both
from tests.util import EditedTipset, assert_event_results_equal, spec_of

pytestmark = pytest.mark.gpu

PASS1_CTA = 128          # receipts per k_pass1_stage CTA (events.cu)
PASS2_PER_WARP_MAX = 16384


@pytest.fixture(scope="session")
def shapes20k(synth_mod):
    return synth_mod.Tipset(synth_mod.default_params(event_shapes=1, seed=0x5A1, n_receipts=20000, events_per_receipt=12, match_ppm=80000))


@pytest.fixture(scope="session")
def shapes33k(synth_mod):
    return synth_mod.Tipset(synth_mod.default_params(event_shapes=1, seed=0x5A2, n_receipts=33000, events_per_receipt=8, match_ppm=600000))


def receipt_leaf(d, root_cid, i):
    """CID of the receipts-AMT leaf (AMT v0, bit width 3) that holds receipt i."""
    height, _, node = cbor2.loads(d[root_cid])
    cid = root_cid
    for h in range(height, 0, -1):
        bmap, links, _ = node
        slot = (i >> (3 * h)) & 7
        cid = links[bin(bmap[0] & ((1 << slot) - 1)).count("1")].value[1:]
        node = cbor2.loads(d[cid])
    return cid


def faulted(ts, index_of, d, rng, drop_leaf, tail_flips=False):
    """ts with the events roots of 2-8 receipts in different pass-1 CTAs damaged — a bit flipped, a byte inserted or deleted, or the
    block dropped — (half of them matching receipts where the CTA has one), and with drop_leaf also the receipts-AMT leaf of a
    matching receipt dropped. tail_flips: every damage is a bit flip in the last 8 bytes (mostly event data: often still valid).
    Only roots no other receipt shares are damaged. Damaged blocks keep their CIDs (the store does not re-hash them)."""
    n = int(ts.n_receipts)
    sel = set(ts.selected.tolist())
    uses = collections.Counter(bytes(ts.events_roots[i]) for i in range(n) if ts.has_events_root[i])
    ctas = rng.choice((n + PASS1_CTA - 1) // PASS1_CTA, size=int(rng.integers(2, 9)), replace=False)
    drop, patch, what = set(), {}, []
    for c in ctas:
        lo, hi = int(c) * PASS1_CTA, min(n, (int(c) + 1) * PASS1_CTA)
        cand = [i for i in range(lo, hi) if ts.has_events_root[i] and uses[bytes(ts.events_roots[i])] == 1]
        hits = [i for i in cand if i in sel]
        i = int(rng.choice(hits if hits and rng.integers(0, 2) else cand))
        k = index_of[bytes(ts.events_roots[i])]
        b = ts.block(k)
        at = int(rng.integers(max(0, len(b) - 8) if tail_flips else 0, len(b)))
        op = 0 if tail_flips else int(rng.integers(0, 4))
        if op == 0:
            b = b[:at] + bytes([b[at] ^ (1 << int(rng.integers(0, 8)))]) + b[at + 1:]
        elif op == 1:
            b = b[:at] + bytes([int(rng.integers(0, 256))]) + b[at:]
        elif op == 2:
            b = b[:at] + b[at + 1:]
        else:
            drop.add(k)
        if op < 3:
            patch[k] = b
        what.append((i, ("flip", "insert", "delete", "drop")[op], at))
    if drop_leaf:
        i = int(rng.choice(ts.selected))
        drop.add(index_of[receipt_leaf(d, bytes(ts.receipts_root), i)])
        what.append((i, "drop receipts leaf", None))
    offs, lens = ts.offsets.copy(), ts.lengths.copy()
    extra = bytearray()
    base = len(ts.blob)
    for k, b in patch.items():
        extra += bytes((16 - (base + len(extra)) % 16) % 16)
        offs[k], lens[k] = base + len(extra), len(b)
        extra += b
    extra += bytes(32)
    keep = [k for k in range(int(ts.n_blocks)) if k not in drop]
    blob = np.concatenate([ts.blob, np.frombuffer(bytes(extra), dtype=np.uint8)])
    return EditedTipset(ts, cids=ts.cids[keep], offsets=offs[keep], lengths=lens[keep], blob=blob, n_blocks=len(keep)), what


def test_multi_fault_error_parity_across_ctas(api, oracle_mod, shapes20k):
    """Each variant gives the oracle's (status, index), or when the oracle succeeds, the oracle's result in every field."""
    ts = shapes20k
    spec = spec_of(ts)
    index_of = {}
    for k in range(int(ts.n_blocks)):
        index_of.setdefault(bytes(ts.cids[k]), k)
    d = ts.as_dict()
    n_err = n_ok = 0
    for v in range(30):
        rng = np.random.default_rng(1000 + v)
        e, what = faulted(ts, index_of, d, rng, drop_leaf=v % 3 == 2, tail_flips=v % 5 == 4)
        o, g = _both(api, oracle_mod, e, spec)
        assert o[0] == g[0], (v, what, o, g)
        if o[0] == "ok":
            n_ok += 1
            assert_event_results_equal(g[1], o[1])
        else:
            n_err += 1
            assert o[1:] == g[1:], (v, what, o, g)
    assert n_err >= 10 and n_ok >= 1, (n_err, n_ok)


@pytest.mark.parametrize("m", [PASS2_PER_WARP_MAX, PASS2_PER_WARP_MAX + 1])
def test_pass2_at_its_per_warp_threshold(api, oracle_mod, shapes33k, monkeypatch, m):
    """Exactly 16 384 (one match per warp) and 16 385 (one per thread) matching receipts, without any environment override."""
    monkeypatch.delenv("IPCFP_PASS2_PER_THREAD", raising=False)
    ts = shapes33k
    sel = ts.selected
    assert len(sel) > m
    has = ts.has_events_root.copy()
    has[int(sel[m]):] = 0
    e = EditedTipset(ts, has_events_root=has)
    exp = oracle_mod.Store.from_tipset(e).generate_event_proof(e, spec_of(e))
    got = api.BlockStore.from_tipset(e).generate_event_proof(e, spec_of(e))
    assert got.matching.tolist() == sel[:m].tolist()
    assert_event_results_equal(got, exp)
