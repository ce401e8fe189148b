"""tests/arena_layouts.py on the CPU: the layouts hold the fixture's blocks at their new offsets, and the C++ oracle (whose
MemoryBlockstore::get clones exactly `len` bytes, so it is length-exact by construction) gives identical results on every layout of
configs 1 and 2; a block shortened in place gives the Python oracle's outcome on a store holding exactly the cut bytes — the expectation
the GPU must meet."""
import hashlib

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import arena_layouts as L
from tests.util import spec_of


def _hashes_to_cid(cid, data):
    cid = bytes(cid)
    if cid[2:4] == b"\xa0\xe4":
        return hashlib.blake2b(data, digest_size=32).digest() == cid[6:]
    if cid[2:4] == b"\xe0\xe4":
        return hashlib.blake2s(data, digest_size=32).digest() == cid[6:]
    return True


def _layouts(ts):
    for filler in L.FILLERS:
        for order in ("index", "shuffled"):
            yield f"{filler}-{order}", L.lay_out(ts.cids, ts.offsets, ts.lengths, ts.blob, filler=filler, order=order, seed=3)
    yield "residues", L.lay_out(ts.cids, ts.offsets, ts.lengths, ts.blob, filler="random", residues=True, tail=0, seed=4)
    yield "residues-next", L.lay_out(ts.cids, ts.offsets, ts.lengths, ts.blob, filler="next", residues=True, tail=0, seed=4)


def _outcome(fn):
    try:
        return fn(), None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _key(r):
    return (r.matching.tolist(), r.n_exec, [p.key() for p in r.proofs], r.witness.cids.tobytes(), r.witness.blocks(), r.data_blob.tobytes())


@pytest.mark.parametrize("cfg", [1, 2])
def test_layouts_hold_the_blocks_and_the_oracle_ignores_the_gaps(synth_mod, oracle_mod, cfg):
    ts = synth_mod.Tipset(synth_mod.config_params(cfg))
    exp = _key(oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts)))
    blocks = L.blocks_of(ts)
    for name, lay in _layouts(ts):
        assert lay.n_blocks == ts.n_blocks and np.array_equal(lay.lengths, ts.lengths), name
        assert [lay.block(i) for i in range(lay.n_blocks)] == blocks, name
        assert all(_hashes_to_cid(lay.cids[i], lay.block(i)) for i in range(lay.n_blocks)), name
        if name.startswith("residues"):
            placed = np.argsort(lay.offsets, kind="stable")
            assert {int(lay.offsets[i]) % 16 for i in placed} == set(range(16)), name
            assert int(lay.offsets[placed[-1]]) + int(lay.lengths[placed[-1]]) == len(lay.blob), name
        if name.endswith("-index"):
            assert all(int(lay.offsets[i]) >= int(lay.offsets[i - 1]) + int(lay.lengths[i - 1]) for i in range(1, lay.n_blocks)), name
        t = lay.over(ts)
        assert _key(oracle_mod.Store.from_tipset(t).generate_event_proof(t, spec_of(t))) == exp, name


def _py_outcome(blocks, ts):
    """The Python oracle (oracle/pyoracle.py, an independent restatement over a {cid: bytes} dict) → (matching, proofs, witness) or
    None when it fails (a decode error, a missing block or a missing message)."""
    from oracle import pyoracle as P
    try:
        r = P.generate_event_proof(blocks, ts, ts.event_signature, ts.topic1, ts.actor_filter)
    except Exception:
        return None
    return r["matching"], r["proofs"], r["witness"]


def test_shortened_in_place_equals_the_exact_size_block(synth_mod, oracle_mod):
    """Every block of the config-1 event call's read set, cut to each length of arena_layouts.shorten_lengths in place (its removed
    suffix, then an echo of it, follows in the arena): the C++ oracle on those arrays gives the outcome the Python oracle gives on a
    dict holding exactly the k bytes — success with the same matches, proofs and witness, or a failure. This is the expectation the
    GPU's group B meets on the same arrays."""
    ts = synth_mod.Tipset(synth_mod.config_params(1))
    lay = L.lay_out(ts.cids, ts.offsets, ts.lengths, ts.blob, filler="echo")
    full = oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts))
    index = {bytes(c): i for i, c in enumerate(lay.cids)}
    base = {bytes(lay.cids[i]): lay.block(i) for i in range(lay.n_blocks)}
    runs = errors = 0
    for c in full.witness.cids:
        i = index[bytes(c)]
        for k in L.shorten_lengths(int(lay.lengths[i])):
            s = L.shortened(lay, i, k)
            got, gerr = _outcome(lambda: oracle_mod.Store.from_tipset(s.over(ts)).generate_event_proof(s.over(ts), spec_of(ts)))
            exact = dict(base)
            exact[bytes(c)] = s.block(i)
            assert len(exact[bytes(c)]) == k
            exp = _py_outcome(exact, ts)
            assert (gerr is None) == (exp is not None), (i, k, gerr)
            if exp is not None:
                assert got.matching.tolist() == exp[0], (i, k)
                assert [(p.exec_index, p.event_index, p.emitter, tuple(p.topics), p.data, p.message_cid) for p in got.proofs] == exp[1], (i, k)
                assert [bytes(x) for x in got.witness.cids] == exp[2], (i, k)
            runs += 1
            errors += gerr is not None
    assert runs > 200 and errors > runs // 2, (runs, errors)


def test_chunked_layout_cuts_where_it_says():
    """The cut rule of ipcfp_store_create's chunked ingest applied to arena_layouts.chunked: chunk 0 = [0, 129) ending exactly at
    64 MiB, chunk 1 starting with a zero-length block and cut at the straddling block, a zero-length last block at blob_size."""
    import synth
    ts = synth.Tipset(synth.config_params(2))
    lay, info = L.chunked(ts.cids, ts.offsets, ts.lengths, ts.blob)
    assert L.first_bad_b2b(lay) is None and len(lay.blob) > 128 << 20
    byte0, cuts = 0, []
    for i in range(lay.n_blocks):
        end = int(lay.offsets[i]) + int(lay.lengths[i])
        assert i == 0 or int(lay.offsets[i]) >= int(lay.offsets[i - 1]) + int(lay.lengths[i - 1])
        if end - byte0 >= 64 << 20 and i + 1 < lay.n_blocks:
            cuts.append(i + 1)
            byte0 = int(lay.offsets[i + 1])
    assert cuts == [129, info["straddle"] + 1]
    assert int(lay.offsets[128]) + int(lay.lengths[128]) == 64 << 20
    assert int(lay.lengths[129]) == 0 and info["first_of_chunk1"] == 130
    s = info["straddle"]
    assert int(lay.offsets[s]) < int(lay.offsets[129]) + (64 << 20) < int(lay.offsets[s]) + int(lay.lengths[s])
    assert int(lay.lengths[-1]) == 0 and int(lay.offsets[-1]) == len(lay.blob)


def test_far_layout_places_blocks_past_4_gib(synth_mod):
    ts = synth_mod.Tipset(synth_mod.config_params(1))
    roots = {bytes(ts.events_roots[i]) for i in range(int(ts.n_receipts)) if ts.has_events_root[i]}
    low = [i for i in range(ts.n_blocks) if bytes(ts.cids[i]) not in roots][:3]
    blocks = dict(zip((bytes(c) for c in ts.cids), L.blocks_of(ts)))
    for straddle32, order in ((False, "index"), (True, "shuffled")):
        lay = L.far(ts.cids, ts.offsets, ts.lengths, ts.blob, low, order=order, straddle32=straddle32)
        assert len(lay.blob) == L.FAR_SIZE
        assert all(lay.block(i) == blocks[bytes(lay.cids[i])] for i in range(lay.n_blocks))
        o, n = lay.offsets.astype(np.int64), lay.lengths.astype(np.int64)
        assert o[0] < 1 << 31 < o[0] + n[0]
        if straddle32:
            assert o[1] < 1 << 32 < o[1] + n[1]
        else:
            assert o[1] + n[1] == 1 << 32 and o[2] == 1 << 32
        assert all(o[k] >= 1 << 32 for k in range(2, lay.n_blocks))
        assert all(o[k] >= 1 << 32 for k in range(lay.n_blocks) if bytes(lay.cids[k]) in roots)
        del lay
