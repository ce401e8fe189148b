"""ipcfp_fetch_plan_to_rpc_json (include/ipcfp.h): the Filecoin.ChainReadObj batch of a fetch plan is Python's json.dumps of the same
batch (compact separators), with CIDs as multibase base32 strings. Host-side rendering: no device is needed."""
import base64
import json

import numpy as np
import pytest


from oracle import pyoracle as P


def _cid_str(c):
    return "b" + base64.b32encode(bytes(c)).decode().lower().rstrip("=")


@pytest.mark.parametrize("n,first_id", [(0, 0), (1, 0), (3, 7), (200, 2**63)])
def test_request_batch_is_json_dumps_of_the_batch(api, n, first_id):
    rng = np.random.default_rng(n)
    cids = np.zeros((n, 38), np.uint8)
    cids[:, :6] = np.frombuffer(P.CID_PREFIX, np.uint8)
    cids[:, 6:] = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    got = api.fetch_plan_to_rpc_json(cids, first_id)
    batch = [{"jsonrpc": "2.0", "method": "Filecoin.ChainReadObj", "params": [{"/": _cid_str(c)}], "id": first_id + k}
             for k, c in enumerate(cids)]
    assert got == json.dumps(batch, separators=(",", ":")).encode()


# ------------------------------------------------------------------------------------------ the per-item code on the CPU
def _cases_file(path, ts, blocks, sspecs, especs, cases):
    """tests/host_fuzz/emu_plan.cu's input: the block set, the tipset, the specs, then per case a keep mask and edited blocks."""
    import struct
    out = [struct.pack("<Q", len(blocks))]
    for c, b in blocks:
        out += [c, struct.pack("<I", len(b)), b]
    cat = lambda a: np.asarray(a, np.uint8).tobytes()   # noqa: E731
    out += [struct.pack("<I", int(ts.n_parents)), cat(ts.parent_cids), cat(ts.parent_txmeta_cids), cat(ts.child_cid), cat(ts.receipts_root),
            cat(ts.parent_state_root), struct.pack("<Q", int(ts.n_receipts)), cat(ts.events_roots), cat(ts.has_events_root)]
    out.append(struct.pack("<I", len(especs)))
    for sig, t1, _ in especs:
        out += [struct.pack("<I", len(sig)), sig.encode(), struct.pack("<I", len(t1)), t1.encode()]
    for _, _, actor in especs:
        out.append(struct.pack("<BQ", actor is not None, actor or 0))
    out.append(struct.pack("<I", len(sspecs)))
    for a, s in sspecs:
        out += [struct.pack("<Q", a), bytes(s)]
    out.append(struct.pack("<I", len(cases)))
    for keep, muts in cases:
        out += [bytes(keep.astype(np.uint8)), struct.pack("<I", len(muts))]
        for i, b in muts:
            out += [struct.pack("<QI", i, len(b)), b]
    open(path, "wb").write(b"".join(out))


@pytest.fixture(scope="module")
def plan_world(synth_mod):
    from tests import rpc_blocks as B
    ts = synth_mod.Tipset(synth_mod.config_params(3, hamt_entries=3000))
    cids, blocks = B.blocks_of(ts)
    pairs = [(bytes(c), b) for c, b in zip(cids, blocks)]
    keys = [bytes(ts.storage_entry(k)[0]) for k in (0, 1, 77)] + [bytes(ts.storage_absent_key(1))]
    sspecs = [(a, P.compute_mapping_slot(k, 0)) for a in (1001, 1002, 1003, 1004, 1005, 1006) for k in keys]
    especs = [(ts.event_signature, ts.topic1, None if ts.actor_filter is None else int(ts.actor_filter))]
    return ts, pairs, sspecs, especs


@pytest.mark.parametrize("sanitize", [False, True])
def test_per_item_code_on_the_cpu_matches_the_restatement(plan_world, tmp_path, sanitize):
    """csrc/plan_items.cuh compiled for the host and driven as csrc/plan.cu drives it (tests/host_fuzz/emu_plan.cu):
    * on seeded partial stores the plan equals tests/plan_rules.py's restatement, CID for CID, with the same needed count;
    * with a TxMeta, message- or events-AMT root or node, receipts-AMT, StateRoot, HAMT, EVM-state or contract-state block replaced by
      bytes that do not decode, the same; with such blocks truncated or with a byte flipped (where the planner may ask for more than
      the restatement, DESIGN.md §2), the planning loop converges without asking for a CID twice and the C++ oracle's bundle on the
      planned store equals its bundle on the whole block set (the same status and index, or the same witness);
    * under AddressSanitizer + UBSan (sanitize=True) the per-item code stays inside the padded buffers on all of them."""
    import random
    import subprocess
    from tests.plan_rules import restate_plan
    from tests.test_host_fuzz import _harness
    ts, pairs, sspecs, especs = plan_world
    exe, env = _harness("emu_plan", with_synth=False, sanitize=sanitize)
    full = dict(pairs)
    index = {c: i for i, (c, _) in reversed(list(enumerate(pairs)))}
    reads = set()
    st = {c: b for c, b in pairs}

    class Logged(dict):
        def get(self, c, d=None):
            reads.add(bytes(c))
            return super().get(c, d)
        __getitem__ = lambda self, c: (reads.add(bytes(c)), dict.__getitem__(self, c))[1]   # noqa: E731
        __contains__ = lambda self, c: (reads.add(bytes(c)), dict.__contains__(self, c))[1]   # noqa: E731

    lg = Logged(st)
    P.generate_event_proof(lg, ts, *especs[0])
    for a, s in sspecs:
        try:
            P.generate_storage_proof(lg, ts, a, s)
        except KeyError:
            pass
    rng = random.Random(5)
    n = len(pairs)
    targets = sorted(reads)
    targets = [bytes(ts.parent_txmeta_cids[0]), bytes(ts.receipts_root), bytes(ts.parent_state_root)] + rng.sample(targets, 21)
    cases, expect = [], []
    for frac in (0.0, 0.3, 0.6, 0.9, 0.98, 1.0):
        keep = np.array([rng.random() < frac for _ in range(n)])
        cases.append((keep, []))
        expect.append({c: full[c] for c, k in zip((c for c, _ in pairs), keep) if k})
    for c in targets:
        i = index[c]
        b = full[c]
        for kind in ("ff", "trunc", "flip"):
            new = b"\xff" if kind == "ff" else (b[:rng.randrange(len(b))] if kind == "trunc" else
                                               (lambda j: b[:j] + bytes([b[j] ^ (1 << rng.randrange(8))]) + b[j + 1:])(rng.randrange(len(b))))
            keep = np.array([rng.random() < 0.5 for _ in range(n)]) if kind == "ff" else np.ones(n, bool)
            cases.append((keep, [(i, new)]))
            if kind == "ff":
                held = {cc: full[cc] for cc, k in zip((cc for cc, _ in pairs), keep) if k}
                if c in held:
                    held[c] = new
                expect.append(held)
            else:
                expect.append(None)
    f = tmp_path / "cases.bin"
    _cases_file(str(f), ts, pairs, sspecs, especs, cases)
    out = subprocess.run([exe, str(f)], capture_output=True, text=True, env=env, timeout=1200)
    assert out.returncode == 0, (out.stdout[-2000:] + out.stderr[-3000:])
    assert "runtime error" not in out.stderr and "AddressSanitizer" not in out.stderr, out.stderr[-3000:]
    lines = out.stdout.splitlines()
    assert len(lines) == 2 * len(cases)
    compared = 0
    for q, held in enumerate(expect):
        tag, nn, *hexes = lines[2 * q].split(" ")
        assert tag == "plan" and lines[2 * q + 1].startswith("loop ")
        if held is None:
            continue
        got = bytes.fromhex(hexes[0]) if hexes and hexes[0] else b""
        exp, n_needed = restate_plan(held, ts, sspecs, especs)
        assert [got[38 * k:38 * k + 38] for k in range(len(got) // 38)] == exp, q
        assert int(nn) == n_needed, q
        compared += 1
    assert compared == 6 + len(targets)
    assert sum(int(lines[2 * q + 1].split()[2]) != 0 for q in range(len(cases))) > len(targets)   # the edits do produce failures
