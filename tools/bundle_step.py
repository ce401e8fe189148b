#!/usr/bin/env python
"""What the UnifiedProofBundle costs on the 1 M-receipt tipset (BASELINE.json configs[3]) with a state tree, 16 storage specs and 2 event
specs, store resident. Usage: python tools/bundle_step.py [--receipts N] [--steps K] [--warmup W]

Four arms, alternated step by step in one process after W warm-up rounds of each:
  1 ipcfp_generate_proof_bundle (uploads the tipset), then ipcfp_bundle_to_json on the host: the route without the resident call
  2 ipcfp_generate_proof_bundle_resident, flags 0
  3 ipcfp_generate_proof_bundle_resident, RESULT_JSON
  4 ipcfp_generate_proof_bundle_resident, RESULT_JSON | WITNESS_BY_REFERENCE
For every arm: median / min / max wall time per step until the results (and, for 1, 3 and 4, the text) are on the host, ms_total and
ms_json (device time, CUDA events; arm 1's ms_total is its bundle call). Arms 1, 3 and 4 must give equal bytes (exit code 1 otherwise).
Prints the card's name and power limit."""
import argparse
import ctypes as C
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.json_step import card  # noqa: E402

EVM_ACTORS = (1001, 1002, 1003, 1004, 1005, 1006)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receipts", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts, with_state_tree=1, hamt_entries=20000))
    keys = [ts.storage_entry(k)[0] for k in (0, 1, 2, 77, 500, 19999)] + [ts.storage_absent_key(k) for k in (1, 2)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys))
    sspecs = [(EVM_ACTORS[k % 6], slots[k % len(slots)]) for k in range(16)]
    especs = [A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter), A.make_event_spec(ts.event_signature, "calib-subnet-2", None)]
    L = api.lib()
    store = api.BlockStore.from_tipset(ts)
    sarr, ns, earr, ne = store._bundle_specs(sspecs, especs)
    d, keep = A.make_tipset_desc(ts)
    tip = store.upload_tipset(ts)
    arms = [("plain + host to_json", None), ("resident flags 0", 0), ("resident RESULT_JSON", A.RESULT_JSON),
            ("resident RESULT_JSON|WITNESS_BY_REF", A.RESULT_JSON | A.WITNESS_BY_REFERENCE)]
    wall = {a[0]: [] for a in arms}
    dev = {a[0]: [] for a in arms}
    djs = {a[0]: [] for a in arms}
    texts = {}
    sizes = {}

    def step(name, flags, keep_text):
        out = C.POINTER(A.BundleC)()
        text_p, n = C.c_void_p(), C.c_uint64()
        t0 = time.perf_counter()
        if flags is None:
            api._check(L.ipcfp_generate_proof_bundle(store._h, C.byref(d), sarr, ns, earr, ne, C.byref(out)))
            api._check(L.ipcfp_bundle_to_json(out, C.byref(d), C.byref(text_p), C.byref(n)))
        else:
            api._check(L.ipcfp_generate_proof_bundle_resident(store._h, tip._h, sarr, ns, earr, ne, flags, C.byref(out)))
        t1 = time.perf_counter()
        b = out.contents
        if keep_text:
            texts[name] = C.string_at(text_p.value, n.value) if flags is None else (C.string_at(b.json, b.json_len) if b.json else None)
            sizes[name] = (int(b.witness.n_blocks), int(b.witness.blob_size), sum(int(b.events[k].contents.n_proofs) for k in range(ne)))
        if flags is None:
            L.ipcfp_json_free(text_p)
        res = (1e3 * (t1 - t0), float(b.ms_total), float(b.ms_json))
        L.ipcfp_bundle_free(out)
        return res

    for _ in range(args.warmup):
        for name, flags in arms:
            step(name, flags, False)
    for k in range(args.steps):
        for name, flags in arms:
            w, t, j = step(name, flags, k == 0)
            wall[name].append(w); dev[name].append(t); djs[name].append(j)
    tip.close()
    ref = texts["plain + host to_json"]
    same = ref == texts["resident RESULT_JSON"] == texts["resident RESULT_JSON|WITNESS_BY_REF"]
    m, blob, n_ev = sizes["resident flags 0"]
    print(f"card: {card()}")
    print(f"receipts {args.receipts}, {ts.n_blocks} blocks in the store; {ns} storage specs, {ne} event specs ({n_ev} event proofs); union "
          f"{m} blocks, {blob} witness blob bytes; JSON {len(ref)} bytes, arms 1/3/4 byte-equal: {same}; {args.steps} steps per arm after "
          f"{args.warmup} warm-up rounds, alternated")
    print(f"{'arm':40s} {'wall ms median [min, max]':>30s} {'ms_total median':>16s} {'ms_json median':>15s}")
    for name, _ in arms:
        w = wall[name]
        print(f"{name:40s} {statistics.median(w):12.3f} [{min(w):7.3f}, {max(w):7.3f}] {statistics.median(dev[name]):16.3f} "
              f"{statistics.median(djs[name]):15.3f}")
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
