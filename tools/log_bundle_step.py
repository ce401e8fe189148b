"""Proof bundles of log filters against the spec bundle on the 1 M-receipt tipset of bench.py (synthetic config 4, with a state tree),
resident store and tipset, one bundle call per step, the two arms alternating in one run:
  spec     ipcfp_generate_proof_bundle_resident with K event specs (the tipset's own, one without an actor filter, one that matches nothing)
  filter   ipcfp_generate_log_bundle_resident with the K filters LogFilter.from_spec gives for them
both with --storage storage specs and the given --flags. K runs over --ks. For each arm and K: the bundle's device time (ms_total, CUDA
events on the store's stream) and the host wall time of the call, median / min / max over --runs after --warmup. The two arms' JSON
texts (IPCFP_RESULT_JSON) are compared byte for byte once per K. Prints one JSON line with the card's name and power limit read in the
same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.json_step import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--receipts", type=int, default=1_000_000)
    ap.add_argument("--storage", type=int, default=16)
    ap.add_argument("--ks", default="1,2,3")
    ap.add_argument("--flags", type=int, default=0)
    args = ap.parse_args()
    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    name = card()
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts, with_state_tree=1, hamt_entries=20000))
    L = api.lib()
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    keys = [ts.storage_entry(k % 20000)[0] for k in range(args.storage)]
    slots = api.compute_mapping_slots(keys, [0] * len(keys)) if keys else []
    sspecs = [(1001 + k % 6, bytes(slots[k])) for k in range(args.storage)]
    all_specs = [api.EventProofSpec(ts.event_signature, ts.topic1, None if ts.actor_filter is None else int(ts.actor_filter)),
                 api.EventProofSpec(ts.event_signature, "calib-subnet-2", None), api.EventProofSpec("NoSuchEvent(bytes32)", "no-such-topic", None)]
    all_filters = [api.LogFilter.from_spec(s) for s in all_specs]
    sarr, ns, _, _ = store._bundle_specs(sspecs, [])

    def call(arm, k, flags):
        out = C.POINTER(A.BundleC)()
        t0 = time.perf_counter()
        if arm == "spec":
            _, _, earr, ne = store._bundle_specs([], all_specs[:k])
            st = L.ipcfp_generate_proof_bundle_resident(store._h, tip._h, sarr, ns, earr, ne, flags, C.byref(out))
        else:
            farr, nf, keep = api._log_filters_c(all_filters[:k])
            st = L.ipcfp_generate_log_bundle_resident(store._h, tip._h, sarr, ns, farr, nf, flags, C.byref(out))
        wall = (time.perf_counter() - t0) * 1e3
        assert st == 0, L.ipcfp_last_error()
        return out, wall

    stat = lambda xs: dict(median=round(statistics.median(xs), 4), min=round(min(xs), 4), max=round(max(xs), 4))   # noqa: E731
    out = dict(card=name, receipts=args.receipts, storage_specs=args.storage, flags=args.flags, ks={})
    for k in (int(x) for x in args.ks.split(",")):
        texts = {}
        for arm in ("spec", "filter"):
            o, _ = call(arm, k, A.RESULT_JSON)
            texts[arm] = C.string_at(o.contents.json, int(o.contents.json_len))
            L.ipcfp_bundle_free(o)
        dev = {"spec": [], "filter": []}
        wall = {"spec": [], "filter": []}
        proofs = 0
        for r in range(args.warmup + args.runs):
            for arm in (("spec", "filter") if r % 2 == 0 else ("filter", "spec")):
                o, w = call(arm, k, args.flags)
                b = o.contents
                proofs = sum(int(b.events[q].contents.n_proofs) for q in range(int(b.n_event_results)))
                if r >= args.warmup:
                    dev[arm].append(b.ms_total)
                    wall[arm].append(w)
                L.ipcfp_bundle_free(o)
        out["ks"][k] = dict(event_proofs=proofs, json_equal=texts["spec"] == texts["filter"], json_bytes=len(texts["spec"]),
                            **{f"{arm}_device_ms": stat(dev[arm]) for arm in dev}, **{f"{arm}_wall_ms": stat(wall[arm]) for arm in wall})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
