"""The logs of given messages on the 1 M-receipt tipset of bench.py (synthetic config 4), resident store and tipset, one call per step:
  log               ipcfp_generate_log_proof_resident with the filter (every receipt's events AMT is read)
  msgs=1, msgs=1000, msgs=65536
                    ipcfp_generate_message_log_proof_resident with the same filter and that many messages drawn from the execution order
                    (65 536 is IPCFP_MESSAGE_MAX, a call's cap; the whole order of 1 M messages takes 16 calls)
for the spec's filter (--filter spec, the default) or the all-wildcard filter (--filter all). For each: the selection / pass 1 part
(ms_pass1: from the execution order to the matching list), the message-AMT walk and dedup (ms_txamt) and the whole step (ms_total),
device time from CUDA events on the store's stream, median / min / max over --runs after --warmup, and the matching receipts and proofs.
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.json_step import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--receipts", type=int, default=1_000_000)
    ap.add_argument("--filter", choices=["spec", "all"], default="spec")
    args = ap.parse_args()
    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    name = card()
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts))
    L = api.lib()
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    spec = api.EventProofSpec(ts.event_signature, ts.topic1, None if ts.actor_filter is None else int(ts.actor_filter))
    flt = api.LogFilter.from_spec(spec) if args.filter == "spec" else api.LogFilter()
    f, fkeep = flt.as_c()
    # the execution order from the all-wildcard result: every receipt of this tipset has a matching event
    out = C.POINTER(A.EventResultC)()
    wf, wkeep = api.LogFilter().as_c()
    assert L.ipcfp_generate_log_proof_resident(store._h, tip._h, C.byref(wf), 0, C.byref(out)) == 0, L.ipcfp_last_error()
    r = out.contents
    n = int(r.n_proofs)
    raw = A._arr(C.cast(r.proofs, C.c_void_p).value, n * C.sizeof(A.EventProofC), np.uint8).reshape(n, C.sizeof(A.EventProofC))
    ex = raw[:, A.EventProofC.exec_index.offset:A.EventProofC.exec_index.offset + 8].copy().view(np.uint64).ravel()
    _, first = np.unique(ex, return_index=True)
    o = A.EventProofC.message_cid.offset
    order = np.ascontiguousarray(raw[first, o:o + 38])
    L.ipcfp_event_result_free(out)
    rng = np.random.default_rng(1)
    cases = {"log": None}
    for k in (1, 1000, A.MESSAGE_MAX):
        cases["msgs=%d" % k] = np.ascontiguousarray(order[np.sort(rng.choice(len(order), size=min(k, len(order)), replace=False))])

    def call(cids):
        out = C.POINTER(A.EventResultC)()
        if cids is None:
            st = L.ipcfp_generate_log_proof_resident(store._h, tip._h, C.byref(f), 0, C.byref(out))
        else:
            idx = np.zeros(len(cids), np.uint64)
            st = L.ipcfp_generate_message_log_proof_resident(store._h, tip._h, cids.ctypes.data, len(cids), C.byref(f), 0, idx.ctypes.data,
                                                             C.byref(out))
        assert st == 0, L.ipcfp_last_error()
        return out

    stat = lambda xs: dict(median=round(statistics.median(xs), 4), min=round(min(xs), 4), max=round(max(xs), 4))   # noqa: E731
    res = dict(card=name, receipts=args.receipts, filter=args.filter, cases={})
    for label, cids in cases.items():
        p1, tx, tot = [], [], []
        for k in range(args.warmup + args.runs):
            o = call(cids)
            r = o.contents
            if k >= args.warmup:
                p1.append(r.ms_pass1)
                tx.append(r.ms_txamt)
                tot.append(r.ms_total)
            if k == 0:
                res["cases"][label] = dict(matching=int(r.n_matching), proofs=int(r.n_proofs), witness_blocks=int(r.witness.n_blocks))
            L.ipcfp_event_result_free(o)
        res["cases"][label].update(txamt_ms=stat(tx), pass1_ms=stat(p1), total_ms=stat(tot))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
