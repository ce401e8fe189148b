"""Message proofs on the 1 M-receipt tipset of bench.py (synthetic config 4), resident store and tipset, one call per step:
  msgs=1, msgs=1000, msgs=65536
      ipcfp_generate_message_proofs_resident, receipt only (the synthetic message CIDs have no blocks, so IPCFP_MESSAGE_WITH_BODY cannot
      run here), on that many messages drawn from the execution order (65 536 is IPCFP_MESSAGE_MAX, a call's cap), beside
      ipcfp_generate_message_log_proof_resident with the all-wildcard filter on the same CIDs, which runs the same execution-order walk
      and selection and then reads the selected receipts' events.
For each: device time from CUDA events on the store's stream — the message-proof call's total and its phases (exec_order: the walk, the
dedup and the selection; walk: the per-request receipts-AMT gets; gather: the data blob; witness), the message-log call's total and its
walk (txamt) — median / min / max over --runs after --warmup, and the host synchronisations. Before timing, every proof is checked:
executed, exec_index equal to the message-log call's, events root equal to the tipset's receipt list. Prints one JSON line with the
card's name and power limit read in the same run."""
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
    args = ap.parse_args()
    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    name = card()
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts))
    L = api.lib()
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
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
    cases = {"msgs=%d" % k: np.ascontiguousarray(order[rng.choice(len(order), size=min(k, len(order)), replace=False)])
             for k in (1, 1000, A.MESSAGE_MAX)}

    def proofs(cids):
        out = C.POINTER(A.MessageResultC)()
        assert L.ipcfp_generate_message_proofs_resident(store._h, tip._h, cids.ctypes.data, len(cids), 0, C.byref(out)) == 0, L.ipcfp_last_error()
        return out

    def message_log(cids):
        out = C.POINTER(A.EventResultC)()
        idx = np.zeros(len(cids), np.uint64)
        assert L.ipcfp_generate_message_log_proof_resident(store._h, tip._h, cids.ctypes.data, len(cids), C.byref(wf), 0, idx.ctypes.data,
                                                           C.byref(out)) == 0, L.ipcfp_last_error()
        return out, idx

    stat = lambda xs: dict(median=round(statistics.median(xs), 4), min=round(min(xs), 4), max=round(max(xs), 4))   # noqa: E731
    res = dict(card=name, receipts=args.receipts, mode="receipt only", cases={})
    for label, cids in cases.items():
        o = proofs(cids)
        got = A.message_result_from_c(o.contents)
        L.ipcfp_message_result_free(o)
        lo, idx = message_log(cids)
        L.ipcfp_event_result_free(lo)
        for p, i in zip(got.proofs, idx):
            assert p.status == A.MESSAGE_EXECUTED and p.exec_index == int(i), label
            assert p.events_root == (bytes(ts.events_roots[int(i)]) if ts.has_events_root[int(i)] else None), label
        res["cases"][label] = dict(proofs=len(got.proofs), witness_blocks=int(got.witness.n_blocks), data_blob_bytes=len(got.data_blob),
                                   host_syncs=got.host_syncs)
        t = {k: [] for k in ("total", "exec_order", "walk", "gather", "witness", "log_total", "log_txamt")}
        for k in range(args.warmup + args.runs):
            o = proofs(cids)
            r = o.contents
            if k >= args.warmup:
                for f in ("total", "exec_order", "walk", "gather", "witness"):
                    t[f].append(getattr(r, "ms_" + f))
            L.ipcfp_message_result_free(o)
            lo, _ = message_log(cids)
            r = lo.contents
            if k >= args.warmup:
                t["log_total"].append(r.ms_total)
                t["log_txamt"].append(r.ms_txamt)
            L.ipcfp_event_result_free(lo)
        res["cases"][label].update({k + "_ms": stat(v) for k, v in t.items()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
