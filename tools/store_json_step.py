"""The block store from Filecoin.ChainReadObj JSON-RPC responses, routes alternated in one process on the same blocks (the 1 M-receipt
tipset's ≈ 1.3 M blocks by default), the responses rendered in three shapes: one batch text, batches of 10 000 (shuffled), one object per
text (shuffled). Per shape:
  device          ipcfp_store_create_rpc_json, without and with IPCFP_STORE_VERIFY_CIDS (parsed on the device);
  host            ipcfp_blocks_from_rpc_json, then ipcfp_store_create (without the flag);
and, as the floor, ipcfp_store_create from the binary arrays, without and with the flag. Every store call returns after the device has
finished; each timing also ends with a device synchronisation. Prints one JSON line: median / min / max wall ms per route, the device
path's parse-kernel time, and the card's name and power limit read in the same run. Every store must hold the same blocks."""
import argparse
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
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--host-runs", type=int, default=1)
    ap.add_argument("--receipts", type=int, default=1_000_000)
    args = ap.parse_args()
    import numpy as np
    import torch

    import synth
    from ipc_filecoin_proofs_b200 import api
    from tests import rpc_blocks as B
    name = card()
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts))
    cids, blocks = B.blocks_of(ts)
    els = [B.element(i, d) for i, d in enumerate(blocks)]
    shuffled = [els[k] for k in np.random.default_rng(1).permutation(len(els))]
    del els
    shapes = {
        "one_batch": lambda: [b"[" + b",".join(shuffled) + b"]"],
        "batches_of_10000": lambda: [b"[" + b",".join(shuffled[a:a + 10000]) + b"]" for a in range(0, len(shuffled), 10000)],
        "one_object_per_text": lambda: shuffled,
    }
    sample = np.random.default_rng(3).choice(len(cids), 200, replace=False)
    ref = api.BlockStore.from_tipset(ts)
    want = {int(i): ref.get(cids[i]) for i in sample}

    def timed(fn, runs, warmup, check=None):
        out, kern = [], []
        for k in range(warmup + runs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = fn()
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) * 1e3
            if k == 0 and check:
                check(st)
            if k >= warmup:
                out.append(dt)
                if hasattr(st, "json_info"):
                    kern.append(st.json_info.ms_kernels)
            st.close()
        r = dict(median_ms=round(statistics.median(out), 2), min_ms=round(min(out), 2), max_ms=round(max(out), 2), runs=len(out))
        if kern:
            r["kernels_median_ms"] = round(statistics.median(kern), 3)
        return r

    def same(st):
        for i, b in want.items():
            assert st.get(cids[i]) == b

    def host_route(texts):
        w = api.blocks_from_rpc_json(cids, texts)
        return api.BlockStore(w.cids, w.offsets, w.lengths, w.blob)

    res = {"card": name, "n_blocks": len(cids), "block_bytes": int(sum(len(b) for b in blocks)), "routes": {}}
    floor = res["routes"]
    floor["binary_store_create"] = timed(lambda: api.BlockStore(ts.cids, ts.offsets, ts.lengths, ts.blob), args.runs, args.warmup, same)
    floor["binary_store_create_verify"] = timed(lambda: api.BlockStore(ts.cids, ts.offsets, ts.lengths, ts.blob, verify_cids=True), args.runs,
                                                args.warmup, same)
    for shape, make in shapes.items():
        texts = make()
        res.setdefault("text_bytes", {})[shape] = int(sum(len(t) for t in texts))

        def dev(verify, texts=texts):
            st = api.BlockStore.from_rpc_json(cids, texts, verify_cids=verify)
            assert st.json_info.parsed_on_device
            return st
        floor[f"{shape}/device"] = timed(lambda: dev(False), args.runs, args.warmup, same)
        floor[f"{shape}/device_verify"] = timed(lambda: dev(True), args.runs, args.warmup, same)
        floor[f"{shape}/host"] = timed(lambda: host_route(texts), args.host_runs, 0, same)
        del texts
    print(json.dumps(res))


if __name__ == "__main__":
    main()
