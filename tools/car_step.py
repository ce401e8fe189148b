"""The block store from a CARv1, routes alternated in one process on the same blocks (the 1 M-receipt tipset's ≈ 1.3 M blocks by default,
written as one CAR in store order):
  car_pinned / car_pinned_verify       ipcfp_store_create_car from pinned memory (ipcfp_host_alloc), without and with IPCFP_STORE_VERIFY_CIDS;
  car_pageable / car_pageable_verify   the same from pageable memory;
  host_pinned / host_pageable          ipcfp_blocks_from_car, then ipcfp_store_create over the CAR (without the flag);
  binary / binary_verify               the floor: ipcfp_store_create from the binary arrays, without and with the flag.
Every timing ends with a device synchronisation; a warm-up round of every route comes first, then the routes take turns. Prints one JSON
line: median / min / max wall ms per route, the device path's parse-kernel time (ms_kernels of ipcfp_store_json_info), and the card's
name and power limit read in the same run, and which path found the sections (parsed_on_device). Every store must hold the same
blocks."""
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
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--receipts", type=int, default=1_000_000)
    args = ap.parse_args()
    import numpy as np
    import torch

    import synth
    from ipc_filecoin_proofs_b200 import api
    from tests import car_files as F
    name = card()
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts))
    car = F.write(F.of_tipset(ts))
    pinned = api.PinnedArray(len(car))
    pinned.array[:] = np.frombuffer(car, np.uint8)
    cids = np.asarray(ts.cids, np.uint8).reshape(-1, 38)
    sample = np.random.default_rng(3).choice(len(cids), 200, replace=False)
    ref = api.BlockStore.from_tipset(ts)
    want = {int(i): ref.get(cids[i]) for i in sample}
    ref.close()

    def from_car(src, verify):
        st = api.BlockStore.from_car(src, verify_cids=verify)
        paths.add(bool(st.car_info.parsed_on_device))
        return st

    def host(src):
        w = api.blocks_from_car(src)
        return api.BlockStore(w.cids, w.offsets, w.lengths, w.blob)

    routes = {
        "car_pinned": lambda: from_car(pinned.array, False),
        "car_pinned_verify": lambda: from_car(pinned.array, True),
        "car_pageable": lambda: from_car(car, False),
        "car_pageable_verify": lambda: from_car(car, True),
        "host_pinned": lambda: host(pinned.array),
        "host_pageable": lambda: host(car),
        "binary": lambda: api.BlockStore(ts.cids, ts.offsets, ts.lengths, ts.blob),
        "binary_verify": lambda: api.BlockStore(ts.cids, ts.offsets, ts.lengths, ts.blob, verify_cids=True),
    }
    paths = set()
    times = {r: [] for r in routes}
    kern = {r: [] for r in routes}
    parse = {r: [] for r in routes}
    for k in range(args.runs + 1):   # round 0 is the warm-up
        for r, fn in routes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = fn()
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) * 1e3
            if k == 0:
                for i, b in want.items():
                    assert st.get(cids[i]) == b, r
            else:
                times[r].append(dt)
                if hasattr(st, "car_info"):
                    kern[r].append(st.car_info.ms_kernels)
                    parse[r].append(st.car_info.ms_parse)
            st.close()
    res = {"card": name, "n_blocks": len(cids), "car_bytes": len(car), "runs": args.runs, "parsed_on_device": sorted(paths), "routes": {}}
    for r, v in times.items():
        res["routes"][r] = dict(median_ms=round(statistics.median(v), 2), min_ms=round(min(v), 2), max_ms=round(max(v), 2))
        if kern[r]:
            res["routes"][r]["kernels_median_ms"] = round(statistics.median(kern[r]), 3)
            res["routes"][r]["ms_parse_median"] = round(statistics.median(parse[r]), 2)
    pinned.free()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
