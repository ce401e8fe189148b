"""The tipset from its Lotus JSON-RPC texts to a device-resident tipset, three routes alternated in one process on the same texts (the
1 M-receipt tipset by default):
  (a) device: BlockStore.upload_tipset_json on the canonical receipt list (parsed on the device);
  (b) host:   the same texts with one trailing space after the receipt list (ipcfp_tipset_desc_from_json, then the upload);
  (c) python: json.loads of the three texts, the descriptor arrays built in Python (base32 decode of every events root), then
              ipcfp_tipset_upload.
Each route ends with a device synchronisation. For every route: median / min / max wall time after warm-up and the text's GB/s; for (a) the
device parse kernels' time (CUDA events inside the call) and the whole parse's wall time. Also the card's name and power limit read in the
same run. All routes must give the same tipset."""
import argparse
import base64
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.json_step import card  # noqa: E402


def python_route(api, store, p, c, r):
    """What a caller does today without the new calls: serde-like deserialisation in Python, base32 per events root, the arrays, the upload."""
    import numpy as np
    parent, child, receipts = json.loads(p), json.loads(c), json.loads(r)

    def cid(s):
        s = s[1:].upper()
        return base64.b32decode(s + "=" * (-len(s) % 8))

    n = len(receipts)
    roots = np.zeros((n, 38), np.uint8)
    has = np.zeros(n, np.uint8)
    for i, rc in enumerate(receipts):
        er = rc.get("EventsRoot")
        if er is not None:
            roots[i] = np.frombuffer(cid(er["/"]), np.uint8)
            has[i] = 1

    class T:
        pass
    t = T()
    t.parent_epoch, t.child_epoch = parent["Height"], child["Height"]
    t.n_parents = len(parent["Cids"])
    t.parent_cids = np.frombuffer(b"".join(cid(x["/"]) for x in parent["Cids"]), np.uint8)
    t.parent_txmeta_cids = np.frombuffer(b"".join(cid(b["Messages"]["/"]) for b in parent["Blocks"]), np.uint8)
    t.child_cid = np.frombuffer(cid(child["Cids"][0]["/"]), np.uint8)
    t.receipts_root = np.frombuffer(cid(child["Blocks"][0]["ParentMessageReceipts"]["/"]), np.uint8)
    t.parent_state_root = np.frombuffer(cid(child["Blocks"][0]["ParentStateRoot"]["/"]), np.uint8)
    t.n_receipts, t.events_roots, t.has_events_root = n, roots, has
    return store.upload_tipset(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--receipts", type=int, default=1_000_000)
    args = ap.parse_args()
    import torch

    import synth
    from ipc_filecoin_proofs_b200 import api
    from tests import rpc_json as R
    print(f"card: {card()}")
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts))
    p, c, r = (x.encode() for x in R.texts(ts))   # the bytes an HTTP client hands over
    r_space = r + b" "
    store = api.BlockStore.from_tipset(ts)
    ref = store.upload_tipset(ts).describe()
    routes = {
        "a": lambda: store.upload_tipset_json(p, c, r),
        "b": lambda: store.upload_tipset_json(p, c, r_space),
        "c": lambda: python_route(api, store, p, c, r),
    }
    wall = {k: [] for k in routes}
    dev = []
    for k in range(args.warmup + args.runs):
        for name, fn in routes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tip = fn()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            info = tip.describe(with_events_roots=(k == 0))
            if k == 0:
                R.assert_desc_equal(info, ref)
            assert info.parsed_on_device == (name == "a")
            if k >= args.warmup:
                wall[name].append(dt * 1e3)
                if name == "a":
                    dev.append((info.ms_kernels, info.ms_parse))
            tip.close()
    total = len(p) + len(c) + len(r)
    print(f"\n{ts.n_receipts} receipts: receipt list {len(r) / 1e6:.1f} MB, tipset texts {(len(p) + len(c)) / 1e3:.1f} KB")
    for name, label in (("a", "(a) upload_tipset_json, device parse"), ("b", "(b) upload_tipset_json, host parse"),
                        ("c", "(c) json.loads + arrays + upload")):
        w = wall[name]
        med = statistics.median(w)
        print(f"  {label:40s} median {med:9.2f} ms [{min(w):9.2f}, {max(w):9.2f}] over {len(w)}   {total / med / 1e6:7.2f} GB/s")
    print(f"  (a) parse kernels (CUDA events) median {statistics.median(d[0] for d in dev):.3f} ms, "
          f"its whole parse incl. H2D median {statistics.median(d[1] for d in dev):.3f} ms")


if __name__ == "__main__":
    main()
