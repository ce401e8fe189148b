"""ipcfp_resolve_addresses on a state tree whose Init actor's address map holds --entries addresses (built with tests/address_trees.py,
the test builders), at 1, 1 000 and 65 536 addresses per call: every address is in the map and every protocol is mixed in (f1, f2, f3,
f410, other f4). Per batch size, after --warmup calls, --runs calls with
  device_ms  the call's own CUDA events on the store's stream (ms_total: upload, Init path, walks, witness, missing list, copies back)
  lookup_ms  the same for the address_map walks alone (ms_lookup)
  wall_ms    host clock around the call (it ends in a device synchronise)
as median / min / max. Parity: every timed call's whole result (IDs, statuses, Init status, missing CIDs, witness CIDs) equals the C++
oracle's (tests/oracle_resolve.cpp, computed once per batch size outside the timed calls), whose IDs and statuses equal the builder's
ground truth; for the 1- and 1 000-address batches the oracle also equals the Python restatement of tests/address_trees.py. Prints one
JSON line with the card's name and power limit read in the same run."""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.json_step import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, default=1_000_000)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="1,1000,65536")
    args = ap.parse_args()
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    from tests import address_trees as T
    from tests import oracle_resolve as O
    from tests import storage_trees as S
    name = card()
    t0 = time.perf_counter()
    blocks = S.Blocks()
    ent = T._entries(random.Random(1), args.entries)
    root = T.state_tree(blocks, ent)
    f = S.Flat(blocks)
    build_s = time.perf_counter() - t0
    store = api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True)
    keys = list(ent)
    out = dict(card=name, entries=args.entries, blocks=int(f.n_blocks), build_s=round(build_s, 1), runs=args.runs, sizes={})
    stat = lambda xs: dict(median=round(statistics.median(xs), 4), min=round(min(xs), 4), max=round(max(xs), 4))   # noqa: E731
    parity = True
    oracle = O.Oracle(blocks)
    for n in (int(x) for x in args.sizes.split(",")):
        addrs = random.Random(n).sample(keys, n)
        want = oracle.resolve(root, addrs)
        parity &= want[0] == [ent[a] for a in addrs] and want[1] == [A.OK] * n and want[2] == A.OK and want[3] == []
        if n <= 1000:
            parity &= T.resolve(blocks, root, addrs) == want
        dev, look, wall = [], [], []
        for k in range(args.warmup + args.runs):
            t1 = time.perf_counter()
            r = store.resolve_addresses(root, addrs)
            w = (time.perf_counter() - t1) * 1e3
            parity &= (r.actor_ids.tolist(), r.status.tolist(), r.init_status) == want[:3]
            parity &= [bytes(c) for c in r.missing] == want[3] and [bytes(c) for c in r.witness.cids] == want[4]
            if k >= args.warmup:
                dev.append(r.ms_total)
                look.append(r.ms_lookup)
                wall.append(w)
        out["sizes"][n] = dict(device_ms=stat(dev), lookup_ms=stat(look), wall_ms=stat(wall), witness_blocks=int(r.witness.n_blocks))
    out["parity"] = bool(parity)
    print(json.dumps(out))
    if not parity:
        sys.exit(1)


if __name__ == "__main__":
    main()
