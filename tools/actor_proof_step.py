"""ipcfp_generate_actor_proofs_resident on a state tree whose actors HAMT holds --entries actors and whose Init actor's address map holds
--entries addresses of every protocol (f1, f2, f3, f410, other f4), each mapped to one of those actors (built with tests/actor_trees.py
and tests/address_trees.py, the test builders), at 1, 1 000 and 65 536 requests per call: half ID addresses, half addresses in the map.
Every 16th actor is an EVM actor with its bytecode; the call runs without and with IPCFP_ACTOR_WITH_CODE. Per batch size and mode, after
--warmup calls, --runs calls with
  device_ms  the call's own CUDA events on the store's stream (ms_total: upload, Init walk, proof walks, code gather, witness, copies)
  walk_ms    the same for the proof walks alone (ms_walk)
  wall_ms    host clock around the call (it ends in a device synchronise)
as median / min / max. Parity: every timed call's proofs, per-proof lists and witness CIDs equal the C++ oracle's (tests/oracle_actors.cpp,
computed once per batch size and mode outside the timed calls); for the 1- and 1 000-request batches the oracle also equals the Python
restatement of tests/actor_trees.py. Prints one JSON line with the card's name and power limit read in the same run."""
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
    from ipc_filecoin_proofs_b200 import api
    from tests import actor_trees as AT
    from tests import address_trees as R
    from tests import oracle_actors as O
    from tests import storage_trees as S
    import synth
    name = card()
    t0 = time.perf_counter()
    blocks = S.Blocks()
    rng = random.Random(1)
    ids = set()
    while len(ids) < args.entries:
        ids.add(rng.randrange(1000, 2 ** rng.choice((20, 32, 64))))
    ids = sorted(ids)
    actors = {}
    for k, aid in enumerate(ids):
        actors[aid] = (AT.evm_actor(blocks, AT.EVM_A, k % 1000) if k % 16 == 0 else
                       AT.actor_state(AT.ACCOUNT, S.cid_of(b"filler-%d" % k), k % 7, AT.bigint(k)))
    amap = {}
    while len(amap) < args.entries:
        amap[R.random_address(rng, R.KINDS[len(amap) % len(R.KINDS)])] = ids[len(amap)]
    root = AT.state_tree(blocks, actors, amap)
    ts = synth.Tipset(synth.config_params(3, hamt_entries=20000))
    hdr, child = S.child_header(ts, root)
    blocks[child] = hdr
    f = S.Flat(blocks)
    tip_ts = S.tipset(ts, f.arrays(), child, root)
    build_s = time.perf_counter() - t0
    store = api.BlockStore(f.cids, f.offsets, f.lengths, f.blob, verify_cids=True)
    tip = store.upload_tipset(tip_ts)
    oracle = O.Oracle(blocks)
    out = dict(card=name, entries=args.entries, blocks=int(f.n_blocks), build_s=round(build_s, 1), runs=args.runs, sizes={})
    stat = lambda xs: dict(median=round(statistics.median(xs), 4), min=round(min(xs), 4), max=round(max(xs), 4))   # noqa: E731
    parity = True
    keys = list(amap)
    for n in (int(x) for x in args.sizes.split(",")):
        r2 = random.Random(n)
        addrs = [R.id_addr(a) for a in r2.sample(ids, n - n // 2)] + r2.sample(keys, n // 2)
        for with_code in (False, True):
            want = oracle.prove(child, root, addrs, [AT.EVM_A], with_code)
            if n <= 1000:
                parity &= AT.prove(blocks, child, root, addrs, [AT.EVM_A], with_code) == want
            dev, walk, wall = [], [], []
            for k in range(args.warmup + args.runs):
                t1 = time.perf_counter()
                r = store.generate_actor_proofs_resident(tip, addrs, [AT.EVM_A], with_code)
                w = (time.perf_counter() - t1) * 1e3
                if k == 0 or k == args.warmup + args.runs - 1:
                    cids = [bytes(c) for c in r.witness.cids]
                    parity &= [vars(p) for p in r.proofs] == want[0] and cids == want[2]
                    parity &= [[cids[j] for j in lst] for lst in r.proof_witness] == want[1]
                if k >= args.warmup:
                    dev.append(r.timings["total"])
                    walk.append(r.timings["walk"])
                    wall.append(w)
            out["sizes"][f"{n}{'+code' if with_code else ''}"] = dict(device_ms=stat(dev), walk_ms=stat(walk), wall_ms=stat(wall),
                                                                     witness_blocks=int(r.witness.n_blocks))
    out["parity"] = bool(parity)
    print(json.dumps(out))
    if not parity:
        sys.exit(1)


if __name__ == "__main__":
    main()
