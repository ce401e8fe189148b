"""Fetch planning on the 1 M-receipt tipset (synthetic config 4):
  full     ipcfp_plan_fetch_resident against the complete store, i.e. the whole traversal with nothing missing: device ms (CUDA events on
           the store's stream) and wall ms, median / min / max over --runs after --warmup;
  loop     api.fetch_until_complete from an empty store, the fetcher answering from the block map with canonical ChainReadObj responses:
           rounds, CIDs per round, plan device ms against store-rebuild wall ms (BlockStore.from_rpc_json over every response so far, then
           the tipset upload) per round. The bundle (IPCFP_RESULT_JSON) of the planned store must equal the full store's.
Prints one JSON line with the card's name and power limit read in the same run."""
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
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--receipts", type=int, default=1_000_000)
    args = ap.parse_args()
    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    from tests import rpc_blocks as B
    from tests.util import spec_of
    name = card()
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts))
    spec = [spec_of(ts)]
    full = api.BlockStore.from_tipset(ts)
    tip = full.upload_tipset(ts)
    dev, wall = [], []
    for k in range(args.warmup + args.runs):
        t0 = time.perf_counter()
        p = full.plan_fetch(tip, [], spec)
        w = (time.perf_counter() - t0) * 1e3
        assert len(p.cids) == 0
        if k >= args.warmup:
            dev.append(p.ms_total)
            wall.append(w)
    stat = lambda xs: dict(median=statistics.median(xs), min=min(xs), max=max(xs))   # noqa: E731
    out = dict(card=name, receipts=args.receipts, blocks=int(full.n_blocks), full=dict(device_ms=stat(dev), wall_ms=stat(wall),
                                                                                        n_needed=p.n_needed, n_levels=p.n_levels))
    cids, blocks = B.blocks_of(ts)
    blk = {bytes(c): b for c, b in zip(cids, blocks)}
    del cids, blocks

    def fetch(cs, first_id):
        return B.render([], elements=[B.element(first_id + k, blk[bytes(c)]) for k, c in enumerate(cs)])

    t0 = time.perf_counter()
    store, stip, rounds, _, _ = api.fetch_until_complete(fetch, lambda s: s.upload_tipset(ts), [], spec, verify_cids=False)
    loop_s = time.perf_counter() - t0
    a = store.generate_proof_bundle_resident(stip, [], spec, A.RESULT_JSON)
    b = full.generate_proof_bundle_resident(tip, [], spec, A.RESULT_JSON)
    assert a.json == b.json
    out["loop"] = dict(rounds=len(rounds), cids=[len(r.cids) for r in rounds], plan_ms=[round(r.ms_plan, 3) for r in rounds],
                       rebuild_ms=[round(r.ms_rebuild, 1) for r in rounds], wall_s=round(loop_s, 2), same_bundle=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
