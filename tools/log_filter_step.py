"""Log filters on the 1 M-receipt tipset of bench.py (synthetic config 4), resident store and tipset, one call per step:
  spec          ipcfp_generate_event_proof_resident with the tipset's spec (bench.py's step)
  filter=spec   ipcfp_generate_log_proof_resident with LogFilter.from_spec(spec)
  topic2        {t0} at topic 0 and 64 values at topic 2 (a constraint past topic 1; three topics needed)
  t1x64, t1x4096  the spec's t1 among 64 / 4 096 values at topic 1 (the large-set path: bitmap + binary search)
  emit1024      topic 0 = {t0}, the spec's actor among 1 024 emitters
  wildcard      no constraint at all (every candidate event of every receipt matches)
For each: pass 1 (ms_pass1) and the whole step (ms_total), device time from CUDA events on the store's stream, median / min / max over
--runs after --warmup, and the matching receipts and proofs. The spec's result and its filter's are compared by SHA-256 over the
proof records, the data blob and the witness CIDs. Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import hashlib
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
    spec = api.EventProofSpec(ts.event_signature, ts.topic1, None if ts.actor_filter is None else int(ts.actor_filter))
    eq = api.LogFilter.from_spec(spec)
    t0, t1 = eq.topics[0][0], eq.topics[1][0]
    rng = np.random.default_rng(1)
    rnd = lambda n: [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(n)]   # noqa: E731
    actor = [int(ts.actor_filter)] if ts.actor_filter is not None else []
    cases = {
        "spec": None,
        "filter=spec": eq,
        "topic2": api.LogFilter(topics=[t0, None, rnd(64)]),
        "t1x64": api.LogFilter(emitters=actor, topics=[t0, [t1] + rnd(63)]),
        "t1x4096": api.LogFilter(emitters=actor, topics=[t0, [t1] + rnd(4095)]),
        "emit1024": api.LogFilter(emitters=actor + [int(x) for x in rng.integers(2**40, 2**62, 1024 - len(actor), dtype=np.uint64)], topics=[t0]),
        "wildcard": api.LogFilter(),
    }
    cspec = spec.as_c()

    def call(flt):
        out = C.POINTER(A.EventResultC)()
        if flt is None:
            st = L.ipcfp_generate_event_proof_resident(store._h, tip._h, C.byref(cspec), 0, C.byref(out))
        else:
            f, keep = flt.as_c()
            st = L.ipcfp_generate_log_proof_resident(store._h, tip._h, C.byref(f), 0, C.byref(out))
        assert st == 0, L.ipcfp_last_error()
        return out

    def digest(r):
        h = hashlib.sha256()
        h.update(A._arr(r.matching_indices, int(r.n_matching), np.uint64).tobytes())
        h.update(A._arr(C.cast(r.proofs, C.c_void_p).value, int(r.n_proofs) * C.sizeof(A.EventProofC), np.uint8).tobytes())
        h.update(A._arr(r.data_blob, int(r.data_blob_size), np.uint8).tobytes())
        h.update(A._arr(r.witness.cids, int(r.witness.n_blocks) * 38, np.uint8).tobytes())
        return h.hexdigest()

    stat = lambda xs: dict(median=round(statistics.median(xs), 4), min=round(min(xs), 4), max=round(max(xs), 4))   # noqa: E731
    out = dict(card=name, receipts=args.receipts, cases={})
    digests = {}
    for label, flt in cases.items():
        p1, tot = [], []
        for k in range(args.warmup + args.runs):
            o = call(flt)
            r = o.contents
            if k >= args.warmup:
                p1.append(r.ms_pass1)
                tot.append(r.ms_total)
            if k == 0:
                digests[label] = digest(r)
                out["cases"][label] = dict(matching=int(r.n_matching), proofs=int(r.n_proofs), witness_blocks=int(r.witness.n_blocks))
            L.ipcfp_event_result_free(o)
        out["cases"][label].update(pass1_ms=stat(p1), total_ms=stat(tot))
    out["filter_equals_spec"] = digests["spec"] == digests["filter=spec"]
    out["wildcard_sha256"] = digests["wildcard"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
