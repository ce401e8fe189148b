#!/usr/bin/env python
"""What the EventProofBundle JSON costs on the 1 M-receipt tipset (BASELINE.json configs[3]), store and tipset resident.
Usage: python tools/json_step.py [--receipts N] [--steps K] [--warmup W]

Five arms, alternated step by step in one process after W warm-up rounds of each:
  1 flags 0                       2 WITNESS_BY_REFERENCE
  3 RESULT_JSON                   4 RESULT_JSON | WITNESS_BY_REFERENCE
  5 flags 0, then ipcfp_event_result_to_json on the host
For every arm: median / min / max wall time per step until the results (and, for 3-5, the text) are on the host, ms_total and ms_json
(device time, CUDA events). Arms 3, 4 and 5 must give equal bytes. Prints the card's name and power limit."""
import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receipts", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts))
    L = api.lib()
    store = api.BlockStore.from_tipset(ts)
    d, keep = A.make_tipset_desc(ts)
    th = C.c_void_p()
    api._check(L.ipcfp_tipset_upload(store._h, C.byref(d), C.byref(th)))
    spec = A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter)
    arms = [("flags 0", 0, False), ("WITNESS_BY_REFERENCE", A.WITNESS_BY_REFERENCE, False), ("RESULT_JSON", A.RESULT_JSON, False),
            ("RESULT_JSON|WITNESS_BY_REFERENCE", A.RESULT_JSON | A.WITNESS_BY_REFERENCE, False), ("flags 0 + host to_json", 0, True)]
    wall = {a[0]: [] for a in arms}
    dev = {a[0]: [] for a in arms}
    djs = {a[0]: [] for a in arms}
    texts = {}

    def step(name, flags, host_json, keep_text):
        out = C.POINTER(A.EventResultC)()
        t0 = time.perf_counter()
        api._check(L.ipcfp_generate_event_proof_resident(store._h, th, C.byref(spec), flags, C.byref(out)))
        text_p, n = C.c_void_p(), C.c_uint64()
        if host_json:
            api._check(L.ipcfp_event_result_to_json(out, C.byref(d), C.byref(text_p), C.byref(n)))
        t1 = time.perf_counter()
        r = out.contents
        if keep_text:
            texts[name] = C.string_at(text_p.value, n.value) if host_json else (C.string_at(r.json, r.json_len) if r.json else None)
        if host_json:
            L.ipcfp_json_free(text_p)
        res = (1e3 * (t1 - t0), float(r.ms_total), float(r.ms_json))
        L.ipcfp_event_result_free(out)
        return res

    for _ in range(args.warmup):
        for name, flags, hj in arms:
            step(name, flags, hj, False)
    for k in range(args.steps):
        for name, flags, hj in arms:
            w, t, j = step(name, flags, hj, k == 0)
            wall[name].append(w); dev[name].append(t); djs[name].append(j)
    L.ipcfp_tipset_free(th)
    same = texts["RESULT_JSON"] == texts["RESULT_JSON|WITNESS_BY_REFERENCE"] == texts["flags 0 + host to_json"]
    print(f"card: {card()}")
    print(f"receipts {args.receipts}, witness blocks {ts.n_blocks} in the store, JSON {len(texts['flags 0 + host to_json'])} bytes, "
          f"arms 3/4/5 byte-equal: {same}; {args.steps} steps per arm after {args.warmup} warm-up rounds, alternated")
    print(f"{'arm':36s} {'wall ms median [min, max]':>30s} {'ms_total median':>16s} {'ms_json median':>15s}")
    for name, _, _ in arms:
        w = wall[name]
        print(f"{name:36s} {statistics.median(w):12.3f} [{min(w):7.3f}, {max(w):7.3f}] {statistics.median(dev[name]):16.3f} "
              f"{statistics.median(djs[name]):15.3f}")
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
