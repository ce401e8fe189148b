#!/usr/bin/env python
"""Minimal driver for ncu: build the configs[3] tipset, ingest, run W warm-up + K resident steps.
Usage: python tools/profile_step.py [--receipts N] [--steps K] [--warmup W] [--verify] [--timeline]

--timeline: the K steps run under torch.profiler (CUDA activities); for every step it prints when, relative to the step's first
GPU activity, the message-AMT walk kernels, pass 1, pass 2 and every device-to-host copy start and end, and the achieved rate of
the witness copy. Run it on its own: tracing slows the host, so its step times are not the benchmark's."""
import argparse
import ctypes as C
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
T0 = time.time()


def log(*a):
    print(f"[{time.time() - T0:7.2f}s]", *a, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receipts", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--verify", action="store_true")
    ap.add_argument("--timeline", action="store_true", help="per-step kernel / copy timeline under torch.profiler (see above)")
    ap.add_argument("--storage", type=int, default=0, help="also run N storage-slot lookups on a 1M-entry HAMT")
    args = ap.parse_args()
    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    log("imports done")
    ts = synth.Tipset(synth.config_params(4, n_receipts=args.receipts))
    log(f"tipset built: {ts.n_blocks} blocks {len(ts.blob) / 1e9:.3f} GB")
    L = api.lib()
    st = api.BlockStore.from_tipset(ts, verify_cids=args.verify)
    log("store created")
    spec = A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter)
    d, keep = A.make_tipset_desc(ts)
    L.ipcfp_tipset_upload.restype = C.c_int32
    L.ipcfp_tipset_upload.argtypes = [C.c_void_p, C.POINTER(A.TipsetDesc), C.POINTER(C.c_void_p)]
    L.ipcfp_generate_event_proof_resident.restype = C.c_int32
    L.ipcfp_generate_event_proof_resident.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(A.EventSpec), C.c_uint32, C.POINTER(C.POINTER(A.EventResultC))]
    tip = C.c_void_p()
    assert L.ipcfp_tipset_upload(st._h, C.byref(d), C.byref(tip)) == 0
    log("tipset uploaded")
    if args.timeline:
        timeline(L, A, st, tip, spec, args.warmup, args.steps)
        return
    for k in range(args.warmup + args.steps):
        out = C.POINTER(A.EventResultC)()
        t = time.time()
        assert L.ipcfp_generate_event_proof_resident(st._h, tip, C.byref(spec), 0, C.byref(out)) == 0, L.ipcfp_last_error()
        r = out.contents
        log(f"step {k}: wall {1e3 * (time.time() - t):.2f} ms; device total {r.ms_total:.3f} txamt {r.ms_txamt:.3f} pass1 {r.ms_pass1:.3f} "
            f"pass2 {r.ms_pass2:.3f} witness {r.ms_witness:.3f}; matching {r.n_matching} witness {r.witness.n_blocks} blocks")
        L.ipcfp_event_result_free(out)
    if args.storage:
        import numpy as np
        ts3 = synth.Tipset(synth.config_params(3))
        st3 = api.BlockStore.from_tipset(ts3, verify_cids=args.verify)
        keys = [ts3.storage_entry(k)[0] for k in range(args.storage)]
        slots = np.frombuffer(b"".join(api.compute_mapping_slots(keys, [0] * len(keys))), dtype=np.uint8)
        for mode in ("fast", "strict", "fast"):
            os.environ.pop("IPCFP_HAMT_STRICT", None)
            if mode == "strict":
                os.environ["IPCFP_HAMT_STRICT"] = "1"
            for k in range(4):
                t = time.time()
                r = st3.read_storage_slots(ts3.storage_root, slots)
                print(f"STORAGE {mode} x{args.storage}: wall {1e3 * (time.time() - t):.2f} ms device {r.ms_total:.3f} ms lookup kernel {r.ms_lookup:.4f} ms nodes {r.lookup_nodes} found {int(r.found.sum())}", flush=True)
    log("done")


def card():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable ({e})"
    return out


def timeline(L, A, st, tip, spec, warmup, steps):
    import json
    import tempfile

    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    torch.zeros(1, device="cuda")
    n_blocks = []

    def step():
        out = C.POINTER(A.EventResultC)()
        assert L.ipcfp_generate_event_proof_resident(st._h, tip, C.byref(spec), 0, C.byref(out)) == 0, L.ipcfp_last_error()
        n_blocks.append(int(out.contents.witness.n_blocks))
        L.ipcfp_event_result_free(out)

    for _ in range(warmup):
        step()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for k in range(steps):
            with record_function(f"ipcfp_step_{k}"):
                step()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    print(f"card: {card()}", flush=True)
    wins = sorted((e["ts"], e["ts"] + e["dur"], e["name"]) for e in events
                  if e.get("cat") == "user_annotation" and e.get("name", "").startswith("ipcfp_step_"))
    gpu = [e for e in events if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    for k, (w0, w1, name) in enumerate(wins):
        m = n_blocks[warmup + k]
        sel = sorted((e for e in gpu if w0 <= e["ts"] < w1), key=lambda e: e["ts"])
        if not sel:
            print(f"{name}: no GPU activity in the step's window")
            continue
        t0 = sel[0]["ts"]
        rel = lambda e: (e["ts"] - t0, e["ts"] + e["dur"] - t0)   # noqa: E731

        def span(label, pred):
            hit = [e for e in sel if e.get("cat") == "kernel" and pred(e["name"])]
            if hit:
                print(f"  {label:34s} {min(rel(e)[0] for e in hit) / 1e3:8.3f} .. {max(rel(e)[1] for e in hit) / 1e3:8.3f} ms  ({len(hit)} launches)")
            else:
                print(f"  {label:34s} none")
        print(f"{name}: first GPU activity = 0, {m} witness blocks")
        span("message-AMT walk (k_amt_*)", lambda n: "k_amt_" in n)
        span("pass 1 (k_pass1*)", lambda n: "k_pass1" in n)
        span("witness gather (k_witness_copy)", lambda n: "k_witness_copy" in n)
        span("execution-order dedup (k_dedup_*)", lambda n: "k_dedup_" in n)
        span("k_pass2", lambda n: "k_pass2" in n)
        span("k_witness_emit", lambda n: "k_witness_emit" in n)
        d2h = [e for e in sel if e.get("cat") == "gpu_memcpy" and "DtoH" in e["name"] and e.get("args", {}).get("bytes", 0) >= 4096]
        # the witness blocks gathered at the snapshot go down in two parts on their own stream, which carries the step's largest copy
        big = max(d2h, key=lambda e: e["args"]["bytes"], default=None)
        side = [e for e in d2h if big is not None and e["args"].get("stream") == big["args"].get("stream")]
        for e in d2h:
            b = e["args"]["bytes"]
            if e in side:
                label = f"witness D2H part {side.index(e) + 1}"
            else:
                label = {38 * m: "witness cids D2H", 8 * m: "witness offsets D2H", 4 * m: "witness lengths D2H"}.get(b, "D2H (late blocks B / results)")
            s0, s1 = rel(e)
            print(f"  {label:34s} {s0 / 1e3:8.3f} .. {s1 / 1e3:8.3f} ms  {b / 1e6:9.3f} MB  {b / max(e['dur'], 1e-3) / 1e3:6.1f} GB/s  stream {e['args'].get('stream')}")
        if side:
            a0, a1 = rel(side[0])[0], rel(side[-1])[1]
            nb = sum(e["args"]["bytes"] for e in side)
            print(f"  witness copy: {nb / 1e6:.1f} MB in {(a1 - a0) / 1e3:.3f} ms from its first byte = {nb / max(a1 - a0, 1e-3) / 1e3:.1f} GB/s")
        print(f"  {'last activity of the step':34s} {max(rel(e)[1] for e in sel) / 1e3:8.3f} ms", flush=True)


if __name__ == "__main__":
    main()
