#!/usr/bin/env python
"""bench.py — receipts/sec scanned (+ witness bytes/sec) of the event-proof hot path on H100.

  python bench.py --gpus N --steps K --warmup W            # this engine (CUDA, through the C ABI)
  python bench.py --impl reference --gpus N --steps K ...   # the reference's CPU algorithm (oracle), host cores
  python bench.py ... --dump-outputs DIR                    # also write the last timed step's results as DIR/<name>.npy

One "step" = one generate_event_proof over the synthetic tipset of BASELINE.json configs[3]
(1 M receipts x 8 events, 0.1 % match rate, events-AMT bit widths 3/5): message-AMT walk + execution
order, pass 1 over every receipt, pass 2 over the matches, witness sort + gather, results to the host.
N > 1 (torchrun): weak scaling — every rank holds a 1 M-receipt shard of an N x 1 M tipset
(configs[4] at N = 8), scans it, and the per-shard witness CID sets are all-gathered (NCCL) and merged.

`value`  : receipts/s with the block store and the tipset descriptor resident in HBM.
`e2e`    : the same metric through the plain C-ABI call sequence a reference-side binding makes with HOST
           buffers: ipcfp_store_create (H2D of every block, index build, Blake2b CID check) +
           ipcfp_generate_event_proof (H2D of the events roots, scan, D2H of the results).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RECEIPTS_PER_GPU = int(os.environ.get("IPCFP_BENCH_RECEIPTS", 1_000_000))


_T0 = time.time()


def log(*a):
    print(f"[{time.time() - _T0:8.2f}s]", *a, file=sys.stderr, flush=True)


def build_tipset(world, rank):
    import synth
    n_total = RECEIPTS_PER_GPU * world
    lo, hi = RECEIPTS_PER_GPU * rank, RECEIPTS_PER_GPU * (rank + 1)
    kw = {}
    if world > 1:
        kw.update(shard_lo=lo, shard_hi=hi)
    p = synth.config_params(4, n_receipts=n_total, **kw)
    t0 = time.time()
    ts = synth.Tipset(p)
    log(f"[rank {rank}] synthetic tipset: {ts.n_blocks} blocks, {len(ts.blob) / 1e9:.3f} GB, built in {time.time() - t0:.1f}s")
    return ts, lo, hi


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx = gpu_index
        self.rows = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "20", "-i", str(self.idx)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._read, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), line.strip()))

    def stop(self, t0, t1):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        for t, line in self.rows:
            f = [x.strip() for x in line.split(",")]
            if len(f) < 8:
                continue
            try:
                mx = float(f[2])
                if t0 - 0.05 <= t <= t1 + 0.05:
                    sm.append(float(f[1]))
                    for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[4:8]):
                        if v.lower().startswith("active"):
                            reasons.add(name)
            except ValueError:
                pass
        if not sm:  # timed region shorter than the sampling period: fall back to all samples
            for t, line in self.rows:
                f = [x.strip() for x in line.split(",")]
                try:
                    sm.append(float(f[1]))
                except (ValueError, IndexError):
                    pass
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


def dist_env():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    return world, rank, local


def peaks():
    return 3350.0, "H100 SXM data sheet: 3.35 TB/s HBM3 (700 W card; not a measured figure)"


def gpu_info(gpu_index):
    """Name and power limit of the card the numbers were measured on."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", str(gpu_index)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(clk)}
    except Exception:
        return None


def dump_outputs(dirpath, res):
    """Writes what generate_event_proof returned (an EventResultPy) as DIR/<name>.npy, float64 for indices and counts, float32 for bytes.
    The witness is large (≈ 147 k blocks, 51 MB at 1 M receipts): a fixed, seeded sample of its rows is written, the same rows for CIDs,
    lengths and block bytes, so that two builds given the same arguments can be compared array for array (≈ 30 MB in all)."""
    from ipc_filecoin_proofs_b200 import _abi as A
    os.makedirs(dirpath, exist_ok=True)
    w = res.witness
    m = w.n_blocks
    rows = np.arange(m) if m <= 16384 else np.sort(np.random.default_rng(0).choice(m, 16384, replace=False))
    blocks = np.frombuffer(b"".join(w.block(int(i)) for i in rows), dtype=np.uint8)[: 8 << 20]
    raw = np.frombuffer(res.raw_proofs.tobytes(), dtype=A.EventProofC).reshape(-1) if len(res.proofs) else None
    fields = ("exec_index", "event_index", "emitter", "n_topics", "data_len", "data_off", "topics_off")
    out = {
        "counts": np.array([len(res.matching), len(res.proofs), m, w.total_bytes, res.n_exec], dtype=np.float64),
        "matching": res.matching.astype(np.float64),
        "proof_fields": np.stack([raw[f].astype(np.float64) for f in fields], axis=1) if raw is not None else np.zeros((0, len(fields))),
        "proof_message_cids": np.array([list(p.message_cid) for p in res.proofs], dtype=np.float32).reshape(-1, A.CID_LEN),
        "proof_data_blob": res.data_blob.astype(np.float32),
        "witness_sample_rows": rows.astype(np.float64),
        "witness_cids": w.cids[rows].astype(np.float32),
        "witness_lengths": w.lengths[rows].astype(np.float64),
        "witness_block_bytes": blocks.astype(np.float32),
    }
    for k, v in out.items():
        np.save(os.path.join(dirpath, k + ".npy"), v)
    return sorted(out)


WORKLOAD = ("BASELINE.json configs[3] per GPU: 1M receipts x 8 events, 0.1% match, events-AMT bit-widths 3/5; generate_event_proof "
            "(message-AMT walk + exec order, pass 1, pass 2, witness sort+gather, results to host)")


def config_dict(world, n_local, **extra):
    """Same keys in both arms (the driver compares them)."""
    d = {k: None for k in ("store_blocks_per_gpu", "store_bytes_per_gpu", "matching_rank0", "proofs_rank0", "matching_total", "proofs_total",
                           "witness_blocks_rank0", "merged_witness_cids", "n_exec", "note")}
    d.update({"workload": WORKLOAD + ("" if world == 1 else f"; N={world}: ONE {world}M-receipt tipset sharded by receipt index range (configs[4] shape at N=8), "
                                 "in-library NCCL protocol: all-to-all + all-reduce for the first-seen dedup of the execution order, all-gather of the witness CID sets"),
         "receipts_per_gpu": int(n_local), "receipts_total": int(n_local) * world,
         "l2": "inputs (1.15 GB/GPU) exceed the 50 MB L2; no flush needed"})
    d.update(extra)
    return d


def digest_proofs(res):
    """sha256 over every EventProof field of a result (EventResultPy), in order."""
    import hashlib
    h = hashlib.sha256()
    for p in res.proofs:
        h.update(repr(p.key()).encode())
    return h.hexdigest()


# ------------------------------------------------------------------------------------------ reference arm
def run_reference(args, world, rank):
    if rank != 0:
        return
    import oracle
    from ipc_filecoin_proofs_b200 import _abi as A
    ts, lo, hi = build_tipset(1, 0)
    spec = A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter)
    cores = os.cpu_count() or 1
    st = oracle.Store.from_tipset(ts)
    d, keep = A.make_tipset_desc(ts)
    L = oracle.lib()

    def step():
        out = C.POINTER(A.EventResultC)()
        rc = L.oracle_generate_event_proof(st._h, C.byref(d), C.byref(spec), 0, cores, C.byref(out))
        assert rc == 0, L.oracle_last_error()
        r = out.contents
        res = (int(r.n_matching), int(r.witness.n_blocks), int(r.witness.blob_size), int(r.n_proofs), int(r.n_exec))
        L.oracle_event_result_free(out)
        return res

    for _ in range(max(args.warmup, 1)):
        step()
    t0 = time.time()
    for _ in range(args.steps):
        nm, wb, wbytes, npf, nex = step()
    dt = time.time() - t0
    val = ts.n_receipts * args.steps / dt
    line = {
        "impl": "reference", "metric": "receipts/sec scanned", "value": val, "unit": "receipts/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "u8", "data": "synthetic",
        "config": config_dict(1, int(ts.n_receipts), store_blocks_per_gpu=int(ts.n_blocks), store_bytes_per_gpu=int(len(ts.blob)), matching_rank0=nm,
                              proofs_rank0=npf, matching_total=nm, proofs_total=npf, witness_blocks_rank0=wb, merged_witness_cids=wb, n_exec=nex,
                              note="the reference arm always scans ONE 1M-receipt tipset on the host (rank 0); at --gpus N > 1 the engine arm scans "
                                   "an N x 1M-receipt tipset (weak scaling): compare receipts/s, not same-input wall time"),
        "witness_bytes_per_s": wbytes * args.steps / dt,
        "cpu_baseline": {"value": val, "unit": "receipts/s", "cores": cores, "kind": "port",
                         "sample": "full workload per step; C++ restatement of the reference (the Rust crate cannot be built here), "
                                   "pass 1 parallelised over receipts on all host threads, the rest single-threaded like the reference"},
        "e2e": {"value": val, "unit": "receipts/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------ engine arm
def storage_section(api, A, L, local, args):
    """configs[2]: 1M-slot EVM storage HAMT, keccak-keyed slot lookups through ipcfp_read_storage_slots (host keys in, values +
    witness out). Kernel time = CUDA events around the lookup kernel; algorithmic bytes = 32 per key + every node on its path."""
    import synth
    import oracle
    t0 = time.time()
    ts3 = synth.Tipset(synth.config_params(3))
    log(f"storage tipset (1M-entry HAMT): {ts3.n_blocks} blocks, {len(ts3.blob) / 1e6:.1f} MB, built in {time.time() - t0:.1f}s")
    st3 = api.BlockStore.from_tipset(ts3, device=local, verify_cids=True)
    ost = oracle.Store.from_tipset(ts3)
    peak, _ = peaks()
    out = {}
    rng = np.random.default_rng(3)
    for nk in (1000, 65536):
        present = rng.choice(1_000_000, size=nk - nk // 10, replace=False)
        keys = [ts3.storage_entry(int(k))[0] for k in present] + [ts3.storage_absent_key(int(k)) for k in range(nk // 10)]
        slots = np.frombuffer(b"".join(api.compute_mapping_slots(keys, [0] * len(keys), device=local)), dtype=np.uint8)
        root = np.ascontiguousarray(ts3.storage_root, dtype=np.uint8)

        def call():   # the plain C-ABI call: host keys in, values + witness (sorted CIDs, block bytes) on the host
            o = C.POINTER(A.SlotResultC)()
            t = time.perf_counter()
            rc = L.ipcfp_read_storage_slots(st3._h, root.ctypes.data, slots.ctypes.data, nk, C.byref(o))
            dt = 1e3 * (time.perf_counter() - t)
            assert rc == 0, L.ipcfp_last_error()
            k = float(o.contents.ms_lookup)
            L.ipcfp_slot_result_free(o)
            return dt, k
        for _ in range(3):
            call()
        ms, walls = [], []
        for _ in range(max(args.steps, 5)):
            dt, k = call()
            walls.append(dt)
            ms.append(k)
        r = st3.read_storage_slots(ts3.storage_root, slots)
        k_ms = float(np.median(ms))
        t = time.time()
        exp = ost.read_storage_slots(ts3.storage_root, slots[: 32 * min(nk, 4096)])
        cpu_s = time.time() - t
        n_cmp = min(nk, 4096)
        same = bool(np.array_equal(exp.values, r.values[:n_cmp]) and np.array_equal(exp.found, r.found[:n_cmp]))
        if nk == 1000:
            expw = ost.read_storage_slots(ts3.storage_root, slots)
            same = same and bool(np.array_equal(expw.witness.cids, r.witness.cids)) and expw.witness.blocks() == r.witness.blocks()
        out[f"lookups_{nk}"] = {
            "lookups": nk, "kernel_ms": k_ms, "lookups_per_s_kernel": nk / (k_ms / 1e3), "call_ms_wall": float(np.median(walls)),
            "lookups_per_s_call": nk / (float(np.median(walls)) / 1e3), "hamt_nodes": r.lookup_nodes, "algorithmic_bytes": r.lookup_bytes,
            "roofline": {"kernel": "k_read_slots", "bound": "hbm", "achieved": r.lookup_bytes / (k_ms / 1e3) / 1e9, "peak": peak, "unit": "GB/s",
                         "frac": r.lookup_bytes / (k_ms / 1e3) / 1e9 / peak, "traffic": None},
            "witness_blocks": int(r.witness.n_blocks), "found": int(r.found.sum()),
            "cpu_baseline": {"value": n_cmp / cpu_s, "unit": "lookups/s", "cores": 1, "kind": "port", "sample": f"the first {n_cmp} lookups, oracle_read_storage_slots"},
            "parity": same,
        }
    st3.close()
    return out


def run_engine(args, world, rank, local):
    import torch
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api

    assert torch.cuda.is_available(), "bench.py needs a CUDA device: the engine has no CPU path"
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        if os.environ.get("NCCL_DEBUG", "").upper() in ("", "VERSION"):
            os.environ["NCCL_DEBUG"] = "WARN"   # keep stdout to the one JSON line
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    L = api.lib()
    ts, lo, hi = build_tipset(world, rank)
    spec = A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter)
    N_local = hi - lo
    bounds = np.array([RECEIPTS_PER_GPU * r for r in range(world + 1)], dtype=np.uint64)

    # pinned host copies of the flat arrays (what a binding would fill from RPC responses)
    def pinned(a):
        a = np.ascontiguousarray(a)
        pa = api.PinnedArray(a.nbytes)
        pa.array[:] = a.view(np.uint8).reshape(-1)
        return pa
    log("allocating pinned host buffers")
    p_cids, p_offs, p_lens, p_blob = pinned(ts.cids), pinned(ts.offsets), pinned(ts.lengths), pinned(ts.blob)
    p_roots, p_has = pinned(ts.events_roots), pinned(ts.has_events_root)
    log("pinned buffers ready")
    d, keep = A.make_tipset_desc(ts)
    d.events_roots = p_roots.array.ctypes.data
    d.has_events_root = p_has.array.ctypes.data
    h2d_bytes = p_cids.array.nbytes + p_offs.array.nbytes + p_lens.array.nbytes + p_blob.array.nbytes + p_roots.array.nbytes + p_has.array.nbytes

    def store_create(flags):
        h = C.c_void_p()
        rc = L.ipcfp_store_create(p_cids.array.ctypes.data, p_offs.array.ctypes.data, p_lens.array.ctypes.data, p_blob.array.ctypes.data,
                                  p_blob.array.nbytes, ts.n_blocks, local, flags, C.byref(h))
        assert rc == 0, L.ipcfp_last_error()
        return h

    # ---- resident-state objects
    store = store_create(A.STORE_VERIFY_CIDS)
    tip = C.c_void_p()
    assert L.ipcfp_tipset_upload(store, C.byref(d), C.byref(tip)) == 0, L.ipcfp_last_error()
    ext_stream = torch.cuda.ExternalStream(L.ipcfp_store_stream(store), device=torch.device("cuda", local))

    comm = None
    if world > 1:
        from ipc_filecoin_proofs_b200 import parallel as PL
        comm = PL.ShardedComm.from_torch_group(L, dist, local)   # the library's own NCCL communicators; torch only carried the id

    def run_shard(store_h, tip_h, flags=0):
        """One step on this rank. N = 1: ipcfp_generate_event_proof_resident. N > 1: ipcfp_generate_event_proof_sharded — local shard
        scan + the cross-shard execution order and witness-CID union, all inside the C-ABI call."""
        out = C.POINTER(A.EventResultC)()
        if world == 1:
            rc = L.ipcfp_generate_event_proof_resident(store_h, tip_h, C.byref(spec), flags, C.byref(out))
            assert rc == 0, L.ipcfp_last_error()
            return out
        return comm.generate_event_proof(store_h, tip_h, spec, bounds, flags)

    stats = {}

    def step_resident(full=True, keep=False):
        """keep: return the result instead of freeing it (the caller frees it outside the timed region)."""
        out = run_shard(store, tip)
        r = out.contents
        m = int(r.witness.n_blocks)
        # (summing 147 k block lengths in numpy costs ~0.1 ms of host time per step: done in the warm-up steps only, the timed steps reuse it)
        wbytes = (int(np.frombuffer((C.c_uint32 * m).from_address(r.witness.lengths), dtype=np.uint32).sum(dtype=np.uint64)) if m else 0) if full \
            else stats.get("witness_bytes", 0)
        stats.update(n_matching=int(r.n_matching), n_proofs=int(r.n_proofs), witness_blocks=m,
                     witness_bytes=wbytes, merged_witness_cids=int(r.n_union_cids) if world > 1 else m, n_exec=int(r.n_exec),
                     total_matching=int(r.total_matching) if world > 1 else int(r.n_matching), total_proofs=int(r.total_proofs) if world > 1 else int(r.n_proofs),
                     ms=dict(total=r.ms_total, txamt=r.ms_txamt, pass1=r.ms_pass1, pass2=r.ms_pass2, witness=r.ms_witness,
                             exchange=r.ms_exchange, fetch=r.ms_fetch, union=r.ms_union),
                     pass1_bytes=int(r.pass1_bytes), pass1_nodes=int(r.pass1_nodes),
                     d2h_bytes=int(r.n_matching) * 4 + int(r.n_proofs) * C.sizeof(A.EventProofC) + int(r.data_blob_size) +
                     int(r.witness.n_blocks) * (38 + 8 + 4) + int(r.witness.blob_size))
        if keep:
            return out
        L.ipcfp_event_result_free(out)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    # ---- resident timing
    log("store + tipset resident; warm-up")
    # the clock sampler starts BEFORE the warm-up steps, so that nothing idles between the last warm-up step and the timed region
    # (a 0.3 s pause there let the GPUs and NCCL's proxy threads fall asleep: the first timed step then took up to 1.6x a normal one)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
        time.sleep(0.3)
    barrier()
    for _ in range(max(args.warmup, 3)):
        step_resident()
    barrier()   # every rank enters the timed region together
    launches0 = api.kernel_launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    phase = {k: [] for k in ("total", "txamt", "pass1", "pass2", "witness", "exchange", "fetch", "union")}
    t_wall0 = time.time()
    ev0.record(ext_stream)
    step_wall = []
    last_out = None
    for i in range(args.steps):
        _t = time.perf_counter()
        last_out = step_resident(False, keep=bool(args.dump_outputs) and i == args.steps - 1)
        step_wall.append(1e3 * (time.perf_counter() - _t))
        for k in phase:
            phase[k].append(stats["ms"][k])
    ev1.record(ext_stream)
    torch.cuda.synchronize()
    t_wall1 = time.time()
    barrier()
    if last_out is not None:
        if rank == 0:
            names = dump_outputs(args.dump_outputs, A.event_result_from_c(last_out.contents))
            log(f"last timed step's results written to {args.dump_outputs}: {', '.join(names)}")
        L.ipcfp_event_result_free(last_out)
    launches = api.kernel_launch_count() - launches0
    # CUDA events on the engine stream bracket the K steps on every rank (each step ends with the results on the host); max over ranks
    dev_ms = ev0.elapsed_time(ev1)
    t_local = torch.tensor([dev_ms, (t_wall1 - t_wall0) * 1e3], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(t_local, op=dist.ReduceOp.MAX)
    dev_ms_max, wall_ms_max = [float(x) for x in t_local.cpu()]
    clocks = sampler.stop(t_wall0, t_wall1) if rank == 0 else None
    pass1_ms = phase["pass1"]
    log(f"resident timing done: {dev_ms_max / args.steps:.3f} ms/step (device), {wall_ms_max / args.steps:.3f} ms/step (wall); per-step wall ms: "
        + ", ".join(f"{x:.2f}" for x in step_wall))

    # ---- parity, outside the timed region: this rank's results + (N > 1) the merged witness CID union, byte for byte against the oracle
    out = run_shard(store, tip, A.SHARDED_UNION_TO_HOST if world > 1 else 0)
    r = out.contents
    got = A.event_result_from_c(r)
    n_union = int(r.n_union_cids)
    # N > 1: the merged witness CID list stays distributed — this rank's partition, entries [union_part_first, +n_union_part) of the sorted set
    n_part, part_first = (int(r.n_union_part), int(r.union_part_first)) if world > 1 else (0, 0)
    union = np.frombuffer((C.c_uint8 * (n_part * 38)).from_address(r.union_cids), dtype=np.uint8).copy() if world > 1 and n_part else np.zeros(0, np.uint8)
    L.ipcfp_event_result_free(out)
    import hashlib
    mine = {"matching": hashlib.sha256(got.matching.tobytes()).hexdigest(), "proofs": digest_proofs(got), "n_exec": int(got.n_exec),
            "witness": hashlib.sha256(got.witness.cids.tobytes()).hexdigest() + hashlib.sha256(b"".join(got.witness.blocks())).hexdigest(),
            "union": (part_first, n_union, union.tobytes()) if world > 1 else None}

    # ---- separately labelled mode (N = 1): the witness BY REFERENCE (IPCFP_WITNESS_BY_REFERENCE) — CIDs / offsets / lengths only, the
    # offsets naming blocks inside the host blob the store was created from, instead of 51 MB of copied block bytes. Not the headline:
    # `value` above stays byte-complete. Its equality with the copied witness is a GPU test (tests/test_zz_witness_by_reference.py).
    by_reference = None
    if world == 1:
        try:
            for _ in range(3):
                L.ipcfp_event_result_free(run_shard(store, tip, A.WITNESS_BY_REFERENCE))
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext_stream)
            for _ in range(args.steps):
                o = run_shard(store, tip, A.WITNESS_BY_REFERENCE)
                rr = o.contents
                ref_counts = (int(rr.n_matching), int(rr.n_proofs), int(rr.witness.n_blocks), int(rr.witness.blob_size))
                L.ipcfp_event_result_free(o)
            e1.record(ext_stream)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            by_reference = {"value": N_local / (ms / 1e3), "unit": "receipts/s", "ms_per_step": ms,
                            "d2h_bytes_per_step": ref_counts[0] * 4 + ref_counts[1] * C.sizeof(A.EventProofC) + ref_counts[2] * (38 + 8 + 4),
                            "same_counts_as_default": ref_counts[:3] == (stats["n_matching"], stats["n_proofs"], stats["witness_blocks"]) and ref_counts[3] == 0,
                            "note": "witness blocks referenced in the caller's own blob, not copied; everything else as in `value`"}
            log(f"by-reference mode: {ms:.3f} ms/step")
        except Exception as e:   # an optional mode must never cost the headline line
            by_reference = {"error": repr(e)[:200]}

    # ---- end-to-end timing (host buffers → results on the host), every step re-ingests the block set
    L.ipcfp_tipset_free(tip)
    L.ipcfp_store_destroy(store)
    e2e_steps = max(1, min(args.steps, 5))
    e2e_parts = []

    def step_e2e():
        t0 = time.time()
        h = store_create(A.STORE_VERIFY_CIDS)
        t1 = time.time()
        tp = C.c_void_p()
        assert L.ipcfp_tipset_upload(h, C.byref(d), C.byref(tp)) == 0, L.ipcfp_last_error()
        out = run_shard(h, tp)
        t2 = time.time()
        L.ipcfp_event_result_free(out)
        L.ipcfp_tipset_free(tp)
        L.ipcfp_store_destroy(h)
        t3 = time.time()
        e2e_parts.append((round(1e3 * (t1 - t0), 2), round(1e3 * (t2 - t1), 2), round(1e3 * (t3 - t2), 2)))

    for _ in range(3):          # W >= 3 warm-up steps here too: the device / pinned pools reach their steady state after two store generations
        step_e2e()
    barrier()
    t0 = time.time()
    for _ in range(e2e_steps):
        step_e2e()
    barrier()
    e2e_ms = (time.time() - t0) * 1e3 / e2e_steps
    t_e2e = torch.tensor([e2e_ms], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(t_e2e, op=dist.ReduceOp.MAX)
    e2e_ms = float(t_e2e.cpu()[0])
    log(f"e2e timing done: {e2e_ms:.2f} ms/step; (store_create, generate, destroy) ms per step: {e2e_parts}")

    # ---- the oracle: CPU baseline (N = 1: single-threaded like the reference, timed) and the parity verdict (all N)
    cpu_baseline = None
    parity = None
    verify = not args.no_cpu_baseline and not os.environ.get("IPCFP_BENCH_NO_VERIFY")
    if world == 1 and verify:
        import oracle
        ost = oracle.Store.from_tipset(ts)
        t0 = time.time()
        exp = ost.generate_event_proof(ts, spec, threads=1)
        dt = time.time() - t0
        theirs = {"matching": hashlib.sha256(exp.matching.tobytes()).hexdigest(), "proofs": digest_proofs(exp), "n_exec": int(exp.n_exec),
                  "witness": hashlib.sha256(exp.witness.cids.tobytes()).hexdigest() + hashlib.sha256(b"".join(exp.witness.blocks())).hexdigest(), "union": None}
        parity = mine == theirs
        cpu_baseline = {"value": ts.n_receipts / dt, "unit": "receipts/s", "cores": 1, "kind": "port",
                        "sample": "the full 1M-receipt workload, 1 repetition, single-threaded C++ restatement of the reference "
                                  "(the reference is single-threaded; its Rust crate cannot be built in this image)",
                        "seconds": dt, "agrees_with_gpu": bool(parity),
                        "compared": "sha256 of: matching indices, every EventProof field incl. message_cid, witness CIDs, witness block bytes; n_exec"}
    elif world > 1 and verify:
        # every rank sends the digests of its own results; rank 0 builds the WHOLE tipset and runs the oracle on all host threads
        allm = [None] * world
        dist.all_gather_object(allm, mine)
        if rank == 0:
            import oracle
            import synth
            t0 = time.time()
            full = synth.Tipset(synth.config_params(4, n_receipts=RECEIPTS_PER_GPU * world))
            fspec = A.make_event_spec(full.event_signature, full.topic1, full.actor_filter)
            ost = oracle.Store.from_tipset(full)
            exp = ost.generate_event_proof(full, fspec, threads=os.cpu_count() or 1)
            # the ranks' partitions, concatenated in rank order, are the oracle's sorted witness CID list byte for byte
            ok = b"".join(m["union"][2] for m in allm) == exp.witness.cids.tobytes()
            ok = ok and all(m["union"][1] == len(exp.witness.cids) for m in allm)
            ok = ok and [m["union"][0] for m in allm] == [sum(len(q["union"][2]) // 38 for q in allm[:k]) for k in range(world)]
            ok = ok and all(m["n_exec"] == int(exp.n_exec) for m in allm)
            for q in range(world):
                qlo, qhi = int(bounds[q]), int(bounds[q + 1])
                sel = exp.matching[(exp.matching >= qlo) & (exp.matching < qhi)]
                ok = ok and hashlib.sha256(sel.tobytes()).hexdigest() == allm[q]["matching"]
                h = hashlib.sha256()
                for p in exp.proofs:
                    if qlo <= p.exec_index < qhi:
                        h.update(repr(p.key()).encode())
                ok = ok and h.hexdigest() == allm[q]["proofs"]
            parity = bool(ok)
            log(f"parity check against the oracle of the whole {world}M-receipt tipset: {parity} ({time.time() - t0:.1f}s)")
        dist.barrier()
    log("verification done")

    storage = None
    if rank == 0 and world == 1 and not args.no_storage:
        storage = storage_section(api, A, L, local, args)
        log("storage section done")

    if rank == 0:
        n_total = N_local * world
        value = n_total * args.steps / (dev_ms_max / 1e3)
        peak, peak_src = peaks()
        p1 = float(np.mean(pass1_ms))
        achieved = stats["pass1_bytes"] / (p1 / 1e3) / 1e9
        step_bytes = stats["pass1_bytes"] + 2 * stats["witness_bytes"] + 50 * stats["n_exec"] // max(world, 1)
        line = {
            "metric": "receipts/sec scanned", "value": value, "unit": "receipts/s", "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": dev_ms_max / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8",
            "data": "synthetic",
            "config": config_dict(world, N_local, store_blocks_per_gpu=int(ts.n_blocks), store_bytes_per_gpu=int(len(ts.blob)),
                                  matching_rank0=stats["n_matching"], proofs_rank0=stats["n_proofs"], matching_total=stats["total_matching"],
                                  proofs_total=stats["total_proofs"], witness_blocks_rank0=stats["witness_blocks"],
                                  merged_witness_cids=stats["merged_witness_cids"], n_exec=stats["n_exec"],
                                  note="the reference arm always scans ONE 1M-receipt tipset on the host (rank 0); at --gpus N > 1 the engine arm scans "
                                       "an N x 1M-receipt tipset (weak scaling): compare receipts/s, not same-input wall time"),
            "parity": parity,
            "by_reference": by_reference,
            "witness_bytes_per_s": stats["witness_bytes"] * world * args.steps / (dev_ms_max / 1e3),
            "wall_ms_per_step": wall_ms_max / args.steps,
            "device_ms_breakdown": {k: float(np.mean(v)) for k, v in phase.items()},
            "step_hbm": {"algorithmic_bytes_per_step_per_gpu": int(step_bytes), "achieved_gbs": step_bytes / (dev_ms_max / args.steps / 1e3) / 1e9,
                         "frac_of_peak": step_bytes / (dev_ms_max / args.steps / 1e3) / 1e9 / peak,
                         "note": "whole step incl. the PCIe copy of the results: pass-1 bytes + witness blocks read and written once + message-AMT nodes"},
            "roofline": {"kernel": os.environ.get("IPCFP_PASS1_STAGE", "k_pass1_stage 128x4x1") + " (pass 1, csrc/events.cu)", "bound": "hbm", "achieved": achieved, "peak": peak,
                         "unit": "GB/s", "frac": achieved / peak,
                         "traffic": None, "algorithmic_bytes_per_launch": stats["pass1_bytes"], "ms_per_launch": p1,
                         "peak_source": peak_src},
            "cpu_baseline": cpu_baseline,
            "e2e": {"value": n_total / (e2e_ms / 1e3), "unit": "receipts/s", "ms_per_step": e2e_ms, "steps": e2e_steps,
                    "h2d_bytes_per_step": int(h2d_bytes), "d2h_bytes_per_step": int(stats["d2h_bytes"]),
                    "parts_ms_rank0": {"store_create": [p[0] for p in e2e_parts[3:]], "generate": [p[1] for p in e2e_parts[3:]], "destroy": [p[2] for p in e2e_parts[3:]]},
                    # what bounds e2e: the H2D of every block over PCIe (ingest = copy + index + Cid ranks + Blake2b check, all under the copy)
                    "ingest_h2d_gbs_rank0": float(h2d_bytes / (max(np.median([p[0] for p in e2e_parts[3:]]), 1e-6) / 1e3) / 1e9)},
            "storage": storage,
            "gpu_launches": int(launches),
            "clocks": clocks,
            "gpu": gpu_info(local),
        }
        print(json.dumps(line), flush=True)
    if comm is not None:
        comm.close()
    if world > 1:
        dist.destroy_process_group()


def main():
    # stdout carries exactly one JSON line: everything else a library prints (e.g. NCCL's version banner) goes to stderr
    real_stdout = os.dup(1)
    os.dup2(2, 1)
    sys.stdout = os.fdopen(real_stdout, "w", buffering=1)
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="engine", choices=["engine", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-storage", action="store_true", help="skip the HAMT storage-lookup section (configs[2])")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one returned (rank 0) as DIR/<name>.npy (float32/float64, < 64 MB)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    world, rank, local = dist_env()
    if args.impl == "reference":
        run_reference(args, world, rank)
    else:
        run_engine(args, world, rank, local)


if __name__ == "__main__":
    main()
