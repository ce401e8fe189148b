"""Storage paths against the route they replace, alternated in one process with a parity check of the outputs:
  mapping  65 536 two-level mapping paths, allowance[k1][k2] (mapping(bytes32 => mapping(uint256 => uint256)) at slot 0) over configs[2]'s
           1 M-slot trie: ipcfp_generate_storage_path_proofs_resident against the composed route, keccak256_batch twice for the slots
           then generate_storage_proofs;
  strings  1 000 strings of 1 KiB (33 slots each) in a trie of their own: the call against keccak256_batch + generate_storage_proofs for
           the header words, the lengths decoded on the host, keccak256_batch + generate_storage_proofs again for the data slots.
Reports, per workload, the call's device time per phase (ms_slots, ms_wave1, ms_wave2, ms_witness, ms_total) and its host
synchronisations, and the composed route's device time (the ms_total of its storage calls) and wall times of both, median / min / max
over --runs after --warmup. Prints one JSON line with the card's name and power limit read in the same run."""
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


def stat(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs))


def run(label, runs, warmup, path_call, composed_call):
    """alternates the two routes; path_call() → PathResultPy, composed_call() → (StorageResultPy list, device ms); parity every run"""
    ph = {k: [] for k in ("slots", "wave1", "wave2", "witness", "total")}
    wall_p, wall_c, dev_c, syncs = [], [], [], 0
    for k in range(warmup + runs):
        t0 = time.perf_counter()
        r = path_call()
        t1 = time.perf_counter()
        parts, ms = composed_call()
        t2 = time.perf_counter()
        import numpy as np
        assert np.array_equal(r.storage.raw_proofs, np.concatenate([p.raw_proofs for p in parts])), f"{label}: proofs differ"
        if k >= warmup:
            for key in ph:
                ph[key].append(r.timings[key])
            wall_p.append((t1 - t0) * 1e3)
            wall_c.append((t2 - t1) * 1e3)
            dev_c.append(ms)
            syncs = r.host_syncs
    return dict(paths=len(r.paths), specs=len(r.specs), call=dict(device_ms={k: stat(v) for k, v in ph.items()}, wall_ms=stat(wall_p), host_syncs=syncs),
                composed=dict(device_ms=stat(dev_c), wall_ms=stat(wall_c)), parity=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--paths", type=int, default=65536)
    ap.add_argument("--strings", type=int, default=1000)
    args = ap.parse_args()
    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    from tests import storage_paths as SP
    name = card()
    out = dict(card=name)

    # ---- mapping: configs[2]
    ts = synth.Tipset(synth.config_params(3))
    store = api.BlockStore.from_tipset(ts)
    tip = store.upload_tipset(ts)
    probe = bytes(32)
    def root_of(a):
        try:
            return bytes(store.generate_storage_proofs(ts, [(a, probe)]).proofs[0].storage_root)
        except A.IpcfpError:
            return None
    actor = next(a for a in range(1000, 1100) if root_of(a) == bytes(ts.storage_root))   # the actor whose contract state is the 1 M-slot trie
    rng = random.Random(1)
    k1 = [ts.storage_entry(rng.randrange(1000))[0] for _ in range(args.paths)]
    k2 = [rng.randrange(2 ** 64) for _ in range(args.paths)]
    paths = [api.StoragePath(actor, 0).mapping(a).mapping(b, "uint256") for a, b in zip(k1, k2)]

    def composed_mapping():
        inner = api.keccak256_batch([a + bytes(32) for a in k1])
        slots = api.keccak256_batch([SP.b32(b) + i for b, i in zip(k2, inner)])
        r = store.generate_storage_proofs(ts, [(actor, s) for s in slots])
        return [r], r.ms_total

    out["mapping"] = run("mapping", args.runs, args.warmup, lambda: store.generate_storage_path_proofs_resident(tip, paths), composed_mapping)
    tip.close()
    store.close()
    del ts

    # ---- strings: 1 000 strings of 1 KiB behind mapping(uint256 => string) at slot 12
    c = SP.Contract()
    storage = {}
    for k in range(args.strings):
        storage.update(SP.encode_string(SP.keccak256(SP.b32(k) + SP.b32(12)), bytes(rng.randrange(32, 127) for _ in range(1024))))
    c.storage = storage
    flat, stip_ts = c.world(synth.Tipset(synth.config_params(3, hamt_entries=20000)))
    store = api.BlockStore(flat.cids, flat.offsets, flat.lengths, flat.blob)
    tip = store.upload_tipset(stip_ts)
    spaths = [api.StoragePath(SP.ACTOR, 12).mapping(k, "uint256").bytes() for k in range(args.strings)]

    def composed_strings():
        heads = api.keccak256_batch([SP.b32(k) + SP.b32(12) for k in range(args.strings)])
        h = store.generate_storage_proofs(stip_ts, [(SP.ACTOR, s) for s in heads])
        bases = api.keccak256_batch(heads)
        data = []
        for q, b in zip(h.proofs, bases):
            n = SP.u256(q.value) >> 1
            data += [(SP.ACTOR, SP.b32(SP.u256(b) + j)) for j in range((n + 31) // 32)]
        d = store.generate_storage_proofs(stip_ts, data)
        # in path order: header, then its data slots
        import numpy as np
        size = h.raw_proofs.size // len(h.proofs)
        per = (len(d.proofs) // args.strings)
        rows = []
        for i in range(args.strings):
            rows.append(h.raw_proofs[i * size:(i + 1) * size])
            rows.append(d.raw_proofs[i * per * size:(i + 1) * per * size])
        merged = A.StorageResultPy([], None, [], 0.0, np.concatenate(rows))
        return [merged], h.ms_total + d.ms_total

    out["strings"] = run("strings", args.runs, args.warmup, lambda: store.generate_storage_path_proofs_resident(tip, spaths), composed_strings)
    tip.close()
    store.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
