"""ipcfp_verify_bundle_json against the composed host flow it replaces, alternated in one process on the same text:
  host:   ipcfp_bundle_from_json → ipcfp_store_create(IPCFP_STORE_VERIFY_CIDS) → ipcfp_verify_storage_proofs / ipcfp_verify_event_proofs
  device: ipcfp_verify_bundle_json (canonical text: device parser)
on the EventProofBundle text of config 1 and of the 1 M-receipt tipset (IPCFP_RESULT_JSON). For every arm: median / min / max wall time
after warm-up, kernel launches per call, and for the device arm the verdict's ms_parse / ms_store / ms_verify split. Also the H2D copy
of the text from pageable memory alone (torch), and the card's name and power limit read in the same run. Both arms must agree."""
import argparse
import ctypes as C
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.json_step import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--receipts", type=int, default=1_000_000)
    args = ap.parse_args()
    import numpy as np
    import torch

    import synth
    from ipc_filecoin_proofs_b200 import _abi as A
    from ipc_filecoin_proofs_b200 import api
    from tests.util import spec_of
    L = api.lib()
    print(f"card: {card()}")
    for name, params in (("config 1", synth.config_params(1)), (f"{args.receipts} receipts", synth.config_params(4, n_receipts=args.receipts))):
        ts = synth.Tipset(params)
        spec = spec_of(ts)
        text = api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec, flags=A.RESULT_JSON | A.WITNESS_BY_REFERENCE).json.encode()

        def host():
            pb = api.ParsedBundle(text)
            c = pb.c
            w = c.witness
            store = C.c_void_p()
            api._check(L.ipcfp_store_create(w.cids, w.offsets, w.lengths, w.blob, w.blob_size, w.n_blocks, 0, A.STORE_VERIFY_CIDS, C.byref(store)))
            n = int(c.n_event_proofs)
            res = np.zeros(max(n, 1), np.uint8)
            api._check(L.ipcfp_verify_event_proofs(store, C.byref(c.tipset), c.event_proofs, n, c.data_blob, c.data_blob_size, C.addressof(spec),
                                                   res.ctypes.data))
            L.ipcfp_store_destroy(store)
            pb.close()
            return [bool(x) for x in res[:n]]

        def device():
            v = api.verify_bundle_json(text, filter_spec=spec)
            assert v.parsed_on_device
            return v

        def h2d():
            t = torch.frombuffer(bytearray(text), dtype=torch.uint8)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            t.to("cuda")
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        wall = {"host": [], "device": [], "h2d": []}
        split, launches = [], {}
        for k in range(args.warmup + args.runs):
            for arm in ("host", "device"):
                n0 = api.kernel_launch_count()
                t0 = time.perf_counter()
                out = host() if arm == "host" else device()
                dt = time.perf_counter() - t0
                launches[arm] = api.kernel_launch_count() - n0
                if arm == "host":
                    want = out
                else:
                    assert out.event_results == want
                    if k >= args.warmup:
                        split.append(out.ms)
                if k >= args.warmup:
                    wall[arm].append(dt * 1e3)
            if k >= args.warmup:
                wall["h2d"].append(h2d() * 1e3)
        print(f"\n{name}: {len(text) / 1e6:.1f} MB of text, {len(want)} event proofs, all verified: {all(want)}")
        for arm, label in (("host", "composed host flow"), ("device", "ipcfp_verify_bundle_json"), ("h2d", "H2D of the text (pageable)")):
            w = wall[arm]
            extra = f"  {launches[arm]} launches" if arm in launches else ""
            print(f"  {label:28s} median {statistics.median(w):9.3f} ms [{min(w):9.3f}, {max(w):9.3f}] over {len(w)}{extra}")
        print("  device split (median ms): " + ", ".join(f"{k} {statistics.median(s[k] for s in split):.3f}" for k in ("parse", "store", "verify", "total")))


if __name__ == "__main__":
    main()
