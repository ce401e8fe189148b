"""Workers for the multi-process tests of the sharded call (spawned by torch.multiprocessing)."""
import os
import sys
import traceback

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PARAMS = dict(seed=123, n_receipts=3000, events_per_receipt=4, match_ppm=30000, dup_msgs=9, n_parents=3)


def _init(rank, world, port, backend):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group(backend, rank=rank, world_size=world)
    return dist


def nccl_worker(rank, world, port, q):
    """One rank per GPU: the library's own protocol (ipcfp_generate_event_proof_sharded over NCCL) against the oracle of the WHOLE
    tipset — every EventProof incl. message_cid, n_exec, the local witness, the merged witness CID union — and the common failure."""
    try:
        import ctypes as C
        import oracle
        import synth
        from ipc_filecoin_proofs_b200 import _abi as A
        from ipc_filecoin_proofs_b200 import api
        from ipc_filecoin_proofs_b200 import parallel as PL
        import torch
        dist = _init(rank, world, port, "gloo")       # carries the 128-byte id only
        dev = rank % torch.cuda.device_count()
        L = api.lib()
        comm = PL.ShardedComm.from_torch_group(L, dist, dev)
        for params in (PARAMS, dict(seed=5, n_receipts=20011, events_per_receipt=8, match_ppm=2000, dup_msgs=0, n_parents=2),
                       dict(seed=9, n_receipts=257, events_per_receipt=3, match_ppm=500000, dup_msgs=40, n_parents=5),
                       # uneven shards: rank 0 owns 70 % of the receipts, so the per-rank match counts differ by hundreds (request padding)
                       dict(seed=11, n_receipts=4001, events_per_receipt=4, match_ppm=300000, dup_msgs=25, n_parents=3, skew=True)):
            params = dict(params)
            skew = params.pop("skew", False)
            N = params["n_receipts"]
            bounds = [N * r // world for r in range(world + 1)]
            if skew and world > 1:
                head = N * 7 // 10
                bounds = [0] + [head + (N - head) * r // (world - 1) for r in range(world)]
            lo, hi = bounds[rank], bounds[rank + 1]
            full = synth.Tipset(synth.default_params(**params))
            shard = synth.Tipset(synth.default_params(shard_lo=lo, shard_hi=hi, **params)) if world > 1 else full
            spec = A.make_event_spec(full.event_signature, full.topic1, full.actor_filter)
            ost = oracle.Store.from_tipset(full)
            exp = ost.generate_event_proof(full, spec)
            exp_shard = ost.generate_event_proof_shard(full, spec, lo, hi, world, rank) if world > 1 else exp
            store = api.BlockStore.from_tipset(shard, device=dev, verify_cids=True)
            d, keep = A.make_tipset_desc(shard)
            tip = C.c_void_p()
            assert L.ipcfp_tipset_upload(store._h, C.byref(d), C.byref(tip)) == 0
            for rep in range(3):                           # later calls reuse every buffer of the communicator
                # rep 0, 2: the witness union stays distributed (this rank's partition); rep 1: the whole list on every rank
                full_union = rep == 1
                if rep == 2:
                    os.environ["IPCFP_UNION_CAP"] = "3"      # pieces of 3 CIDs: the first attempt overflows on every rank, the repeat must deliver
                else:
                    os.environ.pop("IPCFP_UNION_CAP", None)
                out = comm.generate_event_proof(store._h, tip, spec, bounds, A.SHARDED_UNION_TO_HOST | (A.SHARDED_UNION_FULL if full_union else 0))
                r = out.contents
                got = A.event_result_from_c(r)
                n_union, n_part, part_first = int(r.n_union_cids), int(r.n_union_part), int(r.union_part_first)
                union = np.frombuffer((C.c_uint8 * (n_part * 38)).from_address(r.union_cids), dtype=np.uint8).reshape(-1, 38).copy() if n_part else np.zeros((0, 38), np.uint8)
                totals = (int(r.total_matching), int(r.total_proofs), int(r.n_exec))
                L.ipcfp_event_result_free(out)
                assert n_union == len(exp.witness.cids), (n_union, len(exp.witness.cids))
                if full_union:
                    assert (part_first, n_part) == (0, n_union)
                else:
                    parts = [None] * world
                    dist.all_gather_object(parts, (part_first, union.tobytes()))
                    assert [p[0] for p in parts] == [sum(len(q[1]) // 38 for q in parts[:k]) for k in range(world)], [p[0] for p in parts]
                    if world > 1 and n_union > 64 * world:
                        assert all(len(p[1]) for p in parts), "a partition is empty: CIDs are not spread over the ranks"
                    union = np.frombuffer(b"".join(p[1] for p in parts), dtype=np.uint8).reshape(-1, 38)
                os.environ.pop("IPCFP_UNION_CAP", None)
                assert totals == (len(exp.matching), len(exp.proofs), exp.n_exec), (totals, len(exp.matching), len(exp.proofs), exp.n_exec)
                assert got.matching.tolist() == exp_shard.matching.tolist()
                mine = [p for p in exp.proofs if lo <= p.exec_index < hi]
                assert [p.key() for p in got.proofs] == [p.key() for p in mine]                       # message_cid included
                assert np.array_equal(got.witness.cids, exp_shard.witness.cids) and got.witness.blocks() == exp_shard.witness.blocks()
                assert np.array_equal(union, exp.witness.cids), (union.shape, exp.witness.cids.shape)
            # a fault on ONE rank: every rank fails, naming the same error — the one the oracle of the whole tipset names
            if len(exp.matching):
                victim_rcpt = int(exp.matching[len(exp.matching) // 2])
                owner = max(r for r in range(world) if bounds[r] <= victim_rcpt)
                bad = shard
                if owner == rank:
                    from tests.util import EditedTipset
                    cid = bytes(full.events_roots[victim_rcpt])
                    idx = next(i for i in range(shard.n_blocks) if bytes(shard.cids[i]) == cid)
                    blob = shard.blob.copy()
                    blob[int(shard.offsets[idx])] ^= 0xff                                              # root block no longer decodes
                    bad = EditedTipset(shard, blob=blob)
                fidx = next(i for i in range(full.n_blocks) if bytes(full.cids[i]) == bytes(full.events_roots[victim_rcpt]))
                fblob = full.blob.copy()
                fblob[int(full.offsets[fidx])] ^= 0xff
                from tests.util import EditedTipset as ET
                try:
                    oracle.Store.from_tipset(ET(full, blob=fblob)).generate_event_proof(full, spec)
                    raise AssertionError("oracle accepted a damaged block")
                except A.IpcfpError as e:
                    want = (e.status, e.index)
                bstore = api.BlockStore.from_tipset(bad, device=dev)
                btip = C.c_void_p()
                assert L.ipcfp_tipset_upload(bstore._h, C.byref(d), C.byref(btip)) == 0
                try:
                    o2 = comm.generate_event_proof(bstore._h, btip, spec, bounds)
                    L.ipcfp_event_result_free(o2)
                    raise AssertionError("sharded call accepted a damaged block")
                except A.IpcfpError as e:
                    assert (e.status, e.index) == want, ((e.status, e.index), want)
                L.ipcfp_tipset_free(btip)
                bstore.close()
            L.ipcfp_tipset_free(tip)
            store.close()

        def outcome_sharded(shard_ts, N):
            bounds = [N * r // world for r in range(world + 1)]
            spec = A.make_event_spec(shard_ts.event_signature, shard_ts.topic1, shard_ts.actor_filter)
            st_ = api.BlockStore.from_tipset(shard_ts, device=dev)
            d_, k_ = A.make_tipset_desc(shard_ts)
            tp = C.c_void_p()
            assert L.ipcfp_tipset_upload(st_._h, C.byref(d_), C.byref(tp)) == 0
            try:
                o = comm.generate_event_proof(st_._h, tp, spec, bounds, A.SHARDED_UNION_TO_HOST | A.SHARDED_UNION_FULL)
                r_ = o.contents
                g = A.event_result_from_c(r_)
                nu = int(r_.n_union_cids)
                un = np.frombuffer((C.c_uint8 * (nu * 38)).from_address(r_.union_cids), dtype=np.uint8).reshape(-1, 38).copy() if nu else np.zeros((0, 38), np.uint8)
                res = ("ok", g, int(r_.n_exec), un)
                L.ipcfp_event_result_free(o)
                return res
            except A.IpcfpError as e:
                return ("err", e.status, e.index)
            finally:
                L.ipcfp_tipset_free(tp)
                st_.close()

        def outcome_oracle(full_ts):
            spec = A.make_event_spec(full_ts.event_signature, full_ts.topic1, full_ts.actor_filter)
            try:
                return ("ok", oracle.Store.from_tipset(full_ts).generate_event_proof(full_ts, spec))
            except A.IpcfpError as e:
                return ("err", e.status, e.index)

        def compare(got, exp, lo, hi):
            assert got[0] == exp[0], (got[:3] if got[0] == "err" else got[0], exp[:3] if exp[0] == "err" else exp[0])
            if got[0] == "err":
                assert got[1:] == exp[1:], (got, exp)
                return
            g, n_exec, union = got[1], got[2], got[3]
            e = exp[1]
            assert n_exec == e.n_exec
            assert g.matching.tolist() == [int(i) for i in e.matching if lo <= i < hi]
            assert [p.key() for p in g.proofs] == [p.key() for p in e.proofs if lo <= p.exec_index < hi]
            assert np.array_equal(union, e.witness.cids)

        # ---- the LATE path of the protocol: no shard promises its slice early (general walk forced)
        N = PARAMS["n_receipts"]
        lo, hi = N * rank // world, N * (rank + 1) // world
        full = synth.Tipset(synth.default_params(**PARAMS))
        shard = synth.Tipset(synth.default_params(shard_lo=lo, shard_hi=hi, **PARAMS)) if world > 1 else full
        os.environ["IPCFP_BFS_GENERAL"] = "1"
        compare(outcome_sharded(shard, N), outcome_oracle(full), lo, hi)
        del os.environ["IPCFP_BFS_GENERAL"]
        # ---- the STALE path: a message AMT with a hole (its root still promises a dense list): the dense walk of the shard that owns the
        # hole gives up AFTER the early exchange has started; every shard then repeats the exchange with the real slices
        import cbor2
        from tests.test_oracle_cpu import _patched
        dct = full.as_dict()
        tm = cbor2.loads(dct[bytes(full.parent_txmeta_cids[0])])
        root_cid = tm[0].value[1:]
        height, count, node = cbor2.loads(dct[root_cid])
        cur_cid, cur, is_root = root_cid, node, True
        while cur[1]:
            cur_cid = cur[1][0].value[1:]
            cur, is_root = cbor2.loads(dct[cur_cid]), False
        bmap, links, vals = cur
        if len(vals) >= 2:
            slots = [b for b in range(8) if bmap[0] >> b & 1]
            node2 = [bytes([bmap[0] & ~(1 << slots[-1])]), [], vals[:-1]]
            new = cbor2.dumps([height, count, node2]) if is_root else cbor2.dumps(node2)
            full2 = _patched(full, cur_cid, new)
            has = any(bytes(shard.cids[i]) == bytes(cur_cid) for i in range(shard.n_blocks))
            shard2 = _patched(shard, cur_cid, new) if has else shard
            compare(outcome_sharded(shard2, N), outcome_oracle(full2), lo, hi)
        comm.close()
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception:
        q.put((rank, traceback.format_exc()))


def run(worker, world=2):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = []
    for _ in procs:
        results.append(q.get(timeout=600))
    for p in procs:
        p.join(timeout=60)
    bad = [r for r in results if r[1] != "ok"]
    assert not bad, "\n".join(f"rank {r}: {msg}" for r, msg in bad)
