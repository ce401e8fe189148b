"""The multi-GPU event path: one shard's scan against the oracle on one GPU, and the in-library sharded call over NCCL."""
import ctypes as C

import numpy as np
import pytest

from tests import dist_worker


@pytest.mark.gpu
def test_shard_scan_one_gpu(api, oracle_mod, synth_mod):
    """ipcfp_generate_event_proof_shard_resident for rank 0 and then rank 1 of world 2, each on its own shard's store on one GPU,
    against the oracle's shard scan of the whole tipset: the matches, every proof field but message_cid, and the local witness. The
    shard call leaves the execution order to the sharded call, so message_cid is zero and n_exec is 0."""
    from ipc_filecoin_proofs_b200 import _abi as A
    L = api.lib()
    P = dist_worker.PARAMS
    N, world = P["n_receipts"], 2
    full = synth_mod.Tipset(synth_mod.default_params(**P))
    spec = A.make_event_spec(full.event_signature, full.topic1, full.actor_filter)
    ost = oracle_mod.Store.from_tipset(full)
    for rank in range(world):
        lo, hi = N * rank // world, N * (rank + 1) // world
        exp = ost.generate_event_proof_shard(full, spec, lo, hi, world, rank)
        shard = synth_mod.Tipset(synth_mod.default_params(shard_lo=lo, shard_hi=hi, **P))
        store = api.BlockStore.from_tipset(shard, device=0, verify_cids=True)
        d, keep = A.make_tipset_desc(shard)
        tip = C.c_void_p()
        api._check(L.ipcfp_tipset_upload(store._h, C.byref(d), C.byref(tip)))
        out = C.POINTER(A.EventResultC)()
        try:
            api._check(L.ipcfp_generate_event_proof_shard_resident(store._h, tip, C.byref(spec), lo, hi, world, rank, 0, C.byref(out)))
            got = A.event_result_from_c(out.contents)
        finally:
            if out:
                L.ipcfp_event_result_free(out)
            L.ipcfp_tipset_free(tip)
            store.close()
        assert len(exp.proofs), "the shard has no proof to compare"
        assert got.matching.tolist() == exp.matching.tolist()
        assert [p.key()[:-1] for p in got.proofs] == [p.key()[:-1] for p in exp.proofs]
        assert all(p.message_cid == bytes(38) for p in got.proofs) and got.n_exec == 0
        assert np.array_equal(got.witness.cids, exp.witness.cids) and got.witness.blocks() == exp.witness.blocks()


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_sharded_call_over_nccl(world):
    """The in-library protocol (ipcfp_comm_init + ipcfp_generate_event_proof_sharded), one rank per GPU over NCCL, bit-exact against
    the oracle of the whole tipset (proofs incl. message_cid, n_exec, merged witness CID list) and failing together on a fault."""
    if _n_gpus() < world:
        pytest.skip(f"needs {world} visible GPUs")
    dist_worker.run(dist_worker.nccl_worker, world=world)
