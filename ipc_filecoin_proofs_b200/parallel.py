"""Multi-GPU event proofs: one process per GPU, receipts sharded by index range. The library resolves what spans shards (the
execution order, the proofs' message CIDs, the union of the witness CID sets) inside one call per rank; `ShardedComm` makes it."""
import ctypes as C

import numpy as np

from . import _abi as A


class ShardedComm:
    """Thin caller of the library's own cross-shard protocol (`ipcfp_comm_init` / `ipcfp_generate_event_proof_sharded`,
    csrc/parallel.cu): the collectives run inside the C-ABI call over NCCL, on the engine's streams. This class only moves
    the 128-byte communicator id between the ranks (any transport: here an optional torch.distributed group)."""

    def __init__(self, lib, world, rank, device, id_bytes):
        self.L, self.world, self.rank, self.device = lib, world, rank, device
        idb = (C.c_uint8 * A.COMM_ID_BYTES).from_buffer_copy(bytes(id_bytes))
        h = C.c_void_p()
        st = lib.ipcfp_comm_init(idb, world, rank, device, C.byref(h))
        if st != A.OK:
            raise A.IpcfpError(st, lib.ipcfp_last_error().decode(errors="replace"), lib.ipcfp_last_error_index())
        self._h = h

    @staticmethod
    def unique_id(lib):
        buf = (C.c_uint8 * A.COMM_ID_BYTES)()
        st = lib.ipcfp_comm_unique_id(buf)
        if st != A.OK:
            raise A.IpcfpError(st, lib.ipcfp_last_error().decode(errors="replace"), lib.ipcfp_last_error_index())
        return bytes(buf)

    @classmethod
    def from_torch_group(cls, lib, dist, device):
        """Rank 0 makes the id, torch.distributed (any backend) carries it."""
        world, rank = dist.get_world_size(), dist.get_rank()
        box = [cls.unique_id(lib) if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        return cls(lib, world, rank, device, box[0])

    def generate_event_proof(self, store_handle, tipset_handle, spec_c, bounds, flags=0):
        """→ POINTER(EventResultC) (caller frees with ipcfp_event_result_free). bounds: world+1 receipt indices."""
        b = np.ascontiguousarray(bounds, dtype=np.uint64)
        assert len(b) == self.world + 1
        out = C.POINTER(A.EventResultC)()
        st = self.L.ipcfp_generate_event_proof_sharded(self._h, store_handle, tipset_handle, C.byref(spec_c), b.ctypes.data, flags, C.byref(out))
        if st != A.OK:
            raise A.IpcfpError(st, self.L.ipcfp_last_error().decode(errors="replace"), self.L.ipcfp_last_error_index())
        return out

    def close(self):
        if self._h:
            self.L.ipcfp_comm_destroy(self._h)
            self._h = None
