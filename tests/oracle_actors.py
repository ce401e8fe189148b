"""ctypes binding of tests/oracle_actors.cpp, the C++ oracle of ipcfp_generate_actor_proofs_resident (a helper module, not a fixture file).
The library is compiled with g++ once per process into a temporary directory: the checkout may be read-only."""
import ctypes as C
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A
from oracle.pyoracle import cid_sort_key
from tests import actor_trees as AT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=None)
def lib():
    gxx = shutil.which("g++")
    if not gxx:
        raise RuntimeError("g++ is needed to build the actor-proof oracle")
    out = os.path.join(tempfile.mkdtemp(prefix="oracle_actors_"), "liboracle_actors.so")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-o", out, os.path.join(ROOT, "tests", "oracle_actors.cpp")])
    L = C.CDLL(out)
    L.oracle_store_create.restype = C.c_void_p
    L.oracle_store_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.oracle_store_destroy.argtypes = [C.c_void_p]
    L.oracle_actor_proofs.restype = C.c_int32
    L.oracle_actor_proofs.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.POINTER(A.AddressC), C.c_uint64, C.c_void_p, C.c_uint64, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p, C.c_uint64, C.c_void_p,
                                      C.POINTER(C.c_uint64)]
    return L


class Oracle:
    """The oracle over one block set ({cid: bytes}); prove() returns what tests/actor_trees.prove returns (proofs as dicts, per-proof read
    sets, their union) or raises actor_trees.Failure."""

    def __init__(self, blocks):
        cids = b"".join(blocks)
        lens = np.array([len(b) for b in blocks.values()], np.uint32)
        offs = np.concatenate([[0], np.cumsum(lens, dtype=np.uint64)[:-1]]).astype(np.uint64) if len(lens) else np.zeros(0, np.uint64)
        self._keep = (cids, offs, lens, b"".join(blocks.values()) + bytes(16))
        self._h = lib().oracle_store_create(cids, offs.ctypes.data, lens.ctypes.data, self._keep[3], len(lens))

    def prove(self, child, state_root, addrs, evm=(), with_code=False):
        addrs = [bytes(a) for a in addrs]
        n = len(addrs)
        arr = A.make_addresses(addrs)
        ev = b"".join(bytes(c) for c in evm)
        out = (A.ActorProofC * max(n, 1))()
        off = np.zeros(n + 1, np.uint64)
        cs, fail = C.c_uint64(), C.c_uint64()
        code_cap, read_cap = 1 << 16, 64 * max(n, 1)
        while True:
            code, reads = np.zeros(code_cap, np.uint8), np.zeros(38 * read_cap, np.uint8)
            rc = lib().oracle_actor_proofs(self._h, bytes(child), bytes(state_root), arr, n, ev or None, len(evm), int(with_code), C.addressof(out),
                                           code.ctypes.data, code_cap, C.byref(cs), reads.ctypes.data, read_cap, off.ctypes.data, C.byref(fail))
            if rc != A.OK:
                raise AT.Failure(rc, fail.value)
            if cs.value <= code_cap and int(off[n]) <= read_cap:
                break
            code_cap, read_cap = max(code_cap, cs.value), max(read_cap, int(off[n]))
        blob = code[:cs.value].tobytes()
        proofs = [vars(A.actor_proof_from_c(out[i], blob)) for i in range(n)]
        lists = [[reads[38 * k:38 * k + 38].tobytes() for k in range(int(off[i]), int(off[i + 1]))] for i in range(n)]
        union = sorted({c for lst in lists for c in lst}, key=cid_sort_key)
        return proofs, lists, union

    def close(self):
        if self._h:
            lib().oracle_store_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()
