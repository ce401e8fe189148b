"""ctypes binding of tests/oracle_resolve.cpp, the C++ oracle of ipcfp_resolve_addresses (a helper module, not a fixture file). The library
is compiled with g++ once per process into a temporary directory: the checkout may be read-only."""
import ctypes as C
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=None)
def lib():
    gxx = shutil.which("g++")
    if not gxx:
        raise RuntimeError("g++ is needed to build the resolution oracle")
    out = os.path.join(tempfile.mkdtemp(prefix="oracle_resolve_"), "liboracle_resolve.so")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-o", out, os.path.join(ROOT, "tests", "oracle_resolve.cpp")])
    L = C.CDLL(out)
    L.oracle_store_create.restype = C.c_void_p
    L.oracle_store_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.oracle_store_destroy.argtypes = [C.c_void_p]
    L.oracle_resolve_addresses.restype = C.c_int32
    L.oracle_resolve_addresses.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(A.AddressC), C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32),
                                           C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    return L


class Oracle:
    """The oracle over one block set ({cid: bytes}); resolve() returns what tests/address_trees.resolve returns:
    (ids, status, init_status, missing CIDs, read set), both CID lists in `Cid` order."""

    def __init__(self, blocks):
        cids = b"".join(blocks)
        lens = np.array([len(b) for b in blocks.values()], np.uint32)
        offs = np.concatenate([[0], np.cumsum(lens, dtype=np.uint64)[:-1]]).astype(np.uint64) if len(lens) else np.zeros(0, np.uint64)
        self._keep = (cids, offs, lens, b"".join(blocks.values()) + bytes(16))
        self._h = lib().oracle_store_create(cids, offs.ctypes.data, lens.ctypes.data, self._keep[3], len(lens))

    def resolve(self, state_root, addresses):
        n = len(addresses)
        arr = A.make_addresses(addresses)
        ids, st = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.int32)
        init, nm, nr = C.c_int32(), C.c_uint64(), C.c_uint64()
        cap = 64
        while True:
            miss, read = np.zeros(38 * cap, np.uint8), np.zeros(38 * cap, np.uint8)
            rc = lib().oracle_resolve_addresses(self._h, bytes(state_root), arr, n, ids.ctypes.data, st.ctypes.data, C.byref(init),
                                                miss.ctypes.data, cap, C.byref(nm), read.ctypes.data, cap, C.byref(nr))
            assert rc == A.OK
            if max(nm.value, nr.value) <= cap:
                break
            cap = max(nm.value, nr.value)
        split = lambda b, k: [bytes(b[38 * i:38 * i + 38]) for i in range(k)]   # noqa: E731
        return ids[:n].tolist(), st[:n].tolist(), init.value, split(miss, nm.value), split(read, nr.value)

    def close(self):
        if self._h:
            lib().oracle_store_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()
