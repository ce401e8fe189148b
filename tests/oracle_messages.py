"""The message-selected event call restated in Python (ipcfp_generate_message_log_proof, include/ipcfp.h): tests/oracle_logs.py's
generate_log_proof with its receipt loop restricted to the receipts of the given messages, plus the execution-index report, on the Python
oracle's decoders. A filter is oracle_logs' plain pair (emitters, positions); (set(), []) is every log extract_evm_log accepts.

read_set restates which blocks the call reads, the set its fetch planner must converge to.

The second restatement, tests/oracle_messages.cpp (oracle_logs.cpp's generator on oracle/oracle.cpp with the same restriction), is bound
below (CppOracle); it takes the C struct ipcfp_log_filter and 38-byte CIDs. It is compiled with g++ once per process into a temporary
directory: the checkout may be read-only."""
import ctypes as C
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A
from oracle import pyoracle as P
from tests import event_amts as E
from tests import oracle_logs as OL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NOT_EXECUTED = 2 ** 64 - 1


def execution_order(store, ts):
    """The tipset's execution order (reconstruct_execution_order): the message CIDs as bytes."""
    return [bytes(c) for c in P.collect_exec_list(store.get, [bytes(c) for c in ts.parent_txmeta_cids])]


def select(exec_order, n_receipts, message_cids):
    """→ (selected receipts ascending, exec_indices): receipt i is selected when i < n_exec, i < n_receipts and exec[i] is requested."""
    pos = {}
    for i, c in enumerate(exec_order):
        pos.setdefault(c, i)
    idx = [pos.get(bytes(c), NOT_EXECUTED) for c in message_cids]
    return sorted({i for i in idx if i != NOT_EXECUTED and i < n_receipts}), idx


def generate_message_log_proof(store, ts, message_cids, emitters=frozenset(), positions=()):
    """store: dict cid -> bytes. → dict(matching, proofs, witness, exec_indices) as oracle_logs.generate_log_proof returns them; its
    exceptions as that function raises them."""
    def hit(emitter, entries):
        return OL.log_matches(emitters, list(positions), emitter, P.extract_evm_log(entries))

    needed = set(bytes(c) for c in ts.parent_cids)
    needed.add(bytes(ts.child_cid))
    needed.add(bytes(ts.receipts_root))
    txmeta = [bytes(c) for c in ts.parent_txmeta_cids]
    needed.update(txmeta)
    for tx in txmeta:
        rec = P.Recorder(store)
        raw = rec.get(tx)
        if raw is None:
            raise P.MissingBlock(tx)
        bls, secp = P.cbor2.loads(raw)
        for root in (bls, secp):
            P.Amt(P._link(root), rec, 0).for_each(lambda i, v: None)
        needed |= rec.seen
    exec_order = [bytes(c) for c in P.collect_exec_list(store.get, txmeta)]
    selected, exec_indices = select(exec_order, int(ts.n_receipts), message_cids)

    rec_receipts = P.Recorder(store)
    r_amt = P.Amt(bytes(ts.receipts_root), rec_receipts, 0)
    matching = []
    for i in selected:
        if not ts.has_events_root[i]:
            continue
        # the AMT's structure as strictly as the engine and the C++ oracle read it (pyoracle's Amt accepts some refused shapes: a
        # bitmap of the wrong length, links and values in one node, trailing bytes)
        E.walk(store, bytes(ts.events_roots[i]))
        found = []
        P.Amt(bytes(ts.events_roots[i]), P.Recorder(store), 3).for_each(lambda j, se: found.append(j) if hit(*se) else None)
        if found:
            matching.append(i)
    proofs = []
    for i in matching:
        msg = exec_order[i]
        if r_amt.get(i) is None:
            continue
        rec_e = P.Recorder(store)

        def g(j, se, i=i, msg=msg):
            if hit(*se):
                topics, data = P.extract_evm_log(se[1])
                proofs.append((i, j, se[0], tuple(topics), data, msg))

        P.Amt(bytes(ts.events_roots[i]), rec_e, 3).for_each(g)
        needed |= rec_e.seen
    needed |= rec_receipts.seen
    witness = sorted(needed, key=P.cid_sort_key)
    for c in witness:
        if c not in store:
            raise P.MissingBlock(c)
    return dict(matching=matching, proofs=proofs, witness=witness, exec_indices=exec_indices)


def read_set(store, ts, message_cids, emitters=frozenset(), positions=()):
    """Every block the call reads on a complete, valid store: the base roots, the TxMeta blocks and message AMTs, the receipts root, the
    events AMTs of the selected receipts and the receipts-AMT paths of the matching ones."""
    r = generate_message_log_proof(store, ts, message_cids, emitters, positions)
    reads = set(r["witness"])
    exec_order = execution_order(store, ts)
    selected, _ = select(exec_order, int(ts.n_receipts), message_cids)
    for i in selected:
        if ts.has_events_root[i]:
            rec = P.Recorder(store)
            rec.get(bytes(ts.events_roots[i]))
            P.Amt(bytes(ts.events_roots[i]), rec, 3).for_each(lambda j, se: None)
            reads |= rec.seen
    return reads


def events_blocks(store, ts, receipts):
    """The blocks of the events AMTs of the given receipts (those with an events root)."""
    out = set()
    for i in receipts:
        if ts.has_events_root[i]:
            rec = P.Recorder(store)
            rec.get(bytes(ts.events_roots[i]))
            P.Amt(bytes(ts.events_roots[i]), rec, 3).for_each(lambda j, se: None)
            out |= rec.seen
    return out


@functools.lru_cache(maxsize=None)
def cpp_lib():
    gxx = shutil.which("g++")
    if not gxx:
        raise RuntimeError("g++ is needed to build the message oracle")
    out = os.path.join(tempfile.mkdtemp(prefix="oracle_messages_"), "liboracle_messages.so")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-o", out, os.path.join(ROOT, "tests", "oracle_messages.cpp")])
    L = C.CDLL(out)
    L.oracle_store_create.restype = C.c_void_p
    L.oracle_store_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.oracle_store_destroy.argtypes = [C.c_void_p]
    L.oracle_generate_message_log_proof.restype = C.c_int32
    L.oracle_generate_message_log_proof.argtypes = [C.c_void_p, C.POINTER(A.TipsetDesc), C.c_void_p, C.c_uint64, C.POINTER(A.LogFilterC),
                                                    C.c_uint32, C.c_void_p, C.POINTER(C.POINTER(A.EventResultC))]
    L.oracle_event_result_free.argtypes = [C.POINTER(A.EventResultC)]
    L.oracle_last_error.restype = C.c_char_p
    L.oracle_last_error_index.restype = C.c_uint64
    return L


class CppOracle:
    """tests/oracle_messages.cpp over a block set: a tipset-like object's flat arrays, or (cids, offsets, lengths, blob)."""

    def __init__(self, ts=None, arrays=None):
        arrays = arrays if arrays is not None else (ts.cids, ts.offsets, ts.lengths, ts.blob)
        self._keep = tuple(np.ascontiguousarray(a, dtype=t) for a, t in zip(arrays, (np.uint8, np.uint64, np.uint32, np.uint8)))
        c, o, n, b = self._keep
        self._h = cpp_lib().oracle_store_create(c.ctypes.data, o.ctypes.data, n.ctypes.data, b.ctypes.data, len(n))

    def generate(self, ts, message_cids, log_filter=None, flags=0):
        """→ ('ok', A.EventResultPy, exec_indices list) or ('err', status, index)."""
        cids = np.ascontiguousarray(np.frombuffer(b"".join(bytes(c) for c in message_cids), np.uint8) if len(message_cids) else np.zeros(0, np.uint8))
        idx = np.zeros(len(message_cids), np.uint64)
        d, keep = A.make_tipset_desc(ts)
        f, fkeep = log_filter.as_c() if log_filter is not None else (None, None)
        out = C.POINTER(A.EventResultC)()
        L = cpp_lib()
        st = L.oracle_generate_message_log_proof(self._h, C.byref(d), cids.ctypes.data if cids.size else None, len(message_cids),
                                                 C.byref(f) if f is not None else None, flags, idx.ctypes.data if idx.size else None, C.byref(out))
        if st != A.OK:
            return ("err", st, int(L.oracle_last_error_index()))
        try:
            return ("ok", A.event_result_from_c(out.contents), idx.tolist())
        finally:
            L.oracle_event_result_free(out)

    def __del__(self):
        try:
            cpp_lib().oracle_store_destroy(self._h)
        except Exception:
            pass
