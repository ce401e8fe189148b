"""The event generator restated in Python with a log filter as its predicate (the reference's generate_event_proof,
events/generator.rs:60-107, with `matches_log` and the actor filter replaced), on the Python oracle's decoders. A filter here is the
plain pair (emitters, positions): emitters a set of actor IDs (empty: any), positions a list of None (any value) or sets of 32-byte
values; an event matches when extract_evm_log accepts it, its emitter is in the set, it has at least len(positions) topics and
topic k is in positions[k] wherever that is not None. The Python restatement does not use the engine's LogFilter.

The second oracle, tests/oracle_logs.cpp (the C++ oracle's generator with the filter as its predicate), is bound below (CppOracle); it
takes the C struct ipcfp_log_filter. The library is compiled with g++ once per process into a temporary directory: the checkout may be
read-only."""
import ctypes as C
import functools
import os
import shutil
import subprocess
import tempfile

from ipc_filecoin_proofs_b200 import _abi as A
from oracle import pyoracle as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def log_matches(emitters, positions, emitter, log):
    if log is None:
        return False
    topics, _ = log
    if emitters and emitter not in emitters:
        return False
    if len(topics) < len(positions):
        return False
    return all(vals is None or bytes(topics[k]) in vals for k, vals in enumerate(positions))


def filter_of(f):
    """The (emitters, positions) pair of an api.LogFilter."""
    return set(f.emitters), [None if v is None else set(v) for v in f.topics]


def generate_log_proof(store, ts, emitters, positions):
    """store: dict cid -> bytes; ts: the synth.Tipset descriptor attributes. → dict(matching, proofs, witness) as
    pyoracle.generate_event_proof returns them; its exceptions as that function raises them."""
    def hit(emitter, entries):
        return log_matches(emitters, positions, emitter, P.extract_evm_log(entries))

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
    exec_order = P.collect_exec_list(store.get, txmeta)

    rec_receipts = P.Recorder(store)
    r_amt = P.Amt(bytes(ts.receipts_root), rec_receipts, 0)
    matching = []
    for i in range(int(ts.n_receipts)):
        if not ts.has_events_root[i]:
            continue
        found = []
        P.Amt(bytes(ts.events_roots[i]), P.Recorder(store), 3).for_each(lambda j, se: found.append(j) if hit(*se) else None)
        if found:
            matching.append(i)
    proofs = []
    for i in matching:
        if i >= len(exec_order):
            raise IndexError("Missing message at index %d" % i)
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
    return dict(matching=matching, proofs=proofs, witness=witness)


def candidate_logs(store, ts):
    """Every (emitter, topics) that extract_evm_log accepts in the tipset's events AMTs (for choosing filter values)."""
    out = []
    for i in range(int(ts.n_receipts)):
        if not ts.has_events_root[i]:
            continue
        try:
            amt = P.Amt(bytes(ts.events_roots[i]), P.Recorder(store), 3)

            def f(j, se):
                log = P.extract_evm_log(se[1])
                if log is not None:
                    out.append((se[0], [bytes(t) for t in log[0]]))

            amt.for_each(f)
        except Exception:
            continue
    return out


@functools.lru_cache(maxsize=None)
def cpp_lib():
    gxx = shutil.which("g++")
    if not gxx:
        raise RuntimeError("g++ is needed to build the log-filter oracle")
    out = os.path.join(tempfile.mkdtemp(prefix="oracle_logs_"), "liboracle_logs.so")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-o", out, os.path.join(ROOT, "tests", "oracle_logs.cpp")])
    L = C.CDLL(out)
    L.oracle_store_create.restype = C.c_void_p
    L.oracle_store_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.oracle_store_destroy.argtypes = [C.c_void_p]
    L.oracle_generate_log_proof.restype = C.c_int32
    L.oracle_generate_log_proof.argtypes = [C.c_void_p, C.POINTER(A.TipsetDesc), C.POINTER(A.LogFilterC), C.c_uint32, C.c_uint32,
                                            C.POINTER(C.POINTER(A.EventResultC))]
    L.oracle_event_result_free.argtypes = [C.POINTER(A.EventResultC)]
    L.oracle_last_error.restype = C.c_char_p
    L.oracle_last_error_index.restype = C.c_uint64
    return L


class CppOracle:
    """tests/oracle_logs.cpp over a tipset-like object's flat block arrays."""

    def __init__(self, ts):
        import numpy as np
        self._keep = tuple(np.ascontiguousarray(a, dtype=t) for a, t in
                           ((ts.cids, np.uint8), (ts.offsets, np.uint64), (ts.lengths, np.uint32), (ts.blob, np.uint8)))
        c, o, n, b = self._keep
        self._h = cpp_lib().oracle_store_create(c.ctypes.data, o.ctypes.data, n.ctypes.data, b.ctypes.data, len(n))

    def raw(self, ts, log_filter, flags=0, threads=1):
        """→ ('ok', pointer to the ipcfp_event_result, to be released with free()) or ('err', status, index)."""
        d, keep = A.make_tipset_desc(ts)
        f, fkeep = log_filter.as_c()
        out = C.POINTER(A.EventResultC)()
        st = cpp_lib().oracle_generate_log_proof(self._h, C.byref(d), C.byref(f), flags, threads, C.byref(out))
        if st != A.OK:
            return ("err", st, int(cpp_lib().oracle_last_error_index()))
        return ("ok", out)

    @staticmethod
    def free(out):
        cpp_lib().oracle_event_result_free(out)

    def generate(self, ts, log_filter, flags=0, threads=1):
        """→ ('ok', A.EventResultPy) or ('err', status, index)."""
        r = self.raw(ts, log_filter, flags, threads)
        if r[0] != "ok":
            return r
        try:
            return ("ok", A.event_result_from_c(r[1].contents))
        finally:
            self.free(r[1])

    def __del__(self):
        try:
            cpp_lib().oracle_store_destroy(self._h)
        except Exception:
            pass
