"""ctypes front-end of the synthetic tipset builder (synth/synth.cpp).

Test / bench infrastructure: generates the flat block set + tipset descriptor the
engine ingests. CPU only; not part of the product path.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libipcfp_synth.so")


class SynthParams(C.Structure):
    _fields_ = [
        ("seed", C.c_uint64),
        ("n_receipts", C.c_uint64),
        ("events_per_receipt", C.c_uint32),
        ("match_ppm", C.c_uint32),
        ("has_actor_filter", C.c_uint32),
        ("target_actor", C.c_uint64),
        ("bw3_permille", C.c_uint32),
        ("case_a_permille", C.c_uint32),
        ("malformed_permille", C.c_uint32),
        ("null_root_permille", C.c_uint32),
        ("n_parents", C.c_uint32),
        ("dup_msgs", C.c_uint32),
        ("with_state_tree", C.c_uint32),
        ("n_actors", C.c_uint32),
        ("hamt_entries", C.c_uint64),
        ("shard_lo", C.c_uint64),
        ("shard_hi", C.c_uint64),
        ("threads", C.c_uint32),
        ("same_topic1", C.c_uint32),
        ("event_shapes", C.c_uint32),
    ]


def build_lib(force=False):
    src = [os.path.join(_HERE, f) for f in ("synth.cpp", "synth.h", "cpu_crypto.h")]
    if not force and os.path.exists(_LIB_PATH) and all(
            os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in src if os.path.exists(s)):
        return _LIB_PATH
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", _LIB_PATH,
                           os.path.join(_HERE, "synth.cpp")])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build_lib()
        L = C.CDLL(_LIB_PATH)
        L.synth_build.restype = C.c_void_p
        L.synth_build.argtypes = [C.POINTER(SynthParams)]
        L.synth_free.argtypes = [C.c_void_p]
        for name, res in [
            ("synth_n_blocks", C.c_uint64), ("synth_cids", C.c_void_p), ("synth_offsets", C.c_void_p),
            ("synth_lengths", C.c_void_p), ("synth_blob", C.c_void_p), ("synth_blob_size", C.c_uint64),
            ("synth_parent_epoch", C.c_int64), ("synth_child_epoch", C.c_int64), ("synth_n_parents", C.c_uint32),
            ("synth_parent_cids", C.c_void_p), ("synth_parent_txmeta_cids", C.c_void_p), ("synth_child_cid", C.c_void_p),
            ("synth_receipts_root", C.c_void_p), ("synth_parent_state_root", C.c_void_p), ("synth_n_receipts", C.c_uint64),
            ("synth_events_roots", C.c_void_p), ("synth_has_events_root", C.c_void_p), ("synth_event_signature", C.c_char_p),
            ("synth_topic1", C.c_char_p), ("synth_target_actor", C.c_uint64), ("synth_n_selected", C.c_uint64),
            ("synth_selected", C.c_void_p), ("synth_storage_root", C.c_void_p),
        ]:
            f = getattr(L, name)
            f.restype = res
            f.argtypes = [C.c_void_p]
        L.synth_storage_entry.restype = C.c_uint32
        L.synth_storage_entry.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        L.synth_storage_absent_key.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        for name in ("synth_blake2b256", "synth_keccak256", "synth_sha256"):
            getattr(L, name).argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
        _lib = L
    return _lib


def default_params(**kw):
    p = SynthParams()
    lib().synth_default_params(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def _np(ptr, n, dtype):
    if n == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    buf = (C.c_uint8 * (n * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype)


class Tipset:
    """A built synthetic tipset. numpy views alias the C++ object's memory (kept alive by self)."""

    def __init__(self, params=None, **kw):
        self.params = params if params is not None else default_params(**kw)
        L = lib()
        self._h = L.synth_build(C.byref(self.params))
        h = self._h
        n = L.synth_n_blocks(h)
        self.n_blocks = n
        self.cids = _np(L.synth_cids(h), n * 38, np.uint8).reshape(n, 38)
        self.offsets = _np(L.synth_offsets(h), n, np.uint64)
        self.lengths = _np(L.synth_lengths(h), n, np.uint32)
        self.blob = _np(L.synth_blob(h), L.synth_blob_size(h), np.uint8)
        self.parent_epoch = L.synth_parent_epoch(h)
        self.child_epoch = L.synth_child_epoch(h)
        P = L.synth_n_parents(h)
        self.n_parents = P
        self.parent_cids = _np(L.synth_parent_cids(h), P * 38, np.uint8).reshape(P, 38)
        self.parent_txmeta_cids = _np(L.synth_parent_txmeta_cids(h), P * 38, np.uint8).reshape(P, 38)
        self.child_cid = _np(L.synth_child_cid(h), 38, np.uint8)
        self.receipts_root = _np(L.synth_receipts_root(h), 38, np.uint8)
        self.parent_state_root = _np(L.synth_parent_state_root(h), 38, np.uint8)
        N = L.synth_n_receipts(h)
        self.n_receipts = N
        self.events_roots = _np(L.synth_events_roots(h), N * 38, np.uint8).reshape(N, 38)
        self.has_events_root = _np(L.synth_has_events_root(h), N, np.uint8)
        self.event_signature = L.synth_event_signature(h).decode()
        self.topic1 = L.synth_topic1(h).decode()
        self.target_actor = L.synth_target_actor(h)
        self.actor_filter = self.target_actor if self.params.has_actor_filter else None
        self.selected = _np(L.synth_selected(h), L.synth_n_selected(h), np.uint64)
        self.storage_root = _np(L.synth_storage_root(h), 38, np.uint8)

    def block(self, i):
        o = int(self.offsets[i])
        return bytes(self.blob[o:o + int(self.lengths[i])])

    def as_dict(self):
        return {bytes(self.cids[i]): self.block(i) for i in range(self.n_blocks)}

    def storage_entry(self, k):
        key = (C.c_uint8 * 32)()
        val = (C.c_uint8 * 32)()
        n = lib().synth_storage_entry(self._h, k, key, val)
        return bytes(key), bytes(val)[:n]

    def storage_absent_key(self, k):
        key = (C.c_uint8 * 32)()
        lib().synth_storage_absent_key(self._h, k, key)
        return bytes(key)

    def close(self):
        if self._h:
            for a in ("cids", "offsets", "lengths", "blob", "parent_cids", "parent_txmeta_cids", "child_cid", "receipts_root",
                      "parent_state_root", "events_roots", "has_events_root", "selected", "storage_root"):
                setattr(self, a, None)
            lib().synth_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _hash(fn, data):
    out = (C.c_uint8 * 32)()
    getattr(lib(), fn)(bytes(data), len(data), out)
    return bytes(out)


def blake2b256(data):
    return _hash("synth_blake2b256", data)


def keccak256(data):
    return _hash("synth_keccak256", data)


def sha256(data):
    return _hash("synth_sha256", data)


# the BASELINE.json configs (SURVEY.md §8d). seed = 0x1FC0FFEE ^ config_id.
def config_params(config_id, **over):
    base = dict(seed=0x1FC0FFEE ^ config_id)
    if config_id == 1:
        base.update(n_receipts=64, events_per_receipt=8, match_ppm=125000, has_actor_filter=0, same_topic1=1,
                    bw3_permille=0, dup_msgs=2)
    elif config_id == 2:
        base.update(n_receipts=10_000, events_per_receipt=8, match_ppm=10_000, has_actor_filter=1, bw3_permille=100)
    elif config_id == 3:
        base.update(n_receipts=64, events_per_receipt=8, match_ppm=20_000, with_state_tree=1, hamt_entries=1_000_000,
                    n_actors=2048)
    elif config_id == 4:
        base.update(n_receipts=1_000_000, events_per_receipt=8, match_ppm=1_000, has_actor_filter=1, bw3_permille=100,
                    dup_msgs=16)
    elif config_id == 5:
        base.update(n_receipts=8_000_000, events_per_receipt=8, match_ppm=1_000, has_actor_filter=1, bw3_permille=100,
                    dup_msgs=16)
    else:
        raise ValueError(config_id)
    base.update(over)
    return default_params(**base)
