"""Host-side binding of the engine's C ABI (include/ipcfp.h) for tests, bench and Python callers.

Mirrors the reference's API surface for the hot path — `EventProofSpec`, `StorageProofSpec`,
`generate_event_proof`, `read_storage_slot`, `generate_storage_proof`, `generate_proof_bundle`
(reference src/proofs/generator.rs:12-95, events/generator.rs:60-68, storage/decode.rs:36-40,
storage/generator.rs:29-35) — over the CUDA library. There is NO CPU implementation behind these
calls: if libipcfp.so is missing or no CUDA device is present they raise.
"""
import ctypes as C
import os
import subprocess
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _abi as A

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
LIB_PATH = os.path.join(_HERE, "libipcfp.so")


def build_lib(force=False, jobs=8):
    """Compile the CUDA library in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    if force or not os.path.exists(LIB_PATH):
        subprocess.check_call(["make", "-C", _ROOT, "-j%d" % jobs, os.path.relpath(LIB_PATH, _ROOT)])
    else:
        subprocess.check_call(["make", "-C", _ROOT, "-j%d" % jobs, "-s", os.path.relpath(LIB_PATH, _ROOT)])
    return LIB_PATH


_lib = None

_vp, _u64, _u32, _int, _st = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_int32
_P = C.POINTER


def _PP(t):
    return C.POINTER(C.POINTER(t))


_HASH_BATCH = [_vp, _u64, _vp, _vp, _u64, _int, _vp]
_TO_JSON = [_vp, _P(A.TipsetDesc), _P(_vp), _P(_u64)]

# Every function of include/ipcfp.h, in its order: name -> (restype, argtypes). None leaves ctypes' default: the int result of a void
# function, the unchecked argument list of a (void) one. tests/test_abi_bindings.py checks the table against the header.
SIGNATURES = {
    "ipcfp_last_error": (C.c_char_p, None),
    "ipcfp_last_error_index": (_u64, None),
    "ipcfp_version": (C.c_char_p, None),
    "ipcfp_kernel_launch_count": (_u64, None),
    "ipcfp_host_alloc": (_st, [C.c_size_t, _P(_vp)]),
    "ipcfp_host_free": (None, [_vp]),
    "ipcfp_store_create": (_st, [_vp, _vp, _vp, _vp, _u64, _u64, _int, _u32, _P(_vp)]),
    "ipcfp_store_destroy": (None, [_vp]),
    "ipcfp_store_n_blocks": (_u64, [_vp]),
    "ipcfp_store_get": (_st, [_vp, _vp, _vp, _u32, _P(_u32), _P(_int)]),
    "ipcfp_store_has": (_st, [_vp, _vp, _P(_int)]),
    "ipcfp_store_first_bad_block": (_u64, [_vp]),
    "ipcfp_blake2b256_batch": (_st, _HASH_BATCH),
    "ipcfp_keccak256_batch": (_st, _HASH_BATCH),
    "ipcfp_sha256_batch": (_st, _HASH_BATCH),
    "ipcfp_compute_mapping_slots": (_st, [_vp, _vp, _u64, _int, _vp]),
    "ipcfp_generate_event_proof": (_st, [_vp, _P(A.TipsetDesc), _P(A.EventSpec), _u32, _PP(A.EventResultC)]),
    "ipcfp_event_result_free": (None, [_P(A.EventResultC)]),
    "ipcfp_tipset_upload": (_st, [_vp, _P(A.TipsetDesc), _P(_vp)]),
    "ipcfp_tipset_free": (None, [_vp]),
    "ipcfp_generate_event_proof_resident": (_st, [_vp, _vp, _P(A.EventSpec), _u32, _PP(A.EventResultC)]),
    "ipcfp_generate_event_proof_shard_resident": (_st, [_vp, _vp, _P(A.EventSpec), _u64, _u64, _u32, _u32, _u32, _PP(A.EventResultC)]),
    "ipcfp_generate_log_proof_resident": (_st, [_vp, _vp, _P(A.LogFilterC), _u32, _PP(A.EventResultC)]),
    "ipcfp_generate_log_proof": (_st, [_vp, _P(A.TipsetDesc), _P(A.LogFilterC), _u32, _PP(A.EventResultC)]),
    "ipcfp_generate_message_log_proof_resident": (_st, [_vp, _vp, _vp, _u64, _P(A.LogFilterC), _u32, _vp, _PP(A.EventResultC)]),
    "ipcfp_generate_message_log_proof": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _P(A.LogFilterC), _u32, _vp, _PP(A.EventResultC)]),
    "ipcfp_store_stream": (_vp, [_vp]),
    "ipcfp_tipset_desc_from_json": (_st, [C.c_char_p, _u64, C.c_char_p, _u64, C.c_char_p, _u64, _PP(A.ParsedTipsetC)]),
    "ipcfp_parsed_tipset_free": (None, [_P(A.ParsedTipsetC)]),
    "ipcfp_tipset_upload_json": (_st, [_vp, C.c_char_p, _u64, C.c_char_p, _u64, C.c_char_p, _u64, _P(_vp)]),
    "ipcfp_tipset_describe": (_st, [_vp, _int, _P(A.TipsetInfoC)]),
    "ipcfp_blocks_from_rpc_json": (_st, [_vp, _u64, _P(C.c_char_p), _P(_u64), _u64, _PP(A.ParsedBlocksC)]),
    "ipcfp_parsed_blocks_free": (None, [_P(A.ParsedBlocksC)]),
    "ipcfp_store_create_rpc_json": (_st, [_vp, _u64, _P(C.c_char_p), _P(_u64), _u64, _int, _u32, _P(_vp), _P(A.StoreJsonInfoC)]),
    "ipcfp_blocks_from_car": (_st, [_vp, _u64, _PP(A.ParsedBlocksC)]),
    "ipcfp_store_create_car": (_st, [_vp, _u64, _int, _u32, _P(_vp), _P(A.StoreJsonInfoC)]),
    "ipcfp_read_storage_slots": (_st, [_vp, _vp, _vp, _u64, _PP(A.SlotResultC)]),
    "ipcfp_slot_result_free": (None, [_P(A.SlotResultC)]),
    "ipcfp_generate_storage_proofs": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _PP(A.StorageResultC)]),
    "ipcfp_storage_result_free": (None, [_P(A.StorageResultC)]),
    "ipcfp_generate_storage_path_proofs_resident": (_st, [_vp, _vp, _P(A.StoragePathC), _u64, _u32, _PP(A.PathResultC)]),
    "ipcfp_verify_storage_paths": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _P(A.StoragePathC), _u64, _PP(A.PathResultC)]),
    "ipcfp_path_result_free": (None, [_P(A.PathResultC)]),
    "ipcfp_generate_proof_bundle": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _vp, _u64, _PP(A.BundleC)]),
    "ipcfp_generate_proof_bundle_resident": (_st, [_vp, _vp, _vp, _u64, _vp, _u64, _u32, _PP(A.BundleC)]),
    "ipcfp_generate_log_bundle_resident": (_st, [_vp, _vp, _vp, _u64, _P(A.LogFilterC), _u64, _u32, _PP(A.BundleC)]),
    "ipcfp_generate_log_bundle": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _P(A.LogFilterC), _u64, _u32, _PP(A.BundleC)]),
    "ipcfp_bundle_free": (None, [_P(A.BundleC)]),
    "ipcfp_plan_fetch_resident": (_st, [_vp, _vp, _vp, _u64, _vp, _u64, _u32, _PP(A.FetchPlanC)]),
    "ipcfp_plan_fetch": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _vp, _u64, _u32, _PP(A.FetchPlanC)]),
    "ipcfp_fetch_plan_free": (None, [_P(A.FetchPlanC)]),
    "ipcfp_plan_fetch_log_resident": (_st, [_vp, _vp, _P(A.LogFilterC), _u32, _PP(A.FetchPlanC)]),
    "ipcfp_plan_fetch_message_log_resident": (_st, [_vp, _vp, _vp, _u64, _P(A.LogFilterC), _u32, _PP(A.FetchPlanC)]),
    "ipcfp_plan_fetch_log_bundle_resident": (_st, [_vp, _vp, _vp, _u64, _P(A.LogFilterC), _u64, _u32, _PP(A.FetchPlanC)]),
    "ipcfp_plan_fetch_storage_paths_resident": (_st, [_vp, _vp, _P(A.StoragePathC), _u64, _u32, _PP(A.FetchPlanC)]),
    "ipcfp_fetch_plan_to_rpc_json": (_st, [_P(A.FetchPlanC), _u64, _P(_vp), _P(_u64)]),
    "ipcfp_resolve_addresses": (_st, [_vp, _vp, _P(A.AddressC), _u64, _PP(A.ResolveResultC)]),
    "ipcfp_resolve_result_free": (None, [_P(A.ResolveResultC)]),
    "ipcfp_address_parse": (_st, [C.c_char_p, _u64, _P(A.AddressC)]),
    "ipcfp_address_from_eth": (_st, [_vp, _P(A.AddressC)]),
    "ipcfp_generate_actor_proofs_resident": (_st, [_vp, _vp, _P(A.AddressC), _u64, _vp, _u64, _u32, _PP(A.ActorResultC)]),
    "ipcfp_generate_actor_proofs": (_st, [_vp, _P(A.TipsetDesc), _P(A.AddressC), _u64, _vp, _u64, _u32, _PP(A.ActorResultC)]),
    "ipcfp_actor_result_free": (None, [_P(A.ActorResultC)]),
    "ipcfp_plan_fetch_actor_proofs_resident": (_st, [_vp, _vp, _P(A.AddressC), _u64, _vp, _u64, _u32, _PP(A.FetchPlanC)]),
    "ipcfp_verify_actor_proofs": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _vp, _u64, _u32, _vp]),
    "ipcfp_generate_message_proofs_resident": (_st, [_vp, _vp, _vp, _u64, _u32, _PP(A.MessageResultC)]),
    "ipcfp_generate_message_proofs": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _u32, _PP(A.MessageResultC)]),
    "ipcfp_message_result_free": (None, [_P(A.MessageResultC)]),
    "ipcfp_plan_fetch_message_proofs_resident": (_st, [_vp, _vp, _vp, _u64, _u32, _PP(A.FetchPlanC)]),
    "ipcfp_verify_message_proofs": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _vp, _u64, _u32, _vp]),
    "ipcfp_bundle_to_json": (_st, _TO_JSON),
    "ipcfp_event_result_to_json": (_st, _TO_JSON),
    "ipcfp_json_free": (None, [_vp]),
    "ipcfp_bundle_from_json": (_st, [C.c_char_p, _u64, _PP(A.ParsedBundleC)]),
    "ipcfp_parsed_bundle_free": (None, [_P(A.ParsedBundleC)]),
    "ipcfp_verify_event_proofs": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _vp, _u64, _vp, _vp]),
    "ipcfp_verify_storage_proofs": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _vp]),
    "ipcfp_verify_event_proofs_log": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _vp, _u64, _P(A.LogFilterC), _vp]),
    "ipcfp_verify_event_proofs_any": (_st, [_vp, _P(A.TipsetDesc), _vp, _u64, _vp, _u64, _P(A.LogFilterC), _u64, _vp]),
    "ipcfp_verify_bundle_json": (_st, [C.c_char_p, _u64, _int, A.TrustedParentFn, A.TrustedChildFn, _vp, _vp, _PP(A.BundleVerdictC)]),
    "ipcfp_verify_bundle_json_any": (_st, [C.c_char_p, _u64, _int, A.TrustedParentFn, A.TrustedChildFn, _vp, _P(A.LogFilterC), _u64,
                                          _PP(A.BundleVerdictC)]),
    "ipcfp_bundle_verdict_free": (None, [_P(A.BundleVerdictC)]),
    "ipcfp_comm_unique_id": (_st, [_vp]),
    "ipcfp_comm_init": (_st, [_vp, _u32, _u32, _int, _P(_vp)]),
    "ipcfp_comm_destroy": (None, [_vp]),
    "ipcfp_generate_event_proof_sharded": (_st, [_vp, _vp, _vp, _P(A.EventSpec), _vp, _u32, _PP(A.EventResultC)]),
    "ipcfp_generate_event_proof_shard": (_st, [_vp, _P(A.TipsetDesc), _P(A.EventSpec), _u64, _u64, _u32, _u32, _u32, _PP(A.EventResultC)]),
}
EXPORTS = list(SIGNATURES)


def lib():
    """Loads libipcfp.so. Fails loudly when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `make` (or __graft_entry__.build()). There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            f = getattr(L, name)
            if restype is not None:
                f.restype = restype
            if argtypes is not None:
                f.argtypes = argtypes
        _lib = L
    return _lib


def _u8(x):
    if isinstance(x, (bytes, bytearray, memoryview)):
        return np.frombuffer(bytes(x), dtype=np.uint8).copy()
    return np.ascontiguousarray(x, dtype=np.uint8)


def _check(st):
    if st != A.OK:
        L = lib()
        raise A.IpcfpError(st, L.ipcfp_last_error().decode(errors="replace"), L.ipcfp_last_error_index())


def _result(fn, out_type, convert, free, *args):
    """Calls lib().<fn>(*args, &out) for an out_type object → convert(out.contents), then releases the object with lib().<free>."""
    L = lib()
    out = C.POINTER(out_type)()
    _check(getattr(L, fn)(*args, C.byref(out)))
    try:
        return convert(out.contents)
    finally:
        getattr(L, free)(out)


# (out_type, convert, free) of _result for the result kinds several calls return
_EVENT_RESULT = (A.EventResultC, A.event_result_from_c, "ipcfp_event_result_free")
_BUNDLE = (A.BundleC, A.bundle_from_c, "ipcfp_bundle_free")
_FETCH_PLAN = (A.FetchPlanC, A.fetch_plan_from_c, "ipcfp_fetch_plan_free")
_PATH_RESULT = (A.PathResultC, A.path_result_from_c, "ipcfp_path_result_free")


def kernel_launch_count():
    return int(lib().ipcfp_kernel_launch_count())


@dataclass
class EventProofSpec:  # reference src/proofs/generator.rs:18-22
    event_signature: str
    topic_1: str
    actor_id_filter: Optional[int] = None

    def as_c(self):
        return A.make_event_spec(self.event_signature, self.topic_1, self.actor_id_filter)


def _topic32(v):
    if isinstance(v, str):
        v = bytes.fromhex(v[2:] if v[:2] in ("0x", "0X") else v)
    v = bytes(v)
    if len(v) != 32:
        raise ValueError(f"a topic value is 32 bytes, got {len(v)}")
    return v


class LogFilter:
    """An eth_getLogs-style log filter (ipcfp_log_filter): `emitters` — None / [] for any emitter, else actor IDs (resolve Ethereum
    addresses first with resolve_eth_address_to_actor_id); `topics` — one entry per position, each None (any value), a 32-byte value
    (bytes or hex) or a list of them (an empty list is a wildcard, as None). An event matches when extract_evm_log accepts it, its emitter is in the set, it has at least
    len(topics) topics and topic k is in topics[k] wherever that is not None. Trailing None entries count towards the topic minimum,
    as in go-ethereum's filterLogs."""

    def __init__(self, emitters=None, topics=()):
        topics = list(topics)
        if len(topics) > 4:
            raise ValueError("a log filter has at most 4 topic positions")
        self.emitters = [int(e) for e in (emitters or [])]
        self.topics = []
        for t in topics:
            if t is None or (isinstance(t, (list, tuple)) and not t):   # None or an empty list: any value (go-ethereum's rule)
                self.topics.append(None)
            elif isinstance(t, (bytes, bytearray, str)):
                self.topics.append([_topic32(t)])
            else:
                self.topics.append([_topic32(v) for v in t])

    @classmethod
    def from_spec(cls, spec, device=0):
        """The filter an EventProofSpec stands for: topic 0 = keccak256(signature) (hashed on `device`), topic 1 =
        ascii_to_bytes32(topic_1), at least two topics, the actor (if any) as the only emitter."""
        t1 = spec.topic_1.encode()[:32]
        t0 = bytes(keccak256_batch([spec.event_signature.encode()], device)[0])
        return cls(None if spec.actor_id_filter is None else [spec.actor_id_filter], [t0, t1 + bytes(32 - len(t1))])

    def as_c(self):
        """(ipcfp_log_filter, keepalive)"""
        f = A.LogFilterC()
        keep = []
        em = np.ascontiguousarray(self.emitters, dtype=np.uint64)
        keep.append(em)
        f.n_emitters = len(em)
        f.emitters = em.ctypes.data if em.size else None
        f.n_positions = len(self.topics)
        for k, vals in enumerate(self.topics):
            if vals:
                a = np.frombuffer(b"".join(vals), dtype=np.uint8).copy()
                keep.append(a)
                f.n_values[k] = len(vals)
                f.values[k] = a.ctypes.data
        return f, keep

    def matches(self, emitter, topics):
        """The predicate on one extracted log (emitter, list of 32-byte topics)."""
        if self.emitters and emitter not in self.emitters:
            return False
        if len(topics) < len(self.topics):
            return False
        return all(vals is None or bytes(topics[k]) in vals for k, vals in enumerate(self.topics))


def _log_filters_c(log_filters):
    """(ipcfp_log_filter array, count, keepalive) of a sequence of LogFilters"""
    cs, keep = [], []
    for f in log_filters:
        c, k = f.as_c()
        cs.append(c)
        keep.append(k)
    return (A.LogFilterC * max(len(cs), 1))(*cs), len(cs), keep


@dataclass
class StorageProofSpec:  # reference src/proofs/generator.rs:12-15
    actor_id: int
    slot: bytes


def _u256(x):
    """an int (mod 2^256, two's complement for negatives) or 32 bytes → 32 big-endian bytes"""
    if isinstance(x, int):
        return (x % (1 << 256)).to_bytes(32, "big")
    x = bytes(x)
    if len(x) != 32:
        raise ValueError(f"a slot is 32 bytes, got {len(x)}")
    return x


def encode_key(key, key_type=None):
    """A mapping key as Solidity hashes it (keccak256(h(k) ‖ p)): value types as their 32-byte padded form — "address" (20 bytes or hex,
    left-padded), "uint…" / "int…" (two's complement), "bool", "bytes1".."bytes32" (right-padded) — and "bytes" / "string" as their raw
    bytes. key_type None takes 32 bytes as they are."""
    if key_type is None:
        k = bytes(key)
        if len(k) != 32:
            raise ValueError("a key without a type must be 32 bytes")
        return k
    if key_type == "address":
        b = bytes.fromhex(key[2:] if key[:2] in ("0x", "0X") else key) if isinstance(key, str) else bytes(key)
        if len(b) != 20:
            raise ValueError("an address is 20 bytes")
        return bytes(12) + b
    if key_type.startswith("uint") or key_type.startswith("int"):
        return _u256(int(key))
    if key_type == "bool":
        return _u256(1 if key else 0)
    if key_type in ("bytes", "string"):
        return key.encode() if isinstance(key, str) else bytes(key)
    if key_type.startswith("bytes"):
        n = int(key_type[5:])
        b = key.encode() if isinstance(key, str) else bytes(key)
        if not 1 <= n <= 32 or len(b) > n:
            raise ValueError(f"{key_type} key of {len(b)} bytes")
        return b + bytes(32 - len(b))
    raise ValueError(f"unknown key type {key_type!r}")


class StoragePath:
    """A Solidity value by its access path (include/ipcfp.h, "Storage paths"): the state variable's declared slot, then steps —
    .mapping(key, key_type), .array(index) (dynamic: its length word is proven too), .static(index), .field(offset) — and what to read:
    .words(n) (a value type, a struct, a static array; the default is one word) or .bytes() (a bytes / string). Each step returns a new
    path, so a common prefix can be shared:
        StoragePath(actor, 0).mapping(subnet_id, "bytes32").field(3)     # subnets[id].<member at slot offset 3>
    Arrays: elem_slots = slots per element; elem_bytes = the size of a packed value-type element (uint8: 1, address: 20), 0 otherwise."""

    def __init__(self, actor_id, base_slot, steps=(), kind=A.PATH_WORDS, n_words=1):
        self.actor_id = int(actor_id)
        self.base_slot = _u256(base_slot)
        self.steps = tuple(steps)
        self.kind = kind
        self.n_words = n_words

    def _with(self, step=None, **kw):
        d = dict(steps=self.steps + ((step,) if step else ()), kind=self.kind, n_words=self.n_words)
        d.update(kw)
        return StoragePath(self.actor_id, self.base_slot, **d)

    def mapping(self, key, key_type=None):
        return self._with((A.PATH_MAPPING, encode_key(key, key_type), 0, 0, 0))

    def array(self, index, elem_slots=1, elem_bytes=0):
        return self._with((A.PATH_ARRAY, b"", int(index), elem_slots, elem_bytes))

    def static(self, index, elem_slots=1, elem_bytes=0):
        return self._with((A.PATH_STATIC, b"", int(index), elem_slots, elem_bytes))

    def field(self, offset):
        return self._with((A.PATH_FIELD, b"", int(offset), 0, 0))

    def words(self, n=1):
        return self._with(kind=A.PATH_WORDS, n_words=n)

    def bytes(self):
        return self._with(kind=A.PATH_BYTES, n_words=0)

    @staticmethod
    def decode(word, value_type="uint256", byte_offset=0):
        """A packed member of a 32-byte word: its bytes sit byte_offset bytes above the word's low-order end (Solidity packs the first
        member lowest). value_type: "uintN" / "intN" (int), "bool", "address" (20 bytes), "bytesN" (bytes)."""
        word = bytes(word)
        if value_type == "address":
            size = 20
        elif value_type == "bool":
            size = 1
        elif value_type.startswith("uint") or value_type.startswith("int"):
            size = int(value_type.lstrip("uint") or 256) // 8
        elif value_type.startswith("bytes"):
            size = int(value_type[5:])
        else:
            raise ValueError(f"unknown value type {value_type!r}")
        raw = word[32 - byte_offset - size:32 - byte_offset]
        if value_type == "bool":
            return raw != b"\0"
        if value_type.startswith("uint"):
            return int.from_bytes(raw, "big")
        if value_type.startswith("int"):
            return int.from_bytes(raw, "big", signed=True)
        return raw

    def as_c(self):
        """(ipcfp_storage_path, keepalive)"""
        steps = (A.PathStepC * max(len(self.steps), 1))()
        keep = [steps]
        for i, (op, key, index, elem_slots, elem_bytes) in enumerate(self.steps):
            st = steps[i]
            st.op, st.index, st.elem_slots, st.elem_bytes = op, index, elem_slots, elem_bytes
            if key:
                kb = C.create_string_buffer(key, len(key))
                keep.append(kb)
                st.key, st.key_len = C.addressof(kb), len(key)
        c = A.StoragePathC()
        c.actor_id = self.actor_id
        c.base_slot[:] = list(self.base_slot)
        c.n_steps, c.kind, c.n_words = len(self.steps), self.kind, self.n_words
        c.steps = C.addressof(steps) if self.steps else None
        return c, keep


def _paths_c(paths):
    """(ipcfp_storage_path array, count, keepalive) of a sequence of StoragePaths"""
    cs, keep = [], []
    for p in paths:
        c, k = p.as_c()
        cs.append(c)
        keep.append(k)
    return (A.StoragePathC * max(len(cs), 1))(*cs), len(cs), keep


class PinnedArray:
    """Pinned host memory (ipcfp_host_alloc) exposed as a numpy array."""

    def __init__(self, nbytes):
        p = C.c_void_p()
        _check(lib().ipcfp_host_alloc(max(int(nbytes), 1), C.byref(p)))
        self._p = p
        self.array = np.frombuffer((C.c_uint8 * max(int(nbytes), 1)).from_address(p.value), dtype=np.uint8)[:int(nbytes)]

    def free(self):
        if self._p:
            self.array = None
            lib().ipcfp_host_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class BlockStore:
    """Device-resident block store (replaces the reference's Blockstore implementations)."""

    def __init__(self, cids, offsets, lengths, blob, device=0, verify_cids=False):
        cids = np.ascontiguousarray(cids, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        lengths = np.ascontiguousarray(lengths, dtype=np.uint32)
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        self.n_blocks = len(lengths)
        self.device = device
        h = C.c_void_p()
        st = lib().ipcfp_store_create(cids.ctypes.data if cids.size else None, offsets.ctypes.data if offsets.size else None,
                                      lengths.ctypes.data if lengths.size else None, blob.ctypes.data if blob.size else None, blob.size,
                                      self.n_blocks, device, A.STORE_VERIFY_CIDS if verify_cids else 0, C.byref(h))
        self._adopt(st, h)

    def _adopt(self, st, h):
        """Takes the handle a store-creating call returned with status st. On failure the store is released and IpcfpError raised, with
        .first_bad_block (None when no store was made)."""
        self._h = h
        if st != A.OK:
            bad = lib().ipcfp_store_first_bad_block(h) if h else None
            msg, idx = lib().ipcfp_last_error().decode(errors="replace"), lib().ipcfp_last_error_index()
            self.close()
            e = A.IpcfpError(st, msg, idx)
            e.first_bad_block = bad
            raise e

    @classmethod
    def from_tipset(cls, ts, device=0, verify_cids=False):
        return cls(ts.cids, ts.offsets, ts.lengths, ts.blob, device, verify_cids)

    @classmethod
    def from_rpc_json(cls, cids, texts, device=0, verify_cids=False):
        """ipcfp_store_create_rpc_json: the store straight from Filecoin.ChainReadObj responses. cids: (n, 38) — request i asks for CID i
        with "id": i; texts: the response texts as received (str or bytes), each one response object or a batch. Canonical texts are
        parsed on the device. `.json_info` tells which path ran. Failures raise IpcfpError (status, request id or response position) with
        `.first_bad_block` as BlockStore() sets it. Pass verify_cids=True for bytes from an RPC node."""
        cids = np.ascontiguousarray(cids, dtype=np.uint8).reshape(-1, A.CID_LEN)
        arr, lens, keep = _text_array(texts)
        self = cls.__new__(cls)
        self.n_blocks, self.device, self._h = len(cids), device, None
        h, info = C.c_void_p(), A.StoreJsonInfoC()
        st = lib().ipcfp_store_create_rpc_json(cids.ctypes.data if cids.size else None, len(cids), arr, lens, len(keep), device,
                                               A.STORE_VERIFY_CIDS if verify_cids else 0, C.byref(h), C.byref(info))
        self.json_info = A.StoreJsonInfoPy(bool(info.parsed_on_device), float(info.ms_parse), float(info.ms_kernels))
        self._adopt(st, h)
        return self

    @classmethod
    def from_car(cls, car, device=0, verify_cids=False):
        """ipcfp_store_create_car: the store straight from a CARv1 archive (bytes, bytearray, mmap or a uint8 numpy array); block k is
        section k and by-reference offsets index `car`. The sections are found on the device; `.car_info` tells which path ran and its
        times. Failures raise IpcfpError (status, section index) with `.first_bad_block` as BlockStore() sets it."""
        buf = _car_view(car)
        self = cls.__new__(cls)
        self.device, self._h = device, None
        h, info = C.c_void_p(), A.StoreJsonInfoC()
        st = lib().ipcfp_store_create_car(buf.ctypes.data, buf.size, device, A.STORE_VERIFY_CIDS if verify_cids else 0, C.byref(h),
                                          C.byref(info))
        self.car_info = A.StoreJsonInfoPy(bool(info.parsed_on_device), float(info.ms_parse), float(info.ms_kernels))
        self._adopt(st, h)
        self.n_blocks = lib().ipcfp_store_n_blocks(h)
        return self

    def get(self, cid):
        cid = _u8(cid)
        ln = C.c_uint32()
        found = C.c_int()
        _check(lib().ipcfp_store_get(self._h, cid.ctypes.data, None, 0, C.byref(ln), C.byref(found)))
        if not found.value:
            return None
        buf = np.zeros(max(ln.value, 1), dtype=np.uint8)
        _check(lib().ipcfp_store_get(self._h, cid.ctypes.data, buf.ctypes.data, ln.value, C.byref(ln), C.byref(found)))
        return bytes(buf[:ln.value])

    def has(self, cid):
        cid = _u8(cid)
        found = C.c_int()
        _check(lib().ipcfp_store_has(self._h, cid.ctypes.data, C.byref(found)))
        return bool(found.value)

    # --- generate_event_proof (events/generator.rs:60-107)
    def generate_event_proof(self, ts, spec, flags=0):
        d, keep = A.make_tipset_desc(ts)
        cs = spec.as_c() if isinstance(spec, EventProofSpec) else spec
        return _result("ipcfp_generate_event_proof", *_EVENT_RESULT, self._h, C.byref(d), C.byref(cs), flags)

    def generate_log_proof(self, ts, log_filter, flags=0):
        """ipcfp_generate_log_proof: generate_event_proof with a LogFilter as the predicate → A.EventResultPy."""
        d, keep = A.make_tipset_desc(ts)
        return self._log_proof("ipcfp_generate_log_proof", C.byref(d), log_filter, flags)

    def generate_log_proof_resident(self, tip, log_filter, flags=0):
        """ipcfp_generate_log_proof_resident against a ResidentTipset of this store. flags: WITNESS_BY_REFERENCE, RESULT_JSON,
        SCAN_SKIP_TX_AMTS."""
        return self._log_proof("ipcfp_generate_log_proof_resident", tip._h, log_filter, flags)

    def _log_proof(self, fn, tipset, log_filter, flags):
        f, fkeep = log_filter.as_c()
        return _result(fn, *_EVENT_RESULT, self._h, tipset, C.byref(f), flags)

    def generate_message_log_proof(self, ts, message_cids, log_filter=None, flags=0):
        """ipcfp_generate_message_log_proof: the logs of the given messages (message_cids: (n, 38) message CIDs as the message AMTs hold
        them) that match log_filter (None: every log) → (A.EventResultPy, exec_indices): exec_indices[j] is message j's position in the
        execution order, 2**64 - 1 when the tipset did not execute it."""
        d, keep = A.make_tipset_desc(ts)
        return self._message_log_proof("ipcfp_generate_message_log_proof", C.byref(d), message_cids, log_filter, flags)

    def generate_message_log_proof_resident(self, tip, message_cids, log_filter=None, flags=0):
        """ipcfp_generate_message_log_proof_resident against a ResidentTipset of this store → (A.EventResultPy, exec_indices). flags:
        WITNESS_BY_REFERENCE, RESULT_JSON, SCAN_SKIP_TX_AMTS."""
        return self._message_log_proof("ipcfp_generate_message_log_proof_resident", tip._h, message_cids, log_filter, flags)

    @staticmethod
    def _message_args(message_cids, log_filter):
        cids = np.ascontiguousarray(message_cids, dtype=np.uint8).reshape(-1, A.CID_LEN)
        f, fkeep = log_filter.as_c() if log_filter is not None else (None, None)
        return cids, (C.byref(f) if f is not None else None), fkeep

    def _message_log_proof(self, fn, tipset, message_cids, log_filter, flags):
        cids, fp, fkeep = self._message_args(message_cids, log_filter)
        idx = np.zeros(len(cids), np.uint64)
        return _result(fn, *_EVENT_RESULT, self._h, tipset, cids.ctypes.data if cids.size else None, len(cids), fp, flags,
                       idx.ctypes.data if idx.size else None), idx

    def plan_fetch_messages(self, tip, message_cids, log_filter=None, flags=0):
        """ipcfp_plan_fetch_message_log_resident → A.FetchPlanPy: one fetch round for generate_message_log_proof_resident(tip, message_cids,
        log_filter)."""
        cids, fp, fkeep = self._message_args(message_cids, log_filter)
        return _result("ipcfp_plan_fetch_message_log_resident", *_FETCH_PLAN, self._h, tip._h, cids.ctypes.data if cids.size else None,
                       len(cids), fp, flags)

    def generate_event_proof_shard(self, ts, spec, lo, hi, world, rank, flags=0):
        d, keep = A.make_tipset_desc(ts)
        cs = spec.as_c() if isinstance(spec, EventProofSpec) else spec
        return _result("ipcfp_generate_event_proof_shard", *_EVENT_RESULT, self._h, C.byref(d), C.byref(cs), lo, hi, world, rank, flags)

    # --- read_storage_slot (storage/decode.rs:36-97), batched
    def read_storage_slots(self, root, slots):
        root = _u8(root)
        slots = _u8(slots).reshape(-1, 32)
        return _result("ipcfp_read_storage_slots", A.SlotResultC, A.slot_result_from_c, "ipcfp_slot_result_free", self._h, root.ctypes.data,
                       slots.ctypes.data if slots.size else None, len(slots))

    # --- generate_storage_proof (storage/generator.rs:29-67), batched
    def generate_storage_proofs(self, ts, specs):
        specs = [(s.actor_id, s.slot) if isinstance(s, StorageProofSpec) else s for s in specs]
        d, keep = A.make_tipset_desc(ts)
        arr = A.make_storage_specs(specs)
        return _result("ipcfp_generate_storage_proofs", A.StorageResultC, A.storage_result_from_c, "ipcfp_storage_result_free", self._h,
                       C.byref(d), arr, len(specs))

    # --- generate_proof_bundle (proofs/generator.rs:25-95)
    @staticmethod
    def _bundle_specs(storage_specs, event_specs):
        sspecs = [(s.actor_id, s.slot) if isinstance(s, StorageProofSpec) else s for s in storage_specs]
        especs = [s.as_c() if isinstance(s, EventProofSpec) else s for s in event_specs]
        return A.make_storage_specs(sspecs), len(sspecs), (A.EventSpec * len(especs))(*especs), len(especs)

    def generate_proof_bundle(self, ts, storage_specs, event_specs):
        d, keep = A.make_tipset_desc(ts)
        return _result("ipcfp_generate_proof_bundle", *_BUNDLE, self._h, C.byref(d), *self._bundle_specs(storage_specs, event_specs))

    def upload_tipset(self, ts):
        """ipcfp_tipset_upload: the tipset's descriptor on the device, for any number of _resident calls. close() releases it."""
        return ResidentTipset(self, ts)

    def upload_tipset_json(self, parent_text, child_text, receipts_text):
        """ipcfp_tipset_upload_json: the tipset straight from the Lotus JSON-RPC results — the ApiTipset of the parent and of the child
        (ChainGetTipSetByHeight) and the receipt list (ChainGetParentReceipts), each the `result` value as str or bytes. The receipt list is
        parsed on the device when it is canonical. Returns a ResidentTipset; failures raise IpcfpError (status, receipt index)."""
        p, c, r = (_text(x) for x in (parent_text, child_text, receipts_text))
        h = C.c_void_p()
        _check(lib().ipcfp_tipset_upload_json(self._h, p, len(p), c, len(c), r, len(r), C.byref(h)))
        return ResidentTipset(self, None, h)

    def generate_proof_bundle_resident(self, tip, storage_specs, event_specs, flags=0):
        """ipcfp_generate_proof_bundle_resident against a ResidentTipset of this store. flags: WITNESS_BY_REFERENCE, RESULT_JSON."""
        return _result("ipcfp_generate_proof_bundle_resident", *_BUNDLE, self._h, tip._h, *self._bundle_specs(storage_specs, event_specs),
                       flags)

    def plan_fetch(self, tip, storage_specs, event_specs, flags=0):
        """ipcfp_plan_fetch_resident → A.FetchPlanPy: the CIDs this store lacks of the blocks generate_proof_bundle_resident(tip,
        storage_specs, event_specs) would read, as far as the blocks it holds tell (one round; see fetch_until_complete)."""
        return _result("ipcfp_plan_fetch_resident", *_FETCH_PLAN, self._h, tip._h, *self._bundle_specs(storage_specs, event_specs), flags)

    def generate_log_bundle(self, ts, storage_specs, log_filters, flags=0):
        """ipcfp_generate_log_bundle: generate_proof_bundle with LogFilters in place of event specs (events[k] is filter k's result)
        → A.BundlePy. flags: WITNESS_BY_REFERENCE, RESULT_JSON."""
        d, keep = A.make_tipset_desc(ts)
        return self._log_bundle("ipcfp_generate_log_bundle", _BUNDLE, C.byref(d), storage_specs, log_filters, flags)

    def generate_log_bundle_resident(self, tip, storage_specs, log_filters, flags=0):
        """ipcfp_generate_log_bundle_resident against a ResidentTipset of this store → A.BundlePy."""
        return self._log_bundle("ipcfp_generate_log_bundle_resident", _BUNDLE, tip._h, storage_specs, log_filters, flags)

    def plan_fetch_log_bundle(self, tip, storage_specs, log_filters, flags=0):
        """ipcfp_plan_fetch_log_bundle_resident → A.FetchPlanPy: one fetch round for generate_log_bundle_resident(tip, storage_specs,
        log_filters)."""
        return self._log_bundle("ipcfp_plan_fetch_log_bundle_resident", _FETCH_PLAN, tip._h, storage_specs, log_filters, flags)

    def _log_bundle(self, fn, result, tipset, storage_specs, log_filters, flags):
        sarr, ns, _, _ = self._bundle_specs(storage_specs, [])
        farr, nf, fkeep = _log_filters_c(log_filters)
        return _result(fn, *result, self._h, tipset, sarr, ns, farr, nf, flags)

    def generate_storage_path_proofs_resident(self, tip, paths, flags=0):
        """ipcfp_generate_storage_path_proofs_resident → A.PathResultPy: the StoragePaths' expanded specs, values and statuses, and
        .storage, the proofs of the specs (what generate_storage_proofs gives for them). flags: WITNESS_BY_REFERENCE."""
        arr, n, keep = _paths_c(paths)
        return _result("ipcfp_generate_storage_path_proofs_resident", *_PATH_RESULT, self._h, tip._h, arr, n, flags)

    def plan_fetch_storage_paths(self, tip, paths, flags=0):
        """ipcfp_plan_fetch_storage_paths_resident → A.FetchPlanPy: one fetch round for generate_storage_path_proofs_resident."""
        arr, n, keep = _paths_c(paths)
        return _result("ipcfp_plan_fetch_storage_paths_resident", *_FETCH_PLAN, self._h, tip._h, arr, n, flags)

    def plan_fetch_logs(self, tip, log_filter, flags=0):
        """ipcfp_plan_fetch_log_resident → A.FetchPlanPy: one fetch round for generate_log_proof_resident(tip, log_filter)."""
        f, fkeep = log_filter.as_c()
        return _result("ipcfp_plan_fetch_log_resident", *_FETCH_PLAN, self._h, tip._h, C.byref(f), flags)

    def resolve_addresses(self, state_root, addresses):
        """ipcfp_resolve_addresses → A.ResolveResultPy: every address (Address::to_bytes(), or text for address_parse) resolved to its
        actor ID through the Init actor's address map of the state tree at state_root (38 bytes)."""
        root = _u8(state_root)
        if root.size != A.CID_LEN:
            raise ValueError("state_root must be a 38-byte CID")
        addrs = A.make_addresses([address_parse(a) if isinstance(a, str) else a for a in addresses])
        return _result("ipcfp_resolve_addresses", A.ResolveResultC, A.resolve_result_from_c, "ipcfp_resolve_result_free", self._h,
                       root.ctypes.data, addrs, len(addresses))

    def generate_actor_proofs_resident(self, tip, addresses, evm_code_cids=(), with_code=False, flags=0):
        """ipcfp_generate_actor_proofs_resident → A.ActorResultPy: per address (an int actor ID, "f…" / "t…" text, "0x…" Ethereum
        address or Address::to_bytes()) its actor's fields, or a proven absence. evm_code_cids: the EVM actor code CIDs (38 bytes each).
        with_code: ACTOR_WITH_CODE (the bytecode joins the proof). flags: WITNESS_BY_REFERENCE."""
        addrs, n, ev, n_ev, fl = _actor_args(addresses, evm_code_cids, with_code, flags)
        return _result("ipcfp_generate_actor_proofs_resident", A.ActorResultC, A.actor_result_from_c, "ipcfp_actor_result_free", self._h,
                       tip._h, addrs, n, ev.ctypes.data if n_ev else None, n_ev, fl)

    def plan_fetch_actor_proofs(self, tip, addresses, evm_code_cids=(), with_code=False, flags=0):
        """ipcfp_plan_fetch_actor_proofs_resident → A.FetchPlanPy: one fetch round for generate_actor_proofs_resident."""
        addrs, n, ev, n_ev, fl = _actor_args(addresses, evm_code_cids, with_code, flags)
        return _result("ipcfp_plan_fetch_actor_proofs_resident", *_FETCH_PLAN, self._h, tip._h, addrs, n, ev.ctypes.data if n_ev else None,
                       n_ev, fl)

    def generate_message_proofs_resident(self, tip, message_cids, with_body=False, flags=0):
        """ipcfp_generate_message_proofs_resident → A.MessageResultPy: per message CID ((n, 38) bytes, as the message AMTs hold them)
        whether it executed and its receipt; with_body: MESSAGE_WITH_BODY (the message block joins the witness and its fields the
        proof). flags: WITNESS_BY_REFERENCE."""
        cids = np.ascontiguousarray(message_cids, dtype=np.uint8).reshape(-1, A.CID_LEN)
        return _result("ipcfp_generate_message_proofs_resident", A.MessageResultC, A.message_result_from_c, "ipcfp_message_result_free",
                       self._h, tip._h, cids.ctypes.data if cids.size else None, len(cids), flags | (A.MESSAGE_WITH_BODY if with_body else 0))

    def plan_fetch_message_proofs(self, tip, message_cids, with_body=False, flags=0):
        """ipcfp_plan_fetch_message_proofs_resident → A.FetchPlanPy: one fetch round for generate_message_proofs_resident."""
        cids = np.ascontiguousarray(message_cids, dtype=np.uint8).reshape(-1, A.CID_LEN)
        return _result("ipcfp_plan_fetch_message_proofs_resident", *_FETCH_PLAN, self._h, tip._h, cids.ctypes.data if cids.size else None,
                       len(cids), flags | (A.MESSAGE_WITH_BODY if with_body else 0))

    def close(self):
        if self._h:
            lib().ipcfp_store_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ResidentTipset:
    """A tipset descriptor uploaded to a store's device (ipcfp_tipset_upload / ipcfp_tipset_free). Valid while its store lives."""

    def __init__(self, store, ts, handle=None):
        if handle is None:
            d, keep = A.make_tipset_desc(ts)
            handle = C.c_void_p()
            _check(lib().ipcfp_tipset_upload(store._h, C.byref(d), C.byref(handle)))
        self._h = handle
        self.store = store

    def describe(self, with_events_roots=True):
        """ipcfp_tipset_describe → A.TipsetInfoPy: the descriptor the tipset holds (events roots copied back from the device when asked),
        which path parsed its receipt list and how long that took."""
        info = A.TipsetInfoC()
        _check(lib().ipcfp_tipset_describe(self._h, 1 if with_events_roots else 0, C.byref(info)))
        return A.tipset_info_from_c(info.desc, info.parsed_on_device, info.ms_parse, info.ms_kernels)

    def close(self):
        if self._h:
            lib().ipcfp_tipset_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _text(x):
    return x.encode() if isinstance(x, str) else x if isinstance(x, bytes) else bytes(x)


def _text_array(texts):
    """texts (str or bytes each) → (char** array, u64 length array, the bytes objects they point into)."""
    keep = [_text(t) for t in texts]
    arr = (C.c_char_p * max(len(keep), 1))(*keep)
    lens = (C.c_uint64 * max(len(keep), 1))(*[len(t) for t in keep])
    return arr, lens, keep


def blocks_from_rpc_json(cids, texts):
    """ipcfp_blocks_from_rpc_json (host parser, no device): the blocks of Filecoin.ChainReadObj responses in request order, as an
    A.WitnessPy (cids, 16-aligned offsets, lengths, blob). Failures raise IpcfpError with the status and the index include/ipcfp.h gives."""
    cids = np.ascontiguousarray(cids, dtype=np.uint8).reshape(-1, A.CID_LEN)
    arr, lens, keep = _text_array(texts)
    return _result("ipcfp_blocks_from_rpc_json", A.ParsedBlocksC, lambda c: A.witness_from_c(c.blocks), "ipcfp_parsed_blocks_free",
                   cids.ctypes.data if cids.size else None, len(cids), arr, lens, len(keep))


def _car_view(car):
    """The bytes of a CAR (bytes, bytearray, mmap, or a numpy array of uint8) as a flat uint8 array over the same memory where possible."""
    if isinstance(car, np.ndarray):
        if car.dtype != np.uint8:
            raise TypeError("a CAR array must be uint8")
        buf = np.ascontiguousarray(car).reshape(-1)
    else:
        buf = np.frombuffer(car, dtype=np.uint8)
    return buf if buf.size else np.zeros(1, np.uint8)[:0]


def blocks_from_car(car):
    """ipcfp_blocks_from_car (host parser, no device): the sections of a CARv1 in file order, as an A.WitnessPy whose offsets index the
    CAR itself (its blob is a view of `car`). Failures raise IpcfpError with the status and the section index include/ipcfp.h gives."""
    buf = _car_view(car)
    w = _result("ipcfp_blocks_from_car", A.ParsedBlocksC, lambda c: A.witness_from_c(c.blocks), "ipcfp_parsed_blocks_free",
                buf.ctypes.data, buf.size)
    w.blob = buf
    return w


def fetch_plan_to_rpc_json(cids, first_id=0):
    """ipcfp_fetch_plan_to_rpc_json: one Filecoin.ChainReadObj batch (bytes) asking for cids ((n, 38)) with ids first_id + k."""
    cids = np.ascontiguousarray(cids, dtype=np.uint8).reshape(-1, A.CID_LEN)
    p = A.FetchPlanC(len(cids), cids.ctypes.data_as(C.POINTER(C.c_uint8)) if cids.size else None, 0, 0, 0.0)
    out, ln = C.c_void_p(), C.c_uint64()
    _check(lib().ipcfp_fetch_plan_to_rpc_json(C.byref(p), first_id, C.byref(out), C.byref(ln)))
    try:
        return C.string_at(out.value, ln.value)
    finally:
        lib().ipcfp_json_free(out)


@dataclass
class FetchRound:
    """One round of fetch_until_complete: the CIDs requested, the plan's device time, the wall time of the store rebuild after it."""
    cids: np.ndarray
    ms_plan: float
    ms_rebuild: float


def fetch_until_complete(fetch, upload_tipset, storage_specs, event_specs, device=0, verify_cids=True, max_rounds=10000):
    """Plans and fetches rounds until the store holds every block a proof bundle needs (include/ipcfp.h, "Fetch planning").

    fetch(cids, first_id) asks for cids ((k, 38)) and returns the Filecoin.ChainReadObj response texts (request j has "id": first_id + j;
    fetch_plan_to_rpc_json(cids, first_id) is that request); upload_tipset(store) returns the store's ResidentTipset (upload_tipset or
    upload_tipset_json). Starts from an empty store; each round rebuilds it with BlockStore.from_rpc_json over every response so far.
    Returns (store, tipset, rounds, cids, texts): the complete store, its tipset, the FetchRounds, and the CIDs and texts it was built
    from."""
    return _fetch_loop(lambda store, tip: store.plan_fetch(tip, storage_specs, event_specs), fetch, upload_tipset, device, verify_cids,
                       max_rounds)


def fetch_log_bundle_until_complete(fetch, upload_tipset, storage_specs, log_filters, device=0, verify_cids=True, max_rounds=10000):
    """fetch_until_complete for generate_log_bundle_resident(tip, storage_specs, log_filters): the same loop, planned with
    plan_fetch_log_bundle."""
    return _fetch_loop(lambda store, tip: store.plan_fetch_log_bundle(tip, storage_specs, log_filters), fetch, upload_tipset, device,
                       verify_cids, max_rounds)


def fetch_messages_until_complete(fetch, upload_tipset, message_cids, log_filter=None, device=0, verify_cids=True, max_rounds=10000):
    """fetch_until_complete for generate_message_log_proof_resident(tip, message_cids, log_filter): the same loop, planned with
    plan_fetch_messages."""
    return _fetch_loop(lambda store, tip: store.plan_fetch_messages(tip, message_cids, log_filter), fetch, upload_tipset, device, verify_cids,
                       max_rounds)


def fetch_storage_paths_until_complete(fetch, upload_tipset, paths, device=0, verify_cids=True, max_rounds=10000):
    """fetch_until_complete for generate_storage_path_proofs_resident(tip, paths): the same loop, planned with plan_fetch_storage_paths
    (a long bytes / string value takes one round more: its data slots are known once its header word is)."""
    return _fetch_loop(lambda store, tip: store.plan_fetch_storage_paths(tip, paths), fetch, upload_tipset, device, verify_cids, max_rounds)


def _fetch_loop(plan_round, fetch, upload_tipset, device, verify_cids, max_rounds):
    """fetch_until_complete's loop; plan_round(store, tip) → the round's A.FetchPlanPy"""
    import time
    all_cids, texts, rounds = np.zeros((0, A.CID_LEN), np.uint8), [], []
    store = BlockStore(all_cids, np.zeros(0, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.uint8), device=device)
    tip = upload_tipset(store)
    for _ in range(max_rounds):
        plan = plan_round(store, tip)
        if not len(plan.cids):
            return store, tip, rounds, all_cids, texts
        got = fetch(plan.cids, len(all_cids))
        texts += [got] if isinstance(got, (bytes, str)) else list(got)
        all_cids = np.concatenate([all_cids, plan.cids])
        t0 = time.perf_counter()
        tip.close()
        store.close()
        store = BlockStore.from_rpc_json(all_cids, texts, device=device, verify_cids=verify_cids)
        tip = upload_tipset(store)
        rounds.append(FetchRound(plan.cids, plan.ms_total, (time.perf_counter() - t0) * 1e3))
    raise RuntimeError("fetch_until_complete: no fixed point after %d rounds" % max_rounds)


def address_parse(text):
    """ipcfp_address_parse (host, no device): "f…" / "t…" address text → Address::to_bytes(). Malformed text raises IpcfpError."""
    raw = text.encode() if isinstance(text, str) else bytes(text)
    a = A.AddressC()
    _check(lib().ipcfp_address_parse(raw, len(raw), C.byref(a)))
    return a.to_bytes()


def _eth_bytes(eth_addr):
    """The reference's validation of an Ethereum address (src/proofs/common/address.rs:10-21) → 20 bytes; ValueError with its messages."""
    if isinstance(eth_addr, (bytes, bytearray)):
        b = bytes(eth_addr)
    else:
        s = eth_addr
        while s.startswith("0x"):          # trim_start_matches("0x")
            s = s[2:]
        raw = s.encode()
        if len(raw) % 2:
            raise ValueError("Invalid hex in Ethereum address: Odd number of digits")
        for i, c in enumerate(raw):
            if chr(c) not in "0123456789abcdefABCDEF":
                raise ValueError(f"Invalid hex in Ethereum address: Invalid character {chr(c)!r} at position {i}")
        b = bytes.fromhex(s)
    if len(b) != 20:
        raise ValueError(f"Invalid Ethereum address length: expected 20 bytes, got {len(b)}")
    return b


def address_from_eth(eth_addr):
    """ipcfp_address_from_eth (host, no device): "0x…" hex or 20 bytes → Address::to_bytes() of the Filecoin address Lotus's
    EthAddressToFilecoinAddress returns (a masked ID → the ID address, else f410)."""
    b = _eth_bytes(eth_addr)
    a = A.AddressC()
    _check(lib().ipcfp_address_from_eth(b, C.byref(a)))
    return a.to_bytes()


def resolve_eth_address_to_actor_id(store, state_root, eth_addr):
    """The reference's resolve_eth_address_to_actor_id (src/proofs/common/address.rs:8-62) from the state tree at state_root instead of
    two RPC calls: the same validation and messages, then the Init actor's address map. Raises IpcfpError when the address does not
    resolve (status ACTOR_NOT_FOUND, MISSING_BLOCK or DECODE)."""
    r = store.resolve_addresses(state_root, [address_from_eth(eth_addr)])
    st = int(r.status[0])
    if st != A.OK:
        raise A.IpcfpError(st, "Failed to lookup ID address", 0)
    return int(r.actor_ids[0])


@dataclass
class ResolveRound:
    """One round of resolve_until_complete: the CIDs requested and the resolver's device time before it."""
    cids: np.ndarray
    ms_resolve: float


def resolve_until_complete(fetch, state_root, addresses, device=0, verify_cids=True, cids=None, texts=None, max_rounds=10000):
    """Resolves addresses, fetching the blocks the walks lack until none is missing: fetch_until_complete's loop with the resolver's
    missing list as the plan. fetch(cids, first_id) returns the Filecoin.ChainReadObj response texts for cids ((k, 38)) with ids
    first_id + j. cids / texts: blocks the caller already holds (their CIDs and response texts), else an empty store.
    Returns (store, result, rounds, cids, texts)."""
    all_cids = np.zeros((0, A.CID_LEN), np.uint8) if cids is None else np.ascontiguousarray(cids, np.uint8).reshape(-1, A.CID_LEN)
    texts = list(texts or [])
    rounds = []

    def make_store():
        if len(all_cids):
            return BlockStore.from_rpc_json(all_cids, texts, device=device, verify_cids=verify_cids)
        return BlockStore(all_cids, np.zeros(0, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.uint8), device=device)

    store = make_store()
    for _ in range(max_rounds):
        r = store.resolve_addresses(state_root, addresses)
        if not len(r.missing):
            return store, r, rounds, all_cids, texts
        got = fetch(r.missing, len(all_cids))
        texts += [got] if isinstance(got, (bytes, str)) else list(got)
        all_cids = np.concatenate([all_cids, r.missing])
        rounds.append(ResolveRound(r.missing, r.ms_total))
        store.close()
        store = make_store()
    raise RuntimeError("resolve_until_complete: no fixed point after %d rounds" % max_rounds)


def actor_address(a):
    """An actor proof's request → Address::to_bytes(): an int is an actor ID, text is "0x…" (address_from_eth) or "f…" / "t…"
    (address_parse), bytes are taken as they are."""
    if isinstance(a, int):
        if not 0 <= a < 2 ** 64:
            raise ValueError(f"actor ID {a} out of range")
        out = bytearray([0])
        while a >= 0x80:
            out.append((a & 0x7F) | 0x80)
            a >>= 7
        out.append(a)
        return bytes(out)
    if isinstance(a, str):
        return address_from_eth(a) if a.startswith("0x") else address_parse(a)
    return bytes(a)


def _actor_args(addresses, evm_code_cids, with_code, flags):
    raw = [actor_address(a) for a in addresses]
    ev = np.ascontiguousarray(np.frombuffer(b"".join(bytes(c) for c in evm_code_cids), dtype=np.uint8)) if len(evm_code_cids) else np.zeros(0, np.uint8)
    if ev.size % A.CID_LEN:
        raise ValueError("evm_code_cids must be 38-byte CIDs")
    return A.make_addresses(raw), len(raw), ev, ev.size // A.CID_LEN, flags | (A.ACTOR_WITH_CODE if with_code else 0)


def fetch_actor_proofs_until_complete(fetch, upload_tipset, addresses, evm_code_cids=(), with_code=False, device=0, verify_cids=True,
                                      max_rounds=10000):
    """fetch_until_complete for generate_actor_proofs_resident(tip, addresses, evm_code_cids, with_code): the same loop, planned with
    plan_fetch_actor_proofs."""
    return _fetch_loop(lambda store, tip: store.plan_fetch_actor_proofs(tip, addresses, evm_code_cids, with_code), fetch, upload_tipset, device,
                       verify_cids, max_rounds)


def verify_actor_proofs(witness, ts, result, evm_code_cids=(), with_code=False, device=0):
    """ipcfp_verify_actor_proofs over the witness (WitnessPy) as a CID-checked store: every proof of `result` (A.ActorResultPy, or packed
    ipcfp_actor_proof records) replayed against the tipset `ts` → list of bools."""
    raw = np.ascontiguousarray(result.raw_proofs if hasattr(result, "raw_proofs") else result, dtype=np.uint8)
    n = raw.size // C.sizeof(A.ActorProofC)
    _, _, ev, n_ev, fl = _actor_args([], evm_code_cids, with_code, 0)
    store = BlockStore(witness.cids, witness.offsets, witness.lengths, witness.blob, device, verify_cids=True)
    try:
        d, keep = A.make_tipset_desc(ts)
        res = np.zeros(max(n, 1), dtype=np.uint8)
        _check(lib().ipcfp_verify_actor_proofs(store._h, C.byref(d), raw.ctypes.data if n else None, n, ev.ctypes.data if n_ev else None, n_ev,
                                               fl, res.ctypes.data))
        return [bool(x) for x in res[:n]]
    finally:
        store.close()


def fetch_message_proofs_until_complete(fetch, upload_tipset, message_cids, with_body=False, device=0, verify_cids=True, max_rounds=10000):
    """fetch_until_complete for generate_message_proofs_resident(tip, message_cids, with_body): the same loop, planned with
    plan_fetch_message_proofs."""
    return _fetch_loop(lambda store, tip: store.plan_fetch_message_proofs(tip, message_cids, with_body), fetch, upload_tipset, device,
                       verify_cids, max_rounds)


def verify_message_proofs(witness, ts, result, with_body=False, data_blob=None, device=0):
    """ipcfp_verify_message_proofs over the witness (WitnessPy) as a CID-checked store: every proof of `result` (A.MessageResultPy, or
    packed ipcfp_message_proof records with their data_blob) replayed against the tipset `ts` → list of bools."""
    raw = np.ascontiguousarray(result.raw_proofs if hasattr(result, "raw_proofs") else result, dtype=np.uint8)
    blob = np.frombuffer(result.data_blob if data_blob is None else data_blob, dtype=np.uint8)
    n = raw.size // C.sizeof(A.MessageProofC)
    store = BlockStore(witness.cids, witness.offsets, witness.lengths, witness.blob, device, verify_cids=True)
    try:
        d, keep = A.make_tipset_desc(ts)
        res = np.zeros(max(n, 1), dtype=np.uint8)
        _check(lib().ipcfp_verify_message_proofs(store._h, C.byref(d), raw.ctypes.data if n else None, n, blob.ctypes.data if blob.size else None,
                                                 blob.size, A.MESSAGE_WITH_BODY if with_body else 0, res.ctypes.data))
        return [bool(x) for x in res[:n]]
    finally:
        store.close()


def tipset_desc_from_json(parent_text, child_text, receipts_text):
    """ipcfp_tipset_desc_from_json (host parser, no device): the descriptor of the Lotus JSON-RPC texts as an A.TipsetInfoPy. Failures raise
    IpcfpError with the status and the receipt index (UINT64_MAX outside the receipt list's elements)."""
    p, c, r = (_text(x) for x in (parent_text, child_text, receipts_text))
    return _result("ipcfp_tipset_desc_from_json", A.ParsedTipsetC, lambda t: A.tipset_info_from_c(t.desc), "ipcfp_parsed_tipset_free",
                   p, len(p), c, len(c), r, len(r))


def _to_json(fn, obj_ptr, ts):
    d, keep = A.make_tipset_desc(ts)
    out, n = C.c_void_p(), C.c_uint64()
    _check(getattr(lib(), fn)(obj_ptr, C.byref(d), C.byref(out), C.byref(n)))
    try:
        return C.string_at(out.value, n.value).decode()
    finally:
        lib().ipcfp_json_free(out)


def bundle_to_json(bundle_c_ptr, ts):
    """`serde_json::to_string(&UnifiedProofBundle)` of an ipcfp_bundle (POINTER(BundleC) or its address)."""
    return _to_json("ipcfp_bundle_to_json", C.cast(bundle_c_ptr, C.c_void_p), ts)


def event_result_to_json(result_c_ptr, ts):
    """`serde_json::to_string(&EventProofBundle)` of an ipcfp_event_result."""
    return _to_json("ipcfp_event_result_to_json", C.cast(result_c_ptr, C.c_void_p), ts)


class ParsedBundle:
    """`serde_json::from_str::<UnifiedProofBundle | EventProofBundle>` through the C ABI (ipcfp_bundle_from_json): PODs ready for the
    batched verifiers + the witness block arrays. Owns the C object; `.c` is the ipcfp_parsed_bundle."""

    def __init__(self, text):
        raw = text.encode() if isinstance(text, str) else bytes(text)
        self._p = C.POINTER(A.ParsedBundleC)()
        st = lib().ipcfp_bundle_from_json(raw, len(raw), C.byref(self._p))
        if st != A.OK:
            raise A.IpcfpError(st, "ipcfp_bundle_from_json", 0)
        self.c = self._p.contents

    @property
    def witness(self):
        return A.witness_from_c(self.c.witness)

    @property
    def event_proofs_raw(self):
        n = int(self.c.n_event_proofs)
        return A._arr(self.c.event_proofs, n * C.sizeof(A.EventProofC), np.uint8), A._arr(self.c.data_blob, int(self.c.data_blob_size), np.uint8)

    @property
    def storage_proofs_raw(self):
        return A._arr(self.c.storage_proofs, int(self.c.n_storage_proofs) * C.sizeof(A.StorageProofC), np.uint8)

    def tipset_fields(self):
        t = self.c.tipset
        P = int(t.n_parents)
        return dict(parent_epoch=int(t.parent_epoch), child_epoch=int(t.child_epoch),
                    parent_cids=A._arr(t.parent_cids, P * A.CID_LEN, np.uint8).tobytes(),
                    child_cid=A._arr(t.child_cid, A.CID_LEN if t.child_cid else 0, np.uint8).tobytes(),
                    parent_state_root=A._arr(t.child_parent_state_root, A.CID_LEN if t.child_parent_state_root else 0, np.uint8).tobytes())

    def close(self):
        if self._p:
            lib().ipcfp_parsed_bundle_free(self._p)
            self._p = C.POINTER(A.ParsedBundleC)()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BundleVerdict:
    """verify_proof_bundle (src/proofs/verifier.rs:12-60) from the JSON text (ipcfp_verify_bundle_json): storage_results / event_results
    (UnifiedVerificationResult), the parsed proofs (raw PODs, as ParsedBundle has them), the shared tipset fields, the path taken
    (parsed_on_device) and the phase times."""

    def __init__(self, c):
        n_s, n_e = int(c.n_storage_proofs), int(c.n_event_proofs)
        self.storage_results = [bool(x) for x in A._arr(c.storage_results, n_s, np.uint8)] if n_s else []
        self.event_results = [bool(x) for x in A._arr(c.event_results, n_e, np.uint8)] if n_e else []
        self.storage_proofs_raw = A._arr(c.storage_proofs, n_s * C.sizeof(A.StorageProofC), np.uint8).copy() if n_s else np.zeros(0, np.uint8)
        self.event_proofs_raw = A._arr(c.event_proofs, n_e * C.sizeof(A.EventProofC), np.uint8).copy() if n_e else np.zeros(0, np.uint8)
        nb = int(c.data_blob_size)
        self.data_blob = A._arr(c.data_blob, nb, np.uint8).copy() if nb else np.zeros(0, np.uint8)
        t = c.tipset
        P = int(t.n_parents)
        self.tipset = dict(parent_epoch=int(t.parent_epoch), child_epoch=int(t.child_epoch),
                           parent_cids=A._arr(t.parent_cids, P * A.CID_LEN, np.uint8).tobytes() if P else b"",
                           child_cid=A._arr(t.child_cid, A.CID_LEN, np.uint8).tobytes() if t.child_cid else None,
                           parent_state_root=A._arr(t.child_parent_state_root, A.CID_LEN, np.uint8).tobytes() if t.child_parent_state_root else None)
        self.n_blocks, self.witness_bytes = int(c.n_blocks), int(c.witness_bytes)
        self.parsed_on_device = bool(c.parsed_on_device)
        self.ms = dict(total=c.ms_total, parse=c.ms_parse, store=c.ms_store, verify=c.ms_verify)


_VERDICT = (A.BundleVerdictC, BundleVerdict, "ipcfp_bundle_verdict_free")


def _trust_callbacks(trusted_parent, trusted_child):
    cb_p = A.TrustedParentFn(lambda ctx, e, p, n: int(bool(trusted_parent(int(e), C.string_at(p, 38 * n) if n else b""))))\
        if trusted_parent else A.TrustedParentFn()
    cb_c = A.TrustedChildFn(lambda ctx, e, c: int(bool(trusted_child(int(e), C.string_at(c, 38))))) if trusted_child else A.TrustedChildFn()
    return cb_p, cb_c


def verify_bundle_json(text, trusted_parent=None, trusted_child=None, filter_spec=None, device=0):
    """ipcfp_verify_bundle_json. trusted_parent(epoch, parent_cids: bytes) / trusted_child(epoch, child_cid: bytes) → bool, None = accept
    all. filter_spec: an A.EventSpec (check_event) or None. → BundleVerdict; failures raise IpcfpError (status, index)."""
    raw = text.encode() if isinstance(text, str) else bytes(text)
    cb_p, cb_c = _trust_callbacks(trusted_parent, trusted_child)
    return _result("ipcfp_verify_bundle_json", *_VERDICT, raw, len(raw), device, cb_p, cb_c, None,
                   C.addressof(filter_spec) if filter_spec is not None else None)


def verify_bundle_json_any(text, trusted_parent=None, trusted_child=None, log_filters=(), device=0):
    """ipcfp_verify_bundle_json_any: verify_bundle_json with check_event = "matches at least one of log_filters" (LogFilters; empty: no
    check_event). → BundleVerdict; failures raise IpcfpError (status, index)."""
    raw = text.encode() if isinstance(text, str) else bytes(text)
    cb_p, cb_c = _trust_callbacks(trusted_parent, trusted_child)
    farr, nf, fkeep = _log_filters_c(log_filters)
    return _result("ipcfp_verify_bundle_json_any", *_VERDICT, raw, len(raw), device, cb_p, cb_c, None, farr, nf)


def _verify(witness, ts, result, device, fn, *args, blob=True):
    """lib().<fn>(store, descriptor, proofs, n, [data blob, blob size,] *args, results) over the witness (WitnessPy) as a store with every
    block Blake2b-checked against its CID → list of bools, one per proof of `result`. blob: pass result.data_blob."""
    store = BlockStore(witness.cids, witness.offsets, witness.lengths, witness.blob, device, verify_cids=True)
    try:
        d, keep = A.make_tipset_desc(ts)
        n = len(result.proofs)
        res = np.zeros(max(n, 1), dtype=np.uint8)
        raw = np.ascontiguousarray(result.raw_proofs)
        if blob:
            data = np.ascontiguousarray(result.data_blob)
            args = (data.ctypes.data if data.size else None, data.size) + args
        _check(getattr(lib(), fn)(store._h, C.byref(d), raw.ctypes.data if n else None, n, *args, res.ctypes.data))
        return [bool(x) for x in res[:n]]
    finally:
        store.close()


def verify_event_proofs(witness, ts, result, filter_spec=None, device=0):
    """verify_event_proof (events/verifier.rs:51-74) batched on the GPU: the witness (WitnessPy) becomes a store with every block
    Blake2b-checked against its CID, then every proof of `result` (EventResultPy) is replayed. filter_spec (check_event): None, an
    EventProofSpec or a LogFilter (ipcfp_verify_event_proofs_log). → list of bools."""
    if isinstance(filter_spec, LogFilter):
        f, fkeep = filter_spec.as_c()
        return _verify(witness, ts, result, device, "ipcfp_verify_event_proofs_log", C.byref(f))
    fs = filter_spec.as_c() if isinstance(filter_spec, EventProofSpec) else filter_spec
    return _verify(witness, ts, result, device, "ipcfp_verify_event_proofs", C.addressof(fs) if fs is not None else None)


def verify_event_proofs_any(witness, ts, result, log_filters, device=0):
    """verify_event_proofs with check_event = "matches at least one of log_filters" (ipcfp_verify_event_proofs_any; an empty sequence:
    no check_event). result: anything with raw_proofs, data_blob and proofs (A.EventResultPy). → list of bools."""
    farr, nf, fkeep = _log_filters_c(log_filters)
    return _verify(witness, ts, result, device, "ipcfp_verify_event_proofs_any", farr, nf)


def verify_storage_proofs(witness, ts, result, device=0):
    """verify_storage_proof (storage/verifier.rs:24-63) batched on the GPU over a CID-checked witness store."""
    return _verify(witness, ts, result, device, "ipcfp_verify_storage_proofs", blob=False)


def verify_storage_paths(witness, ts, proofs, paths, device=0):
    """ipcfp_verify_storage_paths over the witness (WitnessPy) as a CID-checked store: proofs — an A.StorageResultPy, a list of
    A.StorageProofPy or packed ipcfp_storage_proof records — against the StoragePaths → A.PathResultPy (per path: valid, status, value;
    storage None)."""
    if hasattr(proofs, "raw_proofs"):
        raw = proofs.raw_proofs
    elif isinstance(proofs, np.ndarray):
        raw = proofs
    else:
        raw = A.pack_storage_proofs(proofs)
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    n = raw.size // C.sizeof(A.StorageProofC)
    store = BlockStore(witness.cids, witness.offsets, witness.lengths, witness.blob, device, verify_cids=True)
    try:
        d, keep = A.make_tipset_desc(ts)
        arr, np_, pkeep = _paths_c(paths)
        return _result("ipcfp_verify_storage_paths", *_PATH_RESULT, store._h, C.byref(d), raw.ctypes.data if n else None, n, arr, np_)
    finally:
        store.close()


def _hash_batch(fn, messages, device=0):
    n = len(messages)
    lengths = np.array([len(m) for m in messages], dtype=np.uint32)
    offsets = np.zeros(n, dtype=np.uint64)
    if n:
        offsets[1:] = np.cumsum(lengths[:-1], dtype=np.uint64)
    blob = np.frombuffer(b"".join(bytes(m) for m in messages), dtype=np.uint8) if n else np.zeros(0, dtype=np.uint8)
    out = np.zeros((n, 32), dtype=np.uint8)
    _check(getattr(lib(), fn)(blob.ctypes.data if blob.size else None, blob.size, offsets.ctypes.data if n else None,
                              lengths.ctypes.data if n else None, n, device, out.ctypes.data if n else None))
    return [bytes(r) for r in out]


def blake2b256_batch(messages, device=0):
    return _hash_batch("ipcfp_blake2b256_batch", messages, device)


def keccak256_batch(messages, device=0):
    return _hash_batch("ipcfp_keccak256_batch", messages, device)


def sha256_batch(messages, device=0):
    return _hash_batch("ipcfp_sha256_batch", messages, device)


def compute_mapping_slots(keys32, slot_indices, device=0):
    """compute_mapping_slot (storage/utils.rs:5-12) batched on the GPU."""
    keys = np.ascontiguousarray(np.frombuffer(b"".join(bytes(k) for k in keys32), dtype=np.uint8))
    idx = np.ascontiguousarray(slot_indices, dtype=np.uint64)
    n = len(idx)
    out = np.zeros((n, 32), dtype=np.uint8)
    _check(lib().ipcfp_compute_mapping_slots(keys.ctypes.data if n else None, idx.ctypes.data if n else None, n, device,
                                             out.ctypes.data if n else None))
    return [bytes(r) for r in out]


def calculate_storage_slot(subnet_ascii, subnets_slot_index, device=0):
    """calculate_storage_slot (storage/utils.rs:16-19)."""
    b = subnet_ascii.encode()[:32]
    return compute_mapping_slots([b + bytes(32 - len(b))], [subnets_slot_index], device)[0]
