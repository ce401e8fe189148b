"""ctypes mirror of include/ipcfp.h (POD structs only) + converters to Python result objects.

Shared by the product binding (api.py) and by the test oracle's binding (oracle/__init__.py):
both libraries fill the same structs so parity tests compare field by field.
"""
import ctypes as C
from dataclasses import dataclass, field

import numpy as np

CID_LEN = 38

OK = 0
ERR_INVALID_ARG = -1
ERR_MISSING_BLOCK = -2
ERR_DECODE = -3
ERR_CID_MISMATCH = -4
ERR_MISSING_EXEC = -5
ERR_CUDA = -6
ERR_NCCL = -7
ERR_STATE_ROOT_MISMATCH = -8
ERR_ACTOR_NOT_FOUND = -9
ERR_NO_DEVICE = -10
ERR_UNSUPPORTED = -11

STORE_VERIFY_CIDS = 0x1
SCAN_SKIP_TX_AMTS = 0x1
SHARDED_UNION_TO_HOST = 0x2
SHARDED_UNION_FULL = 0x4
WITNESS_BY_REFERENCE = 0x8
RESULT_JSON = 0x10
ACTOR_WITH_CODE = 0x20
COMM_ID_BYTES = 128


class TipsetDesc(C.Structure):
    _fields_ = [
        ("parent_epoch", C.c_int64),
        ("child_epoch", C.c_int64),
        ("n_parents", C.c_uint32),
        ("parent_cids", C.c_void_p),
        ("parent_txmeta_cids", C.c_void_p),
        ("child_cid", C.c_void_p),
        ("receipts_root", C.c_void_p),
        ("child_parent_state_root", C.c_void_p),
        ("n_receipts", C.c_uint64),
        ("events_roots", C.c_void_p),
        ("has_events_root", C.c_void_p),
    ]


class EventSpec(C.Structure):
    _fields_ = [
        ("event_signature", C.c_char_p),
        ("topic_1", C.c_char_p),
        ("has_actor_id_filter", C.c_uint8),
        ("actor_id_filter", C.c_uint64),
    ]


LOG_FILTER_MAX_VALUES = 65536
MESSAGE_MAX = 65536   # IPCFP_MESSAGE_MAX: message CIDs of one ipcfp_generate_message_log_proof call
LOG_FILTER_MAX_EMITTERS = 65536


class LogFilterC(C.Structure):
    """ipcfp_log_filter"""
    _fields_ = [
        ("n_emitters", C.c_uint64),
        ("emitters", C.c_void_p),
        ("n_positions", C.c_uint32),
        ("_pad", C.c_uint32),
        ("n_values", C.c_uint64 * 4),
        ("values", C.c_void_p * 4),
    ]


class StorageSpec(C.Structure):
    _fields_ = [("actor_id", C.c_uint64), ("slot", C.c_uint8 * 32)]


class Witness(C.Structure):
    _fields_ = [
        ("n_blocks", C.c_uint64),
        ("cids", C.c_void_p),
        ("offsets", C.c_void_p),
        ("lengths", C.c_void_p),
        ("blob", C.c_void_p),
        ("blob_size", C.c_uint64),
    ]


class EventProofC(C.Structure):
    _fields_ = [
        ("exec_index", C.c_uint64),
        ("event_index", C.c_uint64),
        ("emitter", C.c_uint64),
        ("n_topics", C.c_uint32),
        ("data_len", C.c_uint32),
        ("data_off", C.c_uint64),
        ("topics_off", C.c_uint64),
        ("message_cid", C.c_uint8 * CID_LEN),
        ("_pad", C.c_uint8 * 2),
    ]


class EventResultC(C.Structure):
    _fields_ = [
        ("n_matching", C.c_uint64),
        ("matching_indices", C.c_void_p),
        ("n_proofs", C.c_uint64),
        ("proofs", C.POINTER(EventProofC)),
        ("data_blob", C.c_void_p),
        ("data_blob_size", C.c_uint64),
        ("witness", Witness),
        ("n_exec", C.c_uint64),
        ("ms_total", C.c_float),
        ("ms_pass1", C.c_float),
        ("ms_pass2", C.c_float),
        ("ms_txamt", C.c_float),
        ("ms_witness", C.c_float),
        ("pass1_bytes", C.c_uint64),
        ("pass1_nodes", C.c_uint64),
        ("shard_exec_dev", C.c_void_p),
        ("shard_exec_count", C.c_uint64),
        ("shard_raw_total", C.c_uint64),
        ("union_cids_dev", C.c_void_p),
        ("n_union_cids", C.c_uint64),
        ("union_cids", C.c_void_p),
        ("total_matching", C.c_uint64),
        ("total_proofs", C.c_uint64),
        ("ms_exchange", C.c_float),
        ("ms_fetch", C.c_float),
        ("ms_union", C.c_float),
        ("_pad0", C.c_float),
        ("union_part_first", C.c_uint64),
        ("n_union_part", C.c_uint64),
        ("json", C.c_void_p),
        ("json_len", C.c_uint64),
        ("ms_json", C.c_float),
        ("_pad1", C.c_float),
    ]


class StorageProofC(C.Structure):
    _fields_ = [
        ("actor_id", C.c_uint64),
        ("actor_state_cid", C.c_uint8 * CID_LEN),
        ("storage_root", C.c_uint8 * CID_LEN),
        ("slot", C.c_uint8 * 32),
        ("value", C.c_uint8 * 32),
        ("found", C.c_uint8),
        ("_pad", C.c_uint8 * 3),
        ("raw_len", C.c_uint32),
    ]


class ParsedBundleC(C.Structure):
    """ipcfp_parsed_bundle (ipcfp_bundle_from_json)."""
    _fields_ = [
        ("tipset", TipsetDesc),
        ("n_storage_proofs", C.c_uint64),
        ("storage_proofs", C.c_void_p),
        ("n_event_proofs", C.c_uint64),
        ("event_proofs", C.c_void_p),
        ("data_blob", C.c_void_p),
        ("data_blob_size", C.c_uint64),
        ("witness", Witness),
    ]


class ParsedTipsetC(C.Structure):
    """ipcfp_parsed_tipset (ipcfp_tipset_desc_from_json)."""
    _fields_ = [("desc", TipsetDesc)]


class TipsetInfoC(C.Structure):
    """ipcfp_tipset_info (ipcfp_tipset_describe)."""
    _fields_ = [("desc", TipsetDesc), ("parsed_on_device", C.c_uint32), ("ms_parse", C.c_float), ("ms_kernels", C.c_float),
                ("_pad", C.c_uint32)]


@dataclass
class TipsetInfoPy:
    """A tipset descriptor read back from the C ABI, with the attribute names of synth.Tipset (so make_tipset_desc takes it)."""
    parent_epoch: int
    child_epoch: int
    n_parents: int
    parent_cids: np.ndarray          # (n_parents, 38)
    parent_txmeta_cids: np.ndarray   # (n_parents, 38)
    child_cid: np.ndarray            # (38,)
    receipts_root: np.ndarray        # (38,)
    parent_state_root: np.ndarray    # (38,) or None
    n_receipts: int
    events_roots: np.ndarray         # (n_receipts, 38), or None when not read back
    has_events_root: np.ndarray      # (n_receipts,), or None when not read back
    parsed_on_device: bool = False
    ms_parse: float = 0.0
    ms_kernels: float = 0.0


def tipset_info_from_c(d, parsed_on_device=0, ms_parse=0.0, ms_kernels=0.0):
    P, N = int(d.n_parents), int(d.n_receipts)
    roots = _arr(d.events_roots, N * CID_LEN, np.uint8).reshape(N, CID_LEN) if d.events_roots or not N else None
    has = _arr(d.has_events_root, N, np.uint8) if d.has_events_root or not N else None
    return TipsetInfoPy(int(d.parent_epoch), int(d.child_epoch), P, _arr(d.parent_cids, P * CID_LEN, np.uint8).reshape(P, CID_LEN),
                        _arr(d.parent_txmeta_cids, P * CID_LEN, np.uint8).reshape(P, CID_LEN), _arr(d.child_cid, CID_LEN, np.uint8),
                        _arr(d.receipts_root, CID_LEN, np.uint8),
                        _arr(d.child_parent_state_root, CID_LEN, np.uint8) if d.child_parent_state_root else None, N, roots, has,
                        bool(parsed_on_device), float(ms_parse), float(ms_kernels))


class ParsedBlocksC(C.Structure):
    """ipcfp_parsed_blocks (ipcfp_blocks_from_rpc_json)."""
    _fields_ = [("blocks", Witness)]


class StoreJsonInfoC(C.Structure):
    """ipcfp_store_json_info (ipcfp_store_create_rpc_json)."""
    _fields_ = [("parsed_on_device", C.c_uint32), ("ms_parse", C.c_float), ("ms_kernels", C.c_float), ("_pad", C.c_uint32)]


@dataclass
class StoreJsonInfoPy:
    """How ipcfp_store_create_rpc_json built a store: the path that parsed the texts and its times."""
    parsed_on_device: bool
    ms_parse: float
    ms_kernels: float


class FetchPlanC(C.Structure):
    """ipcfp_fetch_plan (ipcfp_plan_fetch_resident)."""
    _fields_ = [("n_missing", C.c_uint64), ("cids", C.POINTER(C.c_uint8)), ("n_needed", C.c_uint64), ("n_levels", C.c_uint32),
                ("ms_total", C.c_float)]


@dataclass
class FetchPlanPy:
    """One round of fetch planning: the CIDs the store lacks ((n, 38), `Cid` order), how many needed blocks it holds, the device walk's
    levels and its time."""
    cids: np.ndarray
    n_needed: int
    n_levels: int
    ms_total: float


def fetch_plan_from_c(p):
    cids = np.ctypeslib.as_array(p.cids, shape=(p.n_missing * CID_LEN,)).copy() if p.n_missing else np.zeros(0, np.uint8)
    return FetchPlanPy(cids.reshape(-1, CID_LEN), int(p.n_needed), int(p.n_levels), float(p.ms_total))


ADDRESS_MAX = 65


class AddressC(C.Structure):
    """ipcfp_address: Address::to_bytes() (protocol byte, then the payload)."""
    _fields_ = [("len", C.c_uint8), ("bytes", C.c_uint8 * ADDRESS_MAX)]

    def to_bytes(self):
        return bytes(self.bytes[:self.len])


def make_addresses(addresses):
    """[bytes] (Address::to_bytes() each) → ctypes array of ipcfp_address. Inputs longer than IPCFP_ADDRESS_MAX do not fit and are
    refused here; other malformed bytes reach the call, which reports them as IPCFP_ERR_INVALID_ARG."""
    parts = []
    for i, a in enumerate(addresses):
        a = bytes(a)
        if len(a) > ADDRESS_MAX:
            raise ValueError(f"address {i}: {len(a)} bytes (at most {ADDRESS_MAX})")
        parts.append(bytes([len(a)]) + a.ljust(ADDRESS_MAX, b"\0"))
    return (AddressC * max(len(addresses), 1)).from_buffer_copy(b"".join(parts) or bytes(C.sizeof(AddressC)))


class ResolveResultC(C.Structure):
    """ipcfp_resolve_result (ipcfp_resolve_addresses)."""
    _fields_ = [("n", C.c_uint64), ("actor_ids", C.c_void_p), ("status", C.c_void_p), ("init_status", C.c_int32), ("_pad", C.c_uint32),
                ("n_missing", C.c_uint64), ("missing_cids", C.c_void_p), ("witness", Witness), ("ms_total", C.c_float), ("ms_lookup", C.c_float)]


@dataclass
class ResolveResultPy:
    """Actor IDs (0 where status != OK), per-address status, the Init path's status, the CIDs the walks lacked ((m, 38), `Cid` order),
    the blocks they read, and the device times."""
    actor_ids: np.ndarray
    status: np.ndarray
    init_status: int
    missing: np.ndarray
    witness: "WitnessPy"
    ms_total: float
    ms_lookup: float


def resolve_result_from_c(r):
    n, m = int(r.n), int(r.n_missing)
    return ResolveResultPy(_arr(r.actor_ids, n, np.uint64), _arr(r.status, n, np.int32), int(r.init_status),
                           _arr(r.missing_cids, m * CID_LEN, np.uint8).reshape(m, CID_LEN), witness_from_c(r.witness), float(r.ms_total),
                           float(r.ms_lookup))


# Actor proofs (include/ipcfp.h, "Actor proofs")
ACTOR_MAX = 65536
ACTOR_FOUND, ACTOR_NO_ADDRESS, ACTOR_NO_ACTOR = 0, 1, 2


class ActorProofC(C.Structure):
    """ipcfp_actor_proof (400 bytes)."""
    _fields_ = [("actor_id", C.c_uint64), ("sequence", C.c_uint64), ("evm_nonce", C.c_uint64), ("code_off", C.c_uint64), ("code_len", C.c_uint64),
                ("status", C.c_uint32), ("balance_negative", C.c_uint8), ("has_delegated", C.c_uint8), ("is_evm", C.c_uint8), ("_pad0", C.c_uint8),
                ("balance", C.c_uint8 * 32), ("code", C.c_uint8 * CID_LEN), ("head", C.c_uint8 * CID_LEN), ("bytecode_cid", C.c_uint8 * CID_LEN),
                ("contract_state", C.c_uint8 * CID_LEN), ("bytecode_hash", C.c_uint8 * 32), ("address", AddressC), ("delegated", AddressC),
                ("_pad1", C.c_uint8 * 4)]


class ActorResultC(C.Structure):
    """ipcfp_actor_result (ipcfp_generate_actor_proofs_resident)."""
    _fields_ = [("n_proofs", C.c_uint64), ("proofs", C.c_void_p), ("witness", Witness), ("proof_witness_offsets", C.c_void_p),
                ("proof_witness_index", C.c_void_p), ("code_blob", C.c_void_p), ("code_blob_size", C.c_uint64), ("ms_total", C.c_float),
                ("ms_init", C.c_float), ("ms_walk", C.c_float), ("ms_code", C.c_float), ("ms_witness", C.c_float), ("host_syncs", C.c_uint32)]


@dataclass
class ActorProof:
    """What the state tree holds for `address` (Address::to_bytes()): status ACTOR_*, the actor ID, ActorState's code, head, sequence,
    balance (a signed int) and delegated address (bytes or None), and for an EVM actor its bytecode CID and hash, EVM nonce, storage root
    (contract_state) and, with ACTOR_WITH_CODE, its bytecode."""
    address: bytes
    status: int
    actor_id: int
    code: bytes
    head: bytes
    sequence: int
    balance: int
    delegated: bytes
    is_evm: bool
    bytecode_cid: bytes
    bytecode_hash: bytes
    evm_nonce: int
    contract_state: bytes
    bytecode: bytes = None


def actor_proof_from_c(p, blob=b""):
    mag = int.from_bytes(bytes(p.balance), "big")
    return ActorProof(p.address.to_bytes(), int(p.status), int(p.actor_id), bytes(p.code), bytes(p.head), int(p.sequence),
                      -mag if p.balance_negative else mag, p.delegated.to_bytes() if p.has_delegated else None, bool(p.is_evm),
                      bytes(p.bytecode_cid), bytes(p.bytecode_hash), int(p.evm_nonce), bytes(p.contract_state),
                      blob[int(p.code_off):int(p.code_off) + int(p.code_len)] if p.code_len and blob else None)


@dataclass
class ActorResultPy:
    proofs: list            # ActorProof per request
    witness: "WitnessPy"
    proof_witness: list     # per proof: indices into witness
    raw_proofs: np.ndarray  # packed ipcfp_actor_proof records (for the verifier)
    timings: dict = field(default_factory=dict)
    host_syncs: int = 0


def actor_result_from_c(r):
    n = int(r.n_proofs)
    raw = _arr(r.proofs, n * C.sizeof(ActorProofC), np.uint8)
    blob = C.string_at(r.code_blob, int(r.code_blob_size)) if r.code_blob_size else b""
    recs = (ActorProofC * max(n, 1)).from_buffer_copy(raw.tobytes() or bytes(C.sizeof(ActorProofC)))
    offs = _arr(r.proof_witness_offsets, n + 1, np.uint64)
    idx = _arr(r.proof_witness_index, int(offs[-1]) if n else 0, np.uint32)
    timings = dict(total=r.ms_total, init=r.ms_init, walk=r.ms_walk, code=r.ms_code, witness=r.ms_witness)
    return ActorResultPy([actor_proof_from_c(recs[i], blob) for i in range(n)], witness_from_c(r.witness),
                         [idx[int(offs[i]):int(offs[i + 1])].tolist() for i in range(n)], raw, timings, int(r.host_syncs))


# Message proofs (include/ipcfp.h, "Message proofs")
MESSAGE_WITH_BODY = 0x40
MESSAGE_EXECUTED, MESSAGE_NOT_EXECUTED, MESSAGE_NO_RECEIPT = 0, 1, 2


class MessageProofC(C.Structure):
    """ipcfp_message_proof (400 bytes)."""
    _fields_ = [("exec_index", C.c_uint64), ("gas_used", C.c_uint64), ("return_off", C.c_uint64), ("return_len", C.c_uint64),
                ("version", C.c_uint64), ("sequence", C.c_uint64), ("gas_limit", C.c_uint64), ("method_num", C.c_uint64),
                ("params_off", C.c_uint64), ("params_len", C.c_uint64), ("status", C.c_uint32), ("exit_code", C.c_uint32),
                ("has_events_root", C.c_uint8), ("has_body", C.c_uint8), ("sig_type", C.c_uint8), ("value_negative", C.c_uint8),
                ("gas_fee_cap_negative", C.c_uint8), ("gas_premium_negative", C.c_uint8), ("_pad0", C.c_uint8 * 2),
                ("value", C.c_uint8 * 32), ("gas_fee_cap", C.c_uint8 * 32), ("gas_premium", C.c_uint8 * 32),
                ("message_cid", C.c_uint8 * CID_LEN), ("events_root", C.c_uint8 * CID_LEN), ("to", AddressC), ("from_", AddressC)]


class MessageResultC(C.Structure):
    """ipcfp_message_result (ipcfp_generate_message_proofs_resident)."""
    _fields_ = [("n_proofs", C.c_uint64), ("proofs", C.c_void_p), ("data_blob", C.c_void_p), ("data_blob_size", C.c_uint64),
                ("witness", Witness), ("n_exec", C.c_uint64), ("ms_total", C.c_float), ("ms_exec_order", C.c_float), ("ms_walk", C.c_float),
                ("ms_gather", C.c_float), ("ms_witness", C.c_float), ("host_syncs", C.c_uint32)]


@dataclass
class MessageProof:
    """Whether `message_cid` executed (status MESSAGE_*, exec_index or None) and its receipt: exit code, return data, gas used and events
    root (bytes or None). With the body (has_body): the Message fields, value / gas_fee_cap / gas_premium as signed ints, to / from as
    Address::to_bytes(), and sig_type (0 for an unsigned Message)."""
    message_cid: bytes
    status: int
    exec_index: int
    exit_code: int
    return_data: bytes
    gas_used: int
    events_root: bytes
    has_body: bool = False
    version: int = 0
    to: bytes = b""
    from_: bytes = b""
    sequence: int = 0
    value: int = 0
    gas_limit: int = 0
    gas_fee_cap: int = 0
    gas_premium: int = 0
    method_num: int = 0
    params: bytes = b""
    sig_type: int = 0


def _signed(mag, negative):
    m = int.from_bytes(bytes(mag), "big")
    return -m if negative else m


def message_proof_from_c(p, blob=b""):
    ro, rl, po, pl = int(p.return_off), int(p.return_len), int(p.params_off), int(p.params_len)
    return MessageProof(bytes(p.message_cid), int(p.status), None if p.exec_index == 2 ** 64 - 1 else int(p.exec_index), int(p.exit_code),
                        blob[ro:ro + rl], int(p.gas_used), bytes(p.events_root) if p.has_events_root else None, bool(p.has_body),
                        int(p.version), p.to.to_bytes() if p.has_body else b"", p.from_.to_bytes() if p.has_body else b"", int(p.sequence),
                        _signed(p.value, p.value_negative), int(p.gas_limit), _signed(p.gas_fee_cap, p.gas_fee_cap_negative),
                        _signed(p.gas_premium, p.gas_premium_negative), int(p.method_num), blob[po:po + pl], int(p.sig_type))


@dataclass
class MessageResultPy:
    proofs: list            # MessageProof per request
    witness: "WitnessPy"
    data_blob: bytes
    raw_proofs: np.ndarray  # packed ipcfp_message_proof records (for the verifier)
    n_exec: int = 0
    timings: dict = field(default_factory=dict)
    host_syncs: int = 0


def message_result_from_c(r):
    n = int(r.n_proofs)
    raw = _arr(r.proofs, n * C.sizeof(MessageProofC), np.uint8)
    blob = C.string_at(r.data_blob, int(r.data_blob_size)) if r.data_blob_size else b""
    recs = (MessageProofC * max(n, 1)).from_buffer_copy(raw.tobytes() or bytes(C.sizeof(MessageProofC)))
    timings = dict(total=r.ms_total, exec_order=r.ms_exec_order, walk=r.ms_walk, gather=r.ms_gather, witness=r.ms_witness)
    return MessageResultPy([message_proof_from_c(recs[i], blob) for i in range(n)], witness_from_c(r.witness), blob, raw, int(r.n_exec),
                           timings, int(r.host_syncs))


TrustedParentFn = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32)
TrustedChildFn = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int64, C.c_void_p)


class BundleVerdictC(C.Structure):
    """ipcfp_bundle_verdict (ipcfp_verify_bundle_json)."""
    _fields_ = [
        ("tipset", TipsetDesc),
        ("n_storage_proofs", C.c_uint64),
        ("storage_proofs", C.c_void_p),
        ("storage_results", C.c_void_p),
        ("n_event_proofs", C.c_uint64),
        ("event_proofs", C.c_void_p),
        ("event_results", C.c_void_p),
        ("data_blob", C.c_void_p),
        ("data_blob_size", C.c_uint64),
        ("n_blocks", C.c_uint64),
        ("witness_bytes", C.c_uint64),
        ("parsed_on_device", C.c_uint32),
        ("ms_total", C.c_float),
        ("ms_parse", C.c_float),
        ("ms_store", C.c_float),
        ("ms_verify", C.c_float),
        ("_pad", C.c_uint32),
    ]


class StorageResultC(C.Structure):
    _fields_ = [
        ("n_proofs", C.c_uint64),
        ("proofs", C.POINTER(StorageProofC)),
        ("witness", Witness),
        ("spec_witness_offsets", C.c_void_p),
        ("spec_witness_index", C.c_void_p),
        ("ms_total", C.c_float),
    ]


# Storage paths (include/ipcfp.h, "Storage paths")
PATH_MAX_PATHS = 65536
PATH_MAX_STEPS = 32
PATH_MAX_KEY = 1024
PATH_MAX_WORDS = 256
PATH_MAX_BYTES = 4096
PATH_MAPPING, PATH_ARRAY, PATH_STATIC, PATH_FIELD = 0, 1, 2, 3
PATH_WORDS, PATH_BYTES = 0, 1
PATH_OK, PATH_INDEX_OUT_OF_RANGE, PATH_BAD_BYTES, PATH_TOO_LONG = 0, 1, 2, 3


class PathStepC(C.Structure):
    """ipcfp_path_step"""
    _fields_ = [("op", C.c_uint32), ("key_len", C.c_uint32), ("key", C.c_void_p), ("index", C.c_uint64), ("elem_slots", C.c_uint32),
                ("elem_bytes", C.c_uint32)]


class StoragePathC(C.Structure):
    """ipcfp_storage_path"""
    _fields_ = [("actor_id", C.c_uint64), ("base_slot", C.c_uint8 * 32), ("n_steps", C.c_uint32), ("kind", C.c_uint32), ("steps", C.c_void_p),
                ("n_words", C.c_uint32), ("_pad", C.c_uint32)]


class PathValueC(C.Structure):
    """ipcfp_path_value"""
    _fields_ = [("status", C.c_uint32), ("valid", C.c_uint32), ("slot", C.c_uint8 * 32), ("byte_offset", C.c_uint32), ("_pad", C.c_uint32),
                ("first_spec", C.c_uint64), ("n_specs", C.c_uint64), ("value_off", C.c_uint64), ("value_len", C.c_uint64)]


class SlotResultC(C.Structure):
    _fields_ = [
        ("n", C.c_uint64),
        ("found", C.c_void_p),
        ("raw_len", C.c_void_p),
        ("values", C.c_void_p),
        ("witness", Witness),
        ("ms_total", C.c_float),
        ("ms_lookup", C.c_float),
        ("lookup_nodes", C.c_uint64),
        ("lookup_bytes", C.c_uint64),
    ]


class BundleC(C.Structure):
    _fields_ = [
        ("storage", C.POINTER(StorageResultC)),
        ("n_event_results", C.c_uint64),
        ("events", C.POINTER(C.POINTER(EventResultC))),
        ("witness", Witness),
        ("json", C.c_void_p),
        ("json_len", C.c_uint64),
        ("ms_total", C.c_float),
        ("ms_json", C.c_float),
    ]


class PathResultC(C.Structure):
    """ipcfp_path_result"""
    _fields_ = [("n_paths", C.c_uint64), ("paths", C.c_void_p), ("n_specs", C.c_uint64), ("specs", C.c_void_p), ("value_blob", C.c_void_p),
                ("value_blob_size", C.c_uint64), ("storage", C.POINTER(StorageResultC)), ("ms_total", C.c_float), ("ms_slots", C.c_float),
                ("ms_wave1", C.c_float), ("ms_wave2", C.c_float), ("ms_witness", C.c_float), ("host_syncs", C.c_uint32)]


def _arr(ptr, n, dtype):
    """Copy n items of dtype from a raw pointer into a fresh numpy array."""
    if n == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    nbytes = n * np.dtype(dtype).itemsize
    buf = (C.c_uint8 * nbytes).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype).copy()


@dataclass
class WitnessPy:
    cids: np.ndarray      # (m, 38) uint8, sorted in Cid Ord
    offsets: np.ndarray   # (m,) uint64
    lengths: np.ndarray   # (m,) uint32
    blob: np.ndarray      # uint8 (blocks in any order)

    @property
    def n_blocks(self):
        return len(self.cids)

    @property
    def total_bytes(self):
        return int(self.lengths.sum())

    def block(self, i):
        o = int(self.offsets[i])
        return bytes(self.blob[o:o + int(self.lengths[i])])

    def blocks(self):
        return [self.block(i) for i in range(self.n_blocks)]

    def as_dict(self):
        return {bytes(self.cids[i]): self.block(i) for i in range(self.n_blocks)}

    def as_c(self):
        """Returns (Witness struct, keepalive) for passing back into C."""
        cids = np.ascontiguousarray(self.cids)
        offs = np.ascontiguousarray(self.offsets)
        lens = np.ascontiguousarray(self.lengths)
        blob = np.ascontiguousarray(self.blob)
        w = Witness(len(cids), cids.ctypes.data, offs.ctypes.data, lens.ctypes.data, blob.ctypes.data, len(blob))
        return w, (cids, offs, lens, blob)


def witness_from_c(w):
    m = int(w.n_blocks)
    return WitnessPy(_arr(w.cids, m * CID_LEN, np.uint8).reshape(m, CID_LEN), _arr(w.offsets, m, np.uint64), _arr(w.lengths, m, np.uint32),
                     _arr(w.blob, int(w.blob_size), np.uint8))


@dataclass
class EventProofPy:
    exec_index: int
    event_index: int
    emitter: int
    topics: list          # list of 32-byte bytes
    data: bytes
    message_cid: bytes

    def key(self):
        return (self.exec_index, self.event_index, self.emitter, tuple(self.topics), self.data, self.message_cid)


@dataclass
class EventResultPy:
    matching: np.ndarray
    proofs: list
    witness: WitnessPy
    n_exec: int
    timings: dict = field(default_factory=dict)
    pass1_bytes: int = 0
    pass1_nodes: int = 0
    raw_proofs: np.ndarray = None   # packed ipcfp_event_proof records (for the verifier)
    data_blob: np.ndarray = None
    json: str = None        # IPCFP_RESULT_JSON: the EventProofBundle text rendered on the device


def event_result_from_c(r):
    matching = _arr(r.matching_indices, int(r.n_matching), np.uint64)
    data = _arr(r.data_blob, int(r.data_blob_size), np.uint8)
    n = int(r.n_proofs)
    raw = _arr(C.cast(r.proofs, C.c_void_p).value, n * C.sizeof(EventProofC), np.uint8)
    proofs = []
    db = data.tobytes()
    for i in range(n):
        p = r.proofs[i]
        topics = [db[p.topics_off + 32 * k: p.topics_off + 32 * (k + 1)] for k in range(p.n_topics)]
        proofs.append(EventProofPy(int(p.exec_index), int(p.event_index), int(p.emitter), topics,
                                   db[p.data_off:p.data_off + p.data_len], bytes(p.message_cid)))
    timings = dict(total=r.ms_total, pass1=r.ms_pass1, pass2=r.ms_pass2, txamt=r.ms_txamt, witness=r.ms_witness)
    text = None
    if r.json:
        text = C.string_at(r.json, int(r.json_len)).decode()
        timings["json"] = r.ms_json
    return EventResultPy(matching, proofs, witness_from_c(r.witness), int(r.n_exec), timings, int(r.pass1_bytes), int(r.pass1_nodes), raw, data, text)


def pack_event_proofs(proofs):
    """list of EventProofPy → (packed ipcfp_event_proof records as uint8, data blob as uint8): the layout the C ABI returns."""
    n = len(proofs)
    recs = (EventProofC * max(n, 1))()
    blob = bytearray()
    for i, p in enumerate(proofs):
        r = recs[i]
        r.exec_index, r.event_index, r.emitter = int(p.exec_index), int(p.event_index), int(p.emitter)
        r.n_topics, r.data_len = len(p.topics), len(p.data)
        r.topics_off = len(blob)
        for t in p.topics:
            blob += bytes(t)
        r.data_off = len(blob)
        blob += bytes(p.data)
        r.message_cid[:] = list(bytes(p.message_cid))
    raw = np.frombuffer(bytes(recs)[:n * C.sizeof(EventProofC)], dtype=np.uint8).copy()
    return raw, np.frombuffer(bytes(blob) + bytes(16), dtype=np.uint8).copy()


def pack_storage_proofs(proofs):
    """list of StorageProofPy → packed ipcfp_storage_proof records as uint8."""
    n = len(proofs)
    recs = (StorageProofC * max(n, 1))()
    for i, p in enumerate(proofs):
        r = recs[i]
        r.actor_id = int(p.actor_id)
        r.actor_state_cid[:] = list(bytes(p.actor_state_cid))
        r.storage_root[:] = list(bytes(p.storage_root))
        r.slot[:] = list(bytes(p.slot))
        r.value[:] = list(bytes(p.value))
        r.found, r.raw_len = int(bool(p.found)), int(p.raw_len)
    return np.frombuffer(bytes(recs)[:n * C.sizeof(StorageProofC)], dtype=np.uint8).copy()


@dataclass
class StorageProofPy:
    actor_id: int
    actor_state_cid: bytes
    storage_root: bytes
    slot: bytes
    value: bytes
    found: bool
    raw_len: int


@dataclass
class StorageResultPy:
    proofs: list
    witness: WitnessPy
    spec_witness: list      # per spec: list of indices into witness
    ms_total: float = 0.0
    raw_proofs: np.ndarray = None


def storage_result_from_c(r):
    n = int(r.n_proofs)
    proofs = []
    for i in range(n):
        p = r.proofs[i]
        proofs.append(StorageProofPy(int(p.actor_id), bytes(p.actor_state_cid), bytes(p.storage_root), bytes(p.slot), bytes(p.value),
                                     bool(p.found), int(p.raw_len)))
    offs = _arr(r.spec_witness_offsets, n + 1, np.uint64)
    idx = _arr(r.spec_witness_index, int(offs[-1]) if n else 0, np.uint32)
    spec_w = [idx[int(offs[i]):int(offs[i + 1])].tolist() for i in range(n)]
    raw = _arr(C.cast(r.proofs, C.c_void_p).value, n * C.sizeof(StorageProofC), np.uint8)
    return StorageResultPy(proofs, witness_from_c(r.witness), spec_w, float(r.ms_total), raw)


@dataclass
class SlotResultPy:
    found: np.ndarray
    raw_len: np.ndarray
    values: np.ndarray   # (n, 32)
    witness: WitnessPy
    ms_total: float = 0.0
    ms_lookup: float = 0.0
    lookup_nodes: int = 0
    lookup_bytes: int = 0


def slot_result_from_c(r):
    n = int(r.n)
    return SlotResultPy(_arr(r.found, n, np.uint8), _arr(r.raw_len, n, np.uint32), _arr(r.values, n * 32, np.uint8).reshape(n, 32),
                        witness_from_c(r.witness), float(r.ms_total), float(r.ms_lookup), int(r.lookup_nodes), int(r.lookup_bytes))


@dataclass
class PathValuePy:
    """One path's outcome: status (PATH_*), valid (the verifier's verdict; 1 from the generator), the final slot, the packed byte offset,
    its expanded specs specs[first_spec : first_spec + n_specs] and its value (the words, or the decoded bytes)."""
    status: int
    valid: bool
    slot: bytes
    byte_offset: int
    first_spec: int
    n_specs: int
    value: bytes


@dataclass
class PathResultPy:
    paths: list             # PathValuePy per path
    specs: list             # the expanded specs, (actor_id, slot) pairs in path order
    storage: StorageResultPy = None   # generate: the proofs of specs; verify: None
    timings: dict = field(default_factory=dict)
    host_syncs: int = 0


def path_result_from_c(r):
    n, m = int(r.n_paths), int(r.n_specs)
    vals = (PathValueC * max(n, 1)).from_address(r.paths) if n else []
    blob = C.string_at(r.value_blob, int(r.value_blob_size)) if r.value_blob_size else b""
    paths = [PathValuePy(int(v.status), bool(v.valid), bytes(v.slot), int(v.byte_offset), int(v.first_spec), int(v.n_specs),
                         blob[int(v.value_off):int(v.value_off) + int(v.value_len)]) for v in (vals[i] for i in range(n))]
    raw = _arr(r.specs, m * C.sizeof(StorageSpec), np.uint8)
    sz = C.sizeof(StorageSpec)
    specs = [(int.from_bytes(raw[sz * i:sz * i + 8].tobytes(), "little"), raw[sz * i + 8:sz * i + 40].tobytes()) for i in range(m)]
    st = storage_result_from_c(r.storage.contents) if r.storage else None
    timings = dict(total=r.ms_total, slots=r.ms_slots, wave1=r.ms_wave1, wave2=r.ms_wave2, witness=r.ms_witness)
    return PathResultPy(paths, specs, st, timings, int(r.host_syncs))


@dataclass
class BundlePy:
    storage: StorageResultPy
    events: list
    witness: WitnessPy
    json: str = None        # IPCFP_RESULT_JSON: the UnifiedProofBundle text rendered on the device
    timings: dict = field(default_factory=dict)


def bundle_from_c(b):
    st = storage_result_from_c(b.storage.contents) if b.storage else None
    ev = [event_result_from_c(b.events[i].contents) for i in range(int(b.n_event_results))]
    timings = dict(total=b.ms_total)
    text = None
    if b.json:
        text = C.string_at(b.json, int(b.json_len)).decode()
        timings["json"] = b.ms_json
    return BundlePy(st, ev, witness_from_c(b.witness), text, timings)


class IpcfpError(RuntimeError):
    def __init__(self, status, msg, index):
        super().__init__(f"ipcfp status {status}: {msg} (index {index})")
        self.status = status
        self.msg = msg
        self.index = index


def make_tipset_desc(ts):
    """Build a TipsetDesc from any object with the synth.Tipset attribute names.
    Returns (desc, keepalive)."""
    keep = []

    def ptr(a):
        a = np.ascontiguousarray(a, dtype=np.uint8)
        keep.append(a)
        return a.ctypes.data if a.size else None

    d = TipsetDesc()
    d.parent_epoch = int(ts.parent_epoch)
    d.child_epoch = int(ts.child_epoch)
    d.n_parents = int(ts.n_parents)
    d.parent_cids = ptr(ts.parent_cids)
    d.parent_txmeta_cids = ptr(ts.parent_txmeta_cids)
    d.child_cid = ptr(ts.child_cid)
    d.receipts_root = ptr(ts.receipts_root)
    d.child_parent_state_root = ptr(ts.parent_state_root)
    d.n_receipts = int(ts.n_receipts)
    d.events_roots = ptr(ts.events_roots)
    d.has_events_root = ptr(ts.has_events_root)
    return d, keep


def make_event_spec(event_signature, topic_1, actor_id_filter=None):
    s = EventSpec()
    s.event_signature = event_signature.encode()
    s.topic_1 = topic_1.encode()
    s.has_actor_id_filter = 0 if actor_id_filter is None else 1
    s.actor_id_filter = 0 if actor_id_filter is None else int(actor_id_filter)
    return s


def make_storage_specs(specs):
    arr = (StorageSpec * len(specs))()
    for i, (actor, slot) in enumerate(specs):
        arr[i].actor_id = int(actor)
        arr[i].slot[:] = list(slot)
    return arr
