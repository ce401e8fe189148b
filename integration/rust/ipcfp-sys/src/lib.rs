//! Raw bindings of `include/ipcfp.h` (what `bindgen` emits, written out by hand).
//! NOT BUILT IN THIS REPO: the build image has no Rust toolchain. Every item mirrors the C header one to one;
//! the reference-side shim (`GpuBlockstore`, `generate_event_proof_gpu`) is sketched in INTEGRATION.md §3.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_int, c_void};

pub const IPCFP_CID_LEN: usize = 38;
pub type ipcfp_status = i32;
pub const IPCFP_OK: ipcfp_status = 0;
pub const IPCFP_ERR_INVALID_ARG: ipcfp_status = -1;
pub const IPCFP_ERR_MISSING_BLOCK: ipcfp_status = -2;
pub const IPCFP_ERR_DECODE: ipcfp_status = -3;
pub const IPCFP_ERR_CID_MISMATCH: ipcfp_status = -4;
pub const IPCFP_ERR_MISSING_EXEC: ipcfp_status = -5;
pub const IPCFP_ERR_CUDA: ipcfp_status = -6;
pub const IPCFP_ERR_NCCL: ipcfp_status = -7;
pub const IPCFP_ERR_STATE_ROOT_MISMATCH: ipcfp_status = -8;
pub const IPCFP_ERR_ACTOR_NOT_FOUND: ipcfp_status = -9;
pub const IPCFP_ERR_NO_DEVICE: ipcfp_status = -10;
pub const IPCFP_ERR_UNSUPPORTED: ipcfp_status = -11;
pub const IPCFP_STORE_VERIFY_CIDS: u32 = 0x1;
pub const IPCFP_SCAN_SKIP_TX_AMTS: u32 = 0x1;
pub const IPCFP_SHARDED_UNION_TO_HOST: u32 = 0x2;
pub const IPCFP_SHARDED_UNION_FULL: u32 = 0x4;
pub const IPCFP_WITNESS_BY_REFERENCE: u32 = 0x8;
pub const IPCFP_RESULT_JSON: u32 = 0x10;
pub const IPCFP_ACTOR_WITH_CODE: u32 = 0x20;
pub const IPCFP_MESSAGE_WITH_BODY: u32 = 0x40;
pub const IPCFP_COMM_ID_BYTES: usize = 128;

#[repr(C)] pub struct ipcfp_store { _p: [u8; 0] }
#[repr(C)] pub struct ipcfp_tipset { _p: [u8; 0] }
#[repr(C)] pub struct ipcfp_comm { _p: [u8; 0] }

#[repr(C)]
pub struct ipcfp_tipset_desc {
    pub parent_epoch: i64,
    pub child_epoch: i64,
    pub n_parents: u32,
    pub parent_cids: *const u8,
    pub parent_txmeta_cids: *const u8,
    pub child_cid: *const u8,
    pub receipts_root: *const u8,
    pub child_parent_state_root: *const u8,
    pub n_receipts: u64,
    pub events_roots: *const u8,
    pub has_events_root: *const u8,
}
#[repr(C)]
pub struct ipcfp_event_spec { pub event_signature: *const c_char, pub topic_1: *const c_char, pub has_actor_id_filter: u8, pub actor_id_filter: u64 }
pub const IPCFP_LOG_FILTER_MAX_VALUES: u32 = 65536;
pub const IPCFP_LOG_FILTER_MAX_EMITTERS: u32 = 65536;
#[repr(C)]
pub struct ipcfp_log_filter { pub n_emitters: u64, pub emitters: *const u64, pub n_positions: u32, pub _pad: u32, pub n_values: [u64; 4],
                              pub values: [*const u8; 4] }
#[repr(C)]
pub struct ipcfp_storage_spec { pub actor_id: u64, pub slot: [u8; 32] }
#[repr(C)]
pub struct ipcfp_witness { pub n_blocks: u64, pub cids: *const u8, pub offsets: *const u64, pub lengths: *const u32, pub blob: *const u8, pub blob_size: u64 }
#[repr(C)]
pub struct ipcfp_event_proof {
    pub exec_index: u64, pub event_index: u64, pub emitter: u64, pub n_topics: u32, pub data_len: u32,
    pub data_off: u64, pub topics_off: u64, pub message_cid: [u8; IPCFP_CID_LEN], pub _pad: [u8; 2],
}
#[repr(C)]
pub struct ipcfp_event_result {
    pub n_matching: u64, pub matching_indices: *const u64, pub n_proofs: u64, pub proofs: *const ipcfp_event_proof,
    pub data_blob: *const u8, pub data_blob_size: u64, pub witness: ipcfp_witness, pub n_exec: u64,
    pub ms_total: f32, pub ms_pass1: f32, pub ms_pass2: f32, pub ms_txamt: f32, pub ms_witness: f32,
    pub pass1_bytes: u64, pub pass1_nodes: u64,
    pub shard_exec_dev: *const c_void, pub shard_exec_count: u64, pub shard_raw_total: u64,
    pub union_cids_dev: *const c_void, pub n_union_cids: u64, pub union_cids: *const u8, pub total_matching: u64, pub total_proofs: u64,
    pub ms_exchange: f32, pub ms_fetch: f32, pub ms_union: f32, pub _pad0: f32,
    pub union_part_first: u64, pub n_union_part: u64,
    pub json: *const c_char, pub json_len: u64, pub ms_json: f32, pub _pad1: f32,
}
#[repr(C)]
pub struct ipcfp_storage_proof {
    pub actor_id: u64, pub actor_state_cid: [u8; IPCFP_CID_LEN], pub storage_root: [u8; IPCFP_CID_LEN],
    pub slot: [u8; 32], pub value: [u8; 32], pub found: u8, pub _pad: [u8; 3], pub raw_len: u32,
}
#[repr(C)]
pub struct ipcfp_storage_result {
    pub n_proofs: u64, pub proofs: *const ipcfp_storage_proof, pub witness: ipcfp_witness,
    pub spec_witness_offsets: *const u64, pub spec_witness_index: *const u32, pub ms_total: f32,
}
#[repr(C)]
pub struct ipcfp_slot_result { pub n: u64, pub found: *const u8, pub raw_len: *const u32, pub values: *const u8, pub witness: ipcfp_witness, pub ms_total: f32, pub ms_lookup: f32,
                                pub lookup_nodes: u64, pub lookup_bytes: u64 }
#[repr(C)]
pub struct ipcfp_parsed_bundle { pub tipset: ipcfp_tipset_desc, pub n_storage_proofs: u64, pub storage_proofs: *const ipcfp_storage_proof,
                                 pub n_event_proofs: u64, pub event_proofs: *const ipcfp_event_proof, pub data_blob: *const u8, pub data_blob_size: u64,
                                 pub witness: ipcfp_witness }
pub type ipcfp_trusted_parent_ts_fn = Option<unsafe extern "C" fn(ctx: *mut c_void, parent_epoch: i64, parent_cids: *const u8, n_parents: u32) -> c_int>;
pub type ipcfp_trusted_child_header_fn = Option<unsafe extern "C" fn(ctx: *mut c_void, child_epoch: i64, child_cid: *const u8) -> c_int>;
#[repr(C)]
pub struct ipcfp_bundle_verdict { pub tipset: ipcfp_tipset_desc, pub n_storage_proofs: u64, pub storage_proofs: *const ipcfp_storage_proof,
                                  pub storage_results: *const u8, pub n_event_proofs: u64, pub event_proofs: *const ipcfp_event_proof,
                                  pub event_results: *const u8, pub data_blob: *const u8, pub data_blob_size: u64, pub n_blocks: u64,
                                  pub witness_bytes: u64, pub parsed_on_device: u32, pub ms_total: f32, pub ms_parse: f32, pub ms_store: f32,
                                  pub ms_verify: f32, pub _pad: u32 }
#[repr(C)]
pub struct ipcfp_parsed_tipset { pub desc: ipcfp_tipset_desc }
#[repr(C)]
pub struct ipcfp_tipset_info { pub desc: ipcfp_tipset_desc, pub parsed_on_device: u32, pub ms_parse: f32, pub ms_kernels: f32,
                               pub _pad: u32 }
#[repr(C)]
pub struct ipcfp_parsed_blocks { pub blocks: ipcfp_witness }
#[repr(C)]
pub struct ipcfp_store_json_info { pub parsed_on_device: u32, pub ms_parse: f32, pub ms_kernels: f32, pub _pad: u32 }
// Storage paths (ipcfp.h, "Storage paths")
pub const IPCFP_PATH_MAX_PATHS: u32 = 65536;
pub const IPCFP_PATH_MAX_STEPS: u32 = 32;
pub const IPCFP_PATH_MAX_KEY: u32 = 1024;
pub const IPCFP_PATH_MAX_WORDS: u32 = 256;
pub const IPCFP_PATH_MAX_BYTES: u32 = 4096;
pub const IPCFP_PATH_MAPPING: u32 = 0;
pub const IPCFP_PATH_ARRAY: u32 = 1;
pub const IPCFP_PATH_STATIC: u32 = 2;
pub const IPCFP_PATH_FIELD: u32 = 3;
pub const IPCFP_PATH_WORDS: u32 = 0;
pub const IPCFP_PATH_BYTES: u32 = 1;
pub const IPCFP_PATH_OK: u32 = 0;
pub const IPCFP_PATH_INDEX_OUT_OF_RANGE: u32 = 1;
pub const IPCFP_PATH_BAD_BYTES: u32 = 2;
pub const IPCFP_PATH_TOO_LONG: u32 = 3;
#[repr(C)]
pub struct ipcfp_path_step { pub op: u32, pub key_len: u32, pub key: *const u8, pub index: u64, pub elem_slots: u32, pub elem_bytes: u32 }
#[repr(C)]
pub struct ipcfp_storage_path { pub actor_id: u64, pub base_slot: [u8; 32], pub n_steps: u32, pub kind: u32, pub steps: *const ipcfp_path_step,
                                pub n_words: u32, pub _pad: u32 }
#[repr(C)]
pub struct ipcfp_path_value { pub status: u32, pub valid: u32, pub slot: [u8; 32], pub byte_offset: u32, pub _pad: u32, pub first_spec: u64,
                              pub n_specs: u64, pub value_off: u64, pub value_len: u64 }
#[repr(C)]
pub struct ipcfp_path_result { pub n_paths: u64, pub paths: *const ipcfp_path_value, pub n_specs: u64, pub specs: *const ipcfp_storage_spec,
                               pub value_blob: *const u8, pub value_blob_size: u64, pub storage: *mut ipcfp_storage_result, pub ms_total: f32,
                               pub ms_slots: f32, pub ms_wave1: f32, pub ms_wave2: f32, pub ms_witness: f32, pub host_syncs: u32 }
#[repr(C)]
pub struct ipcfp_fetch_plan { pub n_missing: u64, pub cids: *const u8, pub n_needed: u64, pub n_levels: u32, pub ms_total: f32 }
pub const IPCFP_ADDRESS_MAX: usize = 65;
#[repr(C)]
#[derive(Clone, Copy)]
pub struct ipcfp_address { pub len: u8, pub bytes: [u8; IPCFP_ADDRESS_MAX] }
#[repr(C)]
pub struct ipcfp_resolve_result { pub n: u64, pub actor_ids: *const u64, pub status: *const ipcfp_status, pub init_status: ipcfp_status, pub _pad: u32,
                                  pub n_missing: u64, pub missing_cids: *const u8, pub witness: ipcfp_witness, pub ms_total: f32, pub ms_lookup: f32 }
pub const IPCFP_ACTOR_MAX: u64 = 65536;
pub const IPCFP_ACTOR_FOUND: u32 = 0;
pub const IPCFP_ACTOR_NO_ADDRESS: u32 = 1;
pub const IPCFP_ACTOR_NO_ACTOR: u32 = 2;
#[repr(C)]
#[derive(Clone, Copy)]
pub struct ipcfp_actor_proof { pub actor_id: u64, pub sequence: u64, pub evm_nonce: u64, pub code_off: u64, pub code_len: u64, pub status: u32,
                               pub balance_negative: u8, pub has_delegated: u8, pub is_evm: u8, pub _pad0: u8, pub balance: [u8; 32],
                               pub code: [u8; 38], pub head: [u8; 38], pub bytecode_cid: [u8; 38], pub contract_state: [u8; 38],
                               pub bytecode_hash: [u8; 32], pub address: ipcfp_address, pub delegated: ipcfp_address, pub _pad1: [u8; 4] }
#[repr(C)]
pub struct ipcfp_actor_result { pub n_proofs: u64, pub proofs: *const ipcfp_actor_proof, pub witness: ipcfp_witness,
                                pub proof_witness_offsets: *const u64, pub proof_witness_index: *const u32, pub code_blob: *const u8,
                                pub code_blob_size: u64, pub ms_total: f32, pub ms_init: f32, pub ms_walk: f32, pub ms_code: f32, pub ms_witness: f32,
                                pub host_syncs: u32 }
pub const IPCFP_MESSAGE_EXECUTED: u32 = 0;
pub const IPCFP_MESSAGE_NOT_EXECUTED: u32 = 1;
pub const IPCFP_MESSAGE_NO_RECEIPT: u32 = 2;
#[repr(C)]
#[derive(Clone, Copy)]
pub struct ipcfp_message_proof { pub exec_index: u64, pub gas_used: u64, pub return_off: u64, pub return_len: u64, pub version: u64, pub sequence: u64,
                                 pub gas_limit: u64, pub method_num: u64, pub params_off: u64, pub params_len: u64, pub status: u32, pub exit_code: u32,
                                 pub has_events_root: u8, pub has_body: u8, pub sig_type: u8, pub value_negative: u8, pub gas_fee_cap_negative: u8,
                                 pub gas_premium_negative: u8, pub _pad0: [u8; 2], pub value: [u8; 32], pub gas_fee_cap: [u8; 32],
                                 pub gas_premium: [u8; 32], pub message_cid: [u8; 38], pub events_root: [u8; 38], pub to: ipcfp_address,
                                 pub from: ipcfp_address }
#[repr(C)]
pub struct ipcfp_message_result { pub n_proofs: u64, pub proofs: *const ipcfp_message_proof, pub data_blob: *const u8, pub data_blob_size: u64,
                                  pub witness: ipcfp_witness, pub n_exec: u64, pub ms_total: f32, pub ms_exec_order: f32, pub ms_walk: f32,
                                  pub ms_gather: f32, pub ms_witness: f32, pub host_syncs: u32 }
#[repr(C)]
pub struct ipcfp_bundle { pub storage: *mut ipcfp_storage_result, pub n_event_results: u64, pub events: *mut *mut ipcfp_event_result, pub witness: ipcfp_witness,
                          pub json: *const c_char, pub json_len: u64, pub ms_total: f32, pub ms_json: f32 }

extern "C" {
    pub fn ipcfp_last_error() -> *const c_char;
    pub fn ipcfp_last_error_index() -> u64;
    pub fn ipcfp_version() -> *const c_char;
    pub fn ipcfp_kernel_launch_count() -> u64;
    pub fn ipcfp_host_alloc(bytes: usize, out: *mut *mut c_void) -> ipcfp_status;
    pub fn ipcfp_host_free(p: *mut c_void);

    pub fn ipcfp_store_create(cids: *const u8, offsets: *const u64, lengths: *const u32, blob: *const u8, blob_size: u64,
                              n_blocks: u64, device: c_int, flags: u32, out: *mut *mut ipcfp_store) -> ipcfp_status;
    pub fn ipcfp_store_destroy(s: *mut ipcfp_store);
    pub fn ipcfp_store_n_blocks(s: *const ipcfp_store) -> u64;
    pub fn ipcfp_store_get(s: *mut ipcfp_store, cid: *const u8, buf: *mut u8, cap: u32, len: *mut u32, found: *mut c_int) -> ipcfp_status;
    pub fn ipcfp_store_has(s: *mut ipcfp_store, cid: *const u8, found: *mut c_int) -> ipcfp_status;
    pub fn ipcfp_store_first_bad_block(s: *const ipcfp_store) -> u64;
    pub fn ipcfp_store_stream(s: *mut ipcfp_store) -> *mut c_void;

    pub fn ipcfp_blake2b256_batch(blob: *const u8, blob_size: u64, offsets: *const u64, lengths: *const u32, n: u64, device: c_int, out: *mut u8) -> ipcfp_status;
    pub fn ipcfp_keccak256_batch(blob: *const u8, blob_size: u64, offsets: *const u64, lengths: *const u32, n: u64, device: c_int, out: *mut u8) -> ipcfp_status;
    pub fn ipcfp_sha256_batch(blob: *const u8, blob_size: u64, offsets: *const u64, lengths: *const u32, n: u64, device: c_int, out: *mut u8) -> ipcfp_status;
    pub fn ipcfp_compute_mapping_slots(keys32: *const u8, slot_indices: *const u64, n: u64, device: c_int, out: *mut u8) -> ipcfp_status;

    pub fn ipcfp_generate_event_proof(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, spec: *const ipcfp_event_spec, flags: u32,
                                      out: *mut *mut ipcfp_event_result) -> ipcfp_status;
    pub fn ipcfp_event_result_free(r: *mut ipcfp_event_result);
    pub fn ipcfp_tipset_upload(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, out: *mut *mut ipcfp_tipset) -> ipcfp_status;
    pub fn ipcfp_tipset_free(t: *mut ipcfp_tipset);
    pub fn ipcfp_tipset_desc_from_json(parent: *const c_char, parent_len: u64, child: *const c_char, child_len: u64, receipts: *const c_char,
                                       receipts_len: u64, out: *mut *mut ipcfp_parsed_tipset) -> ipcfp_status;
    pub fn ipcfp_parsed_tipset_free(p: *mut ipcfp_parsed_tipset);
    pub fn ipcfp_tipset_upload_json(s: *mut ipcfp_store, parent: *const c_char, parent_len: u64, child: *const c_char, child_len: u64,
                                    receipts: *const c_char, receipts_len: u64, out: *mut *mut ipcfp_tipset) -> ipcfp_status;
    pub fn ipcfp_tipset_describe(t: *mut ipcfp_tipset, with_events_roots: c_int, out: *mut ipcfp_tipset_info) -> ipcfp_status;
    pub fn ipcfp_blocks_from_rpc_json(cids: *const u8, n_blocks: u64, texts: *const *const c_char, text_lens: *const u64, n_texts: u64,
                                      out: *mut *mut ipcfp_parsed_blocks) -> ipcfp_status;
    pub fn ipcfp_parsed_blocks_free(p: *mut ipcfp_parsed_blocks);
    pub fn ipcfp_store_create_rpc_json(cids: *const u8, n_blocks: u64, texts: *const *const c_char, text_lens: *const u64, n_texts: u64,
                                       device: c_int, flags: u32, out: *mut *mut ipcfp_store, info: *mut ipcfp_store_json_info) -> ipcfp_status;
    pub fn ipcfp_blocks_from_car(car: *const u8, len: u64, out: *mut *mut ipcfp_parsed_blocks) -> ipcfp_status;
    pub fn ipcfp_store_create_car(car: *const u8, len: u64, device: c_int, flags: u32, out: *mut *mut ipcfp_store,
                                  info: *mut ipcfp_store_json_info) -> ipcfp_status;
    pub fn ipcfp_generate_event_proof_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, spec: *const ipcfp_event_spec, flags: u32,
                                               out: *mut *mut ipcfp_event_result) -> ipcfp_status;
    pub fn ipcfp_generate_log_proof_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, filter: *const ipcfp_log_filter, flags: u32,
                                             out: *mut *mut ipcfp_event_result) -> ipcfp_status;
    pub fn ipcfp_generate_log_proof(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, filter: *const ipcfp_log_filter, flags: u32,
                                    out: *mut *mut ipcfp_event_result) -> ipcfp_status;
    pub fn ipcfp_generate_event_proof_shard(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, spec: *const ipcfp_event_spec, lo: u64, hi: u64,
                                            world_size: u32, rank: u32, flags: u32, out: *mut *mut ipcfp_event_result) -> ipcfp_status;
    pub fn ipcfp_generate_event_proof_shard_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, spec: *const ipcfp_event_spec, lo: u64, hi: u64,
                                                     world_size: u32, rank: u32, flags: u32, out: *mut *mut ipcfp_event_result) -> ipcfp_status;

    pub fn ipcfp_read_storage_slots(s: *mut ipcfp_store, contract_state_root: *const u8, slots: *const u8, k: u64, out: *mut *mut ipcfp_slot_result) -> ipcfp_status;
    pub fn ipcfp_slot_result_free(r: *mut ipcfp_slot_result);
    pub fn ipcfp_generate_storage_proofs(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, specs: *const ipcfp_storage_spec, n_specs: u64,
                                         out: *mut *mut ipcfp_storage_result) -> ipcfp_status;
    pub fn ipcfp_storage_result_free(r: *mut ipcfp_storage_result);
    pub fn ipcfp_generate_storage_path_proofs_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, paths: *const ipcfp_storage_path, n: u64,
                                                       flags: u32, out: *mut *mut ipcfp_path_result) -> ipcfp_status;
    pub fn ipcfp_plan_fetch_storage_paths_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, paths: *const ipcfp_storage_path, n: u64,
                                                   flags: u32, out: *mut *mut ipcfp_fetch_plan) -> ipcfp_status;
    pub fn ipcfp_verify_storage_paths(witness_store: *mut ipcfp_store, t: *const ipcfp_tipset_desc, proofs: *const ipcfp_storage_proof, n_proofs: u64,
                                      paths: *const ipcfp_storage_path, n_paths: u64, out: *mut *mut ipcfp_path_result) -> ipcfp_status;
    pub fn ipcfp_path_result_free(r: *mut ipcfp_path_result);
    pub fn ipcfp_generate_proof_bundle(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, sspecs: *const ipcfp_storage_spec, n_sspecs: u64,
                                       especs: *const ipcfp_event_spec, n_especs: u64, out: *mut *mut ipcfp_bundle) -> ipcfp_status;
    pub fn ipcfp_generate_proof_bundle_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, sspecs: *const ipcfp_storage_spec, n_sspecs: u64,
                                                especs: *const ipcfp_event_spec, n_especs: u64, flags: u32, out: *mut *mut ipcfp_bundle) -> ipcfp_status;
    pub fn ipcfp_generate_log_bundle_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, sspecs: *const ipcfp_storage_spec, n_sspecs: u64,
                                              filters: *const ipcfp_log_filter, n_filters: u64, flags: u32, out: *mut *mut ipcfp_bundle) -> ipcfp_status;
    pub fn ipcfp_generate_log_bundle(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, sspecs: *const ipcfp_storage_spec, n_sspecs: u64,
                                     filters: *const ipcfp_log_filter, n_filters: u64, flags: u32, out: *mut *mut ipcfp_bundle) -> ipcfp_status;
    pub fn ipcfp_bundle_free(b: *mut ipcfp_bundle);
    pub fn ipcfp_plan_fetch_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, sspecs: *const ipcfp_storage_spec, n_sspecs: u64,
                                     especs: *const ipcfp_event_spec, n_especs: u64, flags: u32, out: *mut *mut ipcfp_fetch_plan) -> ipcfp_status;
    pub fn ipcfp_plan_fetch(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, sspecs: *const ipcfp_storage_spec, n_sspecs: u64,
                            especs: *const ipcfp_event_spec, n_especs: u64, flags: u32, out: *mut *mut ipcfp_fetch_plan) -> ipcfp_status;
    pub fn ipcfp_generate_message_log_proof_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, message_cids: *const u8, n: u64,
                                                     filter: *const ipcfp_log_filter, flags: u32, exec_indices: *mut u64,
                                                     out: *mut *mut ipcfp_event_result) -> ipcfp_status;
    pub fn ipcfp_generate_message_log_proof(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, message_cids: *const u8, n: u64,
                                            filter: *const ipcfp_log_filter, flags: u32, exec_indices: *mut u64,
                                            out: *mut *mut ipcfp_event_result) -> ipcfp_status;
    pub fn ipcfp_plan_fetch_message_log_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, message_cids: *const u8, n: u64,
                                                 filter: *const ipcfp_log_filter, flags: u32, out: *mut *mut ipcfp_fetch_plan) -> ipcfp_status;
    pub fn ipcfp_plan_fetch_log_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, filter: *const ipcfp_log_filter, flags: u32,
                                         out: *mut *mut ipcfp_fetch_plan) -> ipcfp_status;
    pub fn ipcfp_plan_fetch_log_bundle_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, sspecs: *const ipcfp_storage_spec, n_sspecs: u64,
                                                filters: *const ipcfp_log_filter, n_filters: u64, flags: u32, out: *mut *mut ipcfp_fetch_plan) -> ipcfp_status;
    pub fn ipcfp_fetch_plan_free(p: *mut ipcfp_fetch_plan);
    pub fn ipcfp_fetch_plan_to_rpc_json(p: *const ipcfp_fetch_plan, first_id: u64, out: *mut *mut c_char, out_len: *mut u64) -> ipcfp_status;
    pub fn ipcfp_resolve_addresses(s: *mut ipcfp_store, state_root: *const u8, addrs: *const ipcfp_address, n: u64,
                                   out: *mut *mut ipcfp_resolve_result) -> ipcfp_status;
    pub fn ipcfp_resolve_result_free(r: *mut ipcfp_resolve_result);
    pub fn ipcfp_address_parse(text: *const c_char, len: u64, out: *mut ipcfp_address) -> ipcfp_status;
    pub fn ipcfp_address_from_eth(eth: *const u8, out: *mut ipcfp_address) -> ipcfp_status;
    pub fn ipcfp_generate_actor_proofs_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, addrs: *const ipcfp_address, n: u64,
                                                evm_code_cids: *const u8, n_evm: u64, flags: u32, out: *mut *mut ipcfp_actor_result) -> ipcfp_status;
    pub fn ipcfp_generate_actor_proofs(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, addrs: *const ipcfp_address, n: u64,
                                       evm_code_cids: *const u8, n_evm: u64, flags: u32, out: *mut *mut ipcfp_actor_result) -> ipcfp_status;
    pub fn ipcfp_actor_result_free(r: *mut ipcfp_actor_result);
    pub fn ipcfp_plan_fetch_actor_proofs_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, addrs: *const ipcfp_address, n: u64,
                                                  evm_code_cids: *const u8, n_evm: u64, flags: u32, out: *mut *mut ipcfp_fetch_plan) -> ipcfp_status;
    pub fn ipcfp_verify_actor_proofs(witness_store: *mut ipcfp_store, t: *const ipcfp_tipset_desc, proofs: *const ipcfp_actor_proof, n: u64,
                                     evm_code_cids: *const u8, n_evm: u64, flags: u32, results: *mut u8) -> ipcfp_status;
    pub fn ipcfp_generate_message_proofs_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, message_cids: *const u8, n: u64, flags: u32,
                                                  out: *mut *mut ipcfp_message_result) -> ipcfp_status;
    pub fn ipcfp_generate_message_proofs(s: *mut ipcfp_store, t: *const ipcfp_tipset_desc, message_cids: *const u8, n: u64, flags: u32,
                                         out: *mut *mut ipcfp_message_result) -> ipcfp_status;
    pub fn ipcfp_message_result_free(r: *mut ipcfp_message_result);
    pub fn ipcfp_plan_fetch_message_proofs_resident(s: *mut ipcfp_store, t: *mut ipcfp_tipset, message_cids: *const u8, n: u64, flags: u32,
                                                    out: *mut *mut ipcfp_fetch_plan) -> ipcfp_status;
    pub fn ipcfp_verify_message_proofs(witness_store: *mut ipcfp_store, t: *const ipcfp_tipset_desc, proofs: *const ipcfp_message_proof, n: u64,
                                       data_blob: *const u8, data_blob_size: u64, flags: u32, results: *mut u8) -> ipcfp_status;

    pub fn ipcfp_bundle_to_json(b: *const ipcfp_bundle, t: *const ipcfp_tipset_desc, out: *mut *mut c_char, out_len: *mut u64) -> ipcfp_status;
    pub fn ipcfp_event_result_to_json(r: *const ipcfp_event_result, t: *const ipcfp_tipset_desc, out: *mut *mut c_char, out_len: *mut u64) -> ipcfp_status;
    pub fn ipcfp_json_free(p: *mut c_char);
    pub fn ipcfp_bundle_from_json(json: *const c_char, len: u64, out: *mut *mut ipcfp_parsed_bundle) -> ipcfp_status;
    pub fn ipcfp_parsed_bundle_free(b: *mut ipcfp_parsed_bundle);
    pub fn ipcfp_verify_event_proofs(witness_store: *mut ipcfp_store, t: *const ipcfp_tipset_desc, proofs: *const ipcfp_event_proof, n_proofs: u64,
                                     data_blob: *const u8, data_blob_size: u64, filter: *const ipcfp_event_spec, results: *mut u8) -> ipcfp_status;
    pub fn ipcfp_verify_event_proofs_log(witness_store: *mut ipcfp_store, t: *const ipcfp_tipset_desc, proofs: *const ipcfp_event_proof, n_proofs: u64,
                                         data_blob: *const u8, data_blob_size: u64, filter: *const ipcfp_log_filter, results: *mut u8) -> ipcfp_status;
    pub fn ipcfp_verify_event_proofs_any(witness_store: *mut ipcfp_store, t: *const ipcfp_tipset_desc, proofs: *const ipcfp_event_proof, n_proofs: u64,
                                         data_blob: *const u8, data_blob_size: u64, filters: *const ipcfp_log_filter, n_filters: u64,
                                         results: *mut u8) -> ipcfp_status;
    pub fn ipcfp_verify_storage_proofs(witness_store: *mut ipcfp_store, t: *const ipcfp_tipset_desc, proofs: *const ipcfp_storage_proof, n_proofs: u64,
                                       results: *mut u8) -> ipcfp_status;
    pub fn ipcfp_verify_bundle_json(json: *const c_char, len: u64, device: c_int, trusted_parent: ipcfp_trusted_parent_ts_fn,
                                    trusted_child: ipcfp_trusted_child_header_fn, trust_ctx: *mut c_void, filter: *const ipcfp_event_spec,
                                    out: *mut *mut ipcfp_bundle_verdict) -> ipcfp_status;
    pub fn ipcfp_verify_bundle_json_any(json: *const c_char, len: u64, device: c_int, trusted_parent: ipcfp_trusted_parent_ts_fn,
                                        trusted_child: ipcfp_trusted_child_header_fn, trust_ctx: *mut c_void, filters: *const ipcfp_log_filter,
                                        n_filters: u64, out: *mut *mut ipcfp_bundle_verdict) -> ipcfp_status;
    pub fn ipcfp_bundle_verdict_free(v: *mut ipcfp_bundle_verdict);
    pub fn ipcfp_comm_unique_id(id: *mut u8) -> ipcfp_status;
    pub fn ipcfp_comm_init(id: *const u8, world_size: u32, rank: u32, device: c_int, out: *mut *mut ipcfp_comm) -> ipcfp_status;
    pub fn ipcfp_comm_destroy(c: *mut ipcfp_comm);
    pub fn ipcfp_generate_event_proof_sharded(c: *mut ipcfp_comm, s: *mut ipcfp_store, t: *mut ipcfp_tipset, spec: *const ipcfp_event_spec,
                                              bounds: *const u64, flags: u32, out: *mut *mut ipcfp_event_result) -> ipcfp_status;
}
