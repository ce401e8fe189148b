/* ipcfp.h — C ABI of the H100-native witness-generation engine.
 *
 * Drop-in boundary for ONE path of consensus-shipyard/ipc-filecoin-proofs: the two-pass
 * receipt/event AMT scan and the HAMT storage-slot lookup. Every entry point cites the
 * reference interface it replaces (paths relative to the reference repo root). The header
 * is bindgen-ready: plain pointers and sizes, POD structs, no C++ or torch types.
 *
 * All compute behind these calls runs in hand-written sm_90a CUDA kernels. There is no
 * CPU implementation in this library: without a CUDA device every call fails with
 * IPCFP_ERR_NO_DEVICE.
 *
 * CIDs are 38-byte binary CIDv1 (`01 | codec | multihash code | 20 | digest[32]`; the
 * Filecoin chain form is `01 71 a0 e4 02 20 <blake2b-256>`), exactly the bytes behind the
 * strings `Cid::try_from(&str)` parses at src/proofs/common/witness.rs:60-63.
 *
 * Ownership: inputs are borrowed for the duration of the call. Outputs are owned by the
 * returned result object and released with the matching ipcfp_*_free. A store handle is
 * bound to one CUDA device; calls on one handle must be serialised by the caller.
 */
#ifndef IPCFP_H
#define IPCFP_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IPCFP_CID_LEN 38

typedef int32_t ipcfp_status;
enum {
    IPCFP_OK = 0,
    IPCFP_ERR_INVALID_ARG = -1,
    IPCFP_ERR_MISSING_BLOCK = -2,   /* anyhow!("missing ...") at witness.rs:47-50, storage/decode.rs:41-43, events/generator.rs:159-161 */
    IPCFP_ERR_DECODE = -3,          /* any serde / AMT / HAMT decode error bubbled by `?`                */
    IPCFP_ERR_CID_MISMATCH = -4,    /* IPCFP_STORE_VERIFY_CIDS: blake2b-256(block) != digest in its CID   */
    IPCFP_ERR_MISSING_EXEC = -5,    /* "Missing message at index" events/generator.rs:244-246             */
    IPCFP_ERR_CUDA = -6,
    IPCFP_ERR_NCCL = -7,
    IPCFP_ERR_STATE_ROOT_MISMATCH = -8, /* "ParentStateRoot mismatch" storage/generator.rs:93-99         */
    IPCFP_ERR_ACTOR_NOT_FOUND = -9,     /* "actor not found" common/decode.rs:39                         */
    IPCFP_ERR_NO_DEVICE = -10,
    IPCFP_ERR_UNSUPPORTED = -11
};

/* Thread-local description of the last failure on this thread ("" if none). */
const char* ipcfp_last_error(void);
/* Index attached to the last failure (receipt index / spec index / block index), or UINT64_MAX. */
uint64_t ipcfp_last_error_index(void);
/* Library version string and the list of kernels compiled in. */
const char* ipcfp_version(void);
/* Number of kernel launches issued by this library on the calling thread since load. */
uint64_t ipcfp_kernel_launch_count(void);

/* Pinned host memory for the flat block arrays (so ingest H2D copies run at PCIe rate). */
ipcfp_status ipcfp_host_alloc(size_t bytes, void** out);
void ipcfp_host_free(void* p);

/* ------------------------------------------------------------------------------------------
 * Block store — replaces the `fvm_ipld_blockstore::Blockstore` implementations the generators
 * are generic over (src/client/blockstore.rs:20-37, src/client/cached_blockstore.rs:53-85):
 * a device-resident arena of IPLD blocks with a CID hash index.
 * ------------------------------------------------------------------------------------------ */
typedef struct ipcfp_store ipcfp_store;

#define IPCFP_STORE_VERIFY_CIDS 0x1u /* Blake2b-256 every block on the GPU and compare with its CID */

/* cids: n*38 bytes; offsets[i]/lengths[i]: block i inside blob. Blocks are used in place at ANY offset / alignment
 * (every device read is an aligned load plus a byte shift). */
ipcfp_status ipcfp_store_create(const uint8_t* cids, const uint64_t* offsets, const uint32_t* lengths,
                                const uint8_t* blob, uint64_t blob_size, uint64_t n_blocks,
                                int device, uint32_t flags, ipcfp_store** out);
void ipcfp_store_destroy(ipcfp_store* s);
uint64_t ipcfp_store_n_blocks(const ipcfp_store* s);
/* Blockstore::get — copies the block into buf (cap bytes). *len receives the block length.
 * Unknown CID: returns IPCFP_OK with *found = 0 (the reference's Ok(None)). */
ipcfp_status ipcfp_store_get(ipcfp_store* s, const uint8_t cid[IPCFP_CID_LEN], uint8_t* buf, uint32_t cap,
                             uint32_t* len, int* found);
/* Blockstore::has */
ipcfp_status ipcfp_store_has(ipcfp_store* s, const uint8_t cid[IPCFP_CID_LEN], int* found);
/* Index of the first block whose CID digest did not match (after a CID_MISMATCH), else UINT64_MAX. */
uint64_t ipcfp_store_first_bad_block(const ipcfp_store* s);

/* ------------------------------------------------------------------------------------------
 * Batched hash primitives (unit parity of the kernels).
 * ------------------------------------------------------------------------------------------ */
/* out[i] = blake2b-256(blob[offsets[i] .. offsets[i]+lengths[i]))   (multihash-codetable Code::Blake2b256,
 * src/proofs/events/utils.rs:65) */
ipcfp_status ipcfp_blake2b256_batch(const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets,
                                    const uint32_t* lengths, uint64_t n, int device, uint8_t* out /* n*32 */);
/* keccak256 (src/proofs/common/evm.rs:62-69, :81-88) */
ipcfp_status ipcfp_keccak256_batch(const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets,
                                   const uint32_t* lengths, uint64_t n, int device, uint8_t* out /* n*32 */);
/* SHA-256 (fvm_ipld_hamt default key hasher) */
ipcfp_status ipcfp_sha256_batch(const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets,
                                const uint32_t* lengths, uint64_t n, int device, uint8_t* out /* n*32 */);
/* compute_mapping_slot(key, slot_index) = keccak256(key32 || u256_be(slot_index))
 * (src/proofs/storage/utils.rs:5-12), batched. */
ipcfp_status ipcfp_compute_mapping_slots(const uint8_t* keys32 /* n*32 */, const uint64_t* slot_indices, uint64_t n,
                                         int device, uint8_t* out /* n*32 */);

/* ------------------------------------------------------------------------------------------
 * Inputs that came over RPC in the reference (src/client/types.rs:13-58).
 * ------------------------------------------------------------------------------------------ */
typedef struct ipcfp_tipset_desc {
    int64_t parent_epoch;                  /* parent.height                                   */
    int64_t child_epoch;                   /* child.height                                    */
    uint32_t n_parents;                    /* parent.cids.len() == parent.blocks.len()        */
    const uint8_t* parent_cids;            /* n_parents*38: parent.cids                       */
    const uint8_t* parent_txmeta_cids;     /* n_parents*38: parent.blocks[i].messages         */
    const uint8_t* child_cid;              /* 38: child.cids[0]                               */
    const uint8_t* receipts_root;          /* 38: child.blocks[0].parent_message_receipts     */
    const uint8_t* child_parent_state_root;/* 38: child.blocks[0].parent_state_root (JSON)    */
    uint64_t n_receipts;                   /* ChainGetParentReceipts(child) length            */
    const uint8_t* events_roots;           /* n_receipts*38: ApiReceipt.events_root           */
    const uint8_t* has_events_root;        /* n_receipts: 0 = None                            */
} ipcfp_tipset_desc;

/* EventProofSpec (src/proofs/generator.rs:18-22) */
typedef struct ipcfp_event_spec {
    const char* event_signature; /* e.g. "NewTopDownMessage(bytes32,uint256)" → topic0 = keccak256 */
    const char* topic_1;         /* ASCII, right-padded to 32 bytes (evm.rs:72-78)                  */
    uint8_t has_actor_id_filter;
    uint64_t actor_id_filter;
} ipcfp_event_spec;

/* An eth_getLogs-style log filter: one predicate over the events extract_evm_log (common/evm.rs:13-59) accepts, with the topics and
 * the emitter the EventProof carries. Topic k of a log is its t(k+1) value (Case B) or bytes 32k..32k+32 of its `topics` blob (Case A,
 * which may hold zero or more than four topics). An event matches when all of these hold:
 *   - extract_evm_log returns Some for it;
 *   - n_emitters == 0, or EventData.emitter is one of emitters[];
 *   - the log has at least n_positions topics;
 *   - for every k < n_positions with n_values[k] > 0, topic k equals one of the 32-byte values[k][..], byte for byte.
 * Duplicates in a set are allowed. A position with n_values[k] == 0 is a wildcard; positions past 3 are never constrained.
 * Trailing wildcards count: n_positions plays the length of go-ethereum's `topics` list, whose filterLogs refuses logs with fewer
 * topics than the list has entries. {n_positions = 3, values = [{A}, {}, {}]} is `[A, null, null]` and needs three topics; a caller
 * who wants only the constrained positions to count sets n_positions to 1 + the highest constrained position ([A] needs one topic).
 * The spec {sig, t1, actor?} is the filter {emitters = [actor] or none, n_positions = 2, values = [{keccak256(sig)}, {ascii_to_bytes32(t1)}]}.
 * IPCFP_ERR_INVALID_ARG: n_positions > 4, n_values[k] > 0 for k >= n_positions, a NULL array with a nonzero count, more than
 * IPCFP_LOG_FILTER_MAX_VALUES values at a position or more than IPCFP_LOG_FILTER_MAX_EMITTERS emitters. Emitters are actor IDs:
 * resolve Ethereum addresses first (ipcfp_resolve_addresses). */
#define IPCFP_LOG_FILTER_MAX_VALUES 65536u
#define IPCFP_LOG_FILTER_MAX_EMITTERS 65536u
typedef struct ipcfp_log_filter {
    uint64_t n_emitters;          /* 0: any emitter; else EventData.emitter must be one of emitters[]        */
    const uint64_t* emitters;     /* actor IDs                                                                */
    uint32_t n_positions;         /* 0..4: an event needs at least this many topics                           */
    uint32_t _pad;
    uint64_t n_values[4];         /* per position; 0 = wildcard                                               */
    const uint8_t* values[4];     /* n_values[k] * 32 bytes; topic k must equal one of them, byte for byte     */
} ipcfp_log_filter;

/* StorageProofSpec (src/proofs/generator.rs:12-15) */
typedef struct ipcfp_storage_spec {
    uint64_t actor_id;
    uint8_t slot[32];
} ipcfp_storage_spec;

/* ------------------------------------------------------------------------------------------
 * Outputs.
 * ------------------------------------------------------------------------------------------ */
/* Vec<ProofBlock> in `Cid` Ord order (src/proofs/common/witness.rs:43-56, common/bundle.rs:11-18) */
typedef struct ipcfp_witness {
    uint64_t n_blocks;
    const uint8_t* cids;      /* n_blocks*38, sorted by (version, codec, multihash) */
    const uint64_t* offsets;  /* n_blocks: block i = blob[offsets[i] .. offsets[i]+lengths[i])   */
    const uint32_t* lengths;  /* n_blocks                                                        */
    const uint8_t* blob;      /* block bytes; blocks may sit in any order / with padding in here (pad bytes unspecified). NULL with IPCFP_WITNESS_BY_REFERENCE: offsets then index the blob given to ipcfp_store_create */
    uint64_t blob_size;
} ipcfp_witness;

/* EventProof + EventData (src/proofs/events/bundle.rs:6-23) minus the per-call constants
 * (epochs, parent tipset CIDs, child block CID) which the caller already holds. */
typedef struct ipcfp_event_proof {
    uint64_t exec_index;
    uint64_t event_index;
    uint64_t emitter;
    uint32_t n_topics;      /* ≤ 4 in Case B; Case A (`topics` key) may carry more — see data_off   */
    uint32_t data_len;
    uint64_t data_off;      /* into ipcfp_event_result.data_blob                                    */
    uint64_t topics_off;    /* into data_blob: n_topics*32 bytes                                    */
    uint8_t message_cid[IPCFP_CID_LEN];
    uint8_t _pad[2];
} ipcfp_event_proof;

typedef struct ipcfp_event_result {
    uint64_t n_matching;
    const uint64_t* matching_indices; /* pass-1 output (events/generator.rs:206-239), ascending */
    uint64_t n_proofs;
    const ipcfp_event_proof* proofs;  /* ordered by (exec_index, event_index)                  */
    const uint8_t* data_blob;
    uint64_t data_blob_size;
    ipcfp_witness witness;            /* EventProofBundle.blocks                                */
    uint64_t n_exec;                  /* length of the reconstructed execution order            */
    /* device-side timing of the last call, milliseconds (CUDA events on the engine stream) */
    float ms_total, ms_pass1, ms_pass2, ms_txamt, ms_witness;
    uint64_t pass1_bytes;             /* algorithmic bytes read by the pass-1 scan kernel       */
    uint64_t pass1_nodes;
    /* shard mode only (ipcfp_generate_event_proof_shard): this shard's slice of the concatenated message list,
     * in order, as 40-byte records {digest[32], prefix[6], 0, 0} in DEVICE memory (valid until the result is
     * freed; free results before destroying the store). proofs[].message_cid is left zero and n_exec is 0:
     * the execution order spans shards, and only ipcfp_generate_event_proof_sharded resolves it. */
    const void* shard_exec_dev;
    uint64_t shard_exec_count;
    uint64_t shard_raw_total;         /* total length of the concatenated message list (all shards) */
    /* ipcfp_generate_event_proof_sharded only: proofs[].message_cid and n_exec are final (resolved across shards inside the
     * call). The union of ALL shards' witness CID sets (the BTreeSet union of src/proofs/common/witness.rs:24-40) has
     * n_union_cids entries in `Cid` order and is left DISTRIBUTED: this rank holds entries [union_part_first, union_part_first +
     * n_union_part) — the CIDs whose first two digest bytes fall into its 1/world share of the 65 536 buckets — so the
     * concatenation of the ranks' parts in rank order is the whole sorted set. With IPCFP_SHARDED_UNION_FULL every rank holds the
     * whole set instead (union_part_first = 0, n_union_part = n_union_cids). union_cids_dev: DEVICE memory, n_union_part*38 bytes,
     * valid until the next sharded call on the same communicator; union_cids: the same on the host with
     * IPCFP_SHARDED_UNION_TO_HOST. total_matching / total_proofs: summed over all shards. */
    const void* union_cids_dev;
    uint64_t n_union_cids;
    const uint8_t* union_cids;
    uint64_t total_matching;
    uint64_t total_proofs;
    float ms_exchange, ms_fetch, ms_union; /* device time of the execution-order exchange (its own stream, under pass 1), the message-CID fetch, the witness union */
    float _pad0;
    uint64_t union_part_first;
    uint64_t n_union_part;
    /* IPCFP_RESULT_JSON only (NULL / 0 otherwise): the EventProofBundle as JSON, byte for byte what ipcfp_event_result_to_json renders
     * for the same call made without the flag. NUL-terminated, json_len bytes without the NUL, owned by the result. ms_json: device time
     * of the rendering and its copy to the host. */
    const char* json;
    uint64_t json_len;
    float ms_json;
    float _pad1;
} ipcfp_event_result;

typedef struct ipcfp_storage_proof {
    uint64_t actor_id;
    uint8_t actor_state_cid[IPCFP_CID_LEN];
    uint8_t storage_root[IPCFP_CID_LEN];
    uint8_t slot[32];
    uint8_t value[32];    /* left_pad_32(raw) (evm.rs:91-100); zero when absent */
    uint8_t found;        /* Hamt::get returned Some                            */
    uint8_t _pad[3];
    uint32_t raw_len;     /* length of the raw value                            */
} ipcfp_storage_proof;

typedef struct ipcfp_storage_result {
    uint64_t n_proofs;
    const ipcfp_storage_proof* proofs;
    ipcfp_witness witness;              /* union over all specs, sorted                          */
    const uint64_t* spec_witness_offsets; /* n_proofs+1                                          */
    const uint32_t* spec_witness_index;   /* per spec: indices into witness (its Vec<ProofBlock>) */
    float ms_total;
} ipcfp_storage_result;

typedef struct ipcfp_slot_result {
    uint64_t n;
    const uint8_t* found;      /* n                                        */
    const uint32_t* raw_len;   /* n                                        */
    const uint8_t* values;     /* n*32, left-padded                        */
    ipcfp_witness witness;     /* blocks touched by the lookups (recorder) */
    float ms_total;
    float ms_lookup;           /* device time of the lookup kernel alone (CUDA events on the engine stream)              */
    uint64_t lookup_nodes;     /* HAMT nodes decoded by the lookups                                                      */
    uint64_t lookup_bytes;     /* algorithmic bytes of the lookups: 32 per key + the bytes of every node on its path      */
} ipcfp_slot_result;

typedef struct ipcfp_bundle {
    ipcfp_storage_result* storage;  /* may be NULL */
    uint64_t n_event_results;
    ipcfp_event_result** events;    /* one per event spec */
    ipcfp_witness witness;          /* UnifiedProofBundle.blocks: BTreeSet<(Cid, data)> order */
    /* IPCFP_RESULT_JSON only (NULL / 0 otherwise): the UnifiedProofBundle as JSON, byte for byte what ipcfp_bundle_to_json renders for the
     * same call made without flags. NUL-terminated, json_len bytes without the NUL, owned by the bundle. */
    const char* json;
    uint64_t json_len;
    float ms_total;                 /* device time of the whole call, milliseconds (CUDA events on the store's stream)                */
    float ms_json;                  /* IPCFP_RESULT_JSON: device time of the rendering and its copy to the host; 0 otherwise          */
} ipcfp_bundle;

/* ------------------------------------------------------------------------------------------
 * Entry points.
 * ------------------------------------------------------------------------------------------ */
#define IPCFP_SCAN_SKIP_TX_AMTS 0x1u  /* find_matching_events only: no record_transaction_amts / base witness;
                                         execution order still built                                          */
#define IPCFP_SHARDED_UNION_TO_HOST 0x2u /* ipcfp_generate_event_proof_sharded: also copy this rank's part of the merged witness CID list to the host */
/* Witness BY REFERENCE (all ipcfp_generate_event_proof* calls): the result's witness carries no block bytes. witness.blob is NULL,
 * blob_size 0, and offsets[i] / lengths[i] locate block i inside the blob the STORE WAS CREATED FROM (the caller's own host array,
 * which it still holds): cids / offsets / lengths arrive as usual, in `Cid` order. Saves copying ≈ 51 MB per 1 M receipts that the
 * host already has; WitnessCollector::materialize (src/proofs/common/witness.rs:43-56) becomes a gather over the caller's blocks. */
#define IPCFP_WITNESS_BY_REFERENCE 0x8u
#define IPCFP_SHARDED_UNION_FULL 0x4u    /* … every rank receives the WHOLE merged list (all-gather + merge of `world` lists on every rank) instead of its partition */
/* JSON result (ipcfp_generate_event_proof, ipcfp_generate_event_proof_resident): the result also carries `json`, the serde_json text of
 * EventProofBundle (src/proofs/events/bundle.rs:5-30), rendered on the device — the text ipcfp_event_result_to_json gives for the same call
 * without the flag. Block bytes are read from the store itself, so IPCFP_RESULT_JSON | IPCFP_WITNESS_BY_REFERENCE is the combination for a
 * caller who wants the wire format: the text, without the ≈ 51 MB (per 1 M receipts) copy of the witness blob it already contains. With
 * IPCFP_SCAN_SKIP_TX_AMTS the text renders what that result holds. Costs one extra host synchronisation per call. Sharded calls
 * (ipcfp_generate_event_proof_shard*, _sharded) refuse the flag with IPCFP_ERR_UNSUPPORTED: a shard's result is not an EventProofBundle. */
#define IPCFP_RESULT_JSON 0x10u

/* generate_event_proof (src/proofs/events/generator.rs:60-107): base witness, message-AMT
 * recording, execution order, two-pass scan (find_matching_events :180-307), materialise. */
ipcfp_status ipcfp_generate_event_proof(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_spec* spec,
                                        uint32_t flags, ipcfp_event_result** out);
void ipcfp_event_result_free(ipcfp_event_result* r);

/* Device-resident tipset descriptor: upload once, scan many specs against it (the reference calls
 * generate_event_proof once per EventProofSpec with the same tipsets, proofs/generator.rs:58-78). */
typedef struct ipcfp_tipset ipcfp_tipset;
ipcfp_status ipcfp_tipset_upload(ipcfp_store* s, const ipcfp_tipset_desc* t, ipcfp_tipset** out);
void ipcfp_tipset_free(ipcfp_tipset* t);
ipcfp_status ipcfp_generate_event_proof_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_event_spec* spec, uint32_t flags,
                                                 ipcfp_event_result** out);
ipcfp_status ipcfp_generate_event_proof_shard_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_event_spec* spec, uint64_t lo,
                                                       uint64_t hi, uint32_t world_size, uint32_t rank, uint32_t flags,
                                                       ipcfp_event_result** out);
/* generate_event_proof with a log filter (ipcfp_log_filter above) in place of the spec's EventMatcher: the same call, flags
 * (IPCFP_WITNESS_BY_REFERENCE, IPCFP_RESULT_JSON, IPCFP_SCAN_SKIP_TX_AMTS) and result, one EventProofBundle. matching_indices are the
 * receipts with at least one matching event; proofs are in (exec_index, event_index) order; a failure is the one the reference's
 * generator with this predicate meets first. The proofs verify with ipcfp_verify_event_proofs (filter NULL or any spec they satisfy)
 * and with ipcfp_verify_event_proofs_log. ipcfp_generate_log_proof = ipcfp_tipset_upload, then the resident call. */
ipcfp_status ipcfp_generate_log_proof_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_log_filter* filter, uint32_t flags,
                                               ipcfp_event_result** out);
ipcfp_status ipcfp_generate_log_proof(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_log_filter* filter, uint32_t flags,
                                      ipcfp_event_result** out);
/* The logs of given messages: eth_getTransactionReceipt(tx).logs with a proof, for the messages a caller names by CID.
 * message_cids (n*38) are message CIDs as the parent blocks' message AMTs hold them: the CIDs reconstruct_execution_order yields (the
 * `Cid` fields of Filecoin.ChainGetParentMessages). filter may be NULL: every log extract_evm_log accepts.
 *   Selection  receipt i is selected when i < n_exec, i < n_receipts and exec[i] is one of message_cids.
 *   Result     what ipcfp_generate_log_proof_resident gives with the same filter (NULL: the all-wildcard filter) and flags
 *              (IPCFP_WITNESS_BY_REFERENCE, IPCFP_RESULT_JSON, IPCFP_SCAN_SKIP_TX_AMTS), with its receipt loop restricted to the selected
 *              receipts: matching_indices are the selected receipts with at least one matching event, proofs are in (exec_index,
 *              event_index) order, the witness is the base witness, the message AMTs and the receipts-AMT paths and events AMTs of the
 *              matching selected receipts. It is an ordinary EventProofBundle: ipcfp_verify_event_proofs* and ipcfp_verify_bundle_json
 *              accept it.
 *   Reads      the events-AMT blocks of unselected receipts are never read: a store that lacks them, or holds other bytes under their
 *              CIDs, gives the same result.
 *   Failures   a fault in the header, TxMeta or message AMTs as ipcfp_generate_log_proof_resident reports it; after that the first fault
 *              of the restricted loop over the selected receipts in ascending order (pass 1's events-AMT decode, then pass 2's reads),
 *              status and index as for the log-filter call.
 *   exec_indices (caller-allocated, n entries): exec_indices[j] is message j's position in the execution order, UINT64_MAX when the
 *              tipset did not execute it. Duplicates are allowed and reported per position; a CID the tipset did not execute is not an
 *              error. Written only when the call succeeds.
 *   Refusals   IPCFP_ERR_INVALID_ARG before any device work: message_cids or exec_indices NULL with n > 0, n > IPCFP_MESSAGE_MAX, an
 *              invalid filter (the rules of ipcfp_log_filter).
 * ipcfp_generate_message_log_proof = ipcfp_tipset_upload, then the resident call. */
#define IPCFP_MESSAGE_MAX 65536u
ipcfp_status ipcfp_generate_message_log_proof_resident(ipcfp_store* s, ipcfp_tipset* t, const uint8_t* message_cids /* n*38 */, uint64_t n,
                                                       const ipcfp_log_filter* filter /* may be NULL */, uint32_t flags, uint64_t* exec_indices,
                                                       ipcfp_event_result** out);
ipcfp_status ipcfp_generate_message_log_proof(ipcfp_store* s, const ipcfp_tipset_desc* t, const uint8_t* message_cids /* n*38 */, uint64_t n,
                                              const ipcfp_log_filter* filter /* may be NULL */, uint32_t flags, uint64_t* exec_indices,
                                              ipcfp_event_result** out);
/* The CUDA stream (cudaStream_t) all work of this store is issued on — for callers that time with
 * CUDA events or order their own device work after the engine's. */
void* ipcfp_store_stream(ipcfp_store* s);

/* ------------------------------------------------------------------------------------------
 * The tipset straight from the Lotus JSON-RPC results (src/client/types.rs:11-58): `parent` and `child` are the `result` values of
 * ChainGetTipSetByHeight (ApiTipset), `receipts` the `result` of ChainGetParentReceipts (Vec<ApiReceipt>) — the values only, not the
 * {"jsonrpc",…} envelope. Not NUL-terminated: each text is exactly its length in bytes.
 *
 * ipcfp_tipset_desc_from_json (host C++, no device) reads them as serde_json::from_str does, then builds the descriptor as
 * extract_child_info / collect_base_witness / find_matching_events do (events/generator.rs:112-145, :199-211):
 *   parent_epoch / child_epoch       parent.Height / child.Height
 *   parent_cids / parent_txmeta_cids parent.Cids[i]["/"] / parent.Blocks[i].Messages["/"]
 *   child_cid                        child.Cids[0]["/"]
 *   receipts_root                    child.Blocks[0].ParentMessageReceipts["/"]
 *   child_parent_state_root          child.Blocks[0].ParentStateRoot["/"]
 *   events_roots / has_events_root   receipts[i].EventsRoot["/"]; a missing or null EventsRoot is None (38 zero bytes, flag 0)
 * serde's derive rules: PascalCase keys, compared after unescaping; unknown keys are skipped (their values must still be valid JSON);
 * a repeated known key is an error. Required: ApiTipset {Cids, Blocks, Height}, ApiBlockHeader {Miner, Parents, ParentStateRoot,
 * ParentMessageReceipts, Messages, Height}, ApiReceipt {ExitCode (u32), Return (string, never decoded), GasUsed (u64)}, CIDMap {"/"}.
 * Integers are plain JSON integers in range ("-0", "1.0", "1e3" are not).
 * Documented deviation: serde's derive also accepts a struct written as a JSON array of its fields; Lotus never writes that form, and
 * it is refused here with IPCFP_ERR_UNSUPPORTED.
 * Statuses: malformed JSON, a wrong type, a missing or repeated field, an integer out of range, an invalid CID string →
 * IPCFP_ERR_INVALID_ARG; a valid CID that is not a 38-byte binary CID or not spelled "b…" (base32) → IPCFP_ERR_UNSUPPORTED (the rule of
 * ipcfp_bundle_from_json); an empty child Cids or Blocks → IPCFP_ERR_INVALID_ARG (the reference panics on the index); parent Cids and
 * Blocks of different lengths → IPCFP_ERR_UNSUPPORTED (the descriptor has one n_parents). The texts are checked in the order parent,
 * child, receipts; within an ApiTipset the structure first, then its CIDs. ipcfp_last_error_index() is the receipt's position for a
 * fault inside one element of the list (its JSON, its fields, its CID), UINT64_MAX for any other fault (the list's brackets and commas,
 * trailing bytes, the tipset texts). *out is released with ipcfp_parsed_tipset_free.
 * ------------------------------------------------------------------------------------------ */
typedef struct ipcfp_parsed_tipset {
    ipcfp_tipset_desc desc;   /* its arrays are owned by the object */
} ipcfp_parsed_tipset;
ipcfp_status ipcfp_tipset_desc_from_json(const char* parent, uint64_t parent_len, const char* child, uint64_t child_len, const char* receipts,
                                         uint64_t receipts_len, ipcfp_parsed_tipset** out);
void ipcfp_parsed_tipset_free(ipcfp_parsed_tipset* p);
/* The same texts straight to a device-resident tipset, for every _resident / _sharded call. The result, status and index are in every
 * case those of ipcfp_tipset_desc_from_json followed by ipcfp_tipset_upload. The two ApiTipset texts are read on the host. The receipt
 * list is parsed on the device when it is in canonical form — no whitespace, every element exactly
 *   {"ExitCode":<u32>,"Return":"<base64 characters and '='>","GasUsed":<u64>,"EventsRoot":null|{"/":"b<61 base32 characters>"}}
 * — with the events roots written straight into the tipset's device arrays. Any other text (whitespace, other key orders, unknown or
 * missing keys, escapes, other CID spellings, texts of 4 GiB or more, and every invalid text) goes through ipcfp_tipset_desc_from_json
 * instead. ipcfp_tipset_describe tells which path ran. */
ipcfp_status ipcfp_tipset_upload_json(ipcfp_store* s, const char* parent, uint64_t parent_len, const char* child, uint64_t child_len,
                                      const char* receipts, uint64_t receipts_len, ipcfp_tipset** out);
/* Read a resident tipset back: its descriptor — the host copies it holds; with with_events_roots != 0 also events_roots /
 * has_events_root, copied back from the device on the first such request (else those two are NULL) — which the host renderers and the
 * verifiers take, and how it was built. Pointers stay valid until ipcfp_tipset_free. */
typedef struct ipcfp_tipset_info {
    ipcfp_tipset_desc desc;
    uint32_t parsed_on_device;   /* 1: the receipt list was parsed on the device; 0: ipcfp_tipset_upload or the host parser     */
    float ms_parse;              /* ipcfp_tipset_upload_json: wall time of the receipt list's parse, its copy to the device included; 0 otherwise */
    float ms_kernels;            /* device parse only: time of its kernels (CUDA events on the store's stream); 0 otherwise     */
    uint32_t _pad;
} ipcfp_tipset_info;
ipcfp_status ipcfp_tipset_describe(ipcfp_tipset* t, int with_events_roots, ipcfp_tipset_info* out);

/* ------------------------------------------------------------------------------------------
 * The block store straight from Filecoin.ChainReadObj JSON-RPC responses (src/client/blockstore.rs:20-28). The caller fetches block i
 * as request i: Filecoin.ChainReadObj([{"/": <CID i>}]) with "id": i, and hands over the response texts exactly as received — each text
 * one JSON-RPC 2.0 response object or a batch (an array of them), not NUL-terminated, the responses in any order, spread over any number
 * of texts. Each response object has "jsonrpc":"2.0", "id" (a JSON integer, 0 <= id < n_blocks) and exactly one of "result" (a string:
 * standard base64 with padding and zero unused bits — the block's bytes) and "error" (any JSON value). Unknown members are skipped; a
 * repeated member is an error; JSON escapes in strings are undone before decoding.
 *
 * ipcfp_blocks_from_rpc_json (host C++, no device) returns the blocks in request order: blocks.cids is a copy of `cids` (n_blocks*38),
 * block i sits at blocks.offsets[i] (16-aligned, ascending), blocks.lengths[i] bytes long, in blocks.blob. Checks, in this order:
 *   1. texts in order, elements in order: a malformed text, an element that breaks the rules above, an id out of range or invalid base64 →
 *      IPCFP_ERR_INVALID_ARG, index = the element's position counted over all texts (a text that does not start with '[' after
 *      whitespace is one element); a fault outside every element (brackets, commas, trailing bytes) → index UINT64_MAX;
 *   2. the smallest id that does not appear exactly once → IPCFP_ERR_INVALID_ARG, index = that id;
 *   3. the smallest id answered with an "error" → IPCFP_ERR_MISSING_BLOCK, index = that id.
 * *out is released with ipcfp_parsed_blocks_free.
 * ------------------------------------------------------------------------------------------ */
typedef struct ipcfp_parsed_blocks {
    ipcfp_witness blocks;   /* host arrays owned by the object; block i = request i */
} ipcfp_parsed_blocks;
ipcfp_status ipcfp_blocks_from_rpc_json(const uint8_t* cids /* n_blocks*38 */, uint64_t n_blocks, const char* const* texts, const uint64_t* text_lens,
                                        uint64_t n_texts, ipcfp_parsed_blocks** out);
void ipcfp_parsed_blocks_free(ipcfp_parsed_blocks* p);
/* The same texts straight to a new block store. The store, status and index are in every case those of ipcfp_blocks_from_rpc_json
 * followed by ipcfp_store_create(blocks.cids, blocks.offsets, blocks.lengths, blocks.blob, blocks.blob_size, n_blocks, device, flags):
 * block i of the store is the block of request i, so ipcfp_store_first_bad_block and every index are request ids. The bytes come from
 * an RPC node: pass IPCFP_STORE_VERIFY_CIDS, which checks every block against its CID (IPCFP_ERR_CID_MISMATCH at the request id; *out is
 * then set, as with ipcfp_store_create). Texts in canonical form are parsed on the device, the base64 decoded straight into the store's
 * arena — each text either one element or "[" elements joined by "," "]", no whitespace, every element exactly
 *   {"jsonrpc":"2.0","result":"<base64>","id":<decimal, no leading zeros>}
 * and all texts together under 4 GiB. Any other input (whitespace, other member orders, escapes, error responses, repeated or missing ids,
 * and every invalid text) goes through ipcfp_blocks_from_rpc_json instead, with the same result.
 * Such a store has no caller blob for by-reference offsets to point into: every generate call on it with IPCFP_WITNESS_BY_REFERENCE
 * returns IPCFP_ERR_UNSUPPORTED (IPCFP_RESULT_JSON reads the store itself and works). info (may be NULL): which path ran and its times.
 * ipcfp_store_create_car fills the same struct, its three fields meaning the same for the CAR's bytes: parsed on the device or by the
 * host parser (ipcfp_blocks_from_car), wall time until the blocks were in the arena, the device parse's kernel time. */
typedef struct ipcfp_store_json_info {
    uint32_t parsed_on_device;   /* 1: the device parsed the texts; 0: ipcfp_blocks_from_rpc_json did                                 */
    float ms_parse;              /* wall time until the blocks were in the store's arena (copy of the texts included), before the index  */
    float ms_kernels;            /* device parse only: time of its kernels (CUDA events on the store's stream); 0 otherwise                */
    uint32_t _pad;
} ipcfp_store_json_info;
ipcfp_status ipcfp_store_create_rpc_json(const uint8_t* cids, uint64_t n_blocks, const char* const* texts, const uint64_t* text_lens, uint64_t n_texts,
                                         int device, uint32_t flags, ipcfp_store** out, ipcfp_store_json_info* info);

/* ------------------------------------------------------------------------------------------
 * The block store straight from a CARv1 archive (https://ipld.io/specs/transport/car/carv1/): what Filecoin.ChainExport, `lotus chain
 * export` and the published snapshots (once decompressed) hold. Varints are unsigned LEB128 below 2^63 in minimal encoding. The rules,
 * checked in file order (the first failure wins):
 *   1. the header: a varint H >= 1, then H bytes inside the buffer that are exactly one DAG-CBOR map (minimal heads, definite lengths)
 *      with the keys "roots" (an array of CIDs: tag 42 over a byte string whose first byte is 0x00; checked for form only, not returned)
 *      and "version" (an unsigned integer), in either order, each once. Its entries are read in order: a version other than 1 →
 *      IPCFP_ERR_UNSUPPORTED (a CARv2 starts with the header {"version": 2}); anything else malformed, a key missing and bytes left over
 *      inside H included → IPCFP_ERR_DECODE; both with index UINT64_MAX;
 *   2. sections from the header's end to len, k = 0, 1, …: a varint L; L = 0, or L bytes not all inside the buffer (a truncated varint
 *      included) → IPCFP_ERR_DECODE at k; the section starts with a CID that must decode under the CID spec (else IPCFP_ERR_DECODE at k)
 *      and be the store's form, CIDv1 with a one-byte codec, a three-byte multihash code and a 32-byte digest: 38 bytes (else
 *      IPCFP_ERR_UNSUPPORTED at k: CIDv0, sha2-256, identity, a two-byte codec); the block is the rest of the section, possibly empty;
 *      a block of 2^32 bytes or more → IPCFP_ERR_UNSUPPORTED at k.
 * ipcfp_blocks_from_car (host C++, no device): the sections in file order, block k = section k. blocks.cids (n*38), and blocks.offsets /
 * blocks.lengths index `car` itself; blocks.blob is NULL and blocks.blob_size = len (the convention of IPCFP_WITNESS_BY_REFERENCE).
 * car NULL or out NULL → IPCFP_ERR_INVALID_ARG. Released with ipcfp_parsed_blocks_free.
 * ------------------------------------------------------------------------------------------ */
ipcfp_status ipcfp_blocks_from_car(const uint8_t* car, uint64_t len, ipcfp_parsed_blocks** out);
/* The same bytes straight to a new store. In every case the store, status and index are those of ipcfp_blocks_from_car followed by
 * ipcfp_store_create(blocks.cids, blocks.offsets, blocks.lengths, car, len, n, device, flags): the arena is the CAR, index k is section
 * k (ipcfp_store_first_bad_block included: IPCFP_ERR_CID_MISMATCH at the section index under IPCFP_STORE_VERIFY_CIDS, *out then set),
 * the rules of ipcfp_store_create apply (duplicate CIDs stay as duplicate entries, the lowest index wins; fewer than 2^31 blocks), and
 * IPCFP_WITNESS_BY_REFERENCE offsets index `car`. The CAR is copied to the device once (pinned memory from ipcfp_host_alloc copies at
 * PCIe rate; pageable memory works too) and its sections are found there, whatever its blocks hold. A CAR the device path does not
 * accept (every invalid CAR) goes through ipcfp_blocks_from_car, over the same device copy, for its status and index; so does any CAR
 * when the device has no room for the parse's scratch (about 0.4 bytes per CAR byte, plus 48 bytes per candidate section). info (may be NULL) is the ipcfp_store_json_info of ipcfp_store_create_rpc_json, with its
 * fields' meanings: parsed_on_device (1: the device found the sections; 0: ipcfp_blocks_from_car did), ms_parse (wall time until the
 * blocks and their arrays were on the device, the copy included, before the index), ms_kernels (device parse only: its kernels' time). */
ipcfp_status ipcfp_store_create_car(const uint8_t* car, uint64_t len, int device, uint32_t flags, ipcfp_store** out, ipcfp_store_json_info* info);

/* read_storage_slot (src/proofs/storage/decode.rs:36-97), batched over k slot keys against one
 * contract_state root, with a RecordingBlockStore-equivalent witness. */
ipcfp_status ipcfp_read_storage_slots(ipcfp_store* s, const uint8_t contract_state_root[IPCFP_CID_LEN],
                                      const uint8_t* slots /* k*32 */, uint64_t k, ipcfp_slot_result** out);
void ipcfp_slot_result_free(ipcfp_slot_result* r);

/* generate_storage_proof (src/proofs/storage/generator.rs:29-67), batched over specs. */
ipcfp_status ipcfp_generate_storage_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* specs,
                                           uint64_t n_specs, ipcfp_storage_result** out);
void ipcfp_storage_result_free(ipcfp_storage_result* r);

/* ------------------------------------------------------------------------------------------
 * Storage paths: a Solidity value named by its access path, with the slots derived and read on the device (DESIGN.md §3, "Storage
 * paths"). A path is the declared slot p of a state variable (base_slot, u256 big-endian) and a list of steps; all slot arithmetic is
 * mod 2^256, as in the EVM:
 *   IPCFP_PATH_MAPPING  slot = keccak256(key ‖ slot). A value-type key is its 32-byte padded form (the caller's); a bytes / string key is
 *                       its raw bytes, 0 to IPCFP_PATH_MAX_KEY of them.
 *   IPCFP_PATH_ARRAY    a dynamic array at slot: slot = keccak256(slot) + (index / per_slot) * elem_slots; the array's length word (the
 *                       slot before the step) is proven too.
 *   IPCFP_PATH_STATIC   a static array at slot: slot = slot + (index / per_slot) * elem_slots.
 *   IPCFP_PATH_FIELD    a struct member: slot = slot + index (the member's slot offset).
 * per_slot = 32 / elem_bytes when the elements are packed (elem_slots = 1 and elem_bytes 1..32), else 1; a packed element sits
 * byte_offset = (index % per_slot) * elem_bytes bytes above the low-order end of its word.
 * kind IPCFP_PATH_WORDS reads n_words (1..IPCFP_PATH_MAX_WORDS) consecutive slots from the final slot: a value type, a whole struct or a
 * static array. kind IPCFP_PATH_BYTES reads a Solidity bytes / string at the final slot: its header word h, then
 *   h & 1 == 0  short: length = (h & 0xff) / 2, which must be <= 31; the bytes are the word's high-order bytes;
 *   h & 1 == 1  long: length = (h - 1) / 2, which must be >= 32; the bytes are in ceil(length / 32) slots from keccak256(slot).
 * A path's EXPANDED SPECS are (actor_id, slot) pairs in this order: the length word of every ARRAY step, in step order; then the value
 * words (the n_words slots, or the header word followed by the data slots in ascending order). The expanded specs of the paths of one
 * call are concatenated in path order.
 * ------------------------------------------------------------------------------------------ */
#define IPCFP_PATH_MAX_PATHS 65536u  /* paths of one call: a failure's index keeps the path in 16 bits beside its spec's position       */
#define IPCFP_PATH_MAX_STEPS 32u     /* steps of one path: one thread derives a path, and every ARRAY step adds a spec to it           */
#define IPCFP_PATH_MAX_KEY 1024u     /* bytes of one MAPPING key: one thread absorbs it into Keccak-256 (at most 8 blocks of 136 bytes) */
#define IPCFP_PATH_MAX_WORDS 256u    /* n_words of a WORDS path: a proof per word, 8 KiB of value                                      */
#define IPCFP_PATH_MAX_BYTES 4096u   /* length of a BYTES value: at most 128 data slots, so one path asks for at most 160 KiB of proof
                                        recorder lists in wave 2 (128 x 320 words)                                                     */
enum { IPCFP_PATH_MAPPING = 0, IPCFP_PATH_ARRAY = 1, IPCFP_PATH_STATIC = 2, IPCFP_PATH_FIELD = 3 };
enum { IPCFP_PATH_WORDS = 0, IPCFP_PATH_BYTES = 1 };
/* Per-path status (not a call failure: the path's proofs are still emitted) */
enum {
    IPCFP_PATH_OK = 0,
    IPCFP_PATH_INDEX_OUT_OF_RANGE = 1,  /* an ARRAY index at or beyond its proven length word (the first such step decides)          */
    IPCFP_PATH_BAD_BYTES = 2,           /* a header word Solidity refuses with Panic 0x22: short with length > 31, long with < 32      */
    IPCFP_PATH_TOO_LONG = 3             /* a long bytes / string over IPCFP_PATH_MAX_BYTES: only its header word is proven              */
};
typedef struct ipcfp_path_step {
    uint32_t op;              /* IPCFP_PATH_MAPPING / _ARRAY / _STATIC / _FIELD                                   */
    uint32_t key_len;         /* MAPPING: bytes at key                                                             */
    const uint8_t* key;       /* MAPPING                                                                           */
    uint64_t index;           /* ARRAY / STATIC: the element index; FIELD: the member's slot offset                */
    uint32_t elem_slots;      /* ARRAY / STATIC: slots per element, >= 1                                           */
    uint32_t elem_bytes;      /* ARRAY / STATIC: 0 (not packed) or the packed element's size, 1..32                */
} ipcfp_path_step;
typedef struct ipcfp_storage_path {
    uint64_t actor_id;
    uint8_t base_slot[32];    /* the state variable's declared slot p, u256 big-endian                               */
    uint32_t n_steps;
    uint32_t kind;            /* IPCFP_PATH_WORDS / IPCFP_PATH_BYTES                                                 */
    const ipcfp_path_step* steps;
    uint32_t n_words;         /* WORDS: 1..IPCFP_PATH_MAX_WORDS; BYTES: ignored                                      */
    uint32_t _pad;
} ipcfp_storage_path;
typedef struct ipcfp_path_value {
    uint32_t status;          /* IPCFP_PATH_*                                                                        */
    uint32_t valid;           /* ipcfp_verify_storage_paths: 1 when every expanded spec has a proof that verifies; generate: 1 */
    uint8_t slot[32];         /* the final slot                                                                      */
    uint32_t byte_offset;     /* a packed last ARRAY / STATIC step: the element's byte offset above the word's low end; else 0 */
    uint32_t _pad;
    uint64_t first_spec;      /* the path's expanded specs: specs[first_spec .. first_spec + n_specs)                 */
    uint64_t n_specs;
    uint64_t value_off;       /* the value: value_blob[value_off .. value_off + value_len) — WORDS: the 32-byte words; BYTES:
                                 the decoded bytes (status OK or INDEX_OUT_OF_RANGE with a valid header; else 0 bytes) */
    uint64_t value_len;
} ipcfp_path_value;
typedef struct ipcfp_path_result {
    uint64_t n_paths;
    const ipcfp_path_value* paths;
    uint64_t n_specs;
    const ipcfp_storage_spec* specs;    /* the expanded specs of every path, concatenated in path order                     */
    const uint8_t* value_blob;
    uint64_t value_blob_size;
    ipcfp_storage_result* storage;      /* generate: the proofs of specs (owned by this result); verify: NULL               */
    /* device time (CUDA events on the store's stream), milliseconds: the whole call, slot derivation, wave 1 (the fixed specs), wave
     * 2 (the data slots, derived and proven), the witness and per-spec lists; host_syncs: host synchronisations the call made */
    float ms_total, ms_slots, ms_wave1, ms_wave2, ms_witness;
    uint32_t host_syncs;
} ipcfp_path_result;
/* Proofs of storage paths. `storage` is, byte for byte, what ipcfp_generate_storage_proofs gives for `specs` (the proofs, the witness
 * union, the per-spec witness lists); every proof is an ordinary StorageProof, and the expanded specs go into every bundle and planner
 * call as ordinary ipcfp_storage_spec. flags: IPCFP_WITNESS_BY_REFERENCE only (any other bit: IPCFP_ERR_INVALID_ARG).
 * Flow: slot derivation (one thread per path, chained Keccak-256 and u256 adds), wave 1 (the fixed specs: length words and value or
 * header words), the expansion (each BYTES path's data-slot count and every path's status from wave 1's words, then a scan), wave 2
 * (the data slots keccak256(slot) + j, derived and proven on the device into the same witness bitmap), one witness materialisation.
 * Host synchronisations: four — the size of wave 2 after the expansion, then the three every storage result takes: the witness
 * count, the end of the witness copy, the end of the call.
 * Failures have the statuses of ipcfp_generate_storage_proofs; the index is the first failing path, and within it the first failing
 * spec in expanded order decides the status. IPCFP_ERR_INVALID_ARG before any device work: a NULL array with a nonzero count, more than
 * IPCFP_PATH_MAX_PATHS paths or IPCFP_PATH_MAX_STEPS steps, a key over IPCFP_PATH_MAX_KEY, an unknown op or kind, elem_bytes over 32,
 * elem_slots = 0, n_words of 0 or over IPCFP_PATH_MAX_WORDS, a tipset without child_parent_state_root. *out is released with
 * ipcfp_path_result_free. */
ipcfp_status ipcfp_generate_storage_path_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_path* paths, uint64_t n,
                                                         uint32_t flags, ipcfp_path_result** out);
/* (the fetch round of this call, ipcfp_plan_fetch_storage_paths_resident, is declared with the other planners below) */
/* Checks storage-path claims against a bundle's storage proofs: every proof is replayed by ipcfp_verify_storage_proofs over the witness
 * store (its failures fail the call, index = the proof). Then, per path, the expanded specs are derived on the device with the length
 * and header words taken from the proofs themselves; each (actor_id, slot) must have a proof in the list that verifies (the first in
 * (actor_id, slot) order when several do). The result's paths[i].valid, status and value are the path's verdict, `specs` the expanded
 * specs derived, `storage` NULL. A proof whose value was changed, a data slot left out or a length word that lies makes the path invalid.
 * A path that is not valid still gets a status and value, read as follows where a spec has no proof that verifies: a length word does
 * not make the index out of range, a bytes / string header reads as zero (no data slots, an empty value), and any other word is that
 * of the first proof in the list with the spec's (actor_id, slot), or zero when there is none. Such a value is not proven.
 * Refusals are the generate call's. *out is released with ipcfp_path_result_free. */
ipcfp_status ipcfp_verify_storage_paths(ipcfp_store* witness_store, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs, uint64_t n_proofs,
                                        const ipcfp_storage_path* paths, uint64_t n_paths, ipcfp_path_result** out);
void ipcfp_path_result_free(ipcfp_path_result* r);

/* generate_proof_bundle (src/proofs/generator.rs:25-95): the storage specs, then the event specs in order, then the union of every
 * proof's blocks (BTreeSet<(Cid, data)>, built on the device). Equivalent to ipcfp_tipset_upload followed by
 * ipcfp_generate_proof_bundle_resident with flags = 0. */
ipcfp_status ipcfp_generate_proof_bundle(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* sspecs,
                                         uint64_t n_sspecs, const ipcfp_event_spec* especs, uint64_t n_especs,
                                         ipcfp_bundle** out);
/* The same against a tipset uploaded once with ipcfp_tipset_upload; it fails where ipcfp_generate_proof_bundle fails, with the same status
 * and index. flags (any other bit: IPCFP_ERR_INVALID_ARG):
 *   IPCFP_WITNESS_BY_REFERENCE  every witness of the bundle (storage->witness, each events[k]->witness and the union `witness`) comes
 *                               by reference: blob NULL, offsets into the blob the store was created from;
 *   IPCFP_RESULT_JSON           the bundle also carries `json`, the UnifiedProofBundle text rendered on the device (block bytes are read
 *                               from the store, so it combines with IPCFP_WITNESS_BY_REFERENCE). One extra host synchronisation.
 * Storage specs need a tipset uploaded with child_parent_state_root (else IPCFP_ERR_INVALID_ARG). */
ipcfp_status ipcfp_generate_proof_bundle_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                                  const ipcfp_event_spec* especs, uint64_t n_especs, uint32_t flags, ipcfp_bundle** out);
/* generate_proof_bundle with log filters in place of event specs: the storage specs in one batch, then filters[0..n_filters) in order
 * (events[k] is filter k's EventProofBundle, what ipcfp_generate_log_proof_resident gives for it with the same IPCFP_WITNESS_BY_REFERENCE
 * bit), then the union of every proof's blocks. Flags, the storage specs' tipset rule and the JSON text are those of
 * ipcfp_generate_proof_bundle_resident; the text is the UnifiedProofBundle ipcfp_bundle_to_json renders for the flagless bundle.
 * An event spec is the filter {emitters = [actor] or none, n_positions = 2, values = [{keccak256(sig)}, {ascii_to_bytes32(t1)}]}, and
 * a bundle of those filters is byte for byte the bundle of the specs. Every filter is checked before any device work: a refused filter
 * gives IPCFP_ERR_INVALID_ARG with its position as the index. Otherwise the status and index of a failure are those of the first
 * generator that fails, in the order storage, filter 0, filter 1, … (the order of the spec bundle). ipcfp_generate_log_bundle =
 * ipcfp_tipset_upload, then the resident call. */
ipcfp_status ipcfp_generate_log_bundle_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                                const ipcfp_log_filter* filters, uint64_t n_filters, uint32_t flags, ipcfp_bundle** out);
ipcfp_status ipcfp_generate_log_bundle(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                       const ipcfp_log_filter* filters, uint64_t n_filters, uint32_t flags, ipcfp_bundle** out);
void ipcfp_bundle_free(ipcfp_bundle* b);

/* ------------------------------------------------------------------------------------------
 * Fetch planning: which blocks to request before ipcfp_generate_proof_bundle_resident can run on a store that does not hold them all.
 * N(S) is the set of blocks the generators of that call would get for this tipset and these specs, as far as decoding the blocks
 * already in the store S finds them (the rules are DESIGN.md §2, "Fetch planning"); the plan is M(S) = N(S) \ S. Each call is one
 * round: fetch the plan's CIDs, build a store from the blocks held so far plus the new ones, upload the tipset to it and call again.
 * Once a plan is empty, ipcfp_generate_proof_bundle_resident on the store gives what it gives on a store with every block: the same
 * bundle, or the same status and index. The planner itself never returns IPCFP_ERR_MISSING_BLOCK or IPCFP_ERR_DECODE; a block that
 * does not decode only has no children here. Any flag bit, or storage specs against a tipset without child_parent_state_root, is
 * IPCFP_ERR_INVALID_ARG. An empty store works (every root is missing). *out is released with ipcfp_fetch_plan_free.
 * ------------------------------------------------------------------------------------------ */
typedef struct ipcfp_fetch_plan {
    uint64_t n_missing;
    const uint8_t* cids;   /* n_missing*38: M(S), unique, in `Cid` order, none of them in the store */
    uint64_t n_needed;     /* blocks of N(S) present in the store                                   */
    uint32_t n_levels;     /* frontier levels of the AMT walk on the device                          */
    float ms_total;        /* CUDA events on the store's stream                                      */
} ipcfp_fetch_plan;
ipcfp_status ipcfp_plan_fetch_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                       const ipcfp_event_spec* especs, uint64_t n_especs, uint32_t flags, ipcfp_fetch_plan** out);
/* ipcfp_tipset_upload, then ipcfp_plan_fetch_resident */
ipcfp_status ipcfp_plan_fetch(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                              const ipcfp_event_spec* especs, uint64_t n_especs, uint32_t flags, ipcfp_fetch_plan** out);
void ipcfp_fetch_plan_free(ipcfp_fetch_plan* p);
/* One fetch round for ipcfp_generate_log_proof_resident: the rules of ipcfp_plan_fetch_resident for event specs, with the filter as
 * rule 3's predicate (the receipts with a matching event add their receipts-AMT paths). Any flag bit is IPCFP_ERR_INVALID_ARG. */
ipcfp_status ipcfp_plan_fetch_log_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_log_filter* filter, uint32_t flags,
                                           ipcfp_fetch_plan** out);
/* One fetch round for ipcfp_generate_message_log_proof_resident: the rules of ipcfp_plan_fetch_log_resident, with two changes. While any
 * TxMeta or message-AMT block is missing (the execution order, and so the selection, needs all of them), the round plans the base roots,
 * the TxMeta blocks and the message AMTs only. Once they are all present, the planner builds the execution order on the device and plans
 * the events AMTs of the selected receipts only, and the receipts-AMT paths of the selected receipts that match. exec_indices is not
 * reported. Refusals are those of the generate call; any flag bit is IPCFP_ERR_INVALID_ARG. */
ipcfp_status ipcfp_plan_fetch_message_log_resident(ipcfp_store* s, ipcfp_tipset* t, const uint8_t* message_cids /* n*38 */, uint64_t n,
                                                   const ipcfp_log_filter* filter /* may be NULL */, uint32_t flags, ipcfp_fetch_plan** out);
/* One fetch round for ipcfp_generate_log_bundle_resident: rules 1–4 of ipcfp_plan_fetch_resident, with rule 3's predicate "matches at
 * least one of filters[]". ipcfp_plan_fetch_log_resident is the case of one filter and no storage spec. Refused filters, flags and
 * storage specs fail as in ipcfp_generate_log_bundle_resident / ipcfp_plan_fetch_resident. */
ipcfp_status ipcfp_plan_fetch_log_bundle_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                                  const ipcfp_log_filter* filters, uint64_t n_filters, uint32_t flags, ipcfp_fetch_plan** out);
/* One fetch round for ipcfp_generate_storage_path_proofs_resident: rule 4 (the storage path) for every expanded spec known without
 * reading storage (the length words and the value or header words), and for a BYTES path's data slots once the store can read its
 * header word (a long header adds one round). From an empty store the rounds end with a store on which the generate call gives what
 * it gives on the complete store: the same result, or the same status and index. Refusals are the generate call's; any flag bit is
 * IPCFP_ERR_INVALID_ARG. */
ipcfp_status ipcfp_plan_fetch_storage_paths_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_path* paths, uint64_t n,
                                                     uint32_t flags, ipcfp_fetch_plan** out);
/* The round as one Filecoin.ChainReadObj batch: request k asks for plan->cids[k] with "id": first_id + k, compact JSON
 *   [{"jsonrpc":"2.0","method":"Filecoin.ChainReadObj","params":[{"/":"b…"}],"id":<first_id + k>},…]
 * With first_id = the number of blocks already held, the responses go straight to ipcfp_store_create_rpc_json with
 * cids = (blocks already held) ++ plan->cids. Host-side rendering: no device is needed. *out is released with ipcfp_json_free. */
ipcfp_status ipcfp_fetch_plan_to_rpc_json(const ipcfp_fetch_plan* p, uint64_t first_id, char** out, uint64_t* out_len);

/* ------------------------------------------------------------------------------------------
 * Address resolution: Filecoin addresses to actor IDs from the state tree itself, in place of the reference's
 * Filecoin.EthAddressToFilecoinAddress + Filecoin.StateLookupID round trip (src/proofs/common/address.rs:8-62). The path is
 * StateRoot [version <= 5, actors, info] -> actors HAMT (width 5) -> the Init actor (ID 1) -> its state, exactly
 * [address_map, next_id, network_name] -> address_map HAMT (width 5, key Address::to_bytes(), value the ActorID as one CBOR unsigned
 * integer) (DESIGN.md §2 "Address resolution", §3). ipcfp_address holds Address::to_bytes(): protocol byte, then the payload.
 * ------------------------------------------------------------------------------------------ */
#define IPCFP_ADDRESS_MAX 65   /* 1 protocol byte + 10-byte LEB128 namespace + 54-byte subaddress */
typedef struct ipcfp_address {
    uint8_t len;
    uint8_t bytes[IPCFP_ADDRESS_MAX];
} ipcfp_address;
typedef struct ipcfp_resolve_result {
    uint64_t n;
    const uint64_t* actor_ids;     /* n; 0 where status != IPCFP_OK                                                           */
    const ipcfp_status* status;    /* n: IPCFP_OK, _ACTOR_NOT_FOUND, _MISSING_BLOCK, _DECODE, or _INVALID_ARG (bytes that are not
                                      an Address); a non-ID address carries init_status when that is not IPCFP_OK               */
    ipcfp_status init_status;      /* StateRoot -> actors HAMT -> Init state, walked once per call                              */
    uint32_t _pad;
    uint64_t n_missing;
    const uint8_t* missing_cids;   /* n_missing*38: the blocks the walks lacked, unique, `Cid` order (ipcfp_fetch_plan's form) */
    ipcfp_witness witness;         /* every block the walks read, the Init path's included, `Cid` order                       */
    float ms_total, ms_lookup;     /* CUDA events on the store's stream: the call, the address_map walks                      */
} ipcfp_resolve_result;
/* n addresses against the state tree at state_root, one device walk per non-ID address. ID addresses (protocol 0) resolve to their
 * own ID with no read (Lotus StateTree.LookupID). Unknown or unresolvable addresses are answers, not failures: the call fails only on
 * null arguments, no device or CUDA errors. Missing blocks are reported in missing_cids, so a caller can fetch them (one
 * Filecoin.ChainReadObj round: ipcfp_fetch_plan_to_rpc_json over a plan holding these CIDs) and call again.
 * *out is released with ipcfp_resolve_result_free. */
ipcfp_status ipcfp_resolve_addresses(ipcfp_store* s, const uint8_t state_root[IPCFP_CID_LEN], const ipcfp_address* addrs, uint64_t n,
                                     ipcfp_resolve_result** out);
void ipcfp_resolve_result_free(ipcfp_resolve_result* r);
/* Host only, no device. ipcfp_address_parse: the text form ("f…" or "t…", read alike; protocols 0–4; lower-case unpadded base32 with the
 * 4-byte Blake2b checksum of to_bytes(); protocol 4 as f4<namespace>f<base32(subaddress ‖ checksum)>) → IPCFP_ERR_INVALID_ARG when
 * malformed. ipcfp_address_from_eth: Lotus EthAddress.ToFilecoinAddress — a masked ID (0xff, eleven zero bytes, the ID big-endian)
 * becomes the ID address, any other address f410 (04 0a ‖ eth). */
ipcfp_status ipcfp_address_parse(const char* text, uint64_t len, ipcfp_address* out);
ipcfp_status ipcfp_address_from_eth(const uint8_t eth[20], ipcfp_address* out);

/* ------------------------------------------------------------------------------------------
 * Actor proofs: what the state tree holds for an address — its actor ID, code, head, nonce (sequence), balance and delegated (f410)
 * address, and for an EVM actor its bytecode CID and hash, EVM nonce and storage root — or a proof that the address or actor is absent
 * (DESIGN.md §2 "Actor proofs", §3). The account half of eth_getProof. A request is an ipcfp_address:
 *   protocol 0 (ID)   the actors HAMT under the child header's ParentStateRoot, key Address::new_id(id).to_bytes();
 *   any other         first the Init actor's address_map (the path of ipcfp_resolve_addresses) under the same ParentStateRoot, then
 *                     the actors HAMT under the ID found there.
 * Every block of both walks goes into the proof's witness: the child header, the StateRoot, the Init path (actors HAMT to ID 1, the
 * InitState) and the address_map path for a non-ID address, the actors HAMT path, the EVM state of an EVM actor and, with
 * IPCFP_ACTOR_WITH_CODE, its bytecode block.
 * Decode contract of the new fields (the rest is DESIGN.md §3's):
 *   ActorState   [code, head, sequence, balance, delegated | null], exactly; delegated must be bytes Address::from_bytes accepts;
 *   balance      fvm bigint_ser: empty bytes = 0; else a sign byte (0 plus, 1 minus; anything else: IPCFP_ERR_DECODE) followed by the
 *                big-endian magnitude, at most 32 bytes (more: IPCFP_ERR_DECODE; total supply is below 2^91). A zero magnitude is
 *                never negative;
 *   EVM actors   those whose code is one of evm_code_cids (the EVM actor code CIDs of the network's manifests; the caller's input, n_evm
 *                may be 0). Their head is read as EvmStateV6, else V5 (the rule of storage proofs); neither: IPCFP_ERR_DECODE. The head
 *                of any other actor is not read.
 * ------------------------------------------------------------------------------------------ */
#define IPCFP_ACTOR_MAX 65536u          /* requests of one call                                                                */
#define IPCFP_ACTOR_WITH_CODE 0x20u     /* flag: the bytecode block of every EVM actor joins its witness and its bytes the code blob */
enum {
    IPCFP_ACTOR_FOUND = 0,              /* the actor and every field below                                                     */
    IPCFP_ACTOR_NO_ADDRESS = 1,         /* a non-ID address proven absent from the address_map; actor_id and the fields are 0   */
    IPCFP_ACTOR_NO_ACTOR = 2            /* actor_id proven absent from the actors HAMT; the fields are 0                        */
};
/* 400 bytes, 8-byte aligned; every byte not named by a field is zero. Offsets: actor_id 0, sequence 8, evm_nonce 16, code_off 24,
 * code_len 32, status 40, balance_negative 44, has_delegated 45, is_evm 46, balance 48, code 80, head 118, bytecode_cid 156,
 * contract_state 194, bytecode_hash 232, address 264, delegated 330. */
typedef struct ipcfp_actor_proof {
    uint64_t actor_id;                  /* the ID (an ID address's own, or the address_map's value)                               */
    uint64_t sequence;                  /* ActorState.sequence (the nonce)                                                        */
    uint64_t evm_nonce;                 /* EVM actors: the EVM state's nonce                                                      */
    uint64_t code_off, code_len;        /* IPCFP_ACTOR_WITH_CODE, EVM actors: the bytecode, code_blob[code_off .. +code_len)       */
    uint32_t status;                    /* IPCFP_ACTOR_*                                                                          */
    uint8_t balance_negative;
    uint8_t has_delegated;
    uint8_t is_evm;                     /* code is one of evm_code_cids                                                           */
    uint8_t _pad0;
    uint8_t balance[32];                /* big-endian magnitude                                                                   */
    uint8_t code[IPCFP_CID_LEN];        /* ActorState.code                                                                        */
    uint8_t head[IPCFP_CID_LEN];        /* ActorState.state                                                                       */
    uint8_t bytecode_cid[IPCFP_CID_LEN];   /* EVM actors                                                                         */
    uint8_t contract_state[IPCFP_CID_LEN]; /* EVM actors: the storage root storage proofs read (their storage_root)             */
    uint8_t bytecode_hash[32];          /* EVM actors: keccak256 of the bytecode                                                  */
    ipcfp_address address;              /* the request                                                                            */
    ipcfp_address delegated;            /* has_delegated: ActorState.delegated_address                                            */
    uint8_t _pad1[4];
} ipcfp_actor_proof;
typedef struct ipcfp_actor_result {
    uint64_t n_proofs;
    const ipcfp_actor_proof* proofs;        /* in request order                                                                   */
    ipcfp_witness witness;                  /* union over all proofs, `Cid` order                                                 */
    const uint64_t* proof_witness_offsets;  /* n_proofs+1                                                                         */
    const uint32_t* proof_witness_index;    /* per proof: indices into witness (its blocks), ascending                            */
    const uint8_t* code_blob;               /* IPCFP_ACTOR_WITH_CODE: the bytecodes, in proof order                               */
    uint64_t code_blob_size;
    /* device time (CUDA events on the store's stream), milliseconds: the whole call, the Init walk, the proofs' walks, the code gather,
     * the witness and per-proof lists; host_syncs: host synchronisations the call made */
    float ms_total, ms_init, ms_walk, ms_code, ms_witness;
    uint32_t host_syncs;
} ipcfp_actor_result;
/* Proofs of n addresses against a resident tipset. Anchored as storage proofs are: the child header's ParentStateRoot must equal the
 * tipset's child_parent_state_root (else IPCFP_ERR_STATE_ROOT_MISMATCH), and the header is in every proof's witness. flags:
 *   IPCFP_WITNESS_BY_REFERENCE  the witness comes by reference (blob NULL, offsets into the blob the store was created from);
 *   IPCFP_ACTOR_WITH_CODE       the bytecode block of every EVM actor (raw codec 0x55, Blake2b-256: a second CID prefix in the store)
 *                               joins the proof's witness and its bytes the code blob; keccak256 of the bytes must equal bytecode_hash,
 *                               else IPCFP_ERR_DECODE.
 * The Init path runs once per call, and only when some address is not an ID address. Absent addresses and actors are answers (status),
 * not failures. Missing blocks, decode errors, a state-tree without an Init actor (IPCFP_ERR_ACTOR_NOT_FOUND) and a state-root mismatch
 * fail the call with the first failing proof's index, as ipcfp_generate_storage_proofs does. IPCFP_ERR_INVALID_ARG before any device
 * work: bytes that are not an Address (ipcfp_resolve_addresses' rule; the index names the request), NULL arrays with nonzero counts, more
 * than IPCFP_ACTOR_MAX requests, another flag bit, a tipset without child_parent_state_root. Host synchronisations: four — the error
 * word (with the bytecode lengths), the witness count, the end of the witness copy, the end of the call. *out is released with
 * ipcfp_actor_result_free. */
ipcfp_status ipcfp_generate_actor_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_address* addrs, uint64_t n,
                                                  const uint8_t* evm_code_cids /* n_evm*38 */, uint64_t n_evm, uint32_t flags,
                                                  ipcfp_actor_result** out);
/* ipcfp_tipset_upload, then the resident call */
ipcfp_status ipcfp_generate_actor_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_address* addrs, uint64_t n,
                                         const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags, ipcfp_actor_result** out);
void ipcfp_actor_result_free(ipcfp_actor_result* r);
/* One ChainReadObj round for the call above: the blocks its walks would read that the store lacks, as far as the blocks it holds tell
 * (the bytecode blocks with IPCFP_ACTOR_WITH_CODE). From an empty store the rounds end with a store on which the generate call gives what
 * it gives on the complete store. flags: those of the generate call; refusals are its refusals. */
ipcfp_status ipcfp_plan_fetch_actor_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_address* addrs, uint64_t n,
                                                    const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags, ipcfp_fetch_plan** out);
/* Replays every proof on the witness store (create it with IPCFP_STORE_VERIFY_CIDS): the header and its ParentStateRoot against t, the
 * Init path and the address_map for a non-ID address, the actors HAMT, every field, the EVM state of an actor whose code is in
 * evm_code_cids, and with IPCFP_ACTOR_WITH_CODE the bytecode block (its length must be code_len and its keccak256 bytecode_hash).
 * Absence claims are checked by walking to the absence again. results[i] = 1 when proof i states exactly what the witness holds. A
 * missing witness block or a decode error fails the call at that proof, as ipcfp_verify_storage_proofs does; refusals are the generate
 * call's (an address of a proof that is not an Address, an unknown status is a 0 verdict). */
ipcfp_status ipcfp_verify_actor_proofs(ipcfp_store* witness_store, const ipcfp_tipset_desc* t, const ipcfp_actor_proof* proofs, uint64_t n,
                                       const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags, uint8_t* results);

/* ------------------------------------------------------------------------------------------
 * Message proofs: whether a message executed in the tipset pair and how it ended — its receipt's exit code, return data, gas used and
 * events root — and, with IPCFP_MESSAGE_WITH_BODY, the message itself (DESIGN.md §2 "Message proofs", §3). The status / gasUsed half of
 * eth_getTransactionReceipt, with the fields eth_getTransactionByHash returns. A request is a message CID as the parent blocks' message
 * AMTs hold it (the request of ipcfp_generate_message_log_proof_resident); duplicates are allowed. Request j's execution position is
 * found in the execution order the event calls rebuild, and its receipt is Amtv0<Receipt>::get(exec_index) under the tipset's
 * receipts_root. The tipset's RPC receipt list (events_roots, n_receipts) and every events AMT are not read.
 * Decode contract of the new fields (the rest is DESIGN.md §3's):
 *   Receipt        [exit_code, return_data, gas_used, events_root | null], exactly; exit_code at most 2^32-1, gas_used a u64;
 *   message block  decided by its shape: array(10) is a Message [version, to, from, sequence, value, gas_limit, gas_fee_cap, gas_premium,
 *                  method_num, params]; array(2) is a SignedMessage [Message, Signature]; anything else is IPCFP_ERR_DECODE.
 *                  version, sequence, gas_limit and method_num are unsigned integers (a negative one: IPCFP_ERR_DECODE); to and from
 *                  bytes Address::from_bytes accepts; value, gas_fee_cap and gas_premium TokenAmounts (the balance rule of actor
 *                  proofs); params bytes; the Signature bytes whose first byte is its type, 1 secp256k1, 2 BLS or 3 delegated (any
 *                  other byte, or no byte: IPCFP_ERR_DECODE). Nothing may follow the block's one item.
 * ------------------------------------------------------------------------------------------ */
#define IPCFP_MESSAGE_WITH_BODY 0x40u   /* flag: the message block of every executed request joins the witness; its fields are decoded */
enum {
    IPCFP_MESSAGE_EXECUTED = 0,         /* executed, with its receipt in every receipt field                                       */
    IPCFP_MESSAGE_NOT_EXECUTED = 1,     /* not in the execution order; exec_index is UINT64_MAX and every other field is 0          */
    IPCFP_MESSAGE_NO_RECEIPT = 2        /* executed, but the receipts AMT has no entry at exec_index; the receipt fields are 0      */
};
/* 400 bytes, 8-byte aligned; every byte not named by a field is zero. Offsets: exec_index 0, gas_used 8, return_off 16, return_len 24,
 * version 32, sequence 40, gas_limit 48, method_num 56, params_off 64, params_len 72, status 80, exit_code 84, has_events_root 88,
 * has_body 89, sig_type 90, value_negative 91, gas_fee_cap_negative 92, gas_premium_negative 93, value 96, gas_fee_cap 128,
 * gas_premium 160, message_cid 192, events_root 230, to 268, from 334. */
typedef struct ipcfp_message_proof {
    uint64_t exec_index;                /* position in the execution order; UINT64_MAX when not executed                          */
    uint64_t gas_used;                  /* Receipt.gas_used                                                                       */
    uint64_t return_off, return_len;    /* Receipt.return_data: data_blob[return_off .. +return_len) (return_off 0 when empty)     */
    uint64_t version;                   /* with the body: Message.version                                                         */
    uint64_t sequence;                  /* with the body: Message.sequence (the nonce)                                            */
    uint64_t gas_limit;                 /* with the body: Message.gas_limit                                                       */
    uint64_t method_num;                /* with the body: Message.method_num                                                      */
    uint64_t params_off, params_len;    /* with the body: Message.params, data_blob[params_off .. +params_len) (0 when empty)      */
    uint32_t status;                    /* IPCFP_MESSAGE_*                                                                        */
    uint32_t exit_code;                 /* Receipt.exit_code                                                                      */
    uint8_t has_events_root;
    uint8_t has_body;                   /* IPCFP_MESSAGE_WITH_BODY and the message executed: the body fields are set              */
    uint8_t sig_type;                   /* with the body: 0 for a Message block, else the Signature's type byte (1, 2 or 3)        */
    uint8_t value_negative, gas_fee_cap_negative, gas_premium_negative;
    uint8_t _pad0[2];
    uint8_t value[32];                  /* with the body: big-endian magnitudes                                                   */
    uint8_t gas_fee_cap[32];
    uint8_t gas_premium[32];
    uint8_t message_cid[IPCFP_CID_LEN]; /* the request                                                                            */
    uint8_t events_root[IPCFP_CID_LEN]; /* has_events_root: Receipt.events_root                                                   */
    ipcfp_address to;                   /* with the body: Message.to                                                              */
    ipcfp_address from;                 /* with the body: Message.from                                                            */
} ipcfp_message_proof;
typedef struct ipcfp_message_result {
    uint64_t n_proofs;
    const ipcfp_message_proof* proofs;  /* in request order                                                                       */
    const uint8_t* data_blob;           /* per proof: its return data, then its params                                            */
    uint64_t data_blob_size;
    ipcfp_witness witness;              /* one union, `Cid` order: the base witness, every parent's message AMTs, the receipts root,
                                         * each executed request's receipts-AMT path and, with the body, the message blocks        */
    uint64_t n_exec;                    /* length of the execution order                                                          */
    /* device time (CUDA events on the store's stream), milliseconds: the whole call, the execution order (the requests' sort, the
     * message-AMT walk and the dedup), the selection and per-request walks, the data-blob gather, the witness; host_syncs: the call's host synchronisations when the message
     * AMTs take the dense walk (the general walk adds its own) */
    float ms_total, ms_exec_order, ms_walk, ms_gather, ms_witness;
    uint32_t host_syncs;
} ipcfp_message_result;
/* Proofs of n messages against a resident tipset. flags: IPCFP_WITNESS_BY_REFERENCE (the witness comes by reference, as for the event
 * calls) and IPCFP_MESSAGE_WITH_BODY. Not executed and no receipt are answers (status), not failures: the first is proven by the message
 * AMTs, which are in the base witness, the second by the receipts-AMT path up to the node that shows the entry absent.
 * Failures: a fault in a header, a TxMeta, a message AMT or the receipts root carries the status and index the message-log call reports
 * for it; then the first fault in request order — a missing or undecodable receipts-AMT node, receipt or message block — with the
 * request's index; then a base-witness block the store lacks (IPCFP_ERR_MISSING_BLOCK). IPCFP_ERR_INVALID_ARG before any device work:
 * message_cids NULL with n > 0, n > IPCFP_MESSAGE_MAX, another flag bit. Host synchronisations: five when the message AMTs take the dense
 * walk — the walk's, the error word with the data lengths, the witness count, the end of the witness copy, the end of the call.
 * *out is released with ipcfp_message_result_free. */
ipcfp_status ipcfp_generate_message_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const uint8_t* message_cids /* n*38 */, uint64_t n,
                                                    uint32_t flags, ipcfp_message_result** out);
/* ipcfp_tipset_upload, then the resident call */
ipcfp_status ipcfp_generate_message_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const uint8_t* message_cids, uint64_t n, uint32_t flags,
                                           ipcfp_message_result** out);
void ipcfp_message_result_free(ipcfp_message_result* r);
/* One ChainReadObj round for the call above: while the execution order cannot be built, the headers, the receipts root, the TxMetas and
 * the message AMTs the store lacks; once it can, also each executed request's receipts-AMT path up to the first block the store lacks
 * and, with IPCFP_MESSAGE_WITH_BODY, its message block. No events AMT is planned. From an empty store the rounds end with a store on
 * which the generate call gives what it gives on the complete store. flags and refusals are the generate call's. */
ipcfp_status ipcfp_plan_fetch_message_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const uint8_t* message_cids, uint64_t n, uint32_t flags,
                                                      ipcfp_fetch_plan** out);
/* Replays every proof on the witness store (create it with IPCFP_STORE_VERIFY_CIDS). The tipset is anchored as ipcfp_verify_event_proofs
 * anchors it: the child header and the parent headers against t, the TxMeta recompute and the execution order rebuilt from the witness.
 * Then per proof: its position in that order (UINT64_MAX when absent) must be exec_index, the receipt at that position (or its absence)
 * every receipt field with the return data compared against data_blob, and with IPCFP_MESSAGE_WITH_BODY the message block every body
 * field with the params compared against data_blob. results[i] = 1 when proof i states exactly what the witness holds, its unnamed
 * bytes zero; headers that do not match t give 0 for every proof. A missing witness block or a decode error fails the call at that
 * proof, as ipcfp_verify_actor_proofs does. IPCFP_ERR_INVALID_ARG: NULL arrays with n > 0, n > IPCFP_MESSAGE_MAX, a flag bit other
 * than IPCFP_MESSAGE_WITH_BODY and IPCFP_WITNESS_BY_REFERENCE. */
ipcfp_status ipcfp_verify_message_proofs(ipcfp_store* witness_store, const ipcfp_tipset_desc* t, const ipcfp_message_proof* proofs, uint64_t n,
                                         const uint8_t* data_blob, uint64_t data_blob_size, uint32_t flags, uint8_t* results);

/* ------------------------------------------------------------------------------------------
 * Wire format (src/proofs/common/bundle.rs:10-45, src/proofs/events/bundle.rs:5-30, src/proofs/storage/bundle.rs:5-14): the JSON
 * `serde_json::to_string` gives for UnifiedProofBundle / EventProofBundle — struct field order, compact, CIDs as "bafy2bzace…"
 * strings, "0x" lower-case hex, base64 block data (ProofBlock.cid as the byte array cid 0.11's Serialize emits). t supplies the
 * fields every proof of the bundle shares (epochs, parent tipset CIDs, child block CID, parent state root). Host-side rendering:
 * no device is needed. *out is a NUL-terminated string of *out_len bytes, released with ipcfp_json_free.
 * ------------------------------------------------------------------------------------------ */
ipcfp_status ipcfp_bundle_to_json(const ipcfp_bundle* b, const ipcfp_tipset_desc* t, char** out, uint64_t* out_len);
ipcfp_status ipcfp_event_result_to_json(const ipcfp_event_result* r, const ipcfp_tipset_desc* t, char** out, uint64_t* out_len);
void ipcfp_json_free(char* p);

/* The way back (csrc/bundle_parse.cpp, host C++): what serde_json::from_str::<UnifiedProofBundle> / ::<EventProofBundle> reads, as
 * the PODs the batched verifiers below take and the flat block arrays ipcfp_store_create takes for the witness store. `tipset` holds
 * the fields every proof of the bundle shares (parent_epoch, child_epoch, n_parents, parent_cids, child_cid,
 * child_parent_state_root; the other members are NULL / 0); a bundle whose proofs disagree on them, CIDs that are not 38 bytes or
 * topics that are not 32 bytes are refused with IPCFP_ERR_UNSUPPORTED, malformed JSON / hex / base32 / base64 with
 * IPCFP_ERR_INVALID_ARG. Blocks are kept in the order given (16-byte aligned inside `witness.blob`); storage proofs come back with
 * found = 1, raw_len = 32 (the wire format carries the padded value only). No device is needed. */
typedef struct ipcfp_parsed_bundle {
    ipcfp_tipset_desc tipset;
    uint64_t n_storage_proofs;
    const ipcfp_storage_proof* storage_proofs;
    uint64_t n_event_proofs;
    const ipcfp_event_proof* event_proofs;
    const uint8_t* data_blob;          /* topics / data of the event proofs (topics_off / data_off index it) */
    uint64_t data_blob_size;
    ipcfp_witness witness;             /* Vec<ProofBlock> */
} ipcfp_parsed_bundle;
ipcfp_status ipcfp_bundle_from_json(const char* json, uint64_t len, ipcfp_parsed_bundle** out);
void ipcfp_parsed_bundle_free(ipcfp_parsed_bundle* b);

/* ------------------------------------------------------------------------------------------
 * Batched verifiers (src/proofs/events/verifier.rs:51-290, src/proofs/storage/verifier.rs:24-170): replay every proof against a
 * store that holds ONLY the witness blocks. Create that store with IPCFP_STORE_VERIFY_CIDS: this is the Blake2b-256 check of every
 * witness block the reference's load_witness_store leaves out (`put_keyed`, events/verifier.rs:79-89). results[i] = the reference's
 * Ok(bool) for proof i; an Err of the reference (missing witness block, decode failure, TxMeta mismatch) fails the call, index =
 * the first proof that meets it. Trust anchors (:124-144) are host-side policy closures and stay with the caller; `filter` (may
 * be NULL) plays check_event: the event must satisfy matches_log of that spec (events/generator.rs:38-40).
 * t: parent_cids / n_parents / epochs / child_cid (events), child_cid / child_parent_state_root (storage) — the fields every
 * proof of one bundle shares (EventProof.parent_tipset_cids …, StorageProof.parent_state_root).
 * ------------------------------------------------------------------------------------------ */
ipcfp_status ipcfp_verify_event_proofs(ipcfp_store* witness_store, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs, uint64_t n_proofs,
                                       const uint8_t* data_blob, uint64_t data_blob_size, const ipcfp_event_spec* filter, uint8_t* results);
ipcfp_status ipcfp_verify_storage_proofs(ipcfp_store* witness_store, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs, uint64_t n_proofs,
                                         uint8_t* results);
/* ipcfp_verify_event_proofs with a log filter as check_event (never NULL): a proof that verifies is true only when its event matches
 * `filter` (emitter set included). Invalid filters are refused as by ipcfp_generate_log_proof. */
ipcfp_status ipcfp_verify_event_proofs_log(ipcfp_store* witness_store, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs,
                                           uint64_t n_proofs, const uint8_t* data_blob, uint64_t data_blob_size, const ipcfp_log_filter* filter,
                                           uint8_t* results);
/* ipcfp_verify_event_proofs with a set of log filters as check_event: results[i] = OR over k of what ipcfp_verify_event_proofs_log gives
 * with filters[k] for proof i. n_filters == 0: no check_event (ipcfp_verify_event_proofs with filter NULL). The check is the last step
 * of a proof's verification, so the status and index of a failing call never depend on the filters: they are those of the unfiltered
 * call. A refused filter gives IPCFP_ERR_INVALID_ARG with its position as the index. This verifies a bundle of
 * ipcfp_generate_log_bundle against the filters it was made from. */
ipcfp_status ipcfp_verify_event_proofs_any(ipcfp_store* witness_store, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs,
                                           uint64_t n_proofs, const uint8_t* data_blob, uint64_t data_blob_size, const ipcfp_log_filter* filters,
                                           uint64_t n_filters, uint8_t* results);

/* ------------------------------------------------------------------------------------------
 * verify_proof_bundle (src/proofs/verifier.rs:12-60) from the JSON text: parse, witness store and verification on the GPU.
 * Accepts EventProofBundle and UnifiedProofBundle text. The result is, in every case, what this composition of the calls above gives:
 *   1. ipcfp_bundle_from_json on the text: its failure status is returned (index UINT64_MAX);
 *   2. trust (verify_trust_anchors / verify_trust_anchor): trusted_child is called once (if the bundle has a proof) with the child epoch
 *      and child block CID, then trusted_parent once (if it has event proofs and the child is trusted) with the parent epoch and parent
 *      tipset CIDs. Both run on the calling thread; non-zero = trusted; NULL = AcceptAll. Untrusted child: every result is false.
 *      Untrusted parent: every event result is false;
 *   3. if a trusted proof is left: a witness store of the blocks in bundle order with IPCFP_STORE_VERIFY_CIDS — a digest mismatch
 *      returns IPCFP_ERR_CID_MISMATCH with the block's position in the bundle as the index (duplicates and up to 8 CID prefixes as in
 *      ipcfp_store_create). With no trusted proof no store is built and the call succeeds whatever the blocks hold;
 *   4. ipcfp_verify_storage_proofs on the trusted storage proofs, then ipcfp_verify_event_proofs on the trusted event proofs with
 *      `filter` (check_event, may be NULL). A verifier failure fails the call; its index counts storage proofs first, then event proofs.
 * Canonical text (what serde_json::to_string, ipcfp_bundle_to_json, ipcfp_event_result_to_json and IPCFP_RESULT_JSON write) is parsed
 * on the device straight into the witness store (parsed_on_device = 1); any other spelling — whitespace, escapes, other key orders or
 * fields, other CID spellings, upper-case hex, out-of-range values — is read by ipcfp_bundle_from_json instead (parsed_on_device = 0),
 * with identical results. *out is released with ipcfp_bundle_verdict_free.
 * ------------------------------------------------------------------------------------------ */
typedef int (*ipcfp_trusted_parent_ts_fn)(void* ctx, int64_t parent_epoch, const uint8_t* parent_cids /* n_parents*38 */, uint32_t n_parents);
typedef int (*ipcfp_trusted_child_header_fn)(void* ctx, int64_t child_epoch, const uint8_t* child_cid /* 38 */);
typedef struct ipcfp_bundle_verdict {
    ipcfp_tipset_desc tipset;                  /* the fields every proof shares, as ipcfp_parsed_bundle.tipset                   */
    uint64_t n_storage_proofs;
    const ipcfp_storage_proof* storage_proofs; /* as ipcfp_bundle_from_json returns them                                         */
    const uint8_t* storage_results;            /* UnifiedVerificationResult.storage_results (0 / 1)                              */
    uint64_t n_event_proofs;
    const ipcfp_event_proof* event_proofs;
    const uint8_t* event_results;              /* UnifiedVerificationResult.event_results (0 / 1)                                */
    const uint8_t* data_blob;                  /* topics / data of event_proofs                                                  */
    uint64_t data_blob_size;
    uint64_t n_blocks;                         /* witness blocks in the bundle                                                   */
    uint64_t witness_bytes;                    /* their decoded bytes (sum of the block lengths)                                 */
    uint32_t parsed_on_device;                 /* 1: device parser; 0: text not in canonical form, read by ipcfp_bundle_from_json */
    /* wall time of the call and of its phases, milliseconds (each phase ends in a host synchronisation): parse (text to PODs and
     * block arrays, including the text's copy to the device), store (witness store with its CID check), verify (both verifiers) */
    float ms_total, ms_parse, ms_store, ms_verify;
    uint32_t _pad;
} ipcfp_bundle_verdict;
ipcfp_status ipcfp_verify_bundle_json(const char* json, uint64_t len, int device, ipcfp_trusted_parent_ts_fn trusted_parent,
                                      ipcfp_trusted_child_header_fn trusted_child, void* trust_ctx, const ipcfp_event_spec* filter,
                                      ipcfp_bundle_verdict** out);
/* ipcfp_verify_bundle_json with "matches at least one of filters[]" as check_event: steps 1–4 above, step 4 calling
 * ipcfp_verify_event_proofs_any (n_filters == 0: no check_event). Every filter is checked first: a refused filter gives
 * IPCFP_ERR_INVALID_ARG with its position as the index. */
ipcfp_status ipcfp_verify_bundle_json_any(const char* json, uint64_t len, int device, ipcfp_trusted_parent_ts_fn trusted_parent,
                                          ipcfp_trusted_child_header_fn trusted_child, void* trust_ctx, const ipcfp_log_filter* filters,
                                          uint64_t n_filters, ipcfp_bundle_verdict** out);
void ipcfp_bundle_verdict_free(ipcfp_bundle_verdict* v);

/* ------------------------------------------------------------------------------------------
 * Multi-GPU (one process per GPU; the library runs the collectives itself, over NCCL).
 * Receipts shard by index range; each rank scans its shard, and one call per rank resolves what spans
 * shards: the execution order, the proofs' message CIDs and the union of the per-shard witness CID sets.
 * ------------------------------------------------------------------------------------------ */
/* In-library protocol (the reference's future-work "Parallel Generation", README.md:384; SURVEY Appendix C): one communicator
 * per process/GPU over NCCL (resolved with dlopen("libnccl.so.2") at init — the library itself links only cudart). Rank 0 makes
 * the id and hands the 128 bytes to the other ranks by any means (MPI, a file, torch.distributed …).
 * ipcfp_generate_event_proof_sharded = generate_event_proof (src/proofs/events/generator.rs:60-107) for ONE tipset whose
 * receipts are split by index range bounds[rank] .. bounds[rank+1] (bounds: world+1 ascending values, bounds[0] = 0,
 * bounds[world] = n_receipts); every rank's store holds the blocks its range needs (events blocks, receipts-AMT paths, its share
 * of the message AMTs, the shared top levels). Inside the call: all-to-all + all-reduce for the first-seen dedup of the
 * execution order (src/proofs/events/utils.rs:48-94), exec index → message CID fetch for the rank's proofs, and the union of the
 * per-shard witness CID sets (range-partitioned all-to-all + merge; see ipcfp_event_result.union_*). All ranks must make the call; they succeed or fail together and a
 * failure names the same (status, index) everywhere — the one the reference's sequential order meets first over all shards.
 * Errors: IPCFP_ERR_NCCL (library missing / communicator failure). */
#define IPCFP_COMM_ID_BYTES 128
typedef struct ipcfp_comm ipcfp_comm;
ipcfp_status ipcfp_comm_unique_id(uint8_t id[IPCFP_COMM_ID_BYTES]);
ipcfp_status ipcfp_comm_init(const uint8_t id[IPCFP_COMM_ID_BYTES], uint32_t world_size, uint32_t rank, int device, ipcfp_comm** out);
void ipcfp_comm_destroy(ipcfp_comm* c);
ipcfp_status ipcfp_generate_event_proof_sharded(ipcfp_comm* c, ipcfp_store* s, ipcfp_tipset* t, const ipcfp_event_spec* spec,
                                                const uint64_t* bounds /* world_size + 1 */, uint32_t flags, ipcfp_event_result** out);

/* One shard's scan on its own, without the cross-shard steps: receipts [lo, hi) only; events_roots/has_events_root in t cover
 * ALL n_receipts. See ipcfp_event_result.shard_exec_dev for what the result leaves unresolved. */
ipcfp_status ipcfp_generate_event_proof_shard(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_spec* spec,
                                              uint64_t lo, uint64_t hi, uint32_t world_size, uint32_t rank,
                                              uint32_t flags, ipcfp_event_result** out);

#ifdef __cplusplus
}
#endif
#endif /* IPCFP_H */
