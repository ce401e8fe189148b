// engine.cuh — host-side objects of the engine (C++17), shared by the translation units.
#pragma once
#include <array>
#include <chrono>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "store.cuh"
#include "rawcid.cuh"

namespace ipcfp {

// Grow-only cache of pinned host buffers so result read-backs run at PCIe rate without paying
// cudaHostAlloc on every call.
// Pinned host buffers should live on the NUMA node the GPU's PCIe root hangs off: a D2H / H2D that crosses the socket
// interconnect loses bandwidth, and with one process per GPU on a two-socket box half of the ranks would otherwise land
// on the far socket. Best effort and silent: the node comes from sysfs, the preference is a thread-local mempolicy
// (MPOL_PREFERRED, so allocation never fails because of it) that lasts for the lifetime of this guard.
struct NumaPrefer {
    bool on = false;
    int old_mode = 0;
    unsigned long old_mask[16] = {};   // the caller's own policy (e.g. numactl) is put back afterwards
    explicit NumaPrefer(int device);
    ~NumaPrefer();
};

struct PinnedPool {
    struct Buf { void* p; size_t cap; };
    std::mutex mu;
    std::vector<Buf> free_list;
    ~PinnedPool();
    void* take(size_t bytes, size_t* cap_out);
    void give(void* p, size_t cap);
};
struct PinnedArray {
    std::shared_ptr<PinnedPool> pool;
    void* p = nullptr;
    size_t cap = 0;
    PinnedArray() {}
    PinnedArray(std::shared_ptr<PinnedPool> pl, size_t bytes) : pool(std::move(pl)) { p = pool->take(bytes ? bytes : 16, &cap); }
    PinnedArray(const PinnedArray&) = delete;
    PinnedArray& operator=(const PinnedArray&) = delete;
    PinnedArray(PinnedArray&& o) noexcept : pool(std::move(o.pool)), p(o.p), cap(o.cap) { o.p = nullptr; }
    PinnedArray& operator=(PinnedArray&& o) noexcept { release(); pool = std::move(o.pool); p = o.p; cap = o.cap; o.p = nullptr; return *this; }
    ~PinnedArray() { release(); }
    void release() { if (p && pool) pool->give(p, cap); p = nullptr; }
    template <class T> T* as() const { return (T*)p; }
};

// ---- Timing and copy helpers of the host code
using Clock = std::chrono::steady_clock;
inline float ms_since(Clock::time_point t0) { return std::chrono::duration<float, std::milli>(Clock::now() - t0).count(); }

// a CUDA event that lives as long as its owner; converts to cudaEvent_t
struct Event {
    cudaEvent_t e = nullptr;
    explicit Event(unsigned flags = cudaEventDefault) { IPCFP_CUDA(cudaEventCreateWithFlags(&e, flags)); }
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    Event(Event&& o) noexcept : e(o.e) { o.e = nullptr; }
    ~Event() { if (e) cudaEventDestroy(e); }
    operator cudaEvent_t() const { return e; }
};
inline float elapsed_ms(cudaEvent_t a, cudaEvent_t b) {
    float ms = 0.f;
    IPCFP_CUDA(cudaEventElapsedTime(&ms, a, b));
    return ms;
}

// H2D copies of byte ranges on a stream of their own, one event per range, so that work on another stream can start on range k while
// the later ranges are still on the wire. The stream is drained before it is destroyed: the source is read for this object's lifetime.
struct ChunkedCopy {
    cudaStream_t st = nullptr;
    std::vector<Event> landed;
    ChunkedCopy() { IPCFP_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); }
    ChunkedCopy(const ChunkedCopy&) = delete;
    ChunkedCopy& operator=(const ChunkedCopy&) = delete;
    ~ChunkedCopy() { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
    // dst[byte0, byte1) = src[byte0, byte1); returns the range's event
    cudaEvent_t copy(uint8_t* dst, const uint8_t* src, uint64_t byte0, uint64_t byte1) {
        if (byte1 > byte0) IPCFP_CUDA(cudaMemcpyAsync(dst + byte0, src + byte0, byte1 - byte0, cudaMemcpyHostToDevice, st));
        landed.emplace_back(cudaEventDisableTiming);
        IPCFP_CUDA(cudaEventRecord(landed.back(), st));
        return landed.back();
    }
    void wait(cudaStream_t consumer, size_t k) const { IPCFP_CUDA(cudaStreamWaitEvent(consumer, landed[k], 0)); }
};

// ---- The store's counter words and events
// dev_words: one slot per counter or fault word a kernel writes. host_words[0, DW_COUNT) mirror them at the same index
// (publish_words(s, first, n) with first + n <= DW_COUNT); the host-only regions behind the mirror receive other device data.
enum DevWord : uint32_t {
    DW_ERR = 0,                            // first error key (report_error)
    DW_FRONTIER_A = 1, DW_FRONTIER_B = 2,  // general walk: frontier counters (ping / pong); k_setup seeds A
    DW_UNKNOWN_CLASSES = 1,                // store ingest: CIDs of no known class
    DW_FIRST_BAD = 2,                      // store ingest: first block whose CID does not match its bytes
    DW_N_EXEC = 3,
    DW_STATS = 4,                          // 4 / 5: nodes / bytes pass 1 (or the slot lookup) read
    DW_N_MATCH = 6,
    DW_N_PROOFS = 7,
    DW_WIT_A = 8, DW_WIT_A_BYTES = 9,      // witness snapshot: blocks, padded bytes
    DW_WIT_B = 10, DW_WIT_B_BYTES = 11,    // late witness blocks, padded bytes
    DW_BLOB_BYTES = 12,                    // topics / data bytes of the proofs
    DW_LEVEL_TOTAL = 13,                   // general walk: the level's exact total
    DW_DENSE_FAIL = 14,                    // the dense walk gave up
    DW_TX_ERR = 15,                        // message-AMT fault key (tx_err_key)
    DW_SPLIT_IDX = 16, DW_SPLIT_BYTES = 17,  // witness gather split: blocks and bytes of the first part
    DW_UNION_SIZE = 18,                    // sharded: size of the replicated witness union
    DW_EXEC_CHECK = 19,                    // sharded: error key of the exec.get check
    DW_JSON_TOTAL0 = 24, DW_JSON_TOTAL1 = 25, DW_JSON_OVERFLOW = 26, DW_JSON_TOTAL2 = 27,
    DW_COUNT = 64
};
constexpr uint32_t MAX_WORLD = 255;   // ranks of one sharded call
// Host-only regions of host_words, each right behind the previous one. The sizes of types defined in a .cu file are asserted there.
constexpr uint32_t HW_PROLOGUE_WORDS = 230;                                   // events.cu: the head of Prologue
constexpr uint32_t HW_JSON_TOTALS_WORDS = DW_JSON_TOTAL2 - DW_JSON_TOTAL0 + 1;  // json.cu: list totals and overflow flag
constexpr uint32_t HW_ANY_SKIP_WORDS = 2;                                     // events.cu: Prologue::misc[0..3], misc[2] = any_skip
constexpr uint32_t HW_PARKED_KEY_WORDS = 1;                                   // verify.cu: the TxMeta check's error key
constexpr uint32_t HW_EXCHANGE_WORDS = 2;                                     // parallel.cu: exchange overflow flag, n_exec
constexpr uint32_t HW_UNION_PARTS_WORDS = 2 * MAX_WORLD;                      // parallel.cu: [partition size, overflow] per rank
constexpr uint32_t HW_PARSE_META_WORDS = 17;                                  // the meta of a device parse: JpMeta (json_parse.cu), the largest
enum HostWord : uint32_t {
    HW_PROLOGUE = DW_COUNT,
    HW_JSON_TOTALS = HW_PROLOGUE + HW_PROLOGUE_WORDS,
    HW_ANY_SKIP = HW_JSON_TOTALS + HW_JSON_TOTALS_WORDS,
    HW_PARKED_KEY = HW_ANY_SKIP + HW_ANY_SKIP_WORDS,
    HW_EXCH_OVERFLOW = HW_PARKED_KEY + HW_PARKED_KEY_WORDS, HW_EXCH_N_EXEC = HW_EXCH_OVERFLOW + 1,
    HW_UNION_PARTS = HW_EXCH_OVERFLOW + HW_EXCHANGE_WORDS,
    HW_PARSE_META = HW_UNION_PARTS + HW_UNION_PARTS_WORDS,   // one parse at a time per store: each parses on a fresh store_shell, or
                                                             // (rpc_json.cu) inside a call on the caller's store, and those are serialised
    HW_END = HW_PARSE_META + HW_PARSE_META_WORDS
};
constexpr uint32_t HW_COUNT = 1024;
static_assert(DW_JSON_TOTAL2 < DW_COUNT, "a mirrored slot never reaches a host-only region (they start at DW_COUNT)");
static_assert(HW_EXCH_N_EXEC < HW_UNION_PARTS, "the exchange words fit their region");
static_assert(HW_END <= HW_COUNT, "the host-only regions fit the mapped words");
// Store::ev: the event-proof step's timeline. storage.cu gives slots 1..3 meanings of its own.
enum StoreEvent : uint32_t {
    EV_BEGIN = 0,
    EV_SETUP = 1, EV_STORAGE_END = 1,
    EV_EXEC_ORDER = 2, EV_LOOKUP_BEGIN = 2,   // execution order done (walk, snapshot, dedup)
    EV_PASS1 = 3, EV_LOOKUP_END = 3,
    EV_PASS2 = 4,
    EV_END = 5,
    EV_WITNESS_SORTED = 6,   // the sorted witness CID list exists on the device (also: the first gather part, for its D2H)
    EV_BLOB_COPIED = 7,      // the witness blob's D2H is done (side stream)
    EV_GATHER_B = 8,         // the second gather part, for its D2H
    EV_RAW_LIST = 9,         // the raw message list of the call is complete (the cross-shard exchange waits for it)
    EV_JSON_BEGIN = 10, EV_JSON_END = 11,
    EV_COUNT = 12
};

struct Store {
    int device = 0;
    cudaStream_t stream = nullptr, stream2 = nullptr;
    unsigned walk_grid = 0;               // CTAs of the persistent message-AMT walk kernels (from their occupancy, set on first use)
    uint64_t n = 0, blob_size = 0;
    DevBuf<uint8_t> arena;
    DevBuf<uint64_t> offsets;
    DevBuf<uint32_t> lengths;
    DevBuf<Digest> digests;
    DevBuf<uint8_t> cls;
    DevBuf<uint64_t> table;
    DevBuf<BlockRec> recs;
    DevBuf<uint32_t> rank_of, block_at_rank;   // `Cid` Ord rank of every block and its inverse (witness bitmaps are indexed by rank)
    StoreView view{};
    DevBuf<StoreView> view_dev;   // device copy, for out-of-line device functions (keeps kernel params off the stack)
    std::vector<std::array<uint8_t, 6>> class_prefix;  // distinct CID prefixes in this store
    std::vector<uint32_t> class_rank;                  // rank of each class in `Cid` Ord
    uint64_t first_bad = UINT64_MAX;
    bool caller_blob = true;   // false: made from JSON-RPC texts (rpc_blocks.cu), no caller blob for IPCFP_WITNESS_BY_REFERENCE offsets
                               // (a store made from a CAR keeps true: its blob is the caller's CAR)
    std::shared_ptr<PinnedPool> pool;
    // small persistent scratch
    DevBuf<unsigned long long> dev_words;  // DW_COUNT slots (DevWord)
    PinnedBuf<uint64_t> host_words;        // HW_COUNT mapped words (HostWord)
    PinnedArray stage;                     // pinned staging (from the process-wide pool) for small per-call uploads: spec, tipset CIDs, walk tables
    cudaEvent_t ev[EV_COUNT] = {};
    ~Store();
    void use() const { IPCFP_CUDA(cudaSetDevice(device)); }
};

// Device-resident copy of an ipcfp_tipset_desc (events roots etc.)
struct TipsetDev {
    int64_t parent_epoch = 0, child_epoch = 0;
    uint32_t n_parents = 0;
    std::vector<uint8_t> parent_cids, txmeta_cids;  // host copies (tiny)
    uint8_t child_cid[38] = {}, receipts_root[38] = {}, child_state_root[38] = {};
    bool has_state_root = false;
    uint64_t n_receipts = 0;
    DevBuf<uint8_t> events_roots;  // n*38
    DevBuf<uint8_t> has_root;      // n
    int device = 0;
    // ipcfp_tipset_upload_json: which path parsed the receipt list and its wall time; ipcfp_tipset_describe: the host copies of the
    // receipt arrays (made on its first request)
    bool parsed_on_device = false;
    float ms_parse = 0.f, ms_kernels = 0.f;
    std::vector<uint8_t> host_roots, host_has;
};

struct ScopedStatus;  // capi.cu
struct Comm;          // parallel.cu: NCCL communicator pair + exchange scratch of one rank

void set_last_error(const std::string& msg, uint64_t index);

// store.cu
Store* store_create(const uint8_t* cids, const uint64_t* offsets, const uint32_t* lengths, const uint8_t* blob, uint64_t blob_size,
                    uint64_t n, int device, uint32_t flags);
void store_get(Store* s, const uint8_t* cid, uint8_t* buf, uint32_t cap, uint32_t* len, int* found);
void hash_batch(int which, const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets, const uint32_t* lengths, uint64_t n, int device,
                uint8_t* out);
void mapping_slots(const uint8_t* keys32, const uint64_t* slot_indices, uint64_t n, int device, uint8_t* out);
void check_device(int device);
// the pieces of store_create, for a caller that writes the blocks on the device itself:
//   store_shell → store_alloc_blocks → (fill cids_dev, offsets, lengths and the blocks) → store_finish
Store* store_shell(int device);   // stream, events, counters; no block yet
// n blocks of blob_size bytes: the arena with its pads zeroed (zero_blocks: all of it), the per-block arrays, cids_dev (n*38) and the
// zeroed hash table, on the store's stream. Returns where block bytes go: offsets index from there.
uint8_t* store_alloc_blocks(Store* s, uint64_t n, uint64_t blob_size, DevBuf<uint8_t>& cids_dev, bool zero_blocks);
// … its two halves, for a caller that fills the arena before it knows n (car.cu): the arena, then the per-block arrays and the index
uint8_t* store_alloc_arena(Store* s, uint64_t blob_size, bool zero_blocks);
void store_alloc_index(Store* s, uint64_t n, DevBuf<uint8_t>& cids_dev);
// the index of the blocks in place, then the CID check of IPCFP_STORE_VERIFY_CIDS in `flags` (first_bad) or a plain synchronisation.
// cids_host: the CIDs on the host, or null; first_prefix: the first CID's 6 prefix bytes (host). blob: the block bytes still landing,
// blocks [bounds[k], bounds[k + 1]) in its range k (null: all on the device already).
void store_finish(Store* s, const uint8_t* cids_dev, const uint8_t* cids_host, const uint8_t* first_prefix, uint32_t flags,
                  const ChunkedCopy* blob = nullptr, const std::vector<uint64_t>& bounds = {});
// A store from input that has a host parser: on_device(store, t0) on a fresh store when try_device and the device is there (false: it
// declined, and the store is dropped); otherwise host_parse's blocks through store_create, over `blob` (null: the parsed blocks' own).
// info is cleared first, and again when the device path declines; the host path sets its ms_parse.
Store* store_create_parsed(int device, uint32_t flags, ipcfp_store_json_info& info, bool try_device,
                           const std::function<bool(Store*, Clock::time_point)>& on_device,
                           const std::function<ipcfp_status(ipcfp_parsed_blocks**)>& host_parse, const uint8_t* blob);
// rpc_blocks.cu — ipcfp_store_create_rpc_json (info: which path ran, its times)
Store* store_create_rpc_json(const uint8_t* cids, uint64_t n_blocks, const char* const* texts, const uint64_t* text_lens, uint64_t n_texts, int device,
                             uint32_t flags, ipcfp_store_json_info& info);
// car.cu — ipcfp_store_create_car (info: which path ran, its times)
Store* store_create_car(const uint8_t* car, uint64_t len, int device, uint32_t flags, ipcfp_store_json_info& info);
// n_words device words at src_dev (null: the mirrored dev_words[dst_first ..]) → host_words[dst_first ..) through mapped host memory,
// on `stream` (null: the store's stream): a tiny kernel instead of a D2H copy, so the read-back never queues behind a large copy on
// the copy engine
void publish_words(Store* s, uint32_t dst_first, uint32_t n_words, const void* src_dev = nullptr, cudaStream_t stream = nullptr);

// events.cu
void tipset_upload(Store* s, const ipcfp_tipset_desc* t, TipsetDev& td);
// rpc_json.cu — ipcfp_tipset_upload_json / ipcfp_tipset_describe
void tipset_upload_json(Store* s, const char* parent, uint64_t parent_len, const char* child, uint64_t child_len, const char* receipts,
                        uint64_t receipts_len, TipsetDev& td);
void tipset_describe(TipsetDev& td, bool with_roots, ipcfp_tipset_info* out);
// the reconstructed execution order of a tipset on the device (reconstruct_execution_order, events/utils.rs:16-30): exec[i] = exec_raw[exec_idx[i]]
struct ExecOrderOut {
    uint64_t n_exec = 0;
    AsyncBuf<RawCid> exec_raw;
    AsyncBuf<uint32_t> exec_idx;
};
// the execution order of a tipset of n_parents parent blocks, from their TxMeta CIDs (n_parents*38, host): the message-AMT walk and the
// dedup that generate_event_proof runs, with no witness and no receipts root (the batched verifier, the message fetch round)
void build_execution_order(Store* s, uint32_t n_parents, const uint8_t* txmeta_cids, ExecOrderOut& out);
ipcfp_event_result* generate_event_proof(Store* s, TipsetDev& td, const ipcfp_event_spec* spec, uint32_t flags, bool sharded, uint64_t lo, uint64_t hi,
                                         Comm* comm = nullptr);
// ipcfp_generate_log_proof_resident: the same call with a log filter as the predicate
ipcfp_event_result* generate_log_proof(Store* s, TipsetDev& td, const ipcfp_log_filter* filter, uint32_t flags);
// ipcfp_generate_message_log_proof_resident: that call with its receipt loop restricted to the receipts of message_cids (n*38, host);
// filter null: every log extract_evm_log accepts. exec_indices[j] (host): request j's execution position, UINT64_MAX when not executed.
ipcfp_event_result* generate_message_log_proof(Store* s, TipsetDev& td, const uint8_t* message_cids, uint64_t n, const ipcfp_log_filter* filter,
                                               uint32_t flags, uint64_t* exec_indices);
// The refusals of a message call, made before any device work: null CIDs with a nonzero count (with_exec: or null exec_indices, which
// the generators write and the fetch plan does not take), more than IPCFP_MESSAGE_MAX CIDs, a refused filter (null: every log)
void message_request_check(const uint8_t* message_cids, uint64_t n, const ipcfp_log_filter* filter, bool with_exec, const uint64_t* exec_indices);
// The host half of EventMatcher::new (events/generator.rs:30-35): m = the spec's t1 = ascii_to_bytes32(topic_1) and actor filter, t0 zero
// (keccak256 of the signature is the caller's, on the device). A spec or field that is null is refused with the message `refusal`.
struct Matcher;
void event_matcher(const ipcfp_event_spec* spec, const char* refusal, Matcher& m);
// plan.cu's selection: has_sel[i] (device, n_receipts) = the receipt has an events root and is selected by message_cids (n*38, host)
// against the execution order exo (the tipset's, built on this store); left as it is when nothing is selected
void message_selection_mask(Store* s, TipsetDev& td, const ExecOrderOut& exo, const uint8_t* message_cids, uint64_t n, uint8_t* has_sel);
// message proofs (message_proof.cu): the execution order of td built with its witness (k_setup's base witness, every message AMT, the
// receipts root; n_receipts only sizes the walk), and request j's position in it. Faults of the message AMTs and the receipts root are
// thrown as generate_message_log_proof throws them; a base-witness block the store lacks is left in missing_base. The call's device
// words are the walk's; DW_N_EXEC is published (read it after the next synchronisation).
struct MessagePositions {
    AsyncBuf<uint32_t> wbits;          // the witness bitmap, by Cid rank
    AsyncBuf<uint64_t> exec_indices;   // n+1: UINT64_MAX where the message is not executed
    uint32_t receipts_root_blk = 0;
    bool missing_base = false;
};
void message_positions(Store* s, TipsetDev& td, const uint8_t* message_cids, uint64_t n, uint32_t flags, MessagePositions& out);
// … and the same positions in an execution order already built (exo): exec_indices (device, n) as message_positions gives them
void message_exec_indices(Store* s, const ExecOrderOut& exo, const uint8_t* message_cids, uint64_t n, uint64_t* exec_indices);
// verify.cu — batched verifiers over a witness store; n_log_filters > 0: check_event is "matches at least one of log_filters[]", in place
// of `filter`
void verify_event_proofs(Store* s, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs, uint64_t n, const uint8_t* data_blob, uint64_t blob_size,
                         const ipcfp_event_spec* filter, uint8_t* results, const ipcfp_log_filter* log_filters = nullptr, uint64_t n_log_filters = 0);
void verify_storage_proofs(Store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs, uint64_t n, uint8_t* results);
// … the same with the proofs (and the data blob, padded by 16 bytes) already in device memory
void verify_event_proofs_dev(Store* s, const ipcfp_tipset_desc* t, const ipcfp_event_proof* d_proofs, uint64_t n, const uint8_t* d_blob, uint64_t blob_size,
                             const ipcfp_event_spec* filter, uint8_t* results, const ipcfp_log_filter* log_filters = nullptr, uint64_t n_log_filters = 0);
void verify_storage_proofs_dev(Store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* d_proofs, uint64_t n, uint8_t* results);
// json_parse.cu — ipcfp_verify_bundle_json
// (log_filters, n_log_filters): check_event of the event verifier, as verify_event_proofs takes it
ipcfp_bundle_verdict* verify_bundle_json(const char* json, uint64_t len, int device, ipcfp_trusted_parent_ts_fn trusted_parent,
                                         ipcfp_trusted_child_header_fn trusted_child, void* trust_ctx, const ipcfp_event_spec* filter,
                                         const ipcfp_log_filter* log_filters = nullptr, uint64_t n_log_filters = 0);
void bundle_verdict_free(ipcfp_bundle_verdict* v);
void event_result_free(ipcfp_event_result* r);
struct WitnessOut;
const WitnessOut& event_result_witness(const ipcfp_event_result* r);   // the witness of a generate_event_proof result, device copies included
// plan.cu — ipcfp_plan_fetch_resident: the CIDs of N(S) \ S for the generators of a proof bundle (DESIGN.md §2, "Fetch planning")
struct FetchPlan {
    std::vector<uint8_t> cids;   // n*38, `Cid` order
    uint64_t n_needed = 0;
    uint32_t n_levels = 0;
    float ms_total = 0.f;
};
// n_log_filters > 0 (with no event specs): rule 3's predicate is "matches at least one of log_filters[]", in place of the event specs'
// has_dev (device, n_receipts; null: the tipset's has-events-root flags): the receipts rules 1 and 3 take, those with a nonzero entry
void plan_fetch(Store* s, TipsetDev& td, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs, const ipcfp_event_spec* especs, uint64_t n_especs,
                FetchPlan& out, const ipcfp_log_filter* log_filters = nullptr, uint64_t n_log_filters = 0, const uint8_t* has_dev = nullptr);
// ipcfp_plan_fetch_message_log_resident: one round for generate_message_log_proof (filter null: the all-wildcard filter)
void plan_fetch_messages(Store* s, TipsetDev& td, const uint8_t* message_cids, uint64_t n, const ipcfp_log_filter* filter, FetchPlan& out);

// storage_path.cu — ipcfp_generate_storage_path_proofs_resident, ipcfp_plan_fetch_storage_paths_resident, ipcfp_verify_storage_paths
// (DESIGN.md §3, "Storage paths")
ipcfp_path_result* generate_storage_path_proofs(Store* s, TipsetDev& td, const ipcfp_storage_path* paths, uint64_t n, uint32_t flags);
void plan_fetch_storage_paths(Store* s, TipsetDev& td, const ipcfp_storage_path* paths, uint64_t n, FetchPlan& out);
ipcfp_path_result* verify_storage_paths(Store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs, uint64_t n_proofs,
                                        const ipcfp_storage_path* paths, uint64_t n_paths);
void path_result_free(ipcfp_path_result* r);

// parallel.cu — in-library cross-shard protocol over NCCL (one process per GPU)
void comm_unique_id(uint8_t* id128);
Comm* comm_init(const uint8_t* id128, uint32_t world, uint32_t rank, int device);
void comm_destroy(Comm* c);
uint32_t comm_world(const Comm* c);
uint32_t comm_rank(const Comm* c);
// One sharded generate_event_proof call's share of the protocol (see the banner in parallel.cu). generate_event_proof drives it:
//   agree_early or agree_slices → start_exchange → positions_for → agree_results → fetch_and_patch → witness_union → finish → fill_result
struct ShardExchange {
    Comm* c;
    Store* s;
    uint64_t lo, hi;
    // H0
    std::vector<uint64_t> nseg_all;
    uint64_t nraw = 0, max_nseg = 0, pos0 = 0, nseg = 0;
    bool peers_ok = true;
    bool all_early = false;          // early H0: every shard promised its slice before its walk was over
    // X
    const RawCid* seg = nullptr;
    uint64_t cap = 0, nwords = 0;
    unsigned long long* n_exec_dev = nullptr;
    unsigned long long* overflow_dev = nullptr;
    // P / F
    uint64_t M = 0;
    const uint32_t* match_rel_dev = nullptr;
    unsigned long long* n_exec_out = nullptr;
    // H0 / H2 (global values, identical on every rank)
    uint64_t g_tx = ~0ull, g_err = ~0ull;
    bool g_missing_base = false, g_overflow = false, g_stale = false;
    uint64_t M_max = 0, nw_max = 0, M_total = 0, proofs_total = 0;
    std::vector<uint64_t> nw_all;
    // W
    bool full_union = false;
    const uint8_t* wit_cids = nullptr;
    uint64_t wit_n = 0;
    uint8_t* union_dev = nullptr;
    ShardExchange(Comm* comm, Store* store, uint64_t lo_, uint64_t hi_);
    void agree_early(bool can_promise, uint64_t planned_nseg, uint64_t nraw_total);
    void agree_slices(uint64_t tx_key, uint64_t err_key, uint64_t nseg_);
    void start_exchange(const void* seg_dev);   // behind EV_RAW_LIST
    void positions_for(const uint32_t* match_rel, uint64_t n_match, unsigned long long* n_exec_out_);
    // H2 after the engine stream's pass-2 synchronisation; true: every shard goes on. A stale early promise repeats H0, X, P and H2.
    bool agree_results(uint64_t tx_key, uint64_t err_key, bool missing_base, uint64_t n_proofs, uint64_t n_witness, bool stale, const void* seg_dev,
                       uint64_t nseg_);
    void fetch_and_patch(ipcfp_event_proof* proofs_dev, uint64_t n_proofs, void* proofs_host);
    void witness_union(const uint8_t* cids_dev, uint64_t n_local, bool full);   // behind EV_WITNESS_SORTED
    void finish();                                                             // joins both protocol streams (the union's retry included)
    void fill_result(ipcfp_event_result& r) const;
    void trace_timeline(cudaEvent_t origin, const char* engine_part) const;
private:
    void gather_results(uint64_t tx_key, uint64_t err_key, bool missing_base, uint64_t n_proofs, uint64_t n_witness, uint64_t exch_overflow, bool stale);
    void patch(ipcfp_event_proof* proofs_dev, uint64_t n_proofs);
    void union_replicated(uint64_t* n_out_dev_word);
    // the union left distributed: this rank's partition (sorted) in union_dev; every rank's [partition size, overflow flag] lands in
    // host words HW_UNION_PARTS with the next sync of the union stream. Any overflow flag set: repeat with union_piece_cap(true).
    uint64_t union_piece_cap(bool cannot_overflow) const;
    void union_partitioned(uint64_t cap);
    void timings(float* ms_exchange, float* ms_fetch, float* ms_union) const;   // after the call's final sync
};

// storage.cu
ipcfp_slot_result* read_storage_slots(Store* s, const uint8_t* root, const uint8_t* slots, uint64_t k);
void slot_result_free(ipcfp_slot_result* r);
// child_cid / state_root: the child block's CID and its header's parent_state_root (38 bytes each, host memory)
ipcfp_storage_result* generate_storage_proofs(Store* s, const uint8_t* child_cid, const uint8_t* state_root, const ipcfp_storage_spec* specs, uint64_t n,
                                              bool by_ref = false);
void storage_result_free(ipcfp_storage_result* r);
const WitnessOut& storage_result_witness(const ipcfp_storage_result* r);
// generate_storage_proofs' second half: the result of n proofs already on the device in spec order (d_out, their recorder lists d_rec /
// d_recn, the witness bitmap they marked): copies, one materialize_witness, the per-spec lists. Its two host synchronisations are
// materialize_witness's, then one at the end; times from s->ev[EV_BEGIN] to s->ev[EV_STORAGE_END].
ipcfp_storage_result* storage_result_finish(Store* s, const ipcfp_storage_proof* d_out, const uint32_t* d_rec, const uint32_t* d_recn, const uint32_t* wbits,
                                            uint64_t n, bool by_ref);
// a storage failure's error key → the Error it throws (status by code, index from the key)
[[noreturn]] void throw_storage_error(uint64_t key);

// witness.cu — materialise a witness bitmap into a sorted ipcfp_witness (host, pinned)
struct WitnessOut {
    PinnedArray cids, offsets, lengths, blob;
    PinnedArray sorted_idx;       // host copy of the block indices in Cid order (u32[n])
    AsyncBuf<uint8_t> cids_dev;   // the same sorted CIDs in device memory (n*38), for the multi-GPU union
    AsyncBuf<uint32_t> idx_dev;   // block index of every entry in device memory (n), for the JSON renderer
    uint64_t n = 0, blob_size = 0;
    void fill(ipcfp_witness& w) const {
        w.n_blocks = n; w.cids = cids.as<uint8_t>(); w.offsets = offsets.as<uint64_t>(); w.lengths = lengths.as<uint32_t>();
        w.blob = blob.as<uint8_t>(); w.blob_size = blob_size;
    }
};
// Two-phase witness materialisation (see witness.cu): snapshot → start_copy → finish_enqueue → finish.
struct WitnessBuilder {
    Store* s;
    cudaStream_t st, st2;
    uint64_t nwords = 0, mA = 0, mB = 0, bytesA = 0, bytesB = 0, host_cap = 0;
    bool have_snapshot = false;
    bool by_ref = false;          // IPCFP_WITNESS_BY_REFERENCE: no block bytes are gathered or copied; offsets are the store's own
    AsyncBuf<uint32_t> idx, plen, bitsA, bitsB;
    AsyncBuf<uint64_t> offs, word_prefix, word_prefixB, scratch;
    AsyncBuf<uint8_t> dblobA, dblobB_keep;
    PinnedArray host_blob;
    explicit WitnessBuilder(Store* store);
    void snapshot(const uint32_t* wbits);        // enqueue; count → dev_words[8]
    // host knows the counts: gather in two parts (the first split_idx blocks = split_bytes bytes, then the rest) so that the D2H of
    // the first part is on the wire while the second is still being gathered
    void start_copy(uint64_t mA, uint64_t bytesA, uint64_t split_idx, uint64_t split_bytes);
    void finish_enqueue(const uint32_t* wbits);  // enqueue; late-block count → dev_words[10], their padded bytes → dev_words[11]
    // late blocks (mB of them, bytesB padded bytes: dev_words[10] and [11] after finish_enqueue), Cid-order index arrays, join
    void finish(uint64_t mB, uint64_t bytesB, WitnessOut& out, bool want_sorted_idx = false);
    void finish_start(uint64_t mB, uint64_t bytesB, WitnessOut& out, bool want_sorted_idx = false);   // … the same without the join: everything enqueued
    void finish_join(WitnessOut& out);                                              // … wait for both streams
};
void materialize_witness(Store* s, const uint32_t* wbits_dev, WitnessOut& out, bool by_ref = false);
// the union of witness lists of this store (the BTreeSet<(Cid, data)> of generate_proof_bundle): every entry's block marks its rank in a
// fresh bitmap (block indices from WitnessOut::idx_dev), which is then materialised as one witness, in `Cid` order
void witness_union(Store* s, const std::vector<const WitnessOut*>& lists, WitnessOut& out, bool by_ref);

// resolve.cu — ipcfp_resolve_addresses (DESIGN.md §2, "Address resolution") and the host-side address codecs
struct ResolveOut {
    std::vector<uint64_t> ids;
    std::vector<int32_t> status;
    int32_t init_status = IPCFP_OK;
    std::vector<uint8_t> missing;   // n*38, unique, `Cid` order
    WitnessOut wit;
    float ms_total = 0.f, ms_lookup = 0.f;
};
void resolve_addresses(Store* s, const uint8_t* state_root, const ipcfp_address* addrs, uint64_t n, ResolveOut& out);
void address_parse(const char* text, uint64_t len, ipcfp_address& out);
void address_from_eth(const uint8_t eth[20], ipcfp_address& out);

// actor.cu — ipcfp_generate_actor_proofs_resident (DESIGN.md §2, "Actor proofs"); the planner (plan.cu) and the verifier (verify.cu) share
// its refusals and its upload
struct ActorArgs;
// the refusals made before any device work (include/ipcfp.h); returns the number of addresses that are not ID addresses
uint64_t actor_request_check(const ipcfp_address* addrs, uint64_t n, const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags);
// one upload of a call's inputs (the child CID, the state root, the EVM code CIDs, the addresses) on the store's stream
struct ActorUpload {
    AsyncBuf<uint8_t> d;
    uint64_t o_evm = 0, o_addrs = 0;
    ActorUpload(Store* s, const uint8_t* child_cid, const uint8_t* state_root, const ipcfp_address* addrs, uint64_t n, const uint8_t* evm,
                uint64_t n_evm);
    void fill(ActorArgs& a, const StoreView& v, uint64_t n, uint64_t n_evm, uint32_t flags) const;   // inputs, sizes, flags
};
ipcfp_actor_result* generate_actor_proofs(Store* s, TipsetDev& td, const ipcfp_address* addrs, uint64_t n, const uint8_t* evm_code_cids, uint64_t n_evm,
                                          uint32_t flags);
void actor_result_free(ipcfp_actor_result* r);
// message_proof.cu — ipcfp_generate_message_proofs_resident (DESIGN.md §2, "Message proofs"); its refusals come before any device work
void message_proof_check(const uint8_t* message_cids, uint64_t n, uint32_t flags);
ipcfp_message_result* generate_message_proofs(Store* s, TipsetDev& td, const uint8_t* message_cids, uint64_t n, uint32_t flags);
void message_result_free(ipcfp_message_result* r);
// plan.cu — ipcfp_plan_fetch_message_proofs_resident; verify.cu — ipcfp_verify_message_proofs
void plan_fetch_message_proofs(Store* s, TipsetDev& td, const uint8_t* message_cids, uint64_t n, uint32_t flags, FetchPlan& out);
void verify_message_proofs(Store* s, const ipcfp_tipset_desc* t, const ipcfp_message_proof* proofs, uint64_t n, const uint8_t* data_blob,
                           uint64_t blob_size, uint32_t flags, uint8_t* results);
// plan.cu — ipcfp_plan_fetch_actor_proofs_resident; verify.cu — ipcfp_verify_actor_proofs
void plan_fetch_actor_proofs(Store* s, TipsetDev& td, const ipcfp_address* addrs, uint64_t n, const uint8_t* evm_code_cids, uint64_t n_evm,
                             uint32_t flags, FetchPlan& out);
void verify_actor_proofs(Store* s, const ipcfp_tipset_desc* t, const ipcfp_actor_proof* proofs, uint64_t n, const uint8_t* evm_code_cids,
                         uint64_t n_evm, uint32_t flags, uint8_t* results);

// json.cu — IPCFP_RESULT_JSON: the EventProofBundle text of one call from what is on the device after k_witness_emit (all pointers device)
struct JsonInputs {
    const ipcfp_event_proof* proofs;   // n_proofs slots as pass 2 wrote them (skipped slots included)
    uint64_t n_proofs;
    const uint8_t* blob;               // topics / data bytes the proofs index
    const uint8_t* cids;               // m*38, sorted witness CIDs
    const uint32_t* idx;               // m, block index of every witness entry
    uint64_t m;
    int64_t parent_epoch, child_epoch;
    uint32_t n_parents;
    const uint8_t* parent_cids;        // n_parents*38
    const uint8_t* child_cid;          // 38
};
// enqueues on the store's stream, synchronises it once (the exact length), enqueues the rendering and the copy into `out` (pinned,
// NUL-terminated; the text is there once the stream has drained); returns the length of the text
uint64_t render_event_json(Store* s, const JsonInputs& in, PinnedArray& out);
// the UnifiedProofBundle text of ipcfp_generate_proof_bundle_resident (all pointers device); the same steps as render_event_json
struct UnifiedJsonInputs {
    const ipcfp_storage_proof* storage;   // n_storage StorageProofs
    uint64_t n_storage;
    const ipcfp_event_proof* proofs;      // n_proofs EventProofs of every spec, in spec order (no skipped slot)
    uint64_t n_proofs;
    const uint8_t* blob;                  // topics / data bytes the proofs index
    const uint8_t* cids;                  // m*38, the union's sorted CIDs
    const uint32_t* idx;                  // m, block index of every union entry
    uint64_t m;
    int64_t parent_epoch, child_epoch;
    uint32_t n_parents;
    const uint8_t* parent_cids;           // n_parents*38
    const uint8_t* child_cid;             // 38
    const uint8_t* state_root;            // 38 (read only when n_storage > 0)
};
uint64_t render_unified_json(Store* s, const UnifiedJsonInputs& in, PinnedArray& out);
// ord[0..m) = the permutation that sorts the blocks idx[0..m) in `Cid` Ord (stable); runs on the store's stream (ingest: the ranks)
size_t sort_by_cid_ws_bytes(uint64_t m);
void sort_by_cid(Store* s, const uint32_t* idx_dev, uint32_t* ord, uint64_t m, void* workspace);

}  // namespace ipcfp
