// parallel.cu — the in-library cross-shard protocol over NCCL (SURVEY Appendix C: ipcfp_comm_init / ipcfp_generate_event_proof_sharded).
//
// One process per GPU. Receipts shard by index range (events/generator.rs:209-301 is independent per receipt); what spans
// shards is (1) the execution order — every message AMT concatenated, first occurrence of a CID wins (events/utils.rs:48-94) —
// and (2) the union of the per-shard witness CID sets (common/witness.rs:24-40). Everything is enqueued on CUDA streams with
// sizes the host already knows; the host waits for its peers twice (H0: does every shard have a message list, how long; H2:
// did every shard get through pass 2, how many matches / witness blocks), both while its own GPU is busy:
//
//   H0   all-gather  {ok, Nraw, nseg}                                      → global positions, exact buffer sizes, common abort
//   X    bucketize by hash(cid) % world → all-to-all (ncclSend/ncclRecv group) → first-seen dedup on the owners → the owners set
//        one bit per NON-first occurrence in a bitmap over the raw positions → all-reduce (sum of disjoint bitmaps = OR)
//        [exchange stream: runs underneath pass 1]
//   P    n_exec = zero bits; exec index i ↔ position of the (i+1)-th zero bit (prefix popcount + select) for the rank's matches;
//        pass 2 runs with the global n_exec (so "Missing message at index" keeps its place in the error order)
//   H2   all-gather  {first error key, matches, proofs, witness blocks}    → all ranks fail together with the SAME error
//   F    all-gather of the wanted positions → every owner copies the CIDs it holds → all-reduce → EventProof.message_cid patched
//   W    the sorted per-shard witness CID lists → bucketed k-way merge + unique: range-partitioned over the ranks (all-to-all of
//        the pieces), or on every rank (all-gather of the lists) with IPCFP_SHARDED_UNION_FULL   [union stream, own communicator]
// NCCL is resolved with dlopen at ipcfp_comm_init (libnccl.so.2: the copy already in the process — e.g. PyTorch's — or the
// system one), so the library itself keeps linking only cudart and loads on machines without NCCL.
#include <algorithm>
#include <cstdio>
#include <dlfcn.h>
#include <nccl.h>
#include <vector>

#include "engine.cuh"
#include "prims.cuh"
#include "rawcid.cuh"
#include "shard_kernels.cuh"

namespace ipcfp {

struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*);
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
    ncclResult_t (*CommDestroy)(ncclComm_t);
    const char* (*GetErrorString)(ncclResult_t);
    ncclResult_t (*GroupStart)();
    ncclResult_t (*GroupEnd)();
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
    ncclResult_t (*GetVersion)(int*);
};
static NcclApi* nccl_api() {
    static std::mutex mu;
    static NcclApi api;
    static bool ready = false;
    std::lock_guard<std::mutex> g(mu);
    if (ready) return &api;
    const char* names[] = {getenv("IPCFP_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    void* h = nullptr;
    for (const char* n : names) if (n && *n && (h = dlopen(n, RTLD_NOW | RTLD_LOCAL))) break;
    if (!h) throw Error(IPCFP_ERR_NCCL, std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : ""));
    auto sym = [&](const char* n) { void* p = dlsym(h, n); if (!p) throw Error(IPCFP_ERR_NCCL, std::string("NCCL symbol missing: ") + n); return p; };
    api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
    api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
    api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
    api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
    api.Send = (decltype(api.Send))sym("ncclSend");
    api.Recv = (decltype(api.Recv))sym("ncclRecv");
    api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
    api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
    api.Broadcast = (decltype(api.Broadcast))sym("ncclBroadcast");
    api.GetVersion = (decltype(api.GetVersion))sym("ncclGetVersion");
    ready = true;
    return &api;
}
#define IPCFP_NCCL(expr)                                                                                                     \
    do {                                                                                                                     \
        ncclResult_t _r = (expr);                                                                                            \
        if (_r != ncclSuccess) throw ::ipcfp::Error(IPCFP_ERR_NCCL, std::string(#expr) + ": " + nccl_api()->GetErrorString(_r)); \
    } while (0)

struct Comm {
    int device = 0;
    uint32_t world = 1, rank = 0;
    ncclComm_t cx = nullptr, cw = nullptr;   // exchange (execution order) / witness union: independent streams, independent communicators
    cudaStream_t sx = nullptr, sw = nullptr;   // exchange / fetch stream (communicator cx); witness-union stream (communicator cw)
    cudaEvent_t ev_a = nullptr, ev_b = nullptr, ev_c = nullptr;
    cudaEvent_t tm[10] = {};                 // timing: exchange begin/end (sx), fetch begin/end, union begin/end (engine stream); [6..8] inside the exchange: bucketize | all-to-all | dedup done
    // grow-only device scratch (allocated during warm-up, then reused)
    DevBuf<uint8_t> sendbuf, recvbuf, gather, merged, recs, part_send;
    DevBuf<unsigned long long> table, words, words2;
    DevBuf<uint32_t> bitmap, bitmap_sum, zeros, flags, starts;
    DevBuf<uint64_t> zprefix, scan_tmp, req, req_pad, req_all, ans, ans_sum, fscan;
    DevBuf<uint32_t> pos_of;
    DevBuf<unsigned long long> part_words;   // partitioned union: [0, W] piece bounds | [W+1, 2W+1) received piece lengths | [n_part, overflow] | the same of all ranks
    PinnedBuf<uint64_t> host;                // mapped: H0 / H2 read-backs
    ~Comm() {
        cudaSetDevice(device);
        NcclApi* n = nullptr;
        try { n = nccl_api(); } catch (...) {}
        if (n) { if (cx) n->CommDestroy(cx); if (cw) n->CommDestroy(cw); }
        if (ev_a) cudaEventDestroy(ev_a);
        if (ev_b) cudaEventDestroy(ev_b);
        if (ev_c) cudaEventDestroy(ev_c);
        for (auto& e : tm) if (e) cudaEventDestroy(e);
        if (sx) cudaStreamDestroy(sx);
        if (sw) cudaStreamDestroy(sw);
    }
};

void comm_unique_id(uint8_t* id128) {
    ncclUniqueId id;
    IPCFP_NCCL(nccl_api()->GetUniqueId(&id));
    static_assert(sizeof id == IPCFP_COMM_ID_BYTES, "ncclUniqueId size");
    memcpy(id128, &id, sizeof id);
}
Comm* comm_init(const uint8_t* id128, uint32_t world, uint32_t rank, int device) {
    check_device(device);
    if (!world || world > 256 || rank >= world) throw Error(IPCFP_ERR_INVALID_ARG, "bad world size / rank");
    NcclApi* n = nccl_api();
    std::unique_ptr<Comm> c(new Comm());
    c->device = device; c->world = world; c->rank = rank;
    {   // the exchange must not queue behind the full-grid scan kernels of the engine stream
        int lo_p = 0, hi_p = 0;
        IPCFP_CUDA(cudaDeviceGetStreamPriorityRange(&lo_p, &hi_p));
        IPCFP_CUDA(cudaStreamCreateWithPriority(&c->sx, cudaStreamNonBlocking, hi_p));
        IPCFP_CUDA(cudaStreamCreateWithPriority(&c->sw, cudaStreamNonBlocking, hi_p));
    }
    IPCFP_CUDA(cudaEventCreateWithFlags(&c->ev_a, cudaEventDisableTiming));
    IPCFP_CUDA(cudaEventCreateWithFlags(&c->ev_b, cudaEventDisableTiming));
    IPCFP_CUDA(cudaEventCreateWithFlags(&c->ev_c, cudaEventDisableTiming));
    for (auto& e : c->tm) IPCFP_CUDA(cudaEventCreate(&e));
    c->host.alloc(4096);    // mapped: [0, 2048) gathered words of H0 / H2
    c->words.alloc(4096);
    c->words2.alloc(4096);
    ncclUniqueId id;
    memcpy(&id, id128, sizeof id);
    IPCFP_NCCL(n->CommInitRank(&c->cx, (int)world, id, (int)rank));
    // the second communicator's id travels over the first one
    ncclUniqueId id2;
    if (rank == 0) IPCFP_NCCL(n->GetUniqueId(&id2));
    IPCFP_CUDA(cudaMemcpyAsync(c->words.p, &id2, sizeof id2, cudaMemcpyHostToDevice, c->sx));
    IPCFP_NCCL(n->Broadcast(c->words.p, c->words.p, sizeof id2, ncclUint8, 0, c->cx, c->sx));
    IPCFP_CUDA(cudaMemcpyAsync(&id2, c->words.p, sizeof id2, cudaMemcpyDeviceToHost, c->sx));
    IPCFP_CUDA(cudaStreamSynchronize(c->sx));
    IPCFP_NCCL(n->CommInitRank(&c->cw, (int)world, id2, (int)rank));
    return c.release();
}
void comm_destroy(Comm* c) { delete c; }
uint32_t comm_world(const Comm* c) { return c->world; }
uint32_t comm_rank(const Comm* c) { return c->rank; }

// ------------------------------------------------------------------------------------------ host side of the protocol
// (the kernels it enqueues are in shard_kernels.cuh)

struct Words8 { uint64_t w[8]; };
__global__ void k_put_words(Words8 v, uint32_t k, unsigned long long* dst) { if (threadIdx.x < k) dst[threadIdx.x] = v.w[threadIdx.x]; }
__global__ void k_fill_words(unsigned long long* dst, uint32_t n, unsigned long long v) { for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = v; }
__global__ void k_publish_words(const unsigned long long* __restrict__ src, unsigned long long* dst_mapped, uint32_t n) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst_mapped[i] = src[i];
    __threadfence_system();
}
// word `field` of every rank's 8-word H2 record → dst[r]
__global__ void k_pick_field(const unsigned long long* __restrict__ gathered, uint32_t world, uint32_t stride, uint32_t field, uint64_t* dst) {
    for (uint32_t r = threadIdx.x; r < world; r += blockDim.x) dst[r] = gathered[(uint64_t)r * stride + field];
}
// Tiny all-gather of k ≤ 8 words per rank whose result the HOST needs. No copy-engine work (the D2H engine is busy with the
// witness blob): the words go up as a kernel parameter and come back through mapped host memory.
static void run_all_gather_host(Comm* c, const uint64_t* mine, uint32_t k, uint64_t* all /* = c->host.p */) {
    NcclApi* n = nccl_api();
    Words8 v{};
    for (uint32_t i = 0; i < k && i < 8; i++) v.w[i] = mine[i];
    k_put_words<<<1, 32, 0, c->sx>>>(v, k, c->words.p); IPCFP_LAUNCH_CHECK();
    IPCFP_NCCL(n->AllGather(c->words.p, c->words2.p, k, ncclUint64, c->cx, c->sx));
    k_publish_words<<<1, 256, 0, c->sx>>>(c->words2.p, (unsigned long long*)c->host.dev, c->world * k); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaStreamSynchronize(c->sx));
    (void)all;
}

ShardExchange::ShardExchange(Comm* comm, Store* store, uint64_t lo_, uint64_t hi_) : c(comm), s(store), lo(lo_), hi(hi_) {
    if (c->device != s->device) throw Error(IPCFP_ERR_INVALID_ARG, "communicator and store are bound to different devices");
    if (c->world > MAX_WORLD) throw Error(IPCFP_ERR_UNSUPPORTED, "world too large");
}

// EARLY H0: can every shard promise the length of its slice already (dense message AMTs: known from the roots), and do all shards see the
// same message list. all_early ⇒ the slices (nseg_all, pos0, nraw) are set as for agree_slices.
void ShardExchange::agree_early(bool can_promise, uint64_t planned_nseg, uint64_t nraw_total) {
    const uint32_t W = c->world;
    uint64_t mine[4] = {can_promise ? 1ull : 0ull, planned_nseg, nraw_total, 0};
    uint64_t* all = c->host.p;
    run_all_gather_host(c, mine, 4, all);
    bool ok = true;
    nseg_all.assign(W, 0);
    nraw = 0; max_nseg = 0;
    for (uint32_t r = 0; r < W; r++) {
        if (!all[4 * r] || all[4 * r + 2] != all[2]) ok = false;
        nseg_all[r] = all[4 * r + 1];
        if (r == c->rank) pos0 = nraw;
        nraw += nseg_all[r];
        max_nseg = std::max(max_nseg, nseg_all[r]);
    }
    if (ok && nraw != all[2]) ok = false;                 // the promised slices must tile the whole list
    if (nraw >= 0xffffffffull) ok = false;
    all_early = ok;
    peers_ok = true;
    nseg = planned_nseg;
}
// H0: does every shard have its slice of the message list, and how long is it. Every rank takes part, also a failing one.
void ShardExchange::agree_slices(uint64_t tx_key, uint64_t err_key, uint64_t nseg_) {
    const uint32_t W = c->world;
    const bool ok = tx_key == IPCFP_NO_ERROR && err_key == IPCFP_NO_ERROR;
    uint64_t mine[4] = {ok ? 1ull : 0ull, ok ? nseg_ : 0, tx_key, err_key};
    uint64_t* all = c->host.p;
    run_all_gather_host(c, mine, 4, all);
    nseg_all.assign(W, 0);
    bool all_ok = true;
    nraw = 0; max_nseg = 0;
    g_tx = g_err = IPCFP_NO_ERROR;
    for (uint32_t r = 0; r < W; r++) {
        if (!all[4 * r]) all_ok = false;
        g_tx = std::min(g_tx, all[4 * r + 2]); g_err = std::min(g_err, all[4 * r + 3]);
        nseg_all[r] = all[4 * r + 1];
        if (r == c->rank) pos0 = nraw;
        nraw += nseg_all[r];
        max_nseg = std::max(max_nseg, nseg_all[r]);
    }
    peers_ok = all_ok;
    nseg = nseg_;
    if (nraw >= 0xffffffffull) throw Error(IPCFP_ERR_UNSUPPORTED, "more than 2^32 messages");
}

// X: bucketize → all-to-all → dedup → duplicate bitmap → all-reduce, all on the exchange stream (runs underneath pass 1)
void ShardExchange::start_exchange(const void* seg_dev) {
    NcclApi* n = nccl_api();
    const uint32_t W = c->world;
    cudaStream_t sx = c->sx;
    seg = (const RawCid*)seg_dev;
    IPCFP_CUDA(cudaStreamWaitEvent(sx, s->ev[EV_RAW_LIST], 0));
    IPCFP_CUDA(cudaEventRecord(c->tm[0], sx));
    cap = exec_seg_cap(max_nseg, W);
    const uint64_t segbytes = XSEG_HDR + cap * 48;
    c->sendbuf.ensure(segbytes * W);
    c->recvbuf.ensure(segbytes * W);
    nwords = (nraw + 31) / 32;
    c->bitmap.ensure(nwords + 64);
    c->bitmap_sum.ensure(nwords + 64);
    c->zeros.ensure(nwords + 64);
    c->zprefix.ensure(nwords + 64);
    c->scan_tmp.ensure(scan_scratch_elems(nwords + 64) + 64);
    const uint64_t slots = exec_table_slots(W, cap);
    c->table.ensure(slots);
    unsigned long long* overflow = c->words.p + 3100;
    IPCFP_CUDA(cudaMemsetAsync(c->bitmap.p, 0, (nwords + 64) * 4, sx));
    IPCFP_CUDA(cudaMemsetAsync(c->table.p, 0, slots * 8, sx));
    IPCFP_CUDA(cudaMemsetAsync(overflow, 0, 8, sx));
    // headers of empty segments must read 0 even when this rank has nothing to send
    for (uint32_t r = 0; r < W; r++) IPCFP_CUDA(cudaMemsetAsync(c->sendbuf.p + r * segbytes, 0, XSEG_HDR, sx));
    if (nseg) {
        const uint32_t nruns = div_up(nseg, XB_RUN);
        AsyncBuf<uint32_t> cnt((uint64_t)W * nruns + 64, sx);
        AsyncBuf<uint64_t> scan((uint64_t)W * nruns + 64, sx), scratch(scan_scratch_elems((uint64_t)W * nruns) + 8, sx), total(1, sx);
        if (W > 32) cnt.zero();
        k_xb_count<<<div_up((uint64_t)nruns * 32, 128), 128, 0, sx>>>(seg, nseg, W, nruns, cnt.p); IPCFP_LAUNCH_CHECK();
        exclusive_scan_u32(cnt.p, scan.p, (uint64_t)W * nruns, total.p, scratch.p, sx);
        k_xb_headers<<<div_up(W, 64), 64, 0, sx>>>(scan.p, total.p, W, nruns, cap, c->sendbuf.p, overflow); IPCFP_LAUNCH_CHECK();
        k_xb_scatter<<<div_up((uint64_t)nruns * 32, 128), 128, 0, sx>>>(seg, nseg, pos0, W, nruns, scan.p, cap, c->sendbuf.p); IPCFP_LAUNCH_CHECK();
    }
    IPCFP_CUDA(cudaEventRecord(c->tm[6], sx));
    // all-to-all of whole segments (fixed size: no count round trip; the valid count travels in the segment header)
    IPCFP_NCCL(n->GroupStart());
    for (uint32_t p = 0; p < W; p++) {
        IPCFP_NCCL(n->Send(c->sendbuf.p + p * segbytes, segbytes, ncclUint8, (int)p, c->cx, sx));
        IPCFP_NCCL(n->Recv(c->recvbuf.p + p * segbytes, segbytes, ncclUint8, (int)p, c->cx, sx));
    }
    IPCFP_NCCL(n->GroupEnd());
    IPCFP_CUDA(cudaEventRecord(c->tm[7], sx));
    uint64_t* seg_off = (uint64_t*)(c->words.p + 2600);   // [0, W]
    k_recv_offsets<<<1, 1, 0, sx>>>(c->recvbuf.p, W, cap, seg_off); IPCFP_LAUNCH_CHECK();
    const unsigned g = div_up(W * cap, 256);
    k_exec_claim_seg<<<g, 256, 0, sx>>>(c->recvbuf.p, seg_off, W, cap, c->table.p, slots - 1); IPCFP_LAUNCH_CHECK();
    k_exec_mark_dups<<<g, 256, 0, sx>>>(c->recvbuf.p, seg_off, W, cap, c->table.p, slots - 1, c->bitmap.p); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaEventRecord(c->tm[8], sx));
    // the owners' bitmaps are disjoint (a position belongs to one CID, a CID to one owner): their sum is their union
    IPCFP_NCCL(n->AllReduce(c->bitmap.p, c->bitmap_sum.p, nwords + 1, ncclUint32, ncclSum, c->cx, sx));
    // n_exec = number of zero bits; prefix zero counts for the select
    if (nwords) { k_zero_counts<<<div_up(nwords, 256), 256, 0, sx>>>(c->bitmap_sum.p, nraw, c->zeros.p); IPCFP_LAUNCH_CHECK(); }
    n_exec_dev = c->words.p + 3101;
    exclusive_scan_u32(c->zeros.p, c->zprefix.p, nwords, (uint64_t*)n_exec_dev, c->scan_tmp.p, sx);
    IPCFP_CUDA(cudaEventRecord(c->ev_a, sx));
    IPCFP_CUDA(cudaEventRecord(c->tm[1], sx));
    overflow_dev = overflow;
}

// P: the global n_exec, raw positions of this rank's matches, and exec.get(i) of events/generator.rs:244-246 for every match — it
// PRECEDES r_amt.get(i) in the reference, so at the same receipt it outranks whatever pass 2 reported (code 0 sorts first in the error
// word). All of it on the exchange stream behind X: the engine stream goes on with the witness and never waits for a peer.
void ShardExchange::positions_for(const uint32_t* match_rel, uint64_t n_match, unsigned long long* n_exec_out_) {
    cudaStream_t st = c->sx;
    n_exec_out = n_exec_out_;
    IPCFP_CUDA(cudaStreamWaitEvent(st, c->ev_a, 0));
    IPCFP_CUDA(cudaMemcpyAsync(n_exec_out, n_exec_dev, 8, cudaMemcpyDeviceToDevice, st));
    publish_words(s, HW_EXCH_OVERFLOW, HW_EXCHANGE_WORDS, overflow_dev, st);   // overflow flag, n_exec: read after the next sync of that stream
    M = n_match;
    c->req.ensure(n_match + 64);
    if (n_match) {
        k_select_positions<<<div_up(n_match, 128), 128, 0, st>>>(match_rel, n_match, lo, c->bitmap_sum.p, c->zprefix.p, nwords, n_exec_dev, c->req.p);
        IPCFP_LAUNCH_CHECK();
    }
    match_rel_dev = match_rel;
    unsigned long long* chk = s->dev_words.p + DW_EXEC_CHECK;   // the check has its own word: it may have to be repeated (stale exchange)
    IPCFP_CUDA(cudaMemsetAsync(chk, 0xff, 8, st));
    if (n_match) { k_check_exec<<<div_up(n_match, 128), 128, 0, st>>>(match_rel, n_match, lo, n_exec_out, chk); IPCFP_LAUNCH_CHECK(); }
    publish_words(s, DW_EXEC_CHECK, 1, nullptr, st);
}

// H2 (the host waits for its peers here while its own GPU sorts the witness). All ranks continue or fail together, naming the same first
// error. When some shard's early promise was wrong, its slice differs from what the running exchange used: every shard repeats the
// exchange with the slices as they really are (late H0), then the positions, the exec.get check and H2.
bool ShardExchange::agree_results(uint64_t tx_key, uint64_t err_key, bool missing_base, uint64_t n_proofs, uint64_t n_witness, bool stale, const void* seg_dev,
                                  uint64_t nseg_) {
    const uint64_t* hw = s->host_words.p;
    IPCFP_CUDA(cudaStreamSynchronize(c->sx));
    uint64_t pend_chk = hw[DW_EXEC_CHECK];
    gather_results(tx_key, std::min(err_key, pend_chk), missing_base, n_proofs, n_witness, hw[HW_EXCH_OVERFLOW], stale);
    if (g_stale && g_tx == IPCFP_NO_ERROR) {
        agree_slices(tx_key, err_key, nseg_);
        if (peers_ok) {
            start_exchange(seg_dev);
            positions_for(match_rel_dev, M, n_exec_out);
            IPCFP_CUDA(cudaStreamSynchronize(c->sx));
            pend_chk = hw[DW_EXEC_CHECK];
        }
        gather_results(tx_key, std::min(err_key, pend_chk), missing_base, n_proofs, n_witness, hw[HW_EXCH_OVERFLOW], false);
    }
    return g_tx == IPCFP_NO_ERROR && g_err == IPCFP_NO_ERROR && !g_missing_base && !g_overflow;
}

// every rank reports how far it got; the global values are the same on every rank
void ShardExchange::gather_results(uint64_t tx_key, uint64_t err_key, bool missing_base, uint64_t n_proofs, uint64_t n_witness, uint64_t exch_overflow, bool stale) {
    const uint32_t W = c->world;
    uint64_t mine[8] = {tx_key, err_key, missing_base ? 1ull : 0ull, M, n_proofs, n_witness, exch_overflow, stale ? 1ull : 0ull};
    uint64_t* all = c->host.p;
    run_all_gather_host(c, mine, 8, all);
    k_pick_field<<<1, 256, 0, c->sx>>>(c->words2.p, W, 8, 5, (uint64_t*)(c->words2.p + 2600)); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaStreamSynchronize(c->sx));
    g_tx = g_err = IPCFP_NO_ERROR; g_missing_base = false; g_overflow = false; g_stale = false;
    M_max = 0; nw_max = 0; M_total = 0; proofs_total = 0;
    nw_all.assign(W, 0);
    for (uint32_t r = 0; r < W; r++) {
        const uint64_t* a = all + 8 * r;
        g_tx = std::min(g_tx, a[0]); g_err = std::min(g_err, a[1]);
        g_missing_base |= a[2] != 0;
        M_max = std::max(M_max, a[3]); M_total += a[3]; proofs_total += a[4];
        nw_all[r] = a[5]; nw_max = std::max(nw_max, a[5]);
        g_overflow |= a[6] != 0;
        g_stale |= a[7] != 0;
    }
}

// F: positions wanted by every rank → the owners answer → EventProof.message_cid of this rank's proofs (pass 2 is complete: the host
// synchronised on it) → proofs_host
void ShardExchange::fetch_and_patch(ipcfp_event_proof* proofs_dev, uint64_t n_proofs, void* proofs_host) {
    cudaStream_t st = c->sx;
    patch(proofs_dev, n_proofs);
    if (n_proofs) IPCFP_CUDA(cudaMemcpyAsync(proofs_host, proofs_dev, n_proofs * sizeof(ipcfp_event_proof), cudaMemcpyDeviceToHost, st));
}
void ShardExchange::patch(ipcfp_event_proof* proofs_dev, uint64_t n_proofs) {
    cudaStream_t st = c->sx;
    IPCFP_CUDA(cudaEventRecord(c->tm[2], st));
    IPCFP_CUDA(cudaEventRecord(c->tm[3], st));
    if (M_max == 0) return;
    NcclApi* n = nccl_api();
    const uint32_t W = c->world;
    c->req_all.ensure((uint64_t)W * M_max + 64);
    c->ans.ensure(((uint64_t)W * M_max + 8) * 5);
    c->ans_sum.ensure(((uint64_t)W * M_max + 8) * 5);
    // this rank's request list, padded to M_max with "nobody's position" (req itself holds M entries: M_max was not known when it was sized)
    c->req_pad.ensure(M_max + 64);
    IPCFP_CUDA(cudaMemsetAsync(c->req_pad.p, 0xff, M_max * 8, st));
    if (M) IPCFP_CUDA(cudaMemcpyAsync(c->req_pad.p, c->req.p, M * 8, cudaMemcpyDeviceToDevice, st));
    IPCFP_NCCL(n->AllGather(c->req_pad.p, c->req_all.p, M_max, ncclUint64, c->cx, st));
    const uint64_t total = (uint64_t)W * M_max;
    k_fetch_positions<<<div_up(total, 256), 256, 0, st>>>(seg, nseg, pos0, c->req_all.p, total, (RawCid*)c->ans.p); IPCFP_LAUNCH_CHECK();
    IPCFP_NCCL(n->AllReduce(c->ans.p, c->ans_sum.p, total * 5, ncclUint64, ncclSum, c->cx, st));
    if (n_proofs) {
        k_patch_message_cids<<<div_up(n_proofs, 128), 128, 0, st>>>(proofs_dev, n_proofs, match_rel_dev, M, lo, (const RawCid*)c->ans_sum.p + (uint64_t)c->rank * M_max);
        IPCFP_LAUNCH_CHECK();
    }
    IPCFP_CUDA(cudaEventRecord(c->tm[3], st));
}

// W: the union of the shards' witness CID sets as soon as this shard's sorted list exists (event after k_witness_emit), on its own
// stream and communicator: it runs beside the message-CID fetch
void ShardExchange::witness_union(const uint8_t* cids_dev, uint64_t n_local, bool full) {
    cudaStream_t sw = c->sw;
    full_union = full; wit_cids = cids_dev; wit_n = n_local;
    IPCFP_CUDA(cudaStreamWaitEvent(sw, s->ev[EV_WITNESS_SORTED], 0));
    if (full) {
        union_replicated((uint64_t*)(s->dev_words.p + DW_UNION_SIZE));
        publish_words(s, DW_UNION_SIZE, 1, nullptr, sw);
    } else union_partitioned(union_piece_cap(false));
}
void ShardExchange::finish() {
    IPCFP_CUDA(cudaStreamSynchronize(c->sx));
    IPCFP_CUDA(cudaStreamSynchronize(c->sw));
    if (full_union) return;
    bool overflow = false;
    for (uint32_t q = 0; q < c->world; q++) overflow |= s->host_words.p[HW_UNION_PARTS + 2 * q + 1] != 0;
    if (overflow) {   // a piece did not fit its slot on some rank (every rank sees the same words): once more with slots that cannot overflow
        union_partitioned(union_piece_cap(true));
        IPCFP_CUDA(cudaStreamSynchronize(c->sw));
    }
}
void ShardExchange::fill_result(ipcfp_event_result& r) const {
    const uint64_t* hw = s->host_words.p;
    r.n_exec = hw[HW_EXCH_N_EXEC];
    r.union_cids_dev = union_dev;
    if (full_union) { r.n_union_cids = r.n_union_part = hw[DW_UNION_SIZE]; r.union_part_first = 0; }
    else {
        r.n_union_cids = 0;
        for (uint32_t q = 0; q < c->world; q++) { if (q == c->rank) r.union_part_first = r.n_union_cids; r.n_union_cids += hw[HW_UNION_PARTS + 2 * q]; }
        r.n_union_part = hw[HW_UNION_PARTS + 2 * c->rank];
    }
    r.total_matching = M_total; r.total_proofs = proofs_total;
    timings(&r.ms_exchange, &r.ms_fetch, &r.ms_union);
}
// union of the per-shard sorted witness CID lists (BTreeSet union of common/witness.rs:24-40) on every rank
void ShardExchange::union_replicated(uint64_t* n_out_dev_word) {
    const uint8_t* cids_dev = wit_cids;
    const uint64_t n_local = wit_n;
    cudaStream_t st = c->sw;
    NcclApi* n = nccl_api();
    const uint32_t W = c->world;
    IPCFP_CUDA(cudaEventRecord(c->tm[4], st));
    const uint64_t capw = nw_max + 1;
    const uint64_t total_cap = (uint64_t)W * capw;
    c->recs.ensure(capw * 40 + 64);
    c->gather.ensure(total_cap * 40 + 64);
    c->starts.ensure((uint64_t)W * (MERGE_BUCKETS + 1) + 64);
    c->pos_of.ensure(total_cap + 64);
    c->flags.ensure(total_cap + 64);
    c->fscan.ensure(total_cap + 64);
    c->merged.ensure(total_cap * 38 + 64);
    c->scan_tmp.ensure(scan_scratch_elems(total_cap + 64) + 64);
    k_cids_to_recs<<<div_up(capw, 256), 256, 0, st>>>(cids_dev, n_local, capw, (RawCid*)c->recs.p); IPCFP_LAUNCH_CHECK();
    IPCFP_NCCL(n->AllGather(c->recs.p, c->gather.p, capw * 40, ncclUint8, c->cw, st));
    uint64_t* counts = (uint64_t*)(c->words2.p + 2600);   // per-rank list lengths, picked out of the H2 records by agree_results
    IPCFP_CUDA(cudaMemsetAsync(c->flags.p, 0, (total_cap + 64) * 4, st));
    const unsigned g = div_up(total_cap, 256);
    k_merge_starts<<<g, 256, 0, st>>>((const RawCid*)c->gather.p, counts, W, capw, c->starts.p, 0, MERGE_BUCKETS); IPCFP_LAUNCH_CHECK();
    k_merge_rank<<<g, 256, 0, st>>>((const RawCid*)c->gather.p, counts, W, capw, c->starts.p, c->pos_of.p, c->flags.p, 0, MERGE_BUCKETS); IPCFP_LAUNCH_CHECK();
    uint64_t total_listed = 0;
    for (uint32_t r = 0; r < W; r++) total_listed += nw_all[r];
    unsigned long long* n_union = c->words2.p + 3000;
    exclusive_scan_u32(c->flags.p, c->fscan.p, total_listed, (uint64_t*)n_union, c->scan_tmp.p, st);
    k_merge_emit38<<<g, 256, 0, st>>>((const RawCid*)c->gather.p, counts, W, capw, c->pos_of.p, c->flags.p, c->fscan.p, c->merged.p); IPCFP_LAUNCH_CHECK();
    union_dev = c->merged.p;
    IPCFP_CUDA(cudaMemcpyAsync(n_out_dev_word, n_union, 8, cudaMemcpyDeviceToDevice, st));
    IPCFP_CUDA(cudaEventRecord(c->tm[5], st));
}
// W, partitioned: the union is left DISTRIBUTED — rank r ends up with the sorted, duplicate-free CIDs whose first two digest bytes
// fall into its 1/world share of the 65 536 buckets, so the concatenation of the partitions in rank order is the BTreeSet order. Every
// rank sends each peer the piece of its sorted list that belongs to it and merges the `world` sorted pieces it receives: bytes on the
// wire and merge work per rank are those of about TWO shard lists, whatever the world size (the all-gather variant above moves and
// merges `world` lists on every rank). Pieces travel in fixed-size slots of `cap` records behind a count header, so that no size has
// to come back to the host in the middle of the protocol; a piece that does not fit raises this rank's overflow word, every rank
// sees every word after the call's last synchronisation, and the caller repeats the union with cap = the longest list (cannot
// overflow). No host synchronisation inside.
uint64_t ShardExchange::union_piece_cap(bool cannot_overflow) const {
    const uint32_t W = c->world;
    if (cannot_overflow) return nw_max + 1;
    if (const char* e = getenv("IPCFP_UNION_CAP")) return (uint64_t)std::max(1, atoi(e));   // tests: force the overflow path
    return union_piece_cap_default(nw_max, W);
}
void ShardExchange::union_partitioned(uint64_t cap) {
    const uint8_t* cids_dev = wit_cids;
    const uint64_t n_local = wit_n;
    cudaStream_t st = c->sw;
    NcclApi* n = nccl_api();
    const uint32_t W = c->world, me = c->rank;
    IPCFP_CUDA(cudaEventRecord(c->tm[4], st));
    const uint64_t stride = cap + 1, total_cap = (uint64_t)W * stride;
    const uint32_t b0 = part_lo(me, W), nb = part_lo(me + 1, W) - b0;
    c->recs.ensure((n_local + 1) * 40 + 64);
    c->part_send.ensure(total_cap * 40 + 64);
    c->gather.ensure(total_cap * 40 + 64);
    c->part_words.ensure(4ull * W + 16);
    c->starts.ensure((uint64_t)W * (nb + 1) + 64);
    c->pos_of.ensure(total_cap + 64);
    c->flags.ensure(total_cap + 64);
    c->fscan.ensure(total_cap + 64);
    c->merged.ensure(total_cap * 38 + 64);
    c->scan_tmp.ensure(scan_scratch_elems(total_cap + 64) + 64);
    unsigned long long* pw = c->part_words.p;
    unsigned long long *bounds_d = pw, *col_d = pw + W + 1, *mine_d = pw + 2 * W + 2 /* [n_part, overflow] */, *all_d = pw + 2 * W + 4 /* 2 words per rank */;
    RawCid* send = (RawCid*)c->part_send.p;
    RawCid* recv = (RawCid*)c->gather.p;
    k_cids_to_recs<<<div_up(n_local + 1, 256), 256, 0, st>>>(cids_dev, n_local, n_local + 1, (RawCid*)c->recs.p); IPCFP_LAUNCH_CHECK();
    k_part_bounds<<<1, 256, 0, st>>>((const RawCid*)c->recs.p, n_local, W, cap, (uint64_t*)bounds_d, send, mine_d + 1); IPCFP_LAUNCH_CHECK();
    if (n_local) { k_part_pack<<<div_up(n_local, 256), 256, 0, st>>>((const RawCid*)c->recs.p, n_local, W, cap, (const uint64_t*)bounds_d, send); IPCFP_LAUNCH_CHECK(); }
    IPCFP_NCCL(n->GroupStart());
    for (uint32_t r = 0; r < W; r++) {
        IPCFP_NCCL(n->Send(send + (uint64_t)r * stride, stride * 40, ncclUint8, (int)r, c->cw, st));
        IPCFP_NCCL(n->Recv(recv + (uint64_t)r * stride, stride * 40, ncclUint8, (int)r, c->cw, st));
    }
    IPCFP_NCCL(n->GroupEnd());
    IPCFP_CUDA(cudaMemsetAsync(c->flags.p, 0, (total_cap + 64) * 4, st));
    k_part_counts<<<1, 256, 0, st>>>(recv, W, cap, (uint64_t*)col_d); IPCFP_LAUNCH_CHECK();
    const unsigned g = div_up(total_cap, 256);
    const RawCid* lists = recv + 1;   // piece r's entries start one record behind its header: same stride
    k_merge_starts<<<g, 256, 0, st>>>(lists, (const uint64_t*)col_d, W, stride, c->starts.p, b0, nb); IPCFP_LAUNCH_CHECK();
    k_merge_rank<<<g, 256, 0, st>>>(lists, (const uint64_t*)col_d, W, stride, c->starts.p, c->pos_of.p, c->flags.p, b0, nb); IPCFP_LAUNCH_CHECK();
    exclusive_scan_u32(c->flags.p, c->fscan.p, total_cap, (uint64_t*)mine_d, c->scan_tmp.p, st);
    k_merge_emit38<<<g, 256, 0, st>>>(lists, (const uint64_t*)col_d, W, stride, c->pos_of.p, c->flags.p, c->fscan.p, c->merged.p); IPCFP_LAUNCH_CHECK();
    // [partition size, overflow] of all ranks → the store's mapped words HW_UNION_PARTS: read after the next sync of this stream
    IPCFP_NCCL(n->AllGather(mine_d, all_d, 2, ncclUint64, c->cw, st));
    publish_words(s, HW_UNION_PARTS, 2 * W, all_d, st);
    union_dev = c->merged.p;
    IPCFP_CUDA(cudaEventRecord(c->tm[5], st));
}
void ShardExchange::timings(float* ms_exchange, float* ms_fetch, float* ms_union) const {
    cudaEventElapsedTime(ms_exchange, c->tm[0], c->tm[1]);
    if (getenv("IPCFP_XCH_TRACE")) {
        float a = 0, b = 0, d = 0, e = 0;
        cudaEventElapsedTime(&a, c->tm[0], c->tm[6]); cudaEventElapsedTime(&b, c->tm[6], c->tm[7]); cudaEventElapsedTime(&d, c->tm[7], c->tm[8]); cudaEventElapsedTime(&e, c->tm[8], c->tm[1]);
        fprintf(stderr, "[ipcfp rank %u] exchange: bucketize %.3f ms | all-to-all %.3f ms | dedup %.3f ms | all-reduce + scan %.3f ms (cap %llu entries/segment)\n", c->rank, a, b, d, e,
                (unsigned long long)cap);
    }
    cudaEventElapsedTime(ms_fetch, c->tm[2], c->tm[3]);
    cudaEventElapsedTime(ms_union, c->tm[4], c->tm[5]);
}
// IPCFP_XCH_TRACE: where the protocol's stages sit on the call's own time axis (ms after `origin`, an event of the engine stream)
void ShardExchange::trace_timeline(cudaEvent_t origin, const char* engine_part) const {
    float t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 6; i++) cudaEventElapsedTime(&t[i], origin, c->tm[i]);
    fprintf(stderr, "[ipcfp rank %u] timeline ms: %s | exchange %.3f-%.3f fetch %.3f-%.3f union %.3f-%.3f\n", c->rank, engine_part, t[0], t[1], t[2], t[3], t[4], t[5]);
}

}  // namespace ipcfp
