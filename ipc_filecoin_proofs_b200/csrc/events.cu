// events.cu — the two-pass receipt/event AMT scan on the GPU.
//
// Replaces, for the data-parallel path, reference src/proofs/events/generator.rs:60-307:
//   k_setup            collect_base_witness (:122-145) + TxMeta decode + AMT root loads
//   k_amt_level/...    record_transaction_amts (:148-177) and build_execution_order
//                      (events/utils.rs:33-94) as ONE level-synchronous, order-preserving BFS
//   k_dedup_*          first-seen dedup of the execution order (utils.rs:56-91)
//   k_pass1_stage      find_matching_events pass 1 (:206-239, pass1_stage.cuh): one lane decodes one
//                      events-AMT root node, its bytes staged through shared memory by the whole warp,
//                      tests (actor_id, topic_0, topic_1) on every StampedEvent, the warp ballots the
//                      matching-receipt bitmap
//   k_pass2<EMIT>      pass 2 (:241-301): per matching receipt, receipts-AMT path walk + full
//                      events-AMT walk, witness bits, EventProof records
//   materialize_witness (witness.cu)   WitnessCollector::materialize (:104)
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include <chrono>
#include <cstddef>
#include <optional>
#include <type_traits>
#include <cooperative_groups.h>
#include "engine.cuh"
#include "hashes.cuh"
#include "ipld.cuh"
#include "prims.cuh"
#include "walk.cuh"
#include "events_items.cuh"
#include "msg_select_items.cuh"
#include "pass1_stage.cuh"
#include "rawcid.cuh"

namespace ipcfp {
namespace cg = cooperative_groups;

// ------------------------------------------------------------------------------------------ pass 1 / pass 2 kernels (per-receipt code: events_items.cuh)
// Pass 1 is k_pass1_stage (pass1_stage.cuh).

// a.per_warp: one matching receipt per WARP (lane 0 walks). A matching receipt is a chain of dependent accesses (hash probe → record →
// strict decode of a 349–413 B node, 7 levels at 1 M receipts, then its events AMT), and 32 lanes on 32 different paths execute that
// chain serialised by divergence: ≈ 1 000 matches in 8 CTAs keep 8 of the GPU's 132 SMs busy. One warp per match is the shape
// k_read_slots uses for the same reason (storage.cu); above 16 384 matches the grid fills the machine either way and one match per
// thread is kept. Same per-item code, so results are identical by construction.
template <class P>
__global__ void __launch_bounds__(128) k_pass2(Pass2ArgsT<P> a) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a.per_warp) { if (threadIdx.x & 31) return; t >>= 5; }
    if (t >= a.n_match) return;
    pass2_item(a, t);
}

// ------------------------------------------------------------------------------------------ message selection (per-item code: msg_select_items.cuh)
// The requests sorted once (msg_sort_key): keys of one slice in the current order, and the final gather
__global__ void k_msg_iota(uint32_t* perm, uint32_t n) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) perm[t] = t;
}
__global__ void k_msg_keys(const RawCid* __restrict__ req, const uint32_t* __restrict__ perm, uint32_t n, uint32_t q, uint32_t* keys) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) keys[t] = msg_sort_key(req[perm[t]], q);
}
__global__ void k_msg_gather(const RawCid* __restrict__ req, const uint32_t* __restrict__ perm, uint32_t n, RawCid* sorted, uint32_t* sorted_pos) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) { sorted[t] = req[perm[t]]; sorted_pos[t] = perm[t]; }
}
// sorted[0..n) = the requests in (CID words, input position) order, sorted_pos their input positions; enqueued on st
static void sort_requests(const RawCid* req, uint32_t n, RawCid* sorted, uint32_t* sorted_pos, cudaStream_t st) {
    if (!n) return;
    const unsigned nb = radix_blocks(n);
    AsyncBuf<uint32_t> keys(n, st), perm(n, st), ka(n, st), pa(n, st), hist((size_t)256 * nb + 256, st);
    AsyncBuf<uint64_t> scan_tmp((size_t)256 * nb + 256, st), scratch(scan_scratch_elems(std::max<uint64_t>((uint64_t)256 * nb, n)) + 8, st);
    k_msg_iota<<<div_up(n, 256), 256, 0, st>>>(perm.p, n); IPCFP_LAUNCH_CHECK();
    for (uint32_t q = MSG_SORT_SLICES; q-- > 0;) {
        k_msg_keys<<<div_up(n, 256), 256, 0, st>>>(req, perm.p, n, q, keys.p); IPCFP_LAUNCH_CHECK();
        radix_sort_pairs(keys.p, perm.p, ka.p, pa.p, n, 32, hist.p, scan_tmp.p, scratch.p, st);
    }
    k_msg_gather<<<div_up(n, 256), 256, 0, st>>>(req, perm.p, n, sorted, sorted_pos); IPCFP_LAUNCH_CHECK();
}
// one thread per execution position: the requests that name it, and the selected-receipt bitmap
__global__ void __launch_bounds__(256) k_msg_select(const RawCid* __restrict__ exec_raw, const uint32_t* __restrict__ exec_idx, const unsigned long long* n_exec,
                                                    const RawCid* __restrict__ sorted, const uint32_t* __restrict__ sorted_pos, uint32_t n, uint64_t n_receipts,
                                                    uint64_t* exec_indices, uint32_t* sel_bits) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *n_exec) return;
    if (msg_select_item(exec_raw, exec_idx, i, sorted, sorted_pos, n, n_receipts, exec_indices)) atomicOr(sel_bits + (i >> 5), 1u << (i & 31));
}
// one selected receipt per warp (lane 0 walks), as k_pass2 takes its matches; above 16 384 one per thread
template <class P>
__global__ void __launch_bounds__(128) k_msg_match(MsgMatchArgsT<P> a) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a.per_warp) { if (threadIdx.x & 31) return; t >>= 5; }
    if (t >= a.n_sel_max || t >= *a.n_sel) return;
    msg_match_item(a, t);
}

// ------------------------------------------------------------------------------------------ setup + message AMT walk
#define IPCFP_MAX_PARENTS 64
static_assert(2 * IPCFP_MAX_PARENTS <= DENSE_MAX_AMTS, "the dense plan's tables hold every message AMT");
// What k_setup leaves for the host and the walk, in one device block. The head (everything before the tables) reaches the host
// in one publish (host words HW_PROLOGUE ..); the tables stay on the device.
struct Prologue {
    uint32_t misc[64 + 2 * IPCFP_MAX_PARENTS];   // [0] receipts-root block, [1] a base-witness CID is missing, [2] any_skip (pass 2), [64 + k] height of AMT k
    uint64_t amt_count[2 * IPCFP_MAX_PARENTS];   // root.count of AMT k
    uint64_t t0[4];                              // keccak256(event signature), the Matcher's t0
    DenseTables plan;                            // the dense walk's plan: ok, rounds, nraw, then the tables
};
static constexpr uint32_t PRO_HEAD_WORDS = (uint32_t)((offsetof(Prologue, plan) + offsetof(DenseTables, per_amt)) / 8);
static_assert(PRO_HEAD_WORDS <= HW_PROLOGUE_WORDS, "the prologue's head fits its host words (HW_PROLOGUE)");
static_assert(offsetof(Prologue, misc) == 0 && 3 * sizeof(uint32_t) <= HW_ANY_SKIP_WORDS * 8, "misc[2] (any_skip) fits its host words (HW_ANY_SKIP)");
struct SetupArgs {
    StoreView store;
    uint32_t n_parents;
    const uint8_t* parent_cids;    // device copies
    const uint8_t* txmeta_cids;
    const uint8_t* child_cid;      // 38
    const uint8_t* receipts_root;  // 38
    uint32_t skip_tx;
    uint32_t skip_receipts;        // execution-order-only mode: the receipts root is not part of the call
    uint32_t* wbits;
    unsigned long long* err;
    unsigned long long* txerr;     // message-AMT fault word (tx_err_key)
    // outputs
    Prologue* pro;
    uint32_t* f_blk; uint32_t* f_meta; uint64_t* f_base;  // initial frontier: one item per message AMT
    unsigned long long* f_count;
    const uint8_t* sig;     // event signature bytes (zero padded to a multiple of 8) and the Matcher whose t0 this kernel fills
    uint32_t sig_len;
    Matcher* matcher;       // null for a log filter: nothing to hash
    // plan_dense: also plan the dense walk (unsharded calls) into pro->plan, against these limits
    uint32_t plan_dense;
    uint64_t frontier_cap, max_raw;
};

// Amtv0::<MessageReceipt>::load(&receipts_root, &rec_receipts) (events/generator.rs:195-196), root validated
__device__ __forceinline__ void setup_receipts_root(const SetupArgs& a) {
    const StoreView& s = a.store;
    int32_t rb = store_lookup(s, a.receipts_root);
    if (rb < 0) { report_error(a.err, ST_RECEIPTS_ROOT, 0, DC_MISSING, 0); return; }
    witness_mark(s, a.wbits, (uint32_t)rb);
    a.pro->misc[0] = (uint32_t)rb;
    uint32_t len;
    const uint8_t* p = store_block(s, (uint32_t)rb, len);
    Rd r(p, len);
    uint32_t bw, h;
    uint64_t cnt;
    amt_root_begin(r, 0, bw, h, cnt);
    AmtNodeHdr hd;
    (void)amt_node_get(r, 3, h, 0, hd, [](Rd& rv, bool) { (void)parse_receipt(rv); });
    if (r.err) report_error(a.err, ST_RECEIPTS_ROOT, 0, DC_DECODE, r.err);
}

// One-CTA prologue, the independent pieces on different warps so their dependent lookups overlap:
//   thread 0        Amtv0::<MessageReceipt>::load(&receipts_root) (events/generator.rs:195-196), root validated
//   threads 32..95  one parent each: TxMeta → BLS / SECP AMT roots (seeds the walk frontier, AMT ordinal 2b + k)
//   thread 96       keccak256(event_signature) → Matcher.t0 (EventMatcher::new, events/generator.rs:30-35)
//   threads 128..   base witness marks (parent headers, child header, receipts root, TxMeta blocks)
//   thread 0, last  (plan_dense) the dense walk's plan from the roots' heights and counts, once every piece above is done
// Errors go through the atomicMin error word, so the one reported is the one the sequential order meets first.
__global__ void __launch_bounds__(256) k_setup(SetupArgs a) {
    const StoreView& s = a.store;
    const uint32_t t = threadIdx.x, P = a.n_parents;
    uint32_t* const amt_height = a.pro->misc + 64;
    uint64_t* const amt_count = a.pro->amt_count;
    if (t >= 128 && !a.skip_tx) {
        for (uint32_t i = t - 128; i < 2 * P + 2; i += 128) {
            const uint8_t* cid = i < P ? a.parent_cids + 38 * i : (i == P ? a.child_cid : (i == P + 1 ? a.receipts_root : a.txmeta_cids + 38 * (i - P - 2)));
            int32_t b = store_lookup(s, cid);
            if (b < 0) a.pro->misc[1] = 1; else witness_mark(s, a.wbits, (uint32_t)b);
        }
    }
    if (t == 96 && a.matcher) {   // a log filter's values arrive raw
        Digest d;
        keccak256(a.sig, a.sig_len, d);
        for (int k = 0; k < 4; k++) a.matcher->t0[k] = a.pro->t0[k] = d.w[k];
    }
    // TxMeta + message AMT roots (needed for the execution order even when skip_tx). An AMT whose root cannot be loaded keeps
    // a sentinel seed (height / count 0): the walk goes on for the others, and the fault the reference meets FIRST wins the word
    if (t >= 32 && t < 96) for (uint32_t b = t - 32; b < P; b += 64) {
        for (uint32_t k = 0; k < 2; k++) { a.f_meta[2 * b + k] = AMT_SENTINEL; a.f_blk[2 * b + k] = 0; a.f_base[2 * b + k] = 0; amt_height[2 * b + k] = 0; amt_count[2 * b + k] = 0; }
        int32_t tb = store_lookup(s, a.txmeta_cids + 38 * b);
        if (tb < 0) { report_tx_error(a.txerr, 3 * b, 0, 31, DC_MISSING, 0); continue; }
        if (!a.skip_tx) witness_mark(s, a.wbits, (uint32_t)tb);
        uint32_t len;
        const uint8_t* p = store_block(s, (uint32_t)tb, len);
        Rd r(p, len);
        rd_array_exact(r, 2);
        uint32_t c0 = rd_cid(r), c1 = rd_cid(r);
        rd_end(r);
        if (r.err) { report_tx_error(a.txerr, 3 * b, 0, 31, DC_DECODE, r.err); continue; }
        for (uint32_t k = 0; k < 2; k++) {
            int32_t rb = store_lookup(s, p + (k ? c1 : c0));
            if (rb < 0) { report_tx_error(a.txerr, 3 * b + 1 + k, 0, 31, DC_MISSING, 0); break; }
            if (!a.skip_tx) witness_mark(s, a.wbits, (uint32_t)rb);
            uint32_t rl;
            const uint8_t* rp = store_block(s, (uint32_t)rb, rl);
            Rd rr(rp, rl);
            uint32_t bw, h;
            uint64_t cnt;
            amt_root_begin(rr, 0, bw, h, cnt);
            if (rr.err) { report_tx_error(a.txerr, 3 * b + 1 + k, 0, 31, DC_DECODE, rr.err); break; }
            const uint32_t amt = 2 * b + k;
            a.f_blk[amt] = (uint32_t)rb;
            a.f_meta[amt] = make_meta(amt, 1, h);
            a.f_base[amt] = 0;
            amt_height[amt] = h;
            amt_count[amt] = cnt;
        }
    }
    if (t == 0) {
        *a.f_count = 2 * P;
        if (!a.skip_receipts) setup_receipts_root(a);
    }
    if (!a.plan_dense) return;
    __syncthreads();   // heights, counts and every fault of the pieces above are in place
    if (t != 0) return;
    // the whole message list (unsharded): every AMT's range is [0, ∞). The ranges are passed in the slots of per_amt that dense_plan
    // overwrites with the clipped range of the same AMT (it reads each before it writes it).
    const uint32_t namt = 2 * P;
    DenseTables& pl = a.pro->plan;
    for (uint32_t k = 0; k < namt; k++) { pl.per_amt[2ull * namt + k] = 0; pl.per_amt[3ull * namt + k] = UINT64_MAX; }
    uint32_t rounds;
    uint64_t nraw;
    const bool ok = dense_plan(namt, amt_height, amt_count, pl.per_amt + 2ull * namt, pl.per_amt + 3ull * namt, a.frontier_cap, a.max_raw, sizeof(DenseTables),
                               pl.fofs, pl.ftot, pl.per_amt, &rounds, &nraw);
    const bool fault = *(volatile unsigned long long*)a.err != IPCFP_NO_ERROR || *(volatile unsigned long long*)a.txerr != IPCFP_NO_ERROR;
    pl.rounds = rounds;
    pl.nraw = nraw;
    pl.ok = ok && !fault;   // a prologue fault: the general walk finds the fault the reference meets first
}

// ---- message-AMT walk, general form: kernels (per-item code: walk.cuh) --------------------------------------
__global__ void __launch_bounds__(128) k_amt_count(StoreView store, Frontier in, const unsigned long long* in_count, uint32_t round, uint32_t last_round,
                                                   uint32_t cap, uint32_t* counts, const uint64_t* rlo, const uint64_t* rhi) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t cnt = *in_count;
    if (cnt > cap) cnt = cap;
    if (t >= cnt) { counts[t] = 0; return; }   // the grid covers exactly the scanned range
    counts[t] = amt_item_count(store, in.blk[t], in.meta[t], in.base[t], round, last_round, rlo, rhi);
}
__global__ void __launch_bounds__(128) k_amt_expand(ExpandArgs a, const uint32_t* counts, unsigned long long* out_count, const unsigned long long* total) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t t = g >> 3;          // frontier item
    const uint32_t j = (uint32_t)g & 7; // lane of the item
    uint64_t cnt = *a.in_count;
    if (cnt > a.cap) cnt = a.cap;
    if (g == 0) {
        unsigned long long n = *total;
        if (a.round < a.last_round && n > a.cap) { report_tx_error(a.err, IPCFP_TX_EIDX_NONE, 0, 0, DC_UNSUPPORTED, 1); n = a.cap; }
        *out_count = n;
    }
    if (t >= cnt) return;
    amt_item_expand(a, t, j, a.in.blk[t], a.in.meta[t], a.in.base[t], counts[t]);
}

// Rounds whose frontier is guaranteed to fit one CTA (≤ 1024 items) run fused in a single launch:
// count, block-wide scan and expand per level with __syncthreads between levels.
#define TOP_CAP 1024
__global__ void __launch_bounds__(TOP_CAP) k_amt_top(ExpandArgs a0, Frontier ping, Frontier pong, unsigned long long* count_io, uint32_t first_round,
                                                      uint32_t n_rounds, uint64_t* scan_tmp) {
    __shared__ uint32_t s_cnt[TOP_CAP];
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_total;
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    Frontier cur = ping, nxt = pong;
    for (uint32_t rr = 0; rr < n_rounds; rr++) {
        uint32_t round = first_round + rr;
        uint64_t cnt = *count_io;
        if (cnt > TOP_CAP) cnt = TOP_CAP;
        uint32_t c = t < cnt ? amt_item_count(a0.store, cur.blk[t], cur.meta[t], cur.base[t], round, a0.last_round, a0.rlo, a0.rhi) : 0;
        // block exclusive scan of c
        uint32_t x = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (uint32_t)o) x += y; }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint32_t v = s_warp[lane], w = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= (uint32_t)o) w += y; }
            s_warp[lane] = w - v;
            if (lane == 31) s_total = w;
        }
        __syncthreads();
        uint32_t ex = s_warp[warp] + x - c;
        scan_tmp[t] = ex;
        s_cnt[t] = c;
        __syncthreads();
        ExpandArgs a = a0;
        a.in = cur; a.out = nxt; a.round = round; a.out_off = scan_tmp;
        for (uint32_t it = t >> 3; it < cnt; it += TOP_CAP / 8) amt_item_expand(a, it, t & 7, cur.blk[it], cur.meta[it], cur.base[it], s_cnt[it]);
        __syncthreads();
        if (t == 0) {
            unsigned long long n = s_total;
            if (round < a0.last_round && n > a0.cap) { report_tx_error(a0.err, IPCFP_TX_EIDX_NONE, 0, 0, DC_UNSUPPORTED, 1); n = a0.cap; }
            *count_io = n;
        }
        __threadfence();
        __syncthreads();
        Frontier tmp = cur; cur = nxt; nxt = tmp;
    }
}

// The message-AMT fault word ranks a fault by the first index below it in 44 bits (tx_err_key). In an AMT of height ≥ 14 indices
// reach 8^15 = 2^45 (and wrap past 2^64 at height 21), so two faults of one AMT can tie on that field, or compare wrongly, and the
// level decides. When the word names a node fault in such an AMT, this kernel (one thread, error path only) walks that AMT in order
// as Amt::for_each does and overwrites the word with the first fault it meets. Its TxMeta and root header decoded (the word names a
// node fault), so only the nodes are checked.
#define TX_KEY_EXACT_HEIGHT 13   // 8^(13+1) = 2^42: every index of an AMT up to this height fits the key's 44-bit base
__global__ void k_amt_first_fault(StoreView s, const uint8_t* txmeta_cids, uint32_t amt, unsigned long long* word) {
    const uint32_t eidx = 3 * (amt >> 1) + 1 + (amt & 1);
    uint32_t len;
    const uint8_t* p = store_block(s, (uint32_t)store_lookup(s, txmeta_cids + 38 * (amt >> 1)), len);
    Rd rt(p, len);
    rd_array_exact(rt, 2);
    const uint32_t c0 = rd_cid(rt), c1 = rd_cid(rt);
    uint32_t blk[DENSE_MAX_ROUNDS + 1], next[DENSE_MAX_ROUNDS + 1];   // per depth: the node's block and the next slot to visit
    blk[0] = (uint32_t)store_lookup(s, p + ((amt & 1) ? c1 : c0));
    next[0] = 0;
    uint32_t height = 0;
    for (int d = 0; d >= 0;) {
        const uint8_t* q = store_block(s, blk[d], len);
        Rd r(q, len);
        if (d == 0) { uint32_t bw; uint64_t c; amt_root_begin(r, 0, bw, height, c); }
        const uint32_t level = height - (uint32_t)d;
        AmtNodeHdr h;
        amt_node_begin(r, 3, h);
        if (next[d] == 0) {   // entering the node: the whole node is decoded (values included), as the reference's load does
            const uint32_t nv = rd_array(r);
            for (uint32_t v = 0; v < nv && !r.err; v++) (void)rd_cid(r);
            amt_node_finish(r, h, nv, level);
            if (r.err) { *word = tx_err_key(eidx, 0, level, DC_DECODE, r.err); return; }
        }
        const uint32_t bm8 = (uint32_t)h.bm.b0 & 0xffu & ~((1u << next[d]) - 1u);
        if (!h.nl || !bm8 || next[d] >= 8) { d--; continue; }
        const uint32_t slot = (uint32_t)__ffs(bm8) - 1;
        next[d] = slot + 1;
        const uint32_t rank = (uint32_t)__popc((uint32_t)h.bm.b0 & ((1u << slot) - 1u));
        const int32_t child = store_lookup(s, q + h.links_off + 43 * rank + 5);
        if (child < 0) { *word = tx_err_key(eidx, 0, level - 1, DC_MISSING, 0); return; }
        d++;
        blk[d] = (uint32_t)child;
        next[d] = 0;
    }
}

// The dense walk (amt_item_dense, walk.cuh) over the plan in a.tables, in two launches: k_amt_dense walks rounds 0 .. rounds-2 as ONE
// persistent cooperative grid with grid.sync() between rounds, k_amt_dense_leaf the last round. A level marks the blocks of the children
// it resolves, so after the first launch every message-AMT block is recorded; the leaf round only writes the raw message list.
// A plan that is not ok raises `fail` (the host then takes the general walk).
#define DENSE_THREADS 256
__global__ void __launch_bounds__(DENSE_THREADS) k_amt_dense(DenseArgs a) {
    const DenseTables& tb = *a.tables;
    if (!tb.ok) { if (blockIdx.x == 0 && threadIdx.x == 0) *a.fail = 1; return; }   // the same in every thread: no one waits in grid.sync
    cg::grid_group grid = cg::this_grid();
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint32_t round = 0; round + 1 < tb.rounds; round++) {
        // `fail` may rise while the round runs: a thread that sees it skips its items but still meets every grid.sync
        if (!*(volatile uint32_t*)a.fail) {
            const Frontier in = (round & 1) ? a.pong : a.ping, out = (round & 1) ? a.ping : a.pong;
            const uint64_t n8 = (uint64_t)tb.ftot[round] * 8;
            for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n8; g += stride)
                amt_item_dense(a, in, out, round, (uint32_t)(g >> 3), (uint32_t)g & 7);
        }
        if (round + 2 < tb.rounds) grid.sync();
    }
}
__global__ void __launch_bounds__(DENSE_THREADS) k_amt_dense_leaf(DenseArgs a) {
    const DenseTables& tb = *a.tables;
    if (!tb.ok) { if (blockIdx.x == 0 && threadIdx.x == 0) *a.fail = 1; return; }
    if (*(volatile uint32_t*)a.fail) return;
    const uint32_t round = tb.rounds - 1;
    const Frontier in = (round & 1) ? a.pong : a.ping, out = (round & 1) ? a.ping : a.pong;
    const uint64_t n8 = (uint64_t)tb.ftot[round] * 8;
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n8; g += (uint64_t)gridDim.x * blockDim.x)
        amt_item_dense(a, in, out, round, (uint32_t)(g >> 3), (uint32_t)g & 7);
}

// first-seen dedup of the raw execution list (events/utils.rs:56-91): hash set keyed by the full
// CID holding the smallest position; an entry survives iff it holds its own position.
__global__ void k_dedup_insert(const RawCid* __restrict__ raw, uint64_t n, unsigned long long* table, uint64_t mask) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    RawCid c = raw[i];
    uint64_t h = rawcid_hash(c);
    uint32_t fp = (uint32_t)(h >> 32) | 1u;
    unsigned long long mine = ((unsigned long long)fp << 32) | (unsigned long long)(i + 1);
    uint64_t slot = h & mask;
    for (;;) {
        unsigned long long e = table[slot];
        if (e == 0) { e = atomicCAS(&table[slot], 0ull, mine); if (e == 0) return; }
        if ((uint32_t)(e >> 32) == fp && rawcid_eq(raw[(uint32_t)e - 1], c)) { atomicMin(&table[slot], mine); return; }
        slot = (slot + 1) & mask;
    }
}
__global__ void k_dedup_flags(const RawCid* __restrict__ raw, uint64_t n, const unsigned long long* __restrict__ table, uint64_t mask,
                              uint32_t* keep_bits) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool keep = false;
    if (i < n) {
        RawCid c = raw[i];
        uint64_t h = rawcid_hash(c);
        uint32_t fp = (uint32_t)(h >> 32) | 1u;
        uint64_t slot = h & mask;
        for (;;) {
            unsigned long long e = table[slot];
            if (e == 0) break;  // cannot happen: every entry was inserted
            if ((uint32_t)(e >> 32) == fp && rawcid_eq(raw[(uint32_t)e - 1], c)) { keep = ((uint32_t)e - 1) == (uint32_t)i; break; }
            slot = (slot + 1) & mask;
        }
    }
    __syncwarp();
    unsigned b = __ballot_sync(0xffffffffu, keep);
    if ((threadIdx.x & 31) == 0) keep_bits[i >> 5] = b;
}

// ------------------------------------------------------------------------------------------ host orchestration
struct EventResultBox {
    ipcfp_event_result r;  // must stay first
    PinnedArray matching, proofs, blob;
    WitnessOut wit;
    PinnedArray union_host;       // sharded calls with IPCFP_SHARDED_UNION_TO_HOST
    PinnedArray json;             // IPCFP_RESULT_JSON: the EventProofBundle text
    AsyncBuf<RawCid> shard_exec;  // shard mode: this shard's slice of the raw execution list, kept on the device
};

static void throw_device_error(uint64_t key) {
    uint32_t stage = (uint32_t)(key >> 56), code = (uint32_t)(key >> 8) & 0xff, detail = (uint32_t)key & 0xff;
    uint64_t index = (key >> 16) & 0xFFFFFFFFFFull;
    ipcfp_status st;
    const char* what;
    switch (code) {
        case DC_MISSING: st = IPCFP_ERR_MISSING_BLOCK; what = "missing block"; break;
        case DC_DECODE: st = IPCFP_ERR_DECODE; what = "decode error"; break;
        case 0:
        case DC_MISSING_EXEC: st = IPCFP_ERR_MISSING_EXEC; what = "Missing message at index"; break;
        case DC_UNSUPPORTED: st = IPCFP_ERR_UNSUPPORTED; what = "unsupported input (frontier overflow)"; break;
        default: st = IPCFP_ERR_DECODE; what = "error"; break;
    }
    uint64_t out_index = UINT64_MAX;
    const char* stage_name = "?";
    switch (stage) {
        case ST_TXMETA:
            stage_name = "message AMTs";
            if (index != 0xFFFFFFFFFFull && index % 3 == 0 && code == DC_MISSING) out_index = index / 3;  // missing TxMeta of parent b
            break;
        case ST_RECEIPTS_ROOT: stage_name = "receipts AMT root"; break;
        case ST_PASS1: stage_name = "pass 1"; out_index = index; break;
        case ST_PASS2: stage_name = "pass 2"; out_index = index; break;
        case ST_WITNESS: stage_name = "materialize"; break;
        default: break;
    }
    throw Error(st, std::string(what) + " in " + stage_name + " (detail " + std::to_string(detail) + ")", out_index);
}

// message-AMT fault word (tx_err_key, common.cuh)
static void throw_tx_error(uint64_t key) {
    const uint32_t eidx = (uint32_t)(key >> 56), code = (uint32_t)(key >> 4) & 7, detail = (uint32_t)key & 15;
    ipcfp_status st;
    const char* what;
    switch (code) {
        case DC_MISSING: st = IPCFP_ERR_MISSING_BLOCK; what = "missing block"; break;
        case DC_UNSUPPORTED: st = IPCFP_ERR_UNSUPPORTED; what = "unsupported input (frontier overflow)"; break;
        default: st = IPCFP_ERR_DECODE; what = "decode error"; break;
    }
    uint64_t out_index = UINT64_MAX;
    if (eidx != IPCFP_TX_EIDX_NONE && eidx % 3 == 0 && code == DC_MISSING) out_index = eidx / 3;   // missing TxMeta of parent b
    throw Error(st, std::string(what) + " in message AMTs (detail " + std::to_string(detail) + ")", out_index);
}
// the failure the reference's sequential order meets first: message-AMT stage before everything else, a missing base-witness block last
static void throw_first(uint64_t tx_key, uint64_t err_key, bool missing_base = false) {
    if (tx_key != IPCFP_NO_ERROR) throw_tx_error(tx_key);
    if (err_key != IPCFP_NO_ERROR) throw_device_error(err_key);
    if (missing_base) throw Error(IPCFP_ERR_MISSING_BLOCK, "missing block (base witness CID not in the store)");
}

void tipset_upload(Store* s, const ipcfp_tipset_desc* t, TipsetDev& td) {
    s->use();
    if (!t || !t->child_cid || !t->receipts_root || (t->n_parents && (!t->parent_cids || !t->parent_txmeta_cids)))
        throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor has null fields");
    if (t->n_parents > IPCFP_MAX_PARENTS) throw Error(IPCFP_ERR_UNSUPPORTED, "too many parent blocks");
    if (t->n_receipts >= 0xffffffffull) throw Error(IPCFP_ERR_UNSUPPORTED, "more than 2^32 receipts");
    if (t->n_receipts && (!t->events_roots || !t->has_events_root)) throw Error(IPCFP_ERR_INVALID_ARG, "events roots missing");
    td.device = s->device;
    td.parent_epoch = t->parent_epoch; td.child_epoch = t->child_epoch; td.n_parents = t->n_parents;
    td.parent_cids.assign(t->parent_cids, t->parent_cids + 38ull * t->n_parents);
    td.txmeta_cids.assign(t->parent_txmeta_cids, t->parent_txmeta_cids + 38ull * t->n_parents);
    memcpy(td.child_cid, t->child_cid, 38);
    memcpy(td.receipts_root, t->receipts_root, 38);
    td.has_state_root = t->child_parent_state_root != nullptr;
    if (td.has_state_root) memcpy(td.child_state_root, t->child_parent_state_root, 38);
    td.n_receipts = t->n_receipts;
    td.events_roots.alloc(t->n_receipts * 38 + 64);
    td.has_root.alloc(t->n_receipts + 64);
    if (t->n_receipts) {
        IPCFP_CUDA(cudaMemcpyAsync(td.events_roots.p, t->events_roots, t->n_receipts * 38, cudaMemcpyHostToDevice, s->stream));
        IPCFP_CUDA(cudaMemcpyAsync(td.has_root.p, t->has_events_root, t->n_receipts, cudaMemcpyHostToDevice, s->stream));
    }
}

namespace {
static constexpr size_t STAGE_TABLES = 32768;   // second half of the store's staging block: dense-walk tables

// The execution order of a tipset (events/generator.rs:122-196: collect_base_witness, record_transaction_amts, build_execution_order):
// k_setup, the message-AMT walk and the first-seen dedup, with the host synchronisations and fault handling around them. Two modes,
// fixed at construction:
//   with witness  (generate_event_proof) base and message-AMT blocks are recorded (unless IPCFP_SCAN_SKIP_TX_AMTS), the receipts root
//                 is loaded, and the witness snapshot and its copy start behind the walk
//   order only    (build_execution_order) no witness and no receipts root: the verifier and the message fetch round
// xch != nullptr: this call is one shard of a multi-GPU call (see EventCall); a failure is then kept in pend_tx / pend_err.
struct ExecOrderBuild {
    Store* s;
    cudaStream_t st;
    const TipsetDev* td;   // with witness: the call's tipset; null: order only
    const bool with_witness;
    uint32_t n_parents;
    const uint8_t* txmeta_cids_h;
    uint64_t n_receipts;
    bool sharded;
    uint64_t lo, hi;
    ShardExchange* xch;
    bool skip_tx, by_ref;
    uint64_t nblk;
    uint64_t pend_tx = IPCFP_NO_ERROR, pend_err = IPCFP_NO_ERROR;   // first failure seen so far (xch mode)
    unsigned long long* dw;
    uint64_t* hw;
    // stage
    size_t tables_off = 0;
    AsyncBuf<uint8_t> small;
    uint8_t* d_cids = nullptr;
    // setup
    AsyncBuf<uint32_t> wbits;
    uint32_t namt = 0;
    uint64_t cap = 0;
    AsyncBuf<uint32_t> fA_blk, fA_meta, fB_blk, fB_meta;
    AsyncBuf<uint64_t> fA_base, fB_base;
    AsyncBuf<Prologue> pro;
    uint32_t* misc = nullptr;
    uint32_t frontier_cap = 0;
    uint64_t max_raw_dev = 0;
    bool force_general = false, plan_on_device = false;
    SetupArgs sa{};   // order only: no parent, child or receipts-root CID (k_setup reads them to record the witness and load the root)
    // walk
    const Prologue* ph;   // the prologue's head as the host reads it, once publish_prologue and a synchronisation have run
    bool early_fault = false, missing_base = false;
    uint32_t receipts_root_blk = 0, last_round = 0;
    // share of the concatenated ("raw") message list this call walks: everything, or — sharded — [Nraw*lo/N, Nraw*hi/N) expressed as
    // one index range per AMT
    std::vector<uint64_t> h_rng = std::vector<uint64_t>(4 * IPCFP_MAX_PARENTS, 0);
    uint64_t nraw_total = 0;
    AsyncBuf<uint32_t> counts;
    AsyncBuf<uint64_t> out_off, scratch;
    unsigned long long *ccount = nullptr, *ncount = nullptr, *total_dev = nullptr;
    AsyncBuf<RawCid> exec_raw;
    uint64_t raw_cap = 0;
    DensePlan plan;
    AsyncBuf<uint64_t> d_foff;
    AsyncBuf<uint32_t> d_flen;
    DenseArgs da;
    AsyncBuf<uint64_t> d_rng;
    AsyncBuf<uint32_t> g_blk[2], g_meta[2];
    AsyncBuf<uint64_t> g_base[2];
    bool dense_used = false, xch_early = false;
    std::optional<WitnessBuilder> wbuild;
    bool early_copy = true;   // with witness: snapshot the witness and start its copy behind the walk (false: the caller materialises wbits)
    uint64_t nraw = 0;
    bool xch_stale = false;
    // dedup
    AsyncBuf<uint32_t> exec_idx, keep_bits;
    unsigned long long* n_exec_dev = nullptr;

    // order only: the tipset of n_parents parent blocks with these TxMeta CIDs (host)
    ExecOrderBuild(Store* s_, uint32_t n_parents_, const uint8_t* txmeta_cids) : ExecOrderBuild(s_, nullptr, n_parents_, txmeta_cids, IPCFP_SCAN_SKIP_TX_AMTS) {}
    // with witness: the tipset td_, the call's flags, its receipt range [lo, hi) and, sharded over NCCL, its exchange
    ExecOrderBuild(Store* s_, const TipsetDev* td_, uint32_t n_parents_, const uint8_t* txmeta_cids, uint32_t flags, bool sharded_ = false,
                   uint64_t lo_ = 0, uint64_t hi_ = 0, ShardExchange* xch_ = nullptr)
        : s(s_), st(s_->stream), td(td_), with_witness(td_ != nullptr), n_parents(n_parents_), txmeta_cids_h(txmeta_cids),
          n_receipts(td_ ? td_->n_receipts : 0), sharded(sharded_), lo(lo_), hi(hi_), xch(xch_), skip_tx((flags & IPCFP_SCAN_SKIP_TX_AMTS) != 0),
          by_ref((flags & IPCFP_WITNESS_BY_REFERENCE) != 0), nblk(s_->n), dw(s_->dev_words.p), hw(s_->host_words.p),
          ph((const Prologue*)(s_->host_words.p + HW_PROLOGUE)) {}

    void note_errors() {   // the fault words as the last publish left them
        if (!xch) { throw_first(hw[DW_TX_ERR], hw[DW_ERR]); return; }
        pend_tx = std::min<uint64_t>(pend_tx, hw[DW_TX_ERR]);
        pend_err = std::min<uint64_t>(pend_err, hw[DW_ERR]);
    }
    void publish_prologue() { publish_words(s, HW_PROLOGUE, PRO_HEAD_WORDS, pro.p); }
    void read_prologue() {   // the fault words as the prologue left them, and its head
        early_fault = hw[DW_ERR] != IPCFP_NO_ERROR || hw[DW_TX_ERR] != IPCFP_NO_ERROR;
        receipts_root_blk = ph->misc[0];
        missing_base = ph->misc[1] != 0;
        last_round = 0;
        for (uint32_t k = 0; k < namt; k++) last_round = std::max(last_round, ph->misc[64 + k]);
        nraw_total = shard_amt_ranges(namt, ph->amt_count, sharded, lo, hi, n_receipts, h_rng.data(), h_rng.data() + 2 * IPCFP_MAX_PARENTS);
    }
    void ensure_scratch(uint64_t n) {   // scan scratch for n items
        if (scratch.n < scan_scratch_elems(n + 64) + 64) scratch.alloc(scan_scratch_elems(n + 64) + 64, st);
    }

    // ---- the call's device words reset; then a head of `head` bytes, which fill_head writes at its host address (zeroed), and the
    // tipset CIDs go up in ONE copy from the store's pinned staging block (no host sync). Returns the head's device address.
    template <class F>
    uint8_t* stage(size_t head, F&& fill_head) {
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_BEGIN], st));
        IPCFP_CUDA(cudaMemsetAsync(dw + DW_ERR, 0xff, 8, st));
        IPCFP_CUDA(cudaMemsetAsync(dw + DW_FRONTIER_A, 0, 40 * 8, st));   // the 40 counters behind the error word
        IPCFP_CUDA(cudaMemsetAsync(dw + DW_TX_ERR, 0xff, 8, st));

        //   head | TxMeta, parent, child, receipts-root CIDs (order only: the TxMeta CIDs)
        const size_t cids_bytes = with_witness ? 38ull * (2 * n_parents + 2) : 38ull * n_parents;
        const size_t small_bytes = head + cids_bytes + 64;
        tables_off = std::max<size_t>(STAGE_TABLES, (small_bytes + 63) & ~(size_t)63);
        if (!s->stage.p || s->stage.cap < tables_off + STAGE_TABLES) s->stage = PinnedArray(s->pool, tables_off + STAGE_TABLES);
        uint8_t* hs = s->stage.as<uint8_t>();
        memset(hs, 0, small_bytes);
        fill_head(hs);
        small.alloc(small_bytes, st);
        d_cids = small.p + head;
        uint8_t* hc = hs + head;
        memcpy(hc, txmeta_cids_h, 38ull * n_parents); hc += 38ull * n_parents;
        if (with_witness) {
            memcpy(hc, td->parent_cids.data(), td->parent_cids.size()); hc += td->parent_cids.size();
            memcpy(hc, td->child_cid, 38); hc += 38;
            memcpy(hc, td->receipts_root, 38);
        }
        IPCFP_CUDA(cudaMemcpyAsync(small.p, hs, small_bytes, cudaMemcpyHostToDevice, st));
        return small.p;
    }

    // ---- the execution order: k_setup (sig / matcher: the event signature whose keccak256 it writes into the Matcher's t0; null for
    // none), the walk and its settlement, the dedup
    void build(const uint8_t* sig, uint32_t sig_len, Matcher* matcher) {
        setup(sig, sig_len, matcher);
        walk();
        settle_walk();
        dedup();
    }

    // ---- witness bitmap + k_setup
    void setup(const uint8_t* sig, uint32_t sig_len, Matcher* matcher) {
        wbits.alloc((nblk + 31) / 32 + 8, st);
        wbits.zero();
        namt = 2 * n_parents;   // k_setup seeds one frontier item per message AMT
        cap = 4 * nblk + 1024;
        fA_blk.alloc(cap, st); fA_meta.alloc(cap, st); fB_blk.alloc(cap, st); fB_meta.alloc(cap, st);
        fA_base.alloc(cap, st); fB_base.alloc(cap, st);
        pro.alloc(1, st);
        pro.zero();
        misc = &pro.p->misc[0];
        frontier_cap = (uint32_t)std::min<uint64_t>(cap, 0xffffffffull);
        // Every message of a parent block is executed, so no message AMT counts more values than there are receipts: a dense walk of an
        // unsharded call writes at most n_parents × n_receipts entries (a plan above that goes to the general walk).
        max_raw_dev = std::min<uint64_t>(8ull * cap, (uint64_t)n_parents * n_receipts + 1024);
        force_general = getenv("IPCFP_BFS_GENERAL") != nullptr;   // read per call: tests toggle it
        // Unsharded calls plan the dense walk on the device (k_setup) and read the prologue back only together with the witness
        // snapshot's counts. A sharded call needs its share's length on the host before its walk (early H0, below), and the
        // order-only mode has no receipt count for the device plan's bound: both read the prologue back first (host synchronisation 1).
        plan_on_device = with_witness && !sharded && !force_general;
        sa.store = s->view; sa.n_parents = n_parents;
        sa.txmeta_cids = d_cids;
        if (with_witness) { sa.parent_cids = d_cids + 38ull * n_parents; sa.child_cid = d_cids + 76ull * n_parents; sa.receipts_root = sa.child_cid + 38; }
        sa.skip_tx = skip_tx; sa.skip_receipts = with_witness ? 0 : 1; sa.wbits = wbits.p; sa.err = dw + DW_ERR; sa.txerr = dw + DW_TX_ERR;
        sa.pro = pro.p;
        sa.f_blk = fA_blk.p; sa.f_meta = fA_meta.p; sa.f_base = fA_base.p; sa.f_count = dw + DW_FRONTIER_A;
        sa.sig = sig; sa.sig_len = sig_len;
        sa.matcher = matcher;
        sa.plan_dense = plan_on_device ? 1 : 0; sa.frontier_cap = frontier_cap; sa.max_raw = max_raw_dev;
        k_setup<<<1, 256, 0, st>>>(sa); IPCFP_LAUNCH_CHECK();
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_SETUP], st));
    }

    // ---- message AMT walk (recording + raw execution list): dense if the plan holds, else general
    void walk() {
        counts.alloc(cap + 1024, st);
        out_off.alloc(cap + 1024, st); scratch.alloc(scan_scratch_elems(std::max<uint64_t>(cap, hi - lo) + 64) + 64, st);
        ccount = dw + DW_FRONTIER_A; ncount = dw + DW_FRONTIER_B; total_dev = dw + DW_LEVEL_TOTAL;
        if (!plan_on_device) {   // the dense walk planned here
            publish_words(s, 0, DW_TX_ERR + 1);
            publish_prologue();
            IPCFP_CUDA(cudaStreamSynchronize(st));
            // A fault seen by the prologue (TxMeta / AMT root / receipts root) is NOT thrown yet: the reference walks the message AMTs
            // before it loads the receipts root, and a fault inside an earlier AMT precedes a missing later root — walk first (general
            // kernels: they cope with the sentinel seeds), then report the first one in the reference's order.
            read_prologue();
            if (namt > 0 && !force_general && !early_fault)
                plan = make_dense_plan(namt, ph->misc + 64, ph->amt_count, h_rng.data(), h_rng.data() + 2 * IPCFP_MAX_PARENTS, frontier_cap, 8ull * cap,
                                       sizeof(DenseTables));
        }
        memset(&da, 0, sizeof da);
        dense_used = plan_on_device || plan.ok;   // device plan: whether it is ok is known at the next synchronisation
        if (dense_used) run_dense(); else run_general();
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_RAW_LIST], st));
    }
    // (a) the dense walk (see k_amt_dense): rounds 0 .. rounds-2 in one cooperative launch, then the leaf round
    void run_dense() {
        if (!plan_on_device) {   // the host's plan goes where k_setup writes it for unsharded calls
            static_assert(sizeof(DenseTables) <= STAGE_TABLES, "the dense plan must fit its staging slot");
            DenseTables* ht = (DenseTables*)(s->stage.as<uint8_t>() + tables_off);
            memset(ht, 0, sizeof *ht);
            ht->ok = 1; ht->rounds = plan.rounds; ht->nraw = plan.nraw;
            std::copy(plan.per_amt.begin(), plan.per_amt.end(), ht->per_amt);
            std::copy(plan.fofs.begin(), plan.fofs.end(), ht->fofs);
            std::copy(plan.ftot.begin(), plan.ftot.end(), ht->ftot);
            IPCFP_CUDA(cudaMemcpyAsync(&pro.p->plan, ht, sizeof(DenseTables), cudaMemcpyHostToDevice, st));
        }
        raw_cap = plan_on_device ? max_raw_dev : plan.nraw;
        exec_raw.alloc(raw_cap + 64, st);
        // a dense walk that succeeds writes every entry of [0, nraw), and the host reads none of it otherwise. A sharded call's early
        // exchange reads the list before the host knows whether the walk succeeded: there an entry the walk did not write must never
        // look like a message CID.
        if (!plan_on_device) exec_raw.zero();
        const DenseTables* tb = &pro.p->plan;
        da.store = s->view;
        da.ping = Frontier{fA_blk.p, fA_meta.p, fA_base.p}; da.pong = Frontier{fB_blk.p, fB_meta.p, fB_base.p};
        da.vals = exec_raw.p;
        da.tables = tb;
        da.vbase = tb->per_amt; da.cnt = tb->per_amt + namt; da.lo = tb->per_amt + 2ull * namt; da.hi = tb->per_amt + 3ull * namt;
        da.fofs = tb->fofs; da.ftot = tb->ftot;
        da.namt = namt; da.record = skip_tx ? 0 : 1; da.wbits = wbits.p; da.fail = (uint32_t*)(dw + DW_DENSE_FAIL);
        // frontier items of a round ≥ 1: an AMT holding c values has at most c/8 + 1 nodes on any level
        uint64_t fmax = 1;
        if (plan_on_device) fmax = max_raw_dev / 8 + namt + 8;
        else for (uint32_t r = 0; r < plan.rounds; r++) fmax = std::max<uint64_t>(fmax, plan.ftot[r]);
        d_foff.alloc(2 * fmax + 8, st); d_flen.alloc(2 * fmax + 8, st);
        da.f_off[0] = d_foff.p; da.f_off[1] = d_foff.p + fmax; da.f_len[0] = d_flen.p; da.f_len[1] = d_flen.p + fmax;
        if (!s->walk_grid) {   // the persistent grid: every CTA of it resident at once
            int per_sm = 0, sms = 0;
            IPCFP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_amt_dense, DENSE_THREADS, 0));
            IPCFP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s->device));
            s->walk_grid = (unsigned)std::max(1, per_sm * sms);
        }
        void* args[] = {&da};
        IPCFP_CUDA(cudaLaunchCooperativeKernel((const void*)k_amt_dense, s->walk_grid, DENSE_THREADS, args, 0, st)); IPCFP_LAUNCH_CHECK();
        k_amt_dense_leaf<<<s->walk_grid, DENSE_THREADS, 0, st>>>(da); IPCFP_LAUNCH_CHECK();
    }
    // (b) the general walk: count → scan → expand per level, any AMT shape, exact errors. It is the fallback, and it sizes every
    // buffer by what it walks rather than by the store: each parent block's AMTs are walked on their own, so parents that share their
    // messages need a frontier per parent while the store holds those nodes once. Below the fused rounds it synchronises once per level
    // and allocates that level's output from the exact total its scan computed.
    void run_general() {
        d_rng.alloc(4 * IPCFP_MAX_PARENTS, st);
        IPCFP_CUDA(cudaMemcpyAsync(d_rng.p, h_rng.data(), h_rng.size() * 8, cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
        auto ensure_g = [&](int i, uint64_t n) {
            if (g_blk[i].n < n) { g_blk[i].alloc(n, st); g_meta[i].alloc(n, st); g_base[i].alloc(n, st); }
        };
        auto gview = [&](int i) { return Frontier{g_blk[i].p, g_meta[i].p, g_base[i].p}; };
        // the fused rounds' last output can be 8 × TOP_CAP items however small the store is: both ping-pong buffers hold that much,
        // and the seeds k_setup wrote move into the first
        ensure_g(0, 8 * TOP_CAP); ensure_g(1, 8 * TOP_CAP);
        IPCFP_CUDA(cudaMemcpyAsync(g_blk[0].p, fA_blk.p, namt * 4ull, cudaMemcpyDeviceToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(g_meta[0].p, fA_meta.p, namt * 4ull, cudaMemcpyDeviceToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(g_base[0].p, fA_base.p, namt * 8ull, cudaMemcpyDeviceToDevice, st));
        int cur = 0;   // g buffer holding the frontier of `round`
        ccount = dw + DW_FRONTIER_A; ncount = dw + DW_FRONTIER_B;
        ExpandArgs ea;
        ea.store = s->view; ea.last_round = last_round; ea.record = skip_tx ? 0 : 1; ea.wbits = wbits.p; ea.err = dw + DW_TX_ERR;
        ea.vals = nullptr; ea.cap = 8 * TOP_CAP;
        ea.rlo = d_rng.p; ea.rhi = d_rng.p + 2 * IPCFP_MAX_PARENTS;
        auto alloc_vals = [&](uint64_t n) {
            raw_cap = n;
            exec_raw.alloc(raw_cap + 64, st);
            exec_raw.zero();
            ea.vals = exec_raw.p;
        };
        // fused single-CTA rounds while the static frontier bound namt · 8^round fits one CTA
        auto bound_of = [&](uint32_t round) { uint64_t b = namt; for (uint32_t k = 0; k < round && b <= TOP_CAP; k++) b *= 8; return b; };
        uint32_t top_rounds = 0;
        while (top_rounds <= last_round && bound_of(top_rounds) <= TOP_CAP) top_rounds++;
        uint32_t round = 0;
        if (top_rounds) {
            if (top_rounds > last_round) alloc_vals(bound_of(last_round) * 8);  // the last round is inside the fused kernel
            ExpandArgs a0 = ea;
            a0.in = gview(0); a0.in_count = ccount; a0.out = gview(1); a0.round = 0; a0.out_off = out_off.p;
            k_amt_top<<<1, TOP_CAP, 0, st>>>(a0, gview(0), gview(1), ccount, 0, top_rounds, out_off.p); IPCFP_LAUNCH_CHECK();
            cur = top_rounds & 1;
            round = top_rounds;
        }
        if (round > last_round) return;   // *ccount holds the number of raw execution entries
        publish_words(s, (uint32_t)(ccount - dw), 1);
        IPCFP_CUDA(cudaStreamSynchronize(st));
        uint64_t items = hw[ccount - dw];
        for (; round <= last_round; round++) {
            const uint64_t slots = (uint64_t)div_up(std::max<uint64_t>(items, 1), 128) * 128;
            if (counts.n < slots) { counts.alloc(slots, st); out_off.alloc(slots, st); }
            ensure_scratch(slots);
            k_amt_count<<<(unsigned)(slots / 128), 128, 0, st>>>(s->view, gview(cur), ccount, round, last_round, (uint32_t)items, counts.p, ea.rlo, ea.rhi);
            IPCFP_LAUNCH_CHECK();
            exclusive_scan_u32(counts.p, out_off.p, slots, (uint64_t*)total_dev, scratch.p, st);
            publish_words(s, DW_LEVEL_TOTAL, 1);
            IPCFP_CUDA(cudaStreamSynchronize(st));
            const uint64_t total = hw[DW_LEVEL_TOTAL];
            if (round == last_round) alloc_vals(total);   // before `a` copies ea.vals
            ExpandArgs a = ea;
            a.in = gview(cur); a.in_count = ccount; a.round = round; a.out_off = out_off.p; a.out = gview(cur ^ 1);
            a.cap = (uint32_t)items;   // clamps the input count; every output position is below `total`
            if (round < last_round) {
                // a level of 2^32 nodes is 64 GB of frontier alone: device memory runs out before this refuses anything
                if (std::max(total, items) >= 0xffffffffull) throw Error(IPCFP_ERR_UNSUPPORTED, "message-AMT walk: a level of 2^32 nodes or more");
                ensure_g(cur ^ 1, std::max(total, items) + 1);
                a.out = gview(cur ^ 1);
                a.cap = (uint32_t)(std::max(total, items) + 1);
                cur ^= 1;
            }
            k_amt_expand<<<div_up(std::max<uint64_t>(items, 1) * 8, 128), 128, 0, st>>>(a, counts.p, ncount, total_dev); IPCFP_LAUNCH_CHECK();
            std::swap(ccount, ncount);
            items = total;
        }
        // *ccount now holds the number of raw execution entries.
    }
    // Witness snapshot: base witness + every message-AMT block are final at this point — start moving them to the host while pass 1 /
    // pass 2 run (witness.cu). Publishes the error word, frontier counters, witness counts, dense-walk flag and gather split.
    void snapshot_and_sync(bool with_prologue) {
        if (wbuild) wbuild->snapshot(wbits.p);
        publish_words(s, 0, DW_SPLIT_BYTES + 1);
        if (with_prologue) publish_prologue();
        IPCFP_CUDA(cudaStreamSynchronize(st));
        if (with_prologue) read_prologue();
    }

    // ---- after the walk: early H0, snapshot, the dense fallback, the first fault of a tall AMT, the capacity check, late H0
    void settle_walk() {
        if (xch) {
            // EARLY H0: with dense message AMTs the length of this shard's slice is known from the roots alone (plan.nraw), so the peers can
            // agree on the slices while the walk is still running and the whole execution-order exchange goes onto the (high-priority)
            // exchange stream right behind it — it then runs under the witness snapshot, the host's sync and pass 1 instead of after them.
            // A shard that cannot promise its slice yet (sparse AMTs → general walk, a fault in the prologue) says so and EVERY shard takes
            // the late path below; a promise that turns out wrong (the dense walk raised its flag) is repaired after pass 2 (`stale`).
            xch->agree_early(plan.ok && !early_fault, plan.ok ? plan.nraw : 0, nraw_total);
            xch_early = xch->all_early;
            if (xch_early) xch->start_exchange(exec_raw.p);
        }
        if (with_witness && early_copy) {
            wbuild.emplace(s);
            wbuild->by_ref = by_ref;
        }
        snapshot_and_sync(plan_on_device);
        if (dense_used && hw[DW_DENSE_FAIL] != 0) {   // the AMTs are not what the dense walk assumes (or its plan was not ok): redo the walk with the general kernels
            dense_used = false;
            k_setup<<<1, 256, 0, st>>>(sa); IPCFP_LAUNCH_CHECK();   // re-seed the frontier (same outputs as before)
            run_general();
            IPCFP_CUDA(cudaEventRecord(s->ev[EV_RAW_LIST], st));
            snapshot_and_sync(false);
        }
        const uint32_t ccount_idx = (uint32_t)(ccount - dw);
        if (!sharded && hw[DW_TX_ERR] != IPCFP_NO_ERROR) {
            // a node fault (level < 31) in a message AMT tall enough for its indices to outgrow the key: resolve it in order
            const uint64_t key = hw[DW_TX_ERR];
            const uint32_t eidx = (uint32_t)(key >> 56), level = 31u - ((uint32_t)(key >> 7) & 31u);
            if (eidx != IPCFP_TX_EIDX_NONE && eidx % 3 != 0 && level < 31) {
                const uint32_t amt = 2 * (eidx / 3) + eidx % 3 - 1;
                if (ph->misc[64 + amt] > TX_KEY_EXACT_HEIGHT) {
                    k_amt_first_fault<<<1, 1, 0, st>>>(s->view, sa.txmeta_cids, amt, dw + DW_TX_ERR); IPCFP_LAUNCH_CHECK();
                    publish_words(s, DW_TX_ERR, 1);
                    IPCFP_CUDA(cudaStreamSynchronize(st));
                }
            }
        }
        note_errors();
        if (!dense_used && hw[ccount_idx] > raw_cap) {
            if (!xch) throw Error(IPCFP_ERR_UNSUPPORTED, "unsupported input (message list longer than the walk's capacity)");
            pend_tx = std::min<uint64_t>(pend_tx, tx_err_key(IPCFP_TX_EIDX_NONE, 0, 0, DC_UNSUPPORTED, 1));
        }
        nraw = dense_used ? (plan_on_device ? ph->plan.nraw : plan.nraw) : std::min<uint64_t>(hw[ccount_idx], raw_cap);
        // early mode: the exchange that is running was fed the PLANNED slice; if the dense walk gave up, the list was rewritten underneath it
        xch_stale = xch_early && (!dense_used || nraw != plan.nraw);
        if (xch && !xch_early && (pend_tx != IPCFP_NO_ERROR || pend_err != IPCFP_NO_ERROR)) {
            // this shard has no message list: tell the peers (H0), then fail — with the first error over ALL shards, like them
            xch->agree_slices(pend_tx, pend_err, 0);
            throw_first(xch->g_tx, xch->g_err);
        }
        if (wbuild) wbuild->start_copy(hw[DW_WIT_A], hw[DW_WIT_A_BYTES], hw[DW_SPLIT_IDX], hw[DW_SPLIT_BYTES]);
        if (xch && !xch_early) {
            // LATE H0 (some shard could not promise its slice before its walk was over): agree on the slices now and start the exchange
            xch->agree_slices(IPCFP_NO_ERROR, IPCFP_NO_ERROR, nraw);
            if (!xch->peers_ok) { IPCFP_CUDA(cudaStreamSynchronize(st)); throw_first(xch->g_tx, xch->g_err); }
            xch->start_exchange(exec_raw.p);
        }
    }

    // ---- first-seen dedup of the raw list: the execution order
    void dedup() {
        exec_idx.alloc(nraw + 32, st); keep_bits.alloc((nraw + 31) / 32 + 8, st);
        n_exec_dev = dw + DW_N_EXEC;
        if (sharded) IPCFP_CUDA(cudaMemsetAsync(n_exec_dev, 0, 8, st));   // execution order is resolved across ranks by the caller
        else if (nraw) {
            // positions in the list are 32-bit (dedup table, exec_idx): 2^32 entries are 160 GB of message CIDs, past device memory
            if (nraw >= 0xffffffffull) throw Error(IPCFP_ERR_UNSUPPORTED, "message list of 2^32 entries or more");
            ensure_scratch((nraw + 31) / 32);   // the general walk's list can outgrow the scratch sized for the store and the receipts
            uint64_t slots = 64;
            while (slots < 2 * nraw) slots <<= 1;
            AsyncBuf<unsigned long long> dtab(slots, st);
            dtab.zero();
            k_dedup_insert<<<div_up(nraw, 256), 256, 0, st>>>(exec_raw.p, nraw, dtab.p, slots - 1); IPCFP_LAUNCH_CHECK();
            k_dedup_flags<<<div_up((nraw + 31) / 32 * 32, 256), 256, 0, st>>>(exec_raw.p, nraw, dtab.p, slots - 1, keep_bits.p); IPCFP_LAUNCH_CHECK();
            AsyncBuf<uint64_t> wp2((nraw + 31) / 32 + 8, st);
            bitmap_to_indices(keep_bits.p, nraw, exec_idx.p, (uint64_t*)n_exec_dev, wp2.p, scratch.p, st);
        } else IPCFP_CUDA(cudaMemsetAsync(n_exec_dev, 0, 8, st));
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_EXEC_ORDER], st));
    }
};

// Requested message CIDs (n*38, host): up as RawCid through pinned memory and sorted once on the device (msg_sort_key), and what
// they select in an execution order (k_msg_select)
struct MsgRequests {
    uint64_t n = 0;
    PinnedArray h;
    AsyncBuf<RawCid> raw, sorted;
    AsyncBuf<uint32_t> pos;
    void stage(Store* s, const uint8_t* cids, uint64_t n_) {
        n = n_;
        if (!n) return;
        cudaStream_t st = s->stream;
        h = PinnedArray(s->pool, n * sizeof(RawCid));
        RawCid* hr = h.as<RawCid>();
        for (uint64_t j = 0; j < n; j++) hr[j] = rawcid_from_bytes(cids + 38 * j);
        raw.alloc(n, st); sorted.alloc(n, st); pos.alloc(n, st);
        IPCFP_CUDA(cudaMemcpyAsync(raw.p, hr, n * sizeof(RawCid), cudaMemcpyHostToDevice, st));
        sort_requests(raw.p, (uint32_t)n, sorted.p, pos.p, st);
    }
    // over the execution order exec_raw[exec_idx[i]], i < *n_exec ≤ n_max: the selected receipts below n_receipts → sel_bits, request
    // j's execution position → exec_indices[j] (left as it is when the message is not executed)
    void select(cudaStream_t st, const RawCid* exec_raw, const uint32_t* exec_idx, const unsigned long long* n_exec, uint64_t n_max, uint64_t n_receipts,
                uint64_t* exec_indices, uint32_t* sel_bits) const {
        if (!n || !n_max) return;
        k_msg_select<<<div_up(n_max, 256), 256, 0, st>>>(exec_raw, exec_idx, n_exec, sorted.p, pos.p, (uint32_t)n, n_receipts, exec_indices, sel_bits);
        IPCFP_LAUNCH_CHECK();
    }
};

// One generate_event_proof call: its arguments, the predicate's and the scan's state and buffers, and its phases, which
// generate_event_proof runs in order; the execution order is the ExecOrderBuild's.
// comm != nullptr: this call is one shard of a multi-GPU call and runs the cross-shard protocol itself (parallel.cu). Failures are then
// not thrown where they are seen: every rank keeps taking part in the collectives and all ranks fail together, with the error the
// reference's sequential order meets first across ALL shards.
// Host synchronisations, per mode:
//   unsharded         snapshot_and_sync after the walk (again after a dense walk that gave up; once more for k_amt_first_fault),
//                     pass1, pass2, read_back's witness join (IPCFP_RESULT_JSON: render_event_json's one before it), fill
//   IPCFP_BFS_GENERAL, sharded, order only (build_execution_order): walk reads the prologue back first; run_general synchronises after
//                     its range upload, after the fused rounds and once per level below them
//   order only:       walk, snapshot_and_sync, then build_execution_order reads n_exec back
//   sharded over NCCL: besides, every H0 / H2 gather, ShardExchange::agree_results and finish, a late H0 that fails, and fill's copy of
//                     the union partition (IPCFP_SHARDED_UNION_TO_HOST)
// P: the predicate. Matcher: `spec` is the call's EventProofSpec (t0 = keccak256(signature) is computed by k_setup). LogFilter: `filter`
// is a log filter (unsharded calls only), its values raw, its large sets uploaded beside it.
template <class P>
struct EventCall {
    Store* s;
    cudaStream_t st;
    TipsetDev& td;
    const ipcfp_event_spec* spec;
    const ipcfp_log_filter* filter = nullptr;
    uint32_t flags;
    bool sharded;
    uint64_t lo, hi;
    Comm* comm;
    std::chrono::steady_clock::time_point t_enter;
    uint64_t N = 0;
    std::unique_ptr<ShardExchange> xch;
    std::optional<ExecOrderBuild> ob;
    unsigned long long* dw;
    uint64_t* hw;
    // stage
    P mh;
    size_t siglen = 0;
    uint8_t* d_sig = nullptr;
    P* d_matcher = nullptr;
    AsyncBuf<uint64_t> d_sets;   // LogFilter: the large sets and their bitmaps, and their pinned host copy
    PinnedArray sets_h;
    // pass 1
    AsyncBuf<uint32_t> match_bits, cnt, nby;
    AsyncBuf<uint64_t> pbase, bbase;
    AsyncBuf<uint32_t> match_rel;
    AsyncBuf<uint64_t> wp3;
    uint64_t n_exec = 0, M = 0, pass1_nodes = 0, pass1_bytes = 0, n_proofs = 0, n_bytes = 0;
    // pass 2 and the result
    std::unique_ptr<EventResultBox> box;
    AsyncBuf<ipcfp_event_proof> d_proofs;
    AsyncBuf<uint8_t> d_blob;
    uint64_t mB = 0;
    bool any_skip = false;
    PinnedArray rel;
    uint64_t json_len = 0;
    // message selection (generate_message_log_proof): the requested CIDs, sorted once on the device, and what they select
    MsgRequests msg;
    PinnedArray exec_indices_h;
    AsyncBuf<uint32_t> sel_bits, sel;
    AsyncBuf<uint64_t> d_exec_indices, wp_sel;
    AsyncBuf<unsigned long long> n_sel;

    EventCall(Store* s_, TipsetDev& td_, const ipcfp_event_spec* spec_, uint32_t flags_, bool sharded_, uint64_t lo_, uint64_t hi_, Comm* comm_)
        : s(s_), st(s_->stream), td(td_), spec(spec_), flags(flags_), sharded(sharded_), lo(lo_), hi(hi_), comm(comm_), dw(s_->dev_words.p),
          hw(s_->host_words.p) {}

    // ---- checks, and the spec + tipset CIDs up in ONE copy from the store's pinned staging block (no host sync)
    void stage() {
        s->use();
        t_enter = std::chrono::steady_clock::now();
        LogFilterHost lfh;
        if constexpr (std::is_same_v<P, Matcher>) {
            event_matcher(spec, "event spec has null fields", mh);
            siglen = strlen(spec->event_signature);
        } else {
            log_filter_build(filter, lfh);
        }
        // a shard's result is not an EventProofBundle: its witness is distributed and its message CIDs are resolved later
        if (sharded && (flags & IPCFP_RESULT_JSON)) throw Error(IPCFP_ERR_UNSUPPORTED, "IPCFP_RESULT_JSON is not available for sharded calls");
        if ((flags & IPCFP_WITNESS_BY_REFERENCE) && !s->caller_blob)
            throw Error(IPCFP_ERR_UNSUPPORTED, "IPCFP_WITNESS_BY_REFERENCE needs a store made from a caller's blob (ipcfp_store_create)");
        if (!sharded) { lo = 0; hi = td.n_receipts; }
        if (lo > hi || hi > td.n_receipts) throw Error(IPCFP_ERR_INVALID_ARG, "receipt range out of bounds");
        N = hi - lo;
        if (comm) {
            if (!sharded) throw Error(IPCFP_ERR_INVALID_ARG, "communicator given for an unsharded call");
            if (s->class_prefix.size() > 1) throw Error(IPCFP_ERR_UNSUPPORTED, "sharded calls need a store with one CID prefix");
            xch.reset(new ShardExchange(comm, s, lo, hi));
        }
        ob.emplace(s, &td, td.n_parents, td.txmeta_cids.data(), flags, sharded, lo, hi, xch.get());

        //   [0,1024) Matcher (t0 is filled in on the device) or LogFilter | signature, zero padded | the tipset CIDs (ExecOrderBuild::stage)
        const size_t sig_cap = (siglen + 64) & ~(size_t)63;
        static_assert(sizeof(P) <= 1024, "the predicate must fit its staging slot");
        uint8_t* d_head = ob->stage(1024 + sig_cap, [&](uint8_t* hs) {
            if constexpr (!std::is_same_v<P, Matcher>) {   // the Matcher is event_matcher's, above
                memset(&mh, 0, sizeof mh);
                if (!lfh.dev.empty()) {   // through pinned memory that lives as long as the call: no host synchronisation
                    sets_h = PinnedArray(s->pool, lfh.dev.size() * 8);
                    memcpy(sets_h.p, lfh.dev.data(), lfh.dev.size() * 8);
                    d_sets.alloc(lfh.dev.size(), st);
                    IPCFP_CUDA(cudaMemcpyAsync(d_sets.p, sets_h.p, lfh.dev.size() * 8, cudaMemcpyHostToDevice, st));
                }
                lfh.place(d_sets.p);
                mh = lfh.f;
            }
            memcpy(hs, &mh, sizeof(P));
            if (siglen) memcpy(hs + 1024, spec->event_signature, siglen);
        });
        d_sig = d_head + 1024;                       // 8-byte aligned
        d_matcher = (P*)d_head;
    }

    // ---- the execution order. The Matcher's t0 is computed by k_setup: it comes from the prologue's head as the builder read it back.
    void exec_order() {
        if constexpr (std::is_same_v<P, Matcher>) {
            ob->build(d_sig, (uint32_t)siglen, d_matcher);
            memcpy(mh.t0, ob->ph->t0, 32);
        } else {
            ob->build(d_sig, (uint32_t)siglen, nullptr);   // a log filter's values arrive raw: nothing to hash
        }
    }

    // ---- pass 1: matching receipts, per-receipt proof counts and bytes
    void pass1() {
        match_bits.alloc((N + 31) / 32 + 8, st); cnt.alloc(N + 8, st); nby.alloc(N + 8, st);
        pbase.alloc(N + 8, st); bbase.alloc(N + 8, st);
        Pass1ArgsT<P> p1;
        p1.store = s->view; p1.store_dev = s->view_dev.p; p1.m_dev = d_matcher; p1.m = mh; p1.events_roots = td.events_roots.p; p1.has_root = td.has_root.p; p1.lo = lo; p1.hi = hi;
        p1.match_bits = match_bits.p; p1.cnt = cnt.p; p1.nbytes = nby.p; p1.err = dw + DW_ERR; p1.stats = dw + DW_STATS;
        if (N) {
            // 4 warps per CTA, 3 CTAs per SM; every lane has a ring of 4 chunks of 128 bytes, one chunk filled per pass (pass1_stage.cuh)
            const int smem = 4 * StageGeom<128, 4, 1>::WARP_BYTES;
            IPCFP_CUDA(cudaFuncSetAttribute(k_pass1_stage<P, 128, 4, 1, 4, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            k_pass1_stage<P, 128, 4, 1, 4, 3><<<div_up(N, 128), 128, smem, st>>>(p1); IPCFP_LAUNCH_CHECK();
        }
        finish_pass1();
    }
    // pass 1's tail: the matching list, the proof and byte offsets, and their counts on the host
    void finish_pass1() {
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_PASS1], st));
        match_rel.alloc(N + 32, st);
        wp3.alloc((N + 31) / 32 + 8, st);
        bitmap_to_indices(match_bits.p, (N + 31) / 32 * 32, match_rel.p, (uint64_t*)(dw + DW_N_MATCH), wp3.p, ob->scratch.p, st);
        exclusive_scan_u32(cnt.p, pbase.p, N, (uint64_t*)(dw + DW_N_PROOFS), ob->scratch.p, st);
        exclusive_scan_u32(nby.p, bbase.p, N, (uint64_t*)(dw + DW_BLOB_BYTES), ob->scratch.p, st);
        publish_words(s, 0, DW_TX_ERR + 1);
        IPCFP_CUDA(cudaStreamSynchronize(st));
        ob->note_errors();
        n_exec = hw[DW_N_EXEC];
        M = hw[DW_N_MATCH];
        pass1_nodes = hw[DW_STATS]; pass1_bytes = hw[DW_STATS + 1];
        n_proofs = hw[DW_N_PROOFS]; n_bytes = hw[DW_BLOB_BYTES];
    }

    // ---- message selection, in place of pass 1 (generate_message_log_proof). The requests go up as RawCid and are sorted on the
    // engine stream ahead of k_setup (msg.stage; the same stream: nothing overlaps); the selection needs the execution order, so it runs
    // behind the dedup.
    // k_msg_select over the execution order → the selected receipts (ascending) and every request's execution index; then the match of
    // the selected receipts only (k_msg_match: pass 1's per-receipt result) → match bits, counts and bytes of those receipts, zero
    // elsewhere; then pass 1's tail. No events AMT of an unselected receipt is read.
    void select_and_match() {
        const uint64_t n_msg = msg.n, nw = (N + 31) / 32 + 8, n_sel_max = std::min<uint64_t>(n_msg, N);
        d_exec_indices.alloc(n_msg + 1, st);
        IPCFP_CUDA(cudaMemsetAsync(d_exec_indices.p, 0xff, (n_msg + 1) * 8, st));
        sel_bits.alloc(nw, st); sel_bits.zero();
        match_bits.alloc(nw, st); match_bits.zero();
        cnt.alloc(N + 8, st); cnt.zero(); nby.alloc(N + 8, st); nby.zero();
        pbase.alloc(N + 8, st); bbase.alloc(N + 8, st);
        n_sel.alloc(1, st); n_sel.zero();
        msg.select(st, ob->exec_raw.p, ob->exec_idx.p, ob->n_exec_dev, ob->nraw, N, d_exec_indices.p, sel_bits.p);
        if (n_sel_max) {
            sel.alloc(n_sel_max + 32, st); wp_sel.alloc(nw, st);
            bitmap_to_indices(sel_bits.p, (N + 31) / 32 * 32, sel.p, (uint64_t*)n_sel.p, wp_sel.p, ob->scratch.p, st);
            MsgMatchArgsT<P> a;
            a.store = s->view; a.store_dev = s->view_dev.p; a.m_dev = d_matcher; a.events_roots = td.events_roots.p; a.has_root = td.has_root.p;
            a.sel = sel.p; a.n_sel = n_sel.p; a.n_sel_max = n_sel_max;
            a.match_bits = match_bits.p; a.cnt = cnt.p; a.nbytes = nby.p; a.err = dw + DW_ERR; a.stats = dw + DW_STATS;
            a.per_warp = n_sel_max <= 16384 ? 1 : 0;
            k_msg_match<<<div_up(a.per_warp ? n_sel_max * 32 : n_sel_max, 128), 128, 0, st>>>(a); IPCFP_LAUNCH_CHECK();
        }
        exec_indices_h = PinnedArray(s->pool, (n_msg + 1) * 8);
        if (n_msg) IPCFP_CUDA(cudaMemcpyAsync(exec_indices_h.p, d_exec_indices.p, n_msg * 8, cudaMemcpyDeviceToHost, st));
        finish_pass1();
    }

    // ---- pass 2: receipts-AMT paths, events walks, EventProofs; the late witness blocks
    void pass2() {
        box.reset(new EventResultBox());
        memset(&box->r, 0, sizeof box->r);
        d_proofs.alloc(n_proofs + 1, st);
        d_blob.alloc(n_bytes + 16, st);
        if (M) {
            Pass2ArgsT<P> p2;
            p2.store = s->view; p2.store_dev = s->view_dev.p; p2.m_dev = d_matcher; p2.m = mh; p2.events_roots = td.events_roots.p; p2.lo = lo; p2.match_rel = match_rel.p; p2.n_match = M;
            p2.receipts_root_blk = ob->receipts_root_blk; p2.exec_cids = ob->exec_raw.p; p2.exec_idx = ob->exec_idx.p; p2.n_exec = ob->n_exec_dev;
            p2.wbits = ob->wbits.p; p2.err = dw + DW_ERR; p2.cnt = cnt.p; p2.proof_base = pbase.p; p2.byte_base = bbase.p;
            p2.proofs = d_proofs.p; p2.blob = d_blob.p; p2.any_skip = ob->misc + 2; p2.resolve_msg = sharded ? 0 : 1;
            p2.per_warp = (M <= 16384 && !getenv("IPCFP_PASS2_PER_THREAD")) ? 1 : 0;
            k_pass2<<<div_up(p2.per_warp ? M * 32 : M, 128), 128, 0, st>>>(p2); IPCFP_LAUNCH_CHECK();
        }
        // pass 2 did not wait for the cross-shard exchange; now that both are done: P (parallel.cu)
        if (xch) xch->positions_for(match_rel.p, M, ob->n_exec_dev);
        // blocks recorded by pass 2 (receipt paths + events AMTs of the matches): the late part of the witness
        ob->wbuild->finish_enqueue(ob->wbits.p);
        publish_words(s, 0, DW_EXEC_CHECK + 1);
        publish_words(s, HW_ANY_SKIP, HW_ANY_SKIP_WORDS, ob->misc);
        IPCFP_CUDA(cudaStreamSynchronize(st));
        ob->note_errors();
        // base-witness CIDs (parent headers, child header, TxMeta) are only dereferenced by WitnessCollector::materialize
        // (common/witness.rs:43-56, events/generator.rs:104), i.e. AFTER every receipts-root / pass-1 / pass-2 failure
        if (!xch && ob->missing_base && !ob->skip_tx) throw_first(IPCFP_NO_ERROR, IPCFP_NO_ERROR, true);
        mB = hw[DW_WIT_B];
        any_skip = ((const uint32_t*)(hw + HW_ANY_SKIP))[2] != 0;
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_PASS2], st));
    }

    // ---- results to the host; the witness's late blocks, Cid order and index arrays (engine stream); the sharded tail beside it; JSON
    void read_back() {
        box->matching = PinnedArray(s->pool, (M + 1) * 8);
        box->proofs = PinnedArray(s->pool, (n_proofs + 1) * sizeof(ipcfp_event_proof));
        box->blob = PinnedArray(s->pool, n_bytes + 16);
        rel = PinnedArray(s->pool, (M + 1) * 4);
        if (M) IPCFP_CUDA(cudaMemcpyAsync(rel.p, match_rel.p, M * 4, cudaMemcpyDeviceToHost, st));
        if (n_proofs && !xch) IPCFP_CUDA(cudaMemcpyAsync(box->proofs.p, d_proofs.p, n_proofs * sizeof(ipcfp_event_proof), cudaMemcpyDeviceToHost, st));
        if (n_bytes) IPCFP_CUDA(cudaMemcpyAsync(box->blob.p, d_blob.p, n_bytes, cudaMemcpyDeviceToHost, st));
        WitnessBuilder& wbuild = *ob->wbuild;
        wbuild.finish_start(mB, hw[DW_WIT_B_BYTES], box->wit);
        if (xch) {
            if (!xch->agree_results(ob->pend_tx, ob->pend_err, ob->missing_base && !ob->skip_tx, n_proofs, hw[DW_WIT_A] + mB, ob->xch_stale, ob->exec_raw.p,
                                    ob->nraw)) {
                wbuild.finish_join(box->wit);   // nothing of this call may be in flight when its buffers go
                throw_first(xch->g_tx, xch->g_err, xch->g_missing_base);
                throw Error(IPCFP_ERR_UNSUPPORTED, "execution-order exchange: bucket overflow (skewed CID hash distribution)");
            }
            xch->fetch_and_patch(d_proofs.p, n_proofs, box->proofs.p);
            xch->witness_union(box->wit.cids_dev.p, box->wit.n, (flags & IPCFP_SHARDED_UNION_FULL) != 0);
        }
        // IPCFP_RESULT_JSON: render the bundle from the device copies (json.cu) while the witness blob copy, if any, is still on the wire
        if (flags & IPCFP_RESULT_JSON) {
            IPCFP_CUDA(cudaEventRecord(s->ev[EV_JSON_BEGIN], st));
            JsonInputs ji{d_proofs.p, n_proofs, d_blob.p, box->wit.cids_dev.p, box->wit.idx_dev.p, box->wit.n,
                          td.parent_epoch, td.child_epoch, td.n_parents, ob->sa.parent_cids, ob->sa.child_cid};
            json_len = render_event_json(s, ji, box->json);
            IPCFP_CUDA(cudaEventRecord(s->ev[EV_JSON_END], st));
        }
        wbuild.finish_join(box->wit);
        if (xch) xch->finish();
    }

    // ---- the result
    ipcfp_event_result* fill() {
        static thread_local std::chrono::steady_clock::time_point t_last_exit = t_enter;
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_END], st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
        {
            uint64_t* mo = box->matching.as<uint64_t>();
            const uint32_t* rp = rel.as<uint32_t>();
            for (uint64_t k = 0; k < M; k++) mo[k] = lo + rp[k];
        }
        if (any_skip) {  // receipts the AMT does not hold (`continue` at :249-251): compact their reserved slots away
            ipcfp_event_proof* pp = box->proofs.as<ipcfp_event_proof>();
            uint64_t w = 0;
            for (uint64_t k = 0; k < n_proofs; k++) if (pp[k].exec_index != UINT64_MAX) pp[w++] = pp[k];
            n_proofs = w;
        }
        ipcfp_event_result& r = box->r;
        r.n_matching = M; r.matching_indices = box->matching.as<uint64_t>();
        r.n_proofs = n_proofs; r.proofs = box->proofs.as<ipcfp_event_proof>();
        r.data_blob = box->blob.as<uint8_t>(); r.data_blob_size = n_bytes;
        box->wit.fill(r.witness);
        r.n_exec = n_exec;
        float ms;
        IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_BEGIN], s->ev[EV_END])); r.ms_total = ms;
        IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_SETUP], s->ev[EV_EXEC_ORDER])); r.ms_txamt = ms;
        IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_EXEC_ORDER], s->ev[EV_PASS1])); r.ms_pass1 = ms;
        IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_PASS1], s->ev[EV_PASS2])); r.ms_pass2 = ms;
        IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_PASS2], s->ev[EV_END])); r.ms_witness = ms;
        r.pass1_bytes = pass1_bytes; r.pass1_nodes = pass1_nodes;
        if (flags & IPCFP_RESULT_JSON) {
            r.json = box->json.as<char>(); r.json_len = json_len;
            IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_JSON_BEGIN], s->ev[EV_JSON_END])); r.ms_json = ms;
        }
        r.shard_raw_total = ob->nraw_total;
        if (sharded) { r.n_exec = 0; r.shard_exec_count = ob->nraw; box->shard_exec = std::move(ob->exec_raw); r.shard_exec_dev = box->shard_exec.p; }
        if (xch) {
            xch->fill_result(r);
            if (getenv("IPCFP_XCH_TRACE")) {
                float t[6]; char buf[384];
                // walk+snapshot done, pass 1 done, pass 2 done, sorted CID list, 51 MB copy done, end
                const int evs[6] = {EV_EXEC_ORDER, EV_PASS1, EV_PASS2, EV_WITNESS_SORTED, EV_BLOB_COPIED, EV_END};
                for (int i = 0; i < 6; i++) cudaEventElapsedTime(&t[i], s->ev[EV_BEGIN], s->ev[evs[i]]);
                const auto t_now = std::chrono::steady_clock::now();
                const double host_call = std::chrono::duration<double, std::milli>(t_now - t_enter).count();
                const double host_gap = std::chrono::duration<double, std::milli>(t_enter - t_last_exit).count();
                snprintf(buf, sizeof buf, "host: gap since last call %.3f, in call %.3f | walk %.3f pass1 %.3f pass2 %.3f sorted %.3f blobD2H %.3f end %.3f", host_gap, host_call,
                         t[0], t[1], t[2], t[3], t[4], t[5]);
                t_last_exit = std::chrono::steady_clock::now();
                xch->trace_timeline(s->ev[EV_BEGIN], buf);
            }
            if (flags & IPCFP_SHARDED_UNION_TO_HOST) {
                box->union_host = PinnedArray(s->pool, r.n_union_part * 38 + 64);
                if (r.n_union_part) IPCFP_CUDA(cudaMemcpyAsync(box->union_host.p, r.union_cids_dev, r.n_union_part * 38, cudaMemcpyDeviceToHost, st));
                IPCFP_CUDA(cudaStreamSynchronize(st));
                r.union_cids = box->union_host.as<uint8_t>();
            }
        }
        return &box.release()->r;
    }
};
}  // namespace

ipcfp_event_result* generate_event_proof(Store* s, TipsetDev& td, const ipcfp_event_spec* spec, uint32_t flags, bool sharded, uint64_t lo, uint64_t hi,
                                         Comm* comm) {
    EventCall<Matcher> c(s, td, spec, flags, sharded, lo, hi, comm);
    c.stage();
    c.exec_order();
    c.pass1();
    c.pass2();
    c.read_back();
    return c.fill();
}

// the same call with a log filter as the predicate (unsharded)
ipcfp_event_result* generate_log_proof(Store* s, TipsetDev& td, const ipcfp_log_filter* filter, uint32_t flags) {
    EventCall<LogFilter> c(s, td, nullptr, flags, false, 0, 0, nullptr);
    c.filter = filter;
    c.stage();
    c.exec_order();
    c.pass1();
    c.pass2();
    c.read_back();
    return c.fill();
}

void event_matcher(const ipcfp_event_spec* spec, const char* refusal, Matcher& m) {
    if (!spec || !spec->event_signature || !spec->topic_1) throw Error(IPCFP_ERR_INVALID_ARG, refusal);
    memset(&m, 0, sizeof m);
    const size_t n1 = strlen(spec->topic_1);
    memcpy(m.t1, spec->topic_1, n1 < 32 ? n1 : 32);   // ascii_to_bytes32 (evm.rs:72-78)
    m.actor = spec->actor_id_filter;
    m.has_actor = spec->has_actor_id_filter ? 1 : 0;
}

void message_request_check(const uint8_t* message_cids, uint64_t n, const ipcfp_log_filter* filter, bool with_exec, const uint64_t* exec_indices) {
    if (with_exec) {
        if (n && (!message_cids || !exec_indices)) throw Error(IPCFP_ERR_INVALID_ARG, "null message CIDs or exec indices with a nonzero count");
    } else if (n && !message_cids) {
        throw Error(IPCFP_ERR_INVALID_ARG, "null message CIDs with a nonzero count");
    }
    if (n > IPCFP_MESSAGE_MAX) throw Error(IPCFP_ERR_INVALID_ARG, "more message CIDs than IPCFP_MESSAGE_MAX");
    if (filter) log_filter_check(filter);
}

// the same call with its receipt loop restricted to the receipts of the given messages (filter null: every log extract_evm_log accepts)
ipcfp_event_result* generate_message_log_proof(Store* s, TipsetDev& td, const uint8_t* message_cids, uint64_t n, const ipcfp_log_filter* filter,
                                               uint32_t flags, uint64_t* exec_indices) {
    message_request_check(message_cids, n, filter, true, exec_indices);
    ipcfp_log_filter any;
    memset(&any, 0, sizeof any);
    EventCall<LogFilter> c(s, td, nullptr, flags, false, 0, 0, nullptr);
    c.filter = filter ? filter : &any;
    c.stage();
    c.msg.stage(s, message_cids, n);
    c.exec_order();
    c.select_and_match();
    c.pass2();
    c.read_back();
    ipcfp_event_result* r = c.fill();
    if (n) memcpy(exec_indices, c.exec_indices_h.p, n * 8);
    return r;
}

void build_execution_order(Store* s, uint32_t n_parents, const uint8_t* txmeta_cids, ExecOrderOut& out) {
    s->use();
    ExecOrderBuild b(s, n_parents, txmeta_cids);
    b.stage(0, [](uint8_t*) {});
    b.build(nullptr, 0, nullptr);
    publish_words(s, DW_N_EXEC, 1);
    IPCFP_CUDA(cudaStreamSynchronize(b.st));
    out.n_exec = b.hw[DW_N_EXEC];
    out.exec_raw = std::move(b.exec_raw);
    out.exec_idx = std::move(b.exec_idx);
}

void message_positions(Store* s, TipsetDev& td, const uint8_t* message_cids, uint64_t n, uint32_t flags, MessagePositions& out) {
    ExecOrderBuild ob(s, &td, td.n_parents, td.txmeta_cids.data(), flags & IPCFP_WITNESS_BY_REFERENCE);
    ob.early_copy = false;
    ob.stage(0, [](uint8_t*) {});
    MsgRequests msg;
    msg.stage(s, message_cids, n);   // read by the walk's synchronisation
    ob.build(nullptr, 0, nullptr);
    cudaStream_t st = s->stream;
    out.exec_indices.alloc(n + 1, st);
    IPCFP_CUDA(cudaMemsetAsync(out.exec_indices.p, 0xff, (n + 1) * 8, st));
    // every executed position is selectable (no receipt count bounds it); the bitmap k_msg_select fills is not read
    AsyncBuf<uint32_t> sel_bits((ob.nraw + 31) / 32 + 8, st);
    msg.select(st, ob.exec_raw.p, ob.exec_idx.p, ob.n_exec_dev, ob.nraw, UINT64_MAX, out.exec_indices.p, sel_bits.p);
    publish_words(s, DW_N_EXEC, 1);
    out.wbits = std::move(ob.wbits);
    out.receipts_root_blk = ob.receipts_root_blk;
    out.missing_base = ob.missing_base;
}

void message_exec_indices(Store* s, const ExecOrderOut& exo, const uint8_t* message_cids, uint64_t n, uint64_t* exec_indices) {
    cudaStream_t st = s->stream;
    IPCFP_CUDA(cudaMemsetAsync(exec_indices, 0xff, n * 8, st));
    if (!n || !exo.n_exec) return;
    MsgRequests req;
    req.stage(s, message_cids, n);
    AsyncBuf<unsigned long long> n_exec(1, st);
    AsyncBuf<uint32_t> sel_bits((exo.n_exec + 31) / 32 + 8, st);   // k_msg_select's bitmap, not read
    const unsigned long long ne = exo.n_exec;
    IPCFP_CUDA(cudaMemcpyAsync(n_exec.p, &ne, 8, cudaMemcpyHostToDevice, st));
    req.select(st, exo.exec_raw.p, exo.exec_idx.p, n_exec.p, exo.n_exec, UINT64_MAX, exec_indices, sel_bits.p);
    IPCFP_CUDA(cudaStreamSynchronize(st));   // the host copies above are read until here
}

__global__ void k_msg_mask(const uint8_t* __restrict__ has_root, const uint32_t* __restrict__ sel_bits, uint64_t n, uint8_t* has_sel) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) has_sel[i] = has_root[i] && ((sel_bits[i >> 5] >> (i & 31)) & 1u) ? 1 : 0;
}
void message_selection_mask(Store* s, TipsetDev& td, const ExecOrderOut& exo, const uint8_t* message_cids, uint64_t n, uint8_t* has_sel) {
    cudaStream_t st = s->stream;
    const uint64_t N = td.n_receipts;
    AsyncBuf<uint32_t> bits((N + 31) / 32 + 8, st);
    bits.zero();
    if (n && exo.n_exec) {
        MsgRequests req;
        req.stage(s, message_cids, n);
        AsyncBuf<uint64_t> idx(n, st);
        AsyncBuf<unsigned long long> n_exec(1, st);
        const unsigned long long ne = exo.n_exec;
        IPCFP_CUDA(cudaMemcpyAsync(n_exec.p, &ne, 8, cudaMemcpyHostToDevice, st));
        req.select(st, exo.exec_raw.p, exo.exec_idx.p, n_exec.p, exo.n_exec, N, idx.p, bits.p);
        if (N) { k_msg_mask<<<div_up(N, 256), 256, 0, st>>>(td.has_root.p, bits.p, N, has_sel); IPCFP_LAUNCH_CHECK(); }
        IPCFP_CUDA(cudaStreamSynchronize(st));   // the host copies above are read until here
    }
}

void event_result_free(ipcfp_event_result* r) { delete reinterpret_cast<EventResultBox*>(r); }
const WitnessOut& event_result_witness(const ipcfp_event_result* r) { return reinterpret_cast<const EventResultBox*>(r)->wit; }

}  // namespace ipcfp
