// plan.cu — ipcfp_plan_fetch_resident: one round of fetch planning for a proof bundle (DESIGN.md §2, "Fetch planning").
//
// N(S) is every block the generators of ipcfp_generate_proof_bundle_resident would `get`, as far as decoding the blocks already in the
// store S finds them; the call returns N(S) \ S in `Cid` order. Per-item code: plan_items.cuh.
//   k_plan_seed_events   level 0: one events-AMT root item per receipt with an events root (the base roots come from the host)
//   k_plan_count         one item per thread: lookup; missing → appended; present → marked needed, expanded once per class (rank
//   k_plan_expand          bitmaps), its children counted, then written behind one atomic cursor. One host sync per level.
//   k_plan_matchers      keccak256(event_signature) of every spec (the Matchers' t0)
//   k_plan_match         rule 3, once no events-AMT block of N(S) is missing: per receipt, pass 1's match, then its receipts-AMT path
//   k_plan_storage       rule 4: per storage spec, generate_storage_proof's path up to the first block the store lacks
//   k_plan_popc          |N(S) ∩ S| from the needed bitmap
// then the missing list is sorted and made unique on the device (sort_unique_cids) and copied back once.
#include <algorithm>
#include <cstring>

#include "engine.cuh"
#include "hashes.cuh"
#include "plan_items.cuh"
#include "prims.cuh"

namespace ipcfp {

enum PlanCounter : uint32_t { PC_CHILDREN = 0, PC_FILL = 1, PC_MISSING = 2, PC_EV_MISSING = 3, PC_NEEDED = 4, PC_COUNT = 8 };

__device__ __forceinline__ void plan_miss(uint8_t* miss, unsigned long long* ctr, const uint8_t* cid) {
    const unsigned long long k = atomicAdd(ctr + PC_MISSING, 1ull);
    for (int b = 0; b < 38; b++) miss[38 * k + b] = cid[b];
}

__global__ void k_plan_seed_events(const uint8_t* __restrict__ roots, const uint8_t* __restrict__ has, uint64_t n, PlanItem* out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = has[i] ? PlanItem{roots + 38 * i, PK_EV_ROOT, 1u << 8} : PlanItem{nullptr, PK_NONE, 0};
}

__global__ void __launch_bounds__(128) k_plan_count(StoreView s, const PlanItem* __restrict__ items, uint64_t n, uint32_t* cnt, uint32_t* blk,
                                                    uint32_t* needed, uint32_t* visited, uint64_t nwords, uint8_t* miss, unsigned long long* ctr) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    cnt[t] = 0;
    const PlanItem it = items[t];
    if (it.kind == PK_NONE) return;
    const int32_t b = store_lookup(s, it.cid);
    if (b < 0) {
        plan_miss(miss, ctr, it.cid);
        if (it.bw_tree >> 8) atomicAdd(ctr + PC_EV_MISSING, 1ull);
        return;
    }
    witness_mark(s, needed, (uint32_t)b);
    if (it.kind == PK_BLOCK) return;
    const uint32_t r = s.rank_of ? s.rank_of[b] : (uint32_t)b, m = 1u << (r & 31);
    if (atomicOr(visited + plan_class(it) * nwords + (r >> 5), m) & m) return;
    uint32_t len;
    const uint8_t* p = store_block(s, (uint32_t)b, len);
    const uint32_t c = plan_children(p, len, it, nullptr);
    cnt[t] = c;
    blk[t] = (uint32_t)b;
    if (c) atomicAdd(ctr + PC_CHILDREN, (unsigned long long)c);
}

__global__ void __launch_bounds__(128) k_plan_expand(StoreView s, const PlanItem* __restrict__ items, uint64_t n, const uint32_t* __restrict__ cnt,
                                                     const uint32_t* __restrict__ blk, PlanItem* out, unsigned long long* ctr) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n || !cnt[t]) return;
    const unsigned long long base = atomicAdd(ctr + PC_FILL, (unsigned long long)cnt[t]);
    uint32_t len;
    const uint8_t* p = store_block(s, blk[t], len);
    (void)plan_children(p, len, items[t], out + base);
}

// EventMatcher::new (events/generator.rs:30-35): sig + sig_off[k] holds spec k's signature, zero padded
__global__ void k_plan_matchers(const uint8_t* sig, const uint64_t* sig_off, const uint32_t* sig_len, uint64_t n, Matcher* m) {
    for (uint64_t k = threadIdx.x; k < n; k += blockDim.x) {
        Digest d;
        keccak256(sig + sig_off[k], sig_len[k], d);
        for (int w = 0; w < 4; w++) m[k].t0[w] = d.w[w];
    }
}

template <class P>
__global__ void __launch_bounds__(128) k_plan_match(StoreView s, const StoreView* s_dev, const uint8_t* __restrict__ roots, const uint8_t* __restrict__ has,
                                                    uint64_t n, const P* m, uint64_t n_specs, const uint8_t* receipts_root, uint32_t* needed,
                                                    uint8_t* miss, unsigned long long* ctr) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !has[i]) return;
    const int32_t rb = store_lookup(s, roots + 38 * i);
    if (rb < 0 || !plan_receipt_matches(s_dev, (uint32_t)rb, m, n_specs)) return;
    const uint8_t* c = plan_receipt_path(s, receipts_root, i, needed);
    if (c) plan_miss(miss, ctr, c);
}

__global__ void __launch_bounds__(128) k_plan_storage(StorageArgs a, uint32_t* needed, uint8_t* miss, unsigned long long* ctr) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n) return;
    const uint8_t* c = plan_storage_path(a, t, needed);
    if (c) plan_miss(miss, ctr, c);
}

__global__ void __launch_bounds__(128) k_plan_actors(ActorArgs a, uint32_t* needed, uint8_t* miss, unsigned long long* ctr) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n) return;
    const uint8_t* c = plan_actor_path(a, t, needed);
    if (c) plan_miss(miss, ctr, c);
}

__global__ void __launch_bounds__(128) k_plan_messages(MsgProofArgs a, const uint8_t* receipts_root, uint32_t* needed, uint8_t* miss,
                                                       unsigned long long* ctr) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n) return;
    const uint8_t* m[2];
    const uint32_t k = plan_message_path(a, receipts_root, t, needed, m);
    for (uint32_t i = 0; i < k; i++) plan_miss(miss, ctr, m[i]);
}

__global__ void k_plan_popc(const uint32_t* __restrict__ bits, uint64_t nwords, unsigned long long* out) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t c = w < nwords ? (uint32_t)__popc(bits[w]) : 0u;
    const uint32_t sum = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && sum) atomicAdd(out, (unsigned long long)sum);
}

void plan_fetch(Store* s, TipsetDev& td, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs, const ipcfp_event_spec* especs, uint64_t n_especs,
                FetchPlan& out, const ipcfp_log_filter* log_filters, uint64_t n_log_filters, const uint8_t* has_dev) {
    if ((n_sspecs && !sspecs) || (n_especs && !especs)) throw Error(IPCFP_ERR_INVALID_ARG, "null specs");
    LogFilterSet fs;
    fs.build(log_filters, n_log_filters);
    const bool events = n_especs || n_log_filters;   // the event path's rules (1–3) apply
    if (n_sspecs && !td.has_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    std::vector<Matcher> mh(n_especs);
    for (uint64_t k = 0; k < n_especs; k++) event_matcher(&especs[k], "event spec has null fields", mh[k]);
    s->use();
    cudaStream_t st = s->stream;
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_BEGIN], st));
    const StoreView& v = s->view;
    const uint64_t nwords = (s->n + 31) / 32 + 1;
    const uint64_t n_rcpt = events ? td.n_receipts : 0;
    const uint8_t* has = has_dev ? has_dev : td.has_root.p;

    // the base roots (collect_base_witness, events/generator.rs:112-145; generate_storage_proof's child header and StateRoot), then every
    // spec's inputs, in one upload
    std::vector<uint8_t> roots;
    std::vector<uint32_t> kinds;
    auto root = [&](const uint8_t* c, uint32_t kind) { roots.insert(roots.end(), c, c + 38); kinds.push_back(kind); };
    if (events) {
        for (uint32_t k = 0; k < td.n_parents; k++) root(td.parent_cids.data() + 38 * k, PK_BLOCK);
        root(td.child_cid, PK_BLOCK);
        root(td.receipts_root, PK_BLOCK);
        for (uint32_t k = 0; k < td.n_parents; k++) root(td.txmeta_cids.data() + 38 * k, PK_TXMETA);
    }
    if (n_sspecs) { root(td.child_cid, PK_BLOCK); root(td.child_state_root, PK_BLOCK); }
    const uint64_t nh = kinds.size();
    std::vector<uint64_t> sig_off(n_especs);
    std::vector<uint32_t> sig_len(n_especs);
    std::vector<uint8_t> sigs;
    for (uint64_t k = 0; k < n_especs; k++) {
        sig_off[k] = sigs.size();
        sig_len[k] = (uint32_t)strlen(especs[k].event_signature);
        sigs.insert(sigs.end(), especs[k].event_signature, especs[k].event_signature + sig_len[k]);
        sigs.resize((sigs.size() + 64) & ~(size_t)63, 0);
    }
    auto up16 = [](uint64_t x) { return (x + 15) & ~15ull; };
    const uint64_t o_roots = 0, o_m = up16(roots.size() + 16), o_so = o_m + up16(n_especs * sizeof(Matcher)), o_sl = o_so + 8 * n_especs,
                   o_sig = up16(o_sl + 4 * n_especs), o_ss = o_sig + up16(sigs.size() + 16), size = o_ss + n_sspecs * sizeof(ipcfp_storage_spec) + 16;
    std::vector<uint8_t> h(size, 0);
    if (!roots.empty()) memcpy(h.data() + o_roots, roots.data(), roots.size());
    if (n_especs) {
        memcpy(h.data() + o_m, mh.data(), n_especs * sizeof(Matcher));
        memcpy(h.data() + o_so, sig_off.data(), 8 * n_especs);
        memcpy(h.data() + o_sl, sig_len.data(), 4 * n_especs);
        memcpy(h.data() + o_sig, sigs.data(), sigs.size());
    }
    if (n_sspecs) memcpy(h.data() + o_ss, sspecs, n_sspecs * sizeof(ipcfp_storage_spec));
    AsyncBuf<uint8_t> d(size, st);
    IPCFP_CUDA(cudaMemcpyAsync(d.p, h.data(), size, cudaMemcpyHostToDevice, st));
    // the log filters and their large sets, in one upload (fs.words outlives the copy: the stream is synchronised before return)
    AsyncBuf<uint64_t> d_lf;
    if (n_log_filters) {
        d_lf.alloc(fs.words.size(), st);
        fs.place(d_lf.p);
        IPCFP_CUDA(cudaMemcpyAsync(d_lf.p, fs.words.data(), fs.words.size() * 8, cudaMemcpyHostToDevice, st));
    }

    AsyncBuf<uint32_t> needed(nwords, st), visited(PLAN_CLASSES * nwords, st);
    needed.zero();
    visited.zero();
    AsyncBuf<unsigned long long> ctr(PC_COUNT, st);
    ctr.zero();
    PinnedArray hc(s->pool, PC_COUNT * 8);
    unsigned long long* hctr = hc.as<unsigned long long>();
    auto read_counters = [&] {
        IPCFP_CUDA(cudaMemcpyAsync(hctr, ctr.p, PC_COUNT * 8, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
    };
    // the missing CIDs: every item, matching receipt and storage spec adds at most one
    AsyncBuf<uint8_t> miss;
    uint64_t n_miss = 0, miss_cap = 0;
    auto ensure_miss = [&](uint64_t extra) {
        if (n_miss + extra <= miss_cap) return;
        const uint64_t cap = std::max(2 * miss_cap, n_miss + extra) + 64;
        AsyncBuf<uint8_t> m2(38 * cap + 16, st);
        if (n_miss) IPCFP_CUDA(cudaMemcpyAsync(m2.p, miss.p, 38 * n_miss, cudaMemcpyDeviceToDevice, st));
        miss = std::move(m2);
        miss_cap = cap;
    };

    // ---- rules 1 and 2 and the base roots: level by level
    uint64_t n = nh + n_rcpt;
    AsyncBuf<PlanItem> cur(std::max<uint64_t>(n, 1), st), nxt;
    AsyncBuf<uint32_t> cnt, blk;
    if (nh) {
        std::vector<PlanItem> seeds(nh);
        for (uint64_t k = 0; k < nh; k++) seeds[k] = PlanItem{d.p + o_roots + 38 * k, kinds[k], kinds[k] == PK_TXMETA ? 3u : 0u};
        IPCFP_CUDA(cudaMemcpyAsync(cur.p, seeds.data(), nh * sizeof(PlanItem), cudaMemcpyHostToDevice, st));
    }
    if (n_rcpt) { k_plan_seed_events<<<div_up(n_rcpt, 256), 256, 0, st>>>(td.events_roots.p, has, n_rcpt, cur.p + nh); IPCFP_LAUNCH_CHECK(); }
    uint32_t levels = 0;
    while (n) {
        ensure_miss(n);
        if (cnt.n < n) { cnt.alloc(n, st); blk.alloc(n, st); }
        IPCFP_CUDA(cudaMemsetAsync(ctr.p + PC_CHILDREN, 0, 16, st));
        k_plan_count<<<div_up(n, 128), 128, 0, st>>>(v, cur.p, n, cnt.p, blk.p, needed.p, visited.p, nwords, miss.p, ctr.p); IPCFP_LAUNCH_CHECK();
        read_counters();
        levels++;
        n_miss = hctr[PC_MISSING];
        const uint64_t total = hctr[PC_CHILDREN];
        if (!total) break;
        nxt.alloc(total, st);
        k_plan_expand<<<div_up(n, 128), 128, 0, st>>>(v, cur.p, n, cnt.p, blk.p, nxt.p, ctr.p); IPCFP_LAUNCH_CHECK();
        std::swap(cur, nxt);
        n = total;
    }
    const bool events_complete = hctr[PC_EV_MISSING] == 0;
    ensure_miss(n_rcpt + n_sspecs);

    // ---- rule 3: the receipts-AMT paths of the matching receipts, once every events-AMT block of N(S) is in the store
    if (n_rcpt && events_complete) {
        const uint8_t* rr = d.p + o_roots + 38ull * (td.n_parents + 1);
        if (n_log_filters) {
            k_plan_match<<<div_up(n_rcpt, 128), 128, 0, st>>>(v, s->view_dev.p, td.events_roots.p, has, n_rcpt, (const LogFilter*)d_lf.p,
                                                              n_log_filters, rr, needed.p, miss.p, ctr.p);
        } else {
            k_plan_matchers<<<1, 32, 0, st>>>(d.p + o_sig, (const uint64_t*)(d.p + o_so), (const uint32_t*)(d.p + o_sl), n_especs, (Matcher*)(d.p + o_m));
            IPCFP_LAUNCH_CHECK();
            k_plan_match<<<div_up(n_rcpt, 128), 128, 0, st>>>(v, s->view_dev.p, td.events_roots.p, has, n_rcpt, (const Matcher*)(d.p + o_m),
                                                              n_especs, rr, needed.p, miss.p, ctr.p);
        }
        IPCFP_LAUNCH_CHECK();
    }
    // ---- rule 4: the storage paths
    if (n_sspecs) {
        StorageArgs a{};
        a.store = v;
        a.child_cid = d.p + o_roots + 38 * (nh - 2);
        a.state_root_json = d.p + o_roots + 38 * (nh - 1);
        a.specs = (const ipcfp_storage_spec*)(d.p + o_ss);
        a.n = n_sspecs;
        k_plan_storage<<<div_up(n_sspecs, 128), 128, 0, st>>>(a, needed.p, miss.p, ctr.p); IPCFP_LAUNCH_CHECK();
    }
    k_plan_popc<<<div_up(nwords, 256), 256, 0, st>>>(needed.p, nwords, ctr.p + PC_NEEDED); IPCFP_LAUNCH_CHECK();
    read_counters();
    n_miss = hctr[PC_MISSING];
    out.n_needed = hctr[PC_NEEDED];
    out.n_levels = levels;

    // ---- M(S): sorted, unique, one copy back
    uint64_t m = 0, mixed = UINT64_MAX;
    if (n_miss) {
        AsyncBuf<uint8_t> sorted(38 * n_miss + 16, st);
        m = sort_unique_cids(st, miss.p, n_miss, sorted.p, &mixed);
        out.cids.resize(38 * m);
        IPCFP_CUDA(cudaMemcpyAsync(out.cids.data(), sorted.p, 38 * m, cudaMemcpyDeviceToHost, st));
    }
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_END], st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    IPCFP_CUDA(cudaEventElapsedTime(&out.ms_total, s->ev[EV_BEGIN], s->ev[EV_END]));
    // The device order is the bytes' order, which is `Cid` order within one prefix. A CID of another prefix (one that no block of the
    // store has, so rarely more than a few) puts the list in `Cid` order on the host.
    if (mixed != UINT64_MAX) sort_cids_host(out.cids);
}

// The message call's round (include/ipcfp.h): the execution order first (the engine's own walk and dedup). While it cannot be built — a
// TxMeta or message-AMT block is missing, or one does not decode, which the generator then reports — no receipt is taken, and the round
// is the base roots, the TxMeta blocks and the message AMTs. Once it is built, the receipts rules 1 and 3 take are the selected ones.
void plan_fetch_messages(Store* s, TipsetDev& td, const uint8_t* message_cids, uint64_t n, const ipcfp_log_filter* filter, FetchPlan& out) {
    message_request_check(message_cids, n, filter, false, nullptr);
    ipcfp_log_filter any;
    memset(&any, 0, sizeof any);
    s->use();
    AsyncBuf<uint8_t> has(td.n_receipts + 64, s->stream);
    has.zero();
    ExecOrderOut exo;
    bool have_order = true;
    try {
        build_execution_order(s, td.n_parents, td.txmeta_cids.data(), exo);
    } catch (Error& e) {
        // a block the walk lacks, or one that does not decode (the generator reports it): no receipt is taken this round. Anything
        // else (device, allocation, unsupported input) is the planner's own failure.
        if (e.status != IPCFP_ERR_MISSING_BLOCK && e.status != IPCFP_ERR_DECODE) throw;
        have_order = false;
    }
    if (have_order) message_selection_mask(s, td, exo, message_cids, n, has.p);
    plan_fetch(s, td, nullptr, 0, nullptr, 0, out, filter ? filter : &any, 1, has.p);
}

// ipcfp_plan_fetch_actor_proofs_resident: each request's walks up to the first block the store lacks (plan_actor_path), one thread each
void plan_fetch_actor_proofs(Store* s, TipsetDev& td, const ipcfp_address* addrs, uint64_t n, const uint8_t* evm, uint64_t n_evm, uint32_t flags,
                             FetchPlan& out) {
    actor_request_check(addrs, n, evm, n_evm, flags);
    if (!td.has_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    s->use();
    cudaStream_t st = s->stream;
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_BEGIN], st));
    const uint64_t nwords = (s->n + 31) / 32 + 1;
    ActorUpload up(s, td.child_cid, td.child_state_root, addrs, n, evm, n_evm);
    ActorArgs a{};
    up.fill(a, s->view, n, n_evm, flags);
    AsyncBuf<uint32_t> needed(nwords, st);
    needed.zero();
    AsyncBuf<unsigned long long> ctr(PC_COUNT, st);
    ctr.zero();
    AsyncBuf<uint8_t> miss(38 * n + 16, st);
    if (n) { k_plan_actors<<<div_up(n, 128), 128, 0, st>>>(a, needed.p, miss.p, ctr.p); IPCFP_LAUNCH_CHECK(); }
    k_plan_popc<<<div_up(nwords, 256), 256, 0, st>>>(needed.p, nwords, ctr.p + PC_NEEDED); IPCFP_LAUNCH_CHECK();
    PinnedArray hc(s->pool, PC_COUNT * 8);
    IPCFP_CUDA(cudaMemcpyAsync(hc.p, ctr.p, PC_COUNT * 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    const uint64_t n_miss = hc.as<unsigned long long>()[PC_MISSING];
    out.n_needed = hc.as<unsigned long long>()[PC_NEEDED];
    out.n_levels = 0;
    uint64_t m = 0, mixed = UINT64_MAX;
    if (n_miss) {
        AsyncBuf<uint8_t> sorted(38 * n_miss + 16, st);
        m = sort_unique_cids(st, miss.p, n_miss, sorted.p, &mixed);
        out.cids.resize(38 * m);
        IPCFP_CUDA(cudaMemcpyAsync(out.cids.data(), sorted.p, 38 * m, cudaMemcpyDeviceToHost, st));
    }
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_END], st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    IPCFP_CUDA(cudaEventElapsedTime(&out.ms_total, s->ev[EV_BEGIN], s->ev[EV_END]));
    if (mixed != UINT64_MAX) sort_cids_host(out.cids);
}

// ipcfp_plan_fetch_message_proofs_resident: the base (headers, receipts root, TxMetas, message AMTs: the message-log planner's rules with no
// receipt taken); once the execution order can be built, each executed request's receipts-AMT path up to the first block the store lacks
// and, with the body, its message block. No events AMT is planned.
void plan_fetch_message_proofs(Store* s, TipsetDev& td, const uint8_t* cids, uint64_t n, uint32_t flags, FetchPlan& out) {
    message_proof_check(cids, n, flags);
    s->use();
    cudaStream_t st = s->stream;
    Event ev[2];
    IPCFP_CUDA(cudaEventRecord(ev[0], st));
    {
        ipcfp_log_filter any;
        memset(&any, 0, sizeof any);
        AsyncBuf<uint8_t> none(td.n_receipts + 64, st);
        none.zero();
        plan_fetch(s, td, nullptr, 0, nullptr, 0, out, &any, 1, none.p);
    }
    auto finish = [&] {
        IPCFP_CUDA(cudaEventRecord(ev[1], st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
        out.ms_total = elapsed_ms(ev[0], ev[1]);
    };
    ExecOrderOut exo;
    try {
        build_execution_order(s, td.n_parents, td.txmeta_cids.data(), exo);
    } catch (Error& e) {
        // a block the walk lacks, or one that does not decode (the generator reports it): the base plan is the round
        if (e.status != IPCFP_ERR_MISSING_BLOCK && e.status != IPCFP_ERR_DECODE) throw;
        finish();
        return;
    }
    if (!n) { finish(); return; }
    AsyncBuf<uint64_t> pos(n + 1, st);
    message_exec_indices(s, exo, cids, n, pos.p);
    AsyncBuf<uint8_t> d_in(64 + 38 * n + 16, st), miss(2 * 38 * n + 16, st);
    IPCFP_CUDA(cudaMemcpyAsync(d_in.p, td.receipts_root, 38, cudaMemcpyHostToDevice, st));
    IPCFP_CUDA(cudaMemcpyAsync(d_in.p + 64, cids, 38 * n, cudaMemcpyHostToDevice, st));
    const uint64_t nwords = (s->n + 31) / 32 + 1;
    AsyncBuf<uint32_t> needed(nwords, st);
    needed.zero();
    AsyncBuf<unsigned long long> ctr(PC_COUNT, st);
    ctr.zero();
    MsgProofArgs a{};
    a.store = s->view; a.cids = d_in.p + 64; a.exec_indices = pos.p; a.n = n; a.with_body = (flags & IPCFP_MESSAGE_WITH_BODY) ? 1 : 0;
    k_plan_messages<<<div_up(n, 128), 128, 0, st>>>(a, d_in.p, needed.p, miss.p, ctr.p); IPCFP_LAUNCH_CHECK();
    k_plan_popc<<<div_up(nwords, 256), 256, 0, st>>>(needed.p, nwords, ctr.p + PC_NEEDED); IPCFP_LAUNCH_CHECK();
    PinnedArray hc(s->pool, PC_COUNT * 8);
    IPCFP_CUDA(cudaMemcpyAsync(hc.p, ctr.p, PC_COUNT * 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    const uint64_t n_miss = hc.as<unsigned long long>()[PC_MISSING];
    out.n_needed += hc.as<unsigned long long>()[PC_NEEDED];   // the paths' blocks are none of the base's
    if (n_miss) {
        std::vector<uint8_t> more(38 * n_miss);
        IPCFP_CUDA(cudaMemcpyAsync(more.data(), miss.p, 38 * n_miss, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
        out.cids.insert(out.cids.end(), more.begin(), more.end());
        sort_cids_host(out.cids);
        std::vector<uint8_t> u;   // unique, in `Cid` order
        for (uint64_t k = 0; k < out.cids.size() / 38; k++)
            if (u.empty() || memcmp(u.data() + u.size() - 38, out.cids.data() + 38 * k, 38)) u.insert(u.end(), out.cids.begin() + 38 * k, out.cids.begin() + 38 * k + 38);
        out.cids.swap(u);
    }
    finish();
}

}  // namespace ipcfp
