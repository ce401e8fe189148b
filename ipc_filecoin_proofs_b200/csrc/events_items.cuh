// events_items.cuh — per-receipt device functions of the event path: the events-AMT walk, pass 1's per-receipt decode, the
// receipts-AMT lookup and pass 2's per-match work (reference events/generator.rs:206-301). The kernels that drive them are in
// events.cu; they live in a header so that tests/host_fuzz can run the very same code on the CPU against the oracle.
#pragma once
#include "ipld.cuh"
#include "log_filter.cuh"
#include "rawcid.cuh"

namespace ipcfp {

// ------------------------------------------------------------------------------------------ events AMT walk
enum WalkMode { WALK_ANY = 0, WALK_COUNT = 1, WALK_EMIT = 2 };



struct EmitCtx {
    ipcfp_event_proof* proofs;   // base for this match
    uint8_t* blob;               // data blob base (whole result)
    uint64_t blob_off;           // running offset for this match
    uint64_t exec_index;
    RawCid msg_cid;
};
struct WalkOut { uint32_t nproofs; uint32_t nbytes; bool any; };

__device__ __forceinline__ void emit_proof(const uint8_t* p, const EvLog& ev, uint64_t j, EmitCtx& ec, uint32_t k) {
    ipcfp_event_proof q;
    q.exec_index = ec.exec_index;
    q.event_index = j;
    q.emitter = ev.emitter;
    q.n_topics = ev.ntopics;
    q.data_len = ev.data_len;
    q.topics_off = ec.blob_off;
    uint8_t* o = ec.blob + ec.blob_off;
    for (uint32_t t = 0; t < ev.ntopics; t++) {
        const uint8_t* src = p + topic_offset(ev, t);
        for (int b = 0; b < 32; b++) o[32 * t + b] = src[b];
    }
    ec.blob_off += 32ull * ev.ntopics;
    q.data_off = ec.blob_off;
    o = ec.blob + ec.blob_off;
    for (uint32_t b = 0; b < ev.data_len; b++) o[b] = p[ev.data_off + b];
    ec.blob_off += ev.data_len;
    for (int b = 0; b < 6; b++) q.message_cid[b] = (uint8_t)(ec.msg_cid.w[4] >> (8 * b));
    for (int b = 0; b < 32; b++) q.message_cid[6 + b] = (uint8_t)(ec.msg_cid.w[b >> 3] >> (8 * (b & 7)));
    q._pad[0] = q._pad[1] = 0;
    ec.proofs[k] = q;
}

// Decodes the values of one events-AMT node. Returns false on a decode error (r.err set).
// PREFETCH: an L2 prefetch 2 lines ahead of the dependent walk before every event (off in the staged pass 1's arena fallback).
// P: the predicate (Matcher for a spec, LogFilter for a log filter; event_matches of either).
template <int MODE, bool PREFETCH = true, class P>
__device__ __forceinline__ void node_events(Rd& r, const uint8_t* p, const AmtNodeHdr& h, uint32_t nv, uint64_t base, const P& m,
                                            WalkOut& wo, EmitCtx* ec) {
    for (uint32_t v = 0; v < nv && !r.err; v++) {
        if (PREFETCH && r.pos + 256 < r.n) prefetch_l2(r.p + r.pos + 256);
        EvLog ev;
        decode_stamped_event(r, ev);
        if (r.err) break;
        if (event_matches(p, ev, m)) {
            wo.any = true;
            if (MODE != WALK_ANY) {
                uint64_t j = base + bm_select(h.bm, v);
                if (MODE == WALK_EMIT) emit_proof(p, ev, j, *ec, wo.nproofs);
                wo.nproofs++;
                wo.nbytes += 32 * ev.ntopics + ev.data_len;
            }
        }
    }
}

// Full in-order walk of Amt<StampedEvent> (v3) rooted at block root_blk — `for_each` of
// fvm_ipld_amt [UPSTREAM]: every reachable node is loaded through the store (and recorded when
// wbits != nullptr). Returns 0 ok, else DevCode; detail in *detail. A Matcher is copied into registers; a LogFilter, whose inline
// sets are indexed per value, is read where it lies.
template <class P> struct PredLocal { using T = const P&; };
template <> struct PredLocal<Matcher> { using T = const Matcher; };
template <int MODE, class P>
static __device__ __noinline__ uint32_t walk_events(const StoreView* sp, uint32_t root_blk, const P* mp, uint32_t* wbits, WalkOut& wo, EmitCtx* ec,
                                uint32_t* detail) {
    const StoreView& s = *sp;
    typename PredLocal<P>::T m = *mp;
    struct Frame { uint32_t blk; uint32_t k; uint64_t base; };
    Frame stk[66];
    int depth = 0;
    stk[0].blk = root_blk; stk[0].k = 0; stk[0].base = 0;
    uint32_t bw = 3, height = 0;
    while (depth >= 0) {
        Frame& f = stk[depth];
        uint32_t len;
        const uint8_t* p = store_block(s, f.blk, len);
        Rd r(p, len);
        if (depth == 0) { uint64_t cnt; amt_root_begin(r, 3, bw, height, cnt); }
        uint32_t lvl = height - (uint32_t)depth;
        AmtNodeHdr h;
        amt_node_begin(r, bw, h);
        if (f.k == 0) {
            uint32_t nv = rd_array(r);
            node_events<MODE>(r, p, h, nv, f.base, m, wo, ec);
            amt_node_finish(r, h, nv, lvl);
            if (r.err) { *detail = r.err; return DC_DECODE; }
        } else if (r.err) { *detail = r.err; return DC_DECODE; }
        if (h.nl == 0 || f.k >= h.nl) { depth--; continue; }
        uint32_t slot = bm_select(h.bm, f.k);
        int32_t child = store_lookup(s, p + h.links_off + 43 * f.k + 5);
        if (child < 0) { *detail = 0; return DC_MISSING; }
        if (wbits) witness_mark(s, wbits, (uint32_t)child);
        uint64_t cbase = f.base + (uint64_t)slot * pow_sat(bw, lvl);
        f.k++;
        depth++;
        stk[depth].blk = (uint32_t)child; stk[depth].k = 0; stk[depth].base = cbase;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------ pass 1
template <class P> struct Pass1ArgsT {
    StoreView store;
    const StoreView* store_dev;    // same view in device memory (for the out-of-line walker)
    const P* m_dev;
    P m;
    const uint8_t* events_roots;
    const uint8_t* has_root;
    uint64_t lo, hi;
    uint32_t* match_bits;          // bit (i - lo)
    uint32_t* cnt;                 // [i - lo] matching events of receipt i  (EventProof count of pass 2)
    uint32_t* nbytes;              // [i - lo] topics+data bytes of those events
    unsigned long long* err;
    unsigned long long* stats;     // [0] nodes scanned, [1] bytes scanned
};
using Pass1Args = Pass1ArgsT<Matcher>;

// ------------------------------------------------------------------------------------------ receipts AMT
// Amtv0<Receipt>::get(i) with recording (events/generator.rs:249): amt_get with every child marked in wbits. missing: as amt_get's.
// Pass 2 runs behind k_setup's setup_receipts_root, which decodes this root node whole: a root node that fails fails the call with
// ST_RECEIPTS_ROOT, which ranks before every pass-2 error, so where the range check sits is not observable here.
__device__ __forceinline__ int receipts_get(const StoreView& s, uint32_t root_blk, uint64_t i, uint32_t* wbits, uint32_t* detail,
                                            const uint8_t** missing = nullptr) {
    const uint8_t* leaf;
    return amt_get(s, root_blk, 0, i, [](Rd& r, bool) { (void)parse_receipt(r); }, &leaf, detail, wbits, missing);
}

// ------------------------------------------------------------------------------------------ pass 2
template <class P> struct Pass2ArgsT {
    StoreView store;
    const StoreView* store_dev;
    const P* m_dev;
    P m;
    const uint8_t* events_roots;
    uint64_t lo;
    const uint32_t* match_rel;     // positions relative to lo, ascending
    uint64_t n_match;
    uint32_t receipts_root_blk;
    const RawCid* exec_cids;       // exec_raw[pos]
    const uint32_t* exec_idx;      // execution order → position in exec_raw
    const unsigned long long* n_exec;
    uint32_t* wbits;
    unsigned long long* err;
    const uint32_t* cnt;           // [i - lo] proofs of receipt i (from pass 1)
    const uint64_t* proof_base;    // [i - lo] exclusive scans over all receipts of the range
    const uint64_t* byte_base;
    ipcfp_event_proof* proofs;
    uint8_t* blob;
    uint32_t* any_skip;            // set when a matching receipt is absent from the receipts AMT
    uint32_t per_warp;             // 1: one matching receipt per warp (lane 0 walks); 0: one per thread
    uint32_t resolve_msg;          // 1: exec.get(i) check + message CID from exec_cids; 0: neither (shard: the execution order spans shards and
                                   // is resolved afterwards — by the caller, or by the in-library protocol with k_check_exec)
};
using Pass2Args = Pass2ArgsT<Matcher>;

// One thread per matching receipt (events/generator.rs:242-301): exec.get(i), r_amt.get(i) with path
// recording, full in-order walk of its events AMT with recording, EventProof emission at the
// offsets pass 1 already counted.
template <class P>
__device__ __forceinline__ void pass2_item(const Pass2ArgsT<P>& a, uint64_t t) {
    uint32_t rel = a.match_rel[t];
    uint64_t i = a.lo + rel;
    // exec.get(i) comes first (:244-246)
    if (a.resolve_msg && i >= *a.n_exec) { report_error(a.err, ST_PASS2, i, DC_MISSING_EXEC, 0); return; }
    uint32_t detail = 0;
    int got = receipts_get(a.store, a.receipts_root_blk, i, a.wbits, &detail);
    if (got < 0) { report_error(a.err, ST_PASS2, i, (uint32_t)(-got), detail); return; }
    ipcfp_event_proof* out = a.proofs + a.proof_base[rel];
    if (got == 0) {  // `continue` at :249-251 — the slots pass 1 reserved stay empty and are dropped on the host
        uint32_t c = a.cnt[rel];
        for (uint32_t k = 0; k < c; k++) out[k].exec_index = 0xFFFFFFFFFFFFFFFFull;
        *a.any_skip = 1;
        return;
    }
    int32_t root = store_lookup(a.store, a.events_roots + 38 * i);
    if (root < 0) { report_error(a.err, ST_PASS2, i, DC_MISSING, 0); return; }
    witness_mark(a.store, a.wbits, (uint32_t)root);
    WalkOut wo{0, 0, false};
    EmitCtx ec;
    ec.proofs = out;
    ec.blob = a.blob;
    ec.blob_off = a.byte_base[rel];
    ec.exec_index = i;
    if (a.resolve_msg == 1) ec.msg_cid = a.exec_cids[a.exec_idx[i]]; else ec.msg_cid = RawCid{};
    uint32_t rc = walk_events<WALK_EMIT>(a.store_dev, (uint32_t)root, a.m_dev, a.wbits, wo, &ec, &detail);
    if (rc) report_error(a.err, ST_PASS2, i, rc, detail);
}
}  // namespace ipcfp
