// plan_items.cuh — per-item device functions of the fetch planner (plan.cu): which blocks the generators of a proof bundle would
// `get`, as far as the blocks already in the store tell, and which of them the store lacks (DESIGN.md §2, "Fetch planning"). They live
// in a header so that tests/host_fuzz can run the very same code on the CPU. Every decoder is the generators' own: amt_root_begin /
// amt_node_begin (ipld.cuh), walk_events and receipts_get (events_items.cuh), storage_proof_one (storage.cuh).
#pragma once
#include "events_items.cuh"
#include "actor_items.cuh"
#include "message_proof_items.cuh"
#include "storage.cuh"

namespace ipcfp {

// ---- whole-AMT walk (rules 1 and 2): one frontier item per block, level by level
enum PlanKind : uint32_t {
    PK_NONE = 0,      // an empty slot (a receipt without an events root)
    PK_BLOCK = 1,     // needed, not expanded: parent / child headers, the receipts root, the StateRoot
    PK_TXMETA = 2,    // [bls_root, secp_root] → two message-AMT roots
    PK_MSG_ROOT = 3,  // AMT v0 root of messages
    PK_EV_ROOT = 4,   // AMT v3 root of StampedEvents
    PK_NODE = 5       // AMT node below a root: every link
};
struct PlanItem {
    const uint8_t* cid;   // 38 bytes in device memory that outlives the call (arena, tipset, uploaded roots), padded by ≥ 16
    uint32_t kind;
    uint32_t bw_tree;     // bit width | tree << 8 (tree 1: an events AMT, whose missing blocks hold back rule 3)
};
// A block expands once per class: the class fixes how it decodes (kind, bit width), so a block reached twice in one class has the
// same children. 12 classes: TxMeta, message root, events root, message node (bw 3), events node at bw 1..8.
#define PLAN_CLASSES 12
__host__ __device__ __forceinline__ uint32_t plan_class(const PlanItem& it) {
    const uint32_t bw = it.bw_tree & 0xff, tree = it.bw_tree >> 8;
    if (it.kind == PK_TXMETA) return 0;
    if (it.kind == PK_MSG_ROOT) return 1;
    if (it.kind == PK_EV_ROOT) return 2;
    return tree ? 3 + bw : 3;   // bw 1..8 → 4..11
}

// The children of one present block under its item's rule; out == nullptr counts them. A block that does not decode under its rule has
// none (the generator, not the planner, reports it).
__device__ __forceinline__ uint32_t plan_children(const uint8_t* p, uint32_t len, const PlanItem& it, PlanItem* out) {
    Rd r(p, len);
    const uint32_t tree = it.bw_tree >> 8;
    if (it.kind == PK_TXMETA) {   // record_transaction_amts (events/generator.rs:148-177): the TxMeta decode of k_setup
        rd_array_exact(r, 2);
        uint32_t c0 = rd_cid(r), c1 = rd_cid(r);
        rd_end(r);
        if (r.err) return 0;
        if (out) {
            out[0] = PlanItem{p + c0, PK_MSG_ROOT, 3};
            out[1] = PlanItem{p + c1, PK_MSG_ROOT, 3};
        }
        return 2;
    }
    uint32_t bw = it.bw_tree & 0xff;
    if (it.kind == PK_MSG_ROOT || it.kind == PK_EV_ROOT) {
        uint32_t height;
        uint64_t cnt;
        amt_root_begin(r, it.kind == PK_MSG_ROOT ? 0 : 3, bw, height, cnt);
        if (r.err) return 0;
    } else if (it.kind != PK_NODE) return 0;
    AmtNodeHdr h;
    amt_node_begin(r, bw, h);
    if (r.err) return 0;
    if (out) for (uint32_t k = 0; k < h.nl; k++) out[k] = PlanItem{p + h.links_off + 43 * k + 5, PK_NODE, bw | (tree << 8)};
    return h.nl;
}

// ---- rule 3: does receipt i match one of the specs (pass 1's rule: walk_events over the whole events AMT, actor filter included)?
// A receipt whose events AMT fails to decode (or, which the gate rules out, lacks a block) does not match.
// P: Matcher (n_specs specs) or LogFilter (n_specs filters: a receipt matches when one of them does).
template <class P>
__device__ __forceinline__ bool plan_receipt_matches(const StoreView* s_dev, uint32_t root_blk, const P* m, uint64_t n_specs) {
    for (uint64_t k = 0; k < n_specs; k++) {
        WalkOut wo{0, 0, false};
        uint32_t detail = 0;
        if (walk_events<WALK_ANY>(s_dev, root_blk, m + k, nullptr, wo, nullptr, &detail)) return false;
        if (wo.any) return true;
    }
    return false;
}

// ---- rules 3 and 4 are paths: each one is followed through the blocks the store holds up to the first it lacks, which is returned
// (nullptr: the path ends in the store). The present blocks are marked in `needed` (rank bitmap).
// Amt::get(i) of the receipts AMT, pass 2's receipts_get. Only a child link can be missing: the root node's decode and the range check
// after it never name a block.
__device__ __forceinline__ const uint8_t* plan_receipt_path(const StoreView& s, const uint8_t* receipts_root, uint64_t i, uint32_t* needed) {
    const int32_t rb = store_lookup(s, receipts_root);
    if (rb < 0) return nullptr;   // the root itself is a PK_BLOCK item
    const uint8_t* miss = nullptr;
    uint32_t detail = 0;
    (void)receipts_get(s, (uint32_t)rb, i, needed, &detail, &miss);
    return miss;
}
// generate_storage_proof for spec t (storage_proof_one): the header is a PK_BLOCK item; a header that does not decode or names another
// ParentStateRoot ends the path, as it ends the generator.
__device__ __forceinline__ const uint8_t* plan_storage_path(const StorageArgs& a, uint64_t t, uint32_t* needed) {
    Recorder rec{nullptr, 0, needed, false};
    rec.rank_of = a.store.rank_of;
    ipcfp_storage_proof q;
    Fail f{0, 0};
    if (storage_proof_one(a, t, rec, q, f) || f.code != DC_MISSING) return nullptr;
    return rec.missing;
}
// ipcfp_generate_actor_proofs_resident for request t: the header, the Init path (a non-ID address; the generator walks it once per
// call, the planner once per request), then actor_proof_one. A path the generator fails on for another reason ends here.
__device__ __forceinline__ const uint8_t* plan_actor_path(const ActorArgs& a, uint64_t t, uint32_t* needed) {
    Recorder rec{nullptr, 0, needed, false};
    rec.rank_of = a.store.rank_of;
    Fail f{0, 0}, init_fail{0, 0};
    const uint8_t* psr;
    if (!actor_header(a, rec, psr, f)) return f.code == DC_MISSING ? rec.missing : nullptr;
    const uint8_t* map = nullptr;
    if (a.addrs[t].bytes[0] != 0 && !resolve_init(a.store, rec, psr, map, init_fail)) return init_fail.code == DC_MISSING ? rec.missing : nullptr;
    ipcfp_actor_proof q;
    memset(&q, 0, sizeof q);
    uint64_t cb;
    if (actor_proof_one(a, a.addrs[t], map, init_fail, rec, q, cb, f) || f.code != DC_MISSING) return nullptr;
    return rec.missing;
}

// message proofs: request t's receipts-AMT path (plan_receipt_path) at its execution position and, with the body, its message block.
// Writes the CIDs the store lacks to miss (at most two) and returns how many; a request that was not executed reads nothing.
__device__ __forceinline__ uint32_t plan_message_path(const MsgProofArgs& a, const uint8_t* receipts_root, uint64_t t, uint32_t* needed,
                                                      const uint8_t* miss[2]) {
    const uint64_t e = a.exec_indices[t];
    if (e == UINT64_MAX) return 0;
    uint32_t k = 0;
    if (const uint8_t* m = plan_receipt_path(a.store, receipts_root, e, needed)) miss[k++] = m;
    if (a.with_body) {
        const uint8_t* c = a.cids + 38 * t;
        const int32_t b = store_lookup(a.store, c);
        if (b < 0) miss[k++] = c;
        else witness_mark(a.store, needed, (uint32_t)b);
    }
    return k;
}

}  // namespace ipcfp
