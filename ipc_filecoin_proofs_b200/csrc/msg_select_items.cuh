// msg_select_items.cuh — per-item device functions of the message-selected event call (ipcfp_generate_message_log_proof_resident,
// DESIGN.md §3 "Logs of given messages"): the requested message CIDs put in order, the execution positions that hold one of them, and
// the per-receipt match of the selected receipts. The kernels that drive them are in events.cu; they live in a header so that
// tests/host_fuzz can run the very same code on the CPU against the Python restatement.
#pragma once
#include "events_items.cuh"

namespace ipcfp {

// a 38-byte CID as RawCid (the layout of the message AMTs' values, rawcid.cuh)
__host__ __device__ __forceinline__ RawCid rawcid_from_bytes(const uint8_t* c) {
    RawCid r;
    for (int k = 0; k < 4; k++) {
        uint64_t w = 0;
        for (int b = 0; b < 8; b++) w |= (uint64_t)c[6 + 8 * k + b] << (8 * b);
        r.w[k] = w;
    }
    uint64_t p = 0;
    for (int b = 0; b < 6; b++) p |= (uint64_t)c[b] << (8 * b);
    r.w[4] = p;
    return r;
}

// a total order on RawCid (the words in turn); any total order serves the binary search
__host__ __device__ __forceinline__ int rawcid_cmp(const RawCid& a, const RawCid& b) {
    for (int k = 0; k < 5; k++)
        if (a.w[k] != b.w[k]) return a.w[k] < b.w[k] ? -1 : 1;
    return 0;
}

// The requests are sorted once by (w[0], …, w[4], input position): an LSD radix sort (prims.cu, stable) over ten 32-bit slices, least
// significant first, starting from the input order. Slice q (0 = most significant) is half q % 2 (0: high) of word q / 2.
#define MSG_SORT_SLICES 10
__host__ __device__ __forceinline__ uint32_t msg_sort_key(const RawCid& c, uint32_t q) {
    const uint64_t w = c.w[q >> 1];
    return (q & 1) ? (uint32_t)w : (uint32_t)(w >> 32);
}

// Execution position i (< n_exec): exec[i] = exec_raw[exec_idx[i]] binary-searched among the sorted requests. Every request that names
// it gets i as its execution index (the execution order holds each CID once, so no two positions write one request); the receipt is
// selected when i < n_receipts. Returns whether it is.
__host__ __device__ __forceinline__ bool msg_select_item(const RawCid* exec_raw, const uint32_t* exec_idx, uint64_t i, const RawCid* sorted,
                                                         const uint32_t* sorted_pos, uint32_t n, uint64_t n_receipts, uint64_t* exec_indices) {
    const RawCid c = exec_raw[exec_idx[i]];
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (rawcid_cmp(sorted[mid], c) < 0) lo = mid + 1; else hi = mid;
    }
    bool hit = false;
    for (uint32_t k = lo; k < n && rawcid_cmp(sorted[k], c) == 0; k++) {
        exec_indices[sorted_pos[k]] = i;
        hit = true;
    }
    return hit && i < n_receipts;
}

// The match of one selected receipt: pass 1's per-receipt result (k_pass1_stage), from the arena decoders alone. A receipt without an
// events root matches nothing; a missing root or a fault in its events AMT is pass 1's fault at that receipt. The events AMT is walked
// in full (walk_events, which decodes the root node as pass 1's arena path does), so counts, bytes and the first fault are pass 1's.
template <class P> struct MsgMatchArgsT {
    StoreView store;
    const StoreView* store_dev;
    const P* m_dev;
    const uint8_t* events_roots;
    const uint8_t* has_root;
    const uint32_t* sel;           // selected receipts, ascending
    const unsigned long long* n_sel;
    uint64_t n_sel_max;            // the grid's bound on *n_sel
    uint32_t* match_bits;          // bit i
    uint32_t* cnt;                 // [i] matching events of receipt i
    uint32_t* nbytes;              // [i] topics+data bytes of those events
    unsigned long long* err;
    unsigned long long* stats;     // [0] roots read, [1] their bytes (+ 38 per CID), as pass 1 counts them
    uint32_t per_warp;             // 1: one selected receipt per warp (lane 0 walks); 0: one per thread
};

template <class P>
__device__ __forceinline__ void msg_match_item(const MsgMatchArgsT<P>& a, uint64_t t) {
    const uint64_t i = a.sel[t];
    if (!a.has_root[i]) return;
    const int32_t blk = store_lookup(a.store, a.events_roots + 38 * i);
    if (blk < 0) { report_error(a.err, ST_PASS1, i, DC_MISSING, 0); return; }
    uint32_t len;
    (void)store_block(a.store, (uint32_t)blk, len);
    atomicAdd(a.stats, 1ull);
    atomicAdd(a.stats + 1, (unsigned long long)(len + 38));
    WalkOut wo{0, 0, false};
    uint32_t detail = 0;
    const uint32_t rc = walk_events<WALK_COUNT>(a.store_dev, (uint32_t)blk, a.m_dev, nullptr, wo, nullptr, &detail);
    if (rc) { report_error(a.err, ST_PASS1, i, rc, detail); return; }
    a.cnt[i] = wo.nproofs;
    a.nbytes[i] = wo.nbytes;
    if (wo.any) atomicOr(a.match_bits + (i >> 5), 1u << (i & 31));
}

}  // namespace ipcfp
