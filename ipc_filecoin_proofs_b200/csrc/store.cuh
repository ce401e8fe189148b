// store.cuh — device-resident IPLD block arena + CID hash index.
//
// Replaces the reference's Blockstore implementations (client/blockstore.rs:20-37,
// client/cached_blockstore.rs:53-85) for the hot path: `get` is a hash probe that returns a
// block INDEX (offset/length into the arena) instead of an owned copy, and RecordingBlockStore
// (common/blockstore.rs:8-39) becomes one bit per block in a witness bitmap.
//
// HBM layout (n blocks, B blob bytes):
//   arena    : [16 B pad][blob as given, any offsets][tail pad]      (store.cu: ARENA_HEAD, ARENA_TAIL)
//   offsets  : u64[n]    lengths: u32[n]
//   digests  : Digest[n] (32 B, raw digest bytes)       cls: u8[n] (CID prefix class)
//   table    : u64[2^k], k = ceil(log2(2n)); slot = fingerprint32 << 32 | (block index + 1)
#pragma once
#include "common.cuh"

namespace ipcfp {

#define IPCFP_MAX_CID_CLASSES 8

// everything a Blockstore::get needs about one block in ONE 64-byte line: the probe compares the digest,
// the hit continues with offset/length from the same line (instead of four scattered arrays)
struct __align__(64) BlockRec { Digest d; uint64_t off; uint32_t len; uint32_t cls; uint64_t pad[2]; };

struct StoreView {
    const uint8_t* blob;      // arena + 16
    const BlockRec* recs;     // n records (hot lookup path)
    const uint64_t* offsets;
    const uint32_t* lengths;
    const Digest* digests;
    const uint8_t* cls;
    const uint64_t* table;
    uint64_t mask;
    uint32_t n;
    uint32_t n_classes;
    uint8_t class_prefix[IPCFP_MAX_CID_CLASSES][8];  // 6 significant bytes each
    // Position of every block in `Cid` Ord among the blocks of this store, computed once at ingest, and its inverse. Witness bitmaps
    // are indexed by RANK, so reading a bitmap in bit order yields the witness already in BTreeSet<Cid> order (no per-call sort).
    // nullptr (host-side test stores) = identity.
    const uint32_t* rank_of;
    const uint32_t* block_at_rank;
};

#ifdef __CUDACC__
__device__ __forceinline__ int cid_class(const StoreView& s, const uint8_t* cid38) {
    for (uint32_t c = 0; c < s.n_classes; c++) {
        bool eq = true;
#pragma unroll
        for (int k = 0; k < 6; k++) eq &= cid38[k] == s.class_prefix[c][k];
        if (eq) return (int)c;
    }
    return -1;
}

// Blockstore::get by (class, digest): block index or -1.
__device__ __forceinline__ int32_t store_find(const StoreView& s, uint32_t cls, const Digest& d) {
    uint64_t h = digest_hash(d, cls);
    uint32_t fp = (uint32_t)(h >> 32) | 1u;
    uint64_t slot = h & s.mask;
    for (;;) {
        uint64_t e = __ldg(s.table + slot);
        if (e == 0) return -1;
        if ((uint32_t)(e >> 32) == fp) {
            uint32_t idx = (uint32_t)e - 1;
            const BlockRec* q = s.recs + idx;
            const ulonglong2 w0 = __ldg((const ulonglong2*)&q->d), w1 = __ldg((const ulonglong2*)&q->d + 1);   // 2 x 16-byte loads, one sector
            if (w0.x == d.w[0] && w0.y == d.w[1] && w1.x == d.w[2] && w1.y == d.w[3] && __ldg(&q->cls) == cls) return (int32_t)idx;
        }
        slot = (slot + 1) & s.mask;
    }
}
// lookup by the 38 raw CID bytes (any alignment)
__device__ __forceinline__ int32_t store_lookup(const StoreView& s, const uint8_t* cid38) {
    int c = cid_class(s, cid38);
    if (c < 0) return -1;
    Digest d = load_digest(cid38 + 6);
    return store_find(s, (uint32_t)c, d);
}
__device__ __forceinline__ const uint8_t* store_block(const StoreView& s, uint32_t idx, uint32_t& len) {
    const BlockRec* q = s.recs + idx;
    len = __ldg(&q->len);
    return s.blob + __ldg(&q->off);
}
// RecordingBlockStore::get side effect: one bit per block, at the block's RANK in `Cid` Ord
__device__ __forceinline__ void witness_mark_rank(uint32_t* wbits, uint32_t r) {
    uint32_t m = 1u << (r & 31);
    uint32_t* w = wbits + (r >> 5);
    if (!(*(volatile uint32_t*)w & m)) atomicOr(w, m);
}
__device__ __forceinline__ void witness_mark(const StoreView& s, uint32_t* wbits, uint32_t idx) {
    witness_mark_rank(wbits, s.rank_of ? __ldg(s.rank_of + idx) : idx);
}
// identity ranks (host-side test stores only)
__device__ __forceinline__ void witness_mark(uint32_t* wbits, uint32_t idx) { witness_mark_rank(wbits, idx); }
#endif

}  // namespace ipcfp
