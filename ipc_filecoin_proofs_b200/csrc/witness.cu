// witness.cu — K4/K6: turn the witness bitmap (one bit per store block, set by every recorded
// Blockstore::get) into the reference's `Vec<ProofBlock>` in `Cid` Ord order.
// Replaces BTreeSet<Cid> + WitnessCollector::materialize (common/witness.rs:9-57).
//
// Two-phase so the bulk of the device→host copy hides behind the scan:
//   snapshot (after the message-AMT walk): bitmap → ordered index list A → block bytes gathered
//            into a 16-byte-padded staging blob → D2H on a second stream while pass 1/2 run;
//   finish   (after pass 2): B = bits set since the snapshot → gathered + copied behind A;
//            A and B are both in `Cid` order already (the bitmap is indexed by the blocks' Cid RANK, computed once per store at
//            ingest), so the merged position of an entry is its own position plus the number of the other list's bits below it:
//            one emit kernel, no per-call sort → cids / offsets / lengths arrays.
// The output keeps block bytes in arrival order (A then B) and the (cid, offset, length) index in `Cid` order.
#include "engine.cuh"
#include "prims.cuh"

namespace ipcfp {

struct ClassRanks { uint8_t r[IPCFP_MAX_CID_CLASSES]; };

__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | (uint64_t)__byte_perm(hi, 0, 0x0123);
}
// lexicographic order of the raw digest bytes
__device__ __forceinline__ int digest_cmp(const Digest& a, const Digest& b) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint64_t x = bswap64(a.w[k]), y = bswap64(b.w[k]);
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}

// ord[i] = i, keys[i] = first four digest bytes (big-endian) of block idx[i]
__global__ void k_digest_keys(const uint32_t* __restrict__ idx, uint64_t m, const Digest* __restrict__ digests, uint32_t* keys, uint32_t* ord) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    uint64_t w0 = digests[idx[i]].w[0];
    keys[i] = __byte_perm((uint32_t)w0, 0, 0x0123);
    ord[i] = (uint32_t)i;
}
__global__ void k_class_keys(const uint32_t* __restrict__ idx, const uint32_t* __restrict__ ord, uint64_t m, const uint8_t* __restrict__ cls,
                             ClassRanks cr, uint32_t* keys) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    keys[i] = cr.r[cls[idx[ord[i]]]];
}
// After the radix passes entries are ordered by (class rank, first 4 digest bytes). Runs with equal
// 4-byte prefixes (≈ m²/2³³ pairs for random digests) are finished by one thread per run.
__global__ void k_tie_fix(const uint32_t* __restrict__ idx, uint32_t* ord, uint64_t m, const Digest* __restrict__ digests,
                          const uint8_t* __restrict__ cls, ClassRanks cr) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    auto key_eq = [&](uint64_t a, uint64_t b) {
        uint32_t x = idx[ord[a]], y = idx[ord[b]];
        return cr.r[cls[x]] == cr.r[cls[y]] && (uint32_t)digests[x].w[0] == (uint32_t)digests[y].w[0];
    };
    if (i > 0 && key_eq(i - 1, i)) return;          // not a run start
    if (i + 1 >= m || !key_eq(i, i + 1)) return;    // run of length 1
    uint64_t j = i + 1;
    while (j + 1 < m && key_eq(i, j + 1)) j++;      // run = [i, j]
    for (uint64_t a = i + 1; a <= j; a++) {         // insertion sort by full digest, stable
        uint32_t v = ord[a];
        Digest dv = digests[idx[v]];
        uint64_t b = a;
        while (b > i && digest_cmp(digests[idx[ord[b - 1]]], dv) > 0) { ord[b] = ord[b - 1]; b--; }
        ord[b] = v;
    }
}

// ord (device, m entries) receives the permutation that sorts idx[] by CID (stable). Runs once per store, at ingest; the caller owns
// the workspace (sort_by_cid_ws_bytes(m) bytes — from the device pool, not stream-ordered: a new store has a new stream).
static inline size_t ws_round(size_t b) { return (b + 255) & ~(size_t)255; }
size_t sort_by_cid_ws_bytes(uint64_t m) {
    const unsigned nb = radix_blocks(m);
    return 3 * ws_round(m * 4 + 64) + ws_round(((size_t)256 * nb + 256) * 4) + ws_round(((size_t)256 * nb + 256) * 8) +
           ws_round((scan_scratch_elems((uint64_t)256 * nb) + 8) * 8);
}
void sort_by_cid(Store* s, const uint32_t* idx_dev, uint32_t* ord, uint64_t m, void* ws) {
    if (m == 0) return;
    cudaStream_t st = s->stream;
    const unsigned nb = radix_blocks(m);
    uint8_t* w = (uint8_t*)ws;
    uint32_t* keys = (uint32_t*)w; w += ws_round(m * 4 + 64);
    uint32_t* keys_alt = (uint32_t*)w; w += ws_round(m * 4 + 64);
    uint32_t* vals_alt = (uint32_t*)w; w += ws_round(m * 4 + 64);
    uint32_t* hist = (uint32_t*)w; w += ws_round(((size_t)256 * nb + 256) * 4);
    uint64_t* scan_tmp = (uint64_t*)w; w += ws_round(((size_t)256 * nb + 256) * 8);
    uint64_t* scratch = (uint64_t*)w;
    ClassRanks cr{};
    for (size_t c = 0; c < s->class_rank.size(); c++) cr.r[c] = (uint8_t)s->class_rank[c];
    k_digest_keys<<<div_up(m, 256), 256, 0, st>>>(idx_dev, m, s->digests.p, keys, ord); IPCFP_LAUNCH_CHECK();
    radix_sort_pairs(keys, ord, keys_alt, vals_alt, m, 32, hist, scan_tmp, scratch, st);
    if (s->class_prefix.size() > 1) {
        k_class_keys<<<div_up(m, 256), 256, 0, st>>>(idx_dev, ord, m, s->cls.p, cr, keys); IPCFP_LAUNCH_CHECK();
        radix_sort_pairs(keys, ord, keys_alt, vals_alt, m, 8, hist, scan_tmp, scratch, st);
    }
    k_tie_fix<<<div_up(m, 256), 256, 0, st>>>(idx_dev, ord, m, s->digests.p, s->cls.p, cr); IPCFP_LAUNCH_CHECK();
}

// idx[] holds RANKS (bit positions of the witness bitmap); bar = StoreView::block_at_rank
__global__ void k_padded_lengths(const uint32_t* __restrict__ idx, uint64_t m, const uint32_t* __restrict__ lengths, const uint32_t* __restrict__ bar, uint32_t* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) out[i] = (lengths[bar[idx[i]]] + 15u) & ~15u;
}
// Σ padded lengths of the late list (its length is only known on the device): out += …
__global__ void k_sum_padded_dev(const uint32_t* __restrict__ idx, const unsigned long long* __restrict__ count, uint64_t n_max, const uint32_t* __restrict__ lengths,
                                 const uint32_t* __restrict__ bar, unsigned long long* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long v = (i < n_max && i < *count) ? (unsigned long long)((lengths[bar[idx[i]]] + 15u) & ~15u) : 0ull;
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(out, v);
}
__global__ void k_andnot(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, uint32_t* out, uint64_t nwords) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nwords) out[i] = a[i] & ~b[i];
}
// one warp per witness block: arena → 16-byte-padded staging blob. 16-byte vector copies when the
// source block is 16-byte aligned (destination slots always are), byte copies otherwise.
__global__ void __launch_bounds__(256) k_witness_copy(const uint32_t* __restrict__ idx, uint64_t m, StoreView v, const uint64_t* __restrict__ offsets,
                                                      uint8_t* out) {
    uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint32_t lane = threadIdx.x & 31;
    if (w >= m) return;
    uint32_t len;
    const uint8_t* src = store_block(v, v.block_at_rank[idx[w]], len);
    uint8_t* dst = out + offsets[w];
    if (((uintptr_t)src & 15) == 0) {
        uint32_t nv = (len + 15) >> 4;  // the arena is padded, reading the tail of the last 16 bytes is safe
        const uint4* s4 = (const uint4*)src;
        uint4* d4 = (uint4*)dst;
        for (uint32_t i = lane; i < nv; i += 32) d4[i] = __ldg(s4 + i);
    } else {
        for (uint32_t i = lane; i < len; i += 32) dst[i] = src[i];
    }
}
// number of set bits of a bitmap below bit r (prefix = exclusive popcount prefix per word, as bitmap_to_indices leaves it)
__device__ __forceinline__ uint32_t bits_below(const uint32_t* __restrict__ bits, const uint64_t* __restrict__ prefix, uint32_t r) {
    return (uint32_t)prefix[r >> 5] + (uint32_t)__popc(bits[r >> 5] & ((1u << (r & 31)) - 1u));
}
// idx = [A: mA ranks ascending][B: m - mA ranks ascending], A and B disjoint. Entry i goes to its merged position f.
// The 38-byte CID records are built in shared memory and stored by the warp as 2-byte units (38·f is always even): the lanes of a
// warp nearly always hold consecutive positions, so each store instruction covers 64 contiguous bytes. One byte store per lane at a
// 38-byte stride touched a sector per lane, 38 times over.
#define EMIT_THREADS 256
__global__ void __launch_bounds__(EMIT_THREADS) k_witness_emit(const uint32_t* __restrict__ idx, const uint64_t* __restrict__ offs, uint64_t m,
                                                               uint64_t mA, uint64_t baseB, const uint32_t* __restrict__ bitsA,
                                                               const uint64_t* __restrict__ prefixA, const uint32_t* __restrict__ bitsB,
                                                               const uint64_t* __restrict__ prefixB, StoreView v, uint8_t* cids, uint64_t* out_offs,
                                                               uint32_t* out_lens, uint32_t* out_idx, int by_ref) {
    __shared__ uint16_t rec[EMIT_THREADS][19];
    __shared__ uint64_t pos[EMIT_THREADS];
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) {
        const uint32_t r = idx[i];
        uint64_t f;
        if (i < mA) f = i + (m > mA ? bits_below(bitsB, prefixB, r) : 0u);
        else f = (i - mA) + bits_below(bitsA, prefixA, r);
        const uint32_t b = v.block_at_rank[r];
        out_offs[f] = by_ref ? v.offsets[b] : offs[i] + (i >= mA ? baseB : 0);   // by reference: where the block sits in the blob the store was created from
        out_lens[f] = v.lengths[b];
        out_idx[f] = b;
        pos[threadIdx.x] = f;
        uint8_t* o = (uint8_t*)rec[threadIdx.x];
        uint32_t c = v.cls[b];
#pragma unroll
        for (int k = 0; k < 6; k++) o[k] = v.class_prefix[c][k];
        Digest d = v.digests[b];
#pragma unroll
        for (int w = 0; w < 4; w++)
#pragma unroll
            for (int k = 0; k < 8; k++) o[6 + 8 * w + k] = (uint8_t)(d.w[w] >> (8 * k));
    }
    __syncwarp();
    const uint32_t lane = threadIdx.x & 31, w0 = threadIdx.x - lane;
    const uint64_t first = i - lane;
    const uint32_t nrec = first < m ? (uint32_t)std::min<uint64_t>(32, m - first) : 0;
    for (uint32_t u = lane; u < nrec * 19; u += 32) {
        const uint32_t q = u / 19, k = u - 19 * q;
        ((uint16_t*)(cids + 38 * pos[w0 + q]))[k] = rec[w0 + q][k];
    }
}

WitnessBuilder::WitnessBuilder(Store* store) : s(store) {
    st = s->stream;
    if (!s->stream2) IPCFP_CUDA(cudaStreamCreateWithFlags(&s->stream2, cudaStreamNonBlocking));
    st2 = s->stream2;
    uint64_t n = s->n;
    nwords = (n + 31) / 32;
    idx.alloc(n + 64, st);
    offs.alloc(n + 64, st);
    plen.alloc(n + 64, st);
    bitsA.alloc(nwords + 8, st);
    word_prefix.alloc(nwords + 8, st);
    word_prefixB.alloc(nwords + 8, st);
    scratch.alloc(scan_scratch_elems(std::max<uint64_t>(nwords, n)) + 8, st);
}

// where to split the snapshot gather: DW_SPLIT_IDX = number of blocks in the first part, DW_SPLIT_BYTES = their padded bytes
__global__ void k_chunk_bounds(const uint64_t* __restrict__ offs, const unsigned long long* count, const unsigned long long* total, unsigned long long* out) {
    const uint64_t m = *count;
    uint64_t ia = m / 8;
    if (ia < 1024) ia = m < 1024 ? m : 1024;
    out[0] = ia;
    out[1] = ia < m ? offs[ia] : *total;
}
// padded length of every candidate slot of idx[] (the count is only known on the device: zero past it)
__global__ void k_padded_lengths_dev(const uint32_t* __restrict__ idx, const unsigned long long* __restrict__ count, uint64_t n_max,
                                     const uint32_t* __restrict__ lengths, const uint32_t* __restrict__ bar, uint32_t* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_max) out[i] = i < *count ? (lengths[bar[idx[i]]] + 15u) & ~15u : 0u;
}
// enqueue: bitmap → idx[0..mA), padded offsets; totals land in DW_WIT_A (mA) and DW_WIT_A_BYTES (bytesA) — the caller
// publishes both and syncs ONCE before start_copy
void WitnessBuilder::snapshot(const uint32_t* wbits) {
    unsigned long long* dw = s->dev_words.p;
    IPCFP_CUDA(cudaMemcpyAsync(bitsA.p, wbits, nwords * 4, cudaMemcpyDeviceToDevice, st));
    bitmap_to_indices(bitsA.p, s->n, idx.p, (uint64_t*)(dw + DW_WIT_A), word_prefix.p, scratch.p, st);
    if (s->n) { k_padded_lengths_dev<<<div_up(s->n, 256), 256, 0, st>>>(idx.p, dw + DW_WIT_A, s->n, s->lengths.p, s->block_at_rank.p, plen.p); IPCFP_LAUNCH_CHECK(); }
    exclusive_scan_u32(plen.p, offs.p, s->n, (uint64_t*)(dw + DW_WIT_A_BYTES), scratch.p, st);
    k_chunk_bounds<<<1, 1, 0, st>>>(offs.p, dw + DW_WIT_A, dw + DW_WIT_A_BYTES, dw + DW_SPLIT_IDX); IPCFP_LAUNCH_CHECK();
    have_snapshot = true;
}
// host knows mA and bytesA: gather (main stream, two parts), D2H on the side stream as soon as each part is there
void WitnessBuilder::start_copy(uint64_t mA_, uint64_t bytesA_, uint64_t split_idx, uint64_t split_bytes) {
    mA = mA_;
    bytesA = bytesA_;
    if (by_ref) {   // nothing to gather or copy: the index arrays are all the host gets (finish_start)
        bytesA = 0;
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_BLOB_COPIED], st2));
        return;
    }
    host_cap = bytesA + bytesA / 8 + (8u << 20);
    host_blob = PinnedArray(s->pool, host_cap);
    host_cap = host_blob.cap;
    dblobA.alloc(bytesA + 64, st);
    const uint64_t ia = std::min(split_idx, mA), ba = ia == mA ? bytesA : std::min(split_bytes, bytesA);
    if (ia) { k_witness_copy<<<div_up(ia * 32, 256), 256, 0, st>>>(idx.p, ia, s->view, offs.p, dblobA.p); IPCFP_LAUNCH_CHECK(); }
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_WITNESS_SORTED], st));
    IPCFP_CUDA(cudaStreamWaitEvent(st2, s->ev[EV_WITNESS_SORTED], 0));
    if (ba) IPCFP_CUDA(cudaMemcpyAsync(host_blob.p, dblobA.p, ba, cudaMemcpyDeviceToHost, st2));
    if (mA > ia) {
        k_witness_copy<<<div_up((mA - ia) * 32, 256), 256, 0, st>>>(idx.p + ia, mA - ia, s->view, offs.p + ia, dblobA.p); IPCFP_LAUNCH_CHECK();
        IPCFP_CUDA(cudaEventRecord(s->ev[EV_GATHER_B], st));
        IPCFP_CUDA(cudaStreamWaitEvent(st2, s->ev[EV_GATHER_B], 0));
        if (bytesA > ba) IPCFP_CUDA(cudaMemcpyAsync((uint8_t*)host_blob.p + ba, dblobA.p + ba, bytesA - ba, cudaMemcpyDeviceToHost, st2));
    }
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_BLOB_COPIED], st2));
}
// enqueue: B = bits & ~A → idx[mA..mA+mB); totals in DW_WIT_B (mB)
void WitnessBuilder::finish_enqueue(const uint32_t* wbits) {
    unsigned long long* dw = s->dev_words.p;
    bitsB.alloc(nwords + 8, st);
    k_andnot<<<div_up(nwords ? nwords : 1, 256), 256, 0, st>>>(wbits, bitsA.p, bitsB.p, nwords); IPCFP_LAUNCH_CHECK();
    bitmap_to_indices(bitsB.p, s->n, idx.p + mA, (uint64_t*)(dw + DW_WIT_B), word_prefixB.p, scratch.p, st);
    // their padded bytes, so that the host learns both numbers with the caller's next synchronisation
    IPCFP_CUDA(cudaMemsetAsync(dw + DW_WIT_B_BYTES, 0, 8, st));
    const uint64_t bound = s->n > mA ? s->n - mA : 0;
    if (bound) { k_sum_padded_dev<<<div_up(bound, 256), 256, 0, st>>>(idx.p + mA, dw + DW_WIT_B, bound, s->lengths.p, s->block_at_rank.p, dw + DW_WIT_B_BYTES); IPCFP_LAUNCH_CHECK(); }
}
void WitnessBuilder::finish(uint64_t mB_, uint64_t bytesB_, WitnessOut& out, bool want_sorted_idx) {
    finish_start(mB_, bytesB_, out, want_sorted_idx);
    finish_join(out);
}
void WitnessBuilder::finish_start(uint64_t mB_, uint64_t bytesB_, WitnessOut& out, bool want_sorted_idx) {
    mB = mB_;
    bytesB = bytesB_;
    unsigned long long* dw = s->dev_words.p;
    uint64_t m = mA + mB;
    if (by_ref) { bytesB = 0; mB_ = 0; }   // (mB stays: the late entries are still listed; only their bytes are not gathered)
    if (mB_) {
        k_padded_lengths<<<div_up(mB, 256), 256, 0, st>>>(idx.p + mA, mB, s->lengths.p, s->block_at_rank.p, plen.p); IPCFP_LAUNCH_CHECK();
        exclusive_scan_u32(plen.p, offs.p + mA, mB, (uint64_t*)(dw + DW_WIT_B_BYTES), scratch.p, st);
    }
    if (bytesA + bytesB > host_cap) {  // rare: more late blocks than the slack — move to a bigger buffer
        IPCFP_CUDA(cudaStreamSynchronize(st2));
        PinnedArray bigger(s->pool, bytesA + bytesB + 64);
        memcpy(bigger.p, host_blob.p, bytesA);
        host_blob = std::move(bigger);
        host_cap = host_blob.cap;
    }
    AsyncBuf<uint8_t> dblobB(bytesB + 64, st);
    if (mB_) {
        k_witness_copy<<<div_up(mB * 32, 256), 256, 0, st>>>(idx.p + mA, mB, s->view, offs.p + mA, dblobB.p); IPCFP_LAUNCH_CHECK();
        IPCFP_CUDA(cudaMemcpyAsync((uint8_t*)host_blob.p + bytesA, dblobB.p, bytesB, cudaMemcpyDeviceToHost, st));
    }
    // index arrays in Cid order
    AsyncBuf<uint32_t> d_lens(m + 8, st), d_idx(m + 8, st);
    AsyncBuf<uint64_t> d_offs(m + 8, st);
    AsyncBuf<uint8_t> d_cids(m * 38 + 64, st);
    if (m) {
        k_witness_emit<<<div_up(m, EMIT_THREADS), EMIT_THREADS, 0, st>>>(idx.p, offs.p, m, mA, bytesA, bitsA.p, word_prefix.p, bitsB.p, word_prefixB.p, s->view, d_cids.p, d_offs.p,
                                                       d_lens.p, d_idx.p, by_ref ? 1 : 0);
        IPCFP_LAUNCH_CHECK();
    }
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_WITNESS_SORTED], st));   // the sorted CID list exists on the device (the multi-GPU union waits for this, not for the copies below)
    out.n = m;
    out.blob_size = bytesA + bytesB;
    out.cids = PinnedArray(s->pool, m * 38 + 64);
    out.offsets = PinnedArray(s->pool, (m + 1) * 8);
    out.lengths = PinnedArray(s->pool, (m + 1) * 4);
    if (want_sorted_idx) out.sorted_idx = PinnedArray(s->pool, (m + 1) * 4);
    if (m) {
        IPCFP_CUDA(cudaMemcpyAsync(out.cids.p, d_cids.p, m * 38, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(out.offsets.p, d_offs.p, m * 8, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(out.lengths.p, d_lens.p, m * 4, cudaMemcpyDeviceToHost, st));
        if (want_sorted_idx) IPCFP_CUDA(cudaMemcpyAsync(out.sorted_idx.p, d_idx.p, m * 4, cudaMemcpyDeviceToHost, st));
    }
    out.cids_dev = std::move(d_cids);
    out.idx_dev = std::move(d_idx);
    dblobB_keep = std::move(dblobB);
}
void WitnessBuilder::finish_join(WitnessOut& out) {
    IPCFP_CUDA(cudaStreamWaitEvent(st, s->ev[EV_BLOB_COPIED], 0));  // the big copy on the side stream
    IPCFP_CUDA(cudaStreamSynchronize(st));
    IPCFP_CUDA(cudaStreamSynchronize(st2));
    out.blob = std::move(host_blob);
}

// single-phase convenience (storage path, bundle union): everything at once
void materialize_witness(Store* s, const uint32_t* wbits_dev, WitnessOut& out, bool by_ref) {
    WitnessBuilder wb(s);
    wb.by_ref = by_ref;
    wb.snapshot(wbits_dev);
    publish_words(s, DW_WIT_A, 2);
    IPCFP_CUDA(cudaStreamSynchronize(s->stream));
    const uint64_t* hw = s->host_words.p;
    wb.start_copy(hw[DW_WIT_A], hw[DW_WIT_A_BYTES], hw[DW_WIT_A], hw[DW_WIT_A_BYTES]);   // one part
    wb.finish(0, 0, out, true);
}

// bit rank_of[idx[i]] of the union bitmap for every entry of one witness list (lists overlap: atomicOr)
__global__ void k_union_mark(const uint32_t* __restrict__ idx, uint64_t m, const uint32_t* __restrict__ rank_of, uint32_t* bits) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint32_t r = rank_of[idx[i]];
    atomicOr(bits + (r >> 5), 1u << (r & 31));
}
// Every entry's block is the one its lookup marked (equal CIDs resolve to one block of the store), so equal CIDs of different lists set one
// bit, and reading the bitmap in bit order is `Cid` order for any number of CID prefixes.
void witness_union(Store* s, const std::vector<const WitnessOut*>& lists, WitnessOut& out, bool by_ref) {
    cudaStream_t st = s->stream;
    AsyncBuf<uint32_t> bits((s->n + 31) / 32 + 8, st);
    bits.zero();
    for (const WitnessOut* w : lists)
        if (w->n) { k_union_mark<<<div_up(w->n, 256), 256, 0, st>>>(w->idx_dev.p, w->n, s->rank_of.p, bits.p); IPCFP_LAUNCH_CHECK(); }
    materialize_witness(s, bits.p, out, by_ref);
}

}  // namespace ipcfp
