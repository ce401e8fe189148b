// shard_kernels.cuh — the kernels of the cross-shard protocol (parallel.cu, DESIGN.md §6: stages X, P, F and W) and the host rules
// that size their buffers. Nothing here talks to NCCL: parallel.cu enqueues these kernels around its collectives, and
// tests/gpu_prims/shard_check.cu drives the same kernels for W simulated ranks on one device, its collectives replaced by copies.
#pragma once
#include <algorithm>

#include "../../include/ipcfp.h"
#include "common.cuh"
#include "rawcid.cuh"

namespace ipcfp {

struct ExecEntry { RawCid c; uint64_t pos; };  // 48 bytes

// ------------------------------------------------------------------------------------------ exchange kernels
#define XSEG_HDR 48   // a segment = [count u64, 40 bytes pad][cap entries of 48 bytes]

// counts per owner from the first sorted position of every owner (nseg where an owner has no entry); writes the segment headers
__global__ void k_exec_seg_headers(const unsigned long long* __restrict__ start, uint64_t nseg, uint32_t world, uint64_t cap, uint8_t* send,
                                   unsigned long long* overflow) {
    if (threadIdx.x || blockIdx.x) return;
    unsigned long long next = nseg;
    for (int r = (int)world - 1; r >= 0; r--) {
        unsigned long long cnt = 0;
        if (start[r] != nseg) { cnt = next - start[r]; next = start[r]; }
        if (cnt > cap) { *overflow = 1; cnt = cap; }
        *(unsigned long long*)(send + (uint64_t)r * (XSEG_HDR + cap * 48)) = cnt;
    }
}
__global__ void k_exec_scatter_seg(const RawCid* __restrict__ seg, const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint64_t nseg,
                                   uint64_t pos0, const unsigned long long* __restrict__ start, uint64_t cap, uint8_t* send) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nseg) return;
    uint32_t owner = keys[j], src = vals[j];
    uint64_t slot = j - start[owner];
    if (slot < cap) {
        ExecEntry e; e.c = seg[src]; e.pos = pos0 + src;
        *(ExecEntry*)(send + (uint64_t)owner * (XSEG_HDR + cap * 48) + XSEG_HDR + slot * 48) = e;
    }
}
// ---- order-preserving partition by owner in three kernels (count per warp run → one scan → scatter), no key / value arrays ----
#define XB_RUN 256u   // consecutive entries one warp handles (8 chunks of 32)
__device__ __forceinline__ uint32_t exec_owner_of(const RawCid& c, uint32_t world) { return (uint32_t)((rawcid_hash(c) >> 32) % world); }
// cnt[owner * nruns + run] = entries of that owner in run `run` of the slice
__global__ void __launch_bounds__(128) k_xb_count(const RawCid* __restrict__ seg, uint64_t nseg, uint32_t world, uint32_t nruns, uint32_t* cnt) {
    const uint32_t run = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (run >= nruns) return;
    const uint64_t base = (uint64_t)run * XB_RUN;
    uint32_t mine = 0;                                   // lane o (< 32) accumulates owner o; world > 32: lanes take owners o, o+32, … in turn
    for (uint32_t c = 0; c < XB_RUN / 32; c++) {
        const uint64_t i = base + c * 32 + lane;
        const uint32_t o = i < nseg ? exec_owner_of(seg[i], world) : 0xffffffffu;
        for (uint32_t ob = 0; ob < world; ob += 32) {
            uint32_t add = 0;
            for (uint32_t k = 0; k < 32 && ob + k < world; k++) { uint32_t b = __ballot_sync(0xffffffffu, o == ob + k); if (lane == k) add = (uint32_t)__popc(b); }
            if (ob == 0) mine += add;
            else if (ob + lane < world && add) atomicAdd(&cnt[(uint64_t)(ob + lane) * nruns + run], add);   // rare: world > 32
        }
    }
    if (lane < world) cnt[(uint64_t)lane * nruns + run] = mine + (world > 32 ? cnt[(uint64_t)lane * nruns + run] : 0u);
}
// segment headers: count per owner from the scan (scan[o * nruns] = entries of all owners before o)
__global__ void k_xb_headers(const uint64_t* __restrict__ scan, const uint64_t* __restrict__ total, uint32_t world, uint32_t nruns, uint64_t cap, uint8_t* send,
                             unsigned long long* overflow) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= world) return;
    const uint64_t a = scan[(uint64_t)o * nruns], b = o + 1 < world ? scan[(uint64_t)(o + 1) * nruns] : *total;
    unsigned long long c = b - a;
    if (c > cap) { *overflow = 1; c = cap; }
    *(unsigned long long*)(send + (uint64_t)o * (XSEG_HDR + cap * 48)) = c;
}
// entries leave in (owner, position) order: slot = entries of that owner in earlier runs + earlier ones of this run
__global__ void __launch_bounds__(128) k_xb_scatter(const RawCid* __restrict__ seg, uint64_t nseg, uint64_t pos0, uint32_t world, uint32_t nruns,
                                                   const uint64_t* __restrict__ scan, uint64_t cap, uint8_t* send) {
    __shared__ uint32_t s_run[4][256];
    const uint32_t run = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    if (run >= nruns) return;
    for (uint32_t o = lane; o < world; o += 32) s_run[wib][o] = 0;
    __syncwarp();
    const uint64_t base = (uint64_t)run * XB_RUN;
    for (uint32_t c = 0; c < XB_RUN / 32; c++) {
        const uint64_t i = base + c * 32 + lane;
        const bool valid = i < nseg;
        RawCid rc{};
        uint32_t o = 0xffffffffu;
        if (valid) { rc = seg[i]; o = exec_owner_of(rc, world); }
        const unsigned m = __match_any_sync(0xffffffffu, o);
        if (valid) {
            const uint32_t rank = (uint32_t)__popc(m & ((1u << lane) - 1u));
            const uint64_t slot = scan[(uint64_t)o * nruns + run] - scan[(uint64_t)o * nruns] + s_run[wib][o] + rank;
            if (slot < cap) {
                ExecEntry e; e.c = rc; e.pos = pos0 + i;
                *(ExecEntry*)(send + (uint64_t)o * (XSEG_HDR + cap * 48) + XSEG_HDR + slot * 48) = e;
            }
        }
        __syncwarp();
        if (valid && (m & ((1u << lane) - 1u)) == 0) s_run[wib][o] += (uint32_t)__popc(m);   // first lane of every owner group
        __syncwarp();
    }
}

// seg_off[0..world] from the received segment headers
__global__ void k_recv_offsets(const uint8_t* __restrict__ recv, uint32_t world, uint64_t cap, uint64_t* seg_off) {
    if (threadIdx.x || blockIdx.x) return;
    uint64_t run = 0;
    for (uint32_t r = 0; r < world; r++) {
        seg_off[r] = run;
        uint64_t c = *(const unsigned long long*)(recv + (uint64_t)r * (XSEG_HDR + cap * 48));
        run += c > cap ? cap : c;
    }
    seg_off[world] = run;
}
__device__ __forceinline__ const ExecEntry* recv_entry_seg(const uint8_t* recv, const uint64_t* seg_off, uint32_t world, uint64_t cap, uint64_t k) {
    uint32_t r = 0;
    while (r + 1 < world && k >= seg_off[r + 1]) r++;
    return (const ExecEntry*)(recv + (uint64_t)r * (XSEG_HDR + cap * 48) + XSEG_HDR) + (k - seg_off[r]);
}
// one canonical slot per distinct CID holding the smallest entry ordinal (= smallest global position: segments arrive in rank
// order and are position-ordered inside)
__global__ void k_exec_claim_seg(const uint8_t* __restrict__ recv, const uint64_t* __restrict__ seg_off, uint32_t world, uint64_t cap,
                                 unsigned long long* table, uint64_t mask) {
    uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= seg_off[world]) return;
    const ExecEntry* e = recv_entry_seg(recv, seg_off, world, cap, k);
    uint64_t h = rawcid_hash(e->c);
    uint32_t fp = (uint32_t)(h >> 40) | 1u;
    unsigned long long mine = ((unsigned long long)fp << 32) | (unsigned long long)(k + 1);
    uint64_t slot = h & mask;
    for (;;) {
        unsigned long long v = table[slot];
        if (v == 0) { v = atomicCAS(&table[slot], 0ull, mine); if (v == 0) return; }
        if ((uint32_t)(v >> 32) == fp && rawcid_eq(recv_entry_seg(recv, seg_off, world, cap, (uint32_t)v - 1)->c, e->c)) { atomicMin(&table[slot], mine); return; }
        slot = (slot + 1) & mask;
    }
}
// every entry that is not the first occurrence of its CID sets the bit of its global position
__global__ void k_exec_mark_dups(const uint8_t* __restrict__ recv, const uint64_t* __restrict__ seg_off, uint32_t world, uint64_t cap,
                                 const unsigned long long* __restrict__ table, uint64_t mask, uint32_t* bitmap) {
    uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= seg_off[world]) return;
    const ExecEntry* e = recv_entry_seg(recv, seg_off, world, cap, k);
    uint64_t h = rawcid_hash(e->c);
    uint32_t fp = (uint32_t)(h >> 40) | 1u;
    uint64_t slot = h & mask;
    for (;;) {
        unsigned long long v = table[slot];
        if (v == 0) return;   // cannot happen: every entry was claimed
        if ((uint32_t)(v >> 32) == fp && rawcid_eq(recv_entry_seg(recv, seg_off, world, cap, (uint32_t)v - 1)->c, e->c)) {
            if ((uint32_t)v - 1 != (uint32_t)k) atomicOr(&bitmap[e->pos >> 5], 1u << (e->pos & 31));
            return;
        }
        slot = (slot + 1) & mask;
    }
}
// zero bits per word of the duplicate bitmap (positions past nraw do not count)
__global__ void k_zero_counts(const uint32_t* __restrict__ bitmap, uint64_t nraw, uint32_t* zeros) {
    uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t nwords = (nraw + 31) / 32;
    if (w >= nwords) return;
    uint32_t valid = (w == nwords - 1 && (nraw & 31)) ? ((1u << (nraw & 31)) - 1u) : 0xffffffffu;
    zeros[w] = (uint32_t)__popc(~bitmap[w] & valid);
}
// exec index i of every matching receipt → raw position of the (i+1)-th zero bit (UINT64_MAX past the end)
__global__ void k_select_positions(const uint32_t* __restrict__ match_rel, uint64_t n_match, uint64_t lo, const uint32_t* __restrict__ bitmap,
                                   const uint64_t* __restrict__ zprefix, uint64_t nwords, const unsigned long long* __restrict__ n_exec,
                                   uint64_t* out) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_match) return;
    const uint64_t i = lo + match_rel[t];
    if (i >= *n_exec) { out[t] = ~0ull; return; }
    uint64_t a = 0, b = nwords;            // largest w with zprefix[w] <= i
    while (b - a > 1) { uint64_t m = (a + b) >> 1; if (zprefix[m] <= i) a = m; else b = m; }
    uint32_t x = ~bitmap[a];
    uint32_t k = (uint32_t)(i - zprefix[a]);
    for (uint32_t j = 0; j < k; j++) x &= x - 1;
    out[t] = a * 32 + (uint64_t)(__ffs((int)x) - 1);
}
__global__ void k_fetch_positions(const RawCid* __restrict__ seg, uint64_t nseg, uint64_t pos0, const uint64_t* __restrict__ req, uint64_t n, RawCid* out) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    uint64_t p = req[j];
    RawCid z{};
    out[j] = (p >= pos0 && p - pos0 < nseg) ? seg[p - pos0] : z;
}
// EventProof.message_cid = exec[exec_index] (events/generator.rs:245, :289): answers are in the order of the matching list
__global__ void k_patch_message_cids(ipcfp_event_proof* proofs, uint64_t n_proofs, const uint32_t* __restrict__ match_rel, uint64_t n_match, uint64_t lo,
                                     const RawCid* __restrict__ answers) {
    uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_proofs) return;
    const uint64_t i = proofs[k].exec_index;
    if (i == 0xFFFFFFFFFFFFFFFFull || i < lo) return;
    const uint32_t rel = (uint32_t)(i - lo);
    uint64_t a = 0, b = n_match;
    while (b - a > 1) { uint64_t m = (a + b) >> 1; if (match_rel[m] <= rel) a = m; else b = m; }
    if (!n_match || match_rel[a] != rel) return;
    const RawCid c = answers[a];
    uint8_t* o = proofs[k].message_cid;
    for (int q = 0; q < 6; q++) o[q] = (uint8_t)(c.w[4] >> (8 * q));
    for (int q = 0; q < 32; q++) o[6 + q] = (uint8_t)(c.w[q >> 3] >> (8 * (q & 7)));
}
// n_exec = nraw − duplicates, published for pass 2 and the host
__global__ void k_set_n_exec(const uint64_t* __restrict__ zprefix_total, unsigned long long* n_exec) { *n_exec = *zprefix_total; }

// ------------------------------------------------------------------------------------------ witness union kernels
// 38-byte CIDs ↔ 40-byte records {digest[32], prefix[6], 0, 0} (aligned words for the merge)
__global__ void k_cids_to_recs(const uint8_t* __restrict__ cids, uint64_t n, uint64_t cap, RawCid* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    RawCid c{};
    if (i < n) {
        const uint8_t* s = cids + 38 * i;
        uint64_t pre = 0;
        for (int q = 0; q < 6; q++) pre |= (uint64_t)s[q] << (8 * q);
        c.w[4] = pre;
        for (int q = 0; q < 32; q++) c.w[q >> 3] |= (uint64_t)s[6 + q] << (8 * (q & 7));
    }
    out[i] = c;
}
__device__ __forceinline__ uint64_t bswap64_p(uint64_t x) {
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | (uint64_t)__byte_perm(hi, 0, 0x0123);
}
// raw byte order of (prefix, digest) — `Cid` Ord for CIDs of one prefix (the Filecoin chain case; the sharded call refuses other stores)
__device__ __forceinline__ int rec_cmp(const RawCid& a, const RawCid& b) {
    uint64_t pa = bswap64_p(a.w[4] << 16), pb = bswap64_p(b.w[4] << 16);
    if (pa != pb) return pa < pb ? -1 : 1;
#pragma unroll
    for (int k = 0; k < 4; k++) { uint64_t x = bswap64_p(a.w[k]), y = bswap64_p(b.w[k]); if (x != y) return x < y ? -1 : 1; }
    return 0;
}
__device__ __forceinline__ uint32_t rec_bucket(const RawCid& a) { return (uint32_t)((a.w[0] & 0xff) << 8 | ((a.w[0] >> 8) & 0xff)); }
#define MERGE_BUCKETS 65536u
// starts[b][B - b0] = first index of list b whose bucket is >= B (B = b0..b0+nb); lists are sorted and hold buckets of [b0, b0+nb) only,
// so every element fills the gap it closes
__global__ void k_merge_starts(const RawCid* __restrict__ lists, const uint64_t* __restrict__ counts, uint32_t world, uint64_t cap, uint32_t* starts,
                               uint32_t b0, uint32_t nb) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (uint64_t)world * cap) return;
    uint32_t b = (uint32_t)(g / cap);
    uint64_t k = g % cap, n = counts[b];
    uint32_t* st = starts + (uint64_t)b * (nb + 1);
    if (n == 0) { if (k == 0) for (uint32_t B = 0; B <= nb; B++) st[B] = 0; return; }
    if (k >= n) return;
    const RawCid* L = lists + (uint64_t)b * cap;
    uint32_t Bk = rec_bucket(L[k]) - b0;
    uint32_t from = k == 0 ? 0 : rec_bucket(L[k - 1]) - b0 + 1;
    for (uint32_t B = from; B <= Bk; B++) st[B] = (uint32_t)k;
    if (k == n - 1) for (uint32_t B = Bk + 1; B <= nb; B++) st[B] = (uint32_t)n;
}
// position of every element in the merged (still non-unique) order + is it the first of its CID
__global__ void k_merge_rank(const RawCid* __restrict__ lists, const uint64_t* __restrict__ counts, uint32_t world, uint64_t cap,
                             const uint32_t* __restrict__ starts, uint32_t* pos_of, uint32_t* keep, uint32_t b0, uint32_t nb) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (uint64_t)world * cap) return;
    uint32_t b = (uint32_t)(g / cap);
    uint64_t k = g % cap;
    if (k >= counts[b]) return;
    const RawCid e = lists[(uint64_t)b * cap + k];
    const uint32_t B = rec_bucket(e) - b0;
    uint64_t pos = 0;
    bool dup = false;
    for (uint32_t q = 0; q < world; q++) {
        const uint32_t* st = starts + (uint64_t)q * (nb + 1);
        uint32_t s0 = st[B], s1 = st[B + 1];
        pos += s0;
        if (q == b) { pos += k - s0; continue; }
        const RawCid* L = lists + (uint64_t)q * cap;
        for (uint32_t x = s0; x < s1; x++) {
            int c = rec_cmp(L[x], e);
            if (c < 0 || (c == 0 && q < b)) pos++;
            if (c == 0 && q < b) dup = true;
            if (c > 0) break;
        }
    }
    pos_of[g] = (uint32_t)pos;
    keep[pos] = dup ? 0u : 1u;
}
__global__ void k_merge_emit38(const RawCid* __restrict__ lists, const uint64_t* __restrict__ counts, uint32_t world, uint64_t cap,
                               const uint32_t* __restrict__ pos_of, const uint32_t* __restrict__ keep, const uint64_t* __restrict__ outidx, uint8_t* out) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (uint64_t)world * cap) return;
    uint32_t b = (uint32_t)(g / cap);
    uint64_t k = g % cap;
    if (k >= counts[b]) return;
    uint32_t pos = pos_of[g];
    if (!keep[pos]) return;
    const RawCid c = lists[(uint64_t)b * cap + k];
    uint8_t* o = out + 38ull * outidx[pos];
    for (int q = 0; q < 6; q++) o[q] = (uint8_t)(c.w[4] >> (8 * q));
    for (int q = 0; q < 32; q++) o[6 + q] = (uint8_t)(c.w[q >> 3] >> (8 * (q & 7)));
}

// ---- partitioned union: rank r owns the CIDs whose bucket (first two digest bytes) lies in [part_lo(r), part_lo(r+1))
__host__ __device__ __forceinline__ uint32_t part_lo(uint32_t r, uint32_t world) { return (uint32_t)(((uint64_t)r * MERGE_BUCKETS + world - 1) / world); }
// One CTA: bounds[r] = first index of the sorted local list whose bucket is >= part_lo(r) (r = 0..world); the header record of piece r
// in the send buffer (piece stride = cap + 1 records) receives min(piece length, cap); *overflow = 1 when a piece does not fit.
__global__ void k_part_bounds(const RawCid* __restrict__ list, uint64_t n, uint32_t world, uint64_t cap, uint64_t* bounds, RawCid* send, unsigned long long* overflow) {
    __shared__ uint64_t b[1025];
    for (uint32_t r = threadIdx.x; r <= world; r += blockDim.x) {
        const uint32_t want = part_lo(r, world);
        uint64_t lo = 0, hi = n;
        while (lo < hi) { uint64_t mid = (lo + hi) >> 1; if (rec_bucket(list[mid]) < want) lo = mid + 1; else hi = mid; }
        b[r] = r == world ? n : lo;
        bounds[r] = b[r];
    }
    if (threadIdx.x == 0) *overflow = 0;
    __syncthreads();
    for (uint32_t r = threadIdx.x; r < world; r += blockDim.x) {
        const uint64_t cnt = b[r + 1] - b[r];
        RawCid h{};
        h.w[0] = cnt < cap ? cnt : cap;
        send[(uint64_t)r * (cap + 1)] = h;
        if (cnt > cap) *overflow = 1;
    }
}
// entry i of the sorted local list → its place in the piece of the rank that owns its bucket
__global__ void k_part_pack(const RawCid* __restrict__ list, uint64_t n, uint32_t world, uint64_t cap, const uint64_t* __restrict__ bounds, RawCid* send) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const RawCid e = list[i];
    const uint32_t dst = (uint32_t)(((uint64_t)rec_bucket(e) * world) >> 16);
    const uint64_t j = i - bounds[dst];
    if (j < cap) send[(uint64_t)dst * (cap + 1) + 1 + j] = e;
}
// piece lengths out of the received headers
__global__ void k_part_counts(const RawCid* __restrict__ recv, uint32_t world, uint64_t cap, uint64_t* counts) {
    for (uint32_t r = threadIdx.x; r < world; r += blockDim.x) counts[r] = recv[(uint64_t)r * (cap + 1)].w[0];
}
// exec.get(i) for every matching receipt against the GLOBAL execution order length (sharded calls: the order spans shards)
__global__ void k_check_exec(const uint32_t* __restrict__ match_rel, uint64_t n_match, uint64_t lo, const unsigned long long* __restrict__ n_exec,
                             unsigned long long* err) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_match) return;
    const uint64_t i = lo + match_rel[t];
    if (i >= *n_exec) report_error(err, ST_PASS2, i, 0 /* DC_MISSING_EXEC, ranked before every other code at the same receipt */, 0);
}

// ------------------------------------------------------------------------------------------ buffer sizes (host)
// X: entries per (sender, owner) segment; a sender with more entries for one owner raises the exchange's overflow word
static inline uint64_t exec_seg_cap(uint64_t max_nseg, uint32_t world) { return max_nseg / world + max_nseg / (4 * world) + 1024; }
// X: the owner's claim table, at most half full: the smallest power of two >= 64 and >= 2 * world * cap
static inline uint64_t exec_table_slots(uint32_t world, uint64_t cap) {
    uint64_t slots = 64;
    while (slots < 2 * (world * cap)) slots <<= 1;
    return slots;
}
// W, partitioned: the default piece slot (records) for lists of at most nw_max CIDs; a balanced list always fits, a skewed one may
// overflow and is retried with nw_max + 1
static inline uint64_t union_piece_cap_default(uint64_t nw_max, uint32_t world) {
    return std::min<uint64_t>(nw_max + 1, 2 * ((nw_max + world - 1) / world) + 1024);
}

}  // namespace ipcfp
