// prims.cu — scan / bitmap compaction / radix sort kernels and the CID sort built on them (see prims.cuh).
#include <algorithm>
#include <cstring>

#include "prims.cuh"

namespace ipcfp {

// ------------------------------------------------------------------------------------------ scan
static constexpr int SCAN_THREADS = 512;
static constexpr int SCAN_ITEMS = 4;
static constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

struct LoadIdentity { __device__ __forceinline__ uint32_t operator()(const uint32_t* in, uint64_t i) const { return in[i]; } };
struct LoadPopc { __device__ __forceinline__ uint32_t operator()(const uint32_t* in, uint64_t i) const { return (uint32_t)__popc(in[i]); } };

__device__ __forceinline__ uint64_t block_exclusive_scan(uint64_t v, uint64_t* total) {
    __shared__ uint64_t warp_sums[SCAN_THREADS / 32];
    __shared__ uint64_t block_total;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint64_t s = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
        uint64_t t = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint64_t y = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += y;
        }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = t - s;
        if (lane == 31) block_total = t;
    }
    __syncthreads();
    uint64_t res = warp_sums[warp] + x - v;
    if (total) *total = block_total;
    __syncthreads();
    return res;
}

template <class Load> __global__ void __launch_bounds__(SCAN_THREADS) k_scan_reduce(const uint32_t* in, uint64_t n, uint64_t* block_sums, Load load) {
    uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_ITEMS;
    uint64_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) if (base + k < n) s += load(in, base + k);
    uint64_t tot;
    block_exclusive_scan(s, &tot);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_block_sums(uint64_t* block_sums, uint64_t nblocks, uint64_t* total_dev) {
    uint64_t carry = 0;
    for (uint64_t base = 0; base < nblocks; base += SCAN_THREADS) {
        uint64_t i = base + threadIdx.x;
        uint64_t v = i < nblocks ? block_sums[i] : 0;
        uint64_t tot;
        uint64_t ex = block_exclusive_scan(v, &tot);
        if (i < nblocks) block_sums[i] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0 && total_dev) *total_dev = carry;
}
template <class Load> __global__ void __launch_bounds__(SCAN_THREADS) k_scan_final(const uint32_t* in, uint64_t* out, uint64_t n, const uint64_t* block_sums, Load load) {
    uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    uint64_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = base + k < n ? load(in, base + k) : 0; s += v[k]; }
    uint64_t ex = block_exclusive_scan(s, nullptr) + block_sums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
}

// The whole scan in one CTA (n ≤ SCAN_SMALL): tiles in sequence with a running carry — one launch instead of three.
static constexpr uint64_t SCAN_SMALL = 8 * SCAN_TILE;
template <class Load> __global__ void __launch_bounds__(SCAN_THREADS) k_scan_small(const uint32_t* in, uint64_t* out, uint64_t n, uint64_t* total_dev, Load load) {
    uint64_t carry = 0;
    for (uint64_t tile = 0; tile < n; tile += SCAN_TILE) {
        uint64_t base = tile + (uint64_t)threadIdx.x * SCAN_ITEMS;
        uint32_t v[SCAN_ITEMS];
        uint64_t s = 0;
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = base + k < n ? load(in, base + k) : 0; s += v[k]; }
        uint64_t tot;
        uint64_t ex = block_exclusive_scan(s, &tot) + carry;
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
        carry += tot;
    }
    if (threadIdx.x == 0 && total_dev) *total_dev = carry;
}
// Second kernel of the two-launch scan: every CTA first adds up the tile sums of the tiles before it (≤ SCAN_FUSED_BLOCKS
// values, L2-resident) instead of waiting for a separate single-CTA pass over them.
static constexpr unsigned SCAN_FUSED_BLOCKS = 8192;
template <class Load> __global__ void __launch_bounds__(SCAN_THREADS) k_scan_final_fused(const uint32_t* in, uint64_t* out, uint64_t n, const uint64_t* block_sums,
                                                                                        uint64_t* total_dev, Load load) {
    uint64_t mine = 0;
    for (uint32_t i = threadIdx.x; i < blockIdx.x; i += SCAN_THREADS) mine += block_sums[i];
    uint64_t prefix;
    block_exclusive_scan(mine, &prefix);
    uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    uint64_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = base + k < n ? load(in, base + k) : 0; s += v[k]; }
    uint64_t tot;
    uint64_t ex = block_exclusive_scan(s, &tot) + prefix;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0 && total_dev) *total_dev = prefix + tot;
}

size_t scan_scratch_elems(uint64_t n) { return (size_t)div_up(n, SCAN_TILE) + 1; }

template <class Load> static void scan_impl(const uint32_t* in, uint64_t* out, uint64_t n, uint64_t* total_dev, uint64_t* scratch, cudaStream_t st, Load load) {
    if (n == 0) {
        if (total_dev) IPCFP_CUDA(cudaMemsetAsync(total_dev, 0, 8, st));
        return;
    }
    if (n <= SCAN_SMALL) { k_scan_small<<<1, SCAN_THREADS, 0, st>>>(in, out, n, total_dev, load); IPCFP_LAUNCH_CHECK(); return; }
    unsigned nb = div_up(n, SCAN_TILE);
    k_scan_reduce<<<nb, SCAN_THREADS, 0, st>>>(in, n, scratch, load); IPCFP_LAUNCH_CHECK();
    if (nb <= SCAN_FUSED_BLOCKS) { k_scan_final_fused<<<nb, SCAN_THREADS, 0, st>>>(in, out, n, scratch, total_dev, load); IPCFP_LAUNCH_CHECK(); return; }
    k_scan_block_sums<<<1, SCAN_THREADS, 0, st>>>(scratch, nb, total_dev); IPCFP_LAUNCH_CHECK();
    k_scan_final<<<nb, SCAN_THREADS, 0, st>>>(in, out, n, scratch, load); IPCFP_LAUNCH_CHECK();
}
void exclusive_scan_u32(const uint32_t* in, uint64_t* out, uint64_t n, uint64_t* total_dev, uint64_t* scratch, cudaStream_t st) {
    scan_impl(in, out, n, total_dev, scratch, st, LoadIdentity());
}

// ------------------------------------------------------------------------------------------ bitmap → indices
__global__ void k_bitmap_scatter(const uint32_t* bits, uint64_t nwords, const uint64_t* word_prefix, uint32_t* out) {
    uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwords) return;
    uint32_t x = bits[w];
    uint64_t o = word_prefix[w];
    while (x) {
        int b = __ffs((int)x) - 1;
        out[o++] = (uint32_t)(w * 32 + (uint64_t)b);
        x &= x - 1;
    }
}
void bitmap_to_indices(const uint32_t* bits, uint64_t nbits, uint32_t* out, uint64_t* total_dev, uint64_t* word_prefix, uint64_t* scratch,
                       cudaStream_t st) {
    uint64_t nwords = (nbits + 31) / 32;
    scan_impl(bits, word_prefix, nwords, total_dev, scratch, st, LoadPopc());
    if (nwords == 0) return;
    k_bitmap_scatter<<<div_up(nwords, 256), 256, 0, st>>>(bits, nwords, word_prefix, out); IPCFP_LAUNCH_CHECK();
}

// 64-bit positions
__global__ void k_bitmap_scatter64(const uint32_t* bits, uint64_t nwords, const uint64_t* word_prefix, uint64_t* out) {
    uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwords) return;
    uint32_t x = bits[w];
    uint64_t o = word_prefix[w];
    while (x) {
        int b = __ffs((int)x) - 1;
        out[o++] = w * 32 + (uint64_t)b;
        x &= x - 1;
    }
}
void bitmap_count64(const uint32_t* bits, uint64_t nbits, uint64_t* total_dev, uint64_t* word_prefix, uint64_t* scratch, cudaStream_t st) {
    scan_impl(bits, word_prefix, (nbits + 31) / 32, total_dev, scratch, st, LoadPopc());
}
void bitmap_scatter64(const uint32_t* bits, uint64_t nbits, const uint64_t* word_prefix, uint64_t* out, cudaStream_t st) {
    const uint64_t nwords = (nbits + 31) / 32;
    if (nwords == 0) return;
    k_bitmap_scatter64<<<div_up(nwords, 256), 256, 0, st>>>(bits, nwords, word_prefix, out); IPCFP_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------ radix sort
static constexpr int RS_THREADS = 256;
static constexpr int RS_WARPS = RS_THREADS / 32;
static constexpr int RS_CHUNKS = 8;                        // 32-key chunks per warp
static constexpr int RS_TILE = RS_THREADS * RS_CHUNKS;     // 2048 keys per block

unsigned radix_blocks(uint64_t n) { return n ? div_up(n, RS_TILE) : 1; }

__global__ void __launch_bounds__(RS_THREADS) k_radix_count(const uint32_t* keys, uint64_t n, int shift, uint32_t* ghist, unsigned nblocks) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    uint64_t base = (uint64_t)blockIdx.x * RS_TILE;
#pragma unroll
    for (int c = 0; c < RS_CHUNKS; c++) {
        uint64_t i = base + (uint64_t)c * RS_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255], 1u);
    }
    __syncthreads();
    ghist[(uint64_t)threadIdx.x * nblocks + blockIdx.x] = h[threadIdx.x];
}

__global__ void __launch_bounds__(RS_THREADS) k_radix_scatter(const uint32_t* keys, const uint32_t* vals, uint32_t* okeys, uint32_t* ovals,
                                                              uint64_t n, int shift, const uint64_t* ghist_scanned, unsigned nblocks) {
    __shared__ uint32_t wh[RS_WARPS][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < RS_WARPS * 256; i += RS_THREADS) (&wh[0][0])[i] = 0;
    __syncthreads();
    // each warp owns a CONTIGUOUS run of RS_CHUNKS*32 keys so that warp order == key order
    uint64_t wbase = (uint64_t)blockIdx.x * RS_TILE + (uint64_t)warp * (RS_CHUNKS * 32);
    uint32_t k[RS_CHUNKS];
#pragma unroll
    for (int c = 0; c < RS_CHUNKS; c++) {
        uint64_t i = wbase + (uint64_t)c * 32 + lane;
        k[c] = i < n ? keys[i] : 0;
        if (i < n) atomicAdd(&wh[warp][(k[c] >> shift) & 255], 1u);
    }
    __syncthreads();
    {
        int d = threadIdx.x;  // 256 threads ↔ 256 digits
        uint32_t run = (uint32_t)ghist_scanned[(uint64_t)d * nblocks + blockIdx.x];
#pragma unroll
        for (int w = 0; w < RS_WARPS; w++) { uint32_t t = wh[w][d]; wh[w][d] = run; run += t; }
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < RS_CHUNKS; c++) {
        uint64_t i = wbase + (uint64_t)c * 32 + lane;
        bool valid = i < n;
        unsigned active = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            uint32_t d = (k[c] >> shift) & 255;
            unsigned m = __match_any_sync(active, d);
            uint32_t rank = (uint32_t)__popc(m & ((1u << lane) - 1));
            uint32_t pos = wh[warp][d] + rank;
            okeys[pos] = k[c];
            ovals[pos] = vals[i];
            __syncwarp(active);
            if (rank == 0) wh[warp][d] += (uint32_t)__popc(m);
        }
        __syncwarp();
    }
}

void radix_sort_pairs(uint32_t* keys, uint32_t* vals, uint32_t* keys_alt, uint32_t* vals_alt, uint64_t n, int nbits, uint32_t* hist,
                      uint64_t* scan_tmp, uint64_t* scratch, cudaStream_t st) {
    if (n <= 1) return;
    unsigned nb = radix_blocks(n);
    uint32_t *ki = keys, *vi = vals, *ko = keys_alt, *vo = vals_alt;
    int passes = (nbits + 7) / 8;
    for (int p = 0; p < passes; p++) {
        k_radix_count<<<nb, RS_THREADS, 0, st>>>(ki, n, 8 * p, hist, nb); IPCFP_LAUNCH_CHECK();
        exclusive_scan_u32(hist, scan_tmp, (uint64_t)256 * nb, nullptr, scratch, st);
        k_radix_scatter<<<nb, RS_THREADS, 0, st>>>(ki, vi, ko, vo, n, 8 * p, scan_tmp, nb); IPCFP_LAUNCH_CHECK();
        uint32_t* t;
        t = ki; ki = ko; ko = t;
        t = vi; vi = vo; vo = t;
    }
    if (ki != keys) {
        IPCFP_CUDA(cudaMemcpyAsync(keys, ki, n * 4, cudaMemcpyDeviceToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(vals, vi, n * 4, cudaMemcpyDeviceToDevice, st));
    }
}

// ------------------------------------------------------------------------------------------ CID sort
// radix sort on digest bytes 0-3 (bytes 6-9 of the CID), then the runs of equal keys put in order by all 38 bytes
__global__ void k_merge_keys(const uint8_t* __restrict__ g, uint64_t n, uint32_t* keys, uint32_t* vals, unsigned long long* mixed) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* c = g + 38 * i;
    bool same = true;
#pragma unroll
    for (int k = 0; k < 6; k++) same &= c[k] == g[k];
    if (!same) atomicMin(mixed, (unsigned long long)i);
    keys[i] = ((uint32_t)c[6] << 24) | ((uint32_t)c[7] << 16) | ((uint32_t)c[8] << 8) | c[9];
    vals[i] = (uint32_t)i;
}
__device__ __forceinline__ int cid_cmp_raw(const uint8_t* a, const uint8_t* b) {
    for (int k = 0; k < 38; k++) if (a[k] != b[k]) return a[k] < b[k] ? -1 : 1;
    return 0;
}
__global__ void k_merge_tie_fix(const uint8_t* __restrict__ g, uint32_t* vals, const uint32_t* __restrict__ keys, uint64_t total) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    if (i > 0 && keys[i - 1] == keys[i]) return;
    if (i + 1 >= total || keys[i] != keys[i + 1]) return;
    uint64_t j = i + 1;
    while (j + 1 < total && keys[j + 1] == keys[i]) j++;
    for (uint64_t a = i + 1; a <= j; a++) {
        uint32_t v = vals[a];
        uint64_t b = a;
        while (b > i && cid_cmp_raw(g + 38ull * vals[b - 1], g + 38ull * v) > 0) { vals[b] = vals[b - 1]; b--; }
        vals[b] = v;
    }
}
__global__ void k_merge_unique_flags(const uint8_t* __restrict__ g, const uint32_t* __restrict__ vals, uint64_t total, uint32_t* bits) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool keep = false;
    if (i < total) keep = i == 0 || cid_cmp_raw(g + 38ull * vals[i - 1], g + 38ull * vals[i]) != 0;
    unsigned b = __ballot_sync(0xffffffffu, keep);
    if ((threadIdx.x & 31) == 0) bits[i >> 5] = b;
}
__global__ void k_merge_emit(const uint8_t* __restrict__ g, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ pos, uint64_t n,
                             uint8_t* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* c = g + 38ull * vals[pos[i]];
    for (int k = 0; k < 38; k++) out[38 * i + k] = c[k];
}

uint64_t sort_unique_cids(cudaStream_t st, const void* cids, uint64_t n, void* out, uint64_t* mixed) {
    *mixed = UINT64_MAX;
    if (!n) return 0;
    const uint8_t* g = (const uint8_t*)cids;
    AsyncBuf<uint32_t> keys(n, st), vals(n, st), ka(n, st), va(n, st), bits((n + 31) / 32 + 8, st), pos(n + 32, st);
    unsigned nb = radix_blocks(n);
    AsyncBuf<uint32_t> hist((size_t)256 * nb + 256, st);
    AsyncBuf<uint64_t> scan_tmp((size_t)256 * nb + 256, st), scratch(scan_scratch_elems(std::max<uint64_t>((uint64_t)256 * nb, n)) + 8, st),
        wp((n + 31) / 32 + 8, st), cnt(2, st);   // cnt[0] = unique count, cnt[1] = first mixed-prefix position
    IPCFP_CUDA(cudaMemsetAsync(cnt.p + 1, 0xff, 8, st));
    k_merge_keys<<<div_up(n, 256), 256, 0, st>>>(g, n, keys.p, vals.p, (unsigned long long*)cnt.p + 1); IPCFP_LAUNCH_CHECK();
    radix_sort_pairs(keys.p, vals.p, ka.p, va.p, n, 32, hist.p, scan_tmp.p, scratch.p, st);
    k_merge_tie_fix<<<div_up(n, 256), 256, 0, st>>>(g, vals.p, keys.p, n); IPCFP_LAUNCH_CHECK();
    k_merge_unique_flags<<<div_up((n + 31) / 32 * 32, 256), 256, 0, st>>>(g, vals.p, n, bits.p); IPCFP_LAUNCH_CHECK();
    bitmap_to_indices(bits.p, n, pos.p, cnt.p, wp.p, scratch.p, st);
    uint64_t h[2] = {0, 0};
    IPCFP_CUDA(cudaMemcpyAsync(h, cnt.p, 16, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    *mixed = h[1];
    const uint64_t m = h[0];
    k_merge_emit<<<div_up(m, 256), 256, 0, st>>>(g, vals.p, pos.p, m, (uint8_t*)out); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaStreamSynchronize(st));
    return m;
}

// `Cid` Ord of 38-byte CIDs: (version, codec, multihash code, size) as varints, then the digest bytes
static bool cid_less(const uint8_t* a, const uint8_t* b) {
    uint32_t pa = 0, pb = 0;
    for (int f = 0; f < 4; f++) {
        uint64_t va = 0, vb = 0;
        for (uint32_t sh = 0; pa < 38; sh += 7) { const uint8_t c = a[pa++]; if (sh < 64) va |= (uint64_t)(c & 0x7f) << sh; if (!(c & 0x80)) break; }
        for (uint32_t sh = 0; pb < 38; sh += 7) { const uint8_t c = b[pb++]; if (sh < 64) vb |= (uint64_t)(c & 0x7f) << sh; if (!(c & 0x80)) break; }
        if (va != vb) return va < vb;
    }
    return std::lexicographical_compare(a + pa, a + 38, b + pb, b + 38);
}

void sort_cids_host(std::vector<uint8_t>& cids) {
    const uint64_t m = cids.size() / 38;
    std::vector<uint32_t> ord(m);
    for (uint32_t k = 0; k < m; k++) ord[k] = k;
    const uint8_t* c = cids.data();
    std::stable_sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) { return cid_less(c + 38ull * x, c + 38ull * y); });
    std::vector<uint8_t> sorted(38 * m);
    for (uint64_t k = 0; k < m; k++) memcpy(sorted.data() + 38 * k, c + 38ull * ord[k], 38);
    cids.swap(sorted);
}

}  // namespace ipcfp
