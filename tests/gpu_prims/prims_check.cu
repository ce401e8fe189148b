// prims_check.cu — the device-wide primitives of csrc/prims.cu against plain CPU references, called directly (not through the C ABI):
//   exclusive_scan_u32   at the sizes where it changes shape: one CTA (n ≤ 16 384), reduce + fused final (≤ 8 192 tiles of 2 048),
//                        reduce + block sums + final (more); inputs of all 0xFFFFFFFF (64-bit totals past 2^32) and random ones;
//   bitmap_to_indices    nbits not a multiple of 32, empty / full / sparse / alternating bitmaps, word counts across the same limits;
//   radix_sort_pairs     8, 16, 24 and 32 key bits (odd and even pass counts), n across 2 048 (one tile) and 131 072 (the histogram
//                        scan leaves the single CTA); equal, two-valued, top-byte-only, sorted, reverse-sorted and random keys. The
//                        result must be the STABLE sort by the low nbits bits, values being the original indices.
// Every output buffer carries a sentinel past its end that must survive.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr \
//        -o prims_check tests/gpu_prims/prims_check.cu ipc_filecoin_proofs_b200/csrc/prims.cu && ./prims_check
// Prints one "ok: ..." line and exits 0, or names the first disagreement and exits 1.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <numeric>
#include <vector>

#include "../../ipc_filecoin_proofs_b200/csrc/prims.cuh"

namespace ipcfp {
void note_launch() {}   // the library counts launches in capi.cu; nothing to count here
}  // namespace ipcfp

using namespace ipcfp;

static uint64_t g_rng = 0x5EED5EEDull;
static uint64_t rnd() {
    uint64_t z = (g_rng += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

template <class T> struct CheckBuf {
    T* p = nullptr;
    explicit CheckBuf(size_t n) { IPCFP_CUDA(cudaMalloc(&p, (n ? n : 1) * sizeof(T))); }
    ~CheckBuf() { cudaFree(p); }
    CheckBuf(const CheckBuf&) = delete;
    CheckBuf& operator=(const CheckBuf&) = delete;
};
template <class T> static void up(T* d, const std::vector<T>& h) { IPCFP_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice)); }
template <class T> static std::vector<T> down(const T* d, size_t n) {
    std::vector<T> h(n);
    IPCFP_CUDA(cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost));
    return h;
}

static const uint64_t SENT64 = 0xA5A5A5A5A5A5A5A5ull;
static const uint32_t SENT32 = 0xA5A5A5A5u;
static uint64_t g_cases = 0;

#define FAIL(...)                         \
    do {                                  \
        fprintf(stderr, "FAIL: ");        \
        fprintf(stderr, __VA_ARGS__);     \
        fprintf(stderr, "\n");            \
        return false;                     \
    } while (0)

// ------------------------------------------------------------------ exclusive_scan_u32
static bool check_scan(uint64_t n, const char* what, const std::vector<uint32_t>& in, cudaStream_t st) {
    CheckBuf<uint32_t> d_in(n);
    CheckBuf<uint64_t> d_out(n + 1), d_total(1), d_scratch(scan_scratch_elems(n));
    if (n) up(d_in.p, in);
    std::vector<uint64_t> sent(n + 1, SENT64);
    up(d_out.p, sent);
    IPCFP_CUDA(cudaMemcpy(d_total.p, &SENT64, 8, cudaMemcpyHostToDevice));
    exclusive_scan_u32(d_in.p, d_out.p, n, d_total.p, d_scratch.p, st);
    IPCFP_CUDA(cudaStreamSynchronize(st));
    std::vector<uint64_t> out = down(d_out.p, n + 1);
    uint64_t total = down(d_total.p, 1)[0];
    uint64_t run = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (out[i] != run) FAIL("scan n=%llu (%s): out[%llu] = %llu, expected %llu", (unsigned long long)n, what, (unsigned long long)i,
                                (unsigned long long)out[i], (unsigned long long)run);
        run += in[i];
    }
    if (out[n] != SENT64) FAIL("scan n=%llu (%s): wrote past the end", (unsigned long long)n, what);
    if (total != run) FAIL("scan n=%llu (%s): total %llu, expected %llu", (unsigned long long)n, what, (unsigned long long)total, (unsigned long long)run);
    g_cases++;
    return true;
}

static bool scans(cudaStream_t st) {
    const uint64_t sizes[] = {0, 1, 2047, 2048, 2049, 16384, 16385, 8192ull * 2048, 8192ull * 2048 + 1, 40000000};
    for (uint64_t n : sizes) {
        std::vector<uint32_t> in(n, 0xFFFFFFFFu);
        if (!check_scan(n, "all 0xFFFFFFFF", in, st)) return false;
        for (auto& x : in) x = (uint32_t)rnd();
        if (!check_scan(n, "random", in, st)) return false;
        for (auto& x : in) x = rnd() % 4 == 0 ? (uint32_t)(rnd() % 5) : 0;
        if (!check_scan(n, "sparse small", in, st)) return false;
    }
    return true;
}

// ------------------------------------------------------------------ bitmap_to_indices
// Bits at positions ≥ nbits of the last word are clear (the callers allocate and clear whole words).
static bool check_bitmap(uint64_t nbits, const char* what, std::vector<uint32_t> bits, cudaStream_t st) {
    const uint64_t nwords = (nbits + 31) / 32;
    if (nbits % 32) bits[nwords - 1] &= (1u << (nbits % 32)) - 1;
    std::vector<uint32_t> ref;
    for (uint64_t w = 0; w < nwords; w++)
        for (uint32_t b = 0; b < 32; b++)
            if (bits[w] >> b & 1) ref.push_back((uint32_t)(w * 32 + b));
    CheckBuf<uint32_t> d_bits(nwords), d_out(ref.size() + 1);
    CheckBuf<uint64_t> d_prefix(nwords), d_total(1), d_scratch(scan_scratch_elems(nwords));
    if (nwords) up(d_bits.p, bits);
    std::vector<uint32_t> sent(ref.size() + 1, SENT32);
    up(d_out.p, sent);
    IPCFP_CUDA(cudaMemcpy(d_total.p, &SENT64, 8, cudaMemcpyHostToDevice));
    bitmap_to_indices(d_bits.p, nbits, d_out.p, d_total.p, d_prefix.p, d_scratch.p, st);
    IPCFP_CUDA(cudaStreamSynchronize(st));
    uint64_t total = down(d_total.p, 1)[0];
    std::vector<uint32_t> out = down(d_out.p, ref.size() + 1);
    if (total != ref.size()) FAIL("bitmap nbits=%llu (%s): count %llu, expected %llu", (unsigned long long)nbits, what, (unsigned long long)total,
                                  (unsigned long long)ref.size());
    for (size_t i = 0; i < ref.size(); i++)
        if (out[i] != ref[i]) FAIL("bitmap nbits=%llu (%s): index %zu is %u, expected %u", (unsigned long long)nbits, what, i, out[i], ref[i]);
    if (out[ref.size()] != SENT32) FAIL("bitmap nbits=%llu (%s): wrote past the last index", (unsigned long long)nbits, what);
    g_cases++;
    return true;
}

static bool bitmaps(cudaStream_t st) {
    // word counts 1, 2, 2 049, 16 384, 16 385, 8 192·2 048 and 8 192·2 048 + 1, each with a partial last word where possible
    const uint64_t sizes[] = {0, 1, 31, 33, 65537, 32ull * 16384 - 3, 32ull * 16384 + 7, 32ull * 8192 * 2048 - 1, 32ull * 8192 * 2048 + 5};
    for (uint64_t nbits : sizes) {
        const uint64_t nwords = (nbits + 31) / 32;
        const bool huge = nwords > 16385;   // the full bitmap of the largest sizes would take 2 GB of indices: alternating covers it
        std::vector<uint32_t> bits(nwords, 0);
        if (!check_bitmap(nbits, "empty", bits, st)) return false;
        for (auto& x : bits) x = rnd() % 64 == 0 ? 1u << (rnd() % 32) : 0;
        if (!check_bitmap(nbits, "sparse", bits, st)) return false;
        for (auto& x : bits) x = 0x55555555u;
        if (!check_bitmap(nbits, "alternating", bits, st)) return false;
        if (!huge) {
            for (auto& x : bits) x = 0xFFFFFFFFu;
            if (!check_bitmap(nbits, "full", bits, st)) return false;
            for (auto& x : bits) x = (uint32_t)rnd();
            if (!check_bitmap(nbits, "random", bits, st)) return false;
        }
    }
    return true;
}

// ------------------------------------------------------------------ radix_sort_pairs
static bool check_sort(uint64_t n, int nbits, const char* what, const std::vector<uint32_t>& keys, cudaStream_t st) {
    const uint32_t mask = nbits >= 32 ? 0xFFFFFFFFu : (1u << nbits) - 1;
    std::vector<uint32_t> idx(n);
    std::iota(idx.begin(), idx.end(), 0u);
    std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return (keys[a] & mask) < (keys[b] & mask); });
    const unsigned nb = radix_blocks(n);
    CheckBuf<uint32_t> k{n + 1}, v{n + 1}, ka{n + 1}, va{n + 1}, hist{(size_t)256 * nb + 256};
    CheckBuf<uint64_t> scan_tmp{(size_t)256 * nb + 256}, scratch{scan_scratch_elems((uint64_t)256 * nb) + 8};
    std::vector<uint32_t> hk(keys), hv(n);
    std::iota(hv.begin(), hv.end(), 0u);
    hk.push_back(SENT32);
    hv.push_back(SENT32);
    up(k.p, hk);
    up(v.p, hv);
    radix_sort_pairs(k.p, v.p, ka.p, va.p, n, nbits, hist.p, scan_tmp.p, scratch.p, st);
    IPCFP_CUDA(cudaStreamSynchronize(st));
    std::vector<uint32_t> ok_ = down(k.p, n + 1), ov = down(v.p, n + 1);
    for (uint64_t i = 0; i < n; i++)
        if (ov[i] != idx[i] || ok_[i] != keys[idx[i]])
            FAIL("radix n=%llu nbits=%d (%s): position %llu holds (key %08x, value %u), the stable sort has (key %08x, value %u)", (unsigned long long)n,
                 nbits, what, (unsigned long long)i, ok_[i], ov[i], keys[idx[i]], idx[i]);
    if (ok_[n] != SENT32 || ov[n] != SENT32) FAIL("radix n=%llu nbits=%d (%s): wrote past the end", (unsigned long long)n, nbits, what);
    g_cases++;
    return true;
}

static bool sorts(cudaStream_t st) {
    const uint64_t sizes[] = {0, 1, 2, 33, 2047, 2048, 2049, 131071, 131072, 131073, 300001, (1u << 20) + 3};
    const int widths[] = {8, 16, 24, 32};
    for (uint64_t n : sizes) {
        for (int nbits : widths) {
            std::vector<uint32_t> keys(n);
            const uint32_t c = (uint32_t)rnd();
            for (auto& x : keys) x = c;
            if (!check_sort(n, nbits, "all equal", keys, st)) return false;
            const uint32_t a = (uint32_t)rnd(), b = (uint32_t)rnd();
            for (auto& x : keys) x = rnd() % 2 ? a : b;
            if (!check_sort(n, nbits, "two values", keys, st)) return false;
            for (auto& x : keys) x = (uint32_t)(rnd() % 256) << 24 | 0x00123456u;
            if (!check_sort(n, nbits, "only the top byte varies", keys, st)) return false;
            for (uint64_t i = 0; i < n; i++) keys[i] = (uint32_t)(i * 2654435761ull >> 7);
            std::sort(keys.begin(), keys.end());
            if (!check_sort(n, nbits, "sorted", keys, st)) return false;
            std::reverse(keys.begin(), keys.end());
            if (!check_sort(n, nbits, "reverse sorted", keys, st)) return false;
            for (auto& x : keys) x = (uint32_t)rnd();
            if (!check_sort(n, nbits, "random", keys, st)) return false;
            for (auto& x : keys) x = (uint32_t)(rnd() % 1000);
            if (!check_sort(n, nbits, "random, many repeats", keys, st)) return false;
        }
    }
    return true;
}

int main() {
    try {
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
            fprintf(stderr, "FAIL: no CUDA device\n");
            return 1;
        }
        cudaStream_t st;
        IPCFP_CUDA(cudaStreamCreate(&st));
        bool ok = scans(st) && bitmaps(st) && sorts(st);
        IPCFP_CUDA(cudaStreamDestroy(st));
        if (!ok) return 1;
        printf("ok: exclusive_scan_u32, bitmap_to_indices and radix_sort_pairs equal the CPU references in %llu cases\n", (unsigned long long)g_cases);
        return 0;
    } catch (const Error& e) {
        fprintf(stderr, "FAIL: %s\n", e.msg.c_str());
        return 1;
    }
}
