// prims_check.cu — the device-wide primitives of csrc/prims.cu against plain CPU references, called directly (not through the C ABI):
//   exclusive_scan_u32   at the sizes where it changes shape: one CTA (n ≤ 16 384), reduce + fused final (≤ 8 192 tiles of 2 048),
//                        reduce + block sums + final (more); inputs of all 0xFFFFFFFF (64-bit totals past 2^32) and random ones;
//   bitmap_to_indices    nbits not a multiple of 32, empty / full / sparse / alternating bitmaps, word counts across the same limits;
//   radix_sort_pairs     8, 16, 24 and 32 key bits (odd and even pass counts), n across 2 048 (one tile) and 131 072 (the histogram
//                        scan leaves the single CTA); equal, two-valued, top-byte-only, sorted, reverse-sorted and random keys. The
//                        result must be the STABLE sort by the low nbits bits, values being the original indices;
//   sort_unique_cids     one-prefix lists of 14 totals across 2 048 and 131 072, digests clustered on the radix key so that
//                        k_merge_tie_fix orders runs of up to 512, against std::sort (the raw byte order) + unique; lists of several
//                        prefixes: ordered by digest bytes 0-3, then the 38 bytes, the first position of another prefix is reported,
//                        and sort_cids_host of the output is the `Cid` order.
// Every output buffer carries a sentinel past its end that must survive.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr \
//        -o prims_check tests/gpu_prims/prims_check.cu ipc_filecoin_proofs_b200/csrc/prims.cu && ./prims_check
// Prints one "ok: ..." line and exits 0, or names the first disagreement and exits 1.
#include <algorithm>
#include <array>
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

// ------------------------------------------------------------------ sort_unique_cids
typedef std::array<uint8_t, 38> Cid38;
static const uint8_t FILECOIN_PREFIX[6] = {0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};   // CIDv1, dag-cbor, blake2b-256, 32 bytes
// Eight valid CIDv1 prefixes in `Cid` order (version, codec, multihash code, size); the varint code makes their raw byte order differ
// (0x407f = ff 80 01 sorts after 0xb220 = a0 e4 02 bytewise). Index 6 is FILECOIN_PREFIX.
static const uint8_t MIXED_PREFIXES[8][6] = {
    {0x01, 0x55, 0xff, 0xff, 0x01, 0x20}, {0x01, 0x55, 0xa0, 0xe4, 0x02, 0x20}, {0x01, 0x70, 0x81, 0x80, 0x02, 0x20},
    {0x01, 0x71, 0xff, 0x80, 0x01, 0x20}, {0x01, 0x71, 0x80, 0x80, 0x02, 0x20}, {0x01, 0x71, 0x92, 0xe4, 0x02, 0x20},
    {0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20}, {0x01, 0x71, 0xff, 0xff, 0x03, 0x20}};

static Cid38 make_cid(const uint8_t* prefix, const uint8_t* digest) {
    Cid38 c;
    std::copy(prefix, prefix + 6, c.begin());
    std::copy(digest, digest + 32, c.begin() + 6);
    return c;
}
static Cid38 random_cid(const uint8_t* prefix) {
    uint8_t d[32];
    for (auto& b : d) b = (uint8_t)rnd();
    return make_cid(prefix, d);
}
// n digests in clusters that share their first four bytes (the radix key) and differ from byte 4 on: the first clusters hold 512 and 300
// members, the rest 2..64, so runs of equal keys longer and shorter than a warp are put in order by k_merge_tie_fix
static std::vector<Cid38> clustered_pool(uint64_t n) {
    std::vector<Cid38> out;
    for (uint64_t g = 0; out.size() < n; g++) {
        uint8_t t[32];
        for (auto& b : t) b = (uint8_t)rnd();
        const uint64_t size = g == 0 ? 512 : g == 1 ? 300 : 2 + rnd() % 63;
        const uint32_t at = 4 + (uint32_t)(rnd() % 27);   // members differ at bytes at, at + 1
        for (uint64_t k = 0; k < size && out.size() < n; k++) {
            uint8_t d[32];
            std::copy(t, t + 32, d);
            d[at] = (uint8_t)(k >> 8);
            d[at + 1] = (uint8_t)k;
            out.push_back(make_cid(FILECOIN_PREFIX, d));
        }
    }
    return out;
}

// One call of sort_unique_cids on `cids`: ordered by digest bytes 0-3 and then the 38 bytes (within one prefix, the raw byte order) with
// duplicates removed, the first position whose prefix differs from entry 0's (UINT64_MAX: none), nothing written past the unique
// entries; with cid_order, sort_cids_host of the output equals cid_order.
static bool check_cid_sort(const char* what, const std::vector<Cid38>& cids, uint64_t want_mixed, cudaStream_t st,
                           const std::vector<Cid38>* cid_order = nullptr) {
    const uint64_t n = cids.size();
    std::vector<Cid38> ref(cids);
    std::sort(ref.begin(), ref.end(), [](const Cid38& x, const Cid38& y) {
        return std::lexicographical_compare(x.begin() + 6, x.begin() + 10, y.begin() + 6, y.begin() + 10) ||
               (std::equal(x.begin() + 6, x.begin() + 10, y.begin() + 6) && x < y);
    });
    ref.erase(std::unique(ref.begin(), ref.end()), ref.end());
    std::vector<uint8_t> in(38 * n);
    for (uint64_t i = 0; i < n; i++) std::copy(cids[i].begin(), cids[i].end(), in.begin() + 38 * i);
    CheckBuf<uint8_t> d_in(38 * n), d_out(38 * (n + 1));
    if (n) up(d_in.p, in);
    up(d_out.p, std::vector<uint8_t>(38 * (n + 1), 0xA5));
    uint64_t mixed = 0;
    const uint64_t m = sort_unique_cids(st, d_in.p, n, d_out.p, &mixed);
    std::vector<uint8_t> out = down(d_out.p, 38 * (n + 1));
    if (m != ref.size()) FAIL("cid sort n=%llu (%s): %llu unique, expected %zu", (unsigned long long)n, what, (unsigned long long)m, ref.size());
    if (mixed != want_mixed)
        FAIL("cid sort n=%llu (%s): first mixed position %llu, expected %llu", (unsigned long long)n, what, (unsigned long long)mixed,
             (unsigned long long)want_mixed);
    for (uint64_t i = 0; i < m; i++)
        if (!std::equal(ref[i].begin(), ref[i].end(), out.begin() + 38 * i)) FAIL("cid sort n=%llu (%s): entry %llu differs", (unsigned long long)n, what, (unsigned long long)i);
    for (uint64_t b = 38 * m; b < out.size(); b++)
        if (out[b] != 0xA5) FAIL("cid sort n=%llu (%s): wrote past the %llu unique entries", (unsigned long long)n, what, (unsigned long long)m);
    if (cid_order) {
        out.resize(38 * m);
        sort_cids_host(out);
        if (cid_order->size() != m) FAIL("cid sort n=%llu (%s): %llu unique, the `Cid` order has %zu", (unsigned long long)n, what, (unsigned long long)m, cid_order->size());
        for (uint64_t i = 0; i < m; i++)
            if (!std::equal((*cid_order)[i].begin(), (*cid_order)[i].end(), out.begin() + 38 * i))
                FAIL("cid sort n=%llu (%s): entry %llu of sort_cids_host differs from the `Cid` order", (unsigned long long)n, what, (unsigned long long)i);
    }
    g_cases++;
    return true;
}

static bool cid_sorts(cudaStream_t st) {
    // one prefix: totals on both sides of one radix tile (2 048) and of the single-CTA scan of the radix histograms (131 072), drawn with
    // replacement from a pool of 3/4 the total, so duplicates are many
    const uint64_t totals[] = {0, 1, 5, 128, 300, 700, 1792, 2047, 2048, 2049, 2200, 131071, 131072, 131073};
    for (uint64_t n : totals) {
        const std::vector<Cid38> pool = clustered_pool(std::max<uint64_t>(8, n * 3 / 4));
        std::vector<Cid38> cids(n);
        for (auto& c : cids) c = pool[rnd() % pool.size()];
        if (!check_cid_sort("one prefix, clustered digests", cids, UINT64_MAX, st)) return false;
    }
    // several prefixes: sorted and unique all the same, the first differing position reported, `Cid` order by sort_cids_host
    auto cid_order = [](std::vector<Cid38> v) {   // the prefixes' rank in MIXED_PREFIXES, then the digest
        auto rank = [](const Cid38& c) { for (int k = 0; k < 8; k++) if (std::equal(c.begin(), c.begin() + 6, MIXED_PREFIXES[k])) return k; return 8; };
        std::sort(v.begin(), v.end(), [&](const Cid38& x, const Cid38& y) { return rank(x) != rank(y) ? rank(x) < rank(y) : x < y; });
        v.erase(std::unique(v.begin(), v.end()), v.end());
        return v;
    };
    std::vector<Cid38> a(9);
    for (auto& c : a) c = random_cid(FILECOIN_PREFIX);
    const Cid38 odd = random_cid(MIXED_PREFIXES[3]);   // multihash code 0x407f: `Cid` order puts it before every FILECOIN_PREFIX CID
    std::vector<Cid38> l1(a.begin(), a.begin() + 7), l2(a.begin(), a.begin() + 3), l3(1, odd);
    l1.push_back(odd);
    l1.insert(l1.end(), a.begin() + 7, a.end());
    l2.push_back(odd);
    l3.insert(l3.end(), a.begin(), a.end());
    std::vector<Cid38> l4(3000);
    for (uint64_t k = 0; k < l4.size(); k++) l4[k] = random_cid(MIXED_PREFIXES[k % 8]);
    const std::pair<const std::vector<Cid38>*, uint64_t> mixed_cases[] = {{&l1, 7}, {&l2, 3}, {&l3, 1}, {&l4, 1}};
    for (const auto& mc : mixed_cases) {
        const std::vector<Cid38> want = cid_order(*mc.first);
        if (!check_cid_sort("several prefixes", *mc.first, mc.second, st, &want)) return false;
    }
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
        bool ok = scans(st) && bitmaps(st) && sorts(st) && cid_sorts(st);
        IPCFP_CUDA(cudaStreamDestroy(st));
        if (!ok) return 1;
        printf("ok: exclusive_scan_u32, bitmap_to_indices, radix_sort_pairs and sort_unique_cids equal the CPU references in %llu cases\n", (unsigned long long)g_cases);
        return 0;
    } catch (const Error& e) {
        fprintf(stderr, "FAIL: %s\n", e.msg.c_str());
        return 1;
    }
}
