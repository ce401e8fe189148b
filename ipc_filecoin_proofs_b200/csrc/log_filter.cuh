// log_filter.cuh — the log-filter predicate (ipcfp_log_filter, DESIGN.md §3 "Log filters", §4 "Where the log filter lives").
//
// LogFilter is the second instance, beside Matcher, of the predicate the event path is templated over (event_matches, node_events,
// walk_events, StageLane::step, k_pass1_stage, k_pass2, k_plan_match, k_verify_events). Small sets travel inside the struct, which
// the scan kernels take as a kernel argument like Matcher: up to LF_INLINE values per position and LF_INLINE emitters, compared with
// static indices (no local memory). A larger set lives in device memory, sorted, behind a bitmap of 64 bits per value indexed by a
// hash of the value: a miss in the bitmap (almost every event that does not match) costs one load, a hit an exact binary search.
#pragma once
#include <algorithm>
#include <cstring>
#include <vector>
#include "ipld.cuh"

namespace ipcfp {

#define LF_INLINE 4   // values per position / emitters held in the struct itself

struct LogFilter {
    uint32_t npos;                 // n_positions: an event needs at least this many topics
    uint32_t ne;                   // emitters; 0: any
    uint32_t nv[4];                // values at position k; 0: any
    uint32_t lb[5];                // large sets: log2 of the bitmap's bits ([0..3] positions, [4] emitters)
    uint32_t _pad;
    uint64_t emit[LF_INLINE];      // ne ≤ LF_INLINE: the emitters
    uint64_t val[4][LF_INLINE][4]; // nv[k] ≤ LF_INLINE: position k's values, little-endian word loads of the 32 bytes
    const uint64_t* big[5];        // large sets in device memory, ascending: [k] 4 words per value of position k, [4] emitters
    const uint32_t* bits[5];       // their bitmaps
};

__host__ __device__ __forceinline__ uint32_t lf_hash32(const uint64_t w[4], uint32_t lb) {
    const uint64_t x = w[0] ^ (w[1] * 0xff51afd7ed558ccdull) ^ (w[2] * 0xc4ceb9fe1a85ec53ull) ^ (w[3] * 0x9e3779b97f4a7c15ull);
    return (uint32_t)((x * 0x9e3779b97f4a7c15ull) >> (64 - lb));
}
__host__ __device__ __forceinline__ uint32_t lf_hash64(uint64_t e, uint32_t lb) { return (uint32_t)((e * 0x9e3779b97f4a7c15ull) >> (64 - lb)); }
__device__ __forceinline__ bool lf_bit(const uint32_t* bits, uint32_t h) { return (bits[h >> 5] >> (h & 31)) & 1u; }

// lexicographic order of the four words (the host sorts the same way)
__device__ __forceinline__ bool lf_less32(const uint64_t* a, const uint64_t w[4]) {
    if (a[0] != w[0]) return a[0] < w[0];
    if (a[1] != w[1]) return a[1] < w[1];
    if (a[2] != w[2]) return a[2] < w[2];
    return a[3] < w[3];
}

__device__ __forceinline__ bool lf_emitter_ok(const LogFilter& f, uint64_t e) {
    if (f.ne == 0) return true;
    if (f.ne <= LF_INLINE) {
        bool ok = false;
#pragma unroll
        for (uint32_t j = 0; j < LF_INLINE; j++) ok |= j < f.ne && f.emit[j] == e;
        return ok;
    }
    if (!lf_bit(f.bits[4], lf_hash64(e, f.lb[4]))) return false;
    const uint64_t* v = f.big[4];
    uint32_t lo = 0, hi = f.ne;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (v[mid] < e) lo = mid + 1; else hi = mid;
    }
    return lo < f.ne && v[lo] == e;
}

// topic k (its 32 bytes as four words) is in position k's set; k must be a compile-time index after unrolling
__device__ __forceinline__ bool lf_value_ok(const LogFilter& f, uint32_t k, const uint64_t w[4]) {
    const uint32_t n = f.nv[k];
    if (n <= LF_INLINE) {
        bool ok = false;
#pragma unroll
        for (uint32_t j = 0; j < LF_INLINE; j++)
            ok |= j < n && f.val[k][j][0] == w[0] && f.val[k][j][1] == w[1] && f.val[k][j][2] == w[2] && f.val[k][j][3] == w[3];
        return ok;
    }
    if (!lf_bit(f.bits[k], lf_hash32(w, f.lb[k]))) return false;
    const uint64_t* v = f.big[k];
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (lf_less32(v + 4ull * mid, w)) lo = mid + 1; else hi = mid;
    }
    if (lo >= n) return false;
    const uint64_t* q = v + 4ull * lo;
    return q[0] == w[0] && q[1] == w[1] && q[2] == w[2] && q[3] == w[3];
}

// the emitter, the topic count and extract_evm_log's Some: everything but the topic values
__device__ __forceinline__ bool lf_candidate(const LogFilter& f, const EvLog& ev) {
    return ev.some && ev.ntopics >= f.npos && lf_emitter_ok(f, ev.emitter);
}

// the whole predicate on an event decoded from block p
__device__ __forceinline__ bool event_matches(const uint8_t* p, const EvLog& ev, const LogFilter& f) {
    if (!lf_candidate(f, ev)) return false;
    bool ok = true;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        if (ok && k < f.npos && f.nv[k]) {
            const uint8_t* q = p + topic_offset(ev, k);
            const uint64_t w[4] = {load_u64_any(q), load_u64_any(q + 8), load_u64_any(q + 16), load_u64_any(q + 24)};
            ok = lf_value_ok(f, k, w);
        }
    }
    return ok;
}

// A set of filters (ipcfp_verify_event_proofs_any's check_event): an event matches when it matches at least one of f[0..n). The
// structs live in device memory, each pointing at its own large sets.
struct LogFilterAny {
    const LogFilter* f;
    uint32_t n;
};
__device__ __forceinline__ bool event_matches(const uint8_t* p, const EvLog& ev, const LogFilterAny& a) {
    for (uint32_t k = 0; k < a.n; k++)
        if (event_matches(p, ev, a.f[k])) return true;
    return false;
}

// ------------------------------------------------------------------------------------------ host side
// The filter as the kernels take it. The large sets and their bitmaps go into `dev` (one upload); place() points the struct at the
// device copy.
struct LogFilterHost {
    LogFilter f;
    std::vector<uint64_t> dev;     // words: large sets and bitmaps
    uint64_t off_big[5], off_bits[5];

    void place(const uint64_t* d) {
        for (int k = 0; k < 5; k++) {
            f.big[k] = off_big[k] == UINT64_MAX ? nullptr : d + off_big[k];
            f.bits[k] = off_bits[k] == UINT64_MAX ? nullptr : (const uint32_t*)(d + off_bits[k]);
        }
    }
};

inline uint32_t lf_bitmap_lb(uint64_t n) {   // 64 bits per value, at least 4096
    uint32_t lb = 12;
    while ((1ull << lb) < 64 * n) lb++;
    return lb;
}

// ipcfp.h's rules; throws Error(IPCFP_ERR_INVALID_ARG) on a refused filter
inline void log_filter_check(const ipcfp_log_filter* in) {
    if (!in) throw Error(IPCFP_ERR_INVALID_ARG, "null log filter");
    if (in->n_positions > 4) throw Error(IPCFP_ERR_INVALID_ARG, "log filter: n_positions > 4");
    if (in->n_emitters > IPCFP_LOG_FILTER_MAX_EMITTERS) throw Error(IPCFP_ERR_INVALID_ARG, "log filter: more emitters than IPCFP_LOG_FILTER_MAX_EMITTERS");
    if (in->n_emitters && !in->emitters) throw Error(IPCFP_ERR_INVALID_ARG, "log filter: null emitters with a nonzero count");
    for (uint32_t k = 0; k < 4; k++) {
        if (in->n_values[k] && k >= in->n_positions) throw Error(IPCFP_ERR_INVALID_ARG, "log filter: values at a position >= n_positions");
        if (in->n_values[k] > IPCFP_LOG_FILTER_MAX_VALUES) throw Error(IPCFP_ERR_INVALID_ARG, "log filter: more values than IPCFP_LOG_FILTER_MAX_VALUES");
        if (in->n_values[k] && !in->values[k]) throw Error(IPCFP_ERR_INVALID_ARG, "log filter: null values with a nonzero count");
    }
}

// Checks the filter (log_filter_check) and builds it.
inline void log_filter_build(const ipcfp_log_filter* in, LogFilterHost& out) {
    log_filter_check(in);
    LogFilter& f = out.f;
    memset(&f, 0, sizeof f);
    out.dev.clear();
    for (int k = 0; k < 5; k++) out.off_big[k] = out.off_bits[k] = UINT64_MAX;
    f.npos = in->n_positions;
    f.ne = (uint32_t)in->n_emitters;
    auto bitmap = [&](int k, uint32_t lb) {
        out.off_bits[k] = out.dev.size();
        out.dev.resize(out.dev.size() + ((1ull << lb) / 64), 0);
        f.lb[k] = lb;
    };
    auto set_bit = [&](int k, uint32_t h) { ((uint32_t*)(out.dev.data() + out.off_bits[k]))[h >> 5] |= 1u << (h & 31); };
    for (uint32_t k = 0; k < 4; k++) {
        const uint64_t n = in->n_values[k];
        f.nv[k] = (uint32_t)n;
        std::vector<uint64_t> w(4 * n);
        if (n) memcpy(w.data(), in->values[k], 32 * n);
        if (n <= LF_INLINE) {
            for (uint64_t j = 0; j < n; j++) for (int q = 0; q < 4; q++) f.val[k][j][q] = w[4 * j + q];
            continue;
        }
        std::vector<uint32_t> idx(n);
        for (uint32_t j = 0; j < n; j++) idx[j] = j;
        std::sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) {
            return std::lexicographical_compare(&w[4 * a], &w[4 * a + 4], &w[4 * b], &w[4 * b + 4]);
        });
        out.off_big[k] = out.dev.size();
        for (uint32_t j : idx) out.dev.insert(out.dev.end(), &w[4 * j], &w[4 * j + 4]);
        bitmap((int)k, lf_bitmap_lb(n));
        for (uint64_t j = 0; j < n; j++) set_bit((int)k, lf_hash32(&w[4 * j], f.lb[k]));
    }
    if (f.ne <= LF_INLINE) {
        for (uint32_t j = 0; j < f.ne; j++) f.emit[j] = in->emitters[j];
    } else {
        std::vector<uint64_t> e(in->emitters, in->emitters + f.ne);
        std::sort(e.begin(), e.end());
        out.off_big[4] = out.dev.size();
        out.dev.insert(out.dev.end(), e.begin(), e.end());
        bitmap(4, lf_bitmap_lb(f.ne));
        for (uint64_t x : e) set_bit(4, lf_hash64(x, f.lb[4]));
    }
}

// filters[0..n) as the kernels take them, in one upload: n LogFilter structs, then every filter's large sets and bitmaps.
// check() / build() check every filter before any is built (a refused filter's Error carries its position); place(d) writes `words`
// for the device copy at d.
struct LogFilterSet {
    std::vector<LogFilterHost> h;
    std::vector<uint64_t> words;
    static constexpr uint64_t FW = (sizeof(LogFilter) + 7) / 8;   // words per struct

    static void check(const ipcfp_log_filter* in, uint64_t n) {
        if (n && !in) throw Error(IPCFP_ERR_INVALID_ARG, "null log filters");
        for (uint64_t k = 0; k < n; k++) {
            try { log_filter_check(&in[k]); }
            catch (Error& e) { e.index = k; throw; }
        }
    }
    void build(const ipcfp_log_filter* in, uint64_t n) {
        check(in, n);
        h.resize(n);
        uint64_t total = FW * n;
        for (uint64_t k = 0; k < n; k++) { log_filter_build(&in[k], h[k]); total += h[k].dev.size(); }
        words.assign(total, 0);
    }
    void place(const uint64_t* d) {
        uint64_t off = FW * h.size();
        for (size_t k = 0; k < h.size(); k++) {
            h[k].place(d + off);
            memcpy(words.data() + FW * k, &h[k].f, sizeof(LogFilter));
            std::copy(h[k].dev.begin(), h[k].dev.end(), words.begin() + off);
            off += h[k].dev.size();
        }
    }
};

}  // namespace ipcfp
