// common.cuh — shared device/host utilities of the H100 witness-generation engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "../../include/ipcfp.h"

namespace ipcfp {

// ------------------------------------------------------------------ host-side error plumbing
struct Error {
    ipcfp_status status;
    std::string msg;
    uint64_t index;
    Error(ipcfp_status s, std::string m, uint64_t i = UINT64_MAX) : status(s), msg(std::move(m)), index(i) {}
};
void note_launch();  // counts kernel launches (ipcfp_kernel_launch_count)

#define IPCFP_CUDA(expr)                                                                                          \
    do {                                                                                                          \
        cudaError_t _e = (expr);                                                                                  \
        if (_e != cudaSuccess)                                                                                    \
            throw ::ipcfp::Error(IPCFP_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));             \
    } while (0)

#define IPCFP_LAUNCH_CHECK()                                                   \
    do {                                                                       \
        ::ipcfp::note_launch();                                                \
        IPCFP_CUDA(cudaGetLastError());                                        \
    } while (0)

static inline unsigned div_up(uint64_t a, uint64_t b) { return (unsigned)((a + b - 1) / b); }

// Process-wide cache of large device buffers (store.cu): a caller that re-ingests per request creates and destroys a store every
// time, and cudaMalloc / cudaFree of a GB-sized arena are slow, device-synchronising calls. A buffer goes back only after the
// stream that used it has drained (Store::~Store synchronises first).
void* dev_pool_take(size_t bytes, size_t* cap_out);
void dev_pool_give(void* p, size_t cap);

// RAII device buffer
template <class T> struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    size_t pool_cap = 0;   // > 0: the memory belongs to the device pool (alloc_pooled)
    DevBuf() {}
    explicit DevBuf(size_t count) { alloc(count); }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n), pool_cap(o.pool_cap) { o.p = nullptr; o.n = 0; o.pool_cap = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept { if (this != &o) { release(); p = o.p; n = o.n; pool_cap = o.pool_cap; o.p = nullptr; o.n = 0; o.pool_cap = 0; } return *this; }
    ~DevBuf() { release(); }
    void alloc(size_t count) {
        release();
        n = count;
        if (count) IPCFP_CUDA(cudaMalloc((void**)&p, count * sizeof(T)));
    }
    void alloc_pooled(size_t count) {
        release();
        n = count;
        if (count) p = (T*)dev_pool_take(count * sizeof(T), &pool_cap);
    }
    void ensure(size_t count) { if (count > n) alloc(count); }
    void release() {
        if (p) { if (pool_cap) dev_pool_give(p, pool_cap); else cudaFree(p); }
        p = nullptr; n = 0; pool_cap = 0;
    }
    size_t bytes() const { return n * sizeof(T); }
};

// stream-ordered device buffer (cudaMallocAsync pool: no implicit device sync, cached between calls)
template <class T> struct AsyncBuf {
    T* p = nullptr;
    size_t n = 0;
    cudaStream_t st = nullptr;
    AsyncBuf() {}
    AsyncBuf(size_t count, cudaStream_t s) { alloc(count, s); }
    AsyncBuf(const AsyncBuf&) = delete;
    AsyncBuf& operator=(const AsyncBuf&) = delete;
    AsyncBuf(AsyncBuf&& o) noexcept : p(o.p), n(o.n), st(o.st) { o.p = nullptr; o.n = 0; }
    AsyncBuf& operator=(AsyncBuf&& o) noexcept { if (this != &o) { release(); p = o.p; n = o.n; st = o.st; o.p = nullptr; o.n = 0; } return *this; }
    ~AsyncBuf() { release(); }
    void alloc(size_t count, cudaStream_t s) {
        release();
        st = s;
        n = count;
        if (count) IPCFP_CUDA(cudaMallocAsync((void**)&p, count * sizeof(T), s));
    }
    void release() { if (p) cudaFreeAsync(p, st); p = nullptr; n = 0; }
    void zero() { if (p) IPCFP_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), st)); }
};

// pinned host scratch for small read-backs (counters, error words)
template <class T> struct PinnedBuf {
    T* p = nullptr;
    T* dev = nullptr;   // device-side alias of the same (mapped) host memory
    size_t n = 0;
    PinnedBuf() {}
    explicit PinnedBuf(size_t count) { alloc(count); }
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
    void alloc(size_t count) {
        if (p) cudaFreeHost(p);
        p = nullptr; dev = nullptr; n = count;
        if (count) {
            IPCFP_CUDA(cudaHostAlloc((void**)&p, count * sizeof(T), cudaHostAllocMapped));
            IPCFP_CUDA(cudaHostGetDevicePointer((void**)&dev, p, 0));
        }
    }
    void ensure(size_t count) { if (count > n) alloc(count); }
    void swap(PinnedBuf& o) { std::swap(p, o.p); std::swap(dev, o.dev); std::swap(n, o.n); }
};

// ------------------------------------------------------------------ device error word
// Kernels report the FIRST failure in the reference's sequential order through one
// atomicMin on a 64-bit key:  [ stage:8 | index:40 | code:8 | detail:8 ].
// stage numbers follow the order in which the reference would hit the failure.
enum Stage : uint32_t {
    ST_TXMETA = 1, ST_TXAMT = 2, ST_RECEIPTS_ROOT = 3, ST_PASS1 = 4, ST_PASS2 = 5, ST_WITNESS = 6,
    ST_STORAGE = 7, ST_INGEST = 8
};
enum DevCode : uint32_t { DC_MISSING = 1, DC_DECODE = 2, DC_MISSING_EXEC = 3, DC_STATE_MISMATCH = 4, DC_ACTOR_NOT_FOUND = 5, DC_UNSUPPORTED = 6, DC_CID_MISMATCH = 7 };

#define IPCFP_NO_ERROR 0xFFFFFFFFFFFFFFFFull

__host__ __device__ static inline uint64_t err_key(uint32_t stage, uint64_t index, uint32_t code, uint32_t detail) {
    return ((uint64_t)stage << 56) | ((index & 0xFFFFFFFFFFull) << 16) | ((uint64_t)(code & 0xff) << 8) | (detail & 0xff);
}
// Faults of the message-AMT stage (TxMeta blocks, BLS / SECP AMT roots and nodes) have their own word, ordered by WHERE the
// reference's sequential, in-order walk (events/generator.rs:148-177, fvm_ipld_amt for_each) would meet them, so that with several
// independent faults the level-synchronous walk still names the one the reference names:
//   [ eidx:8 | base:44 | 31-level:5 | code:3 | detail:4 ]
// eidx = 3·parent + {0 TxMeta, 1 BLS AMT, 2 SECP AMT}; base = first index below the faulting node (a missing child: the child's);
// level = its height above the leaves (faults of the TxMeta / root header: 31). In-order DFS visits a node after everything with a
// smaller base and, on the left-most path (equal base), parents before children — exactly this key order.
#define IPCFP_TX_EIDX_NONE 0xffu
__host__ __device__ static inline uint64_t tx_err_key(uint32_t eidx, uint64_t base, uint32_t level, uint32_t code, uint32_t detail) {
    const uint64_t b = base > 0xFFFFFFFFFFFull ? 0xFFFFFFFFFFFull : base;
    return ((uint64_t)(eidx & 0xff) << 56) | (b << 12) | ((uint64_t)(31u - (level > 31u ? 31u : level)) << 7) | ((uint64_t)(code & 7) << 4) | (detail & 15);
}
#ifdef __CUDACC__
__device__ static inline void report_error(unsigned long long* word, uint32_t stage, uint64_t index, uint32_t code, uint32_t detail) {
    atomicMin(word, (unsigned long long)err_key(stage, index, code, detail));
}
__device__ static inline void report_tx_error(unsigned long long* word, uint32_t eidx, uint64_t base, uint32_t level, uint32_t code, uint32_t detail) {
    atomicMin(word, (unsigned long long)tx_err_key(eidx, base, level, code, detail));
}
#endif

// ------------------------------------------------------------------ CIDs on the device
// A CID is its 6-byte prefix (class id into a small per-store table) + 32-byte digest.
struct Digest { uint64_t w[4]; };  // raw digest bytes, memory order (w[0] = bytes 0..7 little-endian load)

#ifdef __CUDACC__
__device__ __forceinline__ bool digest_eq(const Digest& a, const Digest& b) {
    return a.w[0] == b.w[0] && a.w[1] == b.w[1] && a.w[2] == b.w[2] && a.w[3] == b.w[3];
}
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return x;
}
__device__ __forceinline__ uint64_t digest_hash(const Digest& d, uint32_t cls) { return mix64(d.w[0] ^ (d.w[2] * 0x9E3779B97F4A7C15ULL) ^ cls); }
// unaligned loads from block bytes
__device__ __forceinline__ uint64_t load_u64_le(const uint8_t* p) {
    uint64_t v = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i);
    return v;
}
// 8 bytes at any alignment with two aligned 8-byte loads (may touch up to 15 bytes past q:
// every buffer the engine reads this way is padded by ≥ 16 bytes)
__device__ __forceinline__ uint64_t load_u64_any(const uint8_t* q) {
    uintptr_t a = (uintptr_t)q;
    const uint64_t* b = (const uint64_t*)(a & ~(uintptr_t)7);
    uint32_t s = (uint32_t)(a & 7) * 8;
    uint64_t x0 = b[0], x1 = b[1];
    return (x0 >> s) | ((x1 << 1) << (63 - s));
}
// 16 bytes at any alignment with three aligned 8-byte loads; the byte shift is one word select
// (shift >= 32 bits) plus four 32-bit funnel shifts (shf.r.wrap takes the shift mod 32)
__device__ __forceinline__ void win_load(const uint8_t* q, uint64_t& w0, uint64_t& w1) {
    uintptr_t a = (uintptr_t)q;
    const uint2* b = (const uint2*)(a & ~(uintptr_t)7);
    uint32_t s = (uint32_t)(a & 7) * 8;
    uint2 x0 = b[0], x1 = b[1], x2 = b[2];
    bool up = (s & 32) != 0;
    uint32_t c0 = up ? x0.y : x0.x, c1 = up ? x1.x : x0.y, c2 = up ? x1.y : x1.x, c3 = up ? x2.x : x1.y, c4 = up ? x2.y : x2.x;
    w0 = (uint64_t)__funnelshift_r(c0, c1, s) | ((uint64_t)__funnelshift_r(c1, c2, s) << 32);
    w1 = (uint64_t)__funnelshift_r(c2, c3, s) | ((uint64_t)__funnelshift_r(c3, c4, s) << 32);
}
__device__ __forceinline__ Digest load_digest(const uint8_t* p) {
    uintptr_t a = (uintptr_t)p;
    const uint64_t* b = (const uint64_t*)(a & ~(uintptr_t)7);
    uint32_t s = (uint32_t)(a & 7) * 8;
    uint64_t x0 = b[0], x1 = b[1], x2 = b[2], x3 = b[3], x4 = b[4];
    Digest d;
    d.w[0] = (x0 >> s) | ((x1 << 1) << (63 - s)); d.w[1] = (x1 >> s) | ((x2 << 1) << (63 - s));
    d.w[2] = (x2 >> s) | ((x3 << 1) << (63 - s)); d.w[3] = (x3 >> s) | ((x4 << 1) << (63 - s));
    return d;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
#endif

}  // namespace ipcfp
