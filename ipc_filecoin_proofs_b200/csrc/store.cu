// store.cu — ingest of the flat block set into the device arena, CID hash index build,
// Blake2b-256 CID verification (K1), Blockstore::get/has, batched hash entry points (K1/K2/K2b).
#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <sys/syscall.h>
#include <unistd.h>

#include "engine.cuh"
#include "hashes.cuh"

namespace ipcfp {

// ------------------------------------------------------------------------------------------ NUMA placement of pinned memory
static int gpu_numa_node(int device) {
    static std::mutex mu;
    static std::vector<int> cache;          // per device: -2 unknown, -1 none
    std::lock_guard<std::mutex> g(mu);
    if (device < 0 || device >= 64) return -1;
    if ((int)cache.size() <= device) cache.resize(device + 1, -2);
    if (cache[device] != -2) return cache[device];
    int node = -1;
    char bus[64] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus - 1, device) == cudaSuccess) {
        for (char* c = bus; *c; c++) *c = (char)tolower((unsigned char)*c);
        std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
        if (FILE* f = fopen(path.c_str(), "r")) {
            int v = -1;
            if (fscanf(f, "%d", &v) == 1 && v >= 0 && v < 64) node = v;
            fclose(f);
        }
    } else cudaGetLastError();
    cache[device] = node;
    return node;
}
NumaPrefer::NumaPrefer(int device) {
    if (getenv("IPCFP_NO_NUMA")) return;
    int node = gpu_numa_node(device);
    if (node < 0) return;
    if (syscall(SYS_get_mempolicy, &old_mode, old_mask, 8 * sizeof old_mask, nullptr, 0) != 0) return;
    unsigned long mask = 1ul << node;
    on = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, 8 * sizeof mask + 1) == 0;
}
NumaPrefer::~NumaPrefer() {
    if (!on) return;
    if (old_mode == 0 /* MPOL_DEFAULT */) syscall(SYS_set_mempolicy, 0, nullptr, 0);
    else syscall(SYS_set_mempolicy, old_mode, old_mask, 8 * sizeof old_mask);
}

// ------------------------------------------------------------------------------------------ pinned pool
PinnedPool::~PinnedPool() { for (auto& b : free_list) cudaFreeHost(b.p); }
void* PinnedPool::take(size_t bytes, size_t* cap_out) {
    {
        std::lock_guard<std::mutex> g(mu);
        size_t best = SIZE_MAX, bi = SIZE_MAX;
        for (size_t i = 0; i < free_list.size(); i++)
            if (free_list[i].cap >= bytes && free_list[i].cap < best) { best = free_list[i].cap; bi = i; }
        if (bi != SIZE_MAX && best <= bytes * 4 + (1u << 20)) {
            void* p = free_list[bi].p;
            *cap_out = free_list[bi].cap;
            free_list.erase(free_list.begin() + (long)bi);
            return p;
        }
    }
    size_t cap = bytes < 4096 ? 4096 : bytes + bytes / 8;
    void* p = nullptr;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
    NumaPrefer numa(dev);
    IPCFP_CUDA(cudaMallocHost(&p, cap));
    *cap_out = cap;
    return p;
}
void PinnedPool::give(void* p, size_t cap) {
    std::lock_guard<std::mutex> g(mu);
    free_list.push_back({p, cap});
}

// ------------------------------------------------------------------------------------------ device buffer pool
struct DevPoolEntry { int device; void* p; size_t cap; };
static std::mutex g_dp_mu;
static std::vector<DevPoolEntry> g_dp;
static const size_t DEV_POOL_MAX_ENTRIES = 40;
void* dev_pool_take(size_t bytes, size_t* cap_out) {
    int dev = 0;
    IPCFP_CUDA(cudaGetDevice(&dev));
    {
        std::lock_guard<std::mutex> g(g_dp_mu);
        size_t best = SIZE_MAX, bi = SIZE_MAX;
        for (size_t i = 0; i < g_dp.size(); i++)
            if (g_dp[i].device == dev && g_dp[i].cap >= bytes && g_dp[i].cap < best) { best = g_dp[i].cap; bi = i; }
        if (bi != SIZE_MAX && best <= bytes + bytes / 2 + (1u << 20)) {
            void* p = g_dp[bi].p;
            *cap_out = g_dp[bi].cap;
            g_dp.erase(g_dp.begin() + (long)bi);
            return p;
        }
    }
    size_t cap = bytes + bytes / 16 + 4096;        // a little head-room so that the next, slightly larger store still fits
    void* p = nullptr;
    IPCFP_CUDA(cudaMalloc(&p, cap));
    *cap_out = cap;
    return p;
}
void dev_pool_give(void* p, size_t cap) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); cudaFree(p); return; }
    void* evict = nullptr;
    {
        std::lock_guard<std::mutex> g(g_dp_mu);
        g_dp.push_back(DevPoolEntry{dev, p, cap});
        if (g_dp.size() > DEV_POOL_MAX_ENTRIES) {   // drop the smallest: the big ones are the expensive ones to get back
            size_t si = 0;
            for (size_t i = 1; i < g_dp.size(); i++) if (g_dp[i].cap < g_dp[si].cap) si = i;
            evict = g_dp[si].p;
            g_dp.erase(g_dp.begin() + (long)si);
        }
    }
    if (evict) cudaFree(evict);
}

// mapped counter blocks (host_words) are recycled per device across stores: cudaHostAlloc / cudaFreeHost are
// slow, synchronising calls and a caller that re-ingests per request creates and destroys a store every time
static std::mutex g_hw_mu;
static std::vector<std::pair<int, std::unique_ptr<PinnedBuf<uint64_t>>>> g_hw_cache;
static void host_words_take(int device, PinnedBuf<uint64_t>& out, size_t count) {
    {
        std::lock_guard<std::mutex> g(g_hw_mu);
        for (size_t i = 0; i < g_hw_cache.size(); i++)
            if (g_hw_cache[i].first == device && g_hw_cache[i].second->n >= count) {
                out.swap(*g_hw_cache[i].second);
                g_hw_cache.erase(g_hw_cache.begin() + (long)i);
                return;
            }
    }
    out.alloc(count);
}
static void host_words_give(int device, PinnedBuf<uint64_t>& b) {
    if (!b.p) return;
    std::lock_guard<std::mutex> g(g_hw_mu);
    if (g_hw_cache.size() >= 16) return;   // beyond that the buffer is simply freed by its owner
    std::unique_ptr<PinnedBuf<uint64_t>> keep(new PinnedBuf<uint64_t>());
    keep->swap(b);
    g_hw_cache.emplace_back(device, std::move(keep));
}

Store::~Store() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);     // nothing of this store is in flight when its buffers go back to the pools
    if (stream2) cudaStreamSynchronize(stream2);
    host_words_give(device, host_words);
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
    if (stream2) cudaStreamDestroy(stream2);
}

void check_device(int device) {
    int cnt = 0;
    cudaError_t e = cudaGetDeviceCount(&cnt);
    if (e != cudaSuccess || cnt == 0) {
        cudaGetLastError();
        throw Error(IPCFP_ERR_NO_DEVICE, "no CUDA device: this library has no CPU path");
    }
    if (device < 0 || device >= cnt) throw Error(IPCFP_ERR_INVALID_ARG, "device ordinal out of range");
    IPCFP_CUDA(cudaSetDevice(device));
}

// ------------------------------------------------------------------------------------------ ingest kernels
__global__ void k_extract_digests(const uint8_t* __restrict__ cids, uint32_t n, StoreView v, Digest* digests, uint8_t* cls,
                                  unsigned long long* unknown) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* c = cids + (uint64_t)i * 38;
    int k = cid_class(v, c);
    if (k < 0) { atomicAdd(unknown, 1ull); k = 255; }
    cls[i] = (uint8_t)k;
    digests[i] = load_digest(c + 6);
}

// Insert every block into the open-addressing table. Equal CIDs keep the smallest index
// (the oracle's MemoryBlockstore keeps the first occurrence too).
__global__ void k_build_index(uint32_t n, const Digest* __restrict__ digests, const uint8_t* __restrict__ cls, unsigned long long* table,
                              uint64_t mask) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Digest d = digests[i];
    uint32_t c = cls[i];
    uint64_t h = digest_hash(d, c);
    uint32_t fp = (uint32_t)(h >> 32) | 1u;
    unsigned long long mine = ((unsigned long long)fp << 32) | (unsigned long long)(i + 1);
    uint64_t slot = h & mask;
    for (;;) {
        unsigned long long e = table[slot];
        if (e == 0) {
            e = atomicCAS(&table[slot], 0ull, mine);
            if (e == 0) return;
        }
        if ((uint32_t)(e >> 32) == fp) {
            uint32_t j = (uint32_t)e - 1;
            if (cls[j] == c && digest_eq(digests[j], d)) { atomicMin(&table[slot], mine); return; }
        }
        slot = (slot + 1) & mask;
    }
}

__global__ void k_iota(uint32_t* out, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = i;
}
__global__ void k_invert_perm(const uint32_t* __restrict__ perm, uint32_t n, uint32_t* inv) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) inv[perm[i]] = i;
}
__global__ void k_build_recs(uint32_t n, const Digest* __restrict__ digests, const uint8_t* __restrict__ cls, const uint64_t* __restrict__ offsets,
                             const uint32_t* __restrict__ lengths, BlockRec* recs) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    BlockRec r;
    r.d = digests[i]; r.off = offsets[i]; r.len = lengths[i]; r.cls = cls[i]; r.pad[0] = r.pad[1] = 0;
    recs[i] = r;
}

// K1: Blake2b-256 of every block compared with the digest in its CID (class must be a
// blake2b-256 multihash: code 0xb220; other classes are skipped).
__global__ void __launch_bounds__(128) k_verify_cids(StoreView v, uint32_t lo, uint32_t hi, uint32_t b2b_class_mask, unsigned long long* first_bad) {
    uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hi) return;
    uint32_t c = v.cls[i];
    if (!((b2b_class_mask >> c) & 1)) return;
    uint32_t len;
    const uint8_t* p = store_block(v, i, len);
    Digest d;
    blake2b256(p, len, d);
    if (!digest_eq(d, v.digests[i])) atomicMin(first_bad, (unsigned long long)i);
}

__global__ void k_publish(const unsigned long long* __restrict__ src, unsigned long long* dst, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
    __threadfence_system();
}
void publish_words(Store* s, uint32_t dst_first, uint32_t n_words, const void* src_dev, cudaStream_t stream) {
    const unsigned long long* src = src_dev ? (const unsigned long long*)src_dev : s->dev_words.p + dst_first;
    k_publish<<<div_up(n_words, 64), 64, 0, stream ? stream : s->stream>>>(src, (unsigned long long*)s->host_words.dev + dst_first, n_words);
    IPCFP_LAUNCH_CHECK();
}

__global__ void k_lookup_one(StoreView v, const uint8_t* cid, int32_t* out) { out[0] = store_lookup(v, cid); }

// ------------------------------------------------------------------------------------------ host side
// The arena: ARENA_HEAD zero bytes in front of block 0 (StoreView::blob), the blob_size block bytes, then ARENA_TAIL zero bytes: pass-1
// staging copies whole CH-aligned chunks around the last block.
static const uint64_t ARENA_HEAD = 16, ARENA_TAIL = 32 + 512;

static bool parse_prefix(const uint8_t* p, uint64_t key[4]) {
    size_t pos = 0;
    for (int f = 0; f < 4; f++) {
        uint64_t v = 0;
        int shift = 0;
        for (;;) {
            if (pos >= 6) return false;
            uint8_t c = p[pos++];
            v |= (uint64_t)(c & 0x7f) << shift;
            shift += 7;
            if (!(c & 0x80)) break;
        }
        key[f] = v;
    }
    return pos == 6 && key[3] == 32;
}

static void upload_view(Store* s) {
    if (!s->view_dev.p) s->view_dev.alloc_pooled(1);
    IPCFP_CUDA(cudaMemcpyAsync(s->view_dev.p, &s->view, sizeof(StoreView), cudaMemcpyHostToDevice, s->stream));
}
static void fill_view(Store* s) {
    StoreView& v = s->view;
    v.blob = s->arena.p + ARENA_HEAD;
    v.offsets = s->offsets.p; v.lengths = s->lengths.p; v.digests = s->digests.p; v.cls = s->cls.p; v.table = s->table.p;
    v.recs = s->recs.p;
    v.rank_of = s->rank_of.p; v.block_at_rank = s->block_at_rank.p;
    v.mask = s->table.n - 1;
    v.n = (uint32_t)s->n;
    v.n_classes = (uint32_t)s->class_prefix.size();
    memset(v.class_prefix, 0, sizeof v.class_prefix);
    for (size_t c = 0; c < s->class_prefix.size(); c++) memcpy(v.class_prefix[c], s->class_prefix[c].data(), 6);
}

static void compute_class_ranks(Store* s) {
    size_t nc = s->class_prefix.size();
    std::vector<std::array<uint64_t, 4>> keys(nc);
    for (size_t c = 0; c < nc; c++)
        if (!parse_prefix(s->class_prefix[c].data(), keys[c].data()))
            throw Error(IPCFP_ERR_UNSUPPORTED, "unsupported CID form (need 38-byte CIDv1 with a 32-byte digest)");
    std::vector<uint32_t> order(nc);
    for (size_t c = 0; c < nc; c++) order[c] = (uint32_t)c;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
    s->class_rank.assign(nc, 0);
    for (size_t r = 0; r < nc; r++) s->class_rank[order[r]] = (uint32_t)r;
}

Store* store_shell(int device) {
    check_device(device);
    std::unique_ptr<Store> s(new Store());
    s->device = device;
    {   // one process-wide pinned pool: result buffers are recycled across stores and calls
        static std::mutex pool_mu;
        static std::shared_ptr<PinnedPool> g_pool;
        std::lock_guard<std::mutex> g(pool_mu);
        if (!g_pool) g_pool = std::make_shared<PinnedPool>();
        s->pool = g_pool;
    }
    IPCFP_CUDA(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    for (auto& e : s->ev) IPCFP_CUDA(cudaEventCreate(&e));
    cudaStream_t st = s->stream;
    s->dev_words.alloc_pooled(DW_COUNT);
    host_words_take(device, s->host_words, HW_COUNT);
    {
        cudaMemPool_t mp;
        if (cudaDeviceGetDefaultMemPool(&mp, device) == cudaSuccess) { uint64_t thr = UINT64_MAX; cudaMemPoolSetAttribute(mp, cudaMemPoolAttrReleaseThreshold, &thr); }
    }
    IPCFP_CUDA(cudaMemsetAsync(s->dev_words.p, 0, DW_COUNT * 8, st));
    return s.release();
}

uint8_t* store_alloc_blocks(Store* s, uint64_t n, uint64_t blob_size, DevBuf<uint8_t>& cids_dev, bool zero_blocks) {
    if (n >= 0x7fffffffull) throw Error(IPCFP_ERR_UNSUPPORTED, "more than 2^31 blocks in one store");
    uint8_t* blocks = store_alloc_arena(s, blob_size, zero_blocks);
    store_alloc_index(s, n, cids_dev);
    return blocks;
}

// device allocations
// (from the process-wide device pool: a store created right after one of similar size was destroyed allocates nothing)
uint8_t* store_alloc_arena(Store* s, uint64_t blob_size, bool zero_blocks) {
    cudaStream_t st = s->stream;
    s->blob_size = blob_size;
    s->arena.alloc_pooled(ARENA_HEAD + blob_size + ARENA_TAIL);
    uint8_t* blocks = s->arena.p + ARENA_HEAD;
    if (zero_blocks) {
        IPCFP_CUDA(cudaMemsetAsync(s->arena.p, 0, s->arena.n, st));
    } else {
        IPCFP_CUDA(cudaMemsetAsync(s->arena.p, 0, ARENA_HEAD, st));
        IPCFP_CUDA(cudaMemsetAsync(blocks + blob_size, 0, ARENA_TAIL, st));
    }
    return blocks;
}

void store_alloc_index(Store* s, uint64_t n, DevBuf<uint8_t>& cids_dev) {
    s->n = n;
    s->offsets.alloc_pooled(n + 1);
    s->lengths.alloc_pooled(n + 1);
    s->digests.alloc_pooled(n + 1);
    s->cls.alloc_pooled(n + 1);
    s->recs.alloc_pooled(n + 1);
    s->rank_of.alloc_pooled(n + 1);
    s->block_at_rank.alloc_pooled(n + 1);
    uint64_t slots = 64;
    while (slots < 2 * n) slots <<= 1;
    s->table.alloc_pooled(slots);
    IPCFP_CUDA(cudaMemsetAsync(s->table.p, 0, slots * 8, s->stream));
    cids_dev.alloc_pooled(n * 38 + 16);
}

// Class prefixes, `Cid` ranks, block records and the hash index of the n blocks whose CIDs are at cids_dev (n*38, device) and whose
// offsets / lengths are in the store: everything of the ingest that does not touch block bytes. cids_host: the same CIDs on the host, or
// null (the rare several-prefix path then reads them back). first_prefix: the first CID's 6 prefix bytes (host). Leaves the view
// uploaded; the last synchronisation is the class check's.
static void store_index(Store* s, const uint8_t* cids_dev, const uint8_t* cids_host, const uint8_t* first_prefix, DevBuf<uint8_t>& sort_ws) {
    const uint64_t n = s->n;
    cudaStream_t st = s->stream;
    // CID classes: the first CID's prefix is class 0; anything else is discovered by the kernel
    if (n) { std::array<uint8_t, 6> p0; memcpy(p0.data(), first_prefix, 6); s->class_prefix.push_back(p0); }
    for (int attempt = 0; attempt < 2 && n; attempt++) {
        compute_class_ranks(s);
        fill_view(s);
        unsigned long long* unknown = s->dev_words.p + DW_UNKNOWN_CLASSES;
        IPCFP_CUDA(cudaMemsetAsync(unknown, 0, 8, st));
        k_extract_digests<<<div_up(n, 256), 256, 0, st>>>(cids_dev, (uint32_t)n, s->view, s->digests.p, s->cls.p, unknown);
        IPCFP_LAUNCH_CHECK();
        IPCFP_CUDA(cudaMemcpyAsync(s->host_words.p + DW_UNKNOWN_CLASSES, unknown, 8, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
        if (s->host_words.p[DW_UNKNOWN_CLASSES] == 0) break;
        if (attempt == 1) throw Error(IPCFP_ERR_UNSUPPORTED, "internal: CID classes unresolved");
        // rare path: several CID prefixes in one store — enumerate them on the host
        std::vector<uint8_t> back;
        if (!cids_host) {
            back.resize(n * 38);
            IPCFP_CUDA(cudaMemcpyAsync(back.data(), cids_dev, n * 38, cudaMemcpyDeviceToHost, st));
            IPCFP_CUDA(cudaStreamSynchronize(st));
        }
        const uint8_t* cids = cids_host ? cids_host : back.data();
        for (uint64_t i = 0; i < n; i++) {
            std::array<uint8_t, 6> p;
            memcpy(p.data(), cids + 38 * i, 6);
            if (std::find(s->class_prefix.begin(), s->class_prefix.end(), p) == s->class_prefix.end()) {
                if (s->class_prefix.size() >= IPCFP_MAX_CID_CLASSES) throw Error(IPCFP_ERR_UNSUPPORTED, "too many distinct CID prefixes in one store", i);
                s->class_prefix.push_back(p);
            }
        }
    }
    if (!n) { fill_view(s); }
    if (n) {
        // `Cid` Ord rank of every block (one sort per store, under the blob copy): witness bitmaps are indexed by rank, so that every
        // later call reads its witness out of the bitmap already in BTreeSet<Cid> order
        sort_ws.alloc_pooled(n * 4 + 256 + sort_by_cid_ws_bytes(n));   // released (to the device pool) by the caller: after its final sync
        uint32_t* iota = (uint32_t*)sort_ws.p;
        k_iota<<<div_up(n, 256), 256, 0, st>>>(iota, (uint32_t)n); IPCFP_LAUNCH_CHECK();
        sort_by_cid(s, iota, s->block_at_rank.p, n, sort_ws.p + ((n * 4 + 255) & ~(uint64_t)255));
        k_invert_perm<<<div_up(n, 256), 256, 0, st>>>(s->block_at_rank.p, (uint32_t)n, s->rank_of.p); IPCFP_LAUNCH_CHECK();
        k_build_recs<<<div_up(n, 256), 256, 0, st>>>((uint32_t)n, s->digests.p, s->cls.p, s->offsets.p, s->lengths.p, s->recs.p);
        IPCFP_LAUNCH_CHECK();
        k_build_index<<<div_up(n, 256), 256, 0, st>>>((uint32_t)n, s->digests.p, s->cls.p, (unsigned long long*)s->table.p, s->table.n - 1);
        IPCFP_LAUNCH_CHECK();
    }
    upload_view(s);
}

// the classes whose multihash is Blake2b-256 (0xb220): the blocks IPCFP_STORE_VERIFY_CIDS checks
static uint32_t blake2b_class_mask(const Store* s) {
    uint32_t mask = 0;
    for (size_t c = 0; c < s->class_prefix.size(); c++) {
        uint64_t key[4];
        parse_prefix(s->class_prefix[c].data(), key);
        if (key[2] == 0xb220) mask |= 1u << c;
    }
    return mask;
}

void store_finish(Store* s, const uint8_t* cids_dev, const uint8_t* cids_host, const uint8_t* first_prefix, uint32_t flags, const ChunkedCopy* blob,
                  const std::vector<uint64_t>& bounds) {
    cudaStream_t st = s->stream;
    DevBuf<uint8_t> sort_ws;   // released (to the device pool) after the final synchronisation
    store_index(s, cids_dev, cids_host, first_prefix, sort_ws);
    if (!(flags & IPCFP_STORE_VERIFY_CIDS)) {
        if (blob) blob->wait(st, blob->landed.size() - 1);   // the blob must have landed before anything reads blocks
        IPCFP_CUDA(cudaStreamSynchronize(st));
        return;
    }
    const uint32_t mask = blake2b_class_mask(s);
    unsigned long long* bad = s->dev_words.p + DW_FIRST_BAD;
    IPCFP_CUDA(cudaMemsetAsync(bad, 0xff, 8, st));
    const std::vector<uint64_t> all{0, s->n};
    const std::vector<uint64_t>& b = blob ? bounds : all;
    for (size_t k = 0; k + 1 < b.size(); k++) {   // range k is checked while range k + 1 is on the wire
        if (blob) blob->wait(st, k);
        if (b[k + 1] > b[k]) { k_verify_cids<<<div_up(b[k + 1] - b[k], 128), 128, 0, st>>>(s->view, (uint32_t)b[k], (uint32_t)b[k + 1], mask, bad); IPCFP_LAUNCH_CHECK(); }
    }
    publish_words(s, DW_FIRST_BAD, 1);
    IPCFP_CUDA(cudaStreamSynchronize(st));
    s->first_bad = s->host_words.p[DW_FIRST_BAD];   // reported by the C ABI as IPCFP_ERR_CID_MISMATCH (handle stays valid)
}

Store* store_create(const uint8_t* cids, const uint64_t* offsets, const uint32_t* lengths, const uint8_t* blob, uint64_t blob_size, uint64_t n,
                    int device, uint32_t flags) {
    check_device(device);
    if (n >= 0x7fffffffull) throw Error(IPCFP_ERR_UNSUPPORTED, "more than 2^31 blocks in one store");
    if (n && (!cids || !offsets || !lengths || (!blob && blob_size))) throw Error(IPCFP_ERR_INVALID_ARG, "null input array");
    std::unique_ptr<Store> s(store_shell(device));
    cudaStream_t st = s->stream;
    DevBuf<uint8_t> cids_dev;   // released (to the device pool) when this function returns: after its final sync
    uint8_t* blocks = store_alloc_blocks(s.get(), n, blob_size, cids_dev, false);

    // H2D. The CID array goes first so the index build overlaps the (much larger) blob copy.
    if (n) {
        IPCFP_CUDA(cudaMemcpyAsync(cids_dev.p, cids, n * 38, cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(s->offsets.p, offsets, n * 8, cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(s->lengths.p, lengths, n * 4, cudaMemcpyHostToDevice, st));
    }

    // validate offsets / lengths on the host (metadata only); blocks laid out in index order (the usual case) let the blob travel in
    // CHUNKS whose blocks are Blake2b-checked while the next chunk is still on the wire
    bool monotonic = true;
    for (uint64_t i = 0; i < n; i++) {
        if (offsets[i] > blob_size || (uint64_t)lengths[i] > blob_size - offsets[i]) throw Error(IPCFP_ERR_INVALID_ARG, "block out of blob bounds", i);
        if (i && offsets[i] < offsets[i - 1] + lengths[i - 1]) monotonic = false;
    }
    const bool verify = (flags & IPCFP_STORE_VERIFY_CIDS) && n;
    std::vector<uint64_t> bounds{0}, byte_bounds{0};   // chunk k: blocks [bounds[k], bounds[k + 1]), bytes [byte_bounds[k], byte_bounds[k + 1])
    const uint64_t CHUNK_BYTES = 64ull << 20;
    if (monotonic && verify && blob_size > 2 * CHUNK_BYTES) {
        for (uint64_t i = 0; i + 1 < n; i++)
            if (offsets[i] + lengths[i] - byte_bounds.back() >= CHUNK_BYTES) { bounds.push_back(i + 1); byte_bounds.push_back(offsets[i + 1]); }
    }
    bounds.push_back(n);
    byte_bounds.push_back(blob_size);
    ChunkedCopy copy;
    for (size_t k = 0; k + 1 < bounds.size(); k++) copy.copy(blocks, blob, byte_bounds[k], byte_bounds[k + 1]);
    store_finish(s.get(), cids_dev.p, cids, cids, verify ? flags : 0, &copy, bounds);
    return s.release();
}

Store* store_create_parsed(int device, uint32_t flags, ipcfp_store_json_info& info, bool try_device,
                           const std::function<bool(Store*, Clock::time_point)>& on_device,
                           const std::function<ipcfp_status(ipcfp_parsed_blocks**)>& host_parse, const uint8_t* blob) {
    memset(&info, 0, sizeof info);
    const Clock::time_point t0 = Clock::now();
    if (try_device) {
        bool have_device = true;
        try { check_device(device); }
        catch (const Error&) { have_device = false; }   // the host path's store_create reports it
        if (have_device) {
            std::unique_ptr<Store> s(store_shell(device));
            if (on_device(s.get(), t0)) return s.release();
            memset(&info, 0, sizeof info);
        }
    }
    const Clock::time_point t1 = Clock::now();
    ipcfp_parsed_blocks* pb = nullptr;
    const ipcfp_status st = host_parse(&pb);
    if (st != IPCFP_OK) throw Error(st, ipcfp_last_error(), ipcfp_last_error_index());
    std::unique_ptr<ipcfp_parsed_blocks, void (*)(ipcfp_parsed_blocks*)> keep(pb, ipcfp_parsed_blocks_free);
    info.ms_parse = ms_since(t1);
    const ipcfp_witness& w = pb->blocks;
    return store_create(w.cids, w.offsets, w.lengths, blob ? blob : w.blob, w.blob_size, w.n_blocks, device, flags);
}

void store_get(Store* s, const uint8_t* cid, uint8_t* buf, uint32_t cap, uint32_t* len, int* found) {
    s->use();
    cudaStream_t st = s->stream;
    DevBuf<uint8_t> c(64);
    DevBuf<int32_t> o(4);
    IPCFP_CUDA(cudaMemcpyAsync(c.p, cid, 38, cudaMemcpyHostToDevice, st));
    k_lookup_one<<<1, 1, 0, st>>>(s->view, c.p, o.p); IPCFP_LAUNCH_CHECK();
    int32_t idx = -1;
    IPCFP_CUDA(cudaMemcpyAsync(&idx, o.p, 4, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    *found = idx >= 0;
    if (idx < 0) { if (len) *len = 0; return; }
    uint64_t off; uint32_t l;
    IPCFP_CUDA(cudaMemcpy(&off, s->offsets.p + idx, 8, cudaMemcpyDeviceToHost));
    IPCFP_CUDA(cudaMemcpy(&l, s->lengths.p + idx, 4, cudaMemcpyDeviceToHost));
    if (len) *len = l;
    if (buf && cap) IPCFP_CUDA(cudaMemcpy(buf, s->arena.p + ARENA_HEAD + off, l < cap ? l : cap, cudaMemcpyDeviceToHost));
}

// ------------------------------------------------------------------------------------------ batched hashes
template <int WHICH> __global__ void __launch_bounds__(128) k_hash_batch(const uint8_t* __restrict__ blob, const uint64_t* __restrict__ offsets,
                                                                          const uint32_t* __restrict__ lengths, uint64_t n, uint8_t* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* p = blob + offsets[i];
    uint32_t len = lengths[i];
    uint64_t w[4];
    if (WHICH == 0) { Digest d; blake2b256(p, len, d); w[0] = d.w[0]; w[1] = d.w[1]; w[2] = d.w[2]; w[3] = d.w[3]; }
    else if (WHICH == 1) { Digest d; keccak256(p, len, d); w[0] = d.w[0]; w[1] = d.w[1]; w[2] = d.w[2]; w[3] = d.w[3]; }
    else {
        uint32_t h[8];
        sha256(p, len, h);
#pragma unroll
        for (int k = 0; k < 4; k++) w[k] = (uint64_t)__byte_perm(h[2 * k], 0, 0x0123) | ((uint64_t)__byte_perm(h[2 * k + 1], 0, 0x0123) << 32);
    }
    uint64_t* o = (uint64_t*)(out + 32 * i);
    o[0] = w[0]; o[1] = w[1]; o[2] = w[2]; o[3] = w[3];
}

void hash_batch(int which, const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets, const uint32_t* lengths, uint64_t n, int device,
                uint8_t* out) {
    check_device(device);
    if (n == 0) return;
    for (uint64_t i = 0; i < n; i++)
        if (offsets[i] > blob_size || (uint64_t)lengths[i] > blob_size - offsets[i]) throw Error(IPCFP_ERR_INVALID_ARG, "message out of blob bounds", i);
    DevBuf<uint8_t> dblob(blob_size + 48), dout(n * 32);
    DevBuf<uint64_t> doff(n);
    DevBuf<uint32_t> dlen(n);
    IPCFP_CUDA(cudaMemset(dblob.p, 0, 16));
    IPCFP_CUDA(cudaMemset(dblob.p + 16 + blob_size, 0, 32));
    if (blob_size) IPCFP_CUDA(cudaMemcpy(dblob.p + 16, blob, blob_size, cudaMemcpyHostToDevice));
    IPCFP_CUDA(cudaMemcpy(doff.p, offsets, n * 8, cudaMemcpyHostToDevice));
    IPCFP_CUDA(cudaMemcpy(dlen.p, lengths, n * 4, cudaMemcpyHostToDevice));
    unsigned g = div_up(n, 128);
    if (which == 0) k_hash_batch<0><<<g, 128>>>(dblob.p + 16, doff.p, dlen.p, n, dout.p);
    else if (which == 1) k_hash_batch<1><<<g, 128>>>(dblob.p + 16, doff.p, dlen.p, n, dout.p);
    else k_hash_batch<2><<<g, 128>>>(dblob.p + 16, doff.p, dlen.p, n, dout.p);
    IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaMemcpy(out, dout.p, n * 32, cudaMemcpyDeviceToHost));
}

// compute_mapping_slot (storage/utils.rs:5-12): keccak256(key32 || 24 zero bytes || be64(slot_index))
__global__ void k_mapping_slots(const uint8_t* __restrict__ keys, const uint64_t* __restrict__ idx, uint64_t n, uint8_t* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    __align__(8) uint8_t buf[64];
    for (int k = 0; k < 32; k++) buf[k] = keys[32 * i + k];
    for (int k = 32; k < 56; k++) buf[k] = 0;
    uint64_t s = idx[i];
    for (int k = 0; k < 8; k++) buf[56 + k] = (uint8_t)(s >> (56 - 8 * k));
    // keccak over a local buffer: absorb directly (64 bytes < rate)
    uint64_t st[25];
#pragma unroll
    for (int k = 0; k < 25; k++) st[k] = 0;
    for (int k = 0; k < 8; k++) st[k] = ((const uint64_t*)buf)[k];
    st[8] ^= 0x01ull;
    st[16] ^= 0x8000000000000000ULL;
    keccak_f1600(st);
    uint64_t* o = (uint64_t*)(out + 32 * i);
    o[0] = st[0]; o[1] = st[1]; o[2] = st[2]; o[3] = st[3];
}
void mapping_slots(const uint8_t* keys32, const uint64_t* slot_indices, uint64_t n, int device, uint8_t* out) {
    check_device(device);
    if (!n) return;
    DevBuf<uint8_t> dk(n * 32), dout(n * 32);
    DevBuf<uint64_t> di(n);
    IPCFP_CUDA(cudaMemcpy(dk.p, keys32, n * 32, cudaMemcpyHostToDevice));
    IPCFP_CUDA(cudaMemcpy(di.p, slot_indices, n * 8, cudaMemcpyHostToDevice));
    k_mapping_slots<<<div_up(n, 128), 128>>>(dk.p, di.p, n, dout.p);
    IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaMemcpy(out, dout.p, n * 32, cudaMemcpyDeviceToHost));
}

}  // namespace ipcfp
