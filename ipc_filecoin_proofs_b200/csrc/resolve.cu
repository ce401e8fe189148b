// resolve.cu — ipcfp_resolve_addresses: Filecoin addresses to actor IDs through the Init actor's address map (DESIGN.md §2, "Address
// resolution"), and the host-side address codecs ipcfp_address_parse / ipcfp_address_from_eth. Per-item code: resolve_items.cuh.
//   k_resolve_init   one warp, lane 0: StateRoot → actors HAMT → Init actor → InitState; the call's init_status and address_map root
//   k_resolve        one address per warp, lane 0 walks the address_map HAMT (the shape of k_storage_proofs)
// Every block a walk reads is marked in one rank bitmap, materialised as the call's witness; every walk that lacks a block appends that
// block's CID, and the list is sorted and made unique on the device (sort_unique_cids) before its one copy back.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "engine.cuh"
#include "prims.cuh"
#include "resolve_items.cuh"

namespace ipcfp {

constexpr int32_t RS_PENDING = 1;   // status of an address the kernel resolves (ID and invalid addresses are settled on the host)

struct ResolveArgs {
    StoreView store;
    const uint8_t* state_root;
    const ipcfp_address* addrs;
    uint64_t n;
    int32_t* status;                  // n: RS_PENDING on entry for the walks
    uint64_t* ids;                    // n
    uint32_t* wbits;
    uint8_t* miss;                    // (n + 1) * 38
    unsigned long long* n_miss;
    int32_t* init_status;             // written by k_resolve_init
    const uint8_t** address_map;      // written by k_resolve_init
    uint32_t strict_only;
};

__device__ __forceinline__ void resolve_miss(const ResolveArgs& a, const uint8_t* cid) {
    const unsigned long long k = atomicAdd(a.n_miss, 1ull);
    for (int b = 0; b < 38; b++) a.miss[38 * k + b] = cid[b];
}

__global__ void k_resolve_init(ResolveArgs a) {
    if (threadIdx.x) return;
    Recorder rec{nullptr, 0, a.wbits, false};
    rec.rank_of = a.store.rank_of;
    rec.strict_only = a.strict_only != 0;
    Fail f{0, 0};
    const uint8_t* map = nullptr;
    if (resolve_init(a.store, rec, a.state_root, map, f)) *a.init_status = IPCFP_OK;
    else {
        *a.init_status = resolve_status(f.code);
        if (f.code == DC_MISSING) resolve_miss(a, rec.missing);
    }
    *a.address_map = map;
}

__global__ void __launch_bounds__(128) k_resolve(ResolveArgs a) {
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= a.n || (threadIdx.x & 31) || a.status[t] != RS_PENDING) return;
    const int32_t init = *a.init_status;
    if (init != IPCFP_OK) { a.status[t] = init; return; }
    Recorder rec{nullptr, 0, a.wbits, false};
    rec.rank_of = a.store.rank_of;
    rec.strict_only = a.strict_only != 0;
    Fail f{0, 0};
    uint64_t id;
    const ipcfp_address& ad = a.addrs[t];
    if (resolve_lookup(a.store, rec, *a.address_map, ad.bytes, ad.len, id, f)) { a.status[t] = IPCFP_OK; a.ids[t] = id; return; }
    a.status[t] = resolve_status(f.code);
    if (f.code == DC_MISSING) resolve_miss(a, rec.missing);
}

// ------------------------------------------------------------------------------------------ host: address codecs
static uint32_t leb_put(uint64_t v, uint8_t* out) {
    uint32_t k = 0;
    while (v >= 0x80) { out[k++] = (uint8_t)(v | 0x80); v >>= 7; }
    out[k++] = (uint8_t)v;
    return k;
}

// BLAKE2b with a 4-byte digest (the address checksum): RFC 7693, unkeyed
static void blake2b_4(const uint8_t* msg, size_t len, uint8_t out[4]) {
    static const uint64_t IV[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                                   0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    static const uint8_t SIG[12][16] = {
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
        {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
        {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
        {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
        {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};
    auto rotr = [](uint64_t x, int r) { return (x >> r) | (x << (64 - r)); };
    uint64_t h[8];
    for (int i = 0; i < 8; i++) h[i] = IV[i];
    h[0] ^= 0x01010000ull ^ 4;   // digest length 4, no key
    uint64_t t = 0;
    size_t pos = 0;
    do {
        uint8_t blk[128] = {};
        const size_t take = len - pos > 128 ? 128 : len - pos;
        memcpy(blk, msg + pos, take);
        pos += take;
        t += take;
        const bool last = pos == len;
        uint64_t m[16], v[16];
        for (int i = 0; i < 16; i++) { m[i] = 0; for (int b = 7; b >= 0; b--) m[i] = (m[i] << 8) | blk[8 * i + b]; }
        for (int i = 0; i < 8; i++) { v[i] = h[i]; v[i + 8] = IV[i]; }
        v[12] ^= t;
        if (last) v[14] = ~v[14];
        for (int r = 0; r < 12; r++) {
            const uint8_t* s = SIG[r];
            auto G = [&](int a, int b, int c, int d, uint64_t x, uint64_t y) {
                v[a] = v[a] + v[b] + x; v[d] = rotr(v[d] ^ v[a], 32); v[c] = v[c] + v[d]; v[b] = rotr(v[b] ^ v[c], 24);
                v[a] = v[a] + v[b] + y; v[d] = rotr(v[d] ^ v[a], 16); v[c] = v[c] + v[d]; v[b] = rotr(v[b] ^ v[c], 63);
            };
            G(0, 4, 8, 12, m[s[0]], m[s[1]]); G(1, 5, 9, 13, m[s[2]], m[s[3]]); G(2, 6, 10, 14, m[s[4]], m[s[5]]); G(3, 7, 11, 15, m[s[6]], m[s[7]]);
            G(0, 5, 10, 15, m[s[8]], m[s[9]]); G(1, 6, 11, 12, m[s[10]], m[s[11]]); G(2, 7, 8, 13, m[s[12]], m[s[13]]); G(3, 4, 9, 14, m[s[14]], m[s[15]]);
        }
        for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
    } while (pos < len);
    for (int b = 0; b < 4; b++) out[b] = (uint8_t)(h[0] >> (8 * b));
}

// decimal u64 as Rust's u64::from_str reads it (an optional '+', then digits); fvm_shared refuses more than 20 characters
static bool dec_u64(const char* s, size_t n, uint64_t& v) {
    if (n > 20) return false;
    size_t i = 0;
    if (n && s[0] == '+') i = 1;
    if (i == n) return false;
    v = 0;
    for (; i < n; i++) {
        if (s[i] < '0' || s[i] > '9') return false;
        const uint64_t d = (uint64_t)(s[i] - '0');
        if (v > (UINT64_MAX - d) / 10) return false;
        v = v * 10 + d;
    }
    return true;
}
// RFC 4648 base32, lower case, no padding, trailing bits zero (data_encoding's BASE32_NOPAD rules with the lower-case alphabet)
static bool b32_decode(const char* s, size_t n, std::vector<uint8_t>& out) {
    const size_t r = n % 8;
    if (r == 1 || r == 3 || r == 6) return false;
    out.clear();
    uint32_t acc = 0, bits = 0;
    for (size_t i = 0; i < n; i++) {
        const char c = s[i];
        uint32_t v;
        if (c >= 'a' && c <= 'z') v = (uint32_t)(c - 'a');
        else if (c >= '2' && c <= '7') v = 26u + (uint32_t)(c - '2');
        else return false;
        acc = (acc << 5) | v;
        bits += 5;
        if (bits >= 8) { bits -= 8; out.push_back((uint8_t)(acc >> bits)); acc &= (1u << bits) - 1; }
    }
    return acc == 0;
}

void address_parse(const char* text, uint64_t len, ipcfp_address& out) {
    memset(&out, 0, sizeof out);
    auto bad = [](const char* why) { throw Error(IPCFP_ERR_INVALID_ARG, std::string("invalid address: ") + why); };
    if (len < 3) bad("too short");
    if (text[0] != 'f' && text[0] != 't') bad("unknown network prefix");
    if (text[1] < '0' || text[1] > '4') bad("unknown protocol");
    const uint8_t proto = (uint8_t)(text[1] - '0');
    const char* raw = text + 2;
    size_t n = (size_t)len - 2;
    uint64_t v;
    if (proto == 0) {
        if (!dec_u64(raw, n, v)) bad("ID is not a decimal u64");
        out.bytes[0] = 0;
        out.len = (uint8_t)(1 + leb_put(v, out.bytes + 1));
        return;
    }
    uint8_t head[11];
    uint32_t hl = 0;
    head[hl++] = proto;
    if (proto == 4) {
        const char* f = (const char*)memchr(raw, 'f', n);
        if (!f) bad("delegated address without 'f' separator");
        if (!dec_u64(raw, (size_t)(f - raw), v)) bad("namespace is not a decimal u64");
        hl += leb_put(v, head + hl);
        n -= (size_t)(f - raw) + 1;
        raw = f + 1;
    }
    std::vector<uint8_t> payload;
    if (!b32_decode(raw, n, payload)) bad("payload is not lower-case unpadded base32");
    if (payload.size() < 4) bad("payload shorter than its checksum");
    const size_t pl = payload.size() - 4;
    if ((proto == 1 || proto == 2) && pl != 20) bad("payload length");
    if (proto == 3 && pl != 48) bad("payload length");
    if (proto == 4 && pl > 54) bad("subaddress longer than 54 bytes");
    memcpy(out.bytes, head, hl);
    memcpy(out.bytes + hl, payload.data(), pl);
    out.len = (uint8_t)(hl + pl);
    uint8_t ck[4];
    blake2b_4(out.bytes, out.len, ck);
    if (memcmp(ck, payload.data() + pl, 4) != 0) { memset(&out, 0, sizeof out); bad("checksum mismatch"); }
}

void address_from_eth(const uint8_t eth[20], ipcfp_address& out) {
    memset(&out, 0, sizeof out);
    bool masked = eth[0] == 0xff;
    for (int i = 1; i < 12; i++) masked &= eth[i] == 0;
    if (masked) {
        uint64_t id = 0;
        for (int i = 12; i < 20; i++) id = (id << 8) | eth[i];
        out.bytes[0] = 0;
        out.len = (uint8_t)(1 + leb_put(id, out.bytes + 1));
        return;
    }
    out.bytes[0] = 4;
    out.bytes[1] = 10;   // the Ethereum address manager's namespace
    memcpy(out.bytes + 2, eth, 20);
    out.len = 22;
}

// ------------------------------------------------------------------------------------------ host: the call
void resolve_addresses(Store* s, const uint8_t* state_root, const ipcfp_address* addrs, uint64_t n, ResolveOut& out) {
    if (n && !addrs) throw Error(IPCFP_ERR_INVALID_ARG, "null addresses");
    s->use();
    cudaStream_t st = s->stream;
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_BEGIN], st));
    out.ids.assign(n, 0);
    out.status.assign(n, RS_PENDING);
    uint64_t n_walk = 0;
    for (uint64_t i = 0; i < n; i++) {
        uint64_t id;
        if (!address_valid(addrs[i], &id)) out.status[i] = IPCFP_ERR_INVALID_ARG;
        else if (addrs[i].bytes[0] == 0) { out.status[i] = IPCFP_OK; out.ids[i] = id; }
        else n_walk++;
    }
    const uint64_t nwords = (s->n + 31) / 32 + 8;
    AsyncBuf<uint8_t> d_in(64 + n * sizeof(ipcfp_address) + 16, st), miss(38 * (n + 1) + 16, st);
    AsyncBuf<int32_t> d_status(n + 8, st);
    AsyncBuf<uint64_t> d_ids(n + 8, st), d_words(4, st);   // [0] missing count, [1] init status, [2] address_map pointer
    AsyncBuf<uint32_t> wbits(nwords, st);
    wbits.zero();
    d_words.zero();
    IPCFP_CUDA(cudaMemcpyAsync(d_in.p, state_root, 38, cudaMemcpyHostToDevice, st));
    if (n) {
        IPCFP_CUDA(cudaMemcpyAsync(d_in.p + 64, addrs, n * sizeof(ipcfp_address), cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(d_status.p, out.status.data(), n * 4, cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(d_ids.p, out.ids.data(), n * 8, cudaMemcpyHostToDevice, st));
    }
    ResolveArgs a;
    a.store = s->view; a.state_root = d_in.p; a.addrs = (const ipcfp_address*)(d_in.p + 64); a.n = n; a.status = d_status.p; a.ids = d_ids.p;
    a.wbits = wbits.p; a.miss = miss.p; a.n_miss = (unsigned long long*)d_words.p; a.init_status = (int32_t*)(d_words.p + 1);
    a.address_map = (const uint8_t**)(d_words.p + 2); a.strict_only = getenv("IPCFP_HAMT_STRICT") ? 1 : 0;
    k_resolve_init<<<1, 32, 0, st>>>(a); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_LOOKUP_BEGIN], st));
    if (n_walk) { k_resolve<<<div_up(n * 32, 128), 128, 0, st>>>(a); IPCFP_LAUNCH_CHECK(); }
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_LOOKUP_END], st));
    uint64_t hw[2];
    IPCFP_CUDA(cudaMemcpyAsync(hw, d_words.p, 16, cudaMemcpyDeviceToHost, st));
    if (n) {
        IPCFP_CUDA(cudaMemcpyAsync(out.status.data(), d_status.p, n * 4, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(out.ids.data(), d_ids.p, n * 8, cudaMemcpyDeviceToHost, st));
    }
    materialize_witness(s, wbits.p, out.wit);   // synchronises the stream: hw, status and ids are on the host
    out.init_status = (int32_t)(uint32_t)hw[1];
    uint64_t n_miss = hw[0], m = 0, mixed = UINT64_MAX;
    out.missing.clear();
    if (n_miss) {
        AsyncBuf<uint8_t> sorted(38 * n_miss + 16, st);
        m = sort_unique_cids(st, miss.p, n_miss, sorted.p, &mixed);
        out.missing.resize(38 * m);
        IPCFP_CUDA(cudaMemcpyAsync(out.missing.data(), sorted.p, 38 * m, cudaMemcpyDeviceToHost, st));
    }
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_END], st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (mixed != UINT64_MAX) sort_cids_host(out.missing);
    IPCFP_CUDA(cudaEventElapsedTime(&out.ms_total, s->ev[EV_BEGIN], s->ev[EV_END]));
    IPCFP_CUDA(cudaEventElapsedTime(&out.ms_lookup, s->ev[EV_LOOKUP_BEGIN], s->ev[EV_LOOKUP_END]));
    for (uint64_t i = 0; i < n; i++) if (out.status[i] != IPCFP_OK) out.ids[i] = 0;
}

}  // namespace ipcfp
