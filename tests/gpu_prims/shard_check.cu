// shard_check.cu — the kernels of the cross-shard protocol (csrc/shard_kernels.cuh, DESIGN.md §6 stages X, P, F and W) for W simulated
// ranks on one device, against plain CPU references. Every stage is enqueued the way ShardExchange (csrc/parallel.cu) enqueues it: the
// same kernels, launch shapes, memsets and buffer sizes (exec_seg_cap, exec_table_slots, union_piece_cap_default). The collectives
// become device copies:
//   all-to-all      rank r's receive segment p is rank p's send segment r (one strided copy per receiving rank);
//   all-gather      concatenation;
//   all-reduce(sum) a summing kernel, one receiving rank after the other.
// Ranks run one after the other. All ranks' send buffers share one allocation, rank p's right behind rank p − 1's, and the senders run
// from the last rank down, so a write past the end of one rank's buffer lands in a buffer that is already complete and checked, or in
// the sentinel behind the last one. Every output buffer carries such a sentinel, which must survive. A stage's outputs are checked
// before the next stage reads them, so a wrong count never reaches a kernel as a loop bound.
//
//   X  k_xb_count / k_xb_headers / k_xb_scatter: every segment header (min(count, cap)) and entry in (owner, position) order, the
//      overflow word of every rank; k_recv_offsets, k_exec_claim_seg, k_exec_mark_dups: the summed duplicate bitmap against a
//      first-seen dedup of the raw list, bits past nraw clear;
//   P  k_zero_counts + scan: n_exec; k_select_positions for every exec index and past n_exec (UINT64_MAX); k_check_exec: the key of
//      the smallest exec index >= n_exec (ST_PASS2, code 0) or all ones;
//   F  k_fetch_positions + sum + k_patch_message_cids: every kept proof's message_cid is exec[exec_index], every other proof is
//      untouched, and the answers in rank order are the execution order;
//   W  k_cids_to_recs; the replicated union (k_merge_starts / k_merge_rank / k_merge_emit38: positions, first-of-CID flags, output);
//      the partitioned union (k_part_bounds, k_part_pack, k_part_counts): bounds, headers, pieces, overflow words, each rank's
//      partition, and with forced slot capacities 1 and 3 the retry with nw_max + 1.
// Owners are computed with a host copy of mix64 / rawcid_hash that is checked against the device on every input.
//
//   nvcc <the Makefile's NVFLAGS> -o shard_check tests/gpu_prims/shard_check.cu ipc_filecoin_proofs_b200/csrc/prims.cu
//   ./shard_check [orders.bin out.bin]
// With a file of raw message lists (tests/test_shard_check.py writes it), every list is also exchanged at every world size and the
// rebuilt execution order (the select of every exec index, then the fetch) is written to out.bin. Prints one "ok: ..." line and
// exits 0, or names the first disagreement (kernel, W, case, index) and exits 1.
#include <algorithm>
#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_set>
#include <vector>

#include "../../ipc_filecoin_proofs_b200/csrc/engine.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/prims.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/shard_kernels.cuh"

namespace ipcfp {
void note_launch() {}   // the library counts launches in capi.cu; nothing to count here
}  // namespace ipcfp

using namespace ipcfp;

static uint64_t g_rng = 0x5A4D5EEDull;
static uint64_t rnd() {
    uint64_t z = (g_rng += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static uint64_t g_cases = 0, g_xovf = 0, g_uovf = 0;   // all cases; exchanges with an overflow word raised; unions with a piece overflowing

#define FAIL(...)                         \
    do {                                  \
        fprintf(stderr, "FAIL: ");        \
        fprintf(stderr, __VA_ARGS__);     \
        fprintf(stderr, "\n");            \
        return false;                     \
    } while (0)
#define ULL(x) ((unsigned long long)(x))

// ------------------------------------------------------------------ device buffers with a sentinel
static const uint8_t SENT = 0xA5;
template <class T> struct DBuf {
    T* p = nullptr;
    size_t n = 0, pad = 0;
    // n elements, then `pad` sentinel bytes; the whole allocation starts out as sentinel bytes
    explicit DBuf(size_t n_, size_t pad_ = 256) : n(n_), pad(pad_) {
        IPCFP_CUDA(cudaMalloc((void**)&p, n * sizeof(T) + pad));
        IPCFP_CUDA(cudaMemset(p, SENT, n * sizeof(T) + pad));
    }
    ~DBuf() { cudaFree(p); }
    DBuf(const DBuf&) = delete;
    DBuf& operator=(const DBuf&) = delete;
    bool sentinel_ok() const {
        std::vector<uint8_t> t(pad);
        IPCFP_CUDA(cudaMemcpy(t.data(), (const uint8_t*)p + n * sizeof(T), pad, cudaMemcpyDeviceToHost));
        return std::all_of(t.begin(), t.end(), [](uint8_t b) { return b == SENT; });
    }
};
template <class T> static void up(T* d, const std::vector<T>& h) {
    if (!h.empty()) IPCFP_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
}
template <class T> static std::vector<T> down(const T* d, size_t n) {
    std::vector<T> h(n);
    if (n) IPCFP_CUDA(cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost));
    return h;
}
template <class T> static T down1(const T* d) { return down(d, 1)[0]; }

// ------------------------------------------------------------------ harness kernels (the collectives and the read-back)
__global__ void k_hash_probe(const RawCid* c, uint64_t n, uint64_t* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = rawcid_hash(c[i]);
}
__global__ void k_sum_u32(uint32_t* dst, const uint32_t* src, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] += src[i];
}
__global__ void k_sum_u64(uint64_t* dst, const uint64_t* src, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] += src[i];
}
// the first hbytes of every segment
__global__ void k_gather_hdr(const uint8_t* base, uint64_t nseg, uint64_t stride, uint32_t hbytes, uint8_t* out) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nseg * hbytes) return;
    out[t] = base[(t / hbytes) * stride + t % hbytes];
}
// entries [0, offs[s+1] − offs[s]) of segment s behind its header, all segments back to back (stride, hbytes, esize: multiples of 8)
__global__ void k_compact(const uint8_t* base, uint64_t stride, uint32_t hbytes, uint32_t esize, const uint64_t* offs, uint8_t* out) {
    const uint64_t s = blockIdx.x, a = offs[s], b = offs[s + 1];
    const uint64_t* src = (const uint64_t*)(base + s * stride + hbytes);
    uint64_t* dst = (uint64_t*)(out + a * esize);
    for (uint64_t t = threadIdx.x; t < (b - a) * esize / 8; t += blockDim.x) dst[t] = src[t];
}

// ------------------------------------------------------------------ host copies of the hash, the CID layout and the bucket ranges
static const uint64_t GOLD = 0x9E3779B97F4A7C15ULL;
static const uint64_t M1 = 0xff51afd7ed558ccdULL, M2 = 0xc4ceb9fe1a85ec53ULL;
static uint64_t mix64_h(uint64_t x) {
    x ^= x >> 33; x *= M1; x ^= x >> 33; x *= M2; x ^= x >> 33;
    return x;
}
static uint64_t inv_odd(uint64_t c) {   // c^-1 mod 2^64 (Newton)
    uint64_t y = c;
    for (int i = 0; i < 6; i++) y *= 2 - c * y;
    return y;
}
static uint64_t unmix64_h(uint64_t x) {   // mix64 is a bijection: x ^= x >> 33 is its own inverse
    x ^= x >> 33; x *= inv_odd(M2); x ^= x >> 33; x *= inv_odd(M1); x ^= x >> 33;
    return x;
}
static uint64_t rawcid_hash_h(const RawCid& c) { return mix64_h(c.w[0] ^ (c.w[2] * GOLD) ^ c.w[4]); }
static uint32_t owner_h(const RawCid& c, uint32_t W) { return (uint32_t)((rawcid_hash_h(c) >> 32) % W); }
static bool same(const RawCid& a, const RawCid& b) { return memcmp(&a, &b, sizeof a) == 0; }
struct RawCidHash {
    size_t operator()(const RawCid& c) const { return (size_t)mix64_h(c.w[0] ^ c.w[1] * 3 ^ c.w[2] * 5 ^ c.w[3] * 7 ^ c.w[4] * 11); }
};
struct RawCidEq {
    bool operator()(const RawCid& a, const RawCid& b) const { return same(a, b); }
};

typedef std::array<uint8_t, 38> Cid38;
static const uint8_t FILECOIN_PREFIX[6] = {0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};   // CIDv1, dag-cbor, blake2b-256, 32 bytes
static const uint8_t RAW_SHA_PREFIX[6] = {0x01, 0x55, 0xa0, 0xe4, 0x02, 0x20};    // CIDv1, raw, blake2b-256, 32 bytes
static uint64_t prefix_word(const uint8_t* p) {
    uint64_t w = 0;
    for (int q = 0; q < 6; q++) w |= (uint64_t)p[q] << (8 * q);
    return w;
}
// 38 bytes {prefix[6], digest[32]} ↔ five words {digest bytes in memory order, prefix bytes 0..5 in the low 48 bits}
static RawCid to_raw(const Cid38& c) {
    RawCid r{};
    for (int q = 0; q < 6; q++) r.w[4] |= (uint64_t)c[q] << (8 * q);
    for (int q = 0; q < 32; q++) r.w[q >> 3] |= (uint64_t)c[6 + q] << (8 * (q & 7));
    return r;
}
static Cid38 to_38(const RawCid& r) {
    Cid38 c;
    for (int q = 0; q < 6; q++) c[q] = (uint8_t)(r.w[4] >> (8 * q));
    for (int q = 0; q < 32; q++) c[6 + q] = (uint8_t)(r.w[q >> 3] >> (8 * (q & 7)));
    return c;
}
static RawCid random_raw() {
    RawCid r;
    for (int k = 0; k < 4; k++) r.w[k] = rnd();
    r.w[4] = prefix_word(FILECOIN_PREFIX);
    return r;
}
// a CID whose rawcid_hash is h: w[1], w[3] and the prefix are free, w[0] follows from w[2], w[4] and h
static RawCid cid_with_hash(uint64_t h) {
    RawCid r;
    r.w[1] = rnd(); r.w[2] = rnd(); r.w[3] = rnd();
    r.w[4] = prefix_word(FILECOIN_PREFIX);
    r.w[0] = unmix64_h(h) ^ (r.w[2] * GOLD) ^ r.w[4];
    return r;
}
// a hash whose owner at world size W is o and whose low 32 bits are lo
static uint64_t hash_for(uint32_t o, uint32_t W, uint32_t lo) {
    const uint64_t m = rnd() % ((0x100000000ull - o) / W);
    return ((uint64_t)(o + W * m) << 32) | lo;
}
// the merge order of the witness union: bucket (digest bytes 0, 1), then prefix and digest bytes — within one prefix, the raw byte order
static bool ukey_less(const Cid38& a, const Cid38& b) {
    if (a[6] != b[6]) return a[6] < b[6];
    if (a[7] != b[7]) return a[7] < b[7];
    return a < b;
}
static uint32_t bucket_h(const Cid38& c) { return (uint32_t)c[6] << 8 | c[7]; }
// rank r owns the buckets [ceil(r · 65536 / W), ceil((r + 1) · 65536 / W))
static uint32_t plo_h(uint32_t r, uint32_t W) { return (uint32_t)(((uint64_t)r * 65536 + W - 1) / W); }

// ================================================================== X, P and F: the execution order
struct XCase {
    std::string name;
    uint32_t W;
    std::vector<uint64_t> nseg;   // slice length per rank
    std::vector<RawCid> raw;      // the raw list, all slices back to back
};

// Runs F with the given match lists (exec indices relative to each rank's lo, ascending) and checks the patched proofs; rebuilt:
// the answers of every rank in rank order (the caller passes full match lists when it wants the execution order).
static bool run_fetch(const XCase& xc, const char* mode, const std::vector<uint64_t>& pos0, const std::vector<uint64_t>& lo,
                      const std::vector<uint64_t>& hi, const std::vector<std::vector<uint32_t>>& match, const std::vector<uint64_t>& zpos,
                      const DBuf<RawCid>& d_raw, const DBuf<uint32_t>& bitmap_sum, const DBuf<uint64_t>& zprefix, uint64_t nwords,
                      const DBuf<unsigned long long>& n_exec_d, cudaStream_t st, std::vector<RawCid>* rebuilt) {
    const uint32_t W = xc.W;
    const char* nm = xc.name.c_str();
    const uint64_t n_exec = zpos.size();
    std::vector<uint64_t> moff(W + 1, 0);
    for (uint32_t r = 0; r < W; r++) moff[r + 1] = moff[r] + match[r].size();
    uint64_t M_max = 0;
    for (uint32_t r = 0; r < W; r++) M_max = std::max<uint64_t>(M_max, match[r].size());
    std::vector<uint32_t> rel_all;
    for (auto& m : match) rel_all.insert(rel_all.end(), m.begin(), m.end());
    DBuf<uint32_t> d_rel(rel_all.size());
    up(d_rel.p, rel_all);
    // P again for these matches (positions_for)
    DBuf<uint64_t> req(moff[W]);
    for (uint32_t r = W; r-- > 0;) {
        const uint64_t n_match = match[r].size();
        if (n_match) {
            k_select_positions<<<div_up(n_match, 128), 128, 0, st>>>(d_rel.p + moff[r], n_match, lo[r], bitmap_sum.p, zprefix.p, nwords, n_exec_d.p, req.p + moff[r]);
            IPCFP_LAUNCH_CHECK();
        }
    }
    // proofs: several per exec index, exec_index = UINT64_MAX, indices below lo, indices in range without a match
    std::vector<std::vector<ipcfp_event_proof>> proofs(W);
    std::vector<uint64_t> poff(W + 1, 0);
    for (uint32_t r = 0; r < W; r++) {
        auto add = [&](uint64_t i) {
            ipcfp_event_proof p;
            uint8_t* b = (uint8_t*)&p;
            for (size_t q = 0; q < sizeof p; q++) b[q] = (uint8_t)rnd();
            p.exec_index = i;
            proofs[r].push_back(p);
        };
        add(~0ull);
        if (lo[r]) add(lo[r] - 1);
        for (uint64_t i = lo[r]; i < hi[r]; i++) {
            add(i);
            if (i % 3 == 0) add(i);
            if (i % 7 == 0) add(i);
        }
        add(hi[r]);
        add(~0ull);
        poff[r + 1] = poff[r] + proofs[r].size();
    }
    std::vector<ipcfp_event_proof> pr_all;
    for (auto& v : proofs) pr_all.insert(pr_all.end(), v.begin(), v.end());
    DBuf<ipcfp_event_proof> d_pr(pr_all.size());
    up(d_pr.p, pr_all);
    std::vector<RawCid> ans_h;
    if (M_max) {   // patch(): nothing to fetch when no rank has a match
        const uint64_t total = (uint64_t)W * M_max;
        // all-gather of the request lists, each padded to M_max with "nobody's position"
        DBuf<uint64_t> req_all(total);
        IPCFP_CUDA(cudaMemsetAsync(req_all.p, 0xff, total * 8, st));
        for (uint32_t r = 0; r < W; r++)
            if (moff[r + 1] > moff[r]) IPCFP_CUDA(cudaMemcpyAsync(req_all.p + (uint64_t)r * M_max, req.p + moff[r], (moff[r + 1] - moff[r]) * 8, cudaMemcpyDeviceToDevice, st));
        // every owner answers for the positions of its slice; the all-reduce sums the answers
        DBuf<RawCid> ans(total), ans_sum(total);
        IPCFP_CUDA(cudaMemsetAsync(ans_sum.p, 0, total * sizeof(RawCid), st));
        for (uint32_t q = 0; q < W; q++) {
            k_fetch_positions<<<div_up(total, 256), 256, 0, st>>>(d_raw.p + pos0[q], xc.nseg[q], pos0[q], req_all.p, total, ans.p); IPCFP_LAUNCH_CHECK();
            k_sum_u64<<<div_up(total * 5, 256), 256, 0, st>>>((uint64_t*)ans_sum.p, (const uint64_t*)ans.p, total * 5);
        }
        for (uint32_t r = W; r-- > 0;) {
            const uint64_t n_proofs = proofs[r].size();
            if (n_proofs) {
                k_patch_message_cids<<<div_up(n_proofs, 128), 128, 0, st>>>(d_pr.p + poff[r], n_proofs, d_rel.p + moff[r], match[r].size(), lo[r],
                                                                            ans_sum.p + (uint64_t)r * M_max);
                IPCFP_LAUNCH_CHECK();
            }
        }
        IPCFP_CUDA(cudaStreamSynchronize(st));
        if (!req_all.sentinel_ok() || !ans.sentinel_ok() || !ans_sum.sentinel_ok()) FAIL("k_fetch_positions W=%u case=%s (%s): wrote past the answers", W, nm, mode);
        ans_h = down(ans_sum.p, total);
        for (uint32_t r = 0; r < W; r++)
            for (uint64_t k = 0; k < M_max; k++) {
                const RawCid& got = ans_h[(uint64_t)r * M_max + k];
                RawCid want{};
                if (k < match[r].size()) want = xc.raw[zpos[lo[r] + match[r][k]]];
                if (!same(got, want)) FAIL("k_fetch_positions W=%u case=%s (%s): rank %u answer %llu is not exec[%llu]", W, nm, mode, r, ULL(k), ULL(lo[r] + (k < match[r].size() ? match[r][k] : 0)));
                if (rebuilt && k < match[r].size()) rebuilt->push_back(got);
            }
    }
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (!req.sentinel_ok()) FAIL("k_select_positions W=%u case=%s (%s): wrote past the request list", W, nm, mode);
    if (!d_pr.sentinel_ok()) FAIL("k_patch_message_cids W=%u case=%s (%s): wrote past the proofs", W, nm, mode);
    std::vector<ipcfp_event_proof> got = down(d_pr.p, pr_all.size());
    for (uint32_t r = 0; r < W; r++) {
        std::unordered_set<uint64_t> in_match;
        for (uint32_t m : match[r]) in_match.insert(lo[r] + m);
        for (uint64_t k = 0; k < proofs[r].size(); k++) {
            ipcfp_event_proof want = proofs[r][k];
            const uint64_t i = want.exec_index;
            if (i != ~0ull && i >= lo[r] && in_match.count(i)) {
                if (i >= n_exec) FAIL("harness W=%u case=%s: a match past n_exec", W, nm);
                const Cid38 c = to_38(xc.raw[zpos[i]]);
                memcpy(want.message_cid, c.data(), 38);
            }
            if (memcmp(&want, &got[poff[r] + k], sizeof want))
                FAIL("k_patch_message_cids W=%u case=%s (%s): rank %u proof %llu (exec_index %lld) %s", W, nm, mode, r, ULL(k), (long long)i,
                     in_match.count(i) ? "does not hold exec[exec_index]" : "was touched");
        }
    }
    return true;
}

// One exchange of xc.raw over xc.W ranks: X, P and F. rebuilt (optional): the execution order rebuilt by select + fetch.
static bool run_exchange(const XCase& xc, cudaStream_t st, std::vector<RawCid>* rebuilt = nullptr) {
    const uint32_t W = xc.W;
    const char* nm = xc.name.c_str();
    uint64_t nraw = 0, max_nseg = 0;
    std::vector<uint64_t> pos0(W);
    for (uint32_t r = 0; r < W; r++) { pos0[r] = nraw; nraw += xc.nseg[r]; max_nseg = std::max(max_nseg, xc.nseg[r]); }
    if (nraw != xc.raw.size()) FAIL("harness W=%u case=%s: slices do not tile the raw list", W, nm);
    const uint64_t cap = exec_seg_cap(max_nseg, W), segbytes = XSEG_HDR + cap * 48, slots = exec_table_slots(W, cap), nwords = (nraw + 31) / 32;

    // ---- CPU references: owners, segments, first-seen dedup
    std::vector<uint32_t> own(nraw);
    for (uint64_t i = 0; i < nraw; i++) own[i] = owner_h(xc.raw[i], W);
    std::vector<uint64_t> cnt((uint64_t)W * W, 0);   // [sender * W + owner]
    for (uint32_t p = 0; p < W; p++)
        for (uint64_t i = pos0[p]; i < pos0[p] + xc.nseg[p]; i++) cnt[(uint64_t)p * W + own[i]]++;
    std::vector<bool> ovf_want(W, false);
    bool any_ovf = false;
    for (uint32_t p = 0; p < W; p++)
        for (uint32_t o = 0; o < W; o++)
            if (cnt[(uint64_t)p * W + o] > cap) ovf_want[p] = any_ovf = true;
    std::vector<uint32_t> dup_ref(nwords, 0);
    std::vector<uint64_t> zpos;   // raw position of every exec index
    {
        std::unordered_set<RawCid, RawCidHash, RawCidEq> seen;
        for (uint64_t i = 0; i < nraw; i++) {
            if (seen.insert(xc.raw[i]).second) zpos.push_back(i);
            else dup_ref[i >> 5] |= 1u << (i & 31);
        }
    }
    const uint64_t n_exec = zpos.size();

    DBuf<RawCid> d_raw(nraw);
    up(d_raw.p, xc.raw);
    {   // the host copy of rawcid_hash that placed these CIDs, on every input
        DBuf<uint64_t> h(nraw);
        if (nraw) { k_hash_probe<<<div_up(nraw, 256), 256, 0, st>>>(d_raw.p, nraw, h.p); IPCFP_CUDA(cudaGetLastError()); }
        std::vector<uint64_t> hd = down(h.p, nraw);
        for (uint64_t i = 0; i < nraw; i++)
            if (hd[i] != rawcid_hash_h(xc.raw[i])) FAIL("rawcid_hash W=%u case=%s: the host copy disagrees with the device at entry %llu", W, nm, ULL(i));
    }

    // ---- X, senders (start_exchange: parallel.cu, the sendbuf memsets and the `if (nseg)` block)
    DBuf<uint8_t> send((uint64_t)W * W * segbytes);   // rank p's send buffer at p · W · segbytes
    DBuf<unsigned long long> ovf(W);                  // rank p's overflow word (c->words.p + 3100)
    for (uint32_t p = W; p-- > 0;) {
        uint8_t* sb = send.p + (uint64_t)p * W * segbytes;
        const uint64_t nseg = xc.nseg[p];
        const RawCid* seg = d_raw.p + pos0[p];
        IPCFP_CUDA(cudaMemsetAsync(ovf.p + p, 0, 8, st));
        for (uint32_t r = 0; r < W; r++) IPCFP_CUDA(cudaMemsetAsync(sb + r * segbytes, 0, XSEG_HDR, st));
        if (nseg) {
            const uint32_t nruns = div_up(nseg, XB_RUN);
            {   // leave non-zero bytes in the stream's pool where `cnt` will come from: the kernels may rely on no zero they did not write
                AsyncBuf<uint32_t> junk((uint64_t)W * nruns + 64, st);
                IPCFP_CUDA(cudaMemsetAsync(junk.p, 0xA5, junk.n * 4, st));
            }
            AsyncBuf<uint32_t> cnt_d((uint64_t)W * nruns + 64, st);
            AsyncBuf<uint64_t> scan((uint64_t)W * nruns + 64, st), scratch(scan_scratch_elems((uint64_t)W * nruns) + 8, st), total(1, st);
            if (W > 32) cnt_d.zero();
            k_xb_count<<<div_up((uint64_t)nruns * 32, 128), 128, 0, st>>>(seg, nseg, W, nruns, cnt_d.p); IPCFP_LAUNCH_CHECK();
            exclusive_scan_u32(cnt_d.p, scan.p, (uint64_t)W * nruns, total.p, scratch.p, st);
            k_xb_headers<<<div_up(W, 64), 64, 0, st>>>(scan.p, total.p, W, nruns, cap, sb, ovf.p + p); IPCFP_LAUNCH_CHECK();
            k_xb_scatter<<<div_up((uint64_t)nruns * 32, 128), 128, 0, st>>>(seg, nseg, pos0[p], W, nruns, scan.p, cap, sb); IPCFP_LAUNCH_CHECK();
        }
    }
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (!send.sentinel_ok()) FAIL("k_xb_scatter W=%u case=%s: wrote past the last send buffer", W, nm);
    if (!ovf.sentinel_ok()) FAIL("k_xb_headers W=%u case=%s: wrote past the overflow words", W, nm);
    {
        std::vector<unsigned long long> o = down(ovf.p, W);
        for (uint32_t p = 0; p < W; p++)
            if ((o[p] != 0) != ovf_want[p]) FAIL("k_xb_headers W=%u case=%s: rank %u overflow word %llu, expected %d (cap %llu)", W, nm, p, o[p], (int)ovf_want[p], ULL(cap));
    }
    {   // every header, then every entry in (owner, position) order
        const uint64_t nsegs = (uint64_t)W * W;
        DBuf<uint8_t> hdr(nsegs * XSEG_HDR);
        k_gather_hdr<<<div_up(nsegs * XSEG_HDR, 256), 256, 0, st>>>(send.p, nsegs, segbytes, XSEG_HDR, hdr.p);
        std::vector<uint8_t> h = down(hdr.p, nsegs * XSEG_HDR);
        std::vector<uint64_t> offs(nsegs + 1, 0);
        for (uint64_t s = 0; s < nsegs; s++) {
            uint64_t c;
            memcpy(&c, &h[s * XSEG_HDR], 8);
            const uint64_t want = std::min(cnt[s], cap);
            if (c != want) FAIL("k_xb_headers W=%u case=%s: segment rank %llu → owner %llu says %llu, expected %llu", W, nm, ULL(s / W), ULL(s % W), ULL(c), ULL(want));
            for (int b = 8; b < XSEG_HDR; b++)
                if (h[s * XSEG_HDR + b]) FAIL("k_xb_headers W=%u case=%s: segment rank %llu → owner %llu: header byte %d is not zero", W, nm, ULL(s / W), ULL(s % W), b);
            offs[s + 1] = offs[s] + want;
        }
        DBuf<uint64_t> d_offs(nsegs + 1);
        up(d_offs.p, offs);
        DBuf<uint8_t> comp(offs[nsegs] * 48);
        k_compact<<<(unsigned)nsegs, 128, 0, st>>>(send.p, segbytes, XSEG_HDR, 48, d_offs.p, comp.p);
        IPCFP_CUDA(cudaGetLastError());
        std::vector<uint8_t> e = down(comp.p, offs[nsegs] * 48);
        std::vector<uint64_t> fill(nsegs, 0);
        for (uint32_t p = 0; p < W; p++)
            for (uint64_t i = pos0[p]; i < pos0[p] + xc.nseg[p]; i++) {
                const uint64_t s = (uint64_t)p * W + own[i];
                const uint64_t slot = fill[s]++;
                if (slot >= cap) continue;
                ExecEntry want;
                want.c = xc.raw[i];
                want.pos = i;
                if (memcmp(&want, &e[(offs[s] + slot) * 48], 48))
                    FAIL("k_xb_scatter W=%u case=%s: segment rank %u → owner %u, slot %llu is not raw position %llu", W, nm, p, own[i], ULL(slot), ULL(i));
            }
    }
    g_cases++;
    if (any_ovf && rebuilt) FAIL("k_xb_headers W=%u case=%s: a real message list overflowed its segments (cap %llu)", W, nm, ULL(cap));
    g_xovf += any_ovf;
    if (any_ovf) return true;   // the call refuses it ("bucket overflow"): nothing behind X runs

    // ---- X, owners: all-to-all, claim, mark, all-reduce of the bitmaps
    DBuf<uint8_t> recv((uint64_t)W * segbytes);
    DBuf<uint64_t> seg_off(W + 1);
    DBuf<unsigned long long> table(slots);
    DBuf<uint32_t> bitmap(nwords + 64), bitmap_sum(nwords + 64);
    IPCFP_CUDA(cudaMemsetAsync(bitmap_sum.p, 0, (nwords + 1) * 4, st));
    for (uint32_t o = 0; o < W; o++) {
        IPCFP_CUDA(cudaMemcpy2DAsync(recv.p, segbytes, send.p + (uint64_t)o * segbytes, (uint64_t)W * segbytes, segbytes, W, cudaMemcpyDeviceToDevice, st));
        IPCFP_CUDA(cudaMemsetAsync(bitmap.p, 0, (nwords + 64) * 4, st));
        IPCFP_CUDA(cudaMemsetAsync(table.p, 0, slots * 8, st));
        k_recv_offsets<<<1, 1, 0, st>>>(recv.p, W, cap, seg_off.p); IPCFP_LAUNCH_CHECK();
        std::vector<uint64_t> so = down(seg_off.p, W + 1);
        uint64_t run = 0;
        for (uint32_t r = 0; r <= W; r++) {
            if (so[r] != run) FAIL("k_recv_offsets W=%u case=%s: owner %u, seg_off[%u] = %llu, expected %llu", W, nm, o, r, ULL(so[r]), ULL(run));
            if (r < W) run += cnt[(uint64_t)r * W + o];
        }
        const unsigned g = div_up(W * cap, 256);
        k_exec_claim_seg<<<g, 256, 0, st>>>(recv.p, seg_off.p, W, cap, table.p, slots - 1); IPCFP_LAUNCH_CHECK();
        k_exec_mark_dups<<<g, 256, 0, st>>>(recv.p, seg_off.p, W, cap, table.p, slots - 1, bitmap.p); IPCFP_LAUNCH_CHECK();
        k_sum_u32<<<div_up(nwords + 1, 256), 256, 0, st>>>(bitmap_sum.p, bitmap.p, nwords + 1);
    }
    // ---- P: n_exec and the prefix zero counts
    DBuf<uint32_t> zeros(nwords + 64);
    DBuf<uint64_t> zprefix(nwords + 64), scan_tmp(scan_scratch_elems(nwords + 64) + 64);
    DBuf<unsigned long long> n_exec_d(1);
    if (nwords) { k_zero_counts<<<div_up(nwords, 256), 256, 0, st>>>(bitmap_sum.p, nraw, zeros.p); IPCFP_LAUNCH_CHECK(); }
    exclusive_scan_u32(zeros.p, zprefix.p, nwords, (uint64_t*)n_exec_d.p, scan_tmp.p, st);
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (!recv.sentinel_ok() || !seg_off.sentinel_ok() || !table.sentinel_ok()) FAIL("k_exec_claim_seg W=%u case=%s: wrote past its buffers", W, nm);
    if (!bitmap.sentinel_ok() || !bitmap_sum.sentinel_ok()) FAIL("k_exec_mark_dups W=%u case=%s: wrote past the bitmap", W, nm);
    if (!zeros.sentinel_ok() || !n_exec_d.sentinel_ok()) FAIL("k_zero_counts W=%u case=%s: wrote past its buffers", W, nm);
    {
        std::vector<uint32_t> bm = down(bitmap_sum.p, nwords + 1);
        for (uint64_t w = 0; w <= nwords; w++) {
            const uint32_t want = w < nwords ? dup_ref[w] : 0u;
            if (bm[w] != want) FAIL("k_exec_mark_dups W=%u case=%s: summed bitmap word %llu is %08x, expected %08x", W, nm, ULL(w), bm[w], want);
        }
    }
    if (down1(n_exec_d.p) != n_exec) FAIL("k_zero_counts W=%u case=%s: n_exec %llu, expected %llu", W, nm, down1(n_exec_d.p), ULL(n_exec));

    // ---- P: every exec index and three past n_exec, the receipts split over the ranks by index range
    const uint64_t E = n_exec + 3;
    std::vector<uint64_t> lo(W), hi(W);
    for (uint32_t r = 0; r < W; r++) { lo[r] = E * r / W; hi[r] = E * (r + 1) / W; }
    {
        std::vector<uint32_t> rel(E);
        for (uint32_t r = 0; r < W; r++)
            for (uint64_t i = lo[r]; i < hi[r]; i++) rel[i] = (uint32_t)(i - lo[r]);
        DBuf<uint32_t> d_rel(E);
        up(d_rel.p, rel);
        DBuf<uint64_t> out(E);
        DBuf<unsigned long long> chk(W);
        for (uint32_t r = W; r-- > 0;) {   // positions_for
            const uint64_t n_match = hi[r] - lo[r];
            if (n_match) {
                k_select_positions<<<div_up(n_match, 128), 128, 0, st>>>(d_rel.p + lo[r], n_match, lo[r], bitmap_sum.p, zprefix.p, nwords, n_exec_d.p, out.p + lo[r]);
                IPCFP_LAUNCH_CHECK();
            }
            IPCFP_CUDA(cudaMemsetAsync(chk.p + r, 0xff, 8, st));
            if (n_match) { k_check_exec<<<div_up(n_match, 128), 128, 0, st>>>(d_rel.p + lo[r], n_match, lo[r], n_exec_d.p, chk.p + r); IPCFP_LAUNCH_CHECK(); }
        }
        IPCFP_CUDA(cudaStreamSynchronize(st));
        if (!out.sentinel_ok()) FAIL("k_select_positions W=%u case=%s: wrote past the positions", W, nm);
        if (!chk.sentinel_ok()) FAIL("k_check_exec W=%u case=%s: wrote past the error words", W, nm);
        std::vector<uint64_t> got = down(out.p, E);
        for (uint64_t i = 0; i < E; i++) {
            const uint64_t want = i < n_exec ? zpos[i] : ~0ull;
            if (got[i] != want) FAIL("k_select_positions W=%u case=%s: exec index %llu → %llu, expected %llu", W, nm, ULL(i), ULL(got[i]), ULL(want));
        }
        std::vector<unsigned long long> ck = down(chk.p, W);
        for (uint32_t r = 0; r < W; r++) {
            uint64_t want = ~0ull;   // report_error(err, ST_PASS2, i, 0, 0): [stage 5:8 | index:40 | code 0:8 | detail 0:8]
            for (uint64_t i = lo[r]; i < hi[r]; i++)
                if (i >= n_exec) { want = (5ull << 56) | ((i & 0xFFFFFFFFFFull) << 16); break; }
            if (ck[r] != want) FAIL("k_check_exec W=%u case=%s: rank %u error key %016llx, expected %016llx", W, nm, r, ck[r], ULL(want));
        }
    }
    // ---- F: every exec index (the execution order comes back), then every index but a few
    std::vector<std::vector<uint32_t>> full(W), gaps(W);
    for (uint32_t r = 0; r < W; r++)
        for (uint64_t i = lo[r]; i < std::min(hi[r], n_exec); i++) {
            full[r].push_back((uint32_t)(i - lo[r]));
            if (i % 5 != 2) gaps[r].push_back((uint32_t)(i - lo[r]));
        }
    std::vector<RawCid> order;
    if (!run_fetch(xc, "every index", pos0, lo, hi, full, zpos, d_raw, bitmap_sum, zprefix, nwords, n_exec_d, st, &order)) return false;
    if (order.size() != n_exec) FAIL("k_fetch_positions W=%u case=%s: %zu answers, expected %llu", W, nm, order.size(), ULL(n_exec));
    for (uint64_t i = 0; i < n_exec; i++)
        if (!same(order[i], xc.raw[zpos[i]])) FAIL("k_fetch_positions W=%u case=%s: rebuilt order differs at %llu", W, nm, ULL(i));
    if (!run_fetch(xc, "gaps", pos0, lo, hi, gaps, zpos, d_raw, bitmap_sum, zprefix, nwords, n_exec_d, st, nullptr)) return false;
    if (rebuilt) *rebuilt = order;
    return true;
}

// ------------------------------------------------------------------ exchange cases
enum Content { DISTINCT, ONE_CID, DUP_MIX, STRADDLE, HASHED, ONE_OWNER };
static const char* content_name(Content c) {
    static const char* n[] = {"distinct", "one CID everywhere", "repeats in and across slices", "duplicate runs across slice ends", "hash-built", "one owner"};
    return n[c];
}
// slice shapes
static std::vector<uint64_t> equal_slices(uint32_t W, uint64_t n) {
    std::vector<uint64_t> s(W);
    for (uint32_t r = 0; r < W; r++) s[r] = n / W + (r < n % W);
    return s;
}
static std::vector<uint64_t> slices_on(uint32_t W, uint64_t n, const std::vector<bool>& on) {
    uint32_t k = 0;
    for (bool b : on) k += b;
    std::vector<uint64_t> s(W, 0);
    uint32_t j = 0;
    for (uint32_t r = 0; r < W; r++)
        if (on[r]) { s[r] = n / k + (j < n % k); j++; }
    return s;
}

static std::vector<RawCid> make_raw(Content c, uint32_t W, const std::vector<uint64_t>& nseg) {
    uint64_t n = 0, max_nseg = 0;
    for (uint64_t x : nseg) { n += x; max_nseg = std::max(max_nseg, x); }
    std::vector<RawCid> raw;
    raw.reserve(n);
    switch (c) {
    case DISTINCT:
        while (raw.size() < n) raw.push_back(random_raw());
        break;
    case ONE_CID: {
        const RawCid x = random_raw();
        raw.assign(n, x);
        break;
    }
    case DUP_MIX: {   // drawn from a pool of a third of the length: repeats inside slices and across them
        std::vector<RawCid> pool(std::max<uint64_t>(1, n / 3));
        for (auto& x : pool) x = random_raw();
        while (raw.size() < n) raw.push_back(pool[rnd() % pool.size()]);
        break;
    }
    case STRADDLE: {   // runs of one CID across every slice end, some of them CIDs seen before
        std::vector<uint64_t> ends;
        uint64_t a = 0;
        for (uint64_t x : nseg) { a += x; ends.push_back(a); }
        std::vector<RawCid> used;
        while (raw.size() < n) {
            const uint64_t at = raw.size();
            auto e = std::lower_bound(ends.begin(), ends.end(), at + 1);
            uint64_t len = 1 + rnd() % 4;
            if (e != ends.end() && *e - at <= 40) len = *e - at + 1 + rnd() % 40;   // reaches past the next slice end
            RawCid x = used.empty() || rnd() % 3 ? random_raw() : used[rnd() % used.size()];
            used.push_back(x);
            for (uint64_t k = 0; k < len && raw.size() < n; k++) raw.push_back(x);
        }
        break;
    }
    case HASHED: {   // CIDs aimed at the owners' claim tables
        const uint64_t slots = exec_table_slots(W, exec_seg_cap(max_nseg, W)), mask = slots - 1;
        int lbits = 0;
        while ((1ull << lbits) < slots) lbits++;
        std::vector<RawCid> pool;
        while (pool.size() < std::max<uint64_t>(8, n / 2)) {
            const uint32_t o = (uint32_t)(rnd() % W);
            const uint64_t h = hash_for(o, W, (uint32_t)rnd());
            switch (rnd() % 4) {
            case 0: {   // the same hash: differ only in w[1], only in w[3]
                RawCid x = cid_with_hash(h), y = x, z = x;
                y.w[1] ^= 1 + rnd();
                z.w[3] ^= 1 + rnd();
                pool.insert(pool.end(), {x, y, z});
                break;
            }
            case 1:   // the same slot and owner, other fingerprints
                for (int k = 0; k < 4; k++) pool.push_back(cid_with_hash(hash_for(o, W, (uint32_t)(h & mask))));
                break;
            case 2:   // the same slot, owner and fingerprint, another hash (bits between the slot and the owner differ)
                for (int k = 0; k < 4; k++) pool.push_back(cid_with_hash((h & ~0xFFFFFFFFull) | (h & mask) | (lbits < 32 ? (rnd() << lbits) & 0xFFFFFFFFull : 0)));
                break;
            default:   // probe chains that start in the last slots and wrap to slot 0
                for (int k = 0; k < 6; k++) pool.push_back(cid_with_hash(hash_for(o, W, (uint32_t)(mask - (uint64_t)(k % 3)))));
            }
        }
        while (raw.size() < n) raw.push_back(pool[rnd() % pool.size()]);
        break;
    }
    case ONE_OWNER: {   // every entry on owner W − 1, a few repeated
        while (raw.size() < n) {
            RawCid x = cid_with_hash(hash_for(W - 1, W, (uint32_t)rnd()));
            raw.push_back(x);
            if (rnd() % 8 == 0 && raw.size() < n) raw.push_back(raw[rnd() % raw.size()]);
        }
        break;
    }
    }
    return raw;
}

static bool xcase(const std::string& shape, Content c, uint32_t W, std::vector<uint64_t> nseg, cudaStream_t st) {
    XCase xc;
    xc.W = W;
    xc.nseg = std::move(nseg);
    xc.name = shape + ", " + content_name(c);
    xc.raw = make_raw(c, W, xc.nseg);
    return run_exchange(xc, st);
}

static bool exchanges(uint32_t W, cudaStream_t st) {
    const bool big = W >= 64;
    const uint64_t k = big ? 4 * W : 128;   // the "equal" totals: 32k, 32k + 1, 32k + 31
    std::vector<bool> on(W, true);
    if (!xcase("nraw 0", DISTINCT, W, std::vector<uint64_t>(W, 0), st)) return false;
    if (!xcase("equal, nraw = 0 mod 32", DISTINCT, W, equal_slices(W, 32 * k), st)) return false;
    if (!xcase("equal, nraw = 1 mod 32", DUP_MIX, W, equal_slices(W, 32 * k + 1), st)) return false;
    if (!xcase("equal, nraw = 31 mod 32", STRADDLE, W, equal_slices(W, 32 * k + 31), st)) return false;
    if (!xcase("equal, nraw = 0 mod 32", ONE_CID, W, equal_slices(W, 32 * k), st)) return false;
    if (!xcase("equal", HASHED, W, equal_slices(W, 32 * k + 17), st)) return false;
    if (!xcase("equal", ONE_OWNER, W, equal_slices(W, big ? 4 * W : 2000), st)) return false;
    std::vector<bool> only0(W, false), onlyl(W, false), no0(W, true), nol(W, true), odd(W, false);
    only0[0] = true; onlyl[W - 1] = true; no0[0] = W == 1; nol[W - 1] = W == 1;
    for (uint32_t r = 0; r < W; r += 2) odd[r] = true;
    if (!xcase("all on rank 0", DUP_MIX, W, slices_on(W, 3001, only0), st)) return false;
    if (!xcase("all on the last rank", ONE_CID, W, slices_on(W, 1000, onlyl), st)) return false;
    if (!xcase("all on the last rank", HASHED, W, slices_on(W, 2500, onlyl), st)) return false;
    if (!xcase("rank 0 empty", STRADDLE, W, slices_on(W, 40 * W + 7, no0), st)) return false;
    if (!xcase("last rank empty", DUP_MIX, W, slices_on(W, 40 * W + 9, nol), st)) return false;
    if (!xcase("every other rank empty", STRADDLE, W, slices_on(W, 40 * W + 31, odd), st)) return false;
    if (!xcase("one entry per rank", DUP_MIX, W, std::vector<uint64_t>(W, 1), st)) return false;
    const uint64_t lens[] = {31, 32, 33, 255, 256, 257};
    const Content lc[] = {DUP_MIX, STRADDLE, DISTINCT, STRADDLE, DUP_MIX, HASHED};
    for (int i = 0; i < 6; i++)
        if (!xcase("slices of " + std::to_string(lens[i]), lc[i], W, std::vector<uint64_t>(W, lens[i]), st)) return false;
    // every entry of rank 0 on one owner, at the length where that segment stops fitting and one below it; the other ranks hold 32
    if (W > 1) {
        uint64_t n = 1024;
        while (n <= exec_seg_cap(n, W)) n++;
        for (uint64_t m : {n - 1, n}) {
            std::vector<uint64_t> s(W, 32);
            s[0] = m;
            if (!xcase("rank 0 holds " + std::to_string(m) + (m > exec_seg_cap(m, W) ? " (overflows)" : " (fits)"), ONE_OWNER, W, s, st)) return false;
        }
    }
    return true;
}

// ================================================================== W: the witness union
struct UCase {
    std::string name;
    uint32_t W;
    std::vector<std::vector<Cid38>> lists;   // per rank, sorted by ukey_less, unique
};

static std::vector<uint8_t> flat38(const std::vector<Cid38>& v) {
    std::vector<uint8_t> b(38 * v.size());
    for (size_t i = 0; i < v.size(); i++) memcpy(&b[38 * i], v[i].data(), 38);
    return b;
}

// the local lists of every rank (38-byte CIDs) back to back
struct ULists {
    std::vector<uint64_t> off, n;
    uint64_t nw_max = 0;
    DBuf<uint8_t>* d = nullptr;
    explicit ULists(const UCase& uc) {
        std::vector<uint8_t> all;
        off.push_back(0);
        for (auto& l : uc.lists) {
            std::vector<uint8_t> b = flat38(l);
            all.insert(all.end(), b.begin(), b.end());
            n.push_back(l.size());
            off.push_back(all.size());
            nw_max = std::max<uint64_t>(nw_max, l.size());
        }
        d = new DBuf<uint8_t>(all.size());
        up(d->p, all);
    }
    ~ULists() { delete d; }
};

static bool run_replicated(const UCase& uc, const ULists& L, const std::vector<Cid38>& U, cudaStream_t st) {
    const uint32_t W = uc.W;
    const char* nm = uc.name.c_str();
    // union_replicated: parallel.cu
    const uint64_t capw = L.nw_max + 1, total_cap = (uint64_t)W * capw;
    DBuf<RawCid> gather(total_cap);   // the all-gather of every rank's capw records
    for (uint32_t r = W; r-- > 0;) {
        k_cids_to_recs<<<div_up(capw, 256), 256, 0, st>>>(L.d->p + L.off[r], L.n[r], capw, gather.p + (uint64_t)r * capw); IPCFP_LAUNCH_CHECK();
    }
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (!gather.sentinel_ok()) FAIL("k_cids_to_recs W=%u case=%s: wrote past the records", W, nm);
    {
        std::vector<RawCid> g = down(gather.p, total_cap);
        for (uint32_t r = 0; r < W; r++)
            for (uint64_t k = 0; k < capw; k++) {
                RawCid want{};
                if (k < L.n[r]) want = to_raw(uc.lists[r][k]);
                if (!same(g[(uint64_t)r * capw + k], want)) FAIL("k_cids_to_recs W=%u case=%s: rank %u record %llu", W, nm, r, ULL(k));
            }
    }
    DBuf<uint64_t> counts(W);
    up(counts.p, L.n);
    DBuf<uint32_t> flags(total_cap + 64), starts((uint64_t)W * (MERGE_BUCKETS + 1) + 64), pos_of(total_cap + 64);
    DBuf<uint64_t> fscan(total_cap + 64), scan_tmp(scan_scratch_elems(total_cap + 64) + 64);
    DBuf<uint8_t> merged(total_cap * 38 + 64);
    DBuf<unsigned long long> n_union(1);
    IPCFP_CUDA(cudaMemsetAsync(flags.p, 0, (total_cap + 64) * 4, st));
    const unsigned g = div_up(total_cap, 256);
    k_merge_starts<<<g, 256, 0, st>>>(gather.p, counts.p, W, capw, starts.p, 0, MERGE_BUCKETS); IPCFP_LAUNCH_CHECK();
    k_merge_rank<<<g, 256, 0, st>>>(gather.p, counts.p, W, capw, starts.p, pos_of.p, flags.p, 0, MERGE_BUCKETS); IPCFP_LAUNCH_CHECK();
    uint64_t total_listed = 0;
    for (uint32_t r = 0; r < W; r++) total_listed += L.n[r];
    exclusive_scan_u32(flags.p, fscan.p, total_listed, (uint64_t*)n_union.p, scan_tmp.p, st);
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (!starts.sentinel_ok()) FAIL("k_merge_starts W=%u case=%s: wrote past the bucket starts", W, nm);
    if (!flags.sentinel_ok() || !pos_of.sentinel_ok()) FAIL("k_merge_rank W=%u case=%s: wrote past its buffers", W, nm);
    {   // the merged order is stable: equal CIDs by rank; an element is kept when it is the first of its CID
        std::vector<std::pair<uint32_t, uint64_t>> order;
        for (uint32_t r = 0; r < W; r++)
            for (uint64_t k = 0; k < L.n[r]; k++) order.push_back({r, k});
        std::stable_sort(order.begin(), order.end(), [&](const std::pair<uint32_t, uint64_t>& a, const std::pair<uint32_t, uint64_t>& b) {
            return ukey_less(uc.lists[a.first][a.second], uc.lists[b.first][b.second]);
        });
        std::vector<uint32_t> po = down(pos_of.p, total_cap), fl = down(flags.p, total_cap + 64);
        for (uint64_t q = 0; q < order.size(); q++) {
            const uint32_t r = order[q].first;
            const uint64_t k = order[q].second;
            if (po[(uint64_t)r * capw + k] != q) FAIL("k_merge_rank W=%u case=%s: rank %u element %llu at merged position %u, expected %llu", W, nm, r, ULL(k), po[(uint64_t)r * capw + k], ULL(q));
            const bool first = q == 0 || uc.lists[order[q - 1].first][order[q - 1].second] != uc.lists[r][k];
            if (fl[q] != (first ? 1u : 0u)) FAIL("k_merge_rank W=%u case=%s: merged position %llu flag %u, expected %d", W, nm, ULL(q), fl[q], (int)first);
        }
        for (uint64_t q = order.size(); q < total_cap + 64; q++)
            if (fl[q]) FAIL("k_merge_rank W=%u case=%s: flag set at %llu, past the %llu listed", W, nm, ULL(q), ULL(total_listed));
    }
    k_merge_emit38<<<g, 256, 0, st>>>(gather.p, counts.p, W, capw, pos_of.p, flags.p, fscan.p, merged.p); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaStreamSynchronize(st));
    const uint64_t nu = down1(n_union.p);
    if (nu != U.size()) FAIL("k_merge_emit38 W=%u case=%s: replicated union of %llu CIDs, expected %zu", W, nm, ULL(nu), U.size());
    if (!merged.sentinel_ok()) FAIL("k_merge_emit38 W=%u case=%s: wrote past the union", W, nm);
    std::vector<uint8_t> m = down(merged.p, total_cap * 38 + 64);
    for (uint64_t i = 0; i < nu; i++)
        if (memcmp(&m[38 * i], U[i].data(), 38)) FAIL("k_merge_emit38 W=%u case=%s: replicated union entry %llu differs", W, nm, ULL(i));
    for (uint64_t b = 38 * nu; b < m.size(); b++)
        if (m[b] != SENT) FAIL("k_merge_emit38 W=%u case=%s: wrote byte %llu, past the union", W, nm, ULL(b));
    return true;
}

// union_partitioned(cap): parallel.cu. → *overflow: some rank raised its overflow word (each checked against the rule)
static bool run_partitioned(const UCase& uc, const ULists& L, const std::vector<Cid38>& U, uint64_t cap, bool* overflow, cudaStream_t st) {
    const uint32_t W = uc.W;
    const char* nm = uc.name.c_str();
    const uint64_t stride = cap + 1, total_cap = (uint64_t)W * stride;
    // every rank's piece lengths by the plain bucket ranges
    std::vector<std::vector<uint64_t>> bnd(W, std::vector<uint64_t>(W + 1));
    std::vector<bool> ovf_want(W, false);
    for (uint32_t p = 0; p < W; p++) {
        const auto& l = uc.lists[p];
        for (uint32_t r = 0; r <= W; r++) {
            uint64_t i = 0;
            while (r < W && i < l.size() && bucket_h(l[i]) < plo_h(r, W)) i++;
            bnd[p][r] = r == W ? l.size() : i;
        }
        for (uint32_t r = 0; r < W; r++)
            if (bnd[p][r + 1] - bnd[p][r] > cap) ovf_want[p] = true;
    }
    std::vector<uint64_t> roff(W + 1, 0);
    for (uint32_t p = 0; p < W; p++) roff[p + 1] = roff[p] + L.n[p] + 1;
    DBuf<RawCid> recs(roff[W]);
    // the send buffers of all ranks back to back; a piece may not spill past its slots: room for a whole list behind the last one
    DBuf<RawCid> send((uint64_t)W * total_cap, (L.nw_max + 8) * sizeof(RawCid));
    DBuf<uint64_t> bounds((uint64_t)W * (W + 1));
    DBuf<unsigned long long> mine(2ull * W);   // [n_part, overflow] per rank
    for (uint32_t p = W; p-- > 0;) {
        const uint64_t n_local = L.n[p];
        RawCid* sp = send.p + (uint64_t)p * total_cap;
        k_cids_to_recs<<<div_up(n_local + 1, 256), 256, 0, st>>>(L.d->p + L.off[p], n_local, n_local + 1, recs.p + roff[p]); IPCFP_LAUNCH_CHECK();
        k_part_bounds<<<1, 256, 0, st>>>(recs.p + roff[p], n_local, W, cap, bounds.p + (uint64_t)p * (W + 1), sp, mine.p + 2 * p + 1); IPCFP_LAUNCH_CHECK();
        if (n_local) { k_part_pack<<<div_up(n_local, 256), 256, 0, st>>>(recs.p + roff[p], n_local, W, cap, bounds.p + (uint64_t)p * (W + 1), sp); IPCFP_LAUNCH_CHECK(); }
    }
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (!recs.sentinel_ok()) FAIL("k_cids_to_recs W=%u case=%s cap %llu: wrote past the records", W, nm, ULL(cap));
    if (!bounds.sentinel_ok()) FAIL("k_part_bounds W=%u case=%s cap %llu: wrote past the bounds", W, nm, ULL(cap));
    if (!send.sentinel_ok()) FAIL("k_part_pack W=%u case=%s cap %llu: wrote past the last send buffer", W, nm, ULL(cap));
    {
        std::vector<RawCid> rc = down(recs.p, roff[W]);
        for (uint32_t p = 0; p < W; p++)
            for (uint64_t k = 0; k <= L.n[p]; k++) {
                RawCid want{};
                if (k < L.n[p]) want = to_raw(uc.lists[p][k]);
                if (!same(rc[roff[p] + k], want)) FAIL("k_cids_to_recs W=%u case=%s: rank %u record %llu", W, nm, p, ULL(k));
            }
        std::vector<uint64_t> b = down(bounds.p, (uint64_t)W * (W + 1));
        for (uint32_t p = 0; p < W; p++)
            for (uint32_t r = 0; r <= W; r++)
                if (b[(uint64_t)p * (W + 1) + r] != bnd[p][r])
                    FAIL("k_part_bounds W=%u case=%s: rank %u bound %u is %llu, expected %llu", W, nm, p, r, ULL(b[(uint64_t)p * (W + 1) + r]), ULL(bnd[p][r]));
        std::vector<unsigned long long> mw = down(mine.p, 2ull * W);
        *overflow = false;
        for (uint32_t p = 0; p < W; p++) {
            if ((mw[2 * p + 1] != 0) != ovf_want[p]) FAIL("k_part_bounds W=%u case=%s cap %llu: rank %u overflow word %llu, expected %d", W, nm, ULL(cap), p, mw[2 * p + 1], (int)ovf_want[p]);
            *overflow |= ovf_want[p];
        }
    }
    {   // headers {min(length, cap), 0, 0, 0, 0} and the first min(length, cap) entries of every piece
        const uint64_t npieces = (uint64_t)W * W;
        DBuf<uint8_t> hdr(npieces * 40);
        k_gather_hdr<<<div_up(npieces * 40, 256), 256, 0, st>>>((const uint8_t*)send.p, npieces, stride * 40, 40, hdr.p);
        std::vector<uint8_t> h = down(hdr.p, npieces * 40);
        std::vector<uint64_t> offs(npieces + 1, 0);
        for (uint64_t s = 0; s < npieces; s++) {
            const uint32_t p = (uint32_t)(s / W), r = (uint32_t)(s % W);
            RawCid want{};
            want.w[0] = std::min(bnd[p][r + 1] - bnd[p][r], cap);
            if (memcmp(&h[s * 40], &want, 40)) {
                uint64_t c;
                memcpy(&c, &h[s * 40], 8);
                FAIL("k_part_bounds W=%u case=%s cap %llu: piece rank %u → %u header says %llu, expected %llu (or other header words are not zero)", W, nm, ULL(cap), p, r, ULL(c), ULL(want.w[0]));
            }
            offs[s + 1] = offs[s] + want.w[0];
        }
        DBuf<uint64_t> d_offs(npieces + 1);
        up(d_offs.p, offs);
        DBuf<uint8_t> comp(offs[npieces] * 40);
        k_compact<<<(unsigned)npieces, 128, 0, st>>>((const uint8_t*)send.p, stride * 40, 40, 40, d_offs.p, comp.p);
        IPCFP_CUDA(cudaGetLastError());
        std::vector<uint8_t> e = down(comp.p, offs[npieces] * 40);
        for (uint64_t s = 0; s < npieces; s++) {
            const uint32_t p = (uint32_t)(s / W), r = (uint32_t)(s % W);
            for (uint64_t j = 0; j < offs[s + 1] - offs[s]; j++) {
                const RawCid want = to_raw(uc.lists[p][bnd[p][r] + j]);
                if (memcmp(&e[(offs[s] + j) * 40], &want, 40)) FAIL("k_part_pack W=%u case=%s cap %llu: piece rank %u → %u entry %llu", W, nm, ULL(cap), p, r, ULL(j));
            }
        }
    }
    if (*overflow) { g_cases++; g_uovf++; return true; }   // finish(): every rank repeats the union with cap = nw_max + 1
    // the receiving ranks: all-to-all of the pieces, counts, merge of the pieces
    DBuf<RawCid> recv(total_cap);
    DBuf<uint64_t> col(W);
    uint32_t nb_max = 0;
    for (uint32_t q = 0; q < W; q++) nb_max = std::max(nb_max, part_lo(q + 1, W) - part_lo(q, W));
    DBuf<uint32_t> flags(total_cap + 64), starts((uint64_t)W * (nb_max + 1) + 64), pos_of(total_cap + 64);
    DBuf<uint64_t> fscan(total_cap + 64), scan_tmp(scan_scratch_elems(total_cap + 64) + 64);
    DBuf<uint8_t> merged(total_cap * 38 + 64);
    std::vector<uint8_t> concat;
    for (uint32_t q = 0; q < W; q++) {
        const uint32_t b0 = part_lo(q, W), nb = part_lo(q + 1, W) - b0;
        IPCFP_CUDA(cudaMemcpy2DAsync(recv.p, stride * 40, send.p + (uint64_t)q * stride, total_cap * 40, stride * 40, W, cudaMemcpyDeviceToDevice, st));
        IPCFP_CUDA(cudaMemsetAsync(flags.p, 0, (total_cap + 64) * 4, st));
        IPCFP_CUDA(cudaMemsetAsync(merged.p, SENT, total_cap * 38 + 64, st));
        k_part_counts<<<1, 256, 0, st>>>(recv.p, W, cap, col.p); IPCFP_LAUNCH_CHECK();
        const unsigned g = div_up(total_cap, 256);
        const RawCid* lists = recv.p + 1;
        k_merge_starts<<<g, 256, 0, st>>>(lists, col.p, W, stride, starts.p, b0, nb); IPCFP_LAUNCH_CHECK();
        k_merge_rank<<<g, 256, 0, st>>>(lists, col.p, W, stride, starts.p, pos_of.p, flags.p, b0, nb); IPCFP_LAUNCH_CHECK();
        exclusive_scan_u32(flags.p, fscan.p, total_cap, (uint64_t*)(mine.p + 2 * q), scan_tmp.p, st);
        k_merge_emit38<<<g, 256, 0, st>>>(lists, col.p, W, stride, pos_of.p, flags.p, fscan.p, merged.p); IPCFP_LAUNCH_CHECK();
        std::vector<uint64_t> c = down(col.p, W);
        for (uint32_t p = 0; p < W; p++)
            if (c[p] != bnd[p][q + 1] - bnd[p][q]) FAIL("k_part_counts W=%u case=%s: rank %u, piece of rank %u counts %llu, expected %llu", W, nm, q, p, ULL(c[p]), ULL(bnd[p][q + 1] - bnd[p][q]));
        const uint64_t n_part = down1(mine.p + 2 * q);
        std::vector<uint8_t> m = down(merged.p, total_cap * 38 + 64);
        std::vector<uint8_t> want;
        for (const Cid38& x : U)
            if (bucket_h(x) >= plo_h(q, W) && bucket_h(x) < plo_h(q + 1, W)) want.insert(want.end(), x.begin(), x.end());
        if (n_part * 38 != want.size()) FAIL("k_merge_emit38 W=%u case=%s: rank %u partition of %llu CIDs, expected %zu", W, nm, q, ULL(n_part), want.size() / 38);
        for (uint64_t i = 0; i < n_part; i++)
            if (memcmp(&m[38 * i], &want[38 * i], 38)) FAIL("k_merge_emit38 W=%u case=%s: rank %u partition entry %llu differs", W, nm, q, ULL(i));
        for (uint64_t b = 38 * n_part; b < m.size(); b++)
            if (m[b] != SENT) FAIL("k_merge_emit38 W=%u case=%s: rank %u wrote byte %llu, past its partition", W, nm, q, ULL(b));
        concat.insert(concat.end(), m.begin(), m.begin() + 38 * n_part);
    }
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (!recv.sentinel_ok() || !col.sentinel_ok() || !mine.sentinel_ok()) FAIL("k_part_counts W=%u case=%s: wrote past its buffers", W, nm);
    if (!starts.sentinel_ok() || !flags.sentinel_ok() || !pos_of.sentinel_ok() || !merged.sentinel_ok()) FAIL("k_merge_rank W=%u case=%s: wrote past its buffers", W, nm);
    if (concat != flat38(U)) FAIL("k_merge_emit38 W=%u case=%s: the partitions in rank order are not the union", W, nm);
    g_cases++;
    return true;
}

// forced_cap: 0 = union_piece_cap_default
static bool run_union(const UCase& uc, uint64_t forced_cap, cudaStream_t st) {
    std::vector<Cid38> U;
    for (auto& l : uc.lists) {
        for (size_t i = 1; i < l.size(); i++)
            if (!ukey_less(l[i - 1], l[i])) FAIL("harness W=%u case=%s: a local list is not sorted and unique", uc.W, uc.name.c_str());
        U.insert(U.end(), l.begin(), l.end());
    }
    std::sort(U.begin(), U.end(), ukey_less);
    U.erase(std::unique(U.begin(), U.end()), U.end());
    ULists L(uc);
    if (forced_cap == 0) {
        if (!run_replicated(uc, L, U, st)) return false;
        g_cases++;
    }
    const uint64_t cap = forced_cap ? forced_cap : union_piece_cap_default(L.nw_max, uc.W);
    bool ovf = false;
    if (!run_partitioned(uc, L, U, cap, &ovf, st)) return false;
    if (ovf) {
        if (!run_partitioned(uc, L, U, L.nw_max + 1, &ovf, st)) return false;
        if (ovf) FAIL("k_part_bounds W=%u case=%s: the retry at nw_max + 1 overflowed", uc.W, uc.name.c_str());
    }
    return true;
}

static Cid38 cid_in_bucket(uint32_t b, const uint8_t* prefix = FILECOIN_PREFIX) {
    Cid38 c;
    memcpy(c.data(), prefix, 6);
    for (int q = 0; q < 32; q++) c[6 + q] = (uint8_t)rnd();
    c[6] = (uint8_t)(b >> 8);
    c[7] = (uint8_t)b;
    return c;
}
static std::vector<Cid38> sorted_unique(std::vector<Cid38> v) {
    std::sort(v.begin(), v.end(), ukey_less);
    v.erase(std::unique(v.begin(), v.end()), v.end());
    return v;
}

static bool unions(uint32_t W, cudaStream_t st) {
    const bool big = W >= 64;
    const uint64_t per = big ? 60 : 700;   // CIDs per list
    auto mk = [&](const std::string& name, std::vector<std::vector<Cid38>> lists) {
        UCase uc;
        uc.name = name;
        uc.W = W;
        for (auto& l : lists) uc.lists.push_back(sorted_unique(l));
        return uc;
    };
    auto pool = [&](uint64_t n) {
        std::vector<Cid38> p(n);
        for (auto& c : p) c = cid_in_bucket((uint32_t)(rnd() % 65536));
        return p;
    };
    std::vector<UCase> cases;
    cases.push_back(mk("empty lists", std::vector<std::vector<Cid38>>(W)));
    {
        std::vector<std::vector<Cid38>> l(W);
        l[0] = pool(per);
        cases.push_back(mk("one list on rank 0", l));
        std::vector<std::vector<Cid38>> l2(W);
        l2[W - 1] = pool(per);
        cases.push_back(mk("one list on the last rank", l2));
    }
    cases.push_back(mk("identical lists", std::vector<std::vector<Cid38>>(W, pool(per))));
    {
        std::vector<std::vector<Cid38>> l(W);
        for (auto& x : l) x = pool(per);
        cases.push_back(mk("disjoint lists", l));
    }
    {
        const std::vector<Cid38> p = pool(per * 2);
        std::vector<std::vector<Cid38>> l(W);
        for (auto& x : l)
            for (uint64_t k = 0; k < per; k++) x.push_back(p[rnd() % p.size()]);
        cases.push_back(mk("heavy overlap", l));
    }
    {   // digests starting 0x0000 and 0xffff, and just below / at the first bucket of every rank; shared by neighbouring ranks
        std::vector<Cid38> edge;
        for (uint32_t r = 0; r < W; r++) {
            if (plo_h(r, W)) edge.push_back(cid_in_bucket(plo_h(r, W) - 1));
            edge.push_back(cid_in_bucket(plo_h(r, W)));
        }
        for (int k = 0; k < 3; k++) { edge.push_back(cid_in_bucket(0)); edge.push_back(cid_in_bucket(0xffff)); }
        std::vector<std::vector<Cid38>> l(W);
        for (uint32_t r = 0; r < W; r++)
            for (uint64_t i = 0; i < edge.size(); i++)
                if ((i + r) % 3 != 0) l[r].push_back(edge[i]);
        cases.push_back(mk("bucket edges", l));
    }
    {   // one bucket holds most CIDs of every list
        const uint64_t m = big ? 12 : 150;
        const uint32_t hot = (uint32_t)(rnd() % 65536);
        std::vector<Cid38> hotp(m * 2);
        for (auto& c : hotp) c = cid_in_bucket(hot);
        std::vector<std::vector<Cid38>> l(W);
        for (auto& x : l) {
            for (uint64_t k = 0; k < m; k++) x.push_back(hotp[rnd() % hotp.size()]);
            for (uint64_t k = 0; k < m / 4; k++) x.push_back(cid_in_bucket((uint32_t)(rnd() % 65536)));
        }
        cases.push_back(mk("one hot bucket", l));
    }
    {   // one rank's list holds CIDs of another prefix (the raw codec), some with the digests of other ranks' CIDs
        const std::vector<Cid38> p = pool(per * 2);
        std::vector<std::vector<Cid38>> l(W);
        for (auto& x : l)
            for (uint64_t k = 0; k < per / 2; k++) x.push_back(p[rnd() % p.size()]);
        l[W / 2].clear();
        for (uint64_t k = 0; k < per; k++) {
            Cid38 c = rnd() % 2 ? p[rnd() % p.size()] : cid_in_bucket((uint32_t)(rnd() % 65536));
            memcpy(c.data(), RAW_SHA_PREFIX, 6);
            l[W / 2].push_back(c);
        }
        cases.push_back(mk("another prefix on one rank", l));
    }
    {   // one list much longer than the others, all of it in rank 0's buckets: that piece overflows the default slot from W = 5 on
        std::vector<std::vector<Cid38>> l(W);
        for (auto& x : l) x = pool(8);
        l[0].clear();
        for (uint64_t k = 0; k < (big ? 1100u : 3000u); k++) l[0].push_back(cid_in_bucket((uint32_t)(rnd() % plo_h(1, W))));
        for (uint32_t r = 1; r < W; r += 7) l[r].insert(l[r].end(), l[0].begin(), l[0].begin() + 5);
        cases.push_back(mk("one long list", l));
    }
    for (const UCase& uc : cases)
        if (!run_union(uc, 0, st)) return false;
    // forced slot capacities: the overflow words and headers, then the retry
    for (uint64_t cap : {1ull, 3ull})
        for (size_t i : {size_t(1), size_t(5), size_t(6)}) {
            UCase uc = cases[i];
            uc.name += ", forced cap " + std::to_string(cap);
            if (!run_union(uc, cap, st)) return false;
        }
    return true;
}

// ================================================================== real execution orders from a file
// file: u32 n_cases, then per case u32 name length, name, u64 nraw, nraw × 38 bytes (the raw message list)
// out:  per case and world size: u32 W, u64 n_exec, n_exec × 38 bytes (the rebuilt execution order)
static bool real_orders(const char* in_path, const char* out_path, const std::vector<uint32_t>& worlds, cudaStream_t st) {
    FILE* f = fopen(in_path, "rb");
    if (!f) FAIL("cannot open %s", in_path);
    FILE* o = fopen(out_path, "wb");
    if (!o) { fclose(f); FAIL("cannot open %s", out_path); }
    uint32_t nc = 0;
    bool ok = fread(&nc, 4, 1, f) == 1;
    for (uint32_t c = 0; ok && c < nc; c++) {
        uint32_t ln = 0;
        uint64_t nraw = 0;
        ok = fread(&ln, 4, 1, f) == 1;
        std::string name(ln, ' ');
        ok = ok && fread(&name[0], 1, ln, f) == ln && fread(&nraw, 8, 1, f) == 1;
        std::vector<Cid38> cids(nraw);
        for (uint64_t i = 0; ok && i < nraw; i++) ok = fread(cids[i].data(), 1, 38, f) == 38;
        if (!ok) break;
        XCase xc;
        xc.name = "message lists " + name;
        for (const Cid38& x : cids) xc.raw.push_back(to_raw(x));
        for (uint32_t W : worlds) {
            xc.W = W;
            xc.nseg = equal_slices(W, nraw);
            std::vector<RawCid> order;
            if (!run_exchange(xc, st, &order)) { ok = false; break; }
            const uint64_t n = order.size();
            fwrite(&W, 4, 1, o);
            fwrite(&n, 8, 1, o);
            for (const RawCid& r : order) fwrite(to_38(r).data(), 1, 38, o);
        }
    }
    fclose(f);
    if (fclose(o) != 0) FAIL("cannot write %s", out_path);
    if (!ok) FAIL("real execution orders: stopped (a disagreement above, or a short file %s)", in_path);
    return true;
}

int main(int argc, char** argv) {
    try {
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
            fprintf(stderr, "FAIL: no CUDA device\n");
            return 1;
        }
        {   // the library's setting (store.cu): freed stream-ordered memory stays in the pool for the next allocation
            cudaMemPool_t mp;
            uint64_t thr = UINT64_MAX;
            if (cudaDeviceGetDefaultMemPool(&mp, 0) == cudaSuccess) cudaMemPoolSetAttribute(mp, cudaMemPoolAttrReleaseThreshold, &thr);
        }
        cudaStream_t st;
        IPCFP_CUDA(cudaStreamCreate(&st));
        const std::vector<uint32_t> worlds = {1, 2, 3, 5, 8, 31, 32, 33, 64, 100, MAX_WORLD};
        bool ok = true;
        for (uint32_t W : worlds) {
            ok = exchanges(W, st) && unions(W, st);
            if (!ok) break;
        }
        if (ok && argc >= 3) ok = real_orders(argv[1], argv[2], worlds, st);
        IPCFP_CUDA(cudaStreamDestroy(st));
        if (!ok) return 1;
        printf("ok: the exchange, select, fetch and union kernels equal the CPU references at world sizes 1-%u in %llu cases (%llu exchanges raised "
               "their overflow word, %llu partitioned unions overflowed a piece)\n", MAX_WORLD, ULL(g_cases), ULL(g_xovf), ULL(g_uovf));
        return 0;
    } catch (const Error& e) {
        fprintf(stderr, "FAIL: %s\n", e.msg.c_str());
        return 1;
    }
}
