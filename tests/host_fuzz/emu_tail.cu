// emu_tail.cu — the fast device decoders against the bytes that FOLLOW a block (TEST INFRASTRUCTURE, no GPU needed).
//
// The fast decoders read past the end of the value they decode on purpose (16-byte windows, 8-byte loads, CH-aligned chunk copies)
// and rely on their bound checks to reject anything that ends past the block. Random or zero bytes after a block rarely look like
// the rest of a value, so an off-by-one in those checks can go unnoticed. Here every canonical encoding E (StampedEvents, HAMT
// nodes with ActorState / Vec<u8> / u64 values, the values themselves, message-AMT nodes) is cut at EVERY prefix length k and the
// block length is set to k, with five different continuations after the cut:
//   0  E[k..]            the encoding's own remainder (what an over-reading decoder would want to see)
//   1  E[k..], one byte changed
//   2  E from its start
//   3  00…
//   4  ff…
// Properties, per (encoding, k, tail):
//   * whenever the fast decoder accepts, the strict decoder accepts with identical outputs (offsets, lengths, hit kind, value offset,
//     EvLog fields, next position);
//   * the strict decoder's outcome is the same under all five tails (it never reads past the block length).
//
// Pairs: fast_stamped_event_t over GlobalWin and over StageWin (the launched 128x4x1 ring holding the first 1..4 CH-aligned chunks of the
// span StageLane copies, skew + len + 24 bytes, i.e. every partial residency of a fill) vs parse_stamped_event; hamt_node_lookup_fast vs hamt_node_lookup for HV_ACTOR_STATE / HV_U8VEC / HV_U64;
// skip_u8vec_fast vs parse_u8vec; skip_u64_fast vs rd_uint; amt_item_dense's node-layout check (csrc/walk.cuh) vs amt_node_begin /
// rd_cid / amt_node_finish.
//
//   nvcc -std=c++17 -O2 -o emu_tail tests/host_fuzz/emu_tail.cu && ./emu_tail [encodings] [seed]
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/ipld.cuh"
#ifndef __CUDA_ARCH__
#define prefetch_l2(p) ((void)0)
#endif
#include "../../ipc_filecoin_proofs_b200/csrc/pass1_stage.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/walk.cuh"

using namespace ipcfp;

static uint64_t rng_state;
static uint64_t rnd() {  // SplitMix64
    uint64_t z = (rng_state += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static void put_head(std::vector<uint8_t>& o, int major, uint64_t v) {
    if (v < 24) o.push_back((uint8_t)(major << 5 | v));
    else if (v < 0x100) { o.push_back((uint8_t)(major << 5 | 24)); o.push_back((uint8_t)v); }
    else if (v < 0x10000) { o.push_back((uint8_t)(major << 5 | 25)); o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); }
    else if (v < 0x100000000ull) { o.push_back((uint8_t)(major << 5 | 26)); for (int s = 24; s >= 0; s -= 8) o.push_back((uint8_t)(v >> s)); }
    else { o.push_back((uint8_t)(major << 5 | 27)); for (int s = 56; s >= 0; s -= 8) o.push_back((uint8_t)(v >> s)); }
}
static void put_cid(std::vector<uint8_t>& o) {
    static const uint8_t head[11] = {0xd8, 0x2a, 0x58, 0x27, 0x00, 0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
    o.insert(o.end(), head, head + 11);
    for (int b = 0; b < 32; b++) o.push_back((uint8_t)rnd());
}

// ---- generators: the canonical shapes of tests/host_fuzz/fuzz_events.cu (no mutations: the cut and the tail are the variation)
static void put_entry(std::vector<uint8_t>& o, uint64_t flags, const char* key, uint64_t codec, size_t vlen) {
    put_head(o, 4, 4);
    put_head(o, 0, flags);
    put_head(o, 3, strlen(key));
    o.insert(o.end(), key, key + strlen(key));
    put_head(o, 0, codec);
    put_head(o, 2, vlen);
    for (size_t i = 0; i < vlen; i++) o.push_back((uint8_t)rnd());
}
static std::vector<uint8_t> make_event() {
    std::vector<uint8_t> o;
    put_head(o, 4, 2);
    static const uint64_t emitters[] = {5, 23, 24, 255, 256, 1001, 65535, 65536, 1ull << 32};
    put_head(o, 0, emitters[rnd() % 9]);
    if (rnd() % 6 == 0) {   // Case A
        put_head(o, 4, 2);
        put_entry(o, 3, "topics", 0x55, 32 * (rnd() % 5));
        put_entry(o, 3, "data", 0x55, rnd() % 300);
    } else {
        unsigned nt = 1 + (unsigned)(rnd() % 4);
        bool has_d = rnd() % 4 != 0;
        put_head(o, 4, nt + (has_d ? 1 : 0));
        static const char* tk[] = {"t1", "t2", "t3", "t4"};
        for (unsigned t = 0; t < nt; t++) put_entry(o, rnd() % 8 == 0 ? rnd() % 24 : 3, tk[t], 0x55, rnd() % 16 == 0 ? rnd() % 40 : 32);
        if (has_d) { size_t dl = rnd() % 5 == 0 ? 256 + rnd() % 300 : (rnd() % 3 == 0 ? rnd() % 24 : rnd() % 100); put_entry(o, 3, "d", 0x55, dl); }
    }
    return o;
}
static void put_u8vec(std::vector<uint8_t>& o) {
    size_t vl = rnd() % 4 == 0 ? 24 + rnd() % 40 : rnd() % 34;
    put_head(o, 4, vl);
    for (size_t b = 0; b < vl; b++) put_head(o, 0, rnd() % 3 == 0 ? rnd() % 24 : 24 + rnd() % 232);
}
static void put_u64(std::vector<uint8_t>& o) {
    static const uint64_t v[] = {0, 23, 24, 255, 256, 65535, 65536, 0xffffffffull, 0x100000000ull};
    put_head(o, 0, rnd() % 2 ? v[rnd() % 9] : rnd() >> (rnd() % 64));
}
static std::vector<uint8_t> make_hamt_node(int vkind, std::vector<std::vector<uint8_t>>& keys, uint32_t& bits) {
    uint32_t np = 1 + (uint32_t)(rnd() % 5);
    bits = 0;
    for (uint32_t k = 0; k < np;) { uint32_t b = (uint32_t)(rnd() % 32); if (!(bits >> b & 1)) { bits |= 1u << b; k++; } }
    std::vector<uint8_t> bf;
    for (int s = 24; s >= 0; s -= 8) if (!bf.empty() || (bits >> s) & 0xff) bf.push_back((uint8_t)(bits >> s));
    std::vector<uint8_t> node;
    put_head(node, 4, 2);
    put_head(node, 2, bf.size());
    node.insert(node.end(), bf.begin(), bf.end());
    put_head(node, 4, np);
    for (uint32_t k = 0; k < np; k++) {
        if (rnd() % 4 == 0) { put_cid(node); continue; }
        uint32_t nk = 1 + (uint32_t)(rnd() % 3);
        put_head(node, 4, nk);
        for (uint32_t j = 0; j < nk; j++) {
            put_head(node, 4, 2);
            std::vector<uint8_t> key(vkind == HV_U8VEC ? 32 : 1 + rnd() % 21);
            for (auto& b : key) b = (uint8_t)rnd();
            keys.push_back(key);
            put_head(node, 2, key.size());
            node.insert(node.end(), key.begin(), key.end());
            if (vkind == HV_ACTOR_STATE) {
                put_head(node, 4, 5);
                put_cid(node); put_cid(node);
                put_head(node, 0, rnd() % 100000);
                size_t bl = rnd() % 12;
                put_head(node, 2, bl);
                for (size_t b = 0; b < bl; b++) node.push_back((uint8_t)rnd());
                if (rnd() % 2) node.push_back(0xf6); else { put_head(node, 2, 3); node.push_back(1); node.push_back(2); node.push_back(3); }
            } else if (vkind == HV_U8VEC) put_u8vec(node);
            else put_u64(node);
        }
    }
    return node;
}
// a bw-3 message-AMT node as the dense walk expects it: level 0 (values) or the root [height 0, count, node]
static std::vector<uint8_t> make_amt_node(bool root, uint32_t& nvals) {
    nvals = 1 + (uint32_t)(rnd() % 8);
    std::vector<uint8_t> o;
    if (root) { put_head(o, 4, 3); put_head(o, 0, 0); put_head(o, 0, nvals); }
    o.push_back(0x83); o.push_back(0x41); o.push_back((uint8_t)((1u << nvals) - 1u));
    o.push_back(0x80);
    put_head(o, 4, nvals);
    for (uint32_t v = 0; v < nvals; v++) put_cid(o);
    return o;
}

// ---- the five continuations: the block is E[0..k) at an arena offset `lead` (mod 16), followed by tail t
struct Layout {
    std::vector<uint8_t> mem;
    uint8_t* base;   // 256-byte aligned: chunk arithmetic of StageLane and the aligned loads see real arena alignment
    uint8_t* p;      // the block
};
static void lay_out(Layout& L, const std::vector<uint8_t>& e, uint32_t k, int tail, uint32_t lead, size_t flip_at, uint8_t flip_x) {
    const size_t total = 256 + 16 + lead + 2 * e.size() + 512;
    L.mem.assign(total + 256, 0xEE);
    L.base = (uint8_t*)(((uintptr_t)L.mem.data() + 255) & ~(uintptr_t)255);
    L.p = L.base + 16 + lead;
    memcpy(L.p, e.data(), k);
    uint8_t* t = L.p + k;
    const size_t room = (size_t)(L.mem.data() + L.mem.size() - t) - 64;
    std::vector<uint8_t> tb;
    if (tail <= 1) { tb.assign(e.begin() + k, e.end()); tb.insert(tb.end(), e.begin(), e.end()); }
    else if (tail == 2) { tb = e; tb.insert(tb.end(), e.begin(), e.end()); }
    if (tail == 1) { size_t at = k < e.size() ? flip_at % (e.size() - k) : 0; if (tb.empty()) tb.push_back(0); tb[at] ^= flip_x; }
    const uint8_t fill = tail == 4 ? 0xff : 0x00;
    for (size_t i = 0; i < room; i++) t[i] = i < tb.size() ? tb[i] : fill;
}

static uint64_t g_runs[8], g_fast[8];
static const char* g_names[8] = {"StampedEvent (GlobalWin)", "StampedEvent (StageWin)", "HAMT node, ActorState", "HAMT node, Vec<u8>", "HAMT node, u64",
                                 "Vec<u8> value", "u64 value", "message-AMT node (dense walk)"};
static int fail(int pair, const std::vector<uint8_t>& e, uint32_t k, int tail, const char* what) {
    fprintf(stderr, "TAIL MISMATCH [%s] k %u of %zu, tail %d: %s\nencoding:", g_names[pair], k, e.size(), tail, what);
    for (size_t i = 0; i < e.size(); i++) fprintf(stderr, " %02x", e[i]);
    fprintf(stderr, "\n");
    return 1;
}
static bool same_ev(const EvLog& a, const EvLog& b) {
    if (a.emitter != b.emitter || a.some != b.some || a.case_a != b.case_a || a.ntopics != b.ntopics || a.data_off != b.data_off || a.data_len != b.data_len) return false;
    for (int q = 0; q < 4; q++) if (a.toff[q] != b.toff[q]) return false;
    return true;
}

// strict outcomes, compared across the five tails
struct StrictEv { uint32_t err, pos; EvLog ev; };
struct StrictHamt { uint32_t err; HamtHit hit; };
struct StrictPos { uint32_t err, pos; uint64_t v; };
struct StrictAmt { uint32_t err, nl, nv, vals_off; };

static int run_event(const std::vector<uint8_t>& e, uint32_t lead) {
    using GEO = StageGeom<128, 4, 1>;   // the geometry k_pass1_stage is launched with (csrc/events.cu)
    std::vector<uint8_t> ring(GEO::ROW + 16);
    uint8_t* rbase = (uint8_t*)(((uintptr_t)ring.data() + 15) & ~(uintptr_t)15);
    const size_t flip_at = rnd();
    Layout L;
    for (uint32_t k = 0; k <= e.size(); k++) {
        StrictEv s0{};
        for (int t = 0; t < 5; t++) {
            lay_out(L, e, k, t, lead, flip_at, 0x01);
            Rd r(L.p, k);
            EvLog s;
            memset(&s, 0, sizeof s);
            parse_stamped_event(r, s);
            StrictEv sc{r.err, r.pos, s};
            if (t == 0) s0 = sc;
            else if (sc.err != s0.err || sc.pos != s0.pos || (!sc.err && !same_ev(sc.ev, s0.ev))) return fail(0, e, k, t, "the strict decoder's outcome depends on the bytes after the block");
            // GlobalWin
            EvLog f;
            memset(&f, 0, sizeof f);
            GlobalWin g{L.p};
            uint32_t np = fast_stamped_event_t(g, 0, k, f);
            g_runs[0]++;
            if (np != FAST_FAIL) {
                g_fast[0]++;
                if (r.err || np != r.pos || !same_ev(f, s)) return fail(0, e, k, t, "fast accepted, strict disagrees");
            }
            // StageWin over the lane's ring as StageLane's copies fill it for a node parsed from its first byte: chunks [0, m) of the
            // CH-aligned span holding the block, m = 1 .. min(nchunks, NSLOT) (publish() never requests more than NSLOT chunks ahead of
            // the parse position), every partial residency a fill pass can leave
            StageLane<GEO> lane;
            lane.init(rbase, L.p, k);
            const uint32_t mmax = lane.nchunks < GEO::NSLOT ? lane.nchunks : GEO::NSLOT;
            for (uint32_t m = 1; m <= mmax; m++) {
                for (uint32_t c = 0; c < GEO::RING; c++) rbase[c] = 0xCD;
                for (uint32_t c = 0; c < m; c++) memcpy(rbase + c * GEO::CH, lane.g0 + (size_t)c * GEO::CH, GEO::CH);
                StageWin<GEO> win{rbase, lane.skew, m * GEO::CH, false};
                EvLog f2;
                memset(&f2, 0, sizeof f2);
                uint32_t np2 = fast_stamped_event_t(win, 0, k, f2);
                g_runs[1]++;
                if (!win.shortfall && np2 != FAST_FAIL) {
                    g_fast[1]++;
                    if (r.err || np2 != r.pos || !same_ev(f2, s)) return fail(1, e, k, t, "staged fast path accepted, strict disagrees");
                }
            }
        }
    }
    return 0;
}

static int run_hamt(const std::vector<uint8_t>& e, int vkind, const std::vector<uint8_t>& key, uint32_t idx, uint32_t lead) {
    const int pair = 2 + vkind;
    const size_t flip_at = rnd();
    Layout L;
    for (uint32_t k = 0; k <= e.size(); k++) {
        StrictHamt s0{};
        for (int t = 0; t < 5; t++) {
            lay_out(L, e, k, t, lead, flip_at, 0x01);
            Rd r(L.p, k);
            HamtHit hit;
            hamt_node_lookup(r, vkind, idx, key.data(), (uint32_t)key.size(), hit);
            if (t == 0) s0 = StrictHamt{r.err, hit};
            else if (r.err != s0.err || hit.kind != s0.hit.kind || hit.val_off != s0.hit.val_off || hit.link_off != s0.hit.link_off)
                return fail(pair, e, k, t, "the strict decoder's outcome depends on the bytes after the block");
            HamtHit fh;
            g_runs[pair]++;
            if (hamt_node_lookup_fast(L.p, k, vkind, idx, key.data(), (uint32_t)key.size(), fh)) {
                g_fast[pair]++;
                if (r.err || fh.kind != hit.kind || fh.val_off != hit.val_off || fh.link_off != hit.link_off) return fail(pair, e, k, t, "fast accepted, strict disagrees");
            }
        }
    }
    return 0;
}

static int run_value(const std::vector<uint8_t>& e, bool u8vec, uint32_t lead) {
    const int pair = u8vec ? 5 : 6;
    const size_t flip_at = rnd();
    Layout L;
    for (uint32_t k = 0; k <= e.size(); k++) {
        StrictPos s0{};
        for (int t = 0; t < 5; t++) {
            lay_out(L, e, k, t, lead, flip_at, 0x01);
            Rd r(L.p, k);
            uint64_t v = 0;
            if (u8vec) { uint32_t fo; v = parse_u8vec(r, fo); } else v = rd_uint(r);
            StrictPos sc{r.err, r.pos, r.err ? 0 : v};
            if (t == 0) s0 = sc;
            else if (sc.err != s0.err || sc.pos != s0.pos || sc.v != s0.v) return fail(pair, e, k, t, "the strict decoder's outcome depends on the bytes after the block");
            uint32_t pos = 0;
            const bool ok = u8vec ? skip_u8vec_fast(L.p, k, pos) : skip_u64_fast(L.p, k, pos);
            g_runs[pair]++;
            if (ok) {
                g_fast[pair]++;
                if (r.err || pos != r.pos) return fail(pair, e, k, t, "fast accepted, strict disagrees");
            }
        }
    }
    return 0;
}

// amt_item_dense on one node: round 0 (the root, through the store record) or round 1 (a level-0 node, through the frontier's
// offset/length); fail flag clear = the layout check accepted. Values land in vals[0..n_exp).
static bool dense_accepts(const uint8_t* base, const uint8_t* p, uint32_t len, bool root, uint64_t cnt, RawCid* vals) {
    BlockRec rec;
    memset(&rec, 0, sizeof rec);
    rec.off = (uint64_t)(p - base);
    rec.len = len;
    uint32_t blk = 0, meta = make_meta(0, root ? 1 : 0, 0), fail = 0, f_len = len;
    uint64_t fbase = 0, f_off = rec.off, lo = 0, hi = UINT64_MAX, vbase = 0;
    DenseArgs a;
    memset(&a, 0, sizeof a);
    a.store.blob = base;
    a.store.recs = &rec;
    a.vals = vals;
    a.vbase = &vbase;
    a.cnt = &cnt;
    a.lo = &lo;
    a.hi = &hi;
    a.namt = 1;
    a.fail = &fail;
    a.f_off[1] = &f_off;
    a.f_len[1] = &f_len;
    Frontier in{&blk, &meta, &fbase}, out{nullptr, nullptr, nullptr};
    for (uint32_t j = 0; j < 8; j++) amt_item_dense(a, in, out, root ? 0 : 1, 0, j);
    return fail == 0;
}
static int run_amt(const std::vector<uint8_t>& e, bool root, uint32_t nvals, uint32_t lead) {
    const int pair = 7;
    const size_t flip_at = rnd();
    Layout L;
    for (uint32_t k = 0; k <= e.size(); k++) {
        StrictAmt s0{};
        for (int t = 0; t < 5; t++) {
            lay_out(L, e, k, t, lead, flip_at, 0x01);
            Rd r(L.p, k);
            if (root) { uint32_t bw, h; uint64_t c; amt_root_begin(r, 0, bw, h, c); }
            AmtNodeHdr h;
            amt_node_begin(r, 3, h);
            uint32_t nv = rd_array(r);
            const uint32_t vals_off = r.pos;
            for (uint32_t v = 0; v < nv && !r.err; v++) (void)rd_cid(r);
            amt_node_finish(r, h, nv, 0);
            StrictAmt sc{r.err, r.err ? 0 : h.nl, r.err ? 0 : nv, r.err ? 0 : vals_off};
            if (t == 0) s0 = sc;
            else if (sc.err != s0.err || sc.nl != s0.nl || sc.nv != s0.nv || sc.vals_off != s0.vals_off)
                return fail(pair, e, k, t, "the strict decoder's outcome depends on the bytes after the block");
            RawCid vals[8];
            memset(vals, 0xA5, sizeof vals);
            g_runs[pair]++;
            if (dense_accepts(L.base + 16, L.p, k, root, nvals, vals)) {
                g_fast[pair]++;
                if (r.err || h.nl != 0 || nv != nvals) return fail(pair, e, k, t, "dense layout check accepted, strict disagrees");
                for (uint32_t v = 0; v < nv; v++) {
                    const uint8_t* c = L.p + vals_off + 43 * v + 5;   // the 38 CID bytes the strict decoder found
                    uint64_t w4 = 0, d[4];
                    memcpy(&w4, c, 6);
                    memcpy(d, c + 6, 32);
                    if (vals[v].w[4] != w4 || memcmp(vals[v].w, d, 32) != 0) return fail(pair, e, k, t, "dense walk took another CID than the strict decoder");
                }
            }
        }
    }
    return 0;
}

int main(int argc, char** argv) {
    const uint64_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 200;
    rng_state = argc > 2 ? strtoull(argv[2], nullptr, 10) : 0x7A11ull;
    uint64_t encodings = 0;
    for (uint64_t it = 0; it < n; it++) {
        const uint32_t lead = (uint32_t)(it % 16);   // every residue of the block start mod 16
        if (run_event(make_event(), lead)) return 1;
        encodings++;
        for (int vkind = 0; vkind < 3; vkind++) {
            std::vector<std::vector<uint8_t>> keys;
            uint32_t bits;
            std::vector<uint8_t> node = make_hamt_node(vkind, keys, bits);
            // the looked-up key: one that is there (its slot may be another: any hit kind), or a stranger; slot present or not
            std::vector<uint8_t> key = !keys.empty() && rnd() % 4 ? keys[rnd() % keys.size()] : std::vector<uint8_t>(vkind == HV_U8VEC ? 32 : 3, (uint8_t)rnd());
            uint32_t idx = (uint32_t)(rnd() % 32);
            if (rnd() % 2) { do idx = (uint32_t)(rnd() % 32); while (!(bits >> idx & 1)); }
            if (run_hamt(node, vkind, key, idx, (lead + 5 * vkind) % 16)) return 1;
            encodings++;
        }
        std::vector<uint8_t> v;
        put_u8vec(v);
        if (run_value(v, true, (lead + 3) % 16)) return 1;
        v.clear();
        put_u64(v);
        if (run_value(v, false, (lead + 7) % 16)) return 1;
        uint32_t nvals;
        const bool root = it % 2;
        std::vector<uint8_t> amt = make_amt_node(root, nvals);
        if (run_amt(amt, root, nvals, (lead + 11) % 16)) return 1;
        encodings += 3;
    }
    uint64_t total = 0;
    for (int q = 0; q < 8; q++) {
        total += g_runs[q];
        printf("  %s: %llu (encoding, k, tail) runs, fast path accepted %llu\n", g_names[q], (unsigned long long)g_runs[q], (unsigned long long)g_fast[q]);
    }
    printf("ok: tail bytes: %llu encodings cut at every length under 5 tails, %llu runs; fast == strict wherever the fast path accepts, strict independent of the tail\n",
           (unsigned long long)encodings, (unsigned long long)total);
    return 0;
}
