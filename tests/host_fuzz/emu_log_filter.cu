// emu_log_filter.cu — the log-filter predicate of the event path (csrc/log_filter.cuh) and the staged pass 1 with it
// (csrc/pass1_stage.cuh, StageLane::step<LogFilter>) EXECUTED ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// Per warp: a random filter (0–4 positions, wildcards, inline and large value sets, inline and large emitter sets, duplicates) built by the
// library's own host builder (log_filter_build), and 32 generated / mutated events-AMT root blocks whose events draw their emitters and
// topics from small pools (so that filters hit): Case B with 1–4 topics, Case A with 0–6 topics, void logs, odd codecs and lengths, data
// of any size, at random offsets of one arena. Properties:
//   1. staged == arena: the warp is driven as k_pass1_stage drives it, the asynchronous copies modelled adversarially (a copy poisons its
//      16 destination bytes at once and delivers only at the next wait); a node the staged path takes gives the arena path's (any,
//      #proofs, #bytes), and every well-formed single-node block is taken — the residency check over every constrained position included;
//   2. per item == oracle: every event of every node the arena decoder accepts, event_matches(LogFilter) against the filter evaluated on
//      the C++ oracle's decode (oracle_decode_event: StampedEvent + extract_evm_log) in plain host code.
//
//   nvcc -std=c++17 -O2 -o emu_log_filter tests/host_fuzz/emu_log_filter.cu oracle/oracle.cpp && ./emu_log_filter [warps] [seed]
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/ipld.cuh"
#ifndef __CUDA_ARCH__
#define prefetch_l2(p) ((void)0)
#endif
#include "../../ipc_filecoin_proofs_b200/csrc/pass1_stage.cuh"

using namespace ipcfp;

extern "C" ipcfp_status oracle_decode_event(const uint8_t* p, uint64_t n, uint64_t* consumed, uint64_t* emitter, uint32_t* some, uint32_t* ntopics,
                                            uint8_t* topics_out, uint64_t topics_cap, uint8_t* data_out, uint64_t data_cap, uint64_t* data_len);

struct HostAsync {
    struct Req { uint8_t* dst; const uint8_t* src; };
    std::vector<Req> pend;
    void copy16(uint8_t* dst, const uint8_t* src) { for (int k = 0; k < 16; k++) dst[k] = 0xCD; pend.push_back(Req{dst, src}); }
    void wait_all() { for (auto& q : pend) for (int k = 0; k < 16; k++) q.dst[k] = q.src[k]; pend.clear(); }
};

static uint64_t rng_state;
static uint64_t rnd() {
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

static const int NPOOL = 6;
static uint8_t POOL[NPOOL][32];   // topic values: an address (12 leading zero bytes), zero-heavy and non-UTF-8 bytes, random
static const uint64_t EMITTERS[] = {5, 24, 255, 1001, 65536, (1ull << 40) + 1001};

static void put_bytes(std::vector<uint8_t>& o, const char* key, uint64_t codec, const uint8_t* v, size_t n) {
    put_head(o, 4, 4); put_head(o, 0, 3);
    put_head(o, 3, strlen(key)); o.insert(o.end(), key, key + strlen(key));
    put_head(o, 0, codec);
    put_head(o, 2, n); o.insert(o.end(), v, v + n);
}
static void make_event(std::vector<uint8_t>& o) {
    put_head(o, 4, 2);
    put_head(o, 0, EMITTERS[rnd() % 6]);
    uint8_t buf[7 * 32];
    std::vector<uint8_t> data(rnd() % 4 == 0 ? 200 + rnd() % 800 : rnd() % 64);
    for (auto& b : data) b = (uint8_t)rnd();
    if (rnd() % 3 == 0) {   // Case A: 0–6 topics (rarely a length that is not a multiple of 32)
        unsigned nt = (unsigned)(rnd() % 7);
        for (unsigned t = 0; t < nt; t++) memcpy(buf + 32 * t, POOL[rnd() % NPOOL], 32);
        size_t len = 32 * nt - (nt && rnd() % 20 == 0 ? 1 : 0);
        put_head(o, 4, 2);
        put_bytes(o, "topics", 0x55, buf, len);
        put_bytes(o, "data", 0x55, data.data(), data.size());
    } else {                // Case B: t1..t(nt), sometimes a bad length, a duplicate key or no d
        unsigned nt = 1 + (unsigned)(rnd() % 4);
        bool dup = rnd() % 10 == 0, has_d = rnd() % 4 != 0;
        put_head(o, 4, nt + (dup ? 1 : 0) + (has_d ? 1 : 0));
        static const char* tk[] = {"t1", "t2", "t3", "t4"};
        for (unsigned t = 0; t < nt; t++) put_bytes(o, tk[t], rnd() % 16 == 0 ? rnd() % 24 : 0x55, POOL[rnd() % NPOOL], rnd() % 40 == 0 ? 31 : 32);
        if (dup) put_bytes(o, tk[rnd() % nt], 0x55, POOL[rnd() % NPOOL], 32);   // a later duplicate key wins
        if (has_d) put_bytes(o, "d", 0x55, data.data(), data.size());
    }
}
static std::vector<uint8_t> make_root(bool& wellformed_single) {
    std::vector<uint8_t> o;
    uint32_t bw = rnd() % 2 ? 5u : 3u, width = 1u << bw, nmax = width < 20 ? width : 20;
    uint32_t n = (uint32_t)(rnd() % (nmax + 1));
    std::vector<uint8_t> bm(bw <= 3 ? 1 : (1u << (bw - 3)), 0);
    for (uint32_t k = 0; k < n;) { uint32_t b = (uint32_t)(rnd() % width); if (!(bm[b / 8] >> (b % 8) & 1)) { bm[b / 8] |= (uint8_t)(1u << (b % 8)); k++; } }
    put_head(o, 4, 4); put_head(o, 0, bw); put_head(o, 0, 0); put_head(o, 0, n);
    put_head(o, 4, 3); put_head(o, 2, bm.size()); o.insert(o.end(), bm.begin(), bm.end());
    put_head(o, 4, 0); put_head(o, 4, n);
    for (uint32_t k = 0; k < n; k++) make_event(o);
    wellformed_single = true;
    return o;
}

// a random filter: its C form (owning its arrays) and the same filter as plain host sets
struct RandFilter {
    std::vector<uint64_t> emitters;
    std::vector<std::vector<uint8_t>> vals;   // per position, 32 bytes per value
    ipcfp_log_filter c;
    std::set<uint64_t> em;
    std::vector<std::set<std::vector<uint8_t>>> pos;   // per position; empty = any
};
static void make_filter(RandFilter& f) {
    memset(&f.c, 0, sizeof f.c);
    f.c.n_positions = (uint32_t)(rnd() % 5);
    f.vals.assign(4, {});
    f.pos.assign(f.c.n_positions, {});
    auto size = [] { const uint64_t s[] = {1, 2, LF_INLINE - 1, LF_INLINE, LF_INLINE + 1, 64, 65, 300}; return s[rnd() % 8]; };
    for (uint32_t k = 0; k < f.c.n_positions; k++) {
        if (rnd() % 3 == 0) continue;   // wildcard
        const uint64_t n = size();
        for (uint64_t j = 0; j < n; j++) {
            uint8_t v[32];
            if (rnd() % 4 == 0) memcpy(v, POOL[rnd() % NPOOL], 32); else for (auto& b : v) b = (uint8_t)rnd();
            if (j && rnd() % 8 == 0) memcpy(v, &f.vals[k][32 * (rnd() % j)], 32);   // duplicates
            f.vals[k].insert(f.vals[k].end(), v, v + 32);
            f.pos[k].insert(std::vector<uint8_t>(v, v + 32));
        }
        f.c.n_values[k] = n;
        f.c.values[k] = f.vals[k].data();
    }
    if (rnd() % 2) {
        const uint64_t n = size();
        for (uint64_t j = 0; j < n; j++) {
            const uint64_t e = rnd() % 3 == 0 ? EMITTERS[rnd() % 6] : rnd();
            f.emitters.push_back(e);
            f.em.insert(e);
        }
        f.c.n_emitters = n;
        f.c.emitters = f.emitters.data();
    }
}
static bool host_matches(const RandFilter& f, uint64_t emitter, uint32_t some, uint32_t ntopics, const uint8_t* topics) {
    if (!some || ntopics < f.c.n_positions) return false;
    if (!f.em.empty() && !f.em.count(emitter)) return false;
    for (uint32_t k = 0; k < f.c.n_positions; k++)
        if (!f.pos[k].empty() && !f.pos[k].count(std::vector<uint8_t>(topics + 32 * k, topics + 32 * k + 32))) return false;
    return true;
}

static uint64_t g_taken = 0, g_wf = 0, g_events = 0, g_hits = 0, g_large = 0;

template <int CH, int NSLOT, int CPP>
static int run(uint64_t warps) {
    using GEO = StageGeom<CH, NSLOT, CPP>;
    std::vector<uint8_t> rings(GEO::WARP_BYTES + 16);
    for (uint64_t w = 0; w < warps; w++) {
        RandFilter rf;
        make_filter(rf);
        LogFilterHost lfh;
        log_filter_build(&rf.c, lfh);
        lfh.place(lfh.dev.data());
        const LogFilter& f = lfh.f;
        if (!lfh.dev.empty()) g_large++;
        std::vector<std::vector<uint8_t>> blks(32);
        std::vector<bool> wfs(32, false), have(32, false);
        std::vector<size_t> off(32, 0);
        std::vector<uint8_t> blob;
        for (int l = 0; l < 32; l++) {
            size_t gap = rnd() % 3 == 0 ? rnd() % 300 : 0;
            for (size_t k = 0; k < gap; k++) blob.push_back((uint8_t)rnd());
            if (rnd() % 16 == 0) continue;
            bool w1;
            blks[l] = make_root(w1);
            if (rnd() % 5 == 0) {
                size_t at = rnd() % blks[l].size();
                switch (rnd() % 3) {
                    case 0: blks[l][at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                    case 1: blks[l].erase(blks[l].begin() + (long)at); break;
                    default: blks[l].insert(blks[l].begin() + (long)at, (uint8_t)rnd()); break;
                }
                if (blks[l].empty()) blks[l].push_back(0x84);
                w1 = false;
            }
            have[l] = true; wfs[l] = w1; off[l] = blob.size();
            blob.insert(blob.end(), blks[l].begin(), blks[l].end());
        }
        const size_t total = 16 + blob.size() + 32 + 512;
        std::vector<uint8_t> arena(total + 256 + 64, 0xEE);
        uint8_t* base = (uint8_t*)(((uintptr_t)arena.data() + 255) & ~(uintptr_t)255);
        memset(base, 0, 16);
        memcpy(base + 16, blob.data(), blob.size());
        memset(base + 16 + blob.size(), 0, 32 + 512);
        const uint8_t* lo_ok = base;
        const uint8_t* hi_ok = base + total;
        // ---- 1. the warp, as k_pass1_stage drives it
        for (auto& b : rings) b = 0xAB;
        uint8_t* rbase = (uint8_t*)(((uintptr_t)rings.data() + 15) & ~(uintptr_t)15);
        FillDesc* desc = (FillDesc*)(rbase + 32 * GEO::ROW);
        StageLane<GEO> L[32];
        for (uint32_t l = 0; l < 32; l++) L[l].init(rbase + l * GEO::ROW, have[l] ? base + 16 + off[l] : nullptr, have[l] ? (uint32_t)blks[l].size() : 0);
        HostAsync as;
        bool oob = false;
        auto fill = [&]() {
            for (uint32_t l = 0; l < 32; l++) desc[l] = L[l].publish();
            for (uint32_t l = 0; l < 32; l++)
                stage_fill_lane<GEO>(desc, rbase, l, [&](uint8_t* d, const uint8_t* s) {
                    if (s < lo_ok || s + 16 > hi_ok || d < rbase || d + 16 > rbase + 32 * GEO::ROW) oob = true; else as.copy16(d, s);
                });
        };
        for (uint32_t k = 0; k + CPP < (uint32_t)NSLOT; k += CPP) fill();
        for (uint64_t guard = 0;; guard++) {
            as.wait_all();
            bool alive = false;
            for (uint32_t l = 0; l < 32; l++) { L[l].landed = L[l].front; alive |= L[l].state != 0; }
            if (!alive) break;
            fill();
            for (uint32_t l = 0; l < 32; l++) L[l].step(f);
            if (guard > 100000) { fprintf(stderr, "LF <%d,%d,%d>: no progress (warp %llu)\n", CH, NSLOT, CPP, (unsigned long long)w); return 1; }
        }
        if (oob) { fprintf(stderr, "LF <%d,%d,%d>: a copy left the arena / the rings (warp %llu)\n", CH, NSLOT, CPP, (unsigned long long)w); return 1; }
        for (uint32_t l = 0; l < 32; l++) {
            if (!have[l]) { if (L[l].taken) { fprintf(stderr, "LF: a lane without a node reports a result\n"); return 1; } continue; }
            const uint8_t* p = base + 16 + off[l];
            const uint32_t len = (uint32_t)blks[l].size();
            Rd r(p, len);
            uint32_t bw, height;
            uint64_t cnt;
            amt_root_begin(r, 3, bw, height, cnt);
            AmtNodeHdr h;
            amt_node_begin(r, bw, h);
            uint32_t nv = rd_array(r);
            // ---- 2. per item: every event the arena decoder reads, against the oracle's decode and the plain predicate
            if (!r.err) {
                Rd r2 = r;
                for (uint32_t v = 0; v < nv && !r2.err; v++) {
                    const uint32_t at = r2.pos;
                    EvLog ev;
                    decode_stamped_event(r2, ev);
                    if (r2.err) break;
                    uint64_t used = 0, em = 0, dl = 0;
                    uint32_t some = 0, nt = 0;
                    std::vector<uint8_t> tp(32 * 8), dt(2048);
                    if (oracle_decode_event(p + at, len - at, &used, &em, &some, &nt, tp.data(), tp.size(), dt.data(), dt.size(), &dl) != IPCFP_OK ||
                        used != r2.pos - at) { fprintf(stderr, "LF: the oracle does not decode an event the device decoder accepts (warp %llu)\n", (unsigned long long)w); return 1; }
                    const bool dev = event_matches(p, ev, f), ref = host_matches(rf, em, some, nt, tp.data());
                    g_events++; g_hits += ref;
                    if (dev != ref) {
                        fprintf(stderr, "LF PER-ITEM MISMATCH warp %llu lane %u event %u: device %d oracle %d (emitter %llu some %u ntopics %u, npos %u)\n",
                                (unsigned long long)w, l, v, dev, ref, (unsigned long long)em, some, nt, rf.c.n_positions);
                        return 1;
                    }
                }
            }
            WalkOut wa{0, 0, false};
            node_events<WALK_COUNT>(r, p, h, nv, 0, f, wa, nullptr);
            amt_node_finish(r, h, nv, height);
            if (L[l].taken) {
                g_taken++;
                const WalkOut& ws = L[l].wo;
                if (r.err || h.nl || ws.any != wa.any || ws.nproofs != wa.nproofs || ws.nbytes != wa.nbytes) {
                    fprintf(stderr, "LF STAGE MISMATCH <%d,%d,%d> warp %llu lane %u: staged (any %d np %u nb %u), arena err %u nl %u (any %d np %u nb %u)\n", CH, NSLOT, CPP,
                            (unsigned long long)w, l, ws.any, ws.nproofs, ws.nbytes, r.err, h.nl, wa.any, wa.nproofs, wa.nbytes);
                    return 1;
                }
            }
            if (wfs[l]) {
                g_wf++;
                if (!L[l].taken) { fprintf(stderr, "LF <%d,%d,%d>: a well-formed single-node block was not taken (warp %llu lane %u)\n", CH, NSLOT, CPP, (unsigned long long)w, l); return 1; }
            }
        }
    }
    return 0;
}

int main(int argc, char** argv) {
    uint64_t warps = argc > 1 ? strtoull(argv[1], nullptr, 10) : 1000;
    rng_state = argc > 2 ? strtoull(argv[2], nullptr, 10) : 0xF117E5ull;
    memset(POOL, 0, sizeof POOL);
    for (int i = 12; i < 32; i++) POOL[0][i] = (uint8_t)rnd();            // an address topic
    for (int i = 0; i < 32; i++) POOL[1][i] = (uint8_t)(i % 3 ? 0 : 0xFF);   // zero bytes and non-UTF-8
    for (int k = 2; k < NPOOL; k++) for (int i = 0; i < 32; i++) POOL[k][i] = (uint8_t)rnd();
    POOL[5][0] = POOL[4][0] ^ 1;                                           // differs from POOL[4] in its first byte only
    memcpy(POOL[5] + 1, POOL[4] + 1, 31);
    if (run<128, 4, 1>(warps) || run<64, 4, 2>(warps) || run<64, 8, 2>(warps) || run<256, 2, 1>(warps)) return 1;
    printf("ok: log filter staged == arena and per item == oracle, 4 geometries x %llu warps: %llu nodes taken (%llu well-formed, all taken), %llu events, %llu matching, %llu warps with a large set\n",
           (unsigned long long)warps, (unsigned long long)g_taken, (unsigned long long)g_wf, (unsigned long long)g_events, (unsigned long long)g_hits, (unsigned long long)g_large);
    return 0;
}
