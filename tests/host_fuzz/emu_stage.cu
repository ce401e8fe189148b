// emu_stage.cu — the shared-memory-staged pass 1 (csrc/pass1_stage.cuh) EXECUTED ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// The per-lane code of k_pass1_stage (StageLane: publish / begin / step / finish, StageWin, stage_fill_lane) is compiled for the
// host and driven exactly as the kernel drives it — prologue fills, then { wait, landed = front, any lane alive?, fill, step } —
// for whole warps of 32 generated / mutated events-AMT root blocks laid out at random offsets of one arena, with the asynchronous
// copies modelled ADVERSARIALLY (a copy poisons its 16 destination bytes at once and delivers only at the next wait), against the
// arena decode sequence the kernel falls back to. Properties: a node the staged path takes is accepted by the arena path with the same
// (any, #proofs, #bytes); every well-formed single-node block IS taken; nothing is read outside [arena base, arena end + 512).
//
//   nvcc -std=c++17 -O2 -o emu_stage tests/host_fuzz/emu_stage.cu && ./emu_stage [warps] [seed]
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
#define IPCFP_STAGE_HOST_STATS 1
static unsigned long long g_stage_events = 0, g_stage_slow_events = 0, g_stage_iters = 0;
#include "../../ipc_filecoin_proofs_b200/csrc/pass1_stage.cuh"

using namespace ipcfp;

// host model of the asynchronous copies: a request poisons its destination at once and delivers only at the wait
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
static uint8_t T0[32], T1[32];
static bool g_canonical = false;   // the named synthetic shape: 8 events of t1, t2, d (32 bytes each), emitter < 2^16, bw 5
static void put_entry(std::vector<uint8_t>& o, uint64_t flags, const char* key, uint64_t codec, size_t vlen, const uint8_t* fixed = nullptr, size_t fixed_len = 32) {
    put_head(o, 4, 4);
    put_head(o, 0, flags);
    put_head(o, 3, strlen(key));
    o.insert(o.end(), key, key + strlen(key));
    put_head(o, 0, codec);
    put_head(o, 2, vlen);
    for (size_t i = 0; i < vlen; i++) o.push_back(fixed && i < fixed_len ? fixed[i] : (uint8_t)rnd());   // (a 33..39-byte value with a fixed 32-byte head: found by ASan)
}
static void make_event(std::vector<uint8_t>& o) {
    if (g_canonical) {
        put_head(o, 4, 2); put_head(o, 0, 1000 + rnd() % 16); put_head(o, 4, 3);
        put_entry(o, 3, "t1", 0x55, 32); put_entry(o, 3, "t2", 0x55, 32); put_entry(o, 3, "d", 0x55, 32);
        return;
    }
    put_head(o, 4, 2);
    static const uint64_t emitters[] = {5, 24, 255, 1001, 1001, 65536, (1ull << 40) + 1001};
    put_head(o, 0, emitters[rnd() % 7]);
    unsigned shape = (unsigned)(rnd() % 8);
    bool hit = rnd() % 6 == 0;
    if (shape == 0) {
        put_head(o, 4, 2);
        uint8_t tp[64]; memcpy(tp, T0, 32); memcpy(tp + 32, T1, 32);
        put_entry(o, 3, "topics", 0x55, hit ? 64 : 32 * (rnd() % 5), hit ? tp : nullptr, 64);
        put_entry(o, 3, "data", 0x55, rnd() % 300);
    } else {
        unsigned nt = 1 + (unsigned)(rnd() % 4);
        if (hit && nt < 2) nt = 2;
        bool has_d = rnd() % 4 != 0;
        put_head(o, 4, nt + (has_d ? 1 : 0));
        static const char* tk[] = {"t1", "t2", "t3", "t4"};
        for (unsigned t = 0; t < nt; t++) put_entry(o, 3, tk[t], rnd() % 16 == 0 ? rnd() % 24 : 0x55, rnd() % 32 == 0 ? rnd() % 40 : 32, hit && t < 2 ? (t ? T1 : T0) : nullptr);
        if (has_d) put_entry(o, 3, "d", 0x55, rnd() % 6 == 0 ? 256 + rnd() % 700 : rnd() % 64);
    }
}
static std::vector<uint8_t> make_root(bool& wellformed_single) {
    std::vector<uint8_t> o;
    uint32_t bw = g_canonical ? 5u : (rnd() % 2 ? 5u : 3u), width = 1u << bw, nmax = width < 20 ? width : 20;
    uint32_t n = g_canonical ? 8u : (uint32_t)(rnd() % (nmax + 1));
    std::vector<uint8_t> bm(bw <= 3 ? 1 : (1u << (bw - 3)), 0);
    for (uint32_t k = 0; k < n;) { uint32_t b = (uint32_t)(rnd() % width); if (!(bm[b / 8] >> (b % 8) & 1)) { bm[b / 8] |= (uint8_t)(1u << (b % 8)); k++; } }
    put_head(o, 4, 4); put_head(o, 0, bw); put_head(o, 0, 0); put_head(o, 0, n);
    put_head(o, 4, 3); put_head(o, 2, bm.size()); o.insert(o.end(), bm.begin(), bm.end());
    put_head(o, 4, 0); put_head(o, 4, n);
    for (uint32_t k = 0; k < n; k++) make_event(o);
    wellformed_single = true;
    return o;
}


template <int CH, int NSLOT, int CPP>
static int run(uint64_t warps, uint64_t* taken_out, uint64_t* wf_out, uint64_t* slow_out) {
    using GEO = StageGeom<CH, NSLOT, CPP>;
    uint64_t taken_n = 0, wf = 0;
    Matcher m;
    memset(&m, 0, sizeof m);
    memcpy(m.t0, T0, 32); memcpy(m.t1, T1, 32);
    m.actor = 1001; m.has_actor = rnd() % 2;
    std::vector<uint8_t> rings(GEO::WARP_BYTES + 16);
    for (uint64_t w = 0; w < warps; w++) {
        // 32 blocks (some lanes without a node) at arbitrary offsets of one arena = [16 pad][blob][32 pad][512 slack], 256-byte aligned base
        std::vector<std::vector<uint8_t>> blks(32);
        std::vector<bool> wfs(32, false), have(32, false);
        std::vector<size_t> off(32, 0);
        std::vector<uint8_t> blob;
        for (int l = 0; l < 32; l++) {
            size_t gap = !g_canonical && rnd() % 3 == 0 ? rnd() % 300 : 0;
            for (size_t k = 0; k < gap; k++) blob.push_back((uint8_t)rnd());
            if (!g_canonical && rnd() % 16 == 0) continue;      // receipt without events root / outside the range
            bool w1;
            blks[l] = make_root(w1);
            unsigned nmut = !g_canonical && rnd() % 4 == 0 ? 1 + (unsigned)(rnd() % 2) : 0;
            for (unsigned k = 0; k < nmut; k++) {
                size_t at = rnd() % blks[l].size();
                switch (rnd() % 4) {
                    case 0: blks[l][at] = (uint8_t)rnd(); break;
                    case 1: blks[l][at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                    case 2: blks[l].erase(blks[l].begin() + (long)at); break;
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
        // ---- the warp, as k_pass1_stage drives it
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
        uint64_t guard = 0;
        for (;;) {
            as.wait_all();
            bool alive = false;
            for (uint32_t l = 0; l < 32; l++) { L[l].landed = L[l].front; alive |= L[l].state != 0; }
            if (!alive) break;
            fill();
            for (uint32_t l = 0; l < 32; l++) L[l].step(m);
            g_stage_iters++;
            if (++guard > 100000) { fprintf(stderr, "STAGE <%d,%d,%d>: no progress (warp %llu)\n", CH, NSLOT, CPP, (unsigned long long)w); return 1; }
        }
        if (oob) { fprintf(stderr, "STAGE <%d,%d,%d>: a copy left the arena / the rings (warp %llu)\n", CH, NSLOT, CPP, (unsigned long long)w); return 1; }
        // ---- every lane against the arena path (the kernel's fallback sequence)
        for (uint32_t l = 0; l < 32; l++) {
            if (!have[l]) { if (L[l].taken) { fprintf(stderr, "STAGE: a lane without a node reports a result\n"); return 1; } continue; }
            const uint8_t* p = base + 16 + off[l];
            const uint32_t len = (uint32_t)blks[l].size();
            Rd r(p, len);
            uint32_t bw, height;
            uint64_t cnt;
            amt_root_begin(r, 3, bw, height, cnt);
            AmtNodeHdr h;
            amt_node_begin(r, bw, h);
            uint32_t nv = rd_array(r);
            WalkOut wa{0, 0, false};
            node_events<WALK_COUNT>(r, p, h, nv, 0, m, wa, nullptr);
            amt_node_finish(r, h, nv, height);
            if (L[l].taken) {
                taken_n++;
                const WalkOut& ws = L[l].wo;
                if (r.err || h.nl || ws.any != wa.any || ws.nproofs != wa.nproofs || ws.nbytes != wa.nbytes) {
                    fprintf(stderr, "STAGE MISMATCH <%d,%d,%d> warp %llu lane %u: staged took the node (any %d np %u nb %u), arena err %u nl %u (any %d np %u nb %u); len %u skew %u\n", CH, NSLOT, CPP,
                            (unsigned long long)w, l, ws.any, ws.nproofs, ws.nbytes, r.err, h.nl, wa.any, wa.nproofs, wa.nbytes, len, L[l].skew);
                    return 1;
                }
            }
            if (wfs[l]) {
                wf++;
                if (!L[l].taken) { fprintf(stderr, "STAGE <%d,%d,%d>: a well-formed single-node block was not taken (warp %llu lane %u, len %u)\n", CH, NSLOT, CPP, (unsigned long long)w, l, len); return 1; }
            }
        }
    }
    *taken_out += taken_n; *wf_out += wf;
    (void)slow_out;
    return 0;
}

int main(int argc, char** argv) {
    uint64_t warps = argc > 1 ? strtoull(argv[1], nullptr, 10) : 3000;
    rng_state = argc > 2 ? strtoull(argv[2], nullptr, 10) : 0xC0FFEEull;
    for (int i = 0; i < 32; i++) { T0[i] = (uint8_t)rnd(); T1[i] = (uint8_t)rnd(); }
    uint64_t taken = 0, wf = 0, slow = 0;
    if (argc > 3) {   // canonical-shape statistics per geometry: iterations per warp and events that left the fast path
        g_canonical = true;
        auto one = [&](const char* name, int rc) { printf("  %s: %llu warp iterations, %llu events, %llu through the arena decoder\n", name, g_stage_iters, g_stage_events, g_stage_slow_events); g_stage_iters = g_stage_events = g_stage_slow_events = 0; return rc; };
        if (one("128x4x1", run<128, 4, 1>(warps, &taken, &wf, &slow)) || one("64x4x2", run<64, 4, 2>(warps, &taken, &wf, &slow)) || one("64x8x2", run<64, 8, 2>(warps, &taken, &wf, &slow)) ||
            one("128x4x2", run<128, 4, 2>(warps, &taken, &wf, &slow)) || one("256x2x1", run<256, 2, 1>(warps, &taken, &wf, &slow)))
            return 1;
        g_canonical = false;
    }
    if (run<128, 4, 1>(warps, &taken, &wf, &slow) || run<64, 4, 2>(warps, &taken, &wf, &slow) || run<64, 8, 2>(warps, &taken, &wf, &slow) || run<128, 4, 2>(warps, &taken, &wf, &slow) ||
        run<256, 2, 1>(warps, &taken, &wf, &slow))
        return 1;
    printf("ok: staged pass 1 == arena pass 1 for 5 geometries x %llu warps: %llu nodes taken by the staged path, %llu well-formed single-node blocks (all taken); %llu events, %llu of them through the arena decoder; %llu warp iterations\n",
           (unsigned long long)warps, (unsigned long long)taken, (unsigned long long)wf, g_stage_events, g_stage_slow_events, g_stage_iters);
    return 0;
}
