// pass1_stage.cuh — pass 1 (find_matching_events pass 1, reference events/generator.rs:206-239) with the node bytes STAGED
// THROUGH SHARED MEMORY by warp-cooperative, coalesced 16-byte copies.
//
// Why (DESIGN.md §4): a kernel whose lanes read their nodes straight from the arena makes every 8-byte window load of a warp touch
// 32 different 128-byte lines = 32 L1 wavefronts; with ≈ 80 such loads per node the L1 wavefront queue, not HBM, can be what the
// kernel runs at.
//
// Here a warp owns 32 receipts (lane = receipt, as before: DAG-CBOR is sequential, one lane parses one node) but the BYTES travel
// differently: every lane has a ring of NSLOT chunks of CH bytes in shared memory; a fill pass moves, for every node of the warp,
// its next chunk(s) with `cp.async.cg` — CH/16 consecutive lanes copy one node's chunk, i.e. each copy instruction fetches 32/(CH/16)
// whole chunks of consecutive bytes (full sectors, a handful of wavefronts) — and the lanes parse from shared memory
// (≈ 30-cycle loads, no L1 line traffic). One fill pass is always in flight while the lanes parse the previous one's bytes.
// Chunks are CH-aligned in the ARENA (not in the block), so the 16-byte alignment cp.async needs holds for blocks at any offset.
//
// Only the canonical-shape fast path reads the ring. Anything else — an event the fast path declines, an event larger than the
// ring can show at once, a node with links (taller AMT), any decode problem — goes through the strict arena decoders of
// events_items.cuh, so results are identical by construction; tests/host_fuzz/emu_stage.cu runs this very code on the CPU (with the
// asynchronous copies modelled adversarially) against the arena path.
#pragma once
#include <type_traits>
#include "events_items.cuh"

namespace ipcfp {

template <int CH_, int NSLOT_, int CPP_> struct StageGeom {
    static constexpr uint32_t CH = CH_, NSLOT = NSLOT_, CPP = CPP_;   // chunk bytes, chunks per ring, chunks filled per node and pass
    static constexpr uint32_t RING = CH * NSLOT;
    static constexpr uint32_t ROW = RING + 16;        // 16-byte aligned rows, 4 banks apart
    static constexpr uint32_t G = CH / 16;            // lanes that copy one chunk
    static constexpr uint32_t NPI = 32 / G;           // nodes served by one copy instruction
    static constexpr uint32_t WARP_BYTES = 32 * ROW + 32 * 16;   // rings + fill descriptors
    static_assert((RING & (RING - 1)) == 0 && CH % 16 == 0 && CH >= 64 && G <= 32 && NSLOT >= 2 && CPP >= 1 && CPP < NSLOT, "stage geometry");
};

// what a lane asks the warp to copy for it in the next fill pass (one 16-byte record per lane in shared memory)
struct __align__(16) FillDesc { uint64_t src; uint32_t front; uint32_t nvalid; };


// window source over a lane's ring (same contract as win_load): sets `shortfall` instead of reading bytes that are not resident
template <class GEO> struct StageWin {
    const uint8_t* ring;       // generic pointer to the lane's row
    uint32_t skew;             // block start − chunk 0 start: node offset x lives at ring offset (x + skew) mod RING
    uint32_t resident_end;     // ring coordinate (skew + node offset) up to which bytes have landed
    bool shortfall;
    __device__ __forceinline__ uint2 lds(uint32_t off) const {
        uint2 v;
#ifdef __CUDA_ARCH__
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"((uint32_t)__cvta_generic_to_shared(ring) + (off & (GEO::RING - 1))));
#else
        const uint8_t* q = ring + (off & (GEO::RING - 1));
        v.x = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
        v.y = (uint32_t)q[4] | ((uint32_t)q[5] << 8) | ((uint32_t)q[6] << 16) | ((uint32_t)q[7] << 24);
#endif
        return v;
    }
    __device__ __forceinline__ void load(uint32_t pos, uint64_t& w0, uint64_t& w1) {
        const uint32_t a = skew + pos, a0 = a & ~7u;
        if (a0 + 24 > resident_end) { shortfall = true; w0 = w1 = 0; return; }
        const uint32_t s = (a & 7) * 8;
        const uint2 x0 = lds(a0), x1 = lds(a0 + 8), x2 = lds(a0 + 16);
        const bool up = (s & 32) != 0;
        const uint32_t c0 = up ? x0.y : x0.x, c1 = up ? x1.x : x0.y, c2 = up ? x1.y : x1.x, c3 = up ? x2.x : x1.y, c4 = up ? x2.y : x2.x;
        w0 = (uint64_t)__funnelshift_r(c0, c1, s) | ((uint64_t)__funnelshift_r(c1, c2, s) << 32);
        w1 = (uint64_t)__funnelshift_r(c2, c3, s) | ((uint64_t)__funnelshift_r(c3, c4, s) << 32);
    }
    // 32 bytes at node offset pos == w[0..3]? (pos + 32 must be resident: checked by the caller)
    __device__ __forceinline__ bool eq32(uint32_t pos, const uint64_t w[4]) {
        uint64_t a, b;
        load(pos, a, b);
        if (a != w[0] || b != w[1]) return false;
        load(pos + 16, a, b);
        return a == w[2] && b == w[3];
    }
};

// event_matches for a log filter on an event the fast path decoded from the ring: hit, or have = false when the topic of a constrained
// position is not resident yet (the residency check of the spec's topics 0 and 1, StageLane::step, over every constrained position)
template <class GEO> __device__ __forceinline__ void stage_match(StageWin<GEO>& win, uint32_t skew, const EvLog& ev, const LogFilter& f, bool& have, bool& hit) {
    if (!lf_candidate(f, ev)) return;
    uint32_t hi_off = 0;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        const uint32_t o = topic_offset(ev, k) + 32 + 8;
        if (k < f.npos && f.nv[k] && o > hi_off) hi_off = o;
    }
    if (skew + hi_off > win.resident_end) { have = false; return; }
    bool ok = true;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        if (ok && k < f.npos && f.nv[k]) {
            const uint32_t o = topic_offset(ev, k);
            uint64_t w[4];
            win.load(o, w[0], w[1]);
            win.load(o + 16, w[2], w[3]);
            ok = lf_value_ok(f, k, w);
        }
    }
    hit = ok;
}

// per-lane state of the staged scan (registers on the device)
template <class GEO> struct StageLane {
    uint8_t* ring;          // this lane's row
    const uint8_t* p;       // the block in the arena (slow paths, final checks)
    const uint8_t* g0;      // arena address of chunk 0 (CH-aligned, ≤ p)
    uint32_t len, skew, nchunks;
    uint32_t front;         // chunks requested so far
    uint32_t landed;        // chunks known to have landed (set at the wait)
    uint32_t cur, vi, nv;   // parse position, events done, events of the node
    uint32_t pc, height;    // node header: bitmap popcount, AMT height (final checks)
    uint32_t state;         // 0 idle (no node / finished), 1 header pending, 2 events
    bool taken;             // the staged path produced this node's result (else: the caller re-decodes from the arena)
    WalkOut wo;

    __device__ __forceinline__ void init(uint8_t* row, const uint8_t* blk, uint32_t blen) {
        ring = row; p = blk; len = blen;
        g0 = (const uint8_t*)((uintptr_t)blk & ~(uintptr_t)(GEO::CH - 1));
        skew = (uint32_t)(blk - g0);
        nchunks = blk ? (skew + blen + 24 + GEO::CH - 1) / GEO::CH : 0;
        front = landed = 0; cur = vi = nv = pc = height = 0;
        state = blk ? 1 : 0;
        taken = false;
        wo = WalkOut{0, 0, false};
    }
    // what the next fill pass should bring: chunks [front, min(nchunks, base + NSLOT)) — never a slot the parser may still read
    __device__ __forceinline__ FillDesc publish() {
        const uint32_t base = (skew + cur) / GEO::CH;
        uint32_t lim = base + GEO::NSLOT;
        if (lim > nchunks) lim = nchunks;
        uint32_t nvalid = state != 0 && lim > front ? lim - front : 0;
        if (nvalid > GEO::CPP) nvalid = GEO::CPP;
        FillDesc d;
        d.src = (uint64_t)(uintptr_t)g0 + (uint64_t)front * GEO::CH;
        d.front = front;
        d.nvalid = nvalid;
        front += nvalid;
        return d;
    }
    // node header from the ring: [bw, height, count, [bmap, [links], [values…   (≤ 64 bytes, contiguous in the ring: skew + 64 ≤ RING)
    __device__ __forceinline__ void begin() {
        Rd r(ring + skew, len);
        uint32_t bw;
        uint64_t cnt;
        amt_root_begin(r, 3, bw, height, cnt);
        AmtNodeHdr h;
        amt_node_begin_head(r, bw, h);
        nv = rd_array(r);
        pc = h.pc;
        cur = r.pos;
        if (r.err || h.nl != 0 || r.pos > 48) { state = 0; return; }   // not a plain single-node AMT: the arena path decides
        state = 2;
    }
    __device__ __forceinline__ void finish() {
        // amt_node_finish for a node without links: values only at height 0, popcount == number of values, no trailing bytes
        state = 0;
        taken = !((nv && height != 0) || pc != nv || cur != len);
    }
    // one parse step: at most one event
    template <class P> __device__ __forceinline__ void step(const P& m) {
        if (state == 1) {
            const uint32_t need = skew + (len < 64 ? len : 64);   // every byte begin() may look at
            if (landed * GEO::CH < need && landed < nchunks) return;   // header bytes not there yet
            begin();
            if (state == 0) return;
        }
        if (state != 2) return;
        if (vi >= nv) { finish(); return; }
        StageWin<GEO> win{ring, skew, landed * GEO::CH, false};
        EvLog ev;
        uint32_t nx = fast_stamped_event_t(win, cur, len, ev);
        bool hit = false, have = false;
        if (!win.shortfall && nx != FAST_FAIL) {
            have = true;
            if constexpr (std::is_same_v<P, Matcher>) {
                if ((!m.has_actor || ev.emitter == m.actor) && ev.some && ev.ntopics >= 2) {   // event_matches, topic bytes from the ring
                    const uint32_t o0 = ev.toff[0], o1 = ev.case_a ? ev.toff[0] + 32 : ev.toff[1];
                    const uint32_t hi_off = (o0 > o1 ? o0 : o1) + 32 + 8;                      // + the window's over-read
                    if (skew + hi_off > win.resident_end) have = false;
                    else hit = win.eq32(o0, m.t0) && win.eq32(o1, m.t1);
                }
            } else {
                stage_match(win, skew, ev, m, have, hit);
            }
        }
        if (!have) {
            // bytes missing (wait for the pass in flight) — unless nothing more can arrive for this position, or the fast
            // path declined the event: then the exact decoder reads it from the arena
            if (win.shortfall || nx != FAST_FAIL) { if (landed != front) return; }
            EvLog e2;
            uint32_t err = 0;
#if defined(IPCFP_STAGE_HOST_STATS) && !defined(__CUDA_ARCH__)
            g_stage_slow_events++;
#endif
            nx = slow_stamped_event(p, cur, len, &e2, &err);
            if (err) { state = 0; taken = false; return; }
            ev = e2;
            hit = event_matches(p, ev, m);
        }
#if defined(IPCFP_STAGE_HOST_STATS) && !defined(__CUDA_ARCH__)
        g_stage_events++;
#endif
        if (hit) { wo.any = true; wo.nproofs++; wo.nbytes += 32 * ev.ntopics + ev.data_len; }
        cur = nx;
        vi++;
        if (vi >= nv) finish();
    }
};

// the copies of one fill pass a single lane performs: for every copy instruction j, node (j·NPI + lane / G), piece (lane mod G)
template <class GEO, class Copy>
__device__ __forceinline__ void stage_fill_lane(const FillDesc* desc, uint8_t* warp_rings, uint32_t lane, Copy&& copy16) {
#pragma unroll
    for (uint32_t j = 0; j < 32 / GEO::NPI; j++) {
        const uint32_t k = j * GEO::NPI + lane / GEO::G, piece = lane % GEO::G;
        const FillDesc d = desc[k];
#pragma unroll
        for (uint32_t r = 0; r < GEO::CPP; r++) {
            if (r < d.nvalid) {
                const uint32_t slot = (d.front + r) & (GEO::NSLOT - 1);
                copy16(warp_rings + k * GEO::ROW + slot * GEO::CH + piece * 16, (const uint8_t*)(uintptr_t)(d.src + (uint64_t)r * GEO::CH + piece * 16));
            }
        }
    }
}

#ifdef __CUDACC__
#ifdef __CUDA_ARCH__
__device__ __forceinline__ void cp_async16(uint8_t* dst_smem, const uint8_t* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src) : "memory");
}
#endif

// W warps per CTA, each with its own rings; no CTA-wide synchronisation anywhere.
template <class P, int CH, int NSLOT, int CPP, int W, int MINB>
__global__ void __launch_bounds__(32 * W, MINB) k_pass1_stage(Pass1ArgsT<P> a) {
#ifdef __CUDA_ARCH__
    using GEO = StageGeom<CH, NSLOT, CPP>;
    extern __shared__ __align__(16) uint8_t stage_smem[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t* rings = stage_smem + (size_t)warp * GEO::WARP_BYTES;
    FillDesc* desc = (FillDesc*)(rings + 32 * GEO::ROW);
    const uint64_t i = a.lo + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    // phase 1: Blockstore::get of the events root (hash probe)
    const bool valid = i < a.hi && a.has_root[i];
    int32_t blk = -1;
    if (valid) {
        blk = store_lookup(a.store, a.events_roots + 38 * i);
        if (blk < 0) report_error(a.err, ST_PASS1, i, DC_MISSING, 0);
    }
    uint32_t len = 0;
    const uint8_t* p = nullptr;
    if (blk >= 0) p = store_block(a.store, (uint32_t)blk, len);
    StageLane<GEO> L;
    L.init(rings + lane * GEO::ROW, p, len);
    __syncwarp();
    auto fill = [&]() {
        desc[lane] = L.publish();
        __syncwarp();
        stage_fill_lane<GEO>(desc, rings, lane, [](uint8_t* d, const uint8_t* s) { cp_async16(d, s); });
        asm volatile("cp.async.commit_group;" ::: "memory");
        __syncwarp();                                  // the descriptors may be rewritten
    };
    // prologue: NSLOT − CPP chunks per node in flight before the first wait (the steady state keeps one pass in flight)
    for (uint32_t k = 0; k + CPP < (uint32_t)NSLOT; k += CPP) fill();
    // phase 2: wait for the previous pass, start the next one, parse what has landed
    for (;;) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();                                  // every lane's copies of the passes so far have landed
        L.landed = L.front;
        if (!__any_sync(0xffffffffu, L.state != 0)) break;
        fill();
        L.step(a.m);
    }
    // phase 3: results; nodes the staged path did not take are decoded from the arena (node_events, walk_events)
    bool matched = false;
    uint32_t bytes = 0, nodes = 0, np_ = 0, nb_ = 0;
    if (blk >= 0) {
        bytes = len + 38; nodes = 1;
        WalkOut wo = L.wo;
        if (!L.taken) {
            wo = WalkOut{0, 0, false};
            Rd r(p, len);
            uint32_t bw, height;
            uint64_t cnt;
            amt_root_begin(r, 3, bw, height, cnt);
            AmtNodeHdr h;
            amt_node_begin(r, bw, h);
            uint32_t nv = rd_array(r);
            node_events<WALK_COUNT, false>(r, p, h, nv, 0, a.m, wo, nullptr);
            amt_node_finish(r, h, nv, height);
            if (r.err) { report_error(a.err, ST_PASS1, i, DC_DECODE, r.err); wo = WalkOut{0, 0, false}; }
            else if (h.nl) {
                uint32_t detail = 0;
                wo = WalkOut{0, 0, false};
                uint32_t rc = walk_events<WALK_COUNT>(a.store_dev, (uint32_t)blk, a.m_dev, nullptr, wo, nullptr, &detail);
                if (rc) { report_error(a.err, ST_PASS1, i, rc, detail); wo = WalkOut{0, 0, false}; }
            }
        }
        matched = wo.any;
        np_ = wo.nproofs; nb_ = wo.nbytes;
    }
    if (i < a.hi) { a.cnt[i - a.lo] = np_; a.nbytes[i - a.lo] = nb_; }
    unsigned b = __ballot_sync(0xffffffffu, matched);
    if (lane == 0) a.match_bits[((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5] = b;
    for (int o = 16; o; o >>= 1) { bytes += __shfl_xor_sync(0xffffffffu, bytes, o); nodes += __shfl_xor_sync(0xffffffffu, nodes, o); }
    if (lane == 0 && nodes) { atomicAdd(a.stats, (unsigned long long)nodes); atomicAdd(a.stats + 1, (unsigned long long)bytes); }
#endif
}
#endif

}  // namespace ipcfp
