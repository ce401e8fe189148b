// pass1_ring.cuh — EXPERIMENT (round 2): pass 1 with a per-lane shared-memory ring fed by cp.async.
//
// Why: k_pass1 is bound by the dependent chain "load 16-byte window → parse head → next address": most warp time is spent
// waiting on the first use of a window (long_scoreboard), with neither DRAM nor issue saturated.
// Here every lane streams its node through a private ring of NSLOT chunks of CH bytes (chunk-aligned in the arena, so
// cp.async's 16-byte alignment holds for any block offset): chunks are requested NSLOT-1 ahead of the parser, windows
// come from shared memory (≈ 30 cycles) and L1 is bypassed (cp.async.cg). Only the fast path reads the ring; the strict
// per-event fallback, the topic comparison and nodes with links keep reading the arena.
#pragma once
#include "events_items.cuh"

namespace ipcfp {

// Device: cp.async / ld.shared through the 32-bit shared-window address of the ring. Host build (tests/host_fuzz): the ring is
// ordinary memory and the copies are modelled ADVERSARIALLY — a request poisons its slot at once and delivers the bytes only when
// a wait_group lets it complete — so a missing wait, a slot reused too early or a wrong offset shows up as wrong bytes.
template <int CH, int NSLOT>
struct RingWin {
    static constexpr uint32_t RING = CH * NSLOT;
    static_assert((RING & (RING - 1)) == 0 && CH % 16 == 0 && NSLOT >= 2 && NSLOT <= 4, "ring geometry");
    uint8_t* sp;           // generic pointer to this lane's ring (shared memory on the device)
    const uint8_t* g0;     // arena address of chunk 0 (CH-aligned, ≤ block start)
    const uint8_t* gend;   // end of the arena allocation: nothing is read at or past it
    uint32_t skew;         // block start − g0: node offset x lives at ring offset (x + skew) mod RING
    uint32_t nchunks;      // chunks covering the node plus the 24-byte over-read of a window
    uint32_t issued;       // chunks requested so far (chunk k → slot k mod NSLOT)
    uint32_t done;         // chunks known to have landed
#ifndef __CUDA_ARCH__
    struct Pending { uint8_t* dst; const uint8_t* src; uint32_t valid; };
    Pending pend[8];
    uint32_t npend;
#endif

    __device__ __forceinline__ void init(uint8_t* ring, const uint8_t* p, uint32_t len, const uint8_t* gend_) {
        sp = ring;
        g0 = (const uint8_t*)((uintptr_t)p & ~(uintptr_t)(CH - 1));
        gend = gend_;
        skew = (uint32_t)(p - g0);
        nchunks = (skew + len + 32 + CH - 1) / CH;
        issued = done = 0;
#ifndef __CUDA_ARCH__
        npend = 0;
#endif
    }
    __device__ __forceinline__ void issue_one() {
        // the slot being reused still has an older request aimed at it (chunk issued − NSLOT) unless that one has completed: two
        // copies in flight to the same bytes may land in either order, so make sure at most NSLOT − 1 requests are pending
        if (issued >= (uint32_t)NSLOT) {
            wait_pending<NSLOT - 1>();
            if (done + (NSLOT - 1) < issued) done = issued - (NSLOT - 1);
        }
        const uint8_t* src = g0 + (size_t)issued * CH;
        uint8_t* dstp = sp + (issued % NSLOT) * CH;
#ifdef __CUDA_ARCH__
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(dstp);
        if (src + CH <= gend) {
#pragma unroll
            for (int k = 0; k < CH / 16; k++) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16 * k), "l"(src + 16 * k) : "memory");
        } else {   // last chunk of the arena: read only what exists, zero-fill the rest
#pragma unroll
            for (int k = 0; k < CH / 16; k++) {
                const uint8_t* s = src + 16 * k;
                long long left = gend - s;
                uint32_t sz = left >= 16 ? 16u : (left > 0 ? (uint32_t)left : 0u);
                if (sz == 0) s = gend - 16;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + 16 * k), "l"(s), "r"(sz) : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
#else
        long long left = gend - src;
        pend[npend++] = Pending{dstp, src, left >= (long long)CH ? (uint32_t)CH : (left > 0 ? (uint32_t)left : 0u)};
        for (int k = 0; k < CH; k++) dstp[k] = 0xCD;          // in flight: the slot holds garbage until a wait completes the request
#endif
        issued++;
    }
    template <int N> __device__ __forceinline__ void wait_pending() {
#ifdef __CUDA_ARCH__
        asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
#else
        while (npend > (uint32_t)N) {
            Pending q = pend[0];
            for (uint32_t k = 0; k < (uint32_t)CH; k++) q.dst[k] = k < q.valid ? q.src[k] : 0;
            for (uint32_t k = 1; k < npend; k++) pend[k - 1] = pend[k];
            npend--;
        }
#endif
    }
    // slots of chunks below lo_chunk are free: keep NSLOT chunks requested from there on
    __device__ __forceinline__ void top_up(uint32_t lo_chunk) {
        while (issued < nchunks && issued < lo_chunk + NSLOT) issue_one();
    }
    // chunks 0..hi_chunk must have landed before they are read
    __device__ __forceinline__ void need(uint32_t hi_chunk) {
        if (hi_chunk < done) return;
        uint32_t later = issued - 1 - hi_chunk;          // requests made after hi_chunk may stay in flight
        if (later >= 3) { wait_pending<3>(); done = issued - 3; }
        else if (later == 2) { wait_pending<2>(); done = issued - 2; }
        else if (later == 1) { wait_pending<1>(); done = issued - 1; }
        else { wait_pending<0>(); done = issued; }
    }
    __device__ __forceinline__ uint2 lds(uint32_t off) const {
        uint2 v;
#ifdef __CUDA_ARCH__
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"((uint32_t)__cvta_generic_to_shared(sp) + (off & (RING - 1))));
#else
        const uint8_t* q = sp + (off & (RING - 1));
        v.x = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
        v.y = (uint32_t)q[4] | ((uint32_t)q[5] << 8) | ((uint32_t)q[6] << 16) | ((uint32_t)q[7] << 24);
#endif
        return v;
    }
    // 16 bytes of the node at offset pos (same contract as win_load)
    __device__ __forceinline__ void load(uint32_t pos, uint64_t& w0, uint64_t& w1) {
        const uint32_t a = skew + pos, a0 = a & ~7u;
        top_up(a0 / CH);
        need((a0 + 23) / CH);
        const uint32_t s = (a & 7) * 8;
        const uint2 x0 = lds(a0), x1 = lds(a0 + 8), x2 = lds(a0 + 16);
        const bool up = (s & 32) != 0;
        const uint32_t c0 = up ? x0.y : x0.x, c1 = up ? x1.x : x0.y, c2 = up ? x1.y : x1.x, c3 = up ? x2.x : x1.y, c4 = up ? x2.y : x2.x;
        w0 = (uint64_t)__funnelshift_r(c0, c1, s) | ((uint64_t)__funnelshift_r(c1, c2, s) << 32);
        w1 = (uint64_t)__funnelshift_r(c2, c3, s) | ((uint64_t)__funnelshift_r(c3, c4, s) << 32);
    }
    // generic pointer to node offset 0 for byte-wise reads of the first `upto` bytes (must not wrap: skew + upto ≤ RING)
    __device__ __forceinline__ const uint8_t* head_ptr(uint32_t upto) {
        top_up(0);
        const uint32_t hi = (skew + upto) / CH;
        need(hi < nchunks ? hi : nchunks - 1);
        return sp + skew;
    }
    __device__ __forceinline__ void drain() { wait_pending<0>(); }
};

// Pass 1 for ONE receipt through the ring (the per-lane part of k_pass1_ring). Returns false when the ring path does not take
// the node (malformed head, links = taller AMT, any decode problem): the caller re-decodes it from the arena, which also reports.
template <int CH, int NSLOT>
__device__ __forceinline__ bool pass1_ring_item(RingWin<CH, NSLOT>& ring, const uint8_t* p, uint32_t len, const Matcher& m, WalkOut& wo) {
    wo = WalkOut{0, 0, false};
    bool taken = false;
    Rd r(ring.head_ptr(64), len);               // head of the node byte-wise from the ring (≤ 64 bytes, never wraps)
    uint32_t bw, height;
    uint64_t cnt;
    amt_root_begin(r, 3, bw, height, cnt);
    AmtNodeHdr h;
    amt_node_begin_head(r, bw, h);
    uint32_t nv = rd_array(r);
    if (!r.err && h.nl == 0 && r.pos <= 64) {
        uint32_t pos = r.pos;
        bool bad = false;
        for (uint32_t v = 0; v < nv && !bad; v++) {
            EvLog ev;
            uint32_t nx = fast_stamped_event_t(ring, pos, len, ev);
            if (nx == FAST_FAIL) {               // exact generic decoder, from the arena
                EvLog e2;
                uint32_t err = 0;
                nx = slow_stamped_event(p, pos, len, &e2, &err);
                ev = e2;
                if (err) { bad = true; break; }
            }
            pos = nx;
            if (event_matches(p, ev, m)) {
                wo.any = true;
                wo.nproofs++;
                wo.nbytes += 32 * ev.ntopics + ev.data_len;
            }
        }
        if (!bad) {
            r.pos = pos;
            amt_node_finish(r, h, nv, height);
            taken = !r.err;
        }
    }
    ring.drain();                                // nothing of this lane may still be landing when the CTA retires
    if (!taken) wo = WalkOut{0, 0, false};
    return taken;
}

}  // namespace ipcfp
