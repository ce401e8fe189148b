// pass1_stage.cuh — pass 1 (find_matching_events pass 1, reference events/generator.rs:206-239) with the node bytes STAGED
// THROUGH SHARED MEMORY by warp-cooperative, coalesced 16-byte copies.
//
// Why (DESIGN.md §4): the thread-per-node kernel reads each lane's node straight from the arena, so every 8-byte window load of a
// warp touches 32 different 128-byte lines = 32 L1 wavefronts; with ≈ 80 such loads per node the L1 wavefront queue, not HBM, can
// be what the kernel runs at.
//
// Here a warp owns 32 receipts (lane = receipt, as before: DAG-CBOR is sequential, one lane parses one node) but the BYTES travel
// differently: every lane has a ring of NSLOT chunks of CH bytes in shared memory; a fill pass moves, for every node of the warp,
// its next chunk(s) with `cp.async.cg` — CH/16 consecutive lanes copy one node's chunk, i.e. each copy instruction fetches 32/(CH/16)
// whole chunks of consecutive bytes (full sectors, a handful of wavefronts) — and the lanes parse from shared memory
// (≈ 30-cycle loads, no L1 line traffic). One fill pass is always in flight while the lanes parse the previous one's bytes.
// Chunks are CH-aligned in the ARENA (not in the block), so the 16-byte alignment cp.async needs holds for blocks at any offset.
//
// Only the canonical-shape fast path reads the ring. Anything else — an event the fast path declines, an event larger than the
// ring can show at once, a node with links (taller AMT), any decode problem — goes through the same strict arena decoders as
// k_pass1, so results are identical by construction; tests/host_fuzz/emu_stage.cu runs this very code on the CPU (with the
// asynchronous copies modelled adversarially) against the arena path.
#pragma once
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
    // the same without the residency test (the caller has checked that pos + 24 bytes have landed)
    __device__ __forceinline__ void load_resident(uint32_t pos, uint64_t& w0, uint64_t& w1) const {
        const uint32_t a = skew + pos, a0 = a & ~7u;
        const uint32_t s = (a & 7) * 8;
        const uint2 x0 = lds(a0), x1 = lds(a0 + 8), x2 = lds(a0 + 16);
        const bool up = (s & 32) != 0;
        const uint32_t c0 = up ? x0.y : x0.x, c1 = up ? x1.x : x0.y, c2 = up ? x1.y : x1.x, c3 = up ? x2.x : x1.y, c4 = up ? x2.y : x2.x;
        w0 = (uint64_t)__funnelshift_r(c0, c1, s) | ((uint64_t)__funnelshift_r(c1, c2, s) << 32);
        w1 = (uint64_t)__funnelshift_r(c2, c3, s) | ((uint64_t)__funnelshift_r(c3, c4, s) << 32);
    }
    // 32 resident bytes at node offset pos == w[0..3]? The first 8 bytes decide almost every time.
    __device__ __forceinline__ bool eq32_resident(uint32_t pos, const uint64_t w[4]) const {
        const uint32_t a = skew + pos, a0 = a & ~7u, s = (a & 7) * 8;
        const uint2 x0 = lds(a0), x1 = lds(a0 + 8);
        const uint64_t q0 = (uint64_t)x0.x | ((uint64_t)x0.y << 32), q1 = (uint64_t)x1.x | ((uint64_t)x1.y << 32);
        if (((q0 >> s) | ((q1 << 1) << (63 - s))) != w[0]) return false;
        uint64_t a_, b_;
        load_resident(pos + 8, a_, b_);
        if (a_ != w[1] || b_ != w[2]) return false;
        load_resident(pos + 16, a_, b_);
        return b_ == w[3];
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

// ---- lean event decode for pass 1 ------------------------------------------------------------------------------------------
// Pass 1 only needs, per event: does it decode, does it match, and (for the proofs pass 2 will emit) how many topic / data bytes a
// match carries. fast_stamped_event_t + ev_finish + event_matches keep every offset of every key for the emitter of pass 2; this
// variant keeps bit masks and lengths only, compares t1 / t2 (or the head of `topics`) with the filter while the entry is in the
// window, and never looks at the node again — ≈ 3× fewer instructions per event. Same acceptance as fast_stamped_event_t (the entry
// shapes are decoded by the very same expressions), same meaning as ev_finish + event_matches; whatever it declines (LEAN_FAIL) goes
// to the strict arena decoder; LEAN_SHORT = a byte it needs has not landed in the ring yet (res_end = node offset up to which
// bytes are resident).
#define LEAN_FAIL 0xffffffffu
#define LEAN_SHORT 0xfffffffeu
struct LeanOut { bool hit; uint32_t nbytes; };
template <class Win>
__device__ __forceinline__ uint32_t lean_stamped_event(Win& win, uint32_t pos, uint32_t n, uint32_t res_end, const Matcher& m, LeanOut& out) {
    out.hit = false; out.nbytes = 0;
    if (n - pos < 3) return LEAN_FAIL;
    if (pos + 24 > res_end) return LEAN_SHORT;
    uint64_t w0, w1;
    win.load_resident(pos, w0, w1);
    if ((w0 & 0xff) != 0x82) return LEAN_FAIL;
    const uint32_t eb = (uint32_t)(w0 >> 8) & 0xff;
    if (eb >= 0x1b) return LEAN_FAIL;
    const uint32_t enb = eb < 24 ? 0 : (1u << (eb - 24));
    const uint32_t be = __byte_perm((uint32_t)(w0 >> 16), 0, 0x0123);
    const uint32_t earg = enb ? (be >> (32 - 8 * enb)) : eb;
    const uint32_t emin = eb == 24 ? 24u : (eb == 25 ? 0x100u : (eb == 26 ? 0x10000u : 0u));
    if (earg < emin) return LEAN_FAIL;
    const uint32_t hb = (uint32_t)(w0 >> (16 + 8 * enb)) & 0xffu;
    if ((hb & 0xe0) != 0x80 || (hb & 31) >= 24) return LEAN_FAIL;
    const uint32_t ne = hb & 31;
    uint32_t cur = pos + 3 + enb;
    if (cur > n) return LEAN_FAIL;
    const bool actor_ok = !m.has_actor || earg == m.actor;
    uint32_t have = 0, lenok = 0, d_len = 0, tp_len = 0, da_len = 0;
    bool m0 = false, m1 = false, mA = false;
    for (uint32_t e = 0; e < ne; e++) {
        if (n - cur < 5) return LEAN_FAIL;
        if (cur + 24 > res_end) return LEAN_SHORT;
        win.load_resident(cur, w0, w1);
        const uint32_t lo = (uint32_t)w0, hi = (uint32_t)(w0 >> 32), ll = (uint32_t)w1 & 0xffu;
        const uint32_t tidx = (hi & 0xffu) - (uint32_t)'1';
        const uint32_t fl8 = (lo >> 8) & 0xffu;
        bool canon = (lo & 0xffff00ffu) == 0x74620084u && fl8 < 24u && (hi & 0xff00ff00u) == 0x58001800u && tidx < 4u && ((hi >> 16) & 0xffu) >= 24u && ll >= 24u;
        uint32_t kind = tidx, vlen = ll, voff = cur + 9;
        if ((lo & 0xffff00ffu) == 0x64610084u && fl8 < 24u && (hi & 0xffu) == 0x18u && ((hi >> 8) & 0xffu) >= 24u) {
            const uint32_t vb = (hi >> 16) & 0xffu, b7 = hi >> 24, l16 = (b7 << 8) | ll;
            kind = 4;
            if (vb - 0x40u < 0x18u) { vlen = vb - 0x40u; voff = cur + 7; canon = true; }
            else if (vb == 0x58u && b7 >= 24u) { vlen = b7; voff = cur + 8; canon = true; }
            else if (vb == 0x59u && l16 >= 256u) { vlen = l16; voff = cur + 9; canon = true; }
        }
        if (!canon) {
            uint32_t b0 = (uint32_t)w0 & 0xff, fl = (uint32_t)(w0 >> 8) & 0xff, th = (uint32_t)(w0 >> 16) & 0xff;
            if (b0 != 0x84 || fl >= 24) return LEAN_FAIL;
            uint32_t klen = th - 0x60;
            uint32_t k4 = (uint32_t)(w0 >> 24);
            if (klen == 2) {
                uint32_t idx = ((k4 >> 8) & 0xff) - (uint32_t)'1';
                if ((k4 & 0xff) != 't' || idx >= 4) return LEAN_FAIL;
                kind = idx;
            } else if (klen == 1) {
                if ((k4 & 0xff) != 'd') return LEAN_FAIL;
                kind = 4;
            } else if (klen == 6) {
                uint64_t key = (w0 >> 24) | (w1 << 40);
                if ((key & 0xffffffffffffull) != 0x736369706f74ull) return LEAN_FAIL;  // "topics"
                kind = 5;
            } else if (klen == 4) {
                if (k4 != 0x61746164u) return LEAN_FAIL;          // "data"
                kind = 6;
            } else return LEAN_FAIL;
            uint32_t k = 3 + klen;
            uint32_t cb = win_byte(w0, w1, k);
            uint32_t clen;
            if (cb < 24) clen = 1;
            else if (cb == 24 && win_byte(w0, w1, k + 1) >= 24) clen = 2;
            else return LEAN_FAIL;
            k += clen;
            uint32_t vb = win_byte(w0, w1, k);
            uint32_t vh;
            if (vb >= 0x40 && vb < 0x58) { vlen = vb - 0x40; vh = 1; }
            else if (vb == 0x58) { vlen = win_byte(w0, w1, k + 1); vh = 2; if (vlen < 24) return LEAN_FAIL; }
            else if (vb == 0x59) { vlen = (win_byte(w0, w1, k + 1) << 8) | win_byte(w0, w1, k + 2); vh = 3; if (vlen < 256) return LEAN_FAIL; }
            else return LEAN_FAIL;
            voff = cur + k + vh;
        }
        if (voff > n || vlen > n - voff) return LEAN_FAIL;
        // what extract_evm_log (common/evm.rs:13-59) will look at — last duplicate of a key wins (:14-17)
        if (kind < 4) {
            const uint32_t bit = 1u << kind;
            have |= bit;
            lenok = vlen == 32 ? (lenok | bit) : (lenok & ~bit);
            if (kind < 2 && actor_ok) {                      // topic 0 / topic 1 against the filter, while the value is at hand
                bool eq = false;
                if (vlen == 32) {
                    if (voff + 40 > res_end) return LEAN_SHORT;
                    eq = win.eq32_resident(voff, kind == 0 ? m.t0 : m.t1);
                }
                if (kind == 0) m0 = eq; else m1 = eq;
            }
        } else if (kind == 4) { have |= 16; d_len = vlen; }
        else if (kind == 5) {
            have |= 32; tp_len = vlen;
            mA = false;
            if (actor_ok && vlen >= 64 && vlen % 32 == 0) {
                if (voff + 72 > res_end) return LEAN_SHORT;
                mA = win.eq32_resident(voff, m.t0) && win.eq32_resident(voff + 32, m.t1);
            }
        } else { have |= 64; da_len = vlen; }
        cur = voff + vlen;
    }
    // ev_finish + event_matches: `topics` selects Case A (:20-30); Case B = leading t1.. run, every one of them 32 bytes (:45-56)
    if (have & 32) {
        if (tp_len % 32 == 0 && tp_len >= 64 && mA) { out.hit = true; out.nbytes = tp_len + ((have & 64) ? da_len : 0); }
    } else {
        const uint32_t present = have & 15;
        const uint32_t lead = present == 15 ? 4 : (uint32_t)(__ffs((int)(~present & 15)) - 1);
        const uint32_t lead_mask = (1u << lead) - 1;
        if (lead >= 2 && (lenok & lead_mask) == lead_mask && m0 && m1) { out.hit = true; out.nbytes = 32 * lead + ((have & 16) ? d_len : 0); }
    }
    return cur;
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
    // one parse step with the lean decoder (pass 1's count mode): at most one event
    __device__ __forceinline__ void step_lean(const Matcher& m) {
        if (state == 1) {
            const uint32_t need = skew + (len < 64 ? len : 64);
            if (landed * GEO::CH < need && landed < nchunks) return;
            begin();
            if (state == 0) return;
        }
        if (state != 2) return;
        if (vi >= nv) { finish(); return; }
        StageWin<GEO> win{ring, skew, landed * GEO::CH, false};
        const uint32_t res_end = landed * GEO::CH - skew;    // node offset up to which bytes have landed (landed ≥ 1 here: the header was read)
        LeanOut lo;
        uint32_t nx = lean_stamped_event(win, cur, len, res_end, m, lo);
        if (nx == LEAN_SHORT && landed != front) return;      // the pass in flight brings more
        if (nx >= LEAN_SHORT) {                               // declined, or larger than the ring can show: the exact decoder, from the arena
            EvLog e2;
            uint32_t err = 0;
#if defined(IPCFP_STAGE_HOST_STATS) && !defined(__CUDA_ARCH__)
            g_stage_slow_events++;
#endif
            nx = slow_stamped_event(p, cur, len, &e2, &err);
            if (err) { state = 0; taken = false; return; }
            lo.hit = event_matches(p, e2, m);
            lo.nbytes = 32 * e2.ntopics + e2.data_len;
        }
#if defined(IPCFP_STAGE_HOST_STATS) && !defined(__CUDA_ARCH__)
        g_stage_events++;
#endif
        if (lo.hit) { wo.any = true; wo.nproofs++; wo.nbytes += lo.nbytes; }
        cur = nx;
        vi++;
        if (vi >= nv) finish();
    }
    // one parse step: at most one event
    __device__ __forceinline__ void step(const Matcher& m) {
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
            if ((!m.has_actor || ev.emitter == m.actor) && ev.some && ev.ntopics >= 2) {   // event_matches, topic bytes from the ring
                const uint32_t o0 = ev.toff[0], o1 = ev.case_a ? ev.toff[0] + 32 : ev.toff[1];
                const uint32_t hi_off = (o0 > o1 ? o0 : o1) + 32 + 8;                      // + the window's over-read
                if (skew + hi_off > win.resident_end) have = false;
                else hit = win.eq32(o0, m.t0) && win.eq32(o1, m.t1);
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
template <int CH, int NSLOT, int CPP, int W, int MINB, int LEAN = 0>
__global__ void __launch_bounds__(32 * W, MINB) k_pass1_stage(Pass1Args a) {
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
        if (LEAN) L.step_lean(a.m); else L.step(a.m);
    }
    // phase 3: results; nodes the staged path did not take are decoded from the arena exactly as k_pass1 does
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
            node_events<WALK_COUNT>(r, p, h, nv, 0, a.m, wo, nullptr, 2u);
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
