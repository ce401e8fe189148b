// walk.cuh — per-item device functions and tables of the message-AMT walk (record_transaction_amts + execution order,
// reference events/generator.rs:148-177, events/utils.rs:48-94). The kernels that drive them are in events.cu; they live
// in a header so that tests/host_fuzz can run the very same code on the CPU against the oracle.
#pragma once
#include <algorithm>
#include <vector>

#include "ipld.cuh"
#include "rawcid.cuh"

namespace ipcfp {

// meta of a frontier item: amt ordinal << 16 | is_root << 8 | level
__device__ __forceinline__ uint32_t make_meta(uint32_t amt, uint32_t is_root, uint32_t level) { return (amt << 16) | (is_root << 8) | level; }

#define AMT_SENTINEL 0xffffffffu

struct Frontier { uint32_t* blk; uint32_t* meta; uint64_t* base; };

// slots (children, or values at level 0) of a node at `base` whose index range intersects [rlo, rhi):
// the share of the message AMTs a shard walks (all ones when not sharded)
__device__ __forceinline__ uint32_t slot_mask(uint64_t base, uint32_t level, uint64_t rlo, uint64_t rhi) {
    uint64_t sub = pow_sat(3, level);
    uint32_t m = 0;
#pragma unroll
    for (uint32_t sl = 0; sl < 8; sl++) {
        uint64_t off = sub == ~0ull ? (sl ? ~0ull : 0) : sub * sl;
        uint64_t cb = base + off < base ? ~0ull : base + off;
        uint64_t ce = cb + sub < cb ? ~0ull : cb + sub;
        if (cb < rhi && ce > rlo) m |= 1u << sl;
    }
    return m;
}

// ---- message-AMT walk: order-preserving level-synchronous BFS (count → scan → expand) -----------------
// A frontier item is one AMT node: block index, meta (amt ordinal << 16 | is_root << 8 | level),
// base index. Every level first counts each item's outputs (from the node's bitmap), an exclusive
// scan assigns output slots, then the node is fully decoded/validated and its children (or, in the
// last round, its values) are written in place — so frontiers and the final value list stay in
// (AMT, index) order, which is the reference's in-order `for_each` order. Leaves of shallow AMTs are
// parked (re-emitted unchanged) until the last round.


__device__ __forceinline__ uint32_t amt_item_count(const StoreView& s, uint32_t blk, uint32_t meta, uint64_t base, uint32_t round, uint32_t last_round,
                                                   const uint64_t* rlo, const uint64_t* rhi) {
    if (meta == AMT_SENTINEL) return 0;
    uint32_t level = meta & 0xff, is_root = (meta >> 8) & 1, amt = meta >> 16;
    if (level == 0 && round < last_round) return 1;  // parked
    uint32_t len;
    const uint8_t* p = store_block(s, blk, len);
    Rd r(p, len);
    if (is_root) { uint32_t bw, h; uint64_t c; amt_root_begin(r, 0, bw, h, c); }
    rd_array_exact(r, 3);
    uint32_t bl;
    uint32_t bo = rd_bytes(r, bl);
    if (r.err || bl != 1) return 0;  // reported by the expand pass
    if (level != 0 || round == last_round) return (uint32_t)__popc((uint32_t)p[bo] & slot_mask(base, level, rlo[amt], rhi[amt]));
    return 0;
}

struct ExpandArgs {
    StoreView store;
    Frontier in;
    const unsigned long long* in_count;
    const uint64_t* out_off;   // exclusive scan of the counts
    uint32_t round, last_round, record;
    uint32_t* wbits;
    unsigned long long* err;   // the message-AMT fault word (tx_err_key)
    Frontier out;              // rounds < last_round
    RawCid* vals;              // last round
    uint32_t cap;
    const uint64_t* rlo;       // per message AMT: index range this call walks
    const uint64_t* rhi;
};
// Eight lanes per frontier item (a bw-3 node has ≤ 8 links or values). Every lane runs the same strict decode of
// the node (same bytes → one memory transaction per group; the decode is a few hundred instructions), then lane j
// resolves link j (hash probe + witness mark) or copies value j — the eight dependent store lookups of a node
// proceed in parallel instead of back to back. No lane depends on another, so there is no intra-group sync.
__device__ __forceinline__ void amt_item_expand(const ExpandArgs& a, uint64_t t, uint32_t j, uint32_t blk, uint32_t meta, uint64_t base, uint32_t expect) {
    if (meta == AMT_SENTINEL) return;
    uint32_t level = meta & 0xff, is_root = (meta >> 8) & 1, amt = meta >> 16;
    uint64_t o = a.out_off[t];
    if (level == 0 && a.round < a.last_round) {  // park
        if (j == 0 && o < a.cap) { a.out.blk[o] = blk; a.out.meta[o] = meta; a.out.base[o] = base; }
        return;
    }
    uint32_t len;
    const uint8_t* p = store_block(a.store, blk, len);
    Rd r(p, len);
    if (is_root) { uint32_t bw, h; uint64_t c; amt_root_begin(r, 0, bw, h, c); }
    AmtNodeHdr h;
    amt_node_begin(r, 3, h);
    uint32_t nv = rd_array(r);
    uint32_t vals_off = r.pos;
    for (uint32_t v = 0; v < nv && !r.err; v++) (void)rd_cid(r);
    amt_node_finish(r, h, nv, level);
    uint64_t eidx = 3ull * (amt >> 1) + 1 + (amt & 1);
    const uint32_t smask = slot_mask(base, level, a.rlo[amt], a.rhi[amt]);
    const uint32_t bm8 = (uint32_t)h.bm.b0 & 0xffu;
    uint32_t produced = 0;   // outputs of the whole node (same value in every lane)
    if (r.err) { if (j == 0) report_tx_error(a.err, (uint32_t)eidx, base, level, DC_DECODE, r.err); }
    else if (h.nl || a.round == a.last_round) {
        produced = (uint32_t)__popc(bm8 & smask);
        if (produced > expect) produced = expect;
        const uint32_t n_items = h.nl ? h.nl : nv;                 // == popc(bm8) after amt_node_finish
        if (j < n_items) {
            uint32_t slot = bm_select(h.bm, j);
            uint32_t rank = (uint32_t)__popc(bm8 & smask & ((1u << slot) - 1u));   // selected items before this one
            if (((smask >> slot) & 1) && rank < expect) {
                uint64_t d = o + rank;
                if (h.nl) {
                    int32_t child = store_lookup(a.store, p + h.links_off + 43 * j + 5);
                    if (child < 0) {   // Blockstore::get of child `slot` fails: met after everything below the earlier slots
                        const uint64_t off = (uint64_t)slot * pow_sat(3, level);
                        report_tx_error(a.err, (uint32_t)eidx, base + off < base ? ~0ull : base + off, level - 1, DC_MISSING, 0);
                        if (d < a.cap) a.out.meta[d] = AMT_SENTINEL;
                    }
                    else {
                        if (a.record) witness_mark(a.store, a.wbits, (uint32_t)child);
                        if (d < a.cap) { a.out.blk[d] = (uint32_t)child; a.out.meta[d] = make_meta(amt, 0, level - 1); a.out.base[d] = base + (uint64_t)slot * pow_sat(3, level); }
                    }
                } else {
                    const uint8_t* src = p + vals_off + 43 * j + 5;
                    RawCid c;
                    c.w[4] = load_u64_any(src) & 0xffffffffffffull;
                    Digest dg = load_digest(src + 6);
                    c.w[0] = dg.w[0]; c.w[1] = dg.w[1]; c.w[2] = dg.w[2]; c.w[3] = dg.w[3];
                    a.vals[d] = c;
                }
            }
        }
    }
    // slots promised by the count pass but not produced (malformed node): neutralise them
    if (a.round < a.last_round) for (uint32_t k = produced + j; k < expect; k += 8) if (o + k < a.cap) a.out.meta[o + k] = AMT_SENTINEL;
    if (a.round == a.last_round) for (uint32_t k = produced + j; k < expect; k += 8) { RawCid z{}; a.vals[o + k] = z; }
}

// ---- dense message-AMT walk ---------------------------------------------------------------------------------
// Message AMTs are built from arrays: index i of an AMT with `count` values exists iff i < count. While every
// node's bitmap agrees with that (checked node by node), the position of a node inside its level and of a value
// inside the execution list is plain index arithmetic, so a level is ONE launch — no count pass, no scan — and
// the number of raw entries is known to the host up front. Any surprise (a bitmap that differs, a decode error,
// a missing block) only raises `fail`: the host then re-walks with the general count → scan → expand kernels
// above, which handle sparse AMTs and produce the error the reference's sequential walk would report.
struct DenseTables;
struct DenseArgs {
    StoreView store;
    Frontier ping, pong;     // round r reads (r even ? ping : pong) and writes the other
    RawCid* vals;
    const uint32_t* fofs;    // [(rounds) * namt] first frontier position of each AMT in each round
    const uint32_t* ftot;    // [rounds] frontier items per round
    const uint64_t* vbase;   // per AMT: position of its first owned value in vals
    const uint64_t* cnt;     // per AMT: root.count
    const uint64_t* lo;      // per AMT: owned index range [lo, hi) ⊆ [0, count)
    const uint64_t* hi;
    uint32_t namt, record;
    uint32_t* wbits;
    uint32_t* fail;
    uint64_t* f_off[2];      // where each frontier item's block is (arena offset, length), by round parity — rounds ≥ 1
    uint32_t* f_len[2];
    const DenseTables* tables;   // the kernels of events.cu read the plan's ok flag and round count here
};
// Eight lanes per node. The walk only has to DETECT anything unusual, not name it, so instead of the sequential
// strict decoder the node is matched against the one byte layout a bw-3 node the strict decoder accepts can have:
//     83  41 <bitmap>  8<nl> <nl × 43-byte link>  8<nv> <nv × 43-byte link>  <end>     (root: 83 <height> <count> first)
// with every link  d8 2a 58 27 00 01 …  — all lanes check the frame, lane j checks (and then resolves or copies) item j.
// Whatever this accepts the strict decoder accepts with the same meaning; whatever it rejects goes to the general walk.
__device__ __forceinline__ void amt_item_dense(const DenseArgs& a, const Frontier& in, const Frontier& out, uint32_t round, uint32_t it, uint32_t j) {
    const uint32_t meta = in.meta[it];
    const uint64_t base = in.base[it];
    const uint32_t level = meta & 0xff, is_root = (meta >> 8) & 1, amt = meta >> 16;
    // where the block is: carried with the frontier item by the level above (same record line its lookup compared);
    // the roots (round 0, seeded by k_setup) go through the store
    uint32_t len;
    const uint8_t* p;
    if (round == 0) p = store_block(a.store, in.blk[it], len);
    else { const uint32_t par = round & 1; len = a.f_len[par][it]; p = a.store.blob + a.f_off[par][it]; }
    uint32_t q0 = 0;                                    // offset of the node inside the block
    if (is_root) {
        Rd r(p, len);
        uint32_t bw, h; uint64_t c;
        amt_root_begin(r, 0, bw, h, c);
        if (r.err) { *a.fail = 1; return; }
        q0 = r.pos;
    }
    if (len < q0 + 5) { *a.fail = 1; return; }         // the smallest node (empty) is 5 bytes
    const uint8_t* q = p + q0;
    const uint32_t nlen = len - q0;
    const uint64_t cnt = a.cnt[amt], lo = a.lo[amt], hi = a.hi[amt];
    const uint32_t sh = 3 * level;                      // a child (a value at level 0) spans 2^sh indices; the host admits sh ≤ 60 only
    uint32_t n_exp = 0;                                 // slots a dense AMT has under this node
    if (cnt > base) { uint64_t n = ((cnt - base - 1) >> sh) + 1; n_exp = n > 8 ? 8u : (uint32_t)n; }
    // the three reads of the node — frame head, values-array head, this lane's item — are issued together from the
    // EXPECTED layout (clamped into the block), then checked: one memory round trip instead of three
    const uint32_t exp_nl = level ? n_exp : 0u;
    const uint32_t tpos = min(4u + 43u * exp_nl, nlen - 1u);
    const uint32_t ipos = min((level ? 4u : 5u) + 43u * j, nlen - min(nlen, 8u));   // never starts past the block: the 8-byte read stays inside block + arena padding
    const uint32_t w = (uint32_t)load_u64_any(q);       // 83 41 bm 8n
    const uint32_t tb = q[tpos];
    const uint64_t iw = load_u64_any(q + ipos);
    const uint32_t bm8 = (w >> 16) & 0xffu, nl = (w >> 24) - 0x80u;
    if ((w & 0xffffu) != 0x4183u || nl != exp_nl || 4u + 43u * nl >= nlen) { *a.fail = 1; return; }   // now tpos is the values head
    const uint32_t nv = tb - 0x80u;
    if (nv > 8u || nlen != 5u + 43u * (nl + nv) || (nl && nv) || (nl && level == 0) || (nv && level != 0) || (uint32_t)__popc(bm8) != nl + nv) { *a.fail = 1; return; }
    if (bm8 != (1u << n_exp) - 1u || (level ? nl : nv) != n_exp) { *a.fail = 1; return; }
    if (j >= n_exp) return;
    const uint8_t* item = q + (level ? 4u : 5u) + 43u * j;   // link j (nv == 0) or value j (nl == 0); == q + ipos for a well-formed node
    if ((iw & 0xffffffffffffull) != 0x010027582ad8ull) { *a.fail = 1; return; }   // d8 2a 58 27 00 01
    const uint64_t cb = base + ((uint64_t)j << sh), ce = cb + (1ull << sh);   // indices under slot j
    if (!(cb < hi && ce > lo)) return;                  // not in this call's share
    if (level) {
        int32_t child = store_lookup(a.store, item + 5);
        if (child < 0) { *a.fail = 1; return; }
        const uint64_t d = (uint64_t)a.fofs[(round + 1) * a.namt + amt] + ((cb >> sh) - (lo >> sh));
        const BlockRec* rec = a.store.recs + child;
        const uint32_t par = (round + 1) & 1;
        out.meta[d] = make_meta(amt, 0, level - 1); out.base[d] = cb;
        a.f_off[par][d] = __ldg(&rec->off); a.f_len[par][d] = __ldg(&rec->len);
        if (a.record) witness_mark(a.store, a.wbits, (uint32_t)child);
    } else {
        const uint8_t* src = item + 5;
        RawCid c;
        c.w[4] = load_u64_any(src) & 0xffffffffffffull;
        Digest dg = load_digest(src + 6);
        c.w[0] = dg.w[0]; c.w[1] = dg.w[1]; c.w[2] = dg.w[2]; c.w[3] = dg.w[3];
        a.vals[a.vbase[amt] + (cb - lo)] = c;
    }
}
// ------------------------------------------------------------------------------------------ host side of the walk
// Share of the concatenated ("raw") message list a call walks: everything, or — sharded — [Nraw*lo/N, Nraw*hi/N), expressed as
// one index range per message AMT. Returns Nraw (the sum of the roots' counts).
inline uint64_t shard_amt_ranges(uint32_t namt, const uint64_t* cnts, bool sharded, uint64_t lo, uint64_t hi, uint64_t n_receipts, uint64_t* range_lo,
                                 uint64_t* range_hi) {
    std::vector<uint64_t> rawbase(namt + 1, 0);
    for (uint32_t k = 0; k < namt; k++) rawbase[k + 1] = rawbase[k] + cnts[k];
    const uint64_t nraw_total = rawbase[namt];
    uint64_t glo = 0, ghi = UINT64_MAX;
    if (sharded) {
        glo = n_receipts ? (uint64_t)((__uint128_t)nraw_total * lo / n_receipts) : 0;
        ghi = n_receipts ? (uint64_t)((__uint128_t)nraw_total * hi / n_receipts) : 0;
    }
    for (uint32_t k = 0; k < namt; k++) {
        uint64_t A0 = rawbase[k], A1 = rawbase[k + 1];
        uint64_t l = glo > A0 ? glo - A0 : 0, h = ghi > A0 ? ghi - A0 : 0;
        if (!sharded) { l = 0; h = UINT64_MAX; }
        else if (glo >= A1 && !(A1 == A0 && glo == A0)) { l = h = 0; }          // nothing of this AMT
        else if (ghi >= A1) h = UINT64_MAX;                                      // reaches the tail: also owns indices ≥ count
        if (h < l) h = l;
        range_lo[k] = l; range_hi[k] = h;
    }
    return nraw_total;
}

// Level layout of the dense walk (see k_amt_dense): per round and AMT the first frontier slot, per AMT the first value slot.
// One implementation for both sides: k_setup plans unsharded calls on the device, the host plans sharded ones (and the CPU
// emulations in tests/host_fuzz). Tables have the fixed capacity below, laid out with stride namt:
//   fofs[r * namt + k]   first frontier position of AMT k in round r
//   ftot[r]              frontier items of round r
//   per_amt              vbase[namt] | cnt[namt] | lo[namt] | hi[namt]
// Returns ok; false: the geometry is not one the dense walk takes (the caller uses the general walk).
#define DENSE_MAX_AMTS 128     // 2 message AMTs per parent block, IPCFP_MAX_PARENTS = 64
#define DENSE_MAX_ROUNDS 21    // heights up to 20
__host__ __device__ inline bool dense_plan(uint32_t namt, const uint32_t* heights, const uint64_t* cnts, const uint64_t* range_lo, const uint64_t* range_hi,
                                           uint64_t frontier_cap, uint64_t max_raw, size_t max_table_bytes, uint32_t* fofs, uint32_t* ftot,
                                           uint64_t* per_amt, uint32_t* rounds_out, uint64_t* nraw_out) {
    *rounds_out = 0; *nraw_out = 0;
    bool ok = namt > 0 && namt <= DENSE_MAX_AMTS;
    uint32_t last_round = 0;
    // a root whose count exceeds what its height can hold (8^(height+1)) is NOT dense by construction: every per-node check of
    // amt_item_dense would pass on a completely full tree while count promises more values than exist — the general walk
    // (which never trusts count) takes those
    for (uint32_t k = 0; ok && k < namt; k++) {
        ok = heights[k] <= 20 && cnts[k] <= (1ull << 40) && cnts[k] <= (1ull << (3 * (heights[k] + 1)));
        last_round = heights[k] > last_round ? heights[k] : last_round;
    }
    if (!ok) return false;
    const uint32_t rounds = last_round + 1;
    uint64_t vb = 0;
    for (uint32_t k = 0; k < namt; k++) {
        const uint64_t c = cnts[k];
        const uint64_t l = range_lo[k] < c ? range_lo[k] : c;
        const uint64_t hc = range_hi[k] < c ? range_hi[k] : c, h = hc > l ? hc : l;
        // an EMPTY share strictly inside an AMT (a shard without a single message): the general walk still follows the
        // path to that position (its range test is "child begins before hi and ends after lo"); leave that corner to it
        if (l == h && l > 0) ok = false;
        per_amt[k] = vb; per_amt[namt + k] = c; per_amt[2ull * namt + k] = l; per_amt[3ull * namt + k] = h;
        vb += h - l;
    }
    for (uint32_t r = 0; ok && r < rounds; r++) {
        uint64_t run = 0;
        for (uint32_t k = 0; k < namt; k++) {
            fofs[(size_t)r * namt + k] = (uint32_t)run;
            const uint32_t hk = heights[k];
            if (r > hk) continue;                              // this AMT is shallower: already finished
            const uint64_t l = per_amt[2ull * namt + k], h = per_amt[3ull * namt + k];
            const uint32_t sh = 3 * (hk - r + 1);              // a node of this round spans 2^sh indices
            uint64_t nodes = r == 0 ? 1 : (l < h ? (sh >= 64 ? 1 : ((h - 1) >> sh) - (l >> sh) + 1) : 0);
            run += nodes;
            if (run > frontier_cap) { ok = false; break; }
        }
        ftot[r] = (uint32_t)run;
    }
    const size_t tbytes = (size_t)rounds * namt * 4 + (size_t)rounds * 4 + 4ull * namt * 8 + 64;
    if (vb > max_raw || tbytes > max_table_bytes) ok = false;
    *rounds_out = rounds; *nraw_out = vb;
    return ok;
}

// a plan as the walk kernels read it from device memory (k_setup writes it, or the host uploads it)
struct DenseTables {
    uint32_t ok, rounds;
    uint64_t nraw;
    uint64_t per_amt[4 * DENSE_MAX_AMTS];
    uint32_t fofs[DENSE_MAX_ROUNDS * DENSE_MAX_AMTS];
    uint32_t ftot[DENSE_MAX_ROUNDS];
};

// the same plan in host vectors
struct DensePlan {
    bool ok = false;
    uint32_t rounds = 0;
    uint64_t nraw = 0;
    std::vector<uint32_t> fofs, ftot;
    std::vector<uint64_t> per_amt;   // vbase | cnt | lo | hi
};
inline DensePlan make_dense_plan(uint32_t namt, const uint32_t* heights, const uint64_t* cnts, const uint64_t* range_lo, const uint64_t* range_hi,
                                 uint64_t frontier_cap, uint64_t max_raw, size_t max_table_bytes) {
    DensePlan plan;
    plan.fofs.assign((size_t)DENSE_MAX_ROUNDS * namt, 0);
    plan.ftot.assign(DENSE_MAX_ROUNDS, 0);
    plan.per_amt.assign(4ull * namt, 0);
    plan.ok = dense_plan(namt, heights, cnts, range_lo, range_hi, frontier_cap, max_raw, max_table_bytes, plan.fofs.data(), plan.ftot.data(),
                         plan.per_amt.data(), &plan.rounds, &plan.nraw);
    plan.fofs.resize((size_t)plan.rounds * namt);
    plan.ftot.resize(plan.rounds);
    return plan;
}

}  // namespace ipcfp
