// storage.cuh — per-proof / per-lookup device functions of the storage path (K5), see storage.cu for the kernels and the host
// side. They live in a header so that tests/host_fuzz can run the very same code on the CPU against the oracle:
//   reference src/proofs/storage/generator.rs:29-178  generate_storage_proof
//   reference src/proofs/storage/decode.rs:36-97      read_storage_slot (shape sniffing A1,A2,A3,B1,B2,C)
//   reference src/proofs/common/decode.rs:17-124      get_actor_state, parse_evm_state, HeaderLite
//   fvm_ipld_hamt 0.10 [UPSTREAM]                     Hamt::get with SHA-256 key hashing (K2b)
#pragma once
#include "hashes.cuh"
#include "ipld.cuh"

namespace ipcfp {

// Distinct blocks one storage proof can record, on the longest path the decode contract (DESIGN.md §3) accepts: the child header and the
// StateRoot; the actors HAMT at width 5, whose level k reads hash bits [5k, 5k + 5) and so has at most ⌊256/5⌋ = 51 levels; the EVM
// state; the contract-state block (A1–B2; for C it is the HAMT root itself); a storage HAMT at width 1, at most 256 levels. Wider
// storage HAMTs are shallower (⌊256/bw⌋ ≤ 256). 2 + 51 + 1 + 1 + 256 = 311, rounded up to a multiple of 32 words.
#define REC_FIXED_BLOCKS 4          // header, StateRoot, EVM state, contract-state block
#define REC_CAP 320
static_assert(REC_CAP >= REC_FIXED_BLOCKS + 256 / 5 + 256 / 1, "a storage proof's recorder must hold the longest accepted path");

// RecordingBlockStore of one proof: per-thread list (for the per-spec Vec<ProofBlock>) + union bitmap
struct Recorder {
    uint32_t* list;   // REC_CAP entries, may be nullptr
    uint32_t n;
    uint32_t* wbits;
    bool overflow;
    uint32_t hamt_nodes = 0, hamt_bytes = 0;   // HAMT nodes decoded through this recorder and their bytes (measurement: K5's algorithmic bytes)
    bool strict_only = false;                  // A/B switch (IPCFP_HAMT_STRICT=1): skip the fast node decoder
    const uint32_t* rank_of = nullptr;         // StoreView::rank_of (witness bitmaps are indexed by Cid rank); nullptr = identity
    const uint8_t* missing = nullptr;          // the CID of the last get that found no block (the fetch planner reads it; plan.cu)
    __device__ void note(uint32_t blk) {
        if (wbits) witness_mark_rank(wbits, rank_of ? rank_of[blk] : blk);   // (the verifiers walk without recording)
        if (!list) return;
        for (uint32_t i = 0; i < n; i++) if (list[i] == blk) return;
        if (n < REC_CAP) list[n++] = blk; else overflow = true;   // guard only: no accepted input records more than REC_CAP blocks
    }
};
struct Fail { uint32_t code; uint32_t detail; };
#define SFAIL(c, d) do { f.code = (c); f.detail = (d); return false; } while (0)

// Blockstore::get through a recorder: block index or -1 (recorded either way the reference records
// the CID before forwarding; a missing block never reaches the witness because the call fails)
__device__ __forceinline__ int32_t rec_get(const StoreView& s, Recorder& rec, const uint8_t* cid38) {
    int32_t b = store_lookup(s, cid38);
    if (b >= 0) rec.note((uint32_t)b); else rec.missing = cid38;
    return b;
}

struct ValueRef { uint32_t blk; uint32_t off; };

// Hamt::get. key: keylen bytes. Returns true on success; found/val describe the outcome.
static __device__ bool hamt_get(const StoreView& s, Recorder& rec, const uint8_t* root_cid, uint64_t bw64, int vkind, const uint8_t* key,
                         uint32_t keylen, bool& found, ValueRef& val, Fail& f) {
    found = false;
    if (bw64 < 1 || bw64 > 8) SFAIL(DC_DECODE, CE_HAMT);
    uint32_t bw = (uint32_t)bw64;
    int32_t blk = rec_get(s, rec, root_cid);
    if (blk < 0) SFAIL(DC_MISSING, 0);
    uint32_t h[8];
    sha256(key, keylen, h);
    uint32_t consumed = 0;
    for (;;) {
        uint32_t len;
        const uint8_t* p = store_block(s, (uint32_t)blk, len);
        rec.hamt_nodes++; rec.hamt_bytes += len;
        Rd r(p, len);
        bool depth_ok = consumed + bw <= 256;
        uint32_t idx = depth_ok ? hash_bits(h, consumed, bw) : 0;
        HamtHit hit;
        if (rec.strict_only || !hamt_node_lookup_fast(p, len, vkind, idx, key, keylen, hit)) hamt_node_lookup(r, vkind, idx, key, keylen, hit);   // strict decoder: exact errors
        if (r.err) SFAIL(DC_DECODE, r.err);
        if (!depth_ok) SFAIL(DC_DECODE, CE_HAMT);  // HashBits::next → MaxDepth
        consumed += bw;
        if (hit.kind == 0) return true;
        if (hit.kind == 1) { found = true; val.blk = (uint32_t)blk; val.off = hit.val_off; return true; }
        blk = rec_get(s, rec, p + hit.link_off);
        if (blk < 0) SFAIL(DC_MISSING, 0);
    }
}

// struct SmallMap { v: Vec<(ByteBuf, ByteBuf)> } from a CBOR map; remembers the first pair whose key == slot
static __device__ void dec_small_map(Rd& r, const uint8_t* slot, bool search, bool& hit, uint32_t& voff, uint32_t& vlen) {
    uint32_t n = rd_map(r);
    bool have = false;
    for (uint32_t i = 0; i < n && !r.err; i++) {
        uint32_t kl;
        uint32_t ko = rd_text(r, kl);
        if (r.err) break;
        if (kl == 1 && r.p[ko] == 'v') {
            if (have) { rd_fail(r, CE_FIELD); break; }
            have = true;
            uint32_t np = rd_array(r);
            for (uint32_t j = 0; j < np && !r.err; j++) {
                rd_array_exact(r, 2);
                uint32_t al, bl;
                uint32_t ao = rd_bytes(r, al);
                uint32_t bo = rd_bytes(r, bl);
                if (r.err) break;
                if (search && !hit && al == 32) {
                    bool eq = true;
                    for (int b = 0; b < 32; b++) eq &= r.p[ao + b] == slot[b];
                    if (eq) { hit = true; voff = bo; vlen = bl; }
                }
            }
        } else rd_skip_any(r);
    }
    if (!r.err && !have) rd_fail(r, CE_FIELD);
}

struct SlotValue { bool found; uint32_t raw_len; uint8_t v32[32]; };
__device__ __forceinline__ void value_from_bytes(const uint8_t* p, uint32_t len, SlotValue& out) {  // left_pad_32 (evm.rs:91-100)
    out.found = true; out.raw_len = len;
    for (int i = 0; i < 32; i++) out.v32[i] = 0;
    uint32_t take = len < 32 ? len : 32;
    for (uint32_t i = 0; i < take; i++) out.v32[32 - take + i] = p[len - take + i];
}
static __device__ void value_from_u8vec(const uint8_t* p, uint32_t blen, uint32_t off, SlotValue& out) {
    Rd r(p, blen);
    r.pos = off;
    uint32_t n = rd_array(r);
    out.found = true; out.raw_len = n;
    for (int i = 0; i < 32; i++) out.v32[i] = 0;
    uint32_t skip = n > 32 ? n - 32 : 0, take = n - skip;
    for (uint32_t i = 0; i < n; i++) {
        uint64_t x = rd_uint(r);
        if (i >= skip) out.v32[32 - take + (i - skip)] = (uint8_t)x;
    }
}

// read_storage_slot (storage/decode.rs:36-97)
static __device__ bool read_storage_slot(const StoreView& s, Recorder& rec, const uint8_t* root_cid, const uint8_t* slot, SlotValue& out, Fail& f) {
    out.found = false; out.raw_len = 0;
    for (int i = 0; i < 32; i++) out.v32[i] = 0;
    int32_t blk = rec_get(s, rec, root_cid);
    if (blk < 0) SFAIL(DC_MISSING, 0);
    uint32_t len;
    const uint8_t* p = store_block(s, (uint32_t)blk, len);
    {   // A1: [params, [SmallMap…]] — only the first map is searched; an empty list falls through
        Rd r(p, len);
        rd_array_exact(r, 2);
        uint32_t l;
        (void)rd_bytes(r, l);
        uint32_t n = rd_array(r);
        bool hit = false;
        uint32_t vo = 0, vl = 0;
        for (uint32_t i = 0; i < n && !r.err; i++) dec_small_map(r, slot, i == 0, hit, vo, vl);
        rd_end(r);
        if (!r.err && n > 0) { if (hit) value_from_bytes(p + vo, vl, out); return true; }
    }
    {   // A2: [params, SmallMap]
        Rd r(p, len);
        rd_array_exact(r, 2);
        uint32_t l;
        (void)rd_bytes(r, l);
        bool hit = false;
        uint32_t vo = 0, vl = 0;
        dec_small_map(r, slot, true, hit, vo, vl);
        rd_end(r);
        if (!r.err) { if (hit) value_from_bytes(p + vo, vl, out); return true; }
    }
    {   // A3: SmallMap
        Rd r(p, len);
        bool hit = false;
        uint32_t vo = 0, vl = 0;
        dec_small_map(r, slot, true, hit, vo, vl);
        rd_end(r);
        if (!r.err) { if (hit) value_from_bytes(p + vo, vl, out); return true; }
    }
    const uint8_t* hroot = root_cid;
    uint64_t bw = 5;  // C: direct HAMT, HAMT_BIT_WIDTH
    {   // B1: (root, bitwidth)
        Rd r(p, len);
        rd_array_exact(r, 2);
        uint32_t co = rd_cid(r);
        uint64_t b = rd_uint(r);
        rd_end(r);
        if (!r.err) { hroot = p + co; bw = (uint32_t)b; goto do_hamt; }   // `bw as u32` (storage/decode.rs:79): truncation, not saturation
    }
    {   // B2: { root, bitwidth, … }
        Rd r(p, len);
        uint32_t n = rd_map(r);
        bool hr = false, hb = false;
        uint32_t co = 0;
        uint64_t b = 0;
        for (uint32_t i = 0; i < n && !r.err; i++) {
            uint32_t kl;
            uint32_t ko = rd_text(r, kl);
            if (r.err) break;
            if (kl == 4 && bytes_eq(r.p + ko, "root", 4)) { if (hr) rd_fail(r, CE_FIELD); else { hr = true; co = rd_cid(r); } }
            else if (kl == 8 && bytes_eq(r.p + ko, "bitwidth", 8)) { if (hb) rd_fail(r, CE_FIELD); else { hb = true; b = rd_uint(r); } }
            else rd_skip_any(r);
        }
        if (!r.err && !(hr && hb)) rd_fail(r, CE_FIELD);
        rd_end(r);
        if (!r.err) { hroot = p + co; bw = (uint32_t)b; }                                // `bitwidth as u32` (storage/decode.rs:86)
    }
do_hamt:
    bool found;
    ValueRef vr;
    if (!hamt_get(s, rec, hroot, bw, HV_U8VEC, slot, 32, found, vr, f)) return false;
    if (found) {
        uint32_t bl;
        const uint8_t* bp = store_block(s, vr.blk, bl);
        value_from_u8vec(bp, bl, vr.off, out);
    }
    return true;
}

// HeaderLite (common/decode.rs:100-124): the fields the generators and verifiers read
struct HeaderFields { uint32_t parents_off, n_parents, psr_off, receipts_off, messages_off; int64_t height; };
__device__ __forceinline__ void header_fields(Rd& r, HeaderFields& h) {
    rd_array_exact(r, 16);
    for (int i = 0; i < 5; i++) rd_skip_any(r);
    h.n_parents = rd_array(r);
    h.parents_off = r.pos;
    for (uint32_t i = 0; i < h.n_parents && !r.err; i++) (void)rd_cid(r);
    rd_skip_any(r);
    h.height = rd_int(r);
    h.psr_off = rd_cid(r);
    h.receipts_off = rd_cid(r);
    h.messages_off = rd_cid(r);
    rd_skip_any(r);
    (void)rd_uint(r);
    rd_skip_any(r);
    (void)rd_uint(r);
    rd_skip_any(r);
    rd_end(r);
}
// EvmStateV6 / V5 (common/decode.rs:48-97): offset of contract_state CID bytes
static __device__ bool try_evm_state(const uint8_t* p, uint32_t len, int fields, uint32_t& cs_off) {
    Rd r(p, len);
    rd_array_exact(r, (uint32_t)fields);
    (void)rd_cid(r);
    uint32_t bl;
    (void)rd_bytes(r, bl);
    if (!r.err && bl != 32) rd_fail(r, CE_LEN);
    cs_off = rd_cid(r);
    if (fields == 6) { if (rd_peek_null(r)) r.pos++; else rd_skip_any(r); }
    (void)rd_uint(r);
    if (rd_peek_null(r)) r.pos++; else rd_skip_any(r);
    rd_end(r);
    return !r.err;
}

// Address::new_id(id).to_bytes(), the actors-HAMT key: protocol 0, then the ID as a varint; returns its length
__device__ __forceinline__ uint32_t id_address_key(uint64_t id, uint8_t key[11]) {
    uint32_t kl = 0;
    key[kl++] = 0;
    while (id >= 0x80) { key[kl++] = (uint8_t)(id | 0x80); id >>= 7; }
    key[kl++] = (uint8_t)id;
    return kl;
}
// get_actor_state (common/decode.rs:17-42): StateRoot [version ≤ 5, actors, info] → actors HAMT (width 5) → the ActorState under key;
// state_cid points at its state CID. DC_ACTOR_NOT_FOUND when the actor is absent.
__device__ __forceinline__ bool actor_state(const StoreView& s, Recorder& rec, const uint8_t* state_root, const uint8_t* key, uint32_t keylen,
                                            const uint8_t*& state_cid, Fail& f) {
    const int32_t sb = rec_get(s, rec, state_root);
    if (sb < 0) SFAIL(DC_MISSING, 2);
    uint32_t sl;
    const uint8_t* sp = store_block(s, (uint32_t)sb, sl);
    Rd sr(sp, sl);
    rd_array_exact(sr, 3);
    const uint64_t ver = rd_uint(sr);
    if (!sr.err && ver > 5) rd_fail(sr, CE_RANGE);
    const uint32_t actors_off = rd_cid(sr);
    (void)rd_cid(sr);
    rd_end(sr);
    if (sr.err) SFAIL(DC_DECODE, sr.err);
    bool found;
    ValueRef vr;
    if (!hamt_get(s, rec, sp + actors_off, 5, HV_ACTOR_STATE, key, keylen, found, vr, f)) return false;
    if (!found) SFAIL(DC_ACTOR_NOT_FOUND, 0);
    uint32_t abl;
    const uint8_t* abp = store_block(s, vr.blk, abl);
    Rd ar(abp, abl);
    ar.pos = vr.off;
    uint32_t state_off;
    parse_actor_state(ar, state_off);
    state_cid = abp + state_off;
    return true;
}
// parse_evm_state (common/decode.rs:48-97): the EVM state at state_cid, EvmStateV6 else V5; root points at its contract-state CID
__device__ __forceinline__ bool contract_storage_root(const StoreView& s, Recorder& rec, const uint8_t* state_cid, const uint8_t*& root, Fail& f) {
    const int32_t eb = rec_get(s, rec, state_cid);
    if (eb < 0) SFAIL(DC_MISSING, 3);
    uint32_t el;
    const uint8_t* ep = store_block(s, (uint32_t)eb, el);
    uint32_t cs_off;
    if (!try_evm_state(ep, el, 6, cs_off) && !try_evm_state(ep, el, 5, cs_off)) SFAIL(DC_DECODE, CE_FIELD);
    root = ep + cs_off;
    return true;
}

struct StorageArgs {
    StoreView store;
    const uint8_t* child_cid;
    const uint8_t* state_root_json;
    const ipcfp_storage_spec* specs;
    uint64_t n;
    ipcfp_storage_proof* out;
    uint32_t* rec_list;   // n * REC_CAP
    uint32_t* rec_n;      // n
    uint32_t* wbits;
    unsigned long long* err;
};

static __device__ bool storage_proof_one(const StorageArgs& a, uint64_t t, Recorder& rec, ipcfp_storage_proof& q, Fail& f) {
    const StoreView& s = a.store;
    // extract_and_verify_parent_state (storage/generator.rs:72-103); the header recorder is dropped (:80-83)
    int32_t hb = store_lookup(s, a.child_cid);
    if (hb < 0) SFAIL(DC_MISSING, 1);
    uint32_t hl;
    const uint8_t* hp = store_block(s, (uint32_t)hb, hl);
    Rd hr(hp, hl);
    HeaderFields hf;
    header_fields(hr, hf);
    if (hr.err) SFAIL(DC_DECODE, hr.err);
    const uint8_t* psr = hp + hf.psr_off;
    if (!cid38_equal(psr, a.state_root_json)) SFAIL(DC_STATE_MISMATCH, 0);
    rec.note((uint32_t)hb);  // collector.add_cid(child_cid) (:41)
    // load_actor_and_storage_root (:106-134): add_cid(parent_state_root) + state_recorder.get, get_actor_state, parse_evm_state
    uint8_t key[11];
    const uint32_t kl = id_address_key(a.specs[t].actor_id, key);
    const uint8_t *state_cid, *storage_root;
    if (!actor_state(s, rec, psr, key, kl, state_cid, f) || !contract_storage_root(s, rec, state_cid, storage_root, f)) return false;
    // read_storage_value (:137-155)
    SlotValue sv;
    if (!read_storage_slot(s, rec, storage_root, a.specs[t].slot, sv, f)) return false;
    q.actor_id = a.specs[t].actor_id;
    for (int i = 0; i < 38; i++) { q.actor_state_cid[i] = state_cid[i]; q.storage_root[i] = storage_root[i]; }
    for (int i = 0; i < 32; i++) { q.slot[i] = a.specs[t].slot[i]; q.value[i] = sv.v32[i]; }
    q.found = sv.found; q._pad[0] = q._pad[1] = q._pad[2] = 0;
    q.raw_len = sv.raw_len;
    return true;
}

}  // namespace ipcfp
