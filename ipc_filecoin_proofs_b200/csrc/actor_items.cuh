// actor_items.cuh — per-proof device functions of actor proofs (actor.cu holds the kernels and the host flow; plan_items.cuh and
// verify_items.cuh use them too). They live in a header, as storage.cuh does, so that the same code can be compiled for the host.
//   child header → ParentStateRoot → [Init actor → InitState → address_map (non-ID addresses)] → actors HAMT → ActorState → EVM state
//   fvm_shared ActorState [UPSTREAM]                 [code, head, sequence, balance: TokenAmount, delegated_address: Option<Address>]
//   fvm_shared bigint_ser [UPSTREAM]                 empty bytes = 0; else a sign byte (0 plus, 1 minus), then the big-endian magnitude
//   builtin-actors evm State [UPSTREAM]              EvmStateV6 / V5, read as contract_storage_root reads them
#pragma once
#include "resolve_items.cuh"

namespace ipcfp {

// Distinct blocks one actor proof can record, on the longest accepted path: the child header; the StateRoot; the actors HAMT at width 5
// to the Init actor (⌊256/5⌋ = 51 levels); the InitState; the address_map at width 5 (51 levels); the actors HAMT again to the actor (51
// levels); the EVM state; the bytecode block. The Init path is recorded once per call in a list of its own, so a proof's own list holds
// at most 1 + 51 + 1 + 51 + 1 + 1 blocks; the two lists together hold at most 158.
#define ACTOR_FIXED_BLOCKS 5   // header, StateRoot, InitState, EVM state, bytecode block
static_assert(REC_CAP >= ACTOR_FIXED_BLOCKS + 3 * (256 / 5), "an actor proof's recorder lists must hold the deepest two-HAMT path");

// ActorState with every field located: parse_actor_state's checks, in the same order
struct ActorFields {
    uint32_t code_off, head_off, balance_off, balance_len, delegated_off, delegated_len;
    uint64_t sequence;
    bool has_delegated;
};
__device__ __forceinline__ void parse_actor_state_full(Rd& r, ActorFields& af) {
    rd_array_exact(r, 5);
    af.code_off = rd_cid(r);
    af.head_off = rd_cid(r);
    af.sequence = rd_uint(r);
    af.balance_off = rd_bytes(r, af.balance_len);
    af.has_delegated = !rd_peek_null(r);
    af.delegated_off = 0; af.delegated_len = 0;
    if (af.has_delegated) af.delegated_off = rd_bytes(r, af.delegated_len); else r.pos++;
}

// TokenAmount (bigint_ser) → 32-byte big-endian magnitude and sign. A zero magnitude is never negative (BigInt has no negative zero).
// false: a sign byte other than 0 / 1, or a magnitude over 32 bytes.
__host__ __device__ inline bool decode_balance(const uint8_t* p, uint32_t len, uint8_t out[32], uint8_t& negative) {
    for (int i = 0; i < 32; i++) out[i] = 0;
    negative = 0;
    if (len == 0) return true;
    if (p[0] > 1 || len - 1 > 32) return false;
    const uint32_t m = len - 1;
    bool nonzero = false;
    for (uint32_t i = 0; i < m; i++) { out[32 - m + i] = p[1 + i]; nonzero |= p[1 + i] != 0; }
    negative = (uint8_t)(p[0] == 1 && nonzero);
    return true;
}

// EvmStateV6 / V5 with every field located: try_evm_state's checks, in the same order
struct EvmFields { uint32_t bytecode_off, hash_off, cs_off; uint64_t nonce; };
static __device__ bool evm_state_fields(const uint8_t* p, uint32_t len, int fields, EvmFields& e) {
    Rd r(p, len);
    rd_array_exact(r, (uint32_t)fields);
    e.bytecode_off = rd_cid(r);
    uint32_t bl;
    e.hash_off = rd_bytes(r, bl);
    if (!r.err && bl != 32) rd_fail(r, CE_LEN);
    e.cs_off = rd_cid(r);
    if (fields == 6) { if (rd_peek_null(r)) r.pos++; else rd_skip_any(r); }
    e.nonce = rd_uint(r);
    if (rd_peek_null(r)) r.pos++; else rd_skip_any(r);
    rd_end(r);
    return !r.err;
}

__device__ __forceinline__ bool evm_code(const uint8_t* codes, uint64_t n, const uint8_t* code) {
    for (uint64_t k = 0; k < n; k++) if (cid38_equal(codes + 38 * k, code)) return true;
    return false;
}

struct ActorArgs {
    StoreView store;
    const uint8_t* child_cid;
    const uint8_t* state_root_json;    // the tipset's child_parent_state_root
    const ipcfp_address* addrs;
    uint64_t n;
    const uint8_t* evm_codes;          // n_evm*38: the code CIDs whose actors are EVM actors
    uint64_t n_evm;
    uint32_t with_code;                // IPCFP_ACTOR_WITH_CODE
    uint32_t strict_only;
    const uint8_t** address_map;       // written by the Init walk: the address_map root, nullptr when that walk failed with *init_fail
    Fail* init_fail;
    ipcfp_actor_proof* out;
    uint64_t* code_blk;                // n: the bytecode block of a proof with code, else UINT64_MAX
    uint64_t* code_len;                // n: its length, else 0
    uint32_t* rec_list;                // n * REC_CAP
    uint32_t* rec_n;                   // n
    uint32_t* init_list;               // REC_CAP: the Init path's blocks
    uint32_t* init_n;
    uint32_t* wbits;
    unsigned long long* err;
};

// The child header: its ParentStateRoot must be the tipset's (storage_proof_one's check); psr points at it. The header is recorded.
// A missing header is named in rec.missing, as every other missing block is.
__device__ __forceinline__ bool actor_header(const ActorArgs& a, Recorder& rec, const uint8_t*& psr, Fail& f) {
    const int32_t hb = store_lookup(a.store, a.child_cid);
    if (hb < 0) { rec.missing = a.child_cid; SFAIL(DC_MISSING, 1); }
    uint32_t hl;
    const uint8_t* hp = store_block(a.store, (uint32_t)hb, hl);
    Rd hr(hp, hl);
    HeaderFields hf;
    header_fields(hr, hf);
    if (hr.err) SFAIL(DC_DECODE, hr.err);
    psr = hp + hf.psr_off;
    if (!cid38_equal(psr, a.state_root_json)) SFAIL(DC_STATE_MISMATCH, 0);
    rec.note((uint32_t)hb);
    return true;
}

// The ActorState under actor ID id in the state tree at state_root: StateRoot [version <= 5, actors, info] → actors HAMT (width 5).
// found = false: proven absent. ab / af locate the value.
static __device__ bool actor_lookup(const StoreView& s, Recorder& rec, const uint8_t* state_root, uint64_t id, bool& found, const uint8_t*& ab,
                                    ActorFields& af, Fail& f) {
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
    uint8_t key[11];
    ValueRef vr;
    if (!hamt_get(s, rec, sp + actors_off, 5, HV_ACTOR_STATE, key, id_address_key(id, key), found, vr, f)) return false;
    if (!found) return true;
    uint32_t abl;
    ab = store_block(s, vr.blk, abl);
    Rd ar(ab, abl);
    ar.pos = vr.off;
    parse_actor_state_full(ar, af);
    if (ar.err) SFAIL(DC_DECODE, ar.err);
    return true;
}

// The EVM fields of the state at head (EvmStateV6, else V5); with_code: the bytecode block, whose Keccak-256 must be bytecode_hash. head
// points into the store's block (rec.missing may name it after the caller's proof record is gone).
static __device__ bool actor_evm(const StoreView& s, Recorder& rec, const uint8_t* head, bool with_code, ipcfp_actor_proof& q, uint64_t& code_blk,
                                 Fail& f) {
    const int32_t eb = rec_get(s, rec, head);
    if (eb < 0) SFAIL(DC_MISSING, 3);
    uint32_t el;
    const uint8_t* ep = store_block(s, (uint32_t)eb, el);
    EvmFields e;
    if (!evm_state_fields(ep, el, 6, e) && !evm_state_fields(ep, el, 5, e)) SFAIL(DC_DECODE, CE_FIELD);
    q.is_evm = 1;
    q.evm_nonce = e.nonce;
    for (int i = 0; i < 38; i++) { q.bytecode_cid[i] = ep[e.bytecode_off + i]; q.contract_state[i] = ep[e.cs_off + i]; }
    for (int i = 0; i < 32; i++) q.bytecode_hash[i] = ep[e.hash_off + i];
    if (!with_code) return true;
    const int32_t cb = rec_get(s, rec, ep + e.bytecode_off);
    if (cb < 0) SFAIL(DC_MISSING, 4);
    uint32_t cl;
    const uint8_t* cp = store_block(s, (uint32_t)cb, cl);
    Digest d;
    keccak256(cp, cl, d);
    const uint8_t* db = reinterpret_cast<const uint8_t*>(d.w);
    for (int i = 0; i < 32; i++) if (db[i] != q.bytecode_hash[i]) SFAIL(DC_DECODE, CE_FIELD);
    code_blk = (uint64_t)cb;
    q.code_len = cl;
    return true;
}

// The proof of address ad into q (zeroed by the caller): the header, then (non-ID address) the address_map lookup under the Init path's
// root, then the actor and its fields. An absent address or actor is an answer (status), not a failure. address_map: nullptr when the
// Init path failed with init_fail.
static __device__ bool actor_proof_one(const ActorArgs& a, const ipcfp_address& ad, const uint8_t* address_map, const Fail& init_fail, Recorder& rec,
                                       ipcfp_actor_proof& q, uint64_t& code_blk, Fail& f) {
    const StoreView& s = a.store;
    code_blk = UINT64_MAX;
    const uint8_t* psr;
    if (!actor_header(a, rec, psr, f)) return false;
    q.address = ad;
    uint64_t id = 0;
    if (ad.bytes[0] == 0) (void)address_valid(ad, &id);   // bytes that are not an Address were refused on the host
    else {
        if (!address_map) { f = init_fail; return false; }
        if (!resolve_lookup(s, rec, address_map, ad.bytes, ad.len, id, f)) {
            if (f.code != DC_ACTOR_NOT_FOUND) return false;
            q.status = IPCFP_ACTOR_NO_ADDRESS;
            return true;
        }
    }
    q.actor_id = id;
    bool found;
    const uint8_t* ab = nullptr;
    ActorFields af;
    if (!actor_lookup(s, rec, psr, id, found, ab, af, f)) return false;
    if (!found) { q.status = IPCFP_ACTOR_NO_ACTOR; return true; }
    for (int i = 0; i < 38; i++) { q.code[i] = ab[af.code_off + i]; q.head[i] = ab[af.head_off + i]; }
    q.sequence = af.sequence;
    if (!decode_balance(ab + af.balance_off, af.balance_len, q.balance, q.balance_negative)) SFAIL(DC_DECODE, CE_RANGE);
    if (af.has_delegated) {
        if (!address_bytes_valid(ab + af.delegated_off, af.delegated_len, nullptr)) SFAIL(DC_DECODE, CE_FIELD);
        q.has_delegated = 1;
        q.delegated.len = (uint8_t)af.delegated_len;
        for (uint32_t i = 0; i < af.delegated_len; i++) q.delegated.bytes[i] = ab[af.delegated_off + i];
    }
    if (evm_code(a.evm_codes, a.n_evm, q.code) && !actor_evm(s, rec, ab + af.head_off, a.with_code != 0, q, code_blk, f)) return false;
    q.status = IPCFP_ACTOR_FOUND;
    return true;
}

}  // namespace ipcfp
