// verify_items.cuh — the per-item device code of the GPU-batched verifiers (verify.cu): what ONE thread does for the tipset, for one
// TxMeta block, for one event proof, for one storage proof. Kept apart from the kernels so that tests/host_fuzz/emu_verify.cu can
// compile the very same code for the host and run it, item by item, against the restated CPU verifiers of the test tree — on intact and on
// adversarial bundles, under AddressSanitizer. The kernels in verify.cu only compute the item index and call these.
#pragma once
#include "engine.cuh"
#include "events_items.cuh"
#include "hashes.cuh"
#include "actor_items.cuh"
#include "message_proof_items.cuh"
#include "storage.cuh"

namespace ipcfp {

#define ST_VERIFY 9u

struct VerifyTipsetArgs {
    StoreView store;
    const uint8_t* parent_cids;   // device, n_parents*38 (from the proof / the caller's tipset)
    const uint8_t* child_cid;     // device, 38
    uint32_t n_parents;
    int64_t parent_epoch, child_epoch;
    // outputs
    uint32_t* consistent;         // verify_header_consistency returned true
    uint32_t* receipts_root_blk;  // block of child_hdr.parent_message_receipts (0xffffffff: not in the witness — an error only if a proof gets that far)
    uint8_t* txmeta_cids;         // n_parents*38: hdr.messages of every parent header
    unsigned long long* err;
};
// once per call, one thread: verify_header_consistency (events/verifier.rs:147-181), the parent headers' `messages` links
// (reconstruct_execution_order, events/utils.rs:16-30) and the TxMeta recompute (utils.rs:64-73)
__device__ __forceinline__ void verify_tipset_item(const VerifyTipsetArgs& a) {
    const StoreView& s = a.store;
    *a.consistent = 0;
    *a.receipts_root_blk = 0xffffffffu;
    int32_t cb = store_lookup(s, a.child_cid);
    if (cb < 0) { report_error(a.err, ST_VERIFY, 0, DC_MISSING, 1); return; }
    uint32_t cl;
    const uint8_t* cp = store_block(s, (uint32_t)cb, cl);
    Rd cr(cp, cl);
    HeaderFields ch;
    header_fields(cr, ch);
    if (cr.err) { report_error(a.err, ST_VERIFY, 0, DC_DECODE, cr.err); return; }
    bool same = ch.n_parents == a.n_parents;
    for (uint32_t k = 0; same && k < a.n_parents; k++) same = cid38_equal(cp + ch.parents_off + 43 * k + 5, a.parent_cids + 38 * k);
    if (!same || ch.height != a.child_epoch) return;                           // Ok(false) for every proof
    if (a.n_parents == 0) { report_error(a.err, ST_VERIFY, 0, DC_DECODE, CE_RANGE); return; }   // parent_cids[0] panics in the reference
    int32_t pb0 = store_lookup(s, a.parent_cids);
    if (pb0 < 0) { report_error(a.err, ST_VERIFY, 0, DC_MISSING, 2); return; }
    {
        uint32_t pl;
        const uint8_t* pp = store_block(s, (uint32_t)pb0, pl);
        Rd pr(pp, pl);
        HeaderFields ph;
        header_fields(pr, ph);
        if (pr.err) { report_error(a.err, ST_VERIFY, 0, DC_DECODE, pr.err); return; }
        if (ph.height != a.parent_epoch) return;
    }
    *a.consistent = 1;
    // reconstruct_execution_order: every parent header's `messages`; collect_exec_list(verify_txmeta = true)
    for (uint32_t k = 0; k < a.n_parents; k++) {
        int32_t pb = store_lookup(s, a.parent_cids + 38 * k);
        if (pb < 0) { report_error(a.err, ST_VERIFY, 0, DC_MISSING, 3); return; }
        uint32_t pl;
        const uint8_t* pp = store_block(s, (uint32_t)pb, pl);
        Rd pr(pp, pl);
        HeaderFields ph;
        header_fields(pr, ph);
        if (pr.err) { report_error(a.err, ST_VERIFY, 0, DC_DECODE, pr.err); return; }
        for (int q = 0; q < 38; q++) a.txmeta_cids[38 * k + q] = pp[ph.messages_off + q];
    }
    int32_t rb = store_lookup(s, cp + ch.receipts_off);
    if (rb >= 0) *a.receipts_root_blk = (uint32_t)rb;
}
// put_cbor(&(bls_root, secp_root), Blake2b256) == tx_cid (utils.rs:64-73): the strict decoder accepts only the canonical encoding, so
// re-encoding the decoded pair gives the block's own bytes — the recomputed CID is `dag-cbor | blake2b-256 | Blake2b(block)`
__device__ __forceinline__ void verify_txmeta_item(const StoreView& s, const uint8_t* txmeta_cids, uint32_t k, unsigned long long* err) {
    const uint8_t* cid = txmeta_cids + 38 * k;
    int32_t b = store_lookup(s, cid);
    if (b < 0) return;                                                          // reported as missing TxMeta by the walk
    uint32_t len;
    const uint8_t* p = store_block(s, (uint32_t)b, len);
    Rd r(p, len);
    rd_array_exact(r, 2);
    (void)rd_cid(r); (void)rd_cid(r);
    rd_end(r);
    if (r.err) return;                                                          // reported as a decode error by the walk
    static const uint8_t want[6] = {0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
    bool ok = true;
    for (int q = 0; q < 6; q++) ok &= cid[q] == want[q];
    Digest d;
    blake2b256(p, len, d);
    Digest c = load_digest(cid + 6);
    if (!ok || !digest_eq(d, c)) report_error(err, ST_VERIFY, 0, DC_CID_MISMATCH, (uint32_t)k);
}

// check_event: matches_log of a spec (events/generator.rs:38-40), without its actor filter; nullptr: no predicate
__device__ __forceinline__ bool verify_check(const Matcher* f, const uint8_t* eblk, const EvLog& ev) {
    if (f) {
        if (ev.ntopics < 2) return false;
        const uint32_t o0 = ev.toff[0], o1 = ev.case_a ? ev.toff[0] + 32 : ev.toff[1];
        if (!(eq32(eblk + o0, f->t0) && eq32(eblk + o1, f->t1))) return false;
    }
    return true;
}
// check_event: a set of log filters, emitter sets included; one filter is the set of one
__device__ __forceinline__ bool verify_check(const LogFilterAny* f, const uint8_t* eblk, const EvLog& ev) { return event_matches(eblk, ev, *f); }

template <class F> struct VerifyEventArgsT {
    StoreView store;
    const ipcfp_event_proof* proofs;
    uint64_t n;
    const uint8_t* blob;
    uint64_t blob_size;
    const uint32_t* consistent;
    const uint32_t* receipts_root_blk;
    const RawCid* exec_raw;
    const uint32_t* exec_idx;
    uint64_t n_exec;
    const F* filter;              // nullptr: no predicate (Matcher only)
    uint8_t* results;
    unsigned long long* err;
};
using VerifyEventArgs = VerifyEventArgsT<Matcher>;
template <class F>
__device__ __forceinline__ void verify_event_item(const VerifyEventArgsT<F>& a, uint64_t t) {
    const StoreView& s = a.store;
    const ipcfp_event_proof& p = a.proofs[t];
    a.results[t] = 0;
    if (!*a.consistent) return;
    // verify_execution_order (:184-204)
    if (p.exec_index >= a.n_exec) return;
    {
        const RawCid c = a.exec_raw[a.exec_idx[p.exec_index]];
        bool eq = true;
        for (int q = 0; q < 6; q++) eq &= p.message_cid[q] == (uint8_t)(c.w[4] >> (8 * q));
        for (int q = 0; q < 32; q++) eq &= p.message_cid[6 + q] == (uint8_t)(c.w[q >> 3] >> (8 * (q & 7)));
        if (!eq) return;
    }
    // verify_receipt_and_event (:207-254)
    if (*a.receipts_root_blk == 0xffffffffu) { report_error(a.err, ST_VERIFY, t, DC_MISSING, 4); return; }
    uint32_t detail = 0, ev_off = 0;
    const uint8_t* rblk = nullptr;
    int got = amt_get(s, *a.receipts_root_blk, 0, p.exec_index, [&](Rd& r, bool keep) { const uint32_t o = parse_receipt(r); if (keep) ev_off = o; },
                      &rblk, &detail);
    if (got < 0) { report_error(a.err, ST_VERIFY, t, (uint32_t)(-got), detail); return; }
    if (got == 0 || ev_off == 0xffffffffu) return;
    int32_t eb = store_lookup(s, rblk + ev_off);
    if (eb < 0) { report_error(a.err, ST_VERIFY, t, DC_MISSING, 5); return; }
    EvLog ev;
    const uint8_t* eblk = nullptr;
    got = amt_get(s, (uint32_t)eb, 3, p.event_index, [&](Rd& r, bool keep) { EvLog e; decode_stamped_event(r, e); if (keep && !r.err) ev = e; },
                  &eblk, &detail);
    if (got < 0) { report_error(a.err, ST_VERIFY, t, (uint32_t)(-got), detail); return; }
    if (got == 0) return;
    // verify_event_data_matches (:257-290)
    if (ev.emitter != p.emitter || !ev.some || ev.ntopics != p.n_topics) return;
    if (p.topics_off > a.blob_size || 32ull * p.n_topics > a.blob_size - p.topics_off || p.data_off > a.blob_size || p.data_len > a.blob_size - p.data_off) return;
    for (uint32_t k = 0; k < ev.ntopics; k++) {
        const uint8_t* x = eblk + topic_offset(ev, k);
        const uint8_t* y = a.blob + p.topics_off + 32 * k;
        for (int q = 0; q < 32; q++) if (x[q] != y[q]) return;
    }
    if (ev.data_len != p.data_len) return;
    for (uint32_t q = 0; q < ev.data_len; q++) if (eblk[ev.data_off + q] != a.blob[p.data_off + q]) return;
    if (!verify_check(a.filter, eblk, ev)) return;   // the optional semantic check (check_event)
    a.results[t] = 1;
}

struct VerifyStorageArgs {
    StoreView store;
    const uint8_t* child_cid;
    const uint8_t* state_root_json;   // StorageProof.parent_state_root (the caller's tipset)
    const ipcfp_storage_proof* proofs;
    uint64_t n;
    uint8_t* results;
    unsigned long long* err;
};
__device__ __forceinline__ void verify_storage_item(const VerifyStorageArgs& a, uint64_t t) {
    const StoreView& s = a.store;
    const ipcfp_storage_proof& p = a.proofs[t];
    a.results[t] = 0;
    Recorder rec{nullptr, 0, nullptr, false};   // the verifier records nothing
    // verify_parent_state_root (:98-114)
    int32_t hb = store_lookup(s, a.child_cid);
    if (hb < 0) { report_error(a.err, ST_VERIFY, t, DC_MISSING, 1); return; }
    uint32_t hl;
    const uint8_t* hp = store_block(s, (uint32_t)hb, hl);
    Rd hr(hp, hl);
    HeaderFields hf;
    header_fields(hr, hf);
    if (hr.err) { report_error(a.err, ST_VERIFY, t, DC_DECODE, hr.err); return; }
    const uint8_t* psr = hp + hf.psr_off;
    if (!cid38_equal(psr, a.state_root_json)) return;
    // verify_actor_state (:117-132): get_actor_state (common/decode.rs:17-42)
    Fail f{0, 0};
    uint8_t key[11];
    const uint8_t* state_cid;
    if (!actor_state(s, rec, psr, key, id_address_key(p.actor_id, key), state_cid, f)) { report_error(a.err, ST_VERIFY, t, f.code, f.detail); return; }
    if (!cid38_equal(state_cid, p.actor_state_cid)) return;
    // verify_storage_root (:135-150)
    const uint8_t* storage_root;
    if (!contract_storage_root(s, rec, state_cid, storage_root, f)) { report_error(a.err, ST_VERIFY, t, f.code, f.detail); return; }
    if (!cid38_equal(storage_root, p.storage_root)) return;
    // verify_storage_value (:153-170)
    SlotValue sv;
    if (!read_storage_slot(s, rec, storage_root, p.slot, sv, f)) { report_error(a.err, ST_VERIFY, t, f.code, f.detail); return; }
    for (int q = 0; q < 32; q++) if (sv.v32[q] != p.value[q]) return;
    a.results[t] = 1;
}

struct VerifyActorArgs {
    ActorArgs g;                        // the generator's inputs: the tipset's CIDs, the EVM code CIDs, with_code
    const ipcfp_actor_proof* proofs;
    uint64_t n;
    uint8_t* results;
    unsigned long long* err;
};
__device__ __forceinline__ bool actor_claims_equal(const ipcfp_actor_proof& q, const ipcfp_actor_proof& p, bool with_code) {
    bool eq = q.status == p.status && q.actor_id == p.actor_id && q.sequence == p.sequence && q.evm_nonce == p.evm_nonce &&
              q.balance_negative == p.balance_negative && q.has_delegated == p.has_delegated && q.is_evm == p.is_evm &&
              q.delegated.len == p.delegated.len && (!with_code || q.code_len == p.code_len);
    for (int i = 0; i < 32; i++) eq &= q.balance[i] == p.balance[i] && q.bytecode_hash[i] == p.bytecode_hash[i];
    for (int i = 0; i < 38; i++)
        eq &= q.code[i] == p.code[i] && q.head[i] == p.head[i] && q.bytecode_cid[i] == p.bytecode_cid[i] && q.contract_state[i] == p.contract_state[i];
    for (uint32_t i = 0; eq && i < q.delegated.len; i++) eq &= q.delegated.bytes[i] == p.delegated.bytes[i];
    return eq;
}
// Proof t is replayed on the witness (the generator's walk for its address, the Init path included) and must state what the replay
// finds, absences included. A header naming another ParentStateRoot is a false verdict, as in verify_storage_item.
__device__ __forceinline__ void verify_actor_item(const VerifyActorArgs& a, uint64_t t) {
    const ipcfp_actor_proof& p = a.proofs[t];
    a.results[t] = 0;
    Recorder rec{nullptr, 0, nullptr, false};   // the verifier records nothing
    Fail f{0, 0}, init_fail{0, 0};
    const uint8_t* psr;
    if (!actor_header(a.g, rec, psr, f)) { if (f.code != DC_STATE_MISMATCH) report_error(a.err, ST_VERIFY, t, f.code, f.detail); return; }
    const uint8_t* map = nullptr;
    if (p.address.bytes[0] != 0 && !resolve_init(a.g.store, rec, psr, map, init_fail)) { report_error(a.err, ST_VERIFY, t, init_fail.code, init_fail.detail); return; }
    ipcfp_actor_proof q;
    memset(&q, 0, sizeof q);
    uint64_t cb;
    if (!actor_proof_one(a.g, p.address, map, init_fail, rec, q, cb, f)) { report_error(a.err, ST_VERIFY, t, f.code, f.detail); return; }
    a.results[t] = actor_claims_equal(q, p, a.g.with_code != 0);
}

struct VerifyMessageArgs {
    MsgProofArgs g;                     // the generator's inputs: the proofs' message CIDs, their positions in the rebuilt order, with_body
    const ipcfp_message_proof* proofs;
    const uint8_t* blob;                // the caller's data blob, blob_size bytes (+ 16 of padding)
    uint64_t blob_size;
    const uint32_t* consistent;
    uint8_t* results;
};
__device__ __forceinline__ bool blob_equal(const uint8_t* blob, uint64_t blob_size, uint64_t off, uint64_t len, const uint8_t* x) {
    if (off > blob_size || len > blob_size - off) return false;
    for (uint64_t i = 0; i < len; i++) if (blob[off + i] != x[i]) return false;
    return true;
}
// Proof t is replayed on the witness — its position in the rebuilt execution order, the receipt at that position, with the body the
// message block — and must state exactly what the replay finds: every field, the return data and params against the caller's blob.
__device__ __forceinline__ void verify_message_item(const VerifyMessageArgs& a, uint64_t t) {
    const ipcfp_message_proof& p = a.proofs[t];
    a.results[t] = 0;
    if (!*a.consistent) return;
    ipcfp_message_proof q;
    memset(&q, 0, sizeof q);
    const uint8_t *ret, *par;
    Fail f{0, 0};
    if (a.g.exec_indices[t] != UINT64_MAX && a.g.receipts_root_blk == 0xffffffffu) { report_error(a.g.err, ST_VERIFY, t, DC_MISSING, 4); return; }
    if (!message_proof_one(a.g, t, q, ret, par, f)) { report_error(a.g.err, ST_VERIFY, t, f.code, f.detail); return; }
    q.return_off = p.return_off;
    q.params_off = p.params_off;
    const uint8_t* x = reinterpret_cast<const uint8_t*>(&q);
    const uint8_t* y = reinterpret_cast<const uint8_t*>(&p);
    for (size_t i = 0; i < sizeof q; i++) if (x[i] != y[i]) return;   // the generator's records are zero where no field is
    if (ret && !blob_equal(a.blob, a.blob_size, p.return_off, p.return_len, ret)) return;
    if (par && !blob_equal(a.blob, a.blob_size, p.params_off, p.params_len, par)) return;
    a.results[t] = 1;
}

}  // namespace ipcfp
