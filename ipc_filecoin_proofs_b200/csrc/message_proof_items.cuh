// message_proof_items.cuh — per-request device functions of message proofs (message_proof.cu holds the kernels and the host flow). They
// live in a header, as actor_items.cuh does, so that the same code can be compiled for the host.
//   request CID → its execution position (k_msg_select, msg_select_items.cuh) → Amtv0<Receipt>::get(position) under the receipts root
//   → with IPCFP_MESSAGE_WITH_BODY, the message block under the request CID
//   fvm_shared Receipt [UPSTREAM]          [exit_code, return_data, gas_used, events_root: Option<Cid>]
//   fvm_shared Message [UPSTREAM]          [version, to, from, sequence, value, gas_limit, gas_fee_cap, gas_premium, method_num, params]
//   Lotus SignedMessage [UPSTREAM]         [Message, Signature]; Signature::to_bytes() is its type byte followed by the signature
#pragma once
#include "actor_items.cuh"

namespace ipcfp {

// Receipt with every field located: parse_receipt's checks, in the same order
struct ReceiptFields { uint32_t exit_code, return_off, return_len, events_off; uint64_t gas_used; };
__device__ __forceinline__ void parse_receipt_fields(Rd& r, ReceiptFields& rf) {
    rd_array_exact(r, 4);
    const uint64_t ec = rd_uint(r);
    if (!r.err && ec > 0xffffffffull) rd_fail(r, CE_RANGE);
    rf.exit_code = (uint32_t)ec;
    rf.return_off = rd_bytes(r, rf.return_len);
    rf.gas_used = rd_uint(r);
    rf.events_off = rd_opt_cid(r);
}

// Amtv0<Receipt>::get(i) of the receipts AMT rooted at block root_blk (receipts_get's walk, every child marked in wbits), with the
// receipt found located in rf and its node in *leaf. 1 = Some, 0 = None, < 0 = -DevCode with *detail; missing as amt_get's.
__device__ __forceinline__ int receipt_get_fields(const StoreView& s, uint32_t root_blk, uint64_t i, ReceiptFields& rf, const uint8_t** leaf,
                                                  uint32_t* wbits, uint32_t* detail, const uint8_t** missing = nullptr) {
    return amt_get(s, root_blk, 0, i, [&](Rd& r, bool want) { if (want) parse_receipt_fields(r, rf); else (void)parse_receipt(r); }, leaf, detail,
                   wbits, missing);
}

// A TokenAmount field: bytes decoded by decode_balance
__device__ __forceinline__ void rd_token_amount(Rd& r, uint8_t out[32], uint8_t& negative) {
    uint32_t l;
    const uint32_t o = rd_bytes(r, l);
    if (!r.err && !decode_balance(r.p + o, l, out, negative)) rd_fail(r, CE_RANGE);
}
// An Address field: bytes Address::from_bytes accepts
__device__ __forceinline__ void rd_address(Rd& r, ipcfp_address& a) {
    uint32_t l;
    const uint32_t o = rd_bytes(r, l);
    if (r.err) return;
    if (!address_bytes_valid(r.p + o, l, nullptr)) { rd_fail(r, CE_FIELD); return; }
    a.len = (uint8_t)l;
    for (uint32_t k = 0; k < l; k++) a.bytes[k] = r.p[o + k];
}

// The message block p[0, len) decoded by its shape into q's body fields; params located at *params_off / *params_len. false: the block
// is neither a Message nor a SignedMessage (the CborErr in r.err).
__device__ __forceinline__ uint32_t parse_message_block(const uint8_t* p, uint32_t len, ipcfp_message_proof& q, uint32_t& params_off,
                                                        uint32_t& params_len) {
    Rd r(p, len);
    const uint32_t k = rd_array(r);
    const bool signed_msg = k == 2;
    if (!r.err && k != 10 && k != 2) rd_fail(r, CE_LEN);
    if (signed_msg) rd_array_exact(r, 10);
    q.version = rd_uint(r);
    rd_address(r, q.to);
    rd_address(r, q.from);
    q.sequence = rd_uint(r);
    rd_token_amount(r, q.value, q.value_negative);
    q.gas_limit = rd_uint(r);
    rd_token_amount(r, q.gas_fee_cap, q.gas_fee_cap_negative);
    rd_token_amount(r, q.gas_premium, q.gas_premium_negative);
    q.method_num = rd_uint(r);
    params_off = rd_bytes(r, params_len);
    q.sig_type = 0;
    if (signed_msg) {
        uint32_t sl;
        const uint32_t so = rd_bytes(r, sl);
        if (!r.err && (sl == 0 || p[so] < 1 || p[so] > 3)) rd_fail(r, CE_FIELD);
        if (!r.err) q.sig_type = p[so];
    }
    rd_end(r);
    return r.err;
}

struct MsgProofArgs {
    StoreView store;
    const uint8_t* cids;             // n*38: the requests
    const uint64_t* exec_indices;    // n: each request's execution position, UINT64_MAX when not executed
    uint64_t n;
    uint32_t receipts_root_blk;
    uint32_t with_body;              // IPCFP_MESSAGE_WITH_BODY
    ipcfp_message_proof* out;
    const uint8_t** src;             // 2n: where the return data and the params lie in the store's arena (return data: [0, n))
    uint64_t* len;                   // 2n: their lengths, in the same order
    uint32_t* wbits;
    unsigned long long* err;
};

// The proof of request t into q (zeroed by the caller). Not executed and no receipt are answers; a missing block or a decode error is a
// failure f. missing (may be null): the CID of the block the store lacks.
__device__ __forceinline__ bool message_proof_one(const MsgProofArgs& a, uint64_t t, ipcfp_message_proof& q, const uint8_t*& ret,
                                                  const uint8_t*& par, Fail& f, const uint8_t** missing = nullptr) {
    const uint8_t* cid = a.cids + 38 * t;
    for (int k = 0; k < 38; k++) q.message_cid[k] = cid[k];
    ret = nullptr; par = nullptr;
    const uint64_t e = a.exec_indices[t];
    q.exec_index = e;
    if (e == UINT64_MAX) { q.status = IPCFP_MESSAGE_NOT_EXECUTED; return true; }
    ReceiptFields rf;
    const uint8_t* leaf = nullptr;
    uint32_t detail = 0;
    const int got = receipt_get_fields(a.store, a.receipts_root_blk, e, rf, &leaf, a.wbits, &detail, missing);
    if (got < 0) SFAIL((uint32_t)(-got), detail);
    if (got == 0) q.status = IPCFP_MESSAGE_NO_RECEIPT;
    else {
        q.status = IPCFP_MESSAGE_EXECUTED;
        q.exit_code = rf.exit_code;
        q.gas_used = rf.gas_used;
        q.return_len = rf.return_len;
        ret = leaf + rf.return_off;
        if (rf.events_off != 0xffffffffu) {
            q.has_events_root = 1;
            for (int k = 0; k < 38; k++) q.events_root[k] = leaf[rf.events_off + k];
        }
    }
    if (!a.with_body) return true;
    const int32_t mb = store_lookup(a.store, cid);
    if (mb < 0) { if (missing) *missing = cid; SFAIL(DC_MISSING, 5); }
    if (a.wbits) witness_mark(a.store, a.wbits, (uint32_t)mb);
    uint32_t ml;
    const uint8_t* mp = store_block(a.store, (uint32_t)mb, ml);
    uint32_t po, pl;
    const uint32_t ce = parse_message_block(mp, ml, q, po, pl);
    if (ce) SFAIL(DC_DECODE, ce);
    q.has_body = 1;
    q.params_len = pl;
    par = mp + po;
    return true;
}

}  // namespace ipcfp
