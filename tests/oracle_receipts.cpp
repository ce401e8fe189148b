// oracle_receipts.cpp — the C++ oracle of ipcfp_generate_message_proofs (TEST INFRASTRUCTURE), the second restatement beside
// tests/message_receipts.py: oracle/oracle.cpp's own decoders, Amt<Cid> / Amt<Receipt>, collect_exec_list and WitnessCollector, with
// the message block decoded by its shape (include/ipcfp.h, "Message proofs") and tests/oracle_resolve.cpp's Address check. It includes
// oracle_resolve.cpp (which includes oracle.cpp), so it is built INSTEAD of either, as a shared library (tests/message_receipts.py).
//
//   oracle_message_proofs(store, desc, cids, n, flags, records)   the n records in request order (return_off / params_off into the data
//                                                                 blob); the blob and the witness CIDs (`Cid` order) stay in this
//                                                                 library until the next call: oracle_message_blob, oracle_message_witness
#include <map>

#include "oracle_resolve.cpp"

namespace orc {

static void decode_address(Dec& d, ipcfp_address& a) {
    const Bytes b = d.bytes();
    ipcfp_address x;
    memset(&x, 0, sizeof x);
    if (b.empty() || b.size() > IPCFP_ADDRESS_MAX) fail_decode("address length");
    x.len = (uint8_t)b.size();
    memcpy(x.bytes, b.data(), b.size());
    bool is_id;
    uint64_t id;
    if (!address_from_bytes(x, is_id, id)) fail_decode("not an Address");
    a = x;
}
// TokenAmount (fvm bigint_ser): empty = 0, else a sign byte (0 / 1) and at most 32 magnitude bytes; a zero magnitude is never negative
static void decode_token(Dec& d, uint8_t out[32], uint8_t& negative) {
    const Bytes b = d.bytes();
    memset(out, 0, 32);
    negative = 0;
    if (b.empty()) return;
    if (b[0] > 1 || b.size() - 1 > 32) fail_decode("TokenAmount");
    bool nonzero = false;
    for (size_t i = 1; i < b.size(); i++) { out[32 - (b.size() - 1) + (i - 1)] = b[i]; nonzero |= b[i] != 0; }
    negative = (uint8_t)(b[0] == 1 && nonzero);
}
// array(10): Message; array(2): SignedMessage [Message, Signature]; anything else a decode error
static Bytes decode_message(const Bytes& raw, ipcfp_message_proof& q) {
    Dec d(raw);
    const uint64_t k = d.array();
    if (k != 10 && k != 2) fail_decode("message shape");
    if (k == 2) d.array_exact(10);
    q.version = d.uint();
    decode_address(d, q.to);
    decode_address(d, q.from);
    q.sequence = d.uint();
    decode_token(d, q.value, q.value_negative);
    q.gas_limit = d.uint();
    decode_token(d, q.gas_fee_cap, q.gas_fee_cap_negative);
    decode_token(d, q.gas_premium, q.gas_premium_negative);
    q.method_num = d.uint();
    Bytes params = d.bytes();
    q.sig_type = 0;
    if (k == 2) {
        const Bytes sig = d.bytes();
        if (sig.empty() || sig[0] < 1 || sig[0] > 3) fail_decode("signature type");
        q.sig_type = sig[0];
    }
    d.end();
    return params;
}

struct MessageProofsOut {
    std::vector<ipcfp_message_proof> proofs;
    Bytes blob;
    std::vector<Cid> witness;
};

static MessageProofsOut generate_message_proofs(const Blockstore& net, const TipsetIn& ts, const std::vector<Cid>& msgs, bool with_body) {
    MessageProofsOut out;
    WitnessCollector collector(net);
    for (auto& c : ts.parent_cids) collector.add_cid(c);
    collector.add_cid(ts.child_cid);
    collector.add_cid(ts.receipts_root);
    for (auto& c : ts.txmeta) collector.add_cid(c);
    for (size_t b = 0; b < ts.txmeta.size(); b++) {
        RecordingBlockStore rec(net);
        Bytes raw;
        if (!rec.get(ts.txmeta[b], raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing TxMeta " + cid_hex(ts.txmeta[b]), b);
        auto roots = decode_txmeta(raw);
        for (const Cid* r : {&roots.first, &roots.second}) Amt<Cid>::load(*r, rec, 0).for_each([](uint64_t, const Cid&) {});
        collector.collect_from_recording(rec);
    }
    const std::vector<Cid> exec = collect_exec_list(net, ts.txmeta, false);
    std::map<std::array<uint8_t, 38>, uint64_t> pos;   // the first position of each CID
    for (uint64_t i = 0; i < exec.size(); i++) pos.emplace(exec[i].b, i);
    const auto r_amt = Amt<Receipt>::load(ts.receipts_root, net, 0);
    for (size_t j = 0; j < msgs.size(); j++) {
        ipcfp_message_proof q;
        memset(&q, 0, sizeof q);
        memcpy(q.message_cid, msgs[j].b.data(), 38);
        q.exec_index = UINT64_MAX;
        q.status = IPCFP_MESSAGE_NOT_EXECUTED;
        const auto it = pos.find(msgs[j].b);
        if (it != pos.end()) {
            q.exec_index = it->second;
            try {
                RecordingBlockStore rec(net);
                Amt<Receipt> a = r_amt;
                a.bs = &rec;
                const std::optional<Receipt> r = a.get(q.exec_index);
                collector.collect_from_recording(rec);
                q.status = r ? IPCFP_MESSAGE_EXECUTED : IPCFP_MESSAGE_NO_RECEIPT;
                if (r) {
                    q.exit_code = (uint32_t)r->exit_code;
                    q.gas_used = r->gas_used;
                    q.return_len = r->return_data.size();
                    q.return_off = q.return_len ? out.blob.size() : 0;
                    out.blob.insert(out.blob.end(), r->return_data.begin(), r->return_data.end());
                    if (r->events_root) { q.has_events_root = 1; memcpy(q.events_root, r->events_root->b.data(), 38); }
                }
                if (with_body) {
                    Bytes raw;
                    if (!net.get(msgs[j], raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing message " + cid_hex(msgs[j]));
                    const Bytes params = decode_message(raw, q);
                    q.has_body = 1;
                    q.params_len = params.size();
                    q.params_off = q.params_len ? out.blob.size() : 0;
                    out.blob.insert(out.blob.end(), params.begin(), params.end());
                    collector.add_cid(msgs[j]);
                }
            } catch (Err& e) { e.index = j; throw; }
        }
        out.proofs.push_back(q);
    }
    for (const ProofBlock& b : collector.materialize()) out.witness.push_back(b.cid);
    return out;
}

static MessageProofsOut g_last;

}  // namespace orc

extern "C" ipcfp_status oracle_message_proofs(const oracle_store* s, const ipcfp_tipset_desc* t, const uint8_t* message_cids, uint64_t n,
                                              uint32_t flags, ipcfp_message_proof* out) {
    return orc::guard([&] {
        orc::g_last = orc::MessageProofsOut();
        std::vector<orc::Cid> msgs;
        for (uint64_t j = 0; j < n; j++) msgs.push_back(orc::cid_from(message_cids + 38 * j));
        orc::g_last = orc::generate_message_proofs(s->bs, orc::tipset_in(t), msgs, (flags & IPCFP_MESSAGE_WITH_BODY) != 0);
        if (n) memcpy(out, orc::g_last.proofs.data(), n * sizeof(ipcfp_message_proof));
    });
}
extern "C" const uint8_t* oracle_message_blob(uint64_t* len) {
    *len = orc::g_last.blob.size();
    return orc::g_last.blob.data();
}
extern "C" const uint8_t* oracle_message_witness(uint64_t* n) {
    *n = orc::g_last.witness.size();
    return orc::g_last.witness.empty() ? nullptr : orc::g_last.witness[0].b.data();
}
