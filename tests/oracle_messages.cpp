// oracle_messages.cpp — the C++ oracle of ipcfp_generate_message_log_proof (TEST INFRASTRUCTURE): tests/oracle_logs.cpp's generator (the
// reference's generate_event_proof with a log filter as its predicate, on oracle/oracle.cpp's own decoders, Amt<…>, collect_exec_list and
// WitnessCollector) with its receipt loop restricted to the receipts of the given messages, plus the execution-index report. It includes
// oracle_logs.cpp (which includes oracle.cpp), so it is built INSTEAD of either, never beside them (tests/oracle_messages.py builds it).
//
// Selection (include/ipcfp.h): receipt i is selected when i < n_exec, i < n_receipts and exec[i] is one of the message CIDs, compared as
// 38 raw bytes with std::map, no sorting of our own. A null filter is every log extract_evm_log accepts.
#include <map>

#include "oracle_logs.cpp"

namespace orc {

static EventGenOut generate_message_log_proof(const Blockstore& net, const TipsetIn& ts, const std::vector<Cid>& msgs, const LogPredicate& pred,
                                              uint32_t flags, std::vector<uint64_t>& exec_indices) {
    EventGenOut out;
    WitnessCollector collector(net);
    std::vector<std::unique_ptr<RecordingBlockStore>> tx_recs;
    if (!(flags & IPCFP_SCAN_SKIP_TX_AMTS)) {
        for (auto& c : ts.parent_cids) collector.add_cid(c);
        collector.add_cid(ts.child_cid);
        collector.add_cid(ts.receipts_root);
        for (auto& c : ts.txmeta) collector.add_cid(c);
        for (size_t b = 0; b < ts.txmeta.size(); b++) {
            auto rec = std::make_unique<RecordingBlockStore>(net);
            Bytes raw;
            if (!rec->get(ts.txmeta[b], raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing TxMeta " + cid_hex(ts.txmeta[b]), b);
            auto roots = decode_txmeta(raw);
            for (const Cid* r : {&roots.first, &roots.second}) Amt<Cid>::load(*r, *rec, 0).for_each([](uint64_t, const Cid&) {});
            tx_recs.push_back(std::move(rec));
        }
        for (auto& r : tx_recs) collector.collect_from_recording(*r);
    }
    std::vector<Cid> exec = collect_exec_list(net, ts.txmeta, false);
    out.n_exec = exec.size();
    // the selection
    std::map<std::array<uint8_t, 38>, uint64_t> pos;   // raw bytes: a request need not parse as a CID
    for (uint64_t i = 0; i < exec.size(); i++) pos.emplace(exec[i].b, i);
    std::set<uint64_t> selected;
    exec_indices.assign(msgs.size(), UINT64_MAX);
    for (size_t j = 0; j < msgs.size(); j++) {
        auto it = pos.find(msgs[j].b);
        if (it == pos.end()) continue;
        exec_indices[j] = it->second;
        if (it->second < ts.n_receipts) selected.insert(it->second);
    }
    RecordingBlockStore rec_receipts(net);
    auto r_amt = Amt<Receipt>::load(ts.receipts_root, rec_receipts, 0);
    // pass 1 over the selected receipts in ascending order
    for (uint64_t i : selected) {
        if (!ts.has_root[i]) continue;
        try {
            RecordingBlockStore temp(net);
            auto amt = Amt<StampedEvent>::load(cid_from(ts.events_roots + 38 * i), temp, 3);
            bool has = false;
            amt.for_each([&](uint64_t, const StampedEvent& se) { std::optional<EvmLog> log; if (pred(se, log)) has = true; });
            if (has) out.matching.push_back(i);
        } catch (Err& e) { e.index = i; throw; }
    }
    // pass 2 (every selected receipt is below n_exec: no "Missing message" here)
    std::vector<std::unique_ptr<RecordingBlockStore>> event_recs;
    for (uint64_t i : out.matching) {
        const Cid& msg_cid = exec[i];
        try {
            if (!r_amt.get(i)) continue;
            auto rec_events = std::make_unique<RecordingBlockStore>(net);
            auto e_amt = Amt<StampedEvent>::load(cid_from(ts.events_roots + 38 * i), *rec_events, 3);
            e_amt.for_each([&](uint64_t j, const StampedEvent& se) {
                std::optional<EvmLog> log;
                if (!pred(se, log)) return;
                EventProofRec p;
                p.exec_index = i; p.event_index = j; p.emitter = se.emitter;
                p.topics = log->topics; p.data = log->data; p.message_cid = msg_cid;
                out.proofs.push_back(std::move(p));
            });
            event_recs.push_back(std::move(rec_events));
        } catch (Err& e) { e.index = i; throw; }
    }
    for (auto& r : event_recs) collector.collect_from_recording(*r);
    collector.collect_from_recording(rec_receipts);
    out.blocks = collector.materialize();
    return out;
}

}  // namespace orc

extern "C" ipcfp_status oracle_generate_message_log_proof(const oracle_store* s, const ipcfp_tipset_desc* t, const uint8_t* message_cids, uint64_t n,
                                                          const ipcfp_log_filter* f, uint32_t flags, uint64_t* exec_indices, ipcfp_event_result** out) {
    return orc::guard([&] {
        orc::TipsetIn ts = orc::tipset_in(t);
        std::vector<orc::Cid> msgs;
        for (uint64_t j = 0; j < n; j++) msgs.push_back(orc::cid_from(message_cids + 38 * j));
        ipcfp_log_filter any;
        memset(&any, 0, sizeof any);
        std::vector<uint64_t> idx;
        orc::EventGenOut o = orc::generate_message_log_proof(s->bs, ts, msgs, orc::LogPredicate(f ? *f : any), flags, idx);
        if (n) memcpy(exec_indices, idx.data(), 8 * n);
        *out = orc::box_event(o);
    });
}
