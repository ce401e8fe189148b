// oracle_logs.cpp — the C++ oracle of ipcfp_generate_log_proof (TEST INFRASTRUCTURE): the reference's generate_event_proof
// (events/generator.rs:60-107) restated with a log filter in place of EventMatcher + the actor filter, on oracle/oracle.cpp's own code:
// its strict decoders, Amt<…>, extract_evm_log, collect_exec_list, WitnessCollector and result boxing. This translation unit includes
// oracle.cpp, so it is built INSTEAD of oracle.cpp, never beside it (tests/oracle_logs.py builds it as a shared library).
//
// The predicate is DESIGN.md §3 "Log filters", written here from the C struct alone (std::set membership, no sorting, no hashing):
// extract_evm_log returns Some, the emitter is in the set (or the set is empty), the log has at least n_positions topics, and topic k is
// in values[k] for every k < n_positions with n_values[k] > 0.
#include "../oracle/oracle.cpp"

namespace orc {

struct LogPredicate {
    std::set<uint64_t> emitters;
    uint32_t npos = 0;
    std::vector<std::set<std::array<uint8_t, 32>>> vals;   // per position; empty = any
    explicit LogPredicate(const ipcfp_log_filter& f) : npos(f.n_positions), vals(4) {
        for (uint64_t j = 0; j < f.n_emitters; j++) emitters.insert(f.emitters[j]);
        for (uint32_t k = 0; k < 4; k++)
            for (uint64_t j = 0; j < f.n_values[k]; j++) {
                std::array<uint8_t, 32> v;
                copy_bytes(v.data(), f.values[k] + 32 * j, 32);
                vals[k].insert(v);
            }
    }
    bool operator()(const StampedEvent& se, std::optional<EvmLog>& log) const {
        if (!emitters.empty() && !emitters.count(se.emitter)) return false;
        log = extract_evm_log(se.event);
        if (!log || log->topics.size() < npos) return false;
        for (uint32_t k = 0; k < npos; k++)
            if (!vals[k].empty() && !vals[k].count(log->topics[k])) return false;
        return true;
    }
};

static EventGenOut generate_log_proof(const Blockstore& net, const TipsetIn& ts, const LogPredicate& pred, uint32_t flags, uint32_t threads) {
    EventGenOut out;
    WitnessCollector collector(net);
    std::vector<std::unique_ptr<RecordingBlockStore>> tx_recs;
    if (!(flags & IPCFP_SCAN_SKIP_TX_AMTS)) {
        // collect_base_witness (events/generator.rs:122-145), record_transaction_amts (:148-177)
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
    RecordingBlockStore rec_receipts(net);
    auto r_amt = Amt<Receipt>::load(ts.receipts_root, rec_receipts, 0);
    // pass 1 (:206-239), with the predicate
    auto scan_range = [&](uint64_t a, uint64_t b, std::vector<uint64_t>& dst) {
        for (uint64_t i = a; i < b; i++) {
            if (!ts.has_root[i]) continue;
            try {
                RecordingBlockStore temp(net);
                auto amt = Amt<StampedEvent>::load(cid_from(ts.events_roots + 38 * i), temp, 3);
                bool has = false;
                amt.for_each([&](uint64_t, const StampedEvent& se) { std::optional<EvmLog> log; if (pred(se, log)) has = true; });
                if (has) dst.push_back(i);
            } catch (Err& e) { e.index = i; throw; }
        }
    };
    threads = std::max<uint32_t>(threads, 1);
    std::vector<std::vector<uint64_t>> parts(threads);
    std::vector<std::unique_ptr<Err>> errs(threads);
    std::vector<std::thread> th;
    for (uint32_t t = 0; t < threads; t++)
        th.emplace_back([&, t]() {
            uint64_t a = ts.n_receipts * t / threads, b = ts.n_receipts * (t + 1) / threads;
            try { scan_range(a, b, parts[t]); } catch (Err& e) { errs[t] = std::make_unique<Err>(e); }
        });
    for (auto& x : th) x.join();
    for (uint32_t t = 0; t < threads; t++) { if (errs[t]) throw *errs[t]; out.matching.insert(out.matching.end(), parts[t].begin(), parts[t].end()); }
    // pass 2 (:241-301)
    std::vector<std::unique_ptr<RecordingBlockStore>> event_recs;
    for (uint64_t i : out.matching) {
        if (i >= exec.size()) throw Err(IPCFP_ERR_MISSING_EXEC, "Missing message at index", i);
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

extern "C" ipcfp_status oracle_generate_log_proof(const oracle_store* s, const ipcfp_tipset_desc* t, const ipcfp_log_filter* f, uint32_t flags,
                                                  uint32_t threads, ipcfp_event_result** out) {
    return orc::guard([&] {
        orc::TipsetIn ts = orc::tipset_in(t);
        orc::EventGenOut o = orc::generate_log_proof(s->bs, ts, orc::LogPredicate(*f), flags, threads);
        *out = orc::box_event(o);
    });
}
