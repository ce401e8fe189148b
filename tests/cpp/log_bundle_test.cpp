// log_bundle_test.cpp — the log-filter overloads of include/ipcfp.hpp: generate_proof_bundle with a std::vector<LogFilter> (the filters
// LogFilter::from_spec gives for the specs make the spec bundle, field for field) and verify_proof_bundle_json with a filter set as
// check_event (all of the set's own proofs true, a set that matches nothing: every event proof false, the empty set: no check_event).
//
//   g++ -std=c++17 -o log_bundle_test tests/cpp/log_bundle_test.cpp -Lipc_filecoin_proofs_b200 -lipcfp -Lsynth -lipcfp_synth && ./log_bundle_test cpu|gpu
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../../include/ipcfp.hpp"
#include "../../synth/synth.h"

using namespace ipcfp::host;

static int g_checks = 0;
#define REQUIRE(cond)                                                                      \
    do {                                                                                   \
        g_checks++;                                                                        \
        if (!(cond)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); exit(1); } \
    } while (0)

template <class F>
static ipcfp_status status_of(F&& f) {
    try { f(); } catch (const Error& e) { return e.status; }
    return IPCFP_OK;
}

// a synthetic tipset pair with a state tree, as Lotus would serve it (synth/__init__.py::config_params(3), small HAMT)
struct Fixture {
    synth_tipset* ts = nullptr;
    ApiTipset parent, child;
    std::vector<ApiReceipt> receipts;

    Fixture() {
        synth_params p;
        synth_default_params(&p);
        p.seed = 0x1FC0FFEEull ^ 3u;
        p.n_receipts = 64; p.events_per_receipt = 8; p.match_ppm = 200000; p.with_state_tree = 1; p.hamt_entries = 2000; p.n_actors = 64;
        ts = synth_build(&p);
        REQUIRE(ts != nullptr);
        parent.height = synth_parent_epoch(ts);
        child.height = synth_child_epoch(ts);
        for (uint32_t i = 0; i < synth_n_parents(ts); i++) {
            parent.cids.push_back({Cid::from_bytes(synth_parent_cids(ts) + 38 * i).to_string()});
            ApiBlockHeader h;
            h.messages = {Cid::from_bytes(synth_parent_txmeta_cids(ts) + 38 * i).to_string()};
            h.height = parent.height;
            parent.blocks.push_back(h);
        }
        child.cids.push_back({Cid::from_bytes(synth_child_cid(ts)).to_string()});
        ApiBlockHeader ch;
        ch.parent_message_receipts = {Cid::from_bytes(synth_receipts_root(ts)).to_string()};
        ch.parent_state_root = {Cid::from_bytes(synth_parent_state_root(ts)).to_string()};
        ch.height = child.height;
        for (const auto& c : parent.cids) ch.parents.push_back(c);
        child.blocks.push_back(ch);
        receipts.resize(synth_n_receipts(ts));
        for (uint64_t i = 0; i < receipts.size(); i++)
            if (synth_has_events_root(ts)[i]) receipts[i].events_root = CIDMap{Cid::from_bytes(synth_events_roots(ts) + 38 * i).to_string()};
    }
    ~Fixture() { synth_free(ts); }
    GpuBlockstore store() const {
        return GpuBlockstore::from_flat(synth_cids(ts), synth_offsets(ts), synth_lengths(ts), synth_blob(ts), synth_blob_size(ts), synth_n_blocks(ts), 0, true);
    }
};

static bool yes_ts(int64_t, const std::vector<Cid>&) { return true; }
static bool yes_h(int64_t, const Cid&) { return true; }

static int run_cpu() {
    // more than four topic positions is refused before any call into the library
    LogFilter five;
    five.topics.resize(5);
    REQUIRE(status_of([&] { verify_proof_bundle_json("{}", yes_ts, yes_h, std::vector<LogFilter>{five}); }) == IPCFP_ERR_INVALID_ARG);
    printf("ok: cpu checks of the log-filter overloads (%d checks)\n", g_checks);
    return 0;
}

static int run_gpu() {
    Fixture f;
    GpuBlockstore store = f.store();
    const std::string sig = synth_event_signature(f.ts), t1 = synth_topic1(f.ts);
    const std::vector<EventProofSpec> es = {{sig, t1, std::nullopt}, {sig, "calib-subnet-2", std::nullopt}};
    std::vector<LogFilter> fs;
    for (const auto& e : es) fs.push_back(LogFilter::from_spec(e));
    REQUIRE(fs[0].topics.size() == 2 && fs[0].topics[1][0] == ascii_to_bytes32(t1) && fs[0].emitters.empty());
    H256 slot{};
    const std::vector<StorageProofSpec> ss = {{1001, slot}, {1003, slot}};
    const UnifiedProofBundle a = generate_proof_bundle(store, f.parent, f.child, f.receipts, ss, es);
    const UnifiedProofBundle b = generate_proof_bundle(store, f.parent, f.child, f.receipts, ss, fs);
    REQUIRE(a.storage_proofs.size() == b.storage_proofs.size() && a.event_proofs.size() == b.event_proofs.size() && !a.event_proofs.empty());
    for (size_t i = 0; i < a.storage_proofs.size(); i++) REQUIRE(a.storage_proofs[i] == b.storage_proofs[i]);
    for (size_t i = 0; i < a.event_proofs.size(); i++) REQUIRE(a.event_proofs[i] == b.event_proofs[i]);
    REQUIRE(a.blocks.size() == b.blocks.size());
    for (size_t i = 0; i < a.blocks.size(); i++) REQUIRE(a.blocks[i] == b.blocks[i]);
    const std::string text = to_json(b);
    REQUIRE(text == to_json(a));
    const UnifiedVerificationResult own = verify_proof_bundle_json(text, yes_ts, yes_h, fs);
    REQUIRE(own.storage_results.size() == ss.size() && own.event_results.size() == b.event_proofs.size());
    for (bool x : own.storage_results) REQUIRE(x);
    for (bool x : own.event_results) REQUIRE(x);
    LogFilter nothing;
    nothing.topics = {{H256{}}};
    const UnifiedVerificationResult none = verify_proof_bundle_json(text, yes_ts, yes_h, std::vector<LogFilter>{nothing});
    for (bool x : none.storage_results) REQUIRE(x);
    for (bool x : none.event_results) REQUIRE(!x);
    const UnifiedVerificationResult empty = verify_proof_bundle_json(text, yes_ts, yes_h, std::vector<LogFilter>{});
    const UnifiedVerificationResult plain = verify_proof_bundle_json(text, yes_ts, yes_h);
    REQUIRE(empty.event_results == plain.event_results && empty.storage_results == plain.storage_results);
    // one filter of the two: exactly its own proofs stay true
    const UnifiedVerificationResult first = verify_proof_bundle_json(text, yes_ts, yes_h, std::vector<LogFilter>{fs[0]});
    const EventProofSpec spec0 = es[0];
    const UnifiedVerificationResult by_spec = verify_proof_bundle_json(text, yes_ts, yes_h, &spec0);
    REQUIRE(first.event_results == by_spec.event_results);
    printf("ok: gpu checks of the log-filter overloads, %zu event proofs (%d checks)\n", b.event_proofs.size(), g_checks);
    return 0;
}

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "cpu";
    return mode == "gpu" ? run_gpu() : run_cpu();
}
