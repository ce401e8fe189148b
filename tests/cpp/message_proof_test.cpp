// message_proof_test.cpp — the message overload of include/ipcfp.hpp: generate_event_proof(store, parent, child, receipts,
// std::vector<Cid>, optional LogFilter) → the EventProofBundle restricted to those messages' receipts and every message's execution
// position. Checked against generate_log_proof of the same filter restricted by hand, with duplicates and a CID the tipset did not run.
//
//   g++ -std=c++17 -o message_proof_test tests/cpp/message_proof_test.cpp -Lipc_filecoin_proofs_b200 -lipcfp -Lsynth -lipcfp_synth && ./message_proof_test cpu|gpu
#include <cstdio>
#include <cstdlib>
#include <map>
#include <set>
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

static int run_cpu() {
    // the result type: an empty bundle and no positions until a call fills them; a position is a message's index or none
    const MessageLogProof m;
    REQUIRE(m.bundle.proofs.empty() && m.bundle.blocks.empty() && m.exec_indices.empty());
    printf("ok: cpu checks of the message overload (%d checks)\n", g_checks);
    return 0;
}

static int run_gpu() {
    Fixture f;
    GpuBlockstore store = f.store();
    // every log: each receipt's message CID from the proofs of the all-wildcard filter
    const EventProofBundle all = generate_log_proof(store, f.parent, f.child, f.receipts, LogFilter{});
    std::map<uint64_t, std::string> msg_of;
    for (const auto& p : all.proofs) msg_of[p.exec_index] = p.message_cid;
    REQUIRE(msg_of.size() > 8);
    std::vector<Cid> msgs;
    std::set<uint64_t> picked;
    uint64_t k = 0;
    for (const auto& [i, c] : msg_of) {
        if (k++ % 3) continue;
        msgs.push_back(Cid::try_from(c));
        picked.insert(i);
    }
    msgs.push_back(msgs.front());   // a duplicate
    Cid stranger = msgs.front();
    stranger.bytes[37] ^= 0x5a;     // a CID the tipset did not execute
    msgs.push_back(stranger);
    // more than four topic positions is refused before any call into the library
    LogFilter five;
    five.topics.resize(5);
    REQUIRE(status_of([&] { generate_event_proof(store, f.parent, f.child, f.receipts, msgs, five); }) == IPCFP_ERR_INVALID_ARG);
    for (const std::optional<LogFilter>& flt : {std::optional<LogFilter>{}, std::optional<LogFilter>{LogFilter::from_spec({synth_event_signature(f.ts), synth_topic1(f.ts), std::nullopt})}}) {
        const MessageLogProof m = generate_event_proof(store, f.parent, f.child, f.receipts, msgs, flt);
        const EventProofBundle full = flt ? generate_log_proof(store, f.parent, f.child, f.receipts, *flt) : all;
        std::vector<EventProof> want;
        for (const auto& p : full.proofs) if (picked.count(p.exec_index)) want.push_back(p);
        REQUIRE(m.bundle.proofs.size() == want.size());
        for (size_t i = 0; i < want.size(); i++) REQUIRE(m.bundle.proofs[i] == want[i]);
        REQUIRE(m.exec_indices.size() == msgs.size());
        k = 0;
        for (const auto& [i, c] : msg_of) if (k++ % 3 == 0) REQUIRE(m.exec_indices[(k - 1) / 3] == std::optional<uint64_t>(i));
        REQUIRE(m.exec_indices[msgs.size() - 2] == m.exec_indices[0]);
        REQUIRE(!m.exec_indices.back());
        REQUIRE(!m.bundle.blocks.empty());
        if (!flt) REQUIRE(!want.empty());
    }
    printf("ok: gpu checks of the message overload, %zu messages (%d checks)\n", msgs.size(), g_checks);
    return 0;
}

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "cpu";
    return mode == "gpu" ? run_gpu() : run_cpu();
}
