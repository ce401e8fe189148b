// message_proofs_test.cpp — the message-proof functions of include/ipcfp.hpp: generate_message_proofs, plan_fetch_message_proofs and
// verify_message_proofs. Checked against generate_log_proof's message CIDs and execution positions, the receipt list the tipset was
// described with, a CID the tipset did not execute, a duplicate, a changed claim and the refusals.
//
//   g++ -std=c++17 -o message_proofs_test tests/cpp/message_proofs_test.cpp -Lipc_filecoin_proofs_b200 -lipcfp -Lsynth -lipcfp_synth && ./message_proofs_test cpu|gpu
#include <cstdio>
#include <cstdlib>
#include <map>
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
    static_assert(sizeof(ipcfp_message_proof) == 400 && alignof(ipcfp_message_proof) == 8, "the documented record");
    const MessageProofs m;
    REQUIRE(m.proofs.empty() && m.blocks.empty());
    printf("ok: cpu checks of the message-proof functions (%d checks)\n", g_checks);
    return 0;
}

static int run_gpu() {
    Fixture f;
    GpuBlockstore store = f.store();
    // every receipt's message CID and position, from the proofs of the all-wildcard filter
    const EventProofBundle all = generate_log_proof(store, f.parent, f.child, f.receipts, LogFilter{});
    std::map<uint64_t, std::string> msg_of;
    for (const auto& p : all.proofs) msg_of[p.exec_index] = p.message_cid;
    REQUIRE(msg_of.size() > 8);
    std::vector<Cid> msgs;
    std::vector<uint64_t> pos;
    for (const auto& [i, c] : msg_of) { msgs.push_back(Cid::try_from(c)); pos.push_back(i); }
    msgs.push_back(msgs.front());   // a duplicate
    pos.push_back(pos.front());
    Cid stranger = msgs.front();
    stranger.bytes[37] ^= 0x5a;     // a CID the tipset did not execute
    msgs.push_back(stranger);
    const MessageProofs m = generate_message_proofs(store, f.parent, f.child, f.receipts, msgs);
    REQUIRE(m.proofs.size() == msgs.size() && !m.blocks.empty());
    for (size_t k = 0; k + 1 < msgs.size(); k++) {
        const ipcfp_message_proof& c = m.proofs[k].c;
        REQUIRE(c.status == IPCFP_MESSAGE_EXECUTED && c.exec_index == pos[k] && !c.has_body);
        REQUIRE(memcmp(c.message_cid, msgs[k].bytes.data(), IPCFP_CID_LEN) == 0);
        const auto& er = f.receipts[pos[k]].events_root;
        REQUIRE(c.has_events_root == (er ? 1 : 0));
        if (er) REQUIRE(Cid::from_bytes(c.events_root).to_string() == er->cid);
    }
    REQUIRE(m.proofs.back().c.status == IPCFP_MESSAGE_NOT_EXECUTED && m.proofs.back().c.exec_index == UINT64_MAX);
    // the verifier accepts every proof, and rejects a changed exit code
    const std::vector<bool> ok = verify_message_proofs(m, f.parent, f.child, f.receipts);
    REQUIRE(ok.size() == msgs.size());
    for (bool b : ok) REQUIRE(b);
    MessageProofs bad = m;
    bad.proofs[1].c.exit_code ^= 1;
    const std::vector<bool> v = verify_message_proofs(bad, f.parent, f.child, f.receipts);
    REQUIRE(v[0] && !v[1] && v[2]);
    // the complete store needs nothing; the synthetic messages have no blocks, so the body is missing at the first request
    REQUIRE(plan_fetch_message_proofs(store, f.parent, f.child, f.receipts, msgs).empty());
    REQUIRE(plan_fetch_message_proofs(store, f.parent, f.child, f.receipts, msgs, true).size() == msgs.size() - 2);
    REQUIRE(status_of([&] { generate_message_proofs(store, f.parent, f.child, f.receipts, msgs, true); }) == IPCFP_ERR_MISSING_BLOCK);
    REQUIRE(status_of([&] { generate_message_proofs(store, f.parent, f.child, f.receipts, std::vector<Cid>(IPCFP_MESSAGE_MAX + 1, stranger)); }) ==
            IPCFP_ERR_INVALID_ARG);
    printf("ok: gpu checks of the message-proof functions, %zu messages (%d checks)\n", msgs.size(), g_checks);
    return 0;
}

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "cpu";
    return mode == "gpu" ? run_gpu() : run_cpu();
}
