// actor_proof_test.cpp — the actor-proof functions of include/ipcfp.hpp, driven by tests/test_cpp_actor_proof.py.
//
//   actor_proof_test gpu <case file>   plan_fetch_actor_proofs on a store of the child header alone (it names the StateRoot), then
//                                      generate_actor_proofs with code over the case file's blocks, printed for the test to compare with
//                                      the Python restatement, then verify_actor_proofs on the result and on a proof with a changed balance
// Case file: child CID (38), state root (38), u64 n_evm, n_evm × CID (38), u64 n_blocks, n_blocks × {cid (38), u32 len, bytes},
// u64 n_addrs, n_addrs × {u8 len, bytes}.
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../../include/ipcfp.hpp"

using namespace ipcfp::host;

static int g_checks = 0;
#define REQUIRE(cond)                                                                      \
    do {                                                                                   \
        g_checks++;                                                                        \
        if (!(cond)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); exit(1); } \
    } while (0)

static std::string hex(const uint8_t* p, size_t n) { return to_hex0x(p, n).substr(2); }

static int gpu(const char* path) {
    FILE* f = fopen(path, "rb");
    REQUIRE(f);
    auto rd = [&](void* p, size_t n) { REQUIRE(fread(p, 1, n, f) == n); };
    uint8_t child_b[IPCFP_CID_LEN], root_b[IPCFP_CID_LEN];
    rd(child_b, IPCFP_CID_LEN);
    rd(root_b, IPCFP_CID_LEN);
    uint64_t ne = 0;
    rd(&ne, 8);
    std::vector<Cid> evm(ne);
    for (Cid& c : evm) rd(c.bytes.data(), IPCFP_CID_LEN);
    uint64_t nb = 0;
    rd(&nb, 8);
    std::vector<std::pair<Cid, std::vector<uint8_t>>> blocks(nb);
    for (auto& kv : blocks) {
        rd(kv.first.bytes.data(), IPCFP_CID_LEN);
        uint32_t len = 0;
        rd(&len, 4);
        kv.second.resize(len);
        if (len) rd(kv.second.data(), len);
    }
    uint64_t na = 0;
    rd(&na, 8);
    std::vector<ipcfp_address> addrs(na);
    for (auto& a : addrs) {
        memset(&a, 0, sizeof a);
        rd(&a.len, 1);
        if (a.len) rd(a.bytes, a.len);
    }
    fclose(f);
    const Cid child = Cid::from_bytes(child_b), root = Cid::from_bytes(root_b);
    {
        GpuBlockstore empty = GpuBlockstore::ingest(std::vector<std::pair<Cid, std::vector<uint8_t>>>{{blocks[0].first, blocks[0].second}}, 0, true);
        const std::vector<Cid> plan = plan_fetch_actor_proofs(empty, child, root, addrs, evm, true);
        REQUIRE(plan.size() == 1 && plan[0] == root);   // the header is there: every walk first lacks the StateRoot
    }
    GpuBlockstore store = GpuBlockstore::ingest(blocks, 0, true);
    REQUIRE(plan_fetch_actor_proofs(store, child, root, addrs, evm, true).empty());
    ActorProofs ap = generate_actor_proofs(store, child, root, addrs, evm, true);
    REQUIRE(ap.proofs.size() == na);
    for (const ActorProof& p : ap.proofs) {
        std::string line = "proof " + hex((const uint8_t*)&p.c, sizeof p.c) + " " + (p.bytecode.empty() ? "-" : hex(p.bytecode.data(), p.bytecode.size()));
        for (size_t k : p.witness) line += " " + hex(ap.blocks[k].cid.bytes.data(), IPCFP_CID_LEN);
        printf("%s\n", line.c_str());
    }
    for (const ProofBlock& b : ap.blocks) printf("witness %s %zu\n", hex(b.cid.bytes.data(), IPCFP_CID_LEN).c_str(), b.data.size());
    const std::vector<bool> ok = verify_actor_proofs(ap, child, root, evm, true);
    for (bool v : ok) REQUIRE(v);
    ActorProofs lie = ap;
    lie.proofs[0].c.balance[31] ^= 1;
    REQUIRE(!verify_actor_proofs(lie, child, root, evm, true)[0]);
    printf("ok: %d assertions\n", g_checks);
    return 0;
}

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    if (mode == "gpu" && argc == 3) return gpu(argv[2]);
    fprintf(stderr, "usage: actor_proof_test gpu <case file>\n");
    return 2;
}
