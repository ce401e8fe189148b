// resolve_test.cpp — the address-resolution functions of include/ipcfp.hpp, driven by tests/test_cpp_resolve.py.
//
//   resolve_test cpu                          no device needed: parse_address and the reference's Ethereum-address validation
//   resolve_test gpu <case file> <eth hex>    resolve_addresses over the case file's blocks and addresses, printed for the test to compare
//                                             with the Python restatement; then resolve_eth_address_to_actor_id(<eth hex>)
// Case file: state root (38 bytes), u64 n_blocks, n_blocks × {cid (38), u32 len, bytes}, u64 n_addrs, n_addrs × {u8 len, bytes}.
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

template <class F>
static std::string message_of(F&& f) {
    try { f(); } catch (const Error& e) { return e.what(); }
    return "";
}

static std::string hex(const uint8_t* p, size_t n) { return to_hex0x(p, n).substr(2); }

static int cpu() {
    const ipcfp_address a = parse_address("f410f2oekwcmo2pueydmaq53eic2i62crtbeyuzx2gmy");
    REQUIRE(hex(a.bytes, a.len) == "040ad388ab098ed3e84c0d808776440b48f685198498");
    const ipcfp_address b = eth_to_filecoin_address("0x0xd388ab098ed3e84c0d808776440b48f685198498");
    REQUIRE(b.len == a.len && memcmp(a.bytes, b.bytes, a.len) == 0);
    const ipcfp_address id = parse_address("t01");
    REQUIRE(id.len == 2 && id.bytes[0] == 0 && id.bytes[1] == 1);
    const ipcfp_address m = eth_to_filecoin_address("0xff00000000000000000000000000000000000401");
    REQUIRE(hex(m.bytes, m.len) == "008108");
    REQUIRE(message_of([] { eth_to_filecoin_address("0xabc"); }) == "Invalid hex in Ethereum address: Odd number of digits");
    REQUIRE(message_of([] { eth_to_filecoin_address("0xd388z"); }) == "Invalid hex in Ethereum address: Odd number of digits");
    REQUIRE(message_of([] { eth_to_filecoin_address("0xd388zb"); }) == "Invalid hex in Ethereum address: Invalid character 'z' at position 4");
    REQUIRE(message_of([] { eth_to_filecoin_address("0xd388"); }) == "Invalid Ethereum address length: expected 20 bytes, got 2");
    REQUIRE(message_of([] { parse_address("f1abc"); }).rfind("Failed to parse address 'f1abc'", 0) == 0);
    printf("ok: cpu checks of the address functions of include/ipcfp.hpp, %d assertions\n", g_checks);
    return 0;
}

static int gpu(const char* path, const std::string& eth) {
    FILE* f = fopen(path, "rb");
    REQUIRE(f);
    auto rd = [&](void* p, size_t n) { REQUIRE(fread(p, 1, n, f) == n); };
    uint8_t root[IPCFP_CID_LEN];
    rd(root, IPCFP_CID_LEN);
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
    GpuBlockstore store = GpuBlockstore::ingest(blocks, 0, true);
    const Cid sr = Cid::from_bytes(root);
    const ResolvedAddresses r = resolve_addresses(store, sr, addrs);
    printf("init %d\n", (int)r.init_status);
    for (size_t i = 0; i < na; i++) printf("addr %d %llu\n", (int)r.status[i], (unsigned long long)r.actor_ids[i]);
    for (const Cid& c : r.missing) printf("missing %s\n", hex(c.bytes.data(), IPCFP_CID_LEN).c_str());
    for (const ProofBlock& b : r.witness) printf("witness %s %zu\n", hex(b.cid.bytes.data(), IPCFP_CID_LEN).c_str(), b.data.size());
    printf("eth %llu\n", (unsigned long long)resolve_eth_address_to_actor_id(store, sr, eth));
    ipcfp_status st = IPCFP_OK;
    try { resolve_eth_address_to_actor_id(store, sr, "0x" + std::string(40, '0')); } catch (const Error& e) { st = e.status; }
    printf("unknown %d\n", (int)st);
    printf("ok: %d assertions\n", g_checks);
    return 0;
}

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    if (mode == "cpu") return cpu();
    if (mode == "gpu" && argc == 4) return gpu(argv[2], argv[3]);
    fprintf(stderr, "usage: resolve_test cpu | gpu <case file> <eth hex>\n");
    return 2;
}
