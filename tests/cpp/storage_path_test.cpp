// storage_path_test.cpp — the storage-path functions of include/ipcfp.hpp (StoragePath, generate_storage_path_proofs,
// plan_fetch_storage_paths, verify_storage_paths), driven by tests/test_cpp_storage_path.py.
//
//   storage_path_test <case file>   reads a nested-mapping struct member and two long strings of the contract of tests/storage_paths.py,
//                                   prints every path's status, value and proof count for the test to compare with the restatement,
//                                   then checks that the store needs no further block and that the proofs verify (and a changed
//                                   value does not)
// Case file: child block CID (38), state root (38), u64 n_blocks, n_blocks × {cid (38), u32 len, bytes}, subnet id (32), u64 text key.
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../../include/ipcfp.hpp"

using namespace ipcfp::host;

#define REQUIRE(cond)                                                                      \
    do {                                                                                   \
        if (!(cond)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); exit(1); } \
    } while (0)

static void rd(FILE* f, void* p, size_t n) { REQUIRE(fread(p, 1, n, f) == n); }

int main(int argc, char** argv) {
    REQUIRE(argc == 2);
    FILE* f = fopen(argv[1], "rb");
    REQUIRE(f);
    uint8_t child[38], root[38];
    rd(f, child, 38);
    rd(f, root, 38);
    uint64_t n = 0;
    rd(f, &n, 8);
    std::vector<std::pair<Cid, std::vector<uint8_t>>> blocks(n);
    for (auto& b : blocks) {
        uint8_t c[38];
        uint32_t len = 0;
        rd(f, c, 38);
        rd(f, &len, 4);
        b.first = Cid::from_bytes(c);
        b.second.resize(len);
        if (len) rd(f, b.second.data(), len);
    }
    H256 subnet{};
    uint64_t text_key = 0;
    rd(f, subnet.data(), 32);
    rd(f, &text_key, 8);
    fclose(f);

    GpuBlockstore store = GpuBlockstore::ingest(blocks);
    ApiTipset parent, ch;
    const std::string cc = Cid::from_bytes(child).to_string(), rc = Cid::from_bytes(root).to_string();
    ch.cids.push_back(CIDMap{cc});
    ApiBlockHeader h;
    h.parent_state_root = CIDMap{rc};
    h.parent_message_receipts = CIDMap{cc};
    h.messages = CIDMap{cc};
    ch.blocks.push_back(h);
    H256 key{};
    for (int i = 0; i < 8; i++) key[31 - i] = (uint8_t)(text_key >> (8 * i));
    const StoragePath subnets = StoragePath::at(4242, 0).mapping(subnet);
    const std::vector<StoragePath> paths = {subnets.field(1), subnets.field(2).bytes(), StoragePath::at(4242, 12).mapping(key).bytes()};

    const StoragePathProofs r = generate_storage_path_proofs(store, parent, ch, paths);
    REQUIRE(r.paths.size() == paths.size());
    std::vector<StorageProof> all;
    for (const auto& v : r.paths) {
        printf("path %u %s %zu\n", v.status, to_hex0x(v.value.data(), v.value.size()).c_str(), v.proofs.size());
        all.insert(all.end(), v.proofs.begin(), v.proofs.end());
    }
    REQUIRE(plan_fetch_storage_paths(store, parent, ch, paths).empty());
    const auto trust = [](int64_t, const Cid&) { return true; };
    const auto ok = verify_storage_paths(all, r.blocks, paths, trust);
    for (size_t i = 0; i < ok.size(); i++) {
        REQUIRE(ok[i].valid && ok[i].status == r.paths[i].status && ok[i].value == r.paths[i].value);
    }
    std::vector<StorageProof> bad = all;
    std::string& v = bad.back().value;   // the long string's last data word
    v[2] = v[2] == '0' ? '1' : '0';
    const auto no = verify_storage_paths(bad, r.blocks, paths, trust);
    REQUIRE(no[0].valid && no[1].valid && !no[2].valid);
    const auto untrusted = verify_storage_paths(all, r.blocks, paths, [](int64_t, const Cid&) { return false; });
    REQUIRE(!untrusted[0].valid);
    printf("ok: storage paths through include/ipcfp.hpp\n");
    return 0;
}
