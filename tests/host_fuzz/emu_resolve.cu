// emu_resolve.cu — the per-item code of address resolution (csrc/resolve_items.cuh) executed ON THE CPU (TEST INFRASTRUCTURE, no GPU
// needed), driven as csrc/resolve.cu's kernels drive it: `resolve_init` once per case, then `resolve_lookup` for every address the host
// leaves to the device (valid, not protocol 0), each through its own Recorder over one witness bitmap. tests/test_resolve_host.py writes
// the cases (the catalogue of tests/address_trees.py, dropped blocks, seeded truncations and bit flips) and compares the output with
// that module's restatement; under AddressSanitizer + UBSan it also shows the walks stay inside the padded block buffers.
//
//   emu_resolve <case file>   per case: "case <k> init <status>", "addr <status> <id>" per address, "missing <cid hex>" (sorted, unique),
//                             "witness <cid hex>" (sorted), "end"
// Case file: u64 n_blocks, n_blocks × {cid (38), u32 len, bytes}; u32 n_cases; per case: root (38), u8 strict, u32 n_addrs,
// n_addrs × {u8 len, bytes}, u32 n_drop, n_drop × u64 block index, u32 n_mut, n_mut × {u64 block index, u32 len, bytes}.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/resolve_items.cuh"
#include "host_store.h"

using namespace ipcfp;

static FILE* g_in;
static void rd(void* p, size_t n) {
    if (n && fread(p, 1, n, g_in) != n) { fprintf(stderr, "emu_resolve: truncated case file\n"); exit(2); }
}
template <class T> static T rd1() { T v; rd(&v, sizeof v); return v; }
static std::string hex(const uint8_t* p, size_t n) {
    static const char* D = "0123456789abcdef";
    std::string s;
    for (size_t i = 0; i < n; i++) { s.push_back(D[p[i] >> 4]); s.push_back(D[p[i] & 15]); }
    return s;
}

int main(int argc, char** argv) {
    if (argc != 2 || !(g_in = fopen(argv[1], "rb"))) { fprintf(stderr, "usage: emu_resolve <case file>\n"); return 2; }
    const uint64_t nb = rd1<uint64_t>();
    std::vector<std::vector<uint8_t>> cids(nb, std::vector<uint8_t>(38)), data(nb);
    for (uint64_t i = 0; i < nb; i++) {
        rd(cids[i].data(), 38);
        data[i].resize(rd1<uint32_t>());
        rd(data[i].data(), data[i].size());
    }
    const uint32_t nc = rd1<uint32_t>();
    for (uint32_t k = 0; k < nc; k++) {
        alignas(8) uint8_t root[64] = {};   // the state root sits in a 64-byte slot of the call's upload, as in csrc/resolve.cu
        rd(root, 38);
        const bool strict = rd1<uint8_t>() != 0;
        std::vector<ipcfp_address> addrs(rd1<uint32_t>());
        for (auto& a : addrs) { memset(&a, 0, sizeof a); a.len = rd1<uint8_t>(); rd(a.bytes, a.len); }
        std::set<uint64_t> drop;
        for (uint32_t n = rd1<uint32_t>(); n--;) drop.insert(rd1<uint64_t>());
        std::vector<std::vector<uint8_t>> blk = data;
        for (uint32_t n = rd1<uint32_t>(); n--;) { const uint64_t i = rd1<uint64_t>(); blk[i].resize(rd1<uint32_t>()); rd(blk[i].data(), blk[i].size()); }
        // the case's store: the blocks not dropped, 16-byte aligned as ipcfp_store_create lays them out
        std::vector<uint8_t> c, blob;
        std::vector<uint64_t> offs;
        std::vector<uint32_t> lens;
        for (uint64_t i = 0; i < nb; i++) {
            if (drop.count(i)) continue;
            c.insert(c.end(), cids[i].begin(), cids[i].end());
            blob.resize((blob.size() + 15) & ~(size_t)15);
            offs.push_back(blob.size());
            lens.push_back((uint32_t)blk[i].size());
            blob.insert(blob.end(), blk[i].begin(), blk[i].end());
        }
        const uint64_t n = lens.size();
        HostStore hs(c.data(), offs.data(), lens.data(), blob.data(), blob.size(), n);
        std::vector<uint32_t> wbits((n + 31) / 32 + 8, 0);
        std::set<std::string> missing;
        Recorder rec0{nullptr, 0, wbits.data(), false};
        rec0.strict_only = strict;
        Fail f{0, 0};
        const uint8_t* map = nullptr;
        int init = IPCFP_OK;
        if (!resolve_init(hs.view, rec0, root, map, f)) {
            init = resolve_status(f.code);
            if (f.code == DC_MISSING) missing.insert(hex(rec0.missing, 38));
        }
        printf("case %u init %d\n", k, init);
        for (const ipcfp_address& a : addrs) {
            if (init != IPCFP_OK) { printf("addr %d 0\n", init); continue; }
            Recorder rec{nullptr, 0, wbits.data(), false};
            rec.strict_only = strict;
            Fail g{0, 0};
            uint64_t id = 0;
            if (resolve_lookup(hs.view, rec, map, a.bytes, a.len, id, g)) printf("addr %d %llu\n", IPCFP_OK, (unsigned long long)id);
            else {
                printf("addr %d 0\n", resolve_status(g.code));
                if (g.code == DC_MISSING) missing.insert(hex(rec.missing, 38));
            }
        }
        for (const std::string& m : missing) printf("missing %s\n", m.c_str());
        std::vector<std::string> wit;
        for (uint64_t i = 0; i < n; i++)
            if (wbits[i >> 5] >> (i & 31) & 1) wit.push_back(hex(c.data() + 38 * i, 38));
        std::sort(wit.begin(), wit.end());
        for (const std::string& w : wit) printf("witness %s\n", w.c_str());
        printf("end\n");
    }
    return 0;
}
