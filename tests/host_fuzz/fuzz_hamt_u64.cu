// fuzz_hamt_u64.cu — one address_map HAMT node (the ActorID value kind HV_U64 of csrc/ipld.cuh) through the strict decoder
// `hamt_node_lookup`, the fast decoder `hamt_node_lookup_fast` and the C++ oracle (`oracle_hamt_u64_node_lookup`, tests/oracle_resolve.cpp,
// on oracle/oracle.cpp's HAMT node decoder). TEST INFRASTRUCTURE, no GPU needed. Nodes: up to 6 pointers at bit width 5, links and
// buckets of 1–3 [key, value] pairs with Address::to_bytes()-length keys; values at every CBOR head size, sometimes not minimal, negative,
// bytes, text, null, a float or a map; half the nodes then get one or two random edits. Properties:
//   1. the fast decoder only accepts what the strict one accepts, with the same hit, and it takes every generated unedited node whose
//      values are all minimal unsigned integers;
//   2. the strict decoder and the oracle agree: decode error or not, and the hit (none / the value's integer / the link's CID).
//
//   nvcc -std=c++17 -O2 -o fuzz_hamt_u64 tests/host_fuzz/fuzz_hamt_u64.cu tests/oracle_resolve.cpp -lpthread && ./fuzz_hamt_u64 200000 7
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/ipld.cuh"

extern "C" ipcfp_status oracle_hamt_u64_node_lookup(const uint8_t* p, uint64_t n, uint32_t idx, const uint8_t* key, uint32_t keylen, int32_t* kind,
                                                    uint64_t* value, uint8_t* out38);

using namespace ipcfp;

static uint64_t g_s;
static uint64_t rnd() {  // SplitMix64
    uint64_t z = (g_s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static void put_head(std::vector<uint8_t>& o, int major, uint64_t v, int force_ai = 0) {
    int ai = force_ai ? force_ai : v < 24 ? 0 : v < 0x100 ? 24 : v < 0x10000 ? 25 : v < 0x100000000ull ? 26 : 27;
    if (!ai) { o.push_back((uint8_t)(major << 5 | v)); return; }
    o.push_back((uint8_t)(major << 5 | ai));
    for (int b = (1 << (ai - 24)) - 1; b >= 0; b--) o.push_back((uint8_t)(v >> (8 * b)));
}
static const uint64_t SIZES[] = {0, 23, 24, 255, 256, 65535, 65536, 0xffffffffull, 0x100000000ull, 0xffffffffffffffffull};

int main(int argc, char** argv) {
    const uint64_t iters = argc > 1 ? strtoull(argv[1], nullptr, 10) : 100000;
    g_s = argc > 2 ? strtoull(argv[2], nullptr, 10) : 1;
    uint64_t okn = 0, bad = 0, hits = 0, links = 0, fast_ok = 0;
    std::vector<uint8_t> buf;
    for (uint64_t it = 0; it < iters; it++) {
        const uint32_t np = (uint32_t)(rnd() % 7);
        uint32_t bits = 0;
        for (uint32_t k = 0; k < np;) { uint32_t b = (uint32_t)(rnd() % 32); if (!(bits >> b & 1)) { bits |= 1u << b; k++; } }
        std::vector<uint8_t> bf;
        for (int s = 24; s >= 0; s -= 8) if (!bf.empty() || (bits >> s) & 0xff) bf.push_back((uint8_t)(bits >> s));
        std::vector<uint8_t> node;
        put_head(node, 4, 2);
        put_head(node, 2, bf.size());
        node.insert(node.end(), bf.begin(), bf.end());
        put_head(node, 4, np);
        std::vector<std::vector<uint8_t>> keys;
        bool all_minimal = true;
        for (uint32_t k = 0; k < np; k++) {
            if (rnd() % 4 == 0) {
                static const uint8_t head[11] = {0xd8, 0x2a, 0x58, 0x27, 0x00, 0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
                node.insert(node.end(), head, head + 11);
                for (int b = 0; b < 32; b++) node.push_back((uint8_t)rnd());
                continue;
            }
            const uint32_t nk = 1 + (uint32_t)(rnd() % 3);
            put_head(node, 4, nk);
            for (uint32_t j = 0; j < nk; j++) {
                put_head(node, 4, 2);
                static const uint32_t LENS[] = {2, 11, 21, 22, 49, 1, 65};
                std::vector<uint8_t> key(LENS[rnd() % 7]);
                for (auto& b : key) b = (uint8_t)rnd();
                if (!keys.empty() && rnd() % 16 == 0) key = keys[rnd() % keys.size()];   // a repeated key: the first one wins
                keys.push_back(key);
                put_head(node, 2, key.size());
                node.insert(node.end(), key.begin(), key.end());
                const uint64_t v = rnd() % 2 ? SIZES[rnd() % 10] : rnd() >> (rnd() % 64);
                switch (rnd() % 48) {   // about one value in seven is not a minimal unsigned integer
                    case 0: {   // a head at least as wide as the value needs: not minimal unless it is the natural one
                        const int nat = v < 24 ? 0 : v < 0x100 ? 24 : v < 0x10000 ? 25 : v < 0x100000000ull ? 26 : 27;
                        int ai = 24 + (int)(rnd() % 4);
                        if (ai < nat) ai = nat;
                        put_head(node, 0, v, ai);
                        all_minimal &= ai == nat;
                        break;
                    }
                    case 1: put_head(node, 1, v); all_minimal = false; break;
                    case 2: put_head(node, 2, 1); node.push_back((uint8_t)v); all_minimal = false; break;
                    case 3: put_head(node, 3, 1); node.push_back('7'); all_minimal = false; break;
                    case 4: node.push_back(0xf6); all_minimal = false; break;
                    case 5: node.push_back(0xf9); node.push_back(0x3c); node.push_back(0x00); all_minimal = false; break;
                    case 6: node.push_back(0xa0); all_minimal = false; break;
                    default: put_head(node, 0, v); break;
                }
            }
        }
        const unsigned nmut = it % 2 ? 1 + (unsigned)(rnd() % 2) : 0;
        for (unsigned m = 0; m < nmut; m++) {
            const size_t at = rnd() % node.size();
            switch (rnd() % 4) {
                case 0: node[at] = (uint8_t)rnd(); break;
                case 1: node[at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                case 2: node.erase(node.begin() + (long)at); break;
                default: node.insert(node.begin() + (long)at, (uint8_t)rnd()); break;
            }
            if (node.empty()) node.push_back(0x82);
        }
        std::vector<uint8_t> key = (!keys.empty() && rnd() % 4) ? keys[rnd() % keys.size()] : std::vector<uint8_t>(22, (uint8_t)rnd());
        uint32_t idx = (uint32_t)(rnd() % 32);
        if (bits && rnd() % 2) { do idx = (uint32_t)(rnd() % 32); while (!(bits >> idx & 1)); }
        // the node sits in a buffer padded as the engine's arena is (reads past the end stay inside it)
        const unsigned lead = (unsigned)(rnd() % 16);
        buf.assign(16 + lead, 0xEE);
        buf.insert(buf.end(), node.begin(), node.end());
        buf.insert(buf.end(), 48, (uint8_t)rnd());
        const uint8_t* p = buf.data() + 16 + lead;
        const uint32_t len = (uint32_t)node.size();
        Rd r(p, len);
        HamtHit hit;
        hamt_node_lookup(r, HV_U64, idx, key.data(), (uint32_t)key.size(), hit);
        HamtHit fh;
        if (hamt_node_lookup_fast(p, len, HV_U64, idx, key.data(), (uint32_t)key.size(), fh)) {
            fast_ok++;
            if (r.err || fh.kind != hit.kind || (fh.kind == 1 && fh.val_off != hit.val_off) || (fh.kind == 2 && fh.link_off != hit.link_off)) {
                fprintf(stderr, "FAST/STRICT MISMATCH at iteration %llu: strict err %u kind %d, fast kind %d\n", (unsigned long long)it, r.err, hit.kind, fh.kind);
                return 1;
            }
        } else if (!r.err && nmut == 0 && all_minimal) {
            fprintf(stderr, "FAST: a generated, unedited node with minimal values was not taken (iteration %llu)\n", (unsigned long long)it);
            return 1;
        }
        int32_t okind = 0;
        uint64_t oval = 0;
        uint8_t ocid[38];
        const int ost = (int)oracle_hamt_u64_node_lookup(p, len, idx, key.data(), (uint32_t)key.size(), &okind, &oval, ocid);
        bool ok = (ost == IPCFP_OK) == (r.err == 0);
        if (ok && !r.err) {
            ok = okind == hit.kind;
            if (ok && hit.kind == 2) ok = memcmp(p + hit.link_off, ocid, 38) == 0;
            if (ok && hit.kind == 1) { Rd r2(p, len); r2.pos = hit.val_off; ok = rd_uint(r2) == oval && !r2.err; }
        }
        if (!ok) {
            fprintf(stderr, "NODE MISMATCH at iteration %llu: device err %u kind %d; oracle status %d kind %d\nnode:", (unsigned long long)it, r.err, hit.kind, ost, okind);
            for (size_t k = 0; k < node.size(); k++) fprintf(stderr, " %02x", node[k]);
            fprintf(stderr, "\n");
            return 1;
        }
        if (r.err) bad++; else { okn++; hits += hit.kind == 1; links += hit.kind == 2; }
    }
    printf("ok: %llu address_map nodes agree with the oracle (%llu decoded: %llu values found, %llu links; %llu decode errors; %llu taken by the fast "
           "node decoder)\n", (unsigned long long)iters, (unsigned long long)okn, (unsigned long long)hits, (unsigned long long)links, (unsigned long long)bad,
           (unsigned long long)fast_ok);
    return 0;
}
