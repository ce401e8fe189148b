// emu_storage_paths.cu — the per-path code of the storage-path calls (csrc/storage_path_items.cuh) executed ON THE CPU (TEST
// INFRASTRUCTURE, no GPU needed). tests/test_storage_paths_host.py writes paths and the words storage holds; this program runs them
// as the kernels do — path_fixed_specs (k_path_slots), path_expand on the fixed words (k_path_expand), the data slots keccak256(slot) + j
// (k_path_place_specs), path_value over the words in expanded order (k_path_values) — and prints every path's outcome, which the test
// compares with the Python restatement (tests/storage_paths.py). It also checks keccak_key_slot against hashes.cuh's keccak256 at every
// key length 0..IPCFP_PATH_MAX_KEY.
//
// input (text): n_words, then n_words lines "slot_hex word_hex"; n_paths, then per path "actor base_hex kind n_words n_steps" and
// n_steps lines "op key_len key_hex|- index elem_slots elem_bytes"
// output: per path "status slot_hex byte_offset n_specs spec_hex… value_hex|-"
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/storage_path_items.cuh"

using namespace ipcfp;

static std::vector<uint8_t> unhex(const char* s) {
    std::vector<uint8_t> out;
    if (!strcmp(s, "-")) return out;
    for (size_t i = 0; s[i] && s[i + 1]; i += 2) { unsigned v; sscanf(s + i, "%2x", &v); out.push_back((uint8_t)v); }
    return out;
}
static void hex(const uint8_t* p, size_t n) { for (size_t i = 0; i < n; i++) printf("%02x", p[i]); }

static int keccak_self_check() {
    std::vector<uint8_t> buf(IPCFP_PATH_MAX_KEY + 32 + 64, 0);
    uint64_t x = 88172645463325252ull;
    for (auto& b : buf) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; b = (uint8_t)x; }
    std::vector<uint8_t> msg(buf.size() + 64, 0);
    for (uint32_t len = 0; len <= IPCFP_PATH_MAX_KEY; len++) {
        uint8_t a[32];
        keccak_key_slot(buf.data(), len, buf.data() + IPCFP_PATH_MAX_KEY + 8, a);
        memcpy(msg.data(), buf.data(), len);
        memcpy(msg.data() + len, buf.data() + IPCFP_PATH_MAX_KEY + 8, 32);
        Digest d;
        keccak256(msg.data(), len + 32, d);
        if (memcmp(a, d.w, 32)) { fprintf(stderr, "keccak_key_slot != keccak256 at key length %u\n", len); return 1; }
    }
    return 0;
}

int main(int argc, char** argv) {
    if (keccak_self_check()) return 1;
    if (argc < 2) { fprintf(stderr, "usage: emu_storage_paths input\n"); return 2; }
    FILE* in = fopen(argv[1], "r");
    if (!in) return 2;
    static char a[4096], b[4096];
    std::map<std::string, std::vector<uint8_t>> words;
    unsigned long long nw = 0;
    if (fscanf(in, "%llu", &nw) != 1) return 2;
    for (unsigned long long i = 0; i < nw; i++) { if (fscanf(in, "%s %s", a, b) != 2) return 2; words[a] = unhex(b); }
    auto read = [&](const uint8_t* slot, uint8_t* out) {
        std::string k;
        char t[3];
        for (int i = 0; i < 32; i++) { snprintf(t, 3, "%02x", slot[i]); k += t; }
        auto it = words.find(k);
        if (it == words.end()) memset(out, 0, 32); else memcpy(out, it->second.data(), 32);
    };
    unsigned long long np = 0;
    if (fscanf(in, "%llu", &np) != 1) return 2;
    for (unsigned long long i = 0; i < np; i++) {
        PathDev p;
        memset(&p, 0, sizeof p);
        unsigned long long actor;
        unsigned kind, n_words, n_steps;
        if (fscanf(in, "%llu %s %u %u %u", &actor, a, &kind, &n_words, &n_steps) != 5) return 2;
        p.actor_id = actor;
        std::vector<uint8_t> base = unhex(a);
        memcpy(p.base_slot, base.data(), 32);
        p.n_steps = n_steps; p.kind = kind; p.n_words = kind == IPCFP_PATH_WORDS ? n_words : 0;
        std::vector<PathStepDev> steps(n_steps + 1);
        std::vector<uint8_t> keys;
        uint32_t n_array = 0;
        for (unsigned j = 0; j < n_steps; j++) {
            unsigned op, klen, es, eb;
            unsigned long long index;
            if (fscanf(in, "%u %u %s %llu %u %u", &op, &klen, a, &index, &es, &eb) != 6) return 2;
            std::vector<uint8_t> key = unhex(a);
            PathStepDev& d = steps[j];
            memset(&d, 0, sizeof d);
            d.op = op; d.key_len = klen; d.key_off = keys.size(); d.index = index; d.elem_slots = es; d.elem_bytes = eb;
            keys.insert(keys.end(), key.begin(), key.end());
            n_array += op == IPCFP_PATH_ARRAY;
        }
        keys.resize(keys.size() + 16, 0);
        p.n_fixed = path_n_fixed(n_array, kind, n_words);
        // k_path_slots
        std::vector<ipcfp_storage_spec> fixed(p.n_fixed);
        uint8_t slot[32];
        uint32_t off;
        path_fixed_specs(p, steps.data(), keys.data(), fixed.data(), slot, off);
        // wave 1: the words storage holds under the fixed specs
        std::vector<ipcfp_storage_proof> proofs(p.n_fixed);
        std::vector<uint8_t> ok(p.n_fixed, 1);
        for (uint32_t k = 0; k < p.n_fixed; k++) { memset(&proofs[k], 0, sizeof proofs[k]); read(fixed[k].slot, proofs[k].value); }
        // k_path_expand
        const PathExpansion e = path_expand(p, steps.data(), proofs.data(), ok.data());
        // k_path_place_specs + wave 2
        std::vector<ipcfp_storage_spec> specs(fixed);
        if (e.n_data) {
            uint8_t bs[32];
            keccak_key_slot(nullptr, 0, slot, bs);
            for (uint32_t j = 0; j < e.n_data; j++) {
                ipcfp_storage_spec sp;
                sp.actor_id = p.actor_id;
                path_data_slot(bs, j, sp.slot);
                specs.push_back(sp);
                ipcfp_storage_proof q;
                memset(&q, 0, sizeof q);
                read(sp.slot, q.value);
                proofs.push_back(q);
            }
        }
        // k_path_values
        std::vector<uint8_t> value(e.value_len + 1);
        path_value(p, proofs.data(), e.n_data, e.value_len, value.data());
        printf("%u ", e.status);
        hex(slot, 32);
        printf(" %u %zu", off, specs.size());
        for (auto& s : specs) { printf(" "); hex(s.slot, 32); }
        printf(" ");
        if (e.value_len) hex(value.data(), e.value_len); else printf("-");
        printf("\n");
    }
    fclose(in);
    return 0;
}
