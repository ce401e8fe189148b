// emu_log_bundle.cu — the check_event of ipcfp_verify_event_proofs_any (verify_check(const LogFilterAny*), the last step of
// verify_event_item<LogFilterAny>, csrc/verify_items.cuh) EXECUTED ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// Per case: a random set of 1–5 filters (0–4 positions, wildcards, value and emitter sets of 1–70, so both sides of LF_INLINE, and
// duplicates) laid out by the library's own host builder (LogFilterSet: one word array, every filter placed at its own large sets, here
// in host memory), and 64 events drawn from small pools of emitters and topics so that filters hit: Case B with 0–4 topics, Case A with
// 0–6 topics, void logs, at random offsets of one buffer. For every event the predicate's verdict is printed with the case, one JSON
// object per line, and tests/test_log_bundle_host.py checks it against the Python predicate (api.LogFilter.matches, OR over the set).
//
//   nvcc -std=c++17 -O2 -o emu_log_bundle tests/host_fuzz/emu_log_bundle.cu oracle/oracle.cpp -lpthread && ./emu_log_bundle [cases] [seed]
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/hashes.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/walk.cuh"
#ifndef __CUDA_ARCH__
#define prefetch_l2(p) ((void)0)   // inline PTX: nothing to do on the host
#endif
#include "../../ipc_filecoin_proofs_b200/csrc/verify_items.cuh"

using namespace ipcfp;

static uint64_t rs;
static uint64_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return rs; }

static std::string hex(const uint8_t* p, size_t n) {
    static const char* H = "0123456789abcdef";
    std::string s;
    for (size_t i = 0; i < n; i++) { s.push_back(H[p[i] >> 4]); s.push_back(H[p[i] & 15]); }
    return s;
}

int main(int argc, char** argv) {
    const int cases = argc > 1 ? atoi(argv[1]) : 200;
    rs = argc > 2 ? strtoull(argv[2], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1 : 88172645463325252ull;
    uint8_t pool[8][32];
    for (auto& t : pool) for (auto& b : t) b = (uint8_t)rnd();
    const uint64_t emit_pool[6] = {1001, 1002, 1003, 77, 1ull << 40, 0};
    uint64_t hits = 0, total = 0;
    for (int c = 0; c < cases; c++) {
        const uint32_t nf = (uint32_t)(1 + rnd() % 5);   // the calls take an empty set as no check_event: never this predicate
        std::vector<ipcfp_log_filter> in(nf);
        std::vector<std::vector<uint8_t>> vals;
        std::vector<std::vector<uint64_t>> ems;
        vals.reserve(4 * nf);
        ems.reserve(nf);
        for (uint32_t k = 0; k < nf; k++) {
            ipcfp_log_filter& f = in[k];
            memset(&f, 0, sizeof f);
            if (k && rnd() % 5 == 0) { f = in[k - 1]; continue; }   // a duplicate filter
            f.n_positions = (uint32_t)(rnd() % 5);
            ems.emplace_back();
            const uint32_t ne = rnd() % 3 == 0 ? (uint32_t)(1 + rnd() % (rnd() % 2 ? 4 : 70)) : 0;
            for (uint32_t j = 0; j < ne; j++) ems.back().push_back(j < 3 ? emit_pool[rnd() % 6] : rnd());
            f.n_emitters = ne;
            f.emitters = ne ? ems.back().data() : nullptr;
            for (uint32_t q = 0; q < f.n_positions; q++) {
                if (rnd() % 3 == 0) continue;   // a wildcard
                const uint32_t n = (uint32_t)(1 + rnd() % (rnd() % 2 ? 4 : 70));
                vals.emplace_back(32ull * n);
                for (uint32_t j = 0; j < n; j++) {
                    uint8_t* v = vals.back().data() + 32ull * j;
                    if (j < 2) memcpy(v, pool[rnd() % 8], 32);
                    else for (int b = 0; b < 32; b++) v[b] = (uint8_t)rnd();
                }
                f.n_values[q] = n;
                f.values[q] = vals.back().data();
            }
        }
        LogFilterSet fs;
        fs.build(in.data(), nf);
        std::vector<uint64_t> dev(fs.words.size() + 1);
        fs.place(dev.data());
        std::copy(fs.words.begin(), fs.words.end(), dev.begin());
        const LogFilterAny any{(const LogFilter*)dev.data(), nf};
        std::string line = "{\"filters\":[";
        for (uint32_t k = 0; k < nf; k++) {
            const ipcfp_log_filter& f = in[k];
            line += k ? ",{\"emitters\":[" : "{\"emitters\":[";
            for (uint64_t j = 0; j < f.n_emitters; j++) line += (j ? "," : "") + std::to_string(f.emitters[j]);
            line += "],\"topics\":[";
            for (uint32_t q = 0; q < f.n_positions; q++) {
                line += q ? "," : "";
                if (!f.n_values[q]) { line += "null"; continue; }
                line += "[";
                for (uint64_t j = 0; j < f.n_values[q]; j++) line += (j ? ",\"" : "\"") + hex(f.values[q] + 32 * j, 32) + "\"";
                line += "]";
            }
            line += "]}";
        }
        line += "],\"events\":[";
        for (int e = 0; e < 64; e++) {
            EvLog ev;
            memset(&ev, 0, sizeof ev);
            ev.emitter = emit_pool[rnd() % 6];
            ev.some = rnd() % 8 ? 1u : 0u;
            ev.case_a = (uint32_t)(rnd() & 1);
            ev.ntopics = (uint32_t)(rnd() % (ev.case_a ? 7 : 5));
            const uint32_t skew = (uint32_t)(rnd() % 13);
            std::vector<uint8_t> blk(skew + 32 * 8 + 64 + 16, 0xAB);
            uint8_t tp[6][32];
            for (uint32_t k = 0; k < ev.ntopics; k++) {
                if (rnd() % 4) memcpy(tp[k], pool[rnd() % 8], 32);
                else for (int b = 0; b < 32; b++) tp[k][b] = (uint8_t)rnd();
            }
            if (ev.case_a) {
                ev.toff[0] = skew + 3;
                for (uint32_t k = 0; k < ev.ntopics; k++) memcpy(blk.data() + ev.toff[0] + 32 * k, tp[k], 32);
            } else {
                for (uint32_t k = 0; k < ev.ntopics; k++) {   // Case B: the values apart, in any order
                    ev.toff[k] = skew + 40 * ((k + 1) % 4) + 1;
                    memcpy(blk.data() + ev.toff[k], tp[k], 32);
                }
            }
            const bool got = verify_check(&any, blk.data(), ev);
            hits += got;
            total++;
            line += e ? ",{" : "{";
            line += "\"emitter\":" + std::to_string(ev.emitter) + ",\"some\":" + std::to_string(ev.some) + ",\"topics\":[";
            for (uint32_t k = 0; k < ev.ntopics; k++) line += (k ? ",\"" : "\"") + hex(tp[k], 32) + "\"";
            line += "],\"got\":" + std::string(got ? "1" : "0") + "}";
        }
        line += "]}";
        printf("%s\n", line.c_str());
    }
    printf("ok: %llu events, %llu matches\n", (unsigned long long)total, (unsigned long long)hits);
    return 0;
}
