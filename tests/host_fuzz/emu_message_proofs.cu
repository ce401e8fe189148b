// emu_message_proofs.cu — the per-request code of message proofs (csrc/message_proof_items.cuh) and its planner and verifier items
// (plan_message_path, verify_message_item) executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed), driven as csrc/message_proof.cu,
// csrc/plan.cu and csrc/verify.cu drive them: message_proof_one per request over one witness bitmap, the first failing request deciding;
// then the planner item per request and, when the call succeeds, the verifier item on its proofs and data blob over the same store. The
// execution positions come from the case file (on the GPU they come from the execution order).
// tests/test_message_proofs_host.py writes the cases (the worlds of tests/message_receipts.py, dropped blocks, seeded truncations and bit
// flips) and compares the output with that module's restatement; under AddressSanitizer + UBSan it also shows the receipts-AMT walk and
// the message decoder stay inside the padded block buffers.
//
//   emu_message_proofs <case file>   per case: "fail <status> <index>" or, per proof, "proof <record hex> <return hex or -> <params hex
//                                    or ->" and "marked <cid hex>…" (the blocks the walks marked, in store order); then "plan <cid hex>…"
//                                    (sorted, unique), "verify <0|1>…" (only when the call succeeds) and "end"
// Case file: u64 n_blocks, n_blocks × {cid (38), u32 len, bytes}; u32 n_cases; per case: receipts root (38), u8 with_body, u32 n,
// n × {cid (38), u64 exec_index}, u32 n_drop, n_drop × u64 block index, u32 n_mut, n_mut × {u64 block index, u32 len, bytes}.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/plan_items.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/verify_items.cuh"
#include "host_store.h"

using namespace ipcfp;

static FILE* g_in;
static void rd(void* p, size_t n) {
    if (n && fread(p, 1, n, g_in) != n) { fprintf(stderr, "emu_message_proofs: truncated case file\n"); exit(2); }
}
template <class T> static T rd1() { T v; rd(&v, sizeof v); return v; }
static std::string hex(const uint8_t* p, size_t n) {
    static const char* D = "0123456789abcdef";
    std::string s;
    for (size_t i = 0; i < n; i++) { s.push_back(D[p[i] >> 4]); s.push_back(D[p[i] & 15]); }
    return s;
}

int main(int argc, char** argv) {
    if (argc != 2 || !(g_in = fopen(argv[1], "rb"))) { fprintf(stderr, "usage: emu_message_proofs <case file>\n"); return 2; }
    const uint64_t nb = rd1<uint64_t>();
    std::vector<std::vector<uint8_t>> cids(nb, std::vector<uint8_t>(38)), data(nb);
    for (uint64_t i = 0; i < nb; i++) {
        rd(cids[i].data(), 38);
        data[i].resize(rd1<uint32_t>());
        rd(data[i].data(), data[i].size());
    }
    const uint32_t nc = rd1<uint32_t>();
    for (uint32_t k = 0; k < nc; k++) {
        uint8_t root[38];
        rd(root, 38);
        const bool with_body = rd1<uint8_t>() != 0;
        const uint32_t m = rd1<uint32_t>();
        // the requests as csrc/message_proof.cu uploads them (n*38, padded), the positions beside them
        std::vector<uint8_t> req(64 + 38 * (size_t)m + 64, 0);
        std::vector<uint64_t> pos(m + 1);
        for (uint32_t t = 0; t < m; t++) { rd(req.data() + 64 + 38 * t, 38); pos[t] = rd1<uint64_t>(); }
        std::set<uint64_t> drop;
        for (uint32_t n = rd1<uint32_t>(); n--;) drop.insert(rd1<uint64_t>());
        std::vector<std::vector<uint8_t>> blk = data;
        for (uint32_t n = rd1<uint32_t>(); n--;) { const uint64_t i = rd1<uint64_t>(); blk[i].resize(rd1<uint32_t>()); rd(blk[i].data(), blk[i].size()); }
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
        // the receipts root is k_setup's: a missing or undecodable root fails the call before any request (not modelled here)
        const int32_t rb = store_lookup_host_cid(hs.view, root);
        if (rb < 0) { fprintf(stderr, "emu_message_proofs: the receipts root must be in the store\n"); return 2; }
        std::vector<uint32_t> wbits((n + 31) / 32 + 8, 0);
        MsgProofArgs a{};
        a.store = hs.view;
        a.cids = req.data() + 64;
        a.exec_indices = pos.data();
        a.n = m;
        a.receipts_root_blk = (uint32_t)rb;
        a.with_body = with_body ? 1 : 0;
        a.wbits = wbits.data();
        std::vector<std::string> lines;
        std::vector<ipcfp_message_proof> out(std::max<uint32_t>(m, 1));
        std::vector<uint8_t> data;   // the data blob as csrc/message_proof.cu lays it out
        bool failed = false;
        for (uint64_t t = 0; t < m; t++) {
            ipcfp_message_proof& q = out[t];
            memset(&q, 0, sizeof q);
            const uint8_t *ret, *par;
            Fail f{0, 0};
            if (!message_proof_one(a, t, q, ret, par, f)) {
                printf("fail %d %llu\n", f.code == DC_MISSING ? IPCFP_ERR_MISSING_BLOCK : IPCFP_ERR_DECODE, (unsigned long long)t);
                failed = true;
                break;
            }
            if (ret) { q.return_off = q.return_len ? data.size() : 0; data.insert(data.end(), ret, ret + q.return_len); }
            if (par) { q.params_off = q.params_len ? data.size() : 0; data.insert(data.end(), par, par + q.params_len); }
            lines.push_back("proof " + hex((const uint8_t*)&q, sizeof q) + " " + (ret ? hex(ret, q.return_len) + "-" : std::string("-")) + " " +
                            (par ? hex(par, q.params_len) + "-" : std::string("-")));
        }
        if (!failed) {
            for (const std::string& l : lines) printf("%s\n", l.c_str());
            std::string mk = "marked";
            for (uint64_t b = 0; b < n; b++) if (wbits[b >> 5] >> (b & 31) & 1) mk += " " + hex(c.data() + 38 * b, 38);
            printf("%s\n", mk.c_str());
        }
        // the planner item (k_plan_messages)
        std::set<std::string> plan;
        std::vector<uint32_t> needed((n + 31) / 32 + 8, 0);
        std::vector<uint8_t> root_pad(128, 0);
        memcpy(root_pad.data() + 64, root, 38);
        for (uint64_t t = 0; t < m; t++) {
            const uint8_t* miss[2];
            const uint32_t km = plan_message_path(a, root_pad.data() + 64, t, needed.data(), miss);
            for (uint32_t i = 0; i < km; i++) plan.insert(hex(miss[i], 38));
        }
        std::string pl = "plan";
        for (const std::string& x : plan) pl += " " + x;
        printf("%s\n", pl.c_str());
        // the verifier item (k_verify_messages) on the generated proofs and blob, over the same store
        if (!failed && m) {
            VerifyMessageArgs v{};
            v.g = a;
            v.g.wbits = nullptr;
            unsigned long long err = IPCFP_NO_ERROR;
            v.g.err = &err;
            const uint32_t consistent = 1;
            data.resize(data.size() + 16, 0);
            v.proofs = out.data(); v.blob = data.data(); v.blob_size = data.size() - 16; v.consistent = &consistent;
            std::vector<uint8_t> res(m, 0);
            v.results = res.data();
            for (uint64_t t = 0; t < m; t++) verify_message_item(v, t);
            std::string vl = err == IPCFP_NO_ERROR ? "verify" : "verify-error";
            for (uint8_t r : res) vl += r ? " 1" : " 0";
            printf("%s\n", vl.c_str());
        }
        printf("end\n");
    }
    return 0;
}
