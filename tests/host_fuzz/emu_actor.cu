// emu_actor.cu — the per-proof code of actor proofs (csrc/actor_items.cuh) and its planner and verifier items (plan_actor_path,
// verify_actor_item) executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed), driven as csrc/actor.cu, csrc/plan.cu and csrc/verify.cu
// drive them: the Init walk once per case when some address is not an ID address, then actor_proof_one per request, each through its own
// Recorder; then the planner item per request and, when the call succeeds, the verifier item on its proofs over the same store.
// tests/test_actor_host.py writes the cases (every tree of tests/actor_trees.py, dropped blocks, seeded truncations and bit flips) and
// compares the output with that module's restatement; under AddressSanitizer + UBSan it also shows the walks, the decoders and the
// Keccak-256 of the bytecode stay inside the padded block buffers.
//
//   emu_actor <case file>   per case: "fail <status> <index>" or, per proof, "proof <record hex> <bytecode hex or ->" and
//                           "list <cid hex>…"; then "plan <cid hex>…" (sorted, unique), "verify <0|1>…" (only when the call succeeds), "end"
// Case file: u64 n_blocks, n_blocks × {cid (38), u32 len, bytes}; u32 n_cases; per case: child (38), state root (38), u8 with_code,
// u8 strict, u32 n_evm, n_evm × cid (38), u32 n_addrs, n_addrs × {u8 len, bytes}, u32 n_drop, n_drop × u64 block index,
// u32 n_mut, n_mut × {u64 block index, u32 len, bytes}.
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

using namespace ipcfp;

static FILE* g_in;
static void rd(void* p, size_t n) {
    if (n && fread(p, 1, n, g_in) != n) { fprintf(stderr, "emu_actor: truncated case file\n"); exit(2); }
}
template <class T> static T rd1() { T v; rd(&v, sizeof v); return v; }
static std::string hex(const uint8_t* p, size_t n) {
    static const char* D = "0123456789abcdef";
    std::string s;
    for (size_t i = 0; i < n; i++) { s.push_back(D[p[i] >> 4]); s.push_back(D[p[i] & 15]); }
    return s;
}

// the engine's store over blocks of several CID classes (the bytecode blocks are raw-codec CIDs), laid out as ipcfp_store_create lays
// it out: arena with lead / tail padding, one BlockRec per block, open-addressing index by (class, digest), equal CIDs keep the first
struct ClassStore {
    std::vector<uint8_t> arena;
    std::vector<BlockRec> recs;
    std::vector<uint64_t> table;
    StoreView view;
    ClassStore(const uint8_t* cids, const uint64_t* offs, const uint32_t* lens, const uint8_t* blob, uint64_t blob_size, uint64_t n) {
        arena.assign(16 + blob_size + 32, 0);
        if (blob_size) memcpy(arena.data() + 16, blob, blob_size);
        recs.resize(n);
        memset(&view, 0, sizeof view);
        uint64_t slots = 64;
        while (slots < 2 * n) slots <<= 1;
        table.assign(slots, 0);
        for (uint64_t i = 0; i < n; i++) {
            const uint8_t* c = cids + 38 * i;
            uint32_t cls = 0;
            while (cls < view.n_classes && memcmp(view.class_prefix[cls], c, 6)) cls++;
            if (cls == view.n_classes) {
                if (cls == IPCFP_MAX_CID_CLASSES) { fprintf(stderr, "emu_actor: too many CID classes\n"); exit(2); }
                memcpy(view.class_prefix[cls], c, 6);
                view.n_classes++;
            }
            BlockRec r;
            memset(&r, 0, sizeof r);
            memcpy(r.d.w, c + 6, 32);
            r.off = offs[i]; r.len = lens[i]; r.cls = cls;
            recs[i] = r;
            const uint64_t h = digest_hash(r.d, cls);
            const uint32_t fp = (uint32_t)(h >> 32) | 1u;
            for (uint64_t slot = h & (slots - 1);; slot = (slot + 1) & (slots - 1)) {
                const uint64_t e = table[slot];
                if (e == 0) { table[slot] = ((uint64_t)fp << 32) | (i + 1); break; }
                const BlockRec& q = recs[(uint32_t)e - 1];
                if ((uint32_t)(e >> 32) == fp && digest_eq(q.d, r.d) && q.cls == cls) break;
            }
        }
        view.blob = arena.data() + 16;
        view.recs = recs.data();
        view.table = table.data();
        view.mask = slots - 1;
        view.n = (uint32_t)n;
    }
};

static int status_of(uint32_t code) {
    switch (code) {
        case DC_MISSING: return IPCFP_ERR_MISSING_BLOCK;
        case DC_STATE_MISMATCH: return IPCFP_ERR_STATE_ROOT_MISMATCH;
        case DC_ACTOR_NOT_FOUND: return IPCFP_ERR_ACTOR_NOT_FOUND;
        case DC_UNSUPPORTED: return IPCFP_ERR_UNSUPPORTED;
        default: return IPCFP_ERR_DECODE;
    }
}

int main(int argc, char** argv) {
    if (argc != 2 || !(g_in = fopen(argv[1], "rb"))) { fprintf(stderr, "usage: emu_actor <case file>\n"); return 2; }
    const uint64_t nb = rd1<uint64_t>();
    std::vector<std::vector<uint8_t>> cids(nb, std::vector<uint8_t>(38)), data(nb);
    for (uint64_t i = 0; i < nb; i++) {
        rd(cids[i].data(), 38);
        data[i].resize(rd1<uint32_t>());
        rd(data[i].data(), data[i].size());
    }
    const uint32_t nc = rd1<uint32_t>();
    for (uint32_t k = 0; k < nc; k++) {
        // the call's upload as csrc/actor.cu lays it out: child CID at 0, state root at 64, EVM code CIDs at 128, then the addresses
        std::vector<uint8_t> up(128);
        rd(up.data(), 38);
        rd(up.data() + 64, 38);
        const bool wc = rd1<uint8_t>() != 0, strict = rd1<uint8_t>() != 0;
        const uint32_t n_evm = rd1<uint32_t>();
        up.resize(128 + 38 * n_evm + 16);
        rd(up.data() + 128, 38 * n_evm);
        std::vector<ipcfp_address> addrs(rd1<uint32_t>());
        for (auto& a : addrs) { memset(&a, 0, sizeof a); a.len = rd1<uint8_t>(); rd(a.bytes, a.len); }
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
        ClassStore hs(c.data(), offs.data(), lens.data(), blob.data(), blob.size(), n);
        const uint64_t m = addrs.size();
        ActorArgs a{};
        a.store = hs.view;
        a.child_cid = up.data();
        a.state_root_json = up.data() + 64;
        a.evm_codes = up.data() + 128;
        a.n_evm = n_evm;
        a.addrs = addrs.data();
        a.n = m;
        a.with_code = wc;
        a.strict_only = strict;
        std::vector<uint32_t> wbits((n + 31) / 32 + 8, 0), init_list(REC_CAP), lists(std::max<uint64_t>(m, 1) * REC_CAP);
        // the Init walk (k_actor_init)
        bool any_other = false;
        for (const auto& ad : addrs) any_other |= ad.bytes[0] != 0;
        Fail init_fail{0, 0};
        const uint8_t* map = nullptr;
        uint32_t n_init = 0;
        if (any_other) {
            Recorder rec{init_list.data(), 0, wbits.data(), false};
            rec.strict_only = strict;
            if (!resolve_init(hs.view, rec, a.state_root_json, map, init_fail)) map = nullptr;
            else if (rec.overflow) { map = nullptr; init_fail = Fail{DC_UNSUPPORTED, 2}; }
            n_init = rec.n;
        }
        // the proofs (k_actor_proofs); the first failing proof decides
        std::vector<ipcfp_actor_proof> out(std::max<uint64_t>(m, 1));
        std::vector<std::string> lines;
        bool failed = false;
        for (uint64_t t = 0; t < m && !failed; t++) {
            Recorder rec{lists.data() + t * REC_CAP, 0, wbits.data(), false};
            rec.strict_only = strict;
            ipcfp_actor_proof& q = out[t];
            memset(&q, 0, sizeof q);
            Fail f{0, 0};
            uint64_t cb;
            if (!actor_proof_one(a, addrs[t], map, init_fail, rec, q, cb, f)) {
                printf("fail %d %llu\n", status_of(f.code), (unsigned long long)t);
                failed = true;
                break;
            }
            if (rec.overflow) { printf("fail %d %llu\n", IPCFP_ERR_UNSUPPORTED, (unsigned long long)t); failed = true; break; }
            std::string code = "-";
            if (cb != UINT64_MAX) {
                uint32_t cl;
                const uint8_t* cp = store_block(hs.view, (uint32_t)cb, cl);
                code = hex(cp, cl);
            }
            std::string line = "proof " + hex((const uint8_t*)&q, sizeof q) + " " + code + "\nlist";
            std::set<uint32_t> own(rec.list, rec.list + rec.n);
            if (addrs[t].bytes[0] != 0) own.insert(init_list.begin(), init_list.begin() + n_init);
            for (uint32_t b : own) line += " " + hex(c.data() + 38 * b, 38);
            lines.push_back(line);
        }
        if (!failed) for (const std::string& l : lines) printf("%s\n", l.c_str());
        // the planner item (k_plan_actors)
        std::set<std::string> plan;
        std::vector<uint32_t> needed((n + 31) / 32 + 8, 0);
        for (uint64_t t = 0; t < m; t++) {
            const uint8_t* miss = plan_actor_path(a, t, needed.data());
            if (miss) plan.insert(hex(miss, 38));
        }
        std::string pl = "plan";
        for (const std::string& x : plan) pl += " " + x;
        printf("%s\n", pl.c_str());
        // the verifier item (k_verify_actors) on the generated proofs, over the same store
        if (!failed && m) {
            VerifyActorArgs v{};
            v.g = a;
            v.proofs = out.data();
            v.n = m;
            std::vector<uint8_t> res(m, 0);
            unsigned long long err = IPCFP_NO_ERROR;
            v.results = res.data();
            v.err = &err;
            for (uint64_t t = 0; t < m; t++) verify_actor_item(v, t);
            std::string vl = err == IPCFP_NO_ERROR ? "verify" : "verify-error";
            for (uint8_t r : res) vl += r ? " 1" : " 0";
            printf("%s\n", vl.c_str());
        }
        printf("end\n");
    }
    return 0;
}
