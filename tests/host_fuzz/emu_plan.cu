// emu_plan.cu — the fetch planner (csrc/plan.cu) executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// csrc/plan_items.cuh holds the planner's per-item device code: plan_class / plan_children (the whole-AMT walk of rules 1 and 2),
// plan_receipt_matches and plan_receipt_path (rule 3), plan_storage_path (rule 4). This program compiles them for the host and drives
// them as the kernels of plan.cu do — level by level, item by item, with the per-class visited bitmaps, the needed bitmap and the
// missing list — over a host copy of the store (host_store.h). The input file (written by tests/test_plan_fetch_host.py) holds one
// tipset, its specs, its complete block set and a list of cases; a case keeps a subset of the blocks and may replace some blocks' bytes
// under the same CID. Per case it prints
//   plan <n_needed> <missing CIDs, hex, in Cid order>     the plan against the kept blocks (compared with tests/plan_rules.py)
//   loop <rounds>                                         the planning loop from an empty store, fetching from the (edited) block set
// and checks on its own that the loop converges without requesting a CID twice and that the C++ oracle's generate_proof_bundle on the
// planned store gives what it gives on the whole block set: the same status and error index, or the same witness, block for block.
//
//   nvcc -std=c++17 -O2 -o emu_plan tests/host_fuzz/emu_plan.cu oracle/oracle.cpp -lpthread && ./emu_plan cases.bin
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/common.cuh"
#define prefetch_l2(p) ((void)0)   // inline PTX: nothing to do on the host
#include "../../ipc_filecoin_proofs_b200/csrc/plan_items.cuh"
#include "../../oracle/oracle.h"
#include "host_store.h"

using namespace ipcfp;

[[noreturn]] static void die(const char* what) { fprintf(stderr, "emu_plan: %s\n", what); exit(1); }

struct Reader {
    std::vector<uint8_t> b;
    size_t p = 0;
    const uint8_t* take(size_t n) { if (p + n > b.size()) die("truncated input"); const uint8_t* q = b.data() + p; p += n; return q; }
    template <class T> T get() { T v; memcpy(&v, take(sizeof v), sizeof v); return v; }
    std::string str() { uint32_t n = get<uint32_t>(); return std::string((const char*)take(n), n); }
};

// a buffer the device code may read CIDs from: 16 bytes before and 64 after are in bounds, as on the device
struct Padded {
    std::vector<uint8_t> v;
    explicit Padded(const uint8_t* src = nullptr, size_t n = 0) : v(16 + n + 64, 0) { if (n) memcpy(v.data() + 16, src, n); }
    const uint8_t* p() const { return v.data() + 16; }
};

struct Blocks {   // block i = cids[38i..], bytes[i]
    std::vector<uint8_t> cids;
    std::vector<std::string> bytes;
    size_t n() const { return bytes.size(); }
    void flat(std::vector<uint64_t>& offs, std::vector<uint32_t>& lens, std::vector<uint8_t>& blob) const {
        offs.clear(); lens.clear(); blob.clear();
        for (auto& s : bytes) { offs.push_back(blob.size()); lens.push_back((uint32_t)s.size()); blob.insert(blob.end(), s.begin(), s.end()); }
    }
};

struct Tip {
    uint32_t n_parents;
    Padded parents, txmeta, child, rroot, psr, roots;
    std::vector<uint8_t> has;
    uint64_t n_receipts;
    std::vector<std::string> sigs, topics;
    std::vector<ipcfp_event_spec> especs;
    std::vector<ipcfp_storage_spec> sspecs;
    ipcfp_tipset_desc desc() const {
        ipcfp_tipset_desc d;
        memset(&d, 0, sizeof d);
        d.n_parents = n_parents; d.parent_cids = parents.p(); d.parent_txmeta_cids = txmeta.p(); d.child_cid = child.p();
        d.receipts_root = rroot.p(); d.child_parent_state_root = psr.p(); d.n_receipts = n_receipts; d.events_roots = roots.p();
        d.has_events_root = has.data();
        return d;
    }
};

struct Plan { std::vector<std::string> missing; uint64_t n_needed; };

// plan.cu's plan_fetch, its kernels run item by item
static Plan plan(const Blocks& S, const Tip& t) {
    std::vector<uint64_t> offs;
    std::vector<uint32_t> lens;
    std::vector<uint8_t> blob;
    S.flat(offs, lens, blob);
    StoreView v;
    memset(&v, 0, sizeof v);
    std::unique_ptr<HostStore> hs;
    if (S.n()) { hs.reset(new HostStore(S.cids.data(), offs.data(), lens.data(), blob.data(), blob.size(), S.n())); v = hs->view; }
    const uint64_t nwords = (S.n() + 31) / 32 + 1;
    std::vector<uint32_t> needed(nwords, 0), visited(PLAN_CLASSES * nwords, 0);
    std::vector<std::string> miss;
    const bool ev = !t.especs.empty(), st = !t.sspecs.empty();
    std::vector<PlanItem> cur;
    if (ev) {
        for (uint32_t k = 0; k < t.n_parents; k++) cur.push_back(PlanItem{t.parents.p() + 38 * k, PK_BLOCK, 0});
        cur.push_back(PlanItem{t.child.p(), PK_BLOCK, 0});
        cur.push_back(PlanItem{t.rroot.p(), PK_BLOCK, 0});
        for (uint32_t k = 0; k < t.n_parents; k++) cur.push_back(PlanItem{t.txmeta.p() + 38 * k, PK_TXMETA, 3});
        for (uint64_t i = 0; i < t.n_receipts; i++)
            cur.push_back(t.has[i] ? PlanItem{t.roots.p() + 38 * i, PK_EV_ROOT, 1u << 8} : PlanItem{nullptr, PK_NONE, 0});
    }
    if (st) { cur.push_back(PlanItem{t.child.p(), PK_BLOCK, 0}); cur.push_back(PlanItem{t.psr.p(), PK_BLOCK, 0}); }
    bool ev_missing = false;
    while (!cur.empty()) {   // k_plan_count + k_plan_expand
        std::vector<PlanItem> nxt;
        for (const PlanItem& it : cur) {
            if (it.kind == PK_NONE) continue;
            const int32_t b = store_lookup(v, it.cid);
            if (b < 0) { miss.emplace_back((const char*)it.cid, 38); ev_missing |= (it.bw_tree >> 8) != 0; continue; }
            witness_mark(v, needed.data(), (uint32_t)b);
            if (it.kind == PK_BLOCK) continue;
            const uint32_t r = (uint32_t)b, m = 1u << (r & 31);
            uint32_t& w = visited[plan_class(it) * nwords + (r >> 5)];
            if (w & m) continue;
            w |= m;
            uint32_t len;
            const uint8_t* p = store_block(v, (uint32_t)b, len);
            const uint32_t c = plan_children(p, len, it, nullptr);
            const size_t at = nxt.size();
            nxt.resize(at + c);
            if (c) (void)plan_children(p, len, it, nxt.data() + at);
        }
        cur.swap(nxt);
    }
    if (ev && !ev_missing && t.n_receipts) {   // k_plan_matchers + k_plan_match
        std::vector<Matcher> m(t.especs.size());
        for (size_t k = 0; k < m.size(); k++) {
            memset(&m[k], 0, sizeof(Matcher));
            const std::string& t1 = t.topics[k];
            memcpy(m[k].t1, t1.data(), std::min<size_t>(t1.size(), 32));
            m[k].actor = t.especs[k].actor_id_filter;
            m[k].has_actor = t.especs[k].has_actor_id_filter;
            Padded sig((const uint8_t*)t.sigs[k].data(), t.sigs[k].size());
            Digest d;
            keccak256(sig.p(), (uint32_t)t.sigs[k].size(), d);
            for (int w = 0; w < 4; w++) m[k].t0[w] = d.w[w];
        }
        for (uint64_t i = 0; i < t.n_receipts; i++) {
            if (!t.has[i]) continue;
            const int32_t rb = store_lookup(v, t.roots.p() + 38 * i);
            if (rb < 0 || !plan_receipt_matches(&v, (uint32_t)rb, m.data(), m.size())) continue;
            const uint8_t* c = plan_receipt_path(v, t.rroot.p(), i, needed.data());
            if (c) miss.emplace_back((const char*)c, 38);
        }
    }
    if (st) {   // k_plan_storage
        StorageArgs a;
        memset(&a, 0, sizeof a);
        a.store = v; a.child_cid = t.child.p(); a.state_root_json = t.psr.p(); a.specs = t.sspecs.data(); a.n = t.sspecs.size();
        for (uint64_t k = 0; k < a.n; k++) {
            const uint8_t* c = plan_storage_path(a, k, needed.data());
            if (c) miss.emplace_back((const char*)c, 38);
        }
    }
    std::sort(miss.begin(), miss.end());   // one CID prefix: the bytes' order is `Cid` order
    miss.erase(std::unique(miss.begin(), miss.end()), miss.end());
    uint64_t nn = 0;
    for (uint32_t w : needed) nn += (uint64_t)__builtin_popcount(w);
    return Plan{miss, nn};
}

struct Outcome { int status; uint64_t index; std::vector<std::string> wit; };
static Outcome oracle_bundle(const Blocks& S, const Tip& t) {
    std::vector<uint64_t> offs;
    std::vector<uint32_t> lens;
    std::vector<uint8_t> blob;
    S.flat(offs, lens, blob);
    blob.resize(blob.size() + 16);
    oracle_store* os = oracle_store_create(S.cids.data(), offs.data(), lens.data(), blob.data(), S.n());
    ipcfp_tipset_desc d = t.desc();
    ipcfp_bundle* b = nullptr;
    Outcome o{(int)oracle_generate_proof_bundle(os, &d, t.sspecs.data(), t.sspecs.size(), t.especs.data(), t.especs.size(), &b), 0, {}};
    if (o.status != IPCFP_OK) o.index = oracle_last_error_index();
    else {
        for (uint64_t k = 0; k < b->witness.n_blocks; k++)
            o.wit.push_back(std::string((const char*)b->witness.cids + 38 * k, 38) +
                            std::string((const char*)b->witness.blob + b->witness.offsets[k], b->witness.lengths[k]));
        oracle_bundle_free(b);
    }
    oracle_store_destroy(os);
    return o;
}

static void hex(const std::string& s) { for (unsigned char c : s) printf("%02x", c); }

int main(int argc, char** argv) {
    if (argc < 2) die("usage: emu_plan <cases file>");
    Reader R;
    {
        FILE* f = fopen(argv[1], "rb");
        if (!f) die("cannot open the cases file");
        uint8_t buf[1 << 16];
        size_t n;
        while ((n = fread(buf, 1, sizeof buf, f)) > 0) R.b.insert(R.b.end(), buf, buf + n);
        fclose(f);
    }
    Blocks full;
    const uint64_t n = R.get<uint64_t>();
    for (uint64_t i = 0; i < n; i++) {
        const uint8_t* c = R.take(38);
        full.cids.insert(full.cids.end(), c, c + 38);
        full.bytes.push_back(R.str());
    }
    Tip t;
    t.n_parents = R.get<uint32_t>();
    t.parents = Padded(R.take(38 * t.n_parents), 38 * t.n_parents);
    t.txmeta = Padded(R.take(38 * t.n_parents), 38 * t.n_parents);
    t.child = Padded(R.take(38), 38);
    t.rroot = Padded(R.take(38), 38);
    t.psr = Padded(R.take(38), 38);
    t.n_receipts = R.get<uint64_t>();
    t.roots = Padded(R.take(38 * t.n_receipts), 38 * t.n_receipts);
    const uint8_t* h = R.take(t.n_receipts);
    t.has.assign(h, h + t.n_receipts);
    const uint32_t ne = R.get<uint32_t>();
    for (uint32_t k = 0; k < ne; k++) { t.sigs.push_back(R.str()); t.topics.push_back(R.str()); }
    for (uint32_t k = 0; k < ne; k++) {
        ipcfp_event_spec e;
        memset(&e, 0, sizeof e);
        e.event_signature = t.sigs[k].c_str(); e.topic_1 = t.topics[k].c_str();
        e.has_actor_id_filter = R.get<uint8_t>(); e.actor_id_filter = R.get<uint64_t>();
        t.especs.push_back(e);
    }
    const uint32_t ns = R.get<uint32_t>();
    for (uint32_t k = 0; k < ns; k++) {
        ipcfp_storage_spec s;
        s.actor_id = R.get<uint64_t>();
        memcpy(s.slot, R.take(32), 32);
        t.sspecs.push_back(s);
    }
    const uint32_t n_cases = R.get<uint32_t>();
    for (uint32_t q = 0; q < n_cases; q++) {
        const uint8_t* keep = R.take(n);
        Blocks src = full;
        const uint32_t n_mut = R.get<uint32_t>();
        for (uint32_t k = 0; k < n_mut; k++) { const uint64_t i = R.get<uint64_t>(); src.bytes.at(i) = R.str(); }
        Blocks S;
        for (uint64_t i = 0; i < n; i++)
            if (keep[i]) { S.cids.insert(S.cids.end(), &src.cids[38 * i], &src.cids[38 * i] + 38); S.bytes.push_back(src.bytes[i]); }
        Plan p = plan(S, t);
        printf("plan %llu ", (unsigned long long)p.n_needed);
        for (auto& c : p.missing) hex(c);
        printf("\n");
        // the loop from an empty store over the edited block set
        std::map<std::string, uint64_t> where;
        for (uint64_t i = 0; i < n; i++) where.emplace(std::string((const char*)&src.cids[38 * i], 38), i);
        Blocks held;
        std::map<std::string, int> asked;
        uint32_t rounds = 0;
        for (;; rounds++) {
            if (rounds > 2000) die("the loop does not converge");
            Plan r = plan(held, t);
            uint64_t got = 0;
            for (auto& c : r.missing) {
                auto w = where.find(c);
                if (w == where.end()) continue;   // a CID nobody holds (an edited link): the generator meets it as missing
                if (asked[c]++) die("a CID was requested twice");
                held.cids.insert(held.cids.end(), c.begin(), c.end());
                held.bytes.push_back(src.bytes[w->second]);
                got++;
            }
            if (!got) break;
        }
        const Outcome a = oracle_bundle(held, t), b = oracle_bundle(src, t);
        if (a.status != b.status || a.index != b.index || a.wit != b.wit) {
            fprintf(stderr, "case %u: planned store status %d index %llu (%zu witness blocks), whole block set %d index %llu (%zu)\n", q, a.status,
                    (unsigned long long)a.index, a.wit.size(), b.status, (unsigned long long)b.index, b.wit.size());
            die("the planned store does not give the whole block set's bundle");
        }
        printf("loop %u %d\n", rounds, a.status);
    }
    return 0;
}
