// emu_json_parse.cu — the device bundle parser of ipcfp_verify_bundle_json executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// The per-item functions of csrc/json_parse_items.cuh, compiled for the host and driven as csrc/json_parse.cu drives them — record starts,
// the per-record template checks (records in a shuffled order, the base64 characters of a block in a shuffled lane order), the scans,
// the framing and shared tipset fields, the PODs, the blocks decoded group by group in any order — against ipcfp_bundle_from_json
// (csrc/bundle_parse.cpp, linked as the checker):
//   * random canonical EventProofBundle / UnifiedProofBundle texts rendered by csrc/bundle_json.cpp (edge values as emu_json.cu): the
//     device items must accept every one and give the host parser's PODs field by field;
//   * byte mutations of such texts: each must either be refused by the device items (the call then defers to the host parser) or give
//     exactly the host parser's values; an accept where the host parser refuses is a failure.
// The text the device items read is an exact-size heap buffer followed by JP_PAD zero bytes, as on the device; the framing and tipset
// items, which the host runs on the caller's buffer, read an exact-size copy without padding. Under AddressSanitizer any read outside is a
// report.
//
//   nvcc -std=c++17 -O2 -o emu_json_parse tests/host_fuzz/emu_json_parse.cu ipc_filecoin_proofs_b200/csrc/bundle_json.cpp \
//        ipc_filecoin_proofs_b200/csrc/bundle_parse.cpp && ./emu_json_parse 2000 60000 7
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/json_parse_items.cuh"

using namespace ipcfp;

static uint64_t rs;
static uint64_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return rs; }

static uint64_t pick_u64() {
    static const uint64_t SPECIAL[] = {0, 9, 10, 99, 100, 999, 1000, UINT64_MAX, UINT64_MAX - 1, 10000000000000000000ull};
    switch (rnd() % 4) {
        case 0: return SPECIAL[rnd() % (sizeof SPECIAL / sizeof *SPECIAL)];
        case 1: return rnd() % 1000;
        case 2: return rnd() >> (rnd() % 64);
        default: return rnd();
    }
}
static int64_t pick_i64() {
    static const int64_t SPECIAL[] = {INT64_MIN, INT64_MIN + 1, -1, 0, 1, -10, 9, INT64_MAX};
    switch (rnd() % 3) {
        case 0: return SPECIAL[rnd() % (sizeof SPECIAL / sizeof *SPECIAL)];
        case 1: return (int64_t)(rnd() % 20000000) - 10000000;
        default: return (int64_t)rnd();
    }
}
static void fill(uint8_t* p, uint64_t n) { for (uint64_t i = 0; i < n; i++) p[i] = (uint8_t)rnd(); }
static void fill_cid(uint8_t* c) {
    static const uint8_t pre[6] = {1, 0x71, 0xa0, 0xe4, 2, 0x20};
    fill(c, IPCFP_CID_LEN);
    if (rnd() % 2) memcpy(c, pre, 6);
}

// what the device path yields
struct DevOut {
    JpTipset ts;
    std::vector<uint8_t> parents;
    std::vector<ipcfp_storage_proof> sp;
    std::vector<ipcfp_event_proof> ep;
    std::vector<uint8_t> blob, cids, arena;
    std::vector<uint64_t> offs;
    std::vector<uint32_t> lens;
    uint64_t e_total = 0, b_total = 0, witness_bytes = 0;
};

// csrc/json_parse.cu's flow with the kernels replaced by loops; false = defer
static bool device_parse(const std::string& text, DevOut& o) {
    const uint64_t len = text.size();
    if (len < 2) return false;
    std::vector<char> padded(len + JP_PAD, 0);   // the device copy
    memcpy(padded.data(), text.data(), len);
    const char* t = padded.data();
    // k_jp_mark + bitmap_to_indices
    std::vector<uint32_t> pos;
    for (uint64_t p = 0; p < len; p++) if (t[p] == '{' && jp_kind_at(t, p) != JP_NONE) pos.push_back((uint32_t)p);
    const uint64_t n = pos.size(), cap = len / JP_MIN_RECORD + 1;
    if (n > cap) return false;
    // k_jp_records, in any order
    std::vector<uint64_t> order(n);
    for (uint64_t i = 0; i < n; i++) order[i] = i;
    for (uint64_t q = n; q > 1; q--) std::swap(order[q - 1], order[rnd() % q]);
    uint64_t first[3], last[3], first_start[3], last_end[3];
    for (int k = 0; k < 3; k++) first[k] = last[k] = first_start[k] = last_end[k] = UINT64_MAX;
    std::vector<uint32_t> elen(n + 1, 0), blen(n + 1, 0);
    for (uint64_t i : order) {
        JpRec r;
        if (!jp_record(t, len, pos.data(), n, i, r)) return false;
        if (r.kind == JP_BLOCK) {
            const uint32_t nl = (uint32_t)(1 + rnd() % 40);
            std::vector<uint32_t> lanes(nl);
            for (uint32_t l = 0; l < nl; l++) lanes[l] = l;
            for (uint32_t l = nl; l > 1; l--) std::swap(lanes[l - 1], lanes[rnd() % l]);
            for (uint32_t l : lanes)
                for (uint64_t k = l; k < r.blk.n_chars - r.blk.pads; k += nl) if (!jp_block_char_ok(t, r.blk, k)) return false;
            o.witness_bytes += r.len;
        }
        elen[i] = r.kind == JP_EVENT ? (uint32_t)r.blob_len : 0u;
        blen[i] = r.kind == JP_BLOCK ? (uint32_t)r.blob_len : 0u;
        if (r.first) { first[r.kind] = i; first_start[r.kind] = pos[i]; }
        if (r.last) { last[r.kind] = i; last_end[r.kind] = r.end; }
    }
    std::vector<uint64_t> eoff(n + 1), boff(n + 1);
    for (uint64_t i = 0; i < n; i++) { eoff[i] = o.e_total; o.e_total += elen[i]; boff[i] = o.b_total; o.b_total += blen[i]; }
    // host side of synchronisation 1, on the caller's (unpadded) text
    std::vector<char> exact(text.begin(), text.end());
    uint64_t cnt[3];
    for (int k = 0; k < 3; k++) cnt[k] = first[k] == UINT64_MAX ? 0 : last[k] - first[k] + 1;
    if (!jp_frame_ok(exact.data(), len, cnt, first_start, last_end)) return false;
    if (!jp_tipset(exact.data(), len, cnt, first_start, o.ts)) return false;
    o.parents.resize(38ull * o.ts.n_parents);
    for (uint32_t q = 0; q < o.ts.n_parents; q++) jp_cid_at(exact.data(), o.ts.parents_at + 65ull * q, o.parents.data() + 38ull * q);
    // k_jp_proofs
    const uint64_t nS = cnt[JP_STORAGE], nE = cnt[JP_EVENT], nB = cnt[JP_BLOCK];
    o.sp.resize(nS);
    o.ep.resize(nE);
    o.blob.assign(o.e_total + 16, 0);
    for (uint64_t i = 0; i < nS + nE; i++) {
        uint64_t end;
        if (i < nS) { JpStorage s; if (!jp_storage_proof(t, pos[i], len, s, end, &o.sp[i])) return false; continue; }
        JpEvent r;
        if (!jp_event_proof(t, pos[i], len, r, end)) return false;
        jp_event_write(t, r, eoff[i], o.ep[i - nS], o.blob.data());
    }
    // k_jp_blocks (groups in any order)
    o.cids.assign(38 * nB, 0);
    o.offs.assign(nB, 0);
    o.lens.assign(nB, 0);
    o.arena.assign(o.b_total + 16, 0);
    for (uint64_t j = 0; j < nB; j++) {
        const uint64_t i = first[JP_BLOCK] + j, end = i + 1 < n ? (uint64_t)pos[i + 1] - 1 : len - 2;
        JpBlock b;
        if (!jp_block_head(t, pos[i], end, b, o.cids.data() + 38 * j)) return false;
        o.offs[j] = boff[i];
        o.lens[j] = b.len;
        std::vector<uint8_t> out(b.len + 2, 0xee);   // exact copies: a group writes bytes below len only
        const uint64_t ng = b.n_chars / 4;
        std::vector<uint64_t> gs(ng);
        for (uint64_t g = 0; g < ng; g++) gs[g] = g;
        for (uint64_t g = ng; g > 1; g--) std::swap(gs[g - 1], gs[rnd() % g]);
        for (uint64_t g : gs) jp_block_group(t, b, g, out.data());
        if (out[b.len] != 0xee || out[b.len + 1] != 0xee) { fprintf(stderr, "block %llu: a group wrote past the block\n", (unsigned long long)j); exit(1); }
        memcpy(o.arena.data() + boff[i], out.data(), b.len);
    }
    return true;
}

struct Cov { uint64_t accepted = 0, event_bundles = 0, unified = 0, proofs = 0, sproofs = 0, blocks = 0, mutants = 0, mutants_accepted = 0,
             mutants_host_ok = 0, parents[4] = {}, topics[10] = {}, len_mod3[3] = {}, neg_epoch = 0, min_epoch = 0, empty = 0; };

// the device result equals the host parser's, field by field; when the host refuses, the device must have deferred
static bool same_as_host(const std::string& text, bool dev_ok, const DevOut& d, const char* what, uint64_t id) {
    ipcfp_parsed_bundle* pb = nullptr;
    const ipcfp_status st = ipcfp_bundle_from_json(text.data(), text.size(), &pb);
    if (!dev_ok) { if (pb) ipcfp_parsed_bundle_free(pb); return true; }
    auto fail = [&](const char* m) { fprintf(stderr, "%s %llu: device accepted, %s\n  text: %.300s\n", what, (unsigned long long)id, m, text.c_str()); if (pb) ipcfp_parsed_bundle_free(pb); return false; };
    if (st != IPCFP_OK) return fail("host parser refused");
    const ipcfp_parsed_bundle& h = *pb;
    const ipcfp_tipset_desc& t = h.tipset;
    if (t.parent_epoch != d.ts.parent_epoch || t.child_epoch != d.ts.child_epoch || t.n_parents != d.ts.n_parents) return fail("tipset epochs / parents differ");
    if (t.n_parents && memcmp(t.parent_cids, d.parents.data(), 38ull * t.n_parents)) return fail("parent CIDs differ");
    if (!t.n_parents && t.parent_cids) return fail("parent CIDs not null");
    if ((t.child_cid != nullptr) != d.ts.has_child || (t.child_cid && memcmp(t.child_cid, d.ts.child, 38))) return fail("child CID differs");
    if ((t.child_parent_state_root != nullptr) != d.ts.has_root || (d.ts.has_root && memcmp(t.child_parent_state_root, d.ts.root, 38))) return fail("state root differs");
    if (h.n_storage_proofs != d.sp.size() || (d.sp.size() && memcmp(h.storage_proofs, d.sp.data(), d.sp.size() * sizeof(ipcfp_storage_proof))))
        return fail("storage proofs differ");
    if (h.n_event_proofs != d.ep.size() || (d.ep.size() && memcmp(h.event_proofs, d.ep.data(), d.ep.size() * sizeof(ipcfp_event_proof))))
        return fail("event proofs differ");
    if (h.data_blob_size != d.e_total || (d.e_total && memcmp(h.data_blob, d.blob.data(), d.e_total))) return fail("data blob differs");
    const ipcfp_witness& w = h.witness;
    if (w.n_blocks != d.lens.size() || w.blob_size != d.b_total) return fail("block count / arena size differ");
    uint64_t wb = 0;
    for (uint64_t j = 0; j < w.n_blocks; j++) {
        if (memcmp(w.cids + 38 * j, d.cids.data() + 38 * j, 38) || w.offsets[j] != d.offs[j] || w.lengths[j] != d.lens[j]) return fail("block CID / offset / length differs");
        if (memcmp(w.blob + w.offsets[j], d.arena.data() + d.offs[j], w.lengths[j])) return fail("block bytes differ");
        wb += w.lengths[j];
    }
    if (wb != d.witness_bytes) return fail("witness bytes differ");
    ipcfp_parsed_bundle_free(pb);
    return true;
}

// ---- random canonical bundles through bundle_json.cpp
struct Gen {
    std::vector<uint8_t> tip, data, cids, blob;
    std::vector<ipcfp_event_proof> ep;
    std::vector<ipcfp_storage_proof> sp;
    std::vector<uint64_t> offs;
    std::vector<uint32_t> lens;
};
static std::string make_bundle(Gen& g, bool unified, Cov& cov) {
    const uint32_t P = (uint32_t)(rnd() % 4);
    g.tip.assign(38ull * (P + 2), 0);
    for (uint32_t k = 0; k < P + 2; k++) fill_cid(g.tip.data() + 38ull * k);
    ipcfp_tipset_desc t;
    memset(&t, 0, sizeof t);
    t.parent_epoch = pick_i64(); t.child_epoch = pick_i64(); t.n_parents = P;
    t.parent_cids = g.tip.data(); t.child_cid = g.tip.data() + 38ull * P; t.child_parent_state_root = g.tip.data() + 38ull * (P + 1);
    cov.neg_epoch += t.child_epoch < 0 || t.parent_epoch < 0;
    cov.min_epoch += t.child_epoch == INT64_MIN || t.parent_epoch == INT64_MIN;
    const uint64_t np = rnd() % 5 == 0 ? 0 : rnd() % 8;
    g.ep.assign(np, ipcfp_event_proof{});
    g.data.clear();
    for (uint64_t k = 0; k < np; k++) {
        ipcfp_event_proof& p = g.ep[k];
        memset(&p, 0, sizeof p);
        p.exec_index = pick_u64(); p.event_index = pick_u64(); p.emitter = pick_u64();
        p.n_topics = (uint32_t)(rnd() % 10);
        p.data_len = (uint32_t)(rnd() % 201);
        p.topics_off = g.data.size();
        g.data.resize(g.data.size() + 32ull * p.n_topics + p.data_len);
        fill(g.data.data() + p.topics_off, 32ull * p.n_topics + p.data_len);
        p.data_off = p.topics_off + 32ull * p.n_topics;
        fill_cid(p.message_cid);
        cov.topics[p.n_topics]++;
    }
    if (np) cov.parents[P]++;
    g.data.resize(g.data.size() + 16);
    const uint64_t ns = unified && rnd() % 4 ? rnd() % 5 : 0;
    g.sp.assign(ns, ipcfp_storage_proof{});
    for (uint64_t k = 0; k < ns; k++) {
        ipcfp_storage_proof& s = g.sp[k];
        memset(&s, 0, sizeof s);
        s.actor_id = pick_u64();
        fill_cid(s.actor_state_cid); fill_cid(s.storage_root); fill(s.slot, 32); fill(s.value, 32);
        s.found = 1; s.raw_len = 32;
    }
    const uint64_t m = rnd() % 5 == 0 ? 0 : rnd() % 12;
    g.cids.assign(38 * m + 38, 0);
    for (uint64_t i = 0; i < m; i++) fill_cid(g.cids.data() + 38 * i);
    g.offs.assign(m + 1, 0);
    g.lens.assign(m + 1, 0);
    g.blob.clear();
    for (uint64_t i = 0; i < m; i++) {
        g.lens[i] = (uint32_t)(rnd() % 4 == 0 ? rnd() % 4 : rnd() % 301);
        g.blob.resize(g.blob.size() + rnd() % 5);
        g.offs[i] = g.blob.size();
        g.blob.resize(g.blob.size() + g.lens[i]);
        fill(g.blob.data() + g.offs[i], g.lens[i]);
        cov.len_mod3[g.lens[i] % 3]++;
    }
    g.blob.resize(g.blob.size() + 16);
    ipcfp_witness w;
    memset(&w, 0, sizeof w);
    w.n_blocks = m; w.cids = g.cids.data(); w.offsets = g.offs.data(); w.lengths = g.lens.data(); w.blob = g.blob.data(); w.blob_size = g.blob.size() - 16;
    ipcfp_event_result r;
    memset(&r, 0, sizeof r);
    r.n_proofs = np; r.proofs = g.ep.data(); r.data_blob = g.data.data(); r.data_blob_size = g.data.size() - 16; r.witness = w;
    char* out = nullptr;
    uint64_t out_len = 0;
    ipcfp_status st;
    if (unified) {
        ipcfp_storage_result sr;
        memset(&sr, 0, sizeof sr);
        sr.n_proofs = ns; sr.proofs = g.sp.data();
        ipcfp_event_result* evs[1] = {&r};
        ipcfp_bundle b;
        memset(&b, 0, sizeof b);
        b.storage = ns || rnd() % 2 ? &sr : nullptr;
        b.n_event_results = 1; b.events = evs; b.witness = w;
        st = ipcfp_bundle_to_json(&b, &t, &out, &out_len);
        cov.unified++;
        cov.sproofs += ns;
    } else {
        st = ipcfp_event_result_to_json(&r, &t, &out, &out_len);
        cov.event_bundles++;
    }
    if (st != IPCFP_OK) { fprintf(stderr, "renderer refused\n"); exit(1); }
    std::string s(out, out_len);
    ipcfp_json_free(out);
    cov.proofs += np;
    cov.blocks += m;
    cov.empty += np == 0 && ns == 0 && m == 0;
    return s;
}

static std::string mutate(const std::string& s0) {
    static const char ALPHA[] = "0123456789abcdefxyzABCDEF\"',{}[]:- \n=\\/+.eE";
    std::string s = s0;
    const int k = 1 + (int)(rnd() % 3);
    for (int q = 0; q < k && !s.empty(); q++) {
        const uint64_t at = rnd() % s.size();
        const char c = rnd() % 8 == 0 ? (char)rnd() : ALPHA[rnd() % (sizeof ALPHA - 1)];
        switch (rnd() % 5) {
            case 0: case 1: s[at] = c; break;
            case 2: s.erase(at, 1 + rnd() % 3); break;
            case 3: s.insert(s.begin() + (long)at, c); break;
            default: {   // repeat or drop a span (whole records, separators)
                const uint64_t n = std::min<uint64_t>(1 + rnd() % 400, s.size() - at);
                if (rnd() % 2) s.insert(at, s.substr(at, n)); else s.erase(at, n);
            }
        }
    }
    return s;
}

int main(int argc, char** argv) {
    const uint64_t n_bundles = argc > 1 ? strtoull(argv[1], nullptr, 10) : 2000;
    const uint64_t n_mut = argc > 2 ? strtoull(argv[2], nullptr, 10) : 100000;
    rs = argc > 3 ? strtoull(argv[3], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1 : 88172645463325252ull;
    Cov cov;
    std::vector<std::string> seeds;
    Gen g;
    for (uint64_t id = 0; id < n_bundles; id++) {
        const std::string text = make_bundle(g, id % 2 == 1, cov);
        DevOut d;
        if (!device_parse(text, d)) { fprintf(stderr, "bundle %llu: canonical text refused by the device items\n  %.300s\n", (unsigned long long)id, text.c_str()); return 1; }
        if (!same_as_host(text, true, d, "bundle", id)) return 1;
        cov.accepted++;
        if (text.size() < 20000 && seeds.size() < 64) seeds.push_back(text);
    }
    for (uint64_t id = 0; id < n_mut && !seeds.empty(); id++) {
        const std::string text = mutate(seeds[rnd() % seeds.size()]);
        DevOut d;
        const bool ok = device_parse(text, d);
        ipcfp_parsed_bundle* pb = nullptr;
        if (ipcfp_bundle_from_json(text.data(), text.size(), &pb) == IPCFP_OK) { cov.mutants_host_ok++; ipcfp_parsed_bundle_free(pb); }
        if (!same_as_host(text, ok, d, "mutant", id)) return 1;
        cov.mutants++;
        cov.mutants_accepted += ok;
    }
    bool covered = cov.event_bundles && cov.unified && cov.sproofs && cov.neg_epoch && cov.min_epoch && cov.empty;
    for (int k = 0; k < 4; k++) covered &= cov.parents[k] > 0;
    for (int k = 0; k < 10; k++) covered &= cov.topics[k] > 0;
    for (int k = 0; k < 3; k++) covered &= cov.len_mod3[k] > 0;
    if (!covered) { fprintf(stderr, "coverage incomplete: run more bundles\n"); return 1; }
    printf("ok: device bundle parser == ipcfp_bundle_from_json on %llu canonical bundles (%llu event, %llu unified; %llu event proofs, %llu storage "
           "proofs, %llu blocks) and %llu mutants (%llu accepted by the device items, %llu by the host parser)\n",
           (unsigned long long)cov.accepted, (unsigned long long)cov.event_bundles, (unsigned long long)cov.unified, (unsigned long long)cov.proofs,
           (unsigned long long)cov.sproofs, (unsigned long long)cov.blocks, (unsigned long long)cov.mutants, (unsigned long long)cov.mutants_accepted,
           (unsigned long long)cov.mutants_host_ok);
    return 0;
}
