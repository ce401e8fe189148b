// emu_json_unified.cu — the device renderer of the UnifiedProofBundle text (ipcfp_generate_proof_bundle_resident with IPCFP_RESULT_JSON)
// executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// The StorageProof record (json_storage_len / json_storage_write), the EventProof and ProofBlock records and the unified framing of
// csrc/json_items.cuh, compiled for the host and driven as render_unified_json (csrc/json.cu) drives them — lengths, exclusive scans,
// writers in any order, the lanes of one block in a shuffled order — on random bundles, against ipcfp_bundle_to_json (csrc/bundle_json.cpp,
// compiled into this harness as the checker). Event proofs come from several results, concatenated with their topics / data offsets
// rebased into one data blob, as the engine uploads them. Every buffer the device code reads is exactly as large as the engine's, and the
// output is an exact-size heap buffer, so that under AddressSanitizer any read or write outside them is a report.
//
//   nvcc -std=c++17 -O2 -o emu_json_unified tests/host_fuzz/emu_json_unified.cu oracle/oracle.cpp -lpthread && ./emu_json_unified 3000 7
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/json_items.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/bundle_json.cpp"

using namespace ipcfp;

static uint64_t rs;
static uint64_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return rs; }

static uint64_t pick_u64() {
    static const uint64_t SPECIAL[] = {0, 9, 10, 99, 100, 1000, 1001, UINT64_MAX, UINT64_MAX - 1, 10000000000000000000ull};
    switch (rnd() % 4) {
        case 0: return SPECIAL[rnd() % (sizeof SPECIAL / sizeof *SPECIAL)];
        case 1: return rnd() % 2000;
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
static uint64_t pick_count() {   // 0, 1 or many
    switch (rnd() % 3) {
        case 0: return 0;
        case 1: return 1;
        default: return 2 + rnd() % 14;
    }
}

struct Coverage { uint64_t bundles = 0, storage = 0, events = 0, blocks = 0, bytes = 0, n_storage[3] = {}, n_events[3] = {}, n_blocks[3] = {},
                  actor0 = 0, actor_max = 0, epoch_min = 0, epoch_max = 0, results0 = 0, all_empty = 0; };
static int bucket(uint64_t n) { return n == 0 ? 0 : n == 1 ? 1 : 2; }

static void fill_cid(uint8_t* c) {
    fill(c, IPCFP_CID_LEN);
    if (rnd() % 2) { static const uint8_t pre[6] = {1, 0x71, 0xa0, 0xe4, 2, 0x20}; memcpy(c, pre, 6); }
}

static bool one_case(uint64_t id, Coverage& cov) {
    // ---- tipset constants: device copies (child CID, state root, parent CIDs), one staging area as the engine uploads them
    const uint32_t NP = (uint32_t)(rnd() % 4);
    std::vector<uint8_t> tip(38ull * (2 + NP));
    for (uint32_t k = 0; k < 2 + NP; k++) fill_cid(tip.data() + 38ull * k);
    const uint8_t* child = tip.data();
    const uint8_t* state_root = tip.data() + 38;
    const uint8_t* parents = tip.data() + 76;
    const int64_t pe = pick_i64(), ce = pick_i64();
    cov.epoch_min += ce == INT64_MIN;
    cov.epoch_max += ce == INT64_MAX;

    // ---- storage proofs
    const uint64_t ns = pick_count();
    std::vector<ipcfp_storage_proof> sp(ns + 1);
    for (uint64_t i = 0; i < ns; i++) {
        ipcfp_storage_proof& p = sp[i];
        memset(&p, 0, sizeof p);
        p.actor_id = rnd() % 5 == 0 ? (rnd() % 2 ? 0 : UINT64_MAX) : pick_u64();
        cov.actor0 += p.actor_id == 0;
        cov.actor_max += p.actor_id == UINT64_MAX;
        fill_cid(p.actor_state_cid);
        fill_cid(p.storage_root);
        fill(p.slot, 32);
        fill(p.value, 32);
        p.found = (uint8_t)(rnd() % 2);
        p.raw_len = 32;
    }
    // ---- event results (0..3 of them, some without proofs), each with its own data blob
    const uint64_t nr = rnd() % 4;
    cov.results0 += nr == 0;
    std::vector<std::vector<ipcfp_event_proof>> rp(nr);
    std::vector<std::vector<uint8_t>> rblob(nr);
    std::vector<ipcfp_event_result> rr(nr);
    std::vector<ipcfp_event_result*> rptr(nr);
    uint64_t ne = 0;
    for (uint64_t k = 0; k < nr; k++) {
        const uint64_t n = pick_count();
        rp[k].resize(n + 1);
        for (uint64_t q = 0; q < n; q++) {
            ipcfp_event_proof& p = rp[k][q];
            memset(&p, 0, sizeof p);
            p.exec_index = pick_u64();
            if (p.exec_index == UINT64_MAX) p.exec_index = 0;   // UINT64_MAX marks a skipped slot, which the host compacts away
            p.event_index = pick_u64(); p.emitter = pick_u64();
            p.n_topics = (uint32_t)(rnd() % 6);
            p.data_len = (uint32_t)(rnd() % 120);
            p.topics_off = rblob[k].size();
            rblob[k].resize(rblob[k].size() + 32ull * p.n_topics);
            fill(rblob[k].data() + p.topics_off, 32ull * p.n_topics);
            p.data_off = rblob[k].size();
            rblob[k].resize(rblob[k].size() + p.data_len);
            fill(rblob[k].data() + p.data_off, p.data_len);
            fill_cid(p.message_cid);
        }
        memset(&rr[k], 0, sizeof rr[k]);
        rr[k].n_proofs = n; rr[k].proofs = rp[k].data(); rr[k].data_blob = rblob[k].data(); rr[k].data_blob_size = rblob[k].size();
        rptr[k] = &rr[k];
        ne += n;
    }
    // ---- the union witness: sorted CID list (+ 64, as cids_dev), blocks at any alignment in an arena with the store's pads
    const uint64_t m = pick_count() * (rnd() % 3 + 1);
    std::vector<uint8_t> cids(38 * m + 64);
    for (uint64_t i = 0; i < m; i++) fill_cid(cids.data() + 38 * i);
    std::vector<uint32_t> lens(m + 1);
    std::vector<uint64_t> offs(m + 1);
    uint64_t blob_size = 0;
    for (uint64_t i = 0; i < m; i++) {
        lens[i] = (uint32_t)(rnd() % 4 == 0 ? rnd() % 4 : rnd() % 301);
        blob_size += rnd() % 7;
        offs[i] = blob_size;
        blob_size += lens[i];
    }
    std::vector<uint8_t> arena(16 + blob_size + 16);
    fill(arena.data(), arena.size());
    const uint8_t* blob = arena.data() + 16;
    cov.n_storage[bucket(ns)]++; cov.n_events[bucket(ne)]++; cov.n_blocks[bucket(m)]++;
    cov.all_empty += ns == 0 && ne == 0 && m == 0;

    // ---- the checker: ipcfp_bundle_to_json of the bundle
    ipcfp_storage_result sr;
    memset(&sr, 0, sizeof sr);
    sr.n_proofs = ns; sr.proofs = sp.data();
    ipcfp_bundle b;
    memset(&b, 0, sizeof b);
    b.storage = ns || rnd() % 2 ? &sr : nullptr;   // no storage result and one without proofs render alike
    b.n_event_results = nr; b.events = rptr.data();
    b.witness.n_blocks = m; b.witness.cids = cids.data(); b.witness.offsets = offs.data(); b.witness.lengths = lens.data(); b.witness.blob = blob;
    b.witness.blob_size = blob_size;
    ipcfp_tipset_desc t;
    memset(&t, 0, sizeof t);
    t.parent_epoch = pe; t.child_epoch = ce; t.n_parents = NP; t.parent_cids = parents; t.child_cid = child; t.child_parent_state_root = state_root;
    char* want = nullptr;
    uint64_t want_len = 0;
    if (ipcfp_bundle_to_json(&b, &t, &want, &want_len) != IPCFP_OK) { fprintf(stderr, "case %llu: host renderer refused\n", (unsigned long long)id); return false; }

    // ---- the engine's upload: storage proofs, event proofs concatenated with rebased offsets, one data blob (exact sizes)
    std::vector<ipcfp_storage_proof> d_sp(sp.begin(), sp.begin() + ns);
    std::vector<ipcfp_event_proof> d_ep;
    std::vector<uint8_t> d_blob;
    for (uint64_t k = 0; k < nr; k++) {
        for (uint64_t q = 0; q < rr[k].n_proofs; q++) {
            ipcfp_event_proof p = rp[k][q];
            p.data_off += d_blob.size();
            p.topics_off += d_blob.size();
            d_ep.push_back(p);
        }
        d_blob.insert(d_blob.end(), rblob[k].begin(), rblob[k].end());
    }
    d_blob.resize(d_blob.size() + 16);
    JsonStorageCtx sc{ce, child, state_root};
    JsonProofCtx c{pe, ce, NP, parents, child};

    // ---- the device code, driven as render_unified_json drives it
    std::vector<uint32_t> slen(ns + 1), plen(ne + 1), blen(m + 1);
    for (uint64_t i = 0; i < ns; i++) { uint64_t n = json_storage_len(sc, d_sp[i]); if (n > 0xffffffffull) return false; slen[i] = (uint32_t)n; }
    for (uint64_t k = 0; k < ne; k++) { uint64_t n = json_proof_len(c, d_ep[k], d_blob.data()); if (n > 0xffffffffull) return false; plen[k] = (uint32_t)n; }
    for (uint64_t i = 0; i < m; i++) { uint64_t n = json_block_len(cids.data() + 38 * i, lens[i]); if (n > 0xffffffffull) return false; blen[i] = (uint32_t)n; }
    std::vector<uint64_t> soff(ns + 1), poff(ne + 1), boff(m + 1);
    uint64_t S = 0, P = 0, Q = 0;
    for (uint64_t i = 0; i < ns; i++) { soff[i] = S; S += slen[i]; }
    for (uint64_t k = 0; k < ne; k++) { poff[k] = P; P += plen[k]; }
    for (uint64_t i = 0; i < m; i++) { boff[i] = Q; Q += blen[i]; }
    const uint64_t total = json_u_total_len(S, P, Q);
    char* out = (char*)malloc(total);   // exact size: one byte outside is an ASan report
    memset(out, 0x01, total);           // a byte no writer touches stays 0x01 and differs from the checker's text
    std::vector<uint64_t> order(ns + ne + m);
    for (uint64_t q = 0; q < order.size(); q++) order[q] = q;
    for (uint64_t q = order.size(); q > 1; q--) std::swap(order[q - 1], order[rnd() % q]);
    json_u_frame_write(out, S, P, Q);
    static const uint32_t LANES[] = {32, 32, 1, 3, 7, 64};
    for (uint64_t q : order) {
        if (q < ns) { json_storage_write(out + JSON_STORAGE_HEAD + soff[q], soff[q] == 0, sc, d_sp[q]); continue; }
        if (q < ns + ne) { const uint64_t k = q - ns; json_proof_write(out + json_u_events_at(S) + poff[k], poff[k] == 0, c, d_ep[k], d_blob.data()); continue; }
        const uint64_t i = q - ns - ne;
        const uint32_t nl = LANES[rnd() % (sizeof LANES / sizeof *LANES)];
        std::vector<uint32_t> lanes(nl);
        for (uint32_t l = 0; l < nl; l++) lanes[l] = l;
        for (uint32_t l = nl; l > 1; l--) std::swap(lanes[l - 1], lanes[rnd() % l]);
        std::vector<uint8_t> src(blob + offs[i], blob + offs[i] + lens[i]);   // exact copy: no byte beyond the block may be read
        for (uint32_t l : lanes) json_block_write(out + json_u_blocks_at(S, P) + boff[i], boff[i] == 0, cids.data() + 38 * i, src.data(), lens[i], l, nl);
    }
    bool ok = total == want_len && memcmp(out, want, total) == 0;
    if (!ok) {
        uint64_t d = 0;
        while (d < total && d < want_len && out[d] == want[d]) d++;
        fprintf(stderr, "case %llu: %llu bytes vs %llu from the host renderer, first difference at %llu\n  device: %.80s\n  host:   %.80s\n",
                (unsigned long long)id, (unsigned long long)total, (unsigned long long)want_len, (unsigned long long)d,
                std::string(out + (d > 20 ? d - 20 : 0), std::min<uint64_t>(total - (d > 20 ? d - 20 : 0), 80)).c_str(),
                std::string(want + (d > 20 ? d - 20 : 0), std::min<uint64_t>(want_len - (d > 20 ? d - 20 : 0), 80)).c_str());
    }
    cov.bundles++;
    cov.storage += ns; cov.events += ne; cov.blocks += m; cov.bytes += total;
    free(out);
    ipcfp_json_free(want);
    return ok;
}

int main(int argc, char** argv) {
    const uint64_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 3000;
    rs = argc > 2 ? strtoull(argv[2], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1 : 88172645463325252ull;
    Coverage cov;
    for (uint64_t id = 0; id < n; id++) if (!one_case(id, cov)) return 1;
    // the cases the renderer has to get right must all have occurred
    bool covered = cov.actor0 && cov.actor_max && cov.epoch_min && cov.epoch_max && cov.results0 && cov.all_empty;
    for (int k = 0; k < 3; k++) covered &= cov.n_storage[k] > 0 && cov.n_events[k] > 0 && cov.n_blocks[k] > 0;
    if (!covered) { fprintf(stderr, "coverage incomplete: run more cases\n"); return 1; }
    printf("ok: device UnifiedProofBundle renderer == ipcfp_bundle_to_json for %llu bundles: %llu storage proofs, %llu event proofs, %llu blocks, "
           "%llu bytes\n", (unsigned long long)cov.bundles, (unsigned long long)cov.storage, (unsigned long long)cov.events,
           (unsigned long long)cov.blocks, (unsigned long long)cov.bytes);
    return 0;
}
