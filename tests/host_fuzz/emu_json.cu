// emu_json.cu — the device JSON renderer of IPCFP_RESULT_JSON executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// The per-item functions of csrc/json_items.cuh (record lengths, the proof writer, the lane-split block writer, the framing), compiled for
// the host and driven as the kernels of csrc/json.cu drive them — lengths, exclusive scan, writers in any order, the lanes of one block in a
// shuffled order and in several lane counts — on random event results, against ipcfp_event_result_to_json (csrc/bundle_json.cpp, linked as
// the checker) of the same result with its skipped proof slots compacted away, as the engine's host does. Every buffer the device code
// reads has exactly the padding the engine gives it, and the output is an exact-size heap buffer, so that under AddressSanitizer any read
// or write outside them is a report.
//
//   nvcc -std=c++17 -O2 -o emu_json tests/host_fuzz/emu_json.cu ipc_filecoin_proofs_b200/csrc/bundle_json.cpp && ./emu_json 3000 7
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/json_items.cuh"

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

struct Coverage { uint64_t results = 0, proofs = 0, skipped = 0, skipped_first = 0, no_proofs = 0, no_blocks = 0, blocks = 0, len_mod3[3] = {}, parents[4] = {},
                  neg_epoch = 0, zero_epoch = 0, min_epoch = 0, topics[10] = {}, bytes = 0; };

// one random result; returns false on a difference (details on stderr)
static bool one_case(uint64_t id, Coverage& cov) {
    // ---- tipset constants: device copies padded as the engine's staging buffer (+ 64)
    JsonProofCtx c;
    const uint32_t P = (uint32_t)(rnd() % 4);
    std::vector<uint8_t> tip(38ull * (P + 1) + 64);
    fill(tip.data(), tip.size());
    c.n_parents = P; c.parent_cids = tip.data(); c.child_cid = tip.data() + 38ull * P;
    c.parent_epoch = pick_i64(); c.child_epoch = pick_i64();
    for (int64_t e : {c.parent_epoch, c.child_epoch}) { cov.neg_epoch += e < 0; cov.zero_epoch += e == 0; cov.min_epoch += e == INT64_MIN; }
    cov.parents[P]++;
    // ---- proof slots as pass 2 leaves them, topics / data in one blob (+ 16, as d_blob)
    const uint64_t np = rnd() % 5 == 0 ? 0 : rnd() % 12;
    std::vector<ipcfp_event_proof> slots(np + 1);
    std::vector<uint8_t> data;
    const bool skip_first = rnd() % 4 == 0;
    uint64_t kept = 0;
    for (uint64_t k = 0; k < np; k++) {
        ipcfp_event_proof& p = slots[k];
        memset(&p, 0, sizeof p);
        const bool skip = (k == 0 && skip_first) || rnd() % 5 == 0;
        p.exec_index = skip ? UINT64_MAX : pick_u64();
        if (!skip && p.exec_index == UINT64_MAX) p.exec_index = 0;
        p.event_index = pick_u64(); p.emitter = pick_u64();
        p.n_topics = (uint32_t)(rnd() % 10);
        p.data_len = (uint32_t)(rnd() % 201);
        p.topics_off = data.size();
        data.resize(data.size() + 32ull * p.n_topics);
        fill(data.data() + p.topics_off, 32ull * p.n_topics);
        p.data_off = data.size();
        data.resize(data.size() + p.data_len);
        fill(data.data() + p.data_off, p.data_len);
        fill(p.message_cid, IPCFP_CID_LEN);
        if (skip) { cov.skipped++; if (k == 0) cov.skipped_first++; } else { kept++; cov.topics[p.n_topics]++; }
    }
    cov.proofs += kept;
    cov.no_proofs += kept == 0;
    const uint64_t n_bytes = data.size();
    data.resize(n_bytes + 16);
    // ---- witness: sorted CID list (+ 64, as d_cids), blocks at any alignment in an arena with the store's lead / tail pads
    const uint64_t m = rnd() % 5 == 0 ? 0 : rnd() % 24;
    std::vector<uint8_t> cids(38 * m + 64);
    fill(cids.data(), cids.size());
    for (uint64_t i = 0; i < m; i++) if (rnd() % 2) { static const uint8_t pre[6] = {1, 0x71, 0xa0, 0xe4, 2, 0x20}; memcpy(cids.data() + 38 * i, pre, 6); }
    std::vector<uint32_t> lens(m + 1);
    std::vector<uint64_t> offs(m + 1);
    uint64_t blob_size = 0;
    for (uint64_t i = 0; i < m; i++) {
        lens[i] = (uint32_t)(rnd() % 4 == 0 ? rnd() % 4 : rnd() % 301);
        blob_size += rnd() % 7;
        offs[i] = blob_size;
        blob_size += lens[i];
        cov.len_mod3[lens[i] % 3]++;
    }
    cov.blocks += m;
    cov.no_blocks += m == 0;
    std::vector<uint8_t> arena(16 + blob_size + 16);
    fill(arena.data(), arena.size());
    const uint8_t* blob = arena.data() + 16;

    // ---- the checker: ipcfp_event_result_to_json of the compacted result
    std::vector<ipcfp_event_proof> compact;
    for (uint64_t k = 0; k < np; k++) if (json_proof_kept(slots[k])) compact.push_back(slots[k]);
    ipcfp_event_result r;
    memset(&r, 0, sizeof r);
    r.n_proofs = compact.size(); r.proofs = compact.data(); r.data_blob = data.data(); r.data_blob_size = n_bytes;
    r.witness.n_blocks = m; r.witness.cids = cids.data(); r.witness.offsets = offs.data(); r.witness.lengths = lens.data(); r.witness.blob = blob;
    r.witness.blob_size = blob_size;
    ipcfp_tipset_desc t;
    memset(&t, 0, sizeof t);
    t.parent_epoch = c.parent_epoch; t.child_epoch = c.child_epoch; t.n_parents = P; t.parent_cids = c.parent_cids; t.child_cid = c.child_cid;
    char* want = nullptr;
    uint64_t want_len = 0;
    if (ipcfp_event_result_to_json(&r, &t, &want, &want_len) != IPCFP_OK) { fprintf(stderr, "case %llu: host renderer refused\n", (unsigned long long)id); return false; }

    // ---- the device code, driven as csrc/json.cu drives it
    std::vector<uint32_t> plen(np + 1), blen(m + 1);
    for (uint64_t k = 0; k < np; k++) { uint64_t n = json_proof_len(c, slots[k], data.data()); if (n > 0xffffffffull) return false; plen[k] = (uint32_t)n; }
    for (uint64_t i = 0; i < m; i++) { uint64_t n = json_block_len(cids.data() + 38 * i, lens[i]); if (n > 0xffffffffull) return false; blen[i] = (uint32_t)n; }
    std::vector<uint64_t> poff(np + 1), boff(m + 1);
    uint64_t Pt = 0, Qt = 0;
    for (uint64_t k = 0; k < np; k++) { poff[k] = Pt; Pt += plen[k]; }
    for (uint64_t i = 0; i < m; i++) { boff[i] = Qt; Qt += blen[i]; }
    const uint64_t total = json_total_len(Pt, Qt);
    char* out = (char*)malloc(total ? total : 1);   // exact size: one byte outside is an ASan report
    memset(out, 0x01, total);                       // a byte no writer touches stays 0x01 and differs from the checker's text
    // kernels run in any order; so do their threads
    std::vector<uint64_t> order(np + m);
    for (uint64_t q = 0; q < np + m; q++) order[q] = q;
    for (uint64_t q = order.size(); q > 1; q--) std::swap(order[q - 1], order[rnd() % q]);
    json_frame_write(out, Pt, Qt);
    static const uint32_t LANES[] = {32, 32, 1, 3, 7, 64};
    for (uint64_t q : order) {
        if (q < np) {
            if (json_proof_kept(slots[q])) json_proof_write(out + JSON_PROOFS_HEAD + poff[q], poff[q] == 0, c, slots[q], data.data());
            continue;
        }
        const uint64_t i = q - np;
        const uint32_t nl = LANES[rnd() % (sizeof LANES / sizeof *LANES)];
        std::vector<uint32_t> lanes(nl);
        for (uint32_t l = 0; l < nl; l++) lanes[l] = l;
        for (uint32_t l = nl; l > 1; l--) std::swap(lanes[l - 1], lanes[rnd() % l]);
        // exact copies of the block's bytes: the writer must not read one byte beyond them
        std::vector<uint8_t> src(blob + offs[i], blob + offs[i] + lens[i]);
        for (uint32_t l : lanes) json_block_write(out + json_blocks_at(Pt) + boff[i], boff[i] == 0, cids.data() + 38 * i, src.data(), lens[i], l, nl);
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
    cov.results++;
    cov.bytes += total;
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
    bool covered = cov.skipped_first && cov.no_proofs && cov.no_blocks && cov.neg_epoch && cov.zero_epoch && cov.min_epoch;
    for (int k = 0; k < 3; k++) covered &= cov.len_mod3[k] > 0;
    for (int k = 0; k < 4; k++) covered &= cov.parents[k] > 0;
    for (int k = 0; k < 10; k++) covered &= cov.topics[k] > 0;
    if (!covered) { fprintf(stderr, "coverage incomplete: run more cases\n"); return 1; }
    printf("ok: device JSON renderer == ipcfp_event_result_to_json for %llu results: %llu proofs (%llu skipped slots, %llu of them first), %llu blocks, "
           "%llu bytes\n", (unsigned long long)cov.results, (unsigned long long)cov.proofs, (unsigned long long)cov.skipped,
           (unsigned long long)cov.skipped_first, (unsigned long long)cov.blocks, (unsigned long long)cov.bytes);
    return 0;
}
