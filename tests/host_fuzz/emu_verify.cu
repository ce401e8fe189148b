// emu_verify.cu — the GPU-batched verifiers' per-item device code executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// csrc/verify_items.cuh compiled for the host and driven the way verify.cu drives the kernels:
//   verify_tipset_item   once        header consistency, the parents' `messages` links, the receipts root      (events/verifier.rs:147-181)
//   verify_txmeta_item   per parent  TxMeta recompute                                                          (events/utils.rs:64-73)
//   execution order                  the oracle's raw message list + first-seen dedup stand in for the engine's own walk + dedup kernels
//                                    (those are emulated by emu_events / emu_walk)
//   verify_event_item    per proof   exec[exec_index] == message_cid, receipts / events AMT gets, event data, check_event (:184-290)
//   verify_storage_item  per proof   header → state root → actors HAMT → EVM state → storage slot                (storage/verifier.rs:98-170)
// against oracle_verify_event_proofs / oracle_verify_storage_proofs on bundles the oracle generated — intact, with forged claims
// (every proof field), with a witness block replaced by a mutated copy under its CID, with a witness block missing: the same
// Vec<bool>, or the same status at the same proof index. A verifier is the component that meets hostile input; under
// AddressSanitizer (IPCFP_HOST_FUZZ_SANITIZE) this is also the memory-safety check of its decoders on such input.
//
//   nvcc -std=c++17 -O2 -o emu_verify tests/host_fuzz/emu_verify.cu oracle/oracle.cpp synth/synth.cpp -lpthread && ./emu_verify [cases] [mutations] [seed]
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/hashes.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/walk.cuh"
#ifndef __CUDA_ARCH__
#define prefetch_l2(p) ((void)0)   // inline PTX: nothing to do on the host
#endif
#include "../../ipc_filecoin_proofs_b200/csrc/verify_items.cuh"
#include "../../oracle/oracle.h"
#include "../../synth/synth.h"
#include "host_store.h"

using namespace ipcfp;

static uint64_t rs;
static uint64_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return rs; }

struct Blocks {   // a mutable copy of a witness: flat block arrays
    std::vector<uint8_t> cids, blob;
    std::vector<uint64_t> offs;
    std::vector<uint32_t> lens;
    uint64_t n = 0;
    void from(const ipcfp_witness& w) {
        n = w.n_blocks;
        cids.assign(w.cids, w.cids + 38 * n);
        offs.clear(); lens.assign(w.lengths, w.lengths + n);
        blob.clear();
        for (uint64_t i = 0; i < n; i++) { offs.push_back(blob.size()); blob.insert(blob.end(), w.blob + w.offsets[i], w.blob + w.offsets[i] + w.lengths[i]); }
    }
    ipcfp_witness c() const { ipcfp_witness w; w.n_blocks = n; w.cids = cids.data(); w.offsets = offs.data(); w.lengths = lens.data(); w.blob = blob.data(); w.blob_size = blob.size(); return w; }
    void drop(uint64_t i) {
        cids.erase(cids.begin() + 38 * (long)i, cids.begin() + 38 * (long)(i + 1));
        offs.erase(offs.begin() + (long)i); lens.erase(lens.begin() + (long)i); n--;   // the bytes stay in the blob, unreferenced
    }
    void mutate(uint64_t i) {   // block i keeps its CID and length class, some of its bytes change (or it is truncated / extended)
        std::vector<uint8_t> b(blob.begin() + (long)offs[i], blob.begin() + (long)(offs[i] + lens[i]));
        const unsigned kind = (unsigned)(rnd() % 6);
        if (b.empty() || kind == 0) b.push_back((uint8_t)rnd());
        else if (kind == 1) b.resize(rnd() % b.size());
        else { const unsigned k = 1 + (unsigned)(rnd() % 3); for (unsigned q = 0; q < k; q++) { size_t p = (size_t)(rnd() % b.size()); if (rnd() % 2) b[p] = (uint8_t)rnd(); else b[p] ^= (uint8_t)(1u << (rnd() % 8)); } }
        offs[i] = blob.size(); lens[i] = (uint32_t)b.size();
        blob.insert(blob.end(), b.begin(), b.end());
    }
};

struct Verdict { int status = IPCFP_OK; uint64_t index = UINT64_MAX; std::vector<uint8_t> results; };

static void fail_key(Verdict& v, uint64_t key) {   // csrc/verify.cu throw_verify_error
    const uint32_t code = (uint32_t)(key >> 8) & 0xff;
    v.index = (key >> 16) & 0xFFFFFFFFFFull;
    switch (code) {
        case DC_MISSING: v.status = IPCFP_ERR_MISSING_BLOCK; break;
        case DC_CID_MISMATCH: v.status = IPCFP_ERR_CID_MISMATCH; break;
        case DC_ACTOR_NOT_FOUND: v.status = IPCFP_ERR_ACTOR_NOT_FOUND; break;
        case DC_UNSUPPORTED: v.status = IPCFP_ERR_UNSUPPORTED; break;
        default: v.status = IPCFP_ERR_DECODE; break;
    }
}

// ------------------------------------------------------------------------------------------ event proofs: verify.cu's verify_event_proofs, item by item
static Verdict engine_events(const Blocks& W, const ipcfp_tipset_desc& td, const std::vector<ipcfp_event_proof>& proofs, const std::vector<uint8_t>& blob,
                             const Matcher* filter) {
    Verdict v;
    const uint64_t n = proofs.size();
    v.results.assign(n, 0);
    if (n == 0) return v;   // verify_event_proofs returns before any device work (a bundle without proofs has nothing to verify, events/verifier.rs:60-72)
    HostStore hs(W.cids.data(), W.offs.data(), W.lens.data(), W.blob.data(), W.blob.size(), W.n);
    const uint32_t P = td.n_parents;
    // the device copies: child CID, parent CIDs, room for the TxMeta CIDs — padded as AsyncBuf d_cids is (38*(2P+2) + 64)
    std::vector<uint8_t> d_cids(38ull * (2 * P + 2) + 64, 0);
    memcpy(d_cids.data(), td.child_cid, 38);
    if (P) memcpy(d_cids.data() + 38, td.parent_cids, 38ull * P);
    uint8_t* d_tx = d_cids.data() + 38ull * (P + 1);
    uint32_t flags[2] = {0, 0};
    unsigned long long err = IPCFP_NO_ERROR;
    VerifyTipsetArgs ta;
    memset(&ta, 0, sizeof ta);
    ta.store = hs.view; ta.parent_cids = d_cids.data() + 38; ta.child_cid = d_cids.data(); ta.n_parents = P;
    ta.parent_epoch = td.parent_epoch; ta.child_epoch = td.child_epoch;
    ta.consistent = &flags[0]; ta.receipts_root_blk = &flags[1]; ta.txmeta_cids = d_tx; ta.err = &err;
    verify_tipset_item(ta);
    if (err != IPCFP_NO_ERROR) { fail_key(v, err); return v; }
    std::vector<RawCid> exec_raw;
    std::vector<uint32_t> exec_idx;
    if (flags[0]) {
        unsigned long long txerr = IPCFP_NO_ERROR;
        for (uint32_t k = 0; k < P; k++) verify_txmeta_item(hs.view, d_tx, k, &txerr);
        // the execution order: every BLS / SECP message AMT of every parent, first occurrence wins (events/utils.rs:48-94). The engine
        // runs its own walk + dedup kernels here (emulated elsewhere); a failure of that walk fails the call at proof 0. Its fault key
        // names the parent it met, which is the first parent whose prefix of the parent list fails to walk. verify.cu ranks a TxMeta
        // mismatch at that parent or an earlier one first (the reference checks parent k's TxMeta before it walks parent k's AMTs).
        ipcfp_tipset_desc t2 = td;
        t2.parent_txmeta_cids = d_tx;
        oracle_store* os = oracle_store_create(W.cids.data(), W.offs.data(), W.lens.data(), W.blob.data(), W.n);
        std::vector<uint8_t> raw(38ull * 400000);
        uint64_t nraw = 0;
        ipcfp_status st = oracle_message_list(os, &t2, raw.data(), raw.size() / 38, &nraw);
        uint32_t walk_parent = P;
        if (st != IPCFP_OK) {
            for (uint32_t k = 1; k <= P && walk_parent == P; k++) {
                t2.n_parents = k;
                uint64_t nk = 0;
                if (oracle_message_list(os, &t2, raw.data(), raw.size() / 38, &nk) != IPCFP_OK) walk_parent = k - 1;
            }
            t2.n_parents = P;
        }
        oracle_store_destroy(os);
        if (txerr != IPCFP_NO_ERROR && (st == IPCFP_OK || (uint32_t)(txerr & 0xff) <= walk_parent)) { fail_key(v, txerr); return v; }
        if (st != IPCFP_OK) { v.status = st; v.index = 0; return v; }
        std::unordered_map<std::string, uint32_t> seen;
        exec_raw.resize(nraw);
        for (uint64_t k = 0; k < nraw; k++) {
            const uint8_t* c = raw.data() + 38 * k;
            RawCid rc;
            memcpy(rc.w, c + 6, 32);
            rc.w[4] = 0;
            memcpy(&rc.w[4], c, 6);
            exec_raw[k] = rc;
            if (seen.emplace(std::string((const char*)c, 38), (uint32_t)k).second) exec_idx.push_back((uint32_t)k);
        }
    }
    std::vector<uint8_t> d_blob(blob.begin(), blob.end());
    d_blob.resize(blob.size() + 16, 0);   // AsyncBuf d_blob(blob_size + 16)
    err = IPCFP_NO_ERROR;
    VerifyEventArgs va;
    memset(&va, 0, sizeof va);
    va.store = hs.view; va.proofs = proofs.data(); va.n = n; va.blob = d_blob.data(); va.blob_size = blob.size();
    va.consistent = &flags[0]; va.receipts_root_blk = &flags[1];
    va.exec_raw = exec_raw.data(); va.exec_idx = exec_idx.data(); va.n_exec = exec_idx.size();
    va.filter = filter; va.results = v.results.data(); va.err = &err;
    for (uint64_t t = 0; t < n; t++) verify_event_item(va, t);
    if (err != IPCFP_NO_ERROR) fail_key(v, err);
    return v;
}

// The restated verifiers walk the proofs in order, clear results[i] when they start proof i and stop at the first Err (the reference's
// `?`): with the array pre-set to 2, the proof that failed is the last one that is no longer 2. (Errors raised inside the AMT / HAMT
// helpers carry no index of their own.)
static uint64_t failing_proof(const std::vector<uint8_t>& results) {
    uint64_t i = 0;
    while (i < results.size() && results[i] != 2) i++;
    return i ? i - 1 : 0;
}
static Verdict oracle_events(const Blocks& W, const ipcfp_tipset_desc& td, const std::vector<ipcfp_event_proof>& proofs, const std::vector<uint8_t>& blob,
                             const ipcfp_event_spec* filter) {
    Verdict v;
    v.results.assign(proofs.size(), 2);
    ipcfp_witness w = W.c();
    std::vector<uint8_t> b(blob);
    b.resize(blob.size() + 16, 0);
    v.status = oracle_verify_event_proofs(&w, &td, proofs.data(), proofs.size(), b.data(), filter, v.results.data());
    if (v.status != IPCFP_OK) v.index = failing_proof(v.results);
    return v;
}

static int compare(const char* what, const Verdict& e, const Verdict& o, uint64_t* n_ok, uint64_t* n_err) {
    if (o.status != IPCFP_OK || e.status != IPCFP_OK) {
        const bool same = e.status == o.status && e.index == o.index;
        if (!same) { fprintf(stderr, "EMU MISMATCH (%s): engine status %d index %llu vs oracle status %d index %llu\n", what, e.status, (unsigned long long)e.index, o.status, (unsigned long long)o.index); return 1; }
        (*n_err)++;
        return 0;
    }
    if (e.results != o.results) {
        for (size_t i = 0; i < e.results.size(); i++) if (e.results[i] != o.results[i]) { fprintf(stderr, "EMU MISMATCH (%s): proof %zu engine %u vs oracle %u\n", what, i, e.results[i], o.results[i]); break; }
        return 1;
    }
    (*n_ok)++;
    return 0;
}

// ------------------------------------------------------------------------------------------ storage proofs
static Verdict engine_storage(const Blocks& W, const ipcfp_tipset_desc& td, const std::vector<ipcfp_storage_proof>& proofs) {
    Verdict v;
    v.results.assign(proofs.size(), 0);
    HostStore hs(W.cids.data(), W.offs.data(), W.lens.data(), W.blob.data(), W.blob.size(), W.n);
    std::vector<uint8_t> d_in(128, 0);   // AsyncBuf d_in(128): child CID at 0, the claimed parent state root at 64
    memcpy(d_in.data(), td.child_cid, 38);
    memcpy(d_in.data() + 64, td.child_parent_state_root, 38);
    unsigned long long err = IPCFP_NO_ERROR;
    VerifyStorageArgs a;
    memset(&a, 0, sizeof a);
    a.store = hs.view; a.child_cid = d_in.data(); a.state_root_json = d_in.data() + 64; a.proofs = proofs.data(); a.n = proofs.size(); a.results = v.results.data(); a.err = &err;
    for (uint64_t t = 0; t < proofs.size(); t++) verify_storage_item(a, t);
    if (err != IPCFP_NO_ERROR) fail_key(v, err);
    return v;
}
static Verdict oracle_storage(const Blocks& W, const ipcfp_tipset_desc& td, const std::vector<ipcfp_storage_proof>& proofs) {
    Verdict v;
    v.results.assign(proofs.size(), 2);
    ipcfp_witness w = W.c();
    v.status = oracle_verify_storage_proofs(&w, &td, proofs.data(), proofs.size(), v.results.data());
    if (v.status != IPCFP_OK) v.index = failing_proof(v.results);
    return v;
}

static ipcfp_tipset_desc desc_of(synth_tipset* ts) {
    ipcfp_tipset_desc td;
    memset(&td, 0, sizeof td);
    td.parent_epoch = synth_parent_epoch(ts); td.child_epoch = synth_child_epoch(ts); td.n_parents = synth_n_parents(ts);
    td.parent_cids = synth_parent_cids(ts); td.parent_txmeta_cids = synth_parent_txmeta_cids(ts); td.child_cid = synth_child_cid(ts);
    td.receipts_root = synth_receipts_root(ts); td.child_parent_state_root = synth_parent_state_root(ts); td.n_receipts = synth_n_receipts(ts);
    td.events_roots = synth_events_roots(ts); td.has_events_root = synth_has_events_root(ts);
    return td;
}

int main(int argc, char** argv) {
    uint64_t cases = argc > 1 ? strtoull(argv[1], nullptr, 10) : 8;
    uint64_t muts = argc > 2 ? strtoull(argv[2], nullptr, 10) : 80;
    rs = argc > 3 ? strtoull(argv[3], nullptr, 10) : 0x7E21F7ull;
    uint64_t ev_ok = 0, ev_err = 0, st_ok = 0, st_err = 0, accepted = 0, rejected = 0;
    for (uint64_t c = 0; c < cases; c++) {
        // ---------------- an event bundle from the oracle
        synth_params sp;
        synth_default_params(&sp);
        sp.seed = 9000 + c * 13 + (rs & 0xff);
        static const uint64_t sizes[] = {1, 9, 64, 65, 300, 1500};
        sp.n_receipts = sizes[rnd() % 6];
        static const uint32_t evs[] = {1, 3, 8, 40, 300};
        sp.events_per_receipt = evs[rnd() % 5];
        if (sp.n_receipts * sp.events_per_receipt > 30000) sp.events_per_receipt = 8;
        sp.match_ppm = 20000u << (rnd() % 6);
        if (sp.match_ppm > 1000000) sp.match_ppm = 1000000;
        sp.has_actor_filter = (uint32_t)(rnd() % 2);
        sp.bw3_permille = (uint32_t)(rnd() % 1001);
        sp.case_a_permille = rnd() % 2 ? (uint32_t)(rnd() % 500) : 0;
        sp.null_root_permille = rnd() % 2 ? (uint32_t)(rnd() % 300) : 0;
        sp.n_parents = 1 + (uint32_t)(rnd() % 3);
        sp.dup_msgs = (uint32_t)(rnd() % 4);
        sp.with_state_tree = 0;
        sp.threads = 1;
        synth_tipset* ts = synth_build(&sp);
        ipcfp_tipset_desc td = desc_of(ts);
        oracle_store* os = oracle_store_create(synth_cids(ts), synth_offsets(ts), synth_lengths(ts), synth_blob(ts), synth_n_blocks(ts));
        ipcfp_event_spec spec;
        memset(&spec, 0, sizeof spec);
        spec.event_signature = synth_event_signature(ts); spec.topic_1 = synth_topic1(ts);
        spec.has_actor_id_filter = sp.has_actor_filter ? 1 : 0; spec.actor_id_filter = synth_target_actor(ts);
        ipcfp_event_result* r = nullptr;
        if (oracle_generate_event_proof(os, &td, &spec, 0, 1, &r) != IPCFP_OK) { fprintf(stderr, "oracle_generate_event_proof failed\n"); return 2; }
        Blocks W0;
        W0.from(r->witness);
        std::vector<ipcfp_event_proof> P0(r->proofs, r->proofs + r->n_proofs);
        std::vector<uint8_t> B0(r->data_blob, r->data_blob + r->data_blob_size);
        oracle_event_result_free(r);
        oracle_store_destroy(os);
        // the filter as verify.cu builds the Matcher (keccak on the device code), and a foreign one
        Matcher m_same, m_other;
        memset(&m_same, 0, sizeof m_same);
        {
            std::vector<uint64_t> padded(strlen(spec.event_signature) / 8 + 2, 0);
            memcpy(padded.data(), spec.event_signature, strlen(spec.event_signature));
            Digest d;
            keccak256((const uint8_t*)padded.data(), (uint32_t)strlen(spec.event_signature), d);
            memcpy(m_same.t0, d.w, 32);
            uint8_t t1[32];
            memset(t1, 0, 32);
            memcpy(t1, spec.topic_1, strlen(spec.topic_1) < 32 ? strlen(spec.topic_1) : 32);
            memcpy(m_same.t1, t1, 32);
        }
        m_other = m_same;
        m_other.t1[0] ^= 0x0101;
        ipcfp_event_spec spec_other = spec;
        std::string other_t1 = std::string(spec.topic_1);
        other_t1[0] ^= 1; other_t1[1] ^= 1;
        spec_other.topic_1 = other_t1.c_str();
        for (uint64_t m = 0; m <= muts; m++) {
            Blocks W = W0;
            std::vector<ipcfp_event_proof> P = P0;
            std::vector<uint8_t> B = B0;
            ipcfp_tipset_desc t = td;
            std::vector<uint8_t> pc(td.parent_cids, td.parent_cids + 38 * td.n_parents);
            const char* what = "intact";
            const Matcher* fm = nullptr;
            const ipcfp_event_spec* fs = nullptr;
            if (m > 0) {
                switch (rnd() % 9) {
                    case 0: what = "block mutated"; if (W.n) W.mutate(rnd() % W.n); break;
                    case 1: what = "block missing"; if (W.n) W.drop(rnd() % W.n); break;
                    case 2: what = "two blocks mutated"; if (W.n) { W.mutate(rnd() % W.n); W.mutate(rnd() % W.n); } break;
                    case 3: {   // a forged claim
                        what = "forged proof";
                        if (P.empty()) break;
                        ipcfp_event_proof& p = P[rnd() % P.size()];
                        switch (rnd() % 9) {
                            case 0: p.exec_index += 1 + rnd() % 3; break;
                            case 1: p.exec_index = rnd() % 2 ? UINT64_MAX : rnd(); break;
                            case 2: p.event_index = rnd() % 2 ? p.event_index + 1 : rnd(); break;
                            case 3: p.emitter ^= 1; break;
                            case 4: p.message_cid[rnd() % 38] ^= (uint8_t)(1u << (rnd() % 8)); break;
                            case 5: p.n_topics = (uint32_t)(rnd() % 6); break;
                            case 6: p.data_len += (uint32_t)(rnd() % 3) - 1; break;
                            case 7: p.topics_off = rnd() % 2 ? rnd() : B.size(); break;
                            default: p.data_off = rnd() % 2 ? rnd() : B.size() + 1; break;
                        }
                        break;
                    }
                    case 4: what = "claimed bytes changed"; if (!B.empty()) B[rnd() % B.size()] ^= (uint8_t)(1u << (rnd() % 8)); break;
                    case 5: what = "tipset fields changed"; if (rnd() % 2) t.child_epoch++; else t.parent_epoch--; break;
                    case 6: what = "parent CIDs changed"; if (!pc.empty()) { pc[rnd() % pc.size()] ^= 1; t.parent_cids = pc.data(); } break;
                    case 7: what = "check_event = the spec"; fm = &m_same; fs = &spec; break;
                    default: what = "check_event = another subnet"; fm = &m_other; fs = &spec_other; break;
                }
            }
            Verdict e = engine_events(W, t, P, B, fm);
            // offsets are an artefact of the POD ABI (the reference's EventProof carries hex strings): a proof that names bytes outside
            // the data blob is ABI misuse, which the engine rejects (false) and the restated verifier — it has no blob size — cannot be
            // asked about. Expected: the intact proof's verdicts with that proof rejected.
            std::vector<size_t> outside;
            for (size_t i = 0; i < P.size(); i++)
                if (P[i].topics_off > B.size() || 32ull * P[i].n_topics > B.size() - P[i].topics_off || P[i].data_off > B.size() || P[i].data_len > B.size() - P[i].data_off) outside.push_back(i);
            std::vector<ipcfp_event_proof> Pq = P;
            for (size_t i : outside) Pq[i] = P0[i];
            Verdict o = oracle_events(W, t, Pq, B, fs);
            if (o.status == IPCFP_OK) for (size_t i : outside) o.results[i] = 0;
            if (compare(what, e, o, &ev_ok, &ev_err)) { fprintf(stderr, "  (case %llu, mutation %llu, %llu receipts, %llu proofs)\n", (unsigned long long)c, (unsigned long long)m, (unsigned long long)sp.n_receipts, (unsigned long long)P.size()); return 1; }
            if (m == 0 && !P.empty() && !(e.status == IPCFP_OK && std::all_of(e.results.begin(), e.results.end(), [](uint8_t x) { return x == 1; }))) { fprintf(stderr, "an intact bundle was not accepted\n"); return 1; }
            if (e.status == IPCFP_OK) for (uint8_t x : e.results) (x ? accepted : rejected)++;
        }
        synth_free(ts);

        // ---------------- storage proofs from the oracle (the six root shapes, present / special / absent slots)
        if (c % 2 == 0) {
            synth_params q;
            synth_default_params(&q);
            q.seed = 700 + c;
            q.n_receipts = 8; q.events_per_receipt = 2; q.with_state_tree = 1; q.hamt_entries = 300 + (rnd() % 4000); q.n_actors = 64 + (uint32_t)(rnd() % 500);
            q.threads = 1;
            synth_tipset* t3 = synth_build(&q);
            ipcfp_tipset_desc d3 = desc_of(t3);
            oracle_store* o3 = oracle_store_create(synth_cids(t3), synth_offsets(t3), synth_lengths(t3), synth_blob(t3), synth_n_blocks(t3));
            std::vector<ipcfp_storage_spec> specs;
            for (uint64_t actor = 1001; actor <= 1006; actor++)
                for (int k = 0; k < 3; k++) {
                    ipcfp_storage_spec s;
                    memset(&s, 0, sizeof s);
                    s.actor_id = actor;
                    uint8_t key[32], val[32];
                    if (k == 0) synth_storage_entry(t3, rnd() % q.hamt_entries, key, val);
                    else if (k == 1) synth_storage_entry(t3, q.hamt_entries, key, val);
                    else synth_storage_absent_key(t3, rnd() % 50, key);
                    oracle_compute_mapping_slot(key, 0, s.slot);
                    specs.push_back(s);
                }
            ipcfp_storage_result* sr = nullptr;
            if (oracle_generate_storage_proofs(o3, &d3, specs.data(), specs.size(), &sr) != IPCFP_OK) { fprintf(stderr, "oracle_generate_storage_proofs failed\n"); return 2; }
            Blocks W0s;
            W0s.from(sr->witness);
            std::vector<ipcfp_storage_proof> S0(sr->proofs, sr->proofs + sr->n_proofs);
            oracle_storage_result_free(sr);
            oracle_store_destroy(o3);
            for (uint64_t m = 0; m <= muts; m++) {
                Blocks W = W0s;
                std::vector<ipcfp_storage_proof> S = S0;
                ipcfp_tipset_desc t = d3;
                uint8_t psr[38];
                memcpy(psr, d3.child_parent_state_root, 38);
                const char* what = "storage intact";
                if (m > 0) {
                    switch (rnd() % 5) {
                        case 0: what = "storage block mutated"; W.mutate(rnd() % W.n); break;
                        case 1: what = "storage block missing"; W.drop(rnd() % W.n); break;
                        case 2: {
                            what = "storage claim forged";
                            ipcfp_storage_proof& p = S[rnd() % S.size()];
                            switch (rnd() % 5) {
                                case 0: p.value[rnd() % 32] ^= (uint8_t)(1u << (rnd() % 8)); break;
                                case 1: p.slot[rnd() % 32] ^= 1; break;
                                case 2: p.actor_state_cid[rnd() % 38] ^= 1; break;
                                case 3: p.storage_root[rnd() % 38] ^= 1; break;
                                default: p.actor_id = rnd() % 2 ? p.actor_id + 1 : rnd(); break;
                            }
                            break;
                        }
                        case 3: what = "claimed state root changed"; psr[6 + rnd() % 32] ^= 1; t.child_parent_state_root = psr; break;
                        default: what = "two storage blocks mutated"; W.mutate(rnd() % W.n); W.mutate(rnd() % W.n); break;
                    }
                }
                Verdict e = engine_storage(W, t, S);
                Verdict o = oracle_storage(W, t, S);
                if (compare(what, e, o, &st_ok, &st_err)) { fprintf(stderr, "  (storage case %llu, mutation %llu)\n", (unsigned long long)c, (unsigned long long)m); return 1; }
                if (m == 0 && !(e.status == IPCFP_OK && std::all_of(e.results.begin(), e.results.end(), [](uint8_t x) { return x == 1; }))) { fprintf(stderr, "intact storage proofs were not accepted\n"); return 1; }
                if (e.status == IPCFP_OK) for (uint8_t x : e.results) (x ? accepted : rejected)++;
            }
            synth_free(t3);
        }
    }
    printf("ok: verifiers on the CPU == oracle for %llu bundles: events %llu runs with equal verdicts, %llu failing identically; storage %llu equal, %llu failing identically; "
           "%llu proofs accepted, %llu rejected\n",
           (unsigned long long)cases, (unsigned long long)ev_ok, (unsigned long long)ev_err, (unsigned long long)st_ok, (unsigned long long)st_err,
           (unsigned long long)accepted, (unsigned long long)rejected);
    return 0;
}
