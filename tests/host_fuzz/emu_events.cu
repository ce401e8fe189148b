// emu_events.cu — the event-proof path executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// Per-item device code of `generate_event_proof`, compiled for the host from the product headers and driven item by item:
//   k_setup's sequence (TxMeta → AMT roots, receipts root validation, base witness)        mirrored here from header functions
//   dense message-AMT walk                                                                 amt_item_dense + make_dense_plan (csrc/walk.cuh)
//   first-seen dedup of the raw list                                                       restated here (a hash set)
//   pass 1 per receipt                                                                     k_pass1_stage's arena decode, from node_events / walk_events
//   pass 2 per matching receipt                                                            pass2_item, receipts_get, walk_events<EMIT> (csrc/events_items.cuh)
// against `oracle_generate_event_proof`: matching receipts, every EventProof field, the witness CID set, n_exec — and, with one
// events / receipts block replaced by a mutated copy under the same CID (or removed), the same status at the same index.
//
//   nvcc -std=c++17 -O2 -o emu_events tests/host_fuzz/emu_events.cu oracle/oracle.cpp synth/synth.cpp -lpthread && ./emu_events
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <string>
#include <unordered_set>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/hashes.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/walk.cuh"
#ifndef __CUDA_ARCH__
#define prefetch_l2(p) ((void)0)   // inline PTX: nothing to do on the host
#endif
#include "../../ipc_filecoin_proofs_b200/csrc/events_items.cuh"
#include "../../oracle/oracle.h"
#include "../../synth/synth.h"
#include "host_store.h"
#include "host_walk.h"

using namespace ipcfp;

static uint64_t rs;
static uint64_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return rs; }

struct Blocks {
    std::vector<uint8_t> cids, blob;
    std::vector<uint64_t> offs;
    std::vector<uint32_t> lens;
    uint64_t n;
};
struct ProofRec { uint64_t exec_index, event_index, emitter; std::string topics, data, msg; bool operator==(const ProofRec& o) const { return exec_index == o.exec_index && event_index == o.event_index && emitter == o.emitter && topics == o.topics && data == o.data && msg == o.msg; } };
struct Outcome {
    int status = IPCFP_OK;
    uint64_t index = UINT64_MAX;
    std::vector<uint64_t> matching;
    std::vector<ProofRec> proofs;
    std::set<std::string> witness;
    uint64_t n_exec = 0;
    std::vector<uint32_t> touched;     // engine side: blocks the call read (mutation targets)
    bool used_general = false;
};

static void fail_tx_key(Outcome& o, uint64_t key) {   // csrc/events.cu throw_tx_error
    const uint32_t eidx = (uint32_t)(key >> 56), code = (uint32_t)(key >> 4) & 7;
    o.status = code == DC_MISSING ? IPCFP_ERR_MISSING_BLOCK : (code == DC_UNSUPPORTED ? IPCFP_ERR_UNSUPPORTED : IPCFP_ERR_DECODE);
    o.index = (eidx != IPCFP_TX_EIDX_NONE && eidx % 3 == 0 && code == DC_MISSING) ? eidx / 3 : UINT64_MAX;
}
static void fail_key(Outcome& o, uint64_t key) {   // csrc/events.cu throw_device_error
    uint32_t stage = (uint32_t)(key >> 56), code = (uint32_t)(key >> 8) & 0xff;
    uint64_t index = (key >> 16) & 0xFFFFFFFFFFull;
    switch (code) {
        case DC_MISSING: o.status = IPCFP_ERR_MISSING_BLOCK; break;
        case DC_MISSING_EXEC: o.status = IPCFP_ERR_MISSING_EXEC; break;
        case DC_UNSUPPORTED: o.status = IPCFP_ERR_UNSUPPORTED; break;
        default: o.status = IPCFP_ERR_DECODE; break;
    }
    o.index = (stage == ST_PASS1 || stage == ST_PASS2) ? index : UINT64_MAX;
    if (stage == ST_TXMETA && index != 0xFFFFFFFFFFull && index % 3 == 0 && code == DC_MISSING) o.index = index / 3;   // missing TxMeta of parent b
}

// the engine's device logic, item by item (dense walk first, the general walk when the dense one declines — as the host does)
static bool engine(const Blocks& B, const ipcfp_tipset_desc& td, const char* sig, const char* topic1, bool has_actor, uint64_t actor, Outcome& o, bool sharded = false,
                   uint64_t lo = 0, uint64_t hi = UINT64_MAX) {
    if (!sharded) { lo = 0; hi = td.n_receipts; }
    HostStore hs(B.cids.data(), B.offs.data(), B.lens.data(), B.blob.data(), B.blob.size(), B.n);
    const StoreView& sv = hs.view;
    const uint32_t P = td.n_parents, namt = 2 * P;
    unsigned long long err = IPCFP_NO_ERROR, txerr = IPCFP_NO_ERROR;
    std::vector<uint32_t> wbits((B.n + 31) / 32 + 8, 0);
    // ---- k_setup
    bool missing_base = false;
    auto base = [&](const uint8_t* cid) { int32_t b = store_lookup_host_cid(sv, cid); if (b < 0) missing_base = true; else witness_mark(wbits.data(), (uint32_t)b); };
    for (uint32_t b = 0; b < P; b++) base(td.parent_cids + 38 * b);
    base(td.child_cid); base(td.receipts_root);
    for (uint32_t b = 0; b < P; b++) base(td.parent_txmeta_cids + 38 * b);
    std::vector<uint32_t> heights(namt, 0), f_blk(namt, 0), f_meta(namt, AMT_SENTINEL);
    std::vector<uint64_t> counts(namt, 0);
    for (uint32_t b = 0; b < P; b++) {
        int32_t tb = store_lookup_host_cid(sv, td.parent_txmeta_cids + 38 * b);
        if (tb < 0) { report_tx_error(&txerr, 3 * b, 0, 31, DC_MISSING, 0); continue; }
        witness_mark(wbits.data(), (uint32_t)tb);
        uint32_t len;
        const uint8_t* p = store_block(sv, (uint32_t)tb, len);
        Rd r(p, len);
        rd_array_exact(r, 2);
        uint32_t c0 = rd_cid(r), c1 = rd_cid(r);
        rd_end(r);
        if (r.err) { report_tx_error(&txerr, 3 * b, 0, 31, DC_DECODE, r.err); continue; }
        for (uint32_t k = 0; k < 2; k++) {
            int32_t rb = store_lookup(sv, p + (k ? c1 : c0));
            if (rb < 0) { report_tx_error(&txerr, 3 * b + 1 + k, 0, 31, DC_MISSING, 0); break; }
            witness_mark(wbits.data(), (uint32_t)rb);
            uint32_t rl;
            const uint8_t* rp = store_block(sv, (uint32_t)rb, rl);
            Rd rr(rp, rl);
            uint32_t bw, h;
            uint64_t cnt;
            amt_root_begin(rr, 0, bw, h, cnt);
            if (rr.err) { report_tx_error(&txerr, 3 * b + 1 + k, 0, 31, DC_DECODE, rr.err); break; }
            const uint32_t amt = 2 * b + k;
            f_blk[amt] = (uint32_t)rb; f_meta[amt] = make_meta(amt, 1, h); heights[amt] = h; counts[amt] = cnt;
        }
    }
    uint32_t receipts_root_blk = 0;
    {
        int32_t rb = store_lookup_host_cid(sv, td.receipts_root);
        if (rb < 0) report_error(&err, ST_RECEIPTS_ROOT, 0, DC_MISSING, 0);
        else {
            witness_mark(wbits.data(), (uint32_t)rb);
            receipts_root_blk = (uint32_t)rb;
            uint32_t len;
            const uint8_t* p = store_block(sv, (uint32_t)rb, len);
            Rd r(p, len);
            uint32_t bw, h;
            uint64_t cnt;
            amt_root_begin(r, 0, bw, h, cnt);
            AmtNodeHdr hd;
            amt_node_begin(r, 3, hd);
            uint32_t nv = rd_array(r);
            for (uint32_t v = 0; v < nv && !r.err; v++) parse_receipt(r);
            amt_node_finish(r, hd, nv, h);
            if (r.err) report_error(&err, ST_RECEIPTS_ROOT, 0, DC_DECODE, r.err);
        }
    }
    // a fault seen by the prologue is not thrown yet (csrc/events.cu): the walk runs first (general kernels), then the first fault in
    // the reference's order is reported
    const bool early_fault = err != IPCFP_NO_ERROR || txerr != IPCFP_NO_ERROR;
    // ---- dense walk
    std::vector<uint64_t> rlo(namt), rhi(namt);
    shard_amt_ranges(namt, counts.data(), sharded, lo, hi, td.n_receipts, rlo.data(), rhi.data());
    DensePlan plan = make_dense_plan(namt, heights.data(), counts.data(), rlo.data(), rhi.data(), 4 * B.n + 1024, 8 * (4 * B.n + 1024), 32768);   // the engine's own limits
    std::vector<RawCid> vals;
    uint64_t nraw = 0;
    bool dense_done = false;
    if (plan.ok && !early_fault) {
        uint64_t fmax = 1;
        for (uint32_t r = 0; r < plan.rounds; r++) fmax = std::max<uint64_t>(fmax, plan.ftot[r]);
        std::vector<uint32_t> A_blk(fmax), A_meta(fmax), B_blk(fmax), B_meta(fmax), flen(2 * fmax + 8);
        std::vector<uint64_t> A_base(fmax, 0), B_base(fmax), foff(2 * fmax + 8);
        std::copy(f_blk.begin(), f_blk.end(), A_blk.begin());
        std::copy(f_meta.begin(), f_meta.end(), A_meta.begin());
        vals.assign(plan.nraw + 8, RawCid{});
        uint32_t failflag = 0;
        DenseArgs da;
        memset(&da, 0, sizeof da);
        da.store = sv;
        da.ping = Frontier{A_blk.data(), A_meta.data(), A_base.data()};
        da.pong = Frontier{B_blk.data(), B_meta.data(), B_base.data()};
        da.vals = vals.data();
        da.vbase = plan.per_amt.data(); da.cnt = plan.per_amt.data() + namt; da.lo = plan.per_amt.data() + 2ull * namt; da.hi = plan.per_amt.data() + 3ull * namt;
        da.fofs = plan.fofs.data(); da.ftot = plan.ftot.data();
        da.namt = namt; da.record = 1; da.wbits = wbits.data(); da.fail = &failflag;
        da.f_off[0] = foff.data(); da.f_off[1] = foff.data() + fmax; da.f_len[0] = flen.data(); da.f_len[1] = flen.data() + fmax;
        for (uint32_t round = 0; round < plan.rounds && !failflag; round++) {
            const Frontier in = (round & 1) ? da.pong : da.ping, out = (round & 1) ? da.ping : da.pong;
            for (uint32_t it = 0; it < plan.ftot[round]; it++)
                for (uint32_t j = 0; j < 8; j++) amt_item_dense(da, in, out, round, it, j);
        }
        dense_done = !failflag;
        nraw = plan.nraw;
    }
    o.used_general = !dense_done;
    if (!dense_done) {   // what the host does when the dense walk raises its flag (or does not apply): the general walk, exact errors
        uint32_t last_round = 0;
        for (uint32_t k = 0; k < namt; k++) last_round = std::max(last_round, heights[k]);
        host_general_walk(sv, namt, f_blk, f_meta, last_round, rlo.data(), rhi.data(), 1, wbits.data(), &txerr, 4 * B.n + 1024, vals, nraw);
    }
    if (txerr != IPCFP_NO_ERROR) { fail_tx_key(o, txerr); return true; }
    if (err != IPCFP_NO_ERROR) { fail_key(o, err); return true; }
    // ---- first-seen dedup (k_dedup_insert / k_dedup_flags + compaction)
    std::vector<uint32_t> exec_idx;
    {
        std::unordered_set<std::string> seen;
        for (uint64_t k = 0; k < nraw; k++) if (seen.insert(std::string((const char*)vals[k].w, 40)).second) exec_idx.push_back((uint32_t)k);
    }
    unsigned long long n_exec = exec_idx.size();
    o.n_exec = sharded ? 0 : n_exec;
    // ---- matcher (EventMatcher::new)
    Matcher m;
    memset(&m, 0, sizeof m);
    {   // zero padded to whole 8-byte words, 8-byte aligned: what k_setup's staging block holds (csrc/events.cu)
        std::vector<uint64_t> padded(strlen(sig) / 8 + 2, 0);
        memcpy(padded.data(), sig, strlen(sig));
        Digest d; keccak256((const uint8_t*)padded.data(), (uint32_t)strlen(sig), d); memcpy(m.t0, d.w, 32);
    }
    { uint8_t t1[32]; memset(t1, 0, 32); size_t n1 = strlen(topic1); memcpy(t1, topic1, n1 < 32 ? n1 : 32); memcpy(m.t1, t1, 32); }
    m.actor = actor; m.has_actor = has_actor ? 1 : 0;
    // ---- pass 1 (the per-receipt arena decode of k_pass1_stage)
    const uint64_t N = td.n_receipts;
    std::vector<uint32_t> cnt(N + 1, 0), nby(N + 1, 0), match_rel;
    for (uint64_t i = lo; i < hi; i++) {
        if (!td.has_events_root[i]) continue;
        int32_t blk = store_lookup_host_cid(sv, td.events_roots + 38 * i);
        if (blk < 0) { report_error(&err, ST_PASS1, i, DC_MISSING, 0); continue; }
        o.touched.push_back((uint32_t)blk);
        uint32_t len;
        const uint8_t* p = store_block(sv, (uint32_t)blk, len);
        Rd r(p, len);
        uint32_t bw, height;
        uint64_t c;
        amt_root_begin(r, 3, bw, height, c);
        AmtNodeHdr h;
        amt_node_begin(r, bw, h);
        uint32_t nv = rd_array(r);
        WalkOut wo{0, 0, false};
        node_events<WALK_COUNT>(r, p, h, nv, 0, m, wo, nullptr);
        amt_node_finish(r, h, nv, height);
        if (r.err) { report_error(&err, ST_PASS1, i, DC_DECODE, r.err); continue; }
        if (h.nl) {
            uint32_t detail = 0;
            wo = WalkOut{0, 0, false};
            uint32_t rc = walk_events<WALK_COUNT>(&sv, (uint32_t)blk, &m, nullptr, wo, nullptr, &detail);
            if (rc) { report_error(&err, ST_PASS1, i, rc, detail); continue; }
        }
        if (wo.any) match_rel.push_back((uint32_t)i);
        cnt[i] = wo.nproofs; nby[i] = wo.nbytes;
    }
    if (err != IPCFP_NO_ERROR) { fail_key(o, err); return true; }
    std::vector<uint64_t> pbase(N + 1, 0), bbase(N + 1, 0);
    uint64_t n_proofs = 0, n_bytes = 0;
    for (uint64_t i = 0; i < N; i++) { pbase[i] = n_proofs; bbase[i] = n_bytes; n_proofs += cnt[i]; n_bytes += nby[i]; }
    // ---- pass 2 (the real per-match function)
    std::vector<ipcfp_event_proof> proofs(n_proofs + 1);
    std::vector<uint8_t> blob(n_bytes + 16);
    uint32_t any_skip = 0;
    // the device copy of the events roots is n*38 + 64 bytes (csrc/events.cu, tipset upload): CIDs are loaded as aligned 8-byte words
    std::vector<uint8_t> roots_padded(td.n_receipts * 38 + 64, 0);
    if (td.n_receipts) memcpy(roots_padded.data(), td.events_roots, td.n_receipts * 38);
    Pass2Args p2;
    p2.per_warp = 0;
    memset(&p2, 0, sizeof p2);
    p2.store = sv; p2.store_dev = &sv; p2.m_dev = &m; p2.m = m; p2.events_roots = roots_padded.data(); p2.lo = 0; p2.match_rel = match_rel.data(); p2.n_match = match_rel.size();
    p2.receipts_root_blk = receipts_root_blk; p2.exec_cids = vals.data(); p2.exec_idx = exec_idx.data(); p2.n_exec = &n_exec;
    p2.wbits = wbits.data(); p2.err = &err; p2.cnt = cnt.data(); p2.proof_base = pbase.data(); p2.byte_base = bbase.data();
    p2.proofs = proofs.data(); p2.blob = blob.data(); p2.any_skip = &any_skip; p2.resolve_msg = sharded ? 0 : 1;
    for (uint64_t t = 0; t < match_rel.size(); t++) pass2_item(p2, t);
    if (err != IPCFP_NO_ERROR) { fail_key(o, err); return true; }
    if (missing_base) { o.status = IPCFP_ERR_MISSING_BLOCK; o.index = UINT64_MAX; return true; }   // WitnessCollector::materialize comes last
    for (uint32_t i : match_rel) o.matching.push_back(i);
    for (uint64_t k = 0; k < n_proofs; k++) {
        const ipcfp_event_proof& q = proofs[k];
        if (q.exec_index == UINT64_MAX) continue;             // receipt absent from the receipts AMT: dropped on the host
        ProofRec pr;
        pr.exec_index = q.exec_index; pr.event_index = q.event_index; pr.emitter = q.emitter;
        pr.topics.assign((const char*)blob.data() + q.topics_off, 32ull * q.n_topics);
        pr.data.assign((const char*)blob.data() + q.data_off, q.data_len);
        pr.msg.assign((const char*)q.message_cid, 38);
        o.proofs.push_back(pr);
    }
    for (uint64_t i = 0; i < B.n; i++) if (wbits[i >> 5] >> (i & 31) & 1) { o.witness.insert(std::string((const char*)B.cids.data() + 38 * i, 38)); }
    // mutation targets: everything pass 2 touched lies in the witness; add the receipts root
    for (uint64_t i = 0; i < B.n; i++) if (wbits[i >> 5] >> (i & 31) & 1) o.touched.push_back((uint32_t)i);
    return true;
}

static void oracle_side(const Blocks& B, const ipcfp_tipset_desc& td, const char* sig, const char* topic1, bool has_actor, uint64_t actor, Outcome& o, bool sharded = false,
                        uint64_t lo = 0, uint64_t hi = 0, uint32_t world = 1, uint32_t rank = 0) {
    oracle_store* os = oracle_store_create(B.cids.data(), B.offs.data(), B.lens.data(), B.blob.data(), B.n);
    ipcfp_event_spec spec;
    memset(&spec, 0, sizeof spec);
    spec.event_signature = sig; spec.topic_1 = topic1; spec.has_actor_id_filter = has_actor ? 1 : 0; spec.actor_id_filter = actor;
    ipcfp_event_result* er = nullptr;
    o.status = sharded ? (int)oracle_generate_event_proof_shard(os, &td, &spec, lo, hi, world, rank, 0, 1, &er) : (int)oracle_generate_event_proof(os, &td, &spec, 0, 1, &er);
    if (o.status != IPCFP_OK) o.index = oracle_last_error_index();
    else {
        for (uint64_t k = 0; k < er->n_matching; k++) o.matching.push_back(er->matching_indices[k]);
        for (uint64_t k = 0; k < er->n_proofs; k++) {
            const ipcfp_event_proof& q = er->proofs[k];
            ProofRec pr;
            pr.exec_index = q.exec_index; pr.event_index = q.event_index; pr.emitter = q.emitter;
            pr.topics.assign((const char*)er->data_blob + q.topics_off, 32ull * q.n_topics);
            pr.data.assign((const char*)er->data_blob + q.data_off, q.data_len);
            pr.msg.assign((const char*)q.message_cid, 38);
            o.proofs.push_back(pr);
        }
        for (uint64_t k = 0; k < er->witness.n_blocks; k++) o.witness.insert(std::string((const char*)er->witness.cids + 38 * k, 38));
        o.n_exec = er->n_exec;
        oracle_event_result_free(er);
    }
    oracle_store_destroy(os);
}

static unsigned g_edits = 0;        // byte edits of the current mutation

static int compare(const Blocks& B, const ipcfp_tipset_desc& td, const char* sig, const char* topic1, bool has_actor, uint64_t actor, std::vector<uint32_t>* touched,
                   uint64_t* n_ok, uint64_t* n_err, uint64_t* n_skip) {
    Outcome e, o;
    engine(B, td, sig, topic1, has_actor, actor, e);
    if (e.used_general) (*n_skip)++;
    oracle_side(B, td, sig, topic1, has_actor, actor, o);
    if (touched) *touched = e.touched;
    if (e.status != o.status || (e.status != IPCFP_OK && e.index != o.index)) {
        fprintf(stderr, "EMU MISMATCH: engine status %d index %lld vs oracle status %d index %lld\n", e.status, (long long)e.index, o.status, (long long)o.index);
        return 1;
    }
    if (e.status != IPCFP_OK) { (*n_err)++; return 0; }
    if (e.matching != o.matching) { fprintf(stderr, "EMU MISMATCH: matching receipts differ (%zu vs %zu)\n", e.matching.size(), o.matching.size()); return 1; }
    if (!(e.proofs == o.proofs)) { fprintf(stderr, "EMU MISMATCH: proofs differ (%zu vs %zu)\n", e.proofs.size(), o.proofs.size()); return 1; }
    if (e.n_exec != o.n_exec) { fprintf(stderr, "EMU MISMATCH: n_exec %llu vs %llu\n", (unsigned long long)e.n_exec, (unsigned long long)o.n_exec); return 1; }
    if (e.witness != o.witness) { fprintf(stderr, "EMU MISMATCH: witness sets differ (%zu vs %zu)\n", e.witness.size(), o.witness.size()); return 1; }
    (*n_ok)++;
    return 0;
}

// one shard of a sharded call: message CIDs and the MISSING_EXEC check belong to the cross-shard protocol, everything else is local
static int compare_shard(const Blocks& B, const ipcfp_tipset_desc& td, const char* sig, const char* topic1, bool has_actor, uint64_t actor, uint32_t world, uint32_t rank,
                         uint64_t* n_ok, uint64_t* n_err) {
    const uint64_t lo = td.n_receipts * rank / world, hi = td.n_receipts * (rank + 1) / world;
    Outcome e, o;
    engine(B, td, sig, topic1, has_actor, actor, e, true, lo, hi);
    oracle_side(B, td, sig, topic1, has_actor, actor, o, true, lo, hi, world, rank);
    if (o.status == IPCFP_ERR_MISSING_EXEC) return 0;
    if ((e.status != o.status || e.index != o.index) && o.status != IPCFP_OK && o.index == UINT64_MAX) {
        // the oracle's shard function also builds the WHOLE execution order (a second walk over every message AMT): a fault in a
        // part of the message AMTs this shard does not own surfaces there, while in the engine it belongs to the shard that owns it
        Outcome full;
        engine(B, td, sig, topic1, has_actor, actor, full);
        if (full.status == o.status && full.index == o.index) return 0;
        Outcome ofull;
        oracle_side(B, td, sig, topic1, has_actor, actor, ofull);
        // two faults in the tipset-wide stage (index -1), both visible to this shard: the engine's shard names the one the reference's
        // whole-tipset order meets first (what the cross-shard agreement needs: the minimum over shards is then the reference's error),
        // while the oracle's shard function — a construct of this repo, not of the reference — walks its owned parts first. The
        // whole-tipset results are the normative ones.
        if (e.status == full.status && e.index == full.index && full.status == ofull.status && full.index == ofull.index) { (*n_err)++; return 0; }
        fprintf(stderr, "  (whole-tipset engine run: status %d index %lld; whole-tipset oracle run: status %d index %lld)\n", full.status, (long long)full.index, ofull.status, (long long)ofull.index);
    }
    if (e.status != o.status || (e.status != IPCFP_OK && e.index != o.index)) {
        fprintf(stderr, "EMU MISMATCH (shard %u/%u): engine status %d index %lld vs oracle status %d index %lld\n", rank, world, e.status, (long long)e.index, o.status, (long long)o.index);
        return 1;
    }
    if (e.status != IPCFP_OK) { (*n_err)++; return 0; }
    bool same = e.matching == o.matching && e.proofs.size() == o.proofs.size() && e.witness == o.witness;
    for (size_t k = 0; same && k < e.proofs.size(); k++) { ProofRec a = e.proofs[k], b = o.proofs[k]; a.msg.clear(); b.msg.clear(); same = a == b; }
    if (!same) { fprintf(stderr, "EMU MISMATCH (shard %u/%u): matching %zu/%zu proofs %zu/%zu witness %zu/%zu\n", rank, world, e.matching.size(), o.matching.size(), e.proofs.size(), o.proofs.size(), e.witness.size(), o.witness.size()); return 1; }
    (*n_ok)++;
    return 0;
}

// ---- hand-built events-AMT roots: one whose height·bw wraps modulo 2^64 (bw 5, height 0x3333333333333334 over a chain of 70
// one-link nodes: refused at the root, and walk_events must not follow the chain), and the deepest legal walk (bw 1, height 64, one
// value at 2^64 − 2: 65 frames of walk_events). Under AddressSanitizer a walk deeper than its frame stack is a report.
static void put_head(std::vector<uint8_t>& o, uint32_t major, uint64_t n) {
    if (n < 24) { o.push_back((uint8_t)(major << 5 | n)); return; }
    int sz = n < 0x100 ? 1 : n < 0x10000 ? 2 : n < 0x100000000ull ? 4 : 8;
    o.push_back((uint8_t)(major << 5 | (sz == 1 ? 24 : sz == 2 ? 25 : sz == 4 ? 26 : 27)));
    for (int k = sz - 1; k >= 0; k--) o.push_back((uint8_t)(n >> (8 * k)));
}
static std::vector<uint8_t> put_block(Blocks& B, const std::vector<uint8_t>& b) {
    static const uint8_t prefix[6] = {0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
    std::vector<uint8_t> cid(prefix, prefix + 6);
    uint64_t x = 0x9E3779B97F4A7C15ull * (B.n + 1);
    for (int k = 0; k < 32; k++) { x ^= x >> 29; x *= 0xBF58476D1CE4E5B9ull; cid.push_back((uint8_t)(x >> 56)); }
    while (B.blob.size() % 16) B.blob.push_back(0);
    B.cids.insert(B.cids.end(), cid.begin(), cid.end());
    B.offs.push_back(B.blob.size());
    B.lens.push_back((uint32_t)b.size());
    B.blob.insert(B.blob.end(), b.begin(), b.end());
    B.n++;
    return cid;
}
static std::vector<uint8_t> amt_node(uint32_t bw, uint32_t slot, const std::vector<uint8_t>* link, const std::vector<uint8_t>* value) {
    std::vector<uint8_t> o{0x83};
    const uint32_t blen = bw <= 3 ? 1u : (1u << (bw - 3));
    put_head(o, 2, blen);
    for (uint32_t k = 0; k < blen; k++) o.push_back((link || value) && slot / 8 == k ? (uint8_t)(1u << (slot % 8)) : 0);
    o.push_back(link ? 0x81 : 0x80);
    if (link) { o.insert(o.end(), {0xd8, 0x2a, 0x58, 0x27, 0x00}); o.insert(o.end(), link->begin(), link->end()); }
    o.push_back(value ? 0x81 : 0x80);
    if (value) o.insert(o.end(), value->begin(), value->end());
    return o;
}
static std::vector<uint8_t> amt_root(uint32_t bw, uint64_t height, const std::vector<uint8_t>& node) {
    std::vector<uint8_t> o{0x84};
    put_head(o, 0, bw); put_head(o, 0, height); put_head(o, 0, 1);
    o.insert(o.end(), node.begin(), node.end());
    return o;
}
static int hand_built_roots() {
    Matcher m;
    memset(&m, 0, sizeof m);
    std::vector<uint8_t> ev{0x82, 0x19, 0x03, 0xe9, 0x82};   // [1001, [t1 = 32 × 0x11, t2 = 32 × 0x22]]
    for (uint8_t t : {(uint8_t)0x11, (uint8_t)0x22}) {
        ev.insert(ev.end(), {0x84, 0x03, 0x62, 't', (uint8_t)(t == 0x11 ? '1' : '2'), 0x18, 0x55, 0x58, 0x20});
        ev.insert(ev.end(), 32, t);
    }
    memset(m.t0, 0x11, 32); memset(m.t1, 0x22, 32);
    // the wrapping height
    Blocks B;
    B.n = 0;
    std::vector<uint8_t> c = put_block(B, amt_node(5, 0, nullptr, nullptr));
    for (int d = 0; d < 70; d++) c = put_block(B, amt_node(5, 0, &c, nullptr));
    put_block(B, amt_root(5, 0x3333333333333334ull, amt_node(5, 0, &c, nullptr)));
    // the deepest legal walk: 2^64 − 2 takes slot 0 at height 64, slot 1 at 63 … 1, slot 0 at the leaf
    c = put_block(B, amt_node(1, 0, nullptr, &ev));
    for (int lvl = 1; lvl <= 63; lvl++) c = put_block(B, amt_node(1, 1, &c, nullptr));
    put_block(B, amt_root(1, 64, amt_node(1, 0, &c, nullptr)));
    B.blob.resize(B.blob.size() + 64, 0);
    HostStore hs(B.cids.data(), B.offs.data(), B.lens.data(), B.blob.data(), B.blob.size(), B.n);
    const StoreView& sv = hs.view;
    const uint32_t wrap_root = 71, deep_root = (uint32_t)B.n - 1;
    {
        uint32_t len, bw, height;
        uint64_t cnt;
        const uint8_t* p = store_block(sv, wrap_root, len);
        WalkOut wo{0, 0, false};
        uint32_t detail = 0;
        uint32_t rc = walk_events<WALK_COUNT>(&sv, wrap_root, &m, nullptr, wo, nullptr, &detail);   // first: a walk down the chain overflows
        if (rc != DC_DECODE) { fprintf(stderr, "HAND-BUILT: walk of the wrapping root returned %u, not a decode error\n", rc); return 1; }
        Rd r(p, len);
        amt_root_begin(r, 3, bw, height, cnt);
        if (!r.err) { fprintf(stderr, "HAND-BUILT: root of height 0x3333333333333334 at bit width 5 decoded\n"); return 1; }
    }
    {
        WalkOut wo{0, 0, false};
        uint32_t detail = 0;
        uint32_t rc = walk_events<WALK_COUNT>(&sv, deep_root, &m, nullptr, wo, nullptr, &detail);
        if (rc || wo.nproofs != 1) { fprintf(stderr, "HAND-BUILT: deepest walk returned %u with %u proofs\n", rc, wo.nproofs); return 1; }
        ipcfp_event_proof q[1];
        std::vector<uint8_t> blob(wo.nbytes + 16);
        EmitCtx ec;
        memset(&ec, 0, sizeof ec);
        ec.proofs = q; ec.blob = blob.data(); ec.blob_off = 0; ec.exec_index = 3;
        wo = WalkOut{0, 0, false};
        rc = walk_events<WALK_EMIT>(&sv, deep_root, &m, nullptr, wo, &ec, &detail);
        if (rc || wo.nproofs != 1 || q[0].event_index != 0xFFFFFFFFFFFFFFFEull || q[0].emitter != 1001) {
            fprintf(stderr, "HAND-BUILT: deepest walk emitted event index %llx\n", (unsigned long long)q[0].event_index);
            return 1;
        }
    }
    return 0;
}

int main(int argc, char** argv) {
    if (hand_built_roots()) return 1;
    uint64_t cases = argc > 1 ? strtoull(argv[1], nullptr, 10) : 10;
    uint64_t muts = argc > 2 ? strtoull(argv[2], nullptr, 10) : 60;
    rs = argc > 3 ? strtoull(argv[3], nullptr, 10) : 0xE7E47ull;
    {   // keccak on the host build (the matcher depends on it)
        alignas(8) static const uint8_t abc[16] = {'a', 'b', 'c'};   // the device keccak reads whole aligned 8-byte words: zero padded, as k_setup's input is
        Digest d; keccak256(abc, 3, d);
        uint8_t ref[32]; oracle_keccak256((const uint8_t*)"abc", 3, ref);
        if (memcmp(d.w, ref, 32)) { fprintf(stderr, "host build of keccak256 is broken\n"); return 2; }
        // the DEVICE keccak256 (csrc/hashes.cuh, this very code runs in k_setup / k_hash_batch) on two known answers the reference tree
        // itself holds (vendored forge-std: StdConstants.sol:10 and test/StdUtils.t.sol:267; tests/golden/reference_keccak_vectors.json)
        alignas(8) static const uint8_t m1[16] = {'h', 'e', 'v', 'm', ' ', 'c', 'h', 'e', 'a', 't', ' ', 'c', 'o', 'd', 'e'};
        static const uint8_t vm_addr[20] = {0x71, 0x09, 0x70, 0x9E, 0xCf, 0xa9, 0x1a, 0x80, 0x62, 0x6f, 0xF3, 0x98, 0x9D, 0x68, 0xf6, 0x7F, 0x5b, 0x1D, 0xD1, 0x2D};
        keccak256(m1, 15, d);
        if (memcmp((const uint8_t*)d.w + 12, vm_addr, 20)) { fprintf(stderr, "device keccak256 != forge-std VM address constant\n"); return 2; }
        alignas(8) static const uint8_t m2[8] = {0x60, 0x80};
        static const uint8_t h6080[32] = {0x1a, 0x57, 0x8b, 0x7a, 0x4b, 0x0b, 0x57, 0x55, 0xdb, 0x6d, 0x12, 0x1b, 0x41, 0x18, 0xd4, 0xbc,
                                          0x68, 0xfe, 0x17, 0x0d, 0xca, 0x84, 0x0c, 0x59, 0xbc, 0x92, 0x2f, 0x14, 0x17, 0x5a, 0x76, 0xb0};
        keccak256(m2, 2, d);
        if (memcmp(d.w, h6080, 32)) { fprintf(stderr, "device keccak256 != hashInitCode(hex\"6080\") of forge-std's tests\n"); return 2; }
    }
    uint64_t n_ok = 0, n_err = 0, n_skip = 0;
    for (uint64_t c = 0; c < cases; c++) {
        synth_params sp;
        synth_default_params(&sp);
        sp.seed = 4000 + c * 7 + (rs & 0xff);
        static const uint64_t sizes[] = {0, 1, 8, 9, 40, 64, 65, 257, 700, 2000};   // incl. the empty tipset and the AMT width boundaries
        sp.n_receipts = sizes[rnd() % 10];
        static const uint32_t evs[] = {1, 3, 8, 8, 40, 300};
        sp.events_per_receipt = evs[rnd() % 6];
        if (sp.n_receipts * sp.events_per_receipt > 60000) sp.events_per_receipt = 8;
        sp.match_ppm = 1000u << (rnd() % 10);
        if (sp.match_ppm > 1000000) sp.match_ppm = 1000000;
        sp.has_actor_filter = (uint32_t)(rnd() % 2);
        sp.bw3_permille = (uint32_t)(rnd() % 1001);
        sp.case_a_permille = rnd() % 2 ? (uint32_t)(rnd() % 500) : 0;
        sp.malformed_permille = rnd() % 2 ? (uint32_t)(rnd() % 200) : 0;
        sp.null_root_permille = rnd() % 2 ? (uint32_t)(rnd() % 300) : 0;
        sp.n_parents = 1 + (uint32_t)(rnd() % 3);
        sp.dup_msgs = (uint32_t)(rnd() % 4);
        sp.with_state_tree = 0;
        sp.threads = 1;
        synth_tipset* ts = synth_build(&sp);
        Blocks B;
        B.n = synth_n_blocks(ts);
        B.cids.assign(synth_cids(ts), synth_cids(ts) + 38 * B.n);
        B.offs.assign(synth_offsets(ts), synth_offsets(ts) + B.n);
        B.lens.assign(synth_lengths(ts), synth_lengths(ts) + B.n);
        B.blob.assign(synth_blob(ts), synth_blob(ts) + synth_blob_size(ts));
        ipcfp_tipset_desc td;
        memset(&td, 0, sizeof td);
        td.parent_epoch = synth_parent_epoch(ts); td.child_epoch = synth_child_epoch(ts); td.n_parents = synth_n_parents(ts);
        td.parent_cids = synth_parent_cids(ts); td.parent_txmeta_cids = synth_parent_txmeta_cids(ts); td.child_cid = synth_child_cid(ts);
        td.receipts_root = synth_receipts_root(ts); td.child_parent_state_root = synth_parent_state_root(ts); td.n_receipts = synth_n_receipts(ts);
        td.events_roots = synth_events_roots(ts); td.has_events_root = synth_has_events_root(ts);
        const char* sig = synth_event_signature(ts);
        const char* t1 = synth_topic1(ts);
        const bool has_actor = sp.has_actor_filter != 0;
        const uint64_t actor = synth_target_actor(ts);
        std::vector<uint32_t> touched;
        g_edits = 0;
        if (compare(B, td, sig, t1, has_actor, actor, &touched, &n_ok, &n_err, &n_skip)) { fprintf(stderr, "  (tipset %llu as built)\n", (unsigned long long)c); return 1; }
        for (uint32_t world : {2u, 3u}) for (uint32_t rank = 0; rank < world; rank++)
            if (compare_shard(B, td, sig, t1, has_actor, actor, world, rank, &n_ok, &n_err)) { fprintf(stderr, "  (tipset %llu as built)\n", (unsigned long long)c); return 1; }
        std::vector<uint32_t> targets = touched;   // events blocks, receipts-AMT nodes, message-AMT nodes, TxMeta, headers
        std::sort(targets.begin(), targets.end());
        targets.erase(std::unique(targets.begin(), targets.end()), targets.end());
        for (uint64_t mi = 0; mi < muts && !targets.empty(); mi++) {
            Blocks M = B;
            uint32_t victim = targets[rnd() % targets.size()];
            if (mi % 3 == 0) {   // a SECOND, independent fault in another block: the error named must still be the one the reference meets first
                uint32_t v2 = targets[rnd() % targets.size()];
                if (v2 != victim) {
                    if (rnd() % 2) M.cids[38ull * v2 + 21] ^= 0xa5;                               // missing
                    else {                                                                        // or damaged in place (same length)
                        size_t at = rnd() % B.lens[v2];
                        M.blob[B.offs[v2] + at] ^= (uint8_t)(1u << (rnd() % 8));
                    }
                }
            }
            std::vector<uint8_t> blk(B.blob.begin() + (long)B.offs[victim], B.blob.begin() + (long)B.offs[victim] + B.lens[victim]);
            unsigned nm = 1 + (unsigned)(rnd() % 2);
            g_edits = nm;
            for (unsigned k = 0; k < nm; k++) {
                size_t at = rnd() % blk.size();
                switch (rnd() % 5) {
                    case 0: blk[at] = (uint8_t)rnd(); break;
                    case 1: blk[at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                    case 2: blk.erase(blk.begin() + (long)at); break;
                    case 3: blk.insert(blk.begin() + (long)at, (uint8_t)rnd()); break;
                    default: blk.resize(at); break;
                }
                if (blk.empty()) blk.push_back(0x80);
            }
            while (M.blob.size() % 16) M.blob.push_back(0);
            M.offs[victim] = M.blob.size();
            M.lens[victim] = (uint32_t)blk.size();
            M.blob.insert(M.blob.end(), blk.begin(), blk.end());
            if (rnd() % 12 == 0) { M.cids[38ull * victim + 20] ^= 0x5a; g_edits++; }      // the block is simply not there
            if (mi % 8 == 0 && compare_shard(M, td, sig, t1, has_actor, actor, 2, (uint32_t)(mi / 8 % 2), &n_ok, &n_err)) { fprintf(stderr, "  (tipset %llu, mutation %llu of block %u, shard)\n", (unsigned long long)c, (unsigned long long)mi, victim); return 1; }
            if (compare(M, td, sig, t1, has_actor, actor, nullptr, &n_ok, &n_err, &n_skip)) {
                fprintf(stderr, "  (tipset %llu, mutation %llu of block %u)\n  original:", (unsigned long long)c, (unsigned long long)mi, victim);
                for (uint32_t k = 0; k < B.lens[victim]; k++) fprintf(stderr, " %02x", B.blob[B.offs[victim] + k]);
                fprintf(stderr, "\n  mutated: ");
                for (size_t k = 0; k < blk.size(); k++) fprintf(stderr, " %02x", blk[k]);
                fprintf(stderr, "\n  cid changed: %d\n", memcmp(M.cids.data() + 38ull * victim, B.cids.data() + 38ull * victim, 38) != 0);
                return 1;
            }
        }
        synth_free(ts);
    }
    printf("ok: event path on the CPU == oracle for %llu tipsets: %llu runs equal in every field, %llu runs failing identically, %llu of them through the general walk (one run in three carries two independent faults)\n",
           (unsigned long long)cases, (unsigned long long)n_ok, (unsigned long long)n_err, (unsigned long long)n_skip);
    printf("ok: hand-built roots: a height whose product with the bit width wraps is refused, the 65-frame walk emits index 2^64 - 2\n");
    return 0;
}
