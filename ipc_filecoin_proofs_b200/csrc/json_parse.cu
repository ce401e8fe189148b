// json_parse.cu — ipcfp_verify_bundle_json: verify_proof_bundle (src/proofs/verifier.rs:12-60) from the bundle's JSON text, with the
// parse, the witness store and the verification on the device. The canonical text (json_parse_items.cuh) is parsed here; any other text
// goes through ipcfp_bundle_from_json (csrc/bundle_parse.cpp) and the host-array entry points, so results never depend on the path.
//
// Device path, all on the store's stream:
//   H2D of the text (+ JP_PAD zero bytes)
//   k_jp_mark              one thread per 32 text bytes: bit p of the bitmap = a record starts at p (jp_kind_at)
//   bitmap_to_indices      record starts, ascending (prims.cu)
//   k_jp_records           one warp per record: its template check and its joints (lane 0), the base64 characters of a block (all lanes);
//                          per record the data-blob bytes (event proofs) and 16-aligned arena bytes (blocks), the lists' first / last
//                          records, the defer flag
//   exclusive_scan_u32 ×2  data-blob offsets of the event proofs, arena offsets of the blocks
//   ── host synchronisation 1: the meta words. The host checks the framing and reads the shared tipset fields from the first proofs.
//   k_jp_proofs            one thread per proof: the PODs and the topic / data bytes
//   trust callbacks (host); if a trusted proof is left:
//   k_jp_blocks            one warp per block: CID bytes, offset, length, base64 decoded straight into the new store's arena
//   store_finish (store.cu; host synchronisations of the class check and of the CID check)
//   verify_storage_proofs_dev / verify_event_proofs_dev (verify.cu)
#include <cstring>

#include "engine.cuh"
#include "json_parse_items.cuh"
#include "text_scan.cuh"

namespace ipcfp {

// device meta words of one parse (UINT64_MAX = none, except witness_bytes)
struct JpMeta {
    unsigned long long defer;   // the smallest record index that is not canonical (or n when the count alone is out of range)
    unsigned long long n;       // record starts
    unsigned long long first[3], last[3], first_start[3], last_end[3];
    unsigned long long witness_bytes;
    unsigned long long e_total, b_total;
};
static_assert(sizeof(JpMeta) <= HW_PARSE_META_WORDS * 8, "the meta words fit their host words (HW_PARSE_META)");

__global__ void __launch_bounds__(256) k_jp_mark(const char* __restrict__ t, uint64_t len, uint32_t* bits, uint64_t nwords) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwords) return;
    uint32_t b = 0;
    for (uint32_t k = 0; k < 32; k++) {
        const uint64_t p = 32 * w + k;
        if (p < len && t[p] == '{' && jp_kind_at(t, p) != JP_NONE) b |= 1u << k;
    }
    bits[w] = b;
}

// one warp per record slot of [0, cap); slots past the record count write zero lengths (the scans run over cap)
__global__ void __launch_bounds__(128) k_jp_records(const char* __restrict__ t, uint64_t len, const uint32_t* __restrict__ pos, uint64_t cap,
                                                    JpMeta* meta, uint32_t* elen, uint32_t* blen) {
    const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (w >= cap) return;
    const uint64_t n = meta->n;
    if (n > cap) {   // denser than any canonical text
        if (w == 0 && lane == 0) atomicMin(&meta->defer, (unsigned long long)n);
        return;
    }
    if (w >= n) {
        if (lane == 0) { elen[w] = 0; blen[w] = 0; }
        return;
    }
    JpRec r;
    bool ok = true;
    if (lane == 0) ok = jp_record(t, len, pos, n, w, r);
    ok = __shfl_sync(0xffffffffu, ok, 0);
    const uint32_t kind = __shfl_sync(0xffffffffu, ok ? r.kind : JP_NONE, 0);
    if (ok && kind == JP_BLOCK) {   // the base64 characters, split over the lanes
        JpBlock b;
        b.data_at = __shfl_sync(0xffffffffu, r.blk.data_at, 0);
        b.n_chars = __shfl_sync(0xffffffffu, r.blk.n_chars, 0);
        b.pads = __shfl_sync(0xffffffffu, r.blk.pads, 0);
        bool good = true;
        for (uint64_t k = lane; k < b.n_chars - b.pads; k += 32) good &= jp_block_char_ok(t, b, k);
        ok = __all_sync(0xffffffffu, good);
    }
    if (lane) return;
    if (!ok) { atomicMin(&meta->defer, (unsigned long long)w); elen[w] = 0; blen[w] = 0; return; }
    elen[w] = r.kind == JP_EVENT ? (uint32_t)r.blob_len : 0u;
    blen[w] = r.kind == JP_BLOCK ? (uint32_t)r.blob_len : 0u;
    if (r.first) { meta->first[r.kind] = w; meta->first_start[r.kind] = pos[w]; }
    if (r.last) { meta->last[r.kind] = w; meta->last_end[r.kind] = r.end; }
    if (r.kind == JP_BLOCK) atomicAdd(&meta->witness_bytes, (unsigned long long)r.len);
}

// records [0, nS) are storage proofs, [nS, nS + nE) event proofs (the lists come in that order)
__global__ void __launch_bounds__(128) k_jp_proofs(const char* __restrict__ t, uint64_t len, const uint32_t* __restrict__ pos, uint64_t nS, uint64_t nE,
                                                   const uint64_t* __restrict__ eoff, ipcfp_storage_proof* sp, ipcfp_event_proof* ep, uint8_t* blob) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nS + nE) return;
    uint64_t end;
    if (i < nS) {
        JpStorage s;
        jp_storage_proof(t, pos[i], len, s, end, sp + i);
        return;
    }
    JpEvent r;
    jp_event_proof(t, pos[i], len, r, end);
    ipcfp_event_proof p;
    jp_event_write(t, r, eoff[i], p, blob);
    ep[i - nS] = p;
}

// one warp per block: record first + j is block j of the store
__global__ void __launch_bounds__(128) k_jp_blocks(const char* __restrict__ t, uint64_t len, const uint32_t* __restrict__ pos, uint64_t n, uint64_t first,
                                                   uint64_t nb, const uint64_t* __restrict__ boff, uint8_t* cids, uint64_t* offsets, uint32_t* lengths,
                                                   uint8_t* blob) {
    const uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (j >= nb) return;
    const uint64_t i = first + j;
    const uint64_t end = i + 1 < n ? (uint64_t)pos[i + 1] - 1 : len - 2;
    JpBlock b;
    if (lane == 0) {
        jp_block_head(t, pos[i], end, b, cids + 38 * j);
        offsets[j] = boff[i];
        lengths[j] = b.len;
    }
    b.data_at = __shfl_sync(0xffffffffu, b.data_at, 0);
    b.n_chars = __shfl_sync(0xffffffffu, b.n_chars, 0);
    b.len = __shfl_sync(0xffffffffu, b.len, 0);
    uint8_t* out = blob + boff[i];
    for (uint64_t g = lane; g < b.n_chars / 4; g += 32) jp_block_group(t, b, g, out);
}

// ------------------------------------------------------------------------------------------ host flow
struct VerdictBox {
    ipcfp_bundle_verdict v;   // FIRST member: the handle is a pointer to it
    ipcfp_parsed_bundle* pb = nullptr;   // host path: the parsed bundle the verdict's pointers name
    std::vector<uint8_t> parents, child, root, blob, sres, eres;
    std::vector<ipcfp_storage_proof> sp;
    std::vector<ipcfp_event_proof> ep;
    ~VerdictBox() { if (pb) ipcfp_parsed_bundle_free(pb); }
};

// verify_trust_anchors / verify_trust_anchor of the bundle: each callback at most once
struct Trust { bool child = false, parent = false; };
static Trust ask_trust(const ipcfp_tipset_desc& t, uint64_t nS, uint64_t nE, ipcfp_trusted_parent_ts_fn trusted_parent,
                       ipcfp_trusted_child_header_fn trusted_child, void* ctx) {
    Trust tr;
    if (nS + nE == 0) return tr;
    tr.child = !trusted_child || trusted_child(ctx, t.child_epoch, t.child_cid) != 0;
    if (nE && tr.child) tr.parent = !trusted_parent || trusted_parent(ctx, t.parent_epoch, t.parent_cids, t.n_parents) != 0;
    return tr;
}

// runs the verifiers of the trusted proofs; event failures are indexed after every storage proof
template <class VS, class VE> static void run_verifiers(const Trust& tr, uint64_t nS, uint64_t nE, VS vs, VE ve) {
    if (tr.child && nS) vs();
    if (tr.child && tr.parent && nE) {
        try { ve(); }
        catch (Error& e) { if (e.index != UINT64_MAX) e.index += nS; throw; }
    }
}

// the composition itself, on the host parser's arrays
static void verify_host_path(VerdictBox& B, const char* json, uint64_t len, int device, ipcfp_trusted_parent_ts_fn tp, ipcfp_trusted_child_header_fn tc,
                             void* ctx, const ipcfp_event_spec* filter, const ipcfp_log_filter* lf, uint64_t n_lf,
                             Clock::time_point t0) {
    ipcfp_bundle_verdict& v = B.v;
    const ipcfp_status st = ipcfp_bundle_from_json(json, len, &B.pb);
    if (st != IPCFP_OK) throw Error(st, "ipcfp_bundle_from_json refused the text");
    const ipcfp_parsed_bundle& pb = *B.pb;
    v.tipset = pb.tipset;
    v.n_storage_proofs = pb.n_storage_proofs; v.storage_proofs = pb.storage_proofs;
    v.n_event_proofs = pb.n_event_proofs; v.event_proofs = pb.event_proofs;
    v.data_blob = pb.data_blob; v.data_blob_size = pb.data_blob_size;
    v.n_blocks = pb.witness.n_blocks;
    for (uint64_t i = 0; i < pb.witness.n_blocks; i++) v.witness_bytes += pb.witness.lengths[i];
    B.sres.assign(pb.n_storage_proofs + 1, 0);
    B.eres.assign(pb.n_event_proofs + 1, 0);
    v.storage_results = B.sres.data(); v.event_results = B.eres.data();
    v.ms_parse = ms_since(t0);
    const Trust tr = ask_trust(pb.tipset, pb.n_storage_proofs, pb.n_event_proofs, tp, tc, ctx);
    if (!tr.child || (!pb.n_storage_proofs && !(tr.parent && pb.n_event_proofs))) return;
    const Clock::time_point t1 = Clock::now();
    const ipcfp_witness& w = pb.witness;
    std::unique_ptr<Store> s(store_create(w.cids, w.offsets, w.lengths, w.blob, w.blob_size, w.n_blocks, device, IPCFP_STORE_VERIFY_CIDS));
    if (s->first_bad != UINT64_MAX) throw Error(IPCFP_ERR_CID_MISMATCH, "blake2b-256(block) != CID digest", s->first_bad);
    v.ms_store = ms_since(t1);
    const Clock::time_point t2 = Clock::now();
    run_verifiers(tr, pb.n_storage_proofs, pb.n_event_proofs,
                  [&] { verify_storage_proofs(s.get(), &pb.tipset, pb.storage_proofs, pb.n_storage_proofs, B.sres.data()); },
                  [&] { verify_event_proofs(s.get(), &pb.tipset, pb.event_proofs, pb.n_event_proofs, pb.data_blob, pb.data_blob_size, filter, B.eres.data(), lf, n_lf); });
    v.ms_verify = ms_since(t2);
}

// the device path; false: the text is not canonical (nothing of B has been set)
static bool verify_device_path(VerdictBox& B, const char* json, uint64_t len, int device, ipcfp_trusted_parent_ts_fn tp, ipcfp_trusted_child_header_fn tc,
                               void* ctx, const ipcfp_event_spec* filter, const ipcfp_log_filter* lf, uint64_t n_lf,
                               Clock::time_point t0) {
    if (len < 2 || len > 0xffffff00ull) return false;   // record starts are u32
    try { check_device(device); }
    catch (const Error&) { return false; }   // the host path meets the same failure where the composition does
    std::unique_ptr<Store> s(store_shell(device));
    cudaStream_t st = s->stream;
    const uint64_t cap = len / JP_MIN_RECORD + 1;
    TextScan<JpMeta> sc(s.get(), len, len / 8 + 8, cap, 0xff);
    AsyncBuf<uint32_t> elen(cap + 1, st), blen(cap + 1, st);
    AsyncBuf<uint64_t> eoff(cap + 1, st), boff(cap + 1, st);
    IPCFP_CUDA(cudaMemcpyAsync(sc.text.p, json, len, cudaMemcpyHostToDevice, st));
    IPCFP_CUDA(cudaMemsetAsync(&sc.meta.p->witness_bytes, 0, 8, st));
    sc.starts(k_jp_mark);
    k_jp_records<<<div_up(cap * 32, 128), 128, 0, st>>>(sc.text.p, len, sc.pos.p, cap, sc.meta.p, elen.p, blen.p); IPCFP_LAUNCH_CHECK();
    exclusive_scan_u32(elen.p, eoff.p, cap, (uint64_t*)&sc.meta.p->e_total, sc.scratch.p, st);
    exclusive_scan_u32(blen.p, boff.p, cap, (uint64_t*)&sc.meta.p->b_total, sc.scratch.p, st);
    const JpMeta m = sc.read();   // host synchronisation 1
    if (m.defer != UINT64_MAX || m.n > cap) return false;
    uint64_t cnt[3], first_start[3], last_end[3];
    for (int k = 0; k < 3; k++) { cnt[k] = m.first[k] == UINT64_MAX ? 0 : m.last[k] - m.first[k] + 1; first_start[k] = m.first_start[k]; last_end[k] = m.last_end[k]; }
    if (!jp_frame_ok(json, len, cnt, first_start, last_end)) return false;
    // the shared fields, from the first proof of each list (the device checked that the others repeat them)
    const uint64_t nS = cnt[JP_STORAGE], nE = cnt[JP_EVENT], nB = cnt[JP_BLOCK];
    JpTipset ts;
    if (!jp_tipset(json, len, cnt, first_start, ts)) return false;
    B.parents.resize(38ull * ts.n_parents);
    for (uint32_t q = 0; q < ts.n_parents; q++) jp_cid_at(json, ts.parents_at + 65ull * q, B.parents.data() + 38ull * q);
    if (ts.has_child) B.child.assign(ts.child, ts.child + IPCFP_CID_LEN);
    if (ts.has_root) B.root.assign(ts.root, ts.root + IPCFP_CID_LEN);
    ipcfp_bundle_verdict& v = B.v;
    v.parsed_on_device = 1;
    v.tipset.parent_epoch = ts.parent_epoch;
    v.tipset.child_epoch = ts.child_epoch;
    v.tipset.n_parents = ts.n_parents;
    v.tipset.parent_cids = B.parents.empty() ? nullptr : B.parents.data();
    v.tipset.child_cid = B.child.empty() ? nullptr : B.child.data();
    v.tipset.child_parent_state_root = B.root.empty() ? nullptr : B.root.data();
    v.n_storage_proofs = nS; v.n_event_proofs = nE; v.n_blocks = nB;
    v.witness_bytes = m.witness_bytes;
    v.data_blob_size = m.e_total;
    // the proofs, their data blob, back to the caller
    AsyncBuf<ipcfp_storage_proof> d_sp(nS + 1, st);
    AsyncBuf<ipcfp_event_proof> d_ep(nE + 1, st);
    AsyncBuf<uint8_t> d_blob(m.e_total + 16, st);
    if (nS + nE) { k_jp_proofs<<<div_up(nS + nE, 128), 128, 0, st>>>(sc.text.p, len, sc.pos.p, nS, nE, eoff.p, d_sp.p, d_ep.p, d_blob.p); IPCFP_LAUNCH_CHECK(); }
    B.sp.resize(nS + 1); B.ep.resize(nE + 1); B.blob.assign(m.e_total + 16, 0);
    B.sres.assign(nS + 1, 0); B.eres.assign(nE + 1, 0);
    if (nS) IPCFP_CUDA(cudaMemcpyAsync(B.sp.data(), d_sp.p, nS * sizeof(ipcfp_storage_proof), cudaMemcpyDeviceToHost, st));
    if (nE) IPCFP_CUDA(cudaMemcpyAsync(B.ep.data(), d_ep.p, nE * sizeof(ipcfp_event_proof), cudaMemcpyDeviceToHost, st));
    if (m.e_total) IPCFP_CUDA(cudaMemcpyAsync(B.blob.data(), d_blob.p, m.e_total, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    v.storage_proofs = B.sp.data(); v.event_proofs = B.ep.data(); v.data_blob = B.blob.data();
    v.storage_results = B.sres.data(); v.event_results = B.eres.data();
    v.ms_parse = ms_since(t0);

    const Trust tr = ask_trust(v.tipset, nS, nE, tp, tc, ctx);
    if (!tr.child || (!nS && !(tr.parent && nE))) return true;
    // the witness store, decoded straight into its arena
    const Clock::time_point t1 = Clock::now();
    DevBuf<uint8_t> cids_dev;
    uint8_t* blocks = store_alloc_blocks(s.get(), nB, m.b_total, cids_dev, true);
    uint8_t prefix[6] = {};
    if (nB) {
        k_jp_blocks<<<div_up(nB * 32, 128), 128, 0, st>>>(sc.text.p, len, sc.pos.p, m.n, m.first[JP_BLOCK], nB, boff.p, cids_dev.p, s->offsets.p,
                                                          s->lengths.p, blocks);
        IPCFP_LAUNCH_CHECK();
        JpCur c{json, first_start[JP_BLOCK], len};
        c.lit("{\"cid\":[");
        for (int k = 0; k < 6; k++) { uint64_t x = 0; if (k) c.lit(","); c.u64(x); prefix[k] = (uint8_t)x; }
    }
    store_finish(s.get(), cids_dev.p, nullptr, prefix, IPCFP_STORE_VERIFY_CIDS);
    if (s->first_bad != UINT64_MAX) throw Error(IPCFP_ERR_CID_MISMATCH, "blake2b-256(block) != CID digest", s->first_bad);
    v.ms_store = ms_since(t1);
    const Clock::time_point t2 = Clock::now();
    run_verifiers(tr, nS, nE, [&] { verify_storage_proofs_dev(s.get(), &v.tipset, d_sp.p, nS, B.sres.data()); },
                  [&] { verify_event_proofs_dev(s.get(), &v.tipset, d_ep.p, nE, d_blob.p, m.e_total, filter, B.eres.data(), lf, n_lf); });
    v.ms_verify = ms_since(t2);
    return true;
}

ipcfp_bundle_verdict* verify_bundle_json(const char* json, uint64_t len, int device, ipcfp_trusted_parent_ts_fn trusted_parent,
                                         ipcfp_trusted_child_header_fn trusted_child, void* trust_ctx, const ipcfp_event_spec* filter,
                                         const ipcfp_log_filter* log_filters, uint64_t n_log_filters) {
    const Clock::time_point t0 = Clock::now();
    std::unique_ptr<VerdictBox> B(new VerdictBox());
    memset(&B->v, 0, sizeof B->v);
    if (!verify_device_path(*B, json, len, device, trusted_parent, trusted_child, trust_ctx, filter, log_filters, n_log_filters, t0)) {
        B.reset(new VerdictBox());
        memset(&B->v, 0, sizeof B->v);
        verify_host_path(*B, json, len, device, trusted_parent, trusted_child, trust_ctx, filter, log_filters, n_log_filters, t0);
    }
    B->v.ms_total = ms_since(t0);
    return &B.release()->v;
}
void bundle_verdict_free(ipcfp_bundle_verdict* v) { delete reinterpret_cast<VerdictBox*>(v); }

}  // namespace ipcfp
