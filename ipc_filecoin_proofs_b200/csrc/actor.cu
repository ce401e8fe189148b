// actor.cu — ipcfp_generate_actor_proofs_resident: what the state tree holds for an address (DESIGN.md §2, "Actor proofs"). Per-proof
// code: actor_items.cuh.
//   k_actor_init         one warp, lane 0: StateRoot → actors HAMT → Init actor → InitState (the k_resolve_init walk), recorded in a list of
//                        its own; runs once per call, and only when some address is not an ID address
//   k_actor_proofs       one request per warp, lane 0 walks (the shape of k_storage_proofs): header, address_map, actors HAMT, EVM state,
//                        and with IPCFP_ACTOR_WITH_CODE the bytecode block and its Keccak-256
//   k_actor_code_gather  IPCFP_ACTOR_WITH_CODE: one CTA per proof copies its bytecode into the code blob
// Every block a walk reads is marked in one rank bitmap, materialised as the call's witness; each proof's list is its own recorder list,
// joined with the Init path's list for a non-ID address.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "actor_items.cuh"
#include "engine.cuh"

namespace ipcfp {

__global__ void k_actor_init(ActorArgs a) {
    if (threadIdx.x) return;
    Recorder rec{a.init_list, 0, a.wbits, false};
    rec.rank_of = a.store.rank_of;
    rec.strict_only = a.strict_only != 0;
    Fail f{0, 0};
    const uint8_t* map = nullptr;
    if (!resolve_init(a.store, rec, a.state_root_json, map, f)) { map = nullptr; *a.init_fail = f; }
    else if (rec.overflow) { map = nullptr; *a.init_fail = Fail{DC_UNSUPPORTED, 2}; }   // as k_actor_proofs: the list is the witness
    *a.address_map = map;
    *a.init_n = rec.n;
}

__global__ void __launch_bounds__(128) k_actor_proofs(ActorArgs a) {
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= a.n || (threadIdx.x & 31)) return;
    Recorder rec{a.rec_list + t * REC_CAP, 0, a.wbits, false};
    rec.rank_of = a.store.rank_of;
    rec.strict_only = a.strict_only != 0;
    ipcfp_actor_proof q;
    memset(&q, 0, sizeof q);   // padding included: the proofs reach the caller byte for byte
    Fail f{0, 0};
    uint64_t cb;
    if (!actor_proof_one(a, a.addrs[t], *a.address_map, *a.init_fail, rec, q, cb, f)) { report_error(a.err, ST_STORAGE, t, f.code, f.detail); a.rec_n[t] = 0; return; }
    if (rec.overflow) { report_error(a.err, ST_STORAGE, t, DC_UNSUPPORTED, 2); a.rec_n[t] = 0; return; }
    a.out[t] = q;
    a.rec_n[t] = rec.n;
    a.code_blk[t] = cb;
    a.code_len[t] = q.code_len;
}

__global__ void k_actor_code_gather(StoreView s, const uint64_t* code_blk, const uint64_t* code_off, uint64_t n, uint8_t* blob) {
    for (uint64_t t = blockIdx.x; t < n; t += gridDim.x) {
        const uint64_t b = code_blk[t];
        if (b == UINT64_MAX) continue;
        uint32_t len;
        const uint8_t* p = store_block(s, (uint32_t)b, len);
        for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) blob[code_off[t] + i] = p[i];
    }
}

// ------------------------------------------------------------------------------------------ host
uint64_t actor_request_check(const ipcfp_address* addrs, uint64_t n, const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags) {
    if (flags & ~(uint32_t)(IPCFP_WITNESS_BY_REFERENCE | IPCFP_ACTOR_WITH_CODE)) throw Error(IPCFP_ERR_INVALID_ARG, "unknown flag bit for actor proofs");
    if ((n && !addrs) || (n_evm && !evm_code_cids)) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
    if (n > IPCFP_ACTOR_MAX) throw Error(IPCFP_ERR_INVALID_ARG, "more than IPCFP_ACTOR_MAX addresses");
    uint64_t n_other = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (!address_valid(addrs[i], nullptr)) throw Error(IPCFP_ERR_INVALID_ARG, "bytes that are not an Address", i);
        n_other += addrs[i].bytes[0] != 0;
    }
    return n_other;
}

ActorUpload::ActorUpload(Store* s, const uint8_t* child_cid, const uint8_t* state_root, const ipcfp_address* addrs, uint64_t n,
                         const uint8_t* evm, uint64_t n_evm) {
    cudaStream_t st = s->stream;
    o_evm = 128;
    o_addrs = (o_evm + 38 * n_evm + 15) & ~15ull;
    const uint64_t size = o_addrs + n * sizeof(ipcfp_address) + 16;
    d.alloc(size, st);
    IPCFP_CUDA(cudaMemcpyAsync(d.p, child_cid, 38, cudaMemcpyHostToDevice, st));
    IPCFP_CUDA(cudaMemcpyAsync(d.p + 64, state_root, 38, cudaMemcpyHostToDevice, st));
    if (n_evm) IPCFP_CUDA(cudaMemcpyAsync(d.p + o_evm, evm, 38 * n_evm, cudaMemcpyHostToDevice, st));
    if (n) IPCFP_CUDA(cudaMemcpyAsync(d.p + o_addrs, addrs, n * sizeof(ipcfp_address), cudaMemcpyHostToDevice, st));
}
void ActorUpload::fill(ActorArgs& a, const StoreView& v, uint64_t n, uint64_t n_evm, uint32_t flags) const {
    a.store = v;
    a.child_cid = d.p;
    a.state_root_json = d.p + 64;
    a.evm_codes = d.p + o_evm;
    a.n_evm = n_evm;
    a.addrs = (const ipcfp_address*)(d.p + o_addrs);
    a.n = n;
    a.with_code = (flags & IPCFP_ACTOR_WITH_CODE) ? 1 : 0;
    a.strict_only = getenv("IPCFP_HAMT_STRICT") ? 1 : 0;
}

struct ActorResultBox {
    ipcfp_actor_result r;   // must stay first
    PinnedArray proofs, code;
    WitnessOut wit;
    std::vector<uint64_t> off;
    std::vector<uint32_t> idx;
};

ipcfp_actor_result* generate_actor_proofs(Store* s, TipsetDev& td, const ipcfp_address* addrs, uint64_t n, const uint8_t* evm, uint64_t n_evm,
                                          uint32_t flags) {
    const uint64_t n_other = actor_request_check(addrs, n, evm, n_evm, flags);
    if (!td.has_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    const bool by_ref = (flags & IPCFP_WITNESS_BY_REFERENCE) != 0, with_code = (flags & IPCFP_ACTOR_WITH_CODE) != 0;
    if (by_ref && !s->caller_blob)
        throw Error(IPCFP_ERR_UNSUPPORTED, "IPCFP_WITNESS_BY_REFERENCE needs a store made from a caller's blob (ipcfp_store_create)");
    s->use();
    cudaStream_t st = s->stream;
    unsigned long long* dw = s->dev_words.p;
    uint64_t* hw = s->host_words.p;
    Event ev[4];
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_BEGIN], st));
    IPCFP_CUDA(cudaMemsetAsync(dw, 0xff, 8, st));
    ActorUpload up(s, td.child_cid, td.child_state_root, addrs, n, evm, n_evm);
    AsyncBuf<ipcfp_actor_proof> d_out(n + 1, st);
    AsyncBuf<uint32_t> d_rec(n * REC_CAP + 8, st), d_recn(n + 8, st), d_init(REC_CAP + 8, st), wbits((s->n + 31) / 32 + 8, st);
    AsyncBuf<uint64_t> d_words(4, st), d_code(2 * n + 8, st);   // words: [0] address_map, [1] init Fail, [2] init list length; code: blocks, lengths
    wbits.zero();
    d_words.zero();
    ActorArgs a;
    up.fill(a, s->view, n, n_evm, flags);
    a.address_map = (const uint8_t**)d_words.p; a.init_fail = (Fail*)(d_words.p + 1); a.init_n = (uint32_t*)(d_words.p + 2);
    a.out = d_out.p; a.code_blk = d_code.p; a.code_len = d_code.p + n; a.rec_list = d_rec.p; a.rec_n = d_recn.p; a.init_list = d_init.p; a.wbits = wbits.p; a.err = dw;
    if (n_other) { k_actor_init<<<1, 32, 0, st>>>(a); IPCFP_LAUNCH_CHECK(); }
    IPCFP_CUDA(cudaEventRecord(ev[0], st));
    if (n) { k_actor_proofs<<<div_up(n * 32, 128), 128, 0, st>>>(a); IPCFP_LAUNCH_CHECK(); }
    IPCFP_CUDA(cudaEventRecord(ev[1], st));
    // host synchronisation 1: the error word and the bytecode blocks
    PinnedArray codes(s->pool, (2 * n + 1) * 8);
    IPCFP_CUDA(cudaMemcpyAsync(hw, dw, 8, cudaMemcpyDeviceToHost, st));
    if (n && with_code) IPCFP_CUDA(cudaMemcpyAsync(codes.p, d_code.p + n, n * 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (hw[DW_ERR] != IPCFP_NO_ERROR) throw_storage_error(hw[DW_ERR]);
    std::unique_ptr<ActorResultBox> box(new ActorResultBox());
    memset(&box->r, 0, sizeof box->r);
    // the code blob: bytecodes in proof order
    std::vector<uint64_t> code_off(n + 1, 0), code_len(n, 0);
    uint64_t code_bytes = 0;
    for (uint64_t i = 0; with_code && i < n; i++) {
        code_off[i] = code_bytes;
        code_len[i] = codes.as<uint64_t>()[i];
        code_bytes += code_len[i];
    }
    box->code = PinnedArray(s->pool, code_bytes + 16);
    if (code_bytes) {
        AsyncBuf<uint8_t> d_blob(code_bytes + 16, st);
        AsyncBuf<uint64_t> d_off(n + 1, st);
        IPCFP_CUDA(cudaMemcpyAsync(d_off.p, code_off.data(), 8 * n, cudaMemcpyHostToDevice, st));
        k_actor_code_gather<<<(unsigned)std::min<uint64_t>(n, 65535), 128, 0, st>>>(s->view, d_code.p, d_off.p, n, d_blob.p); IPCFP_LAUNCH_CHECK();
        IPCFP_CUDA(cudaMemcpyAsync(box->code.p, d_blob.p, code_bytes, cudaMemcpyDeviceToHost, st));
    }
    IPCFP_CUDA(cudaEventRecord(ev[2], st));
    // the proofs, the lists, the witness
    box->proofs = PinnedArray(s->pool, (n + 1) * sizeof(ipcfp_actor_proof));
    PinnedArray rec(s->pool, (n * REC_CAP + 8) * 4), recn(s->pool, (n + 8) * 4), init(s->pool, (REC_CAP + 8) * 4), words(s->pool, 32);
    if (n) {
        IPCFP_CUDA(cudaMemcpyAsync(box->proofs.p, d_out.p, n * sizeof(ipcfp_actor_proof), cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(rec.p, d_rec.p, n * REC_CAP * 4, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(recn.p, d_recn.p, n * 4, cudaMemcpyDeviceToHost, st));
    }
    IPCFP_CUDA(cudaMemcpyAsync(init.p, d_init.p, REC_CAP * 4, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaMemcpyAsync(words.p, d_words.p, 32, cudaMemcpyDeviceToHost, st));
    materialize_witness(s, wbits.p, box->wit, by_ref);
    IPCFP_CUDA(cudaEventRecord(ev[3], st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    // per-proof lists: the proof's own blocks, with the Init path's for a non-ID address, as positions in the sorted union
    const uint32_t* sorted_idx = box->wit.sorted_idx.as<uint32_t>();
    std::vector<uint32_t> pos(s->n + 1, UINT32_MAX);
    for (uint64_t i = 0; i < box->wit.n; i++) pos[sorted_idx[i]] = (uint32_t)i;
    const uint32_t n_init = n_other ? (uint32_t)words.as<uint64_t>()[2] : 0;
    ipcfp_actor_proof* proofs = box->proofs.as<ipcfp_actor_proof>();
    box->off.push_back(0);
    std::vector<uint32_t> v;
    for (uint64_t i = 0; i < n; i++) {
        v.clear();
        const uint32_t c = recn.as<uint32_t>()[i];
        for (uint32_t k = 0; k < c; k++) v.push_back(pos[rec.as<uint32_t>()[i * REC_CAP + k]]);
        if (addrs[i].bytes[0] != 0) for (uint32_t k = 0; k < n_init; k++) v.push_back(pos[init.as<uint32_t>()[k]]);
        std::sort(v.begin(), v.end());
        v.erase(std::unique(v.begin(), v.end()), v.end());
        box->idx.insert(box->idx.end(), v.begin(), v.end());
        box->off.push_back(box->idx.size());
        if (with_code) { proofs[i].code_off = code_len[i] ? code_off[i] : 0; proofs[i].code_len = code_len[i]; }
    }
    ipcfp_actor_result& r = box->r;
    r.n_proofs = n;
    r.proofs = proofs;
    box->wit.fill(r.witness);
    r.proof_witness_offsets = box->off.data();
    r.proof_witness_index = box->idx.data();
    r.code_blob = box->code.as<uint8_t>();
    r.code_blob_size = code_bytes;
    r.ms_total = elapsed_ms(s->ev[EV_BEGIN], ev[3]);
    r.ms_init = elapsed_ms(s->ev[EV_BEGIN], ev[0]);
    r.ms_walk = elapsed_ms(ev[0], ev[1]);
    r.ms_code = elapsed_ms(ev[1], ev[2]);
    r.ms_witness = elapsed_ms(ev[2], ev[3]);
    r.host_syncs = 4;   // the error word, materialize_witness's two (witness count, witness copy), the end
    return &box.release()->r;
}
void actor_result_free(ipcfp_actor_result* r) { delete reinterpret_cast<ActorResultBox*>(r); }

}  // namespace ipcfp
