// storage.cu — K5: HAMT storage-slot lookups and storage-proof generation on the GPU.
//
// One thread runs the whole dependent chain of one proof / one lookup with device-side
// Blockstore::get (hash probe) and a device-side recorder:
//   reference src/proofs/storage/generator.rs:29-178  generate_storage_proof
//   reference src/proofs/storage/decode.rs:36-97      read_storage_slot (shape sniffing A1,A2,A3,B1,B2,C)
//   reference src/proofs/common/decode.rs:17-124      get_actor_state, parse_evm_state, HeaderLite
//   fvm_ipld_hamt 0.10 [UPSTREAM]                     Hamt::get with SHA-256 key hashing (K2b)
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>

#include "engine.cuh"
#include "hashes.cuh"
#include "ipld.cuh"
#include "prims.cuh"
#include "storage.cuh"

namespace ipcfp {

// One WARP per proof / lookup, lane 0 walks. The walk is a chain of data-dependent branches over a different node in every lane:
// 32 lookups in one warp execute close to one lane at a time (the kernel time hardly depends on the batch size), so a lookup per warp
// costs the same issue slots, finishes 32 lookups' worth earlier and spreads a small batch over all SMs.
__global__ void __launch_bounds__(128) k_storage_proofs(StorageArgs a) {
    uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= a.n || (threadIdx.x & 31)) return;
    Recorder rec{a.rec_list + t * REC_CAP, 0, a.wbits, false};
    rec.rank_of = a.store.rank_of;
    ipcfp_storage_proof q;
    memset(&q, 0, sizeof q);   // the 4 bytes of tail padding too: the proofs reach the caller byte for byte (raw_proofs, the verifiers)
    Fail f{0, 0};
    if (!storage_proof_one(a, t, rec, q, f)) { report_error(a.err, ST_STORAGE, t, f.code, f.detail); a.rec_n[t] = 0; return; }
    if (rec.overflow) { report_error(a.err, ST_STORAGE, t, DC_UNSUPPORTED, 2); a.rec_n[t] = 0; return; }
    a.out[t] = q;
    a.rec_n[t] = rec.n;
}

struct SlotArgs {
    StoreView store;
    const uint8_t* root_cid;
    const uint8_t* slots;
    uint64_t n;
    uint8_t* found; uint32_t* raw_len; uint8_t* values;
    uint32_t* wbits;
    unsigned long long* err;
    unsigned long long* stats;   // [0] HAMT nodes decoded, [1] their bytes
    uint32_t strict_only;
    uint32_t per_warp;
};
// a.per_warp: one lookup per warp (small and medium batches: latency); else one per thread with the strict decoder, whose uniform
// head-by-head loop keeps the lanes of a warp closer together (large batches, where the grid fills the GPU either way)
__global__ void __launch_bounds__(128) k_read_slots(SlotArgs a) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a.per_warp) { if (threadIdx.x & 31) return; t >>= 5; }
    if (t >= a.n) return;
    Recorder rec{nullptr, 0, a.wbits, false};
    rec.rank_of = a.store.rank_of;
    rec.strict_only = a.strict_only != 0;
    SlotValue sv;
    Fail f{0, 0};
    const bool ok = read_storage_slot(a.store, rec, a.root_cid, a.slots + 32 * t, sv, f);
    atomicAdd(a.stats, (unsigned long long)rec.hamt_nodes);
    atomicAdd(a.stats + 1, (unsigned long long)rec.hamt_bytes);
    if (!ok) { report_error(a.err, ST_STORAGE, t, f.code, f.detail); return; }
    a.found[t] = sv.found;
    a.raw_len[t] = sv.raw_len;
    for (int i = 0; i < 32; i++) a.values[32 * t + i] = sv.v32[i];
}

// ------------------------------------------------------------------------------------------ host
void throw_storage_error(uint64_t key) {
    uint32_t code = (uint32_t)(key >> 8) & 0xff, detail = (uint32_t)key & 0xff;
    uint64_t index = (key >> 16) & 0xFFFFFFFFFFull;
    switch (code) {
        case DC_MISSING: throw Error(IPCFP_ERR_MISSING_BLOCK, "missing block on the storage path (detail " + std::to_string(detail) + ")", index);
        case DC_STATE_MISMATCH: throw Error(IPCFP_ERR_STATE_ROOT_MISMATCH, "ParentStateRoot mismatch: header vs JSON", index);
        case DC_ACTOR_NOT_FOUND: throw Error(IPCFP_ERR_ACTOR_NOT_FOUND, "actor not found", index);
        case DC_UNSUPPORTED: throw Error(IPCFP_ERR_UNSUPPORTED, "recorder overflow", index);
        default: throw Error(IPCFP_ERR_DECODE, "decode error on the storage path (detail " + std::to_string(detail) + ")", index);
    }
}

struct SlotResultBox {
    ipcfp_slot_result r;
    PinnedArray found, raw_len, values;
    WitnessOut wit;
};
ipcfp_slot_result* read_storage_slots(Store* s, const uint8_t* root, const uint8_t* slots, uint64_t k) {
    s->use();
    cudaStream_t st = s->stream;
    unsigned long long* dw = s->dev_words.p;
    uint64_t* hw = s->host_words.p;
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_BEGIN], st));
    IPCFP_CUDA(cudaMemsetAsync(dw, 0xff, 8, st));
    AsyncBuf<uint8_t> d_in(64 + 32 * k, st), d_found(k + 8, st), d_vals(32 * k + 32, st);
    AsyncBuf<uint32_t> d_len(k + 8, st), wbits((s->n + 31) / 32 + 8, st);
    wbits.zero();
    IPCFP_CUDA(cudaMemsetAsync(d_found.p, 0, k + 8, st));
    IPCFP_CUDA(cudaMemsetAsync(d_len.p, 0, (k + 8) * 4, st));
    IPCFP_CUDA(cudaMemsetAsync(d_vals.p, 0, 32 * k + 32, st));
    IPCFP_CUDA(cudaMemcpyAsync(d_in.p, root, 38, cudaMemcpyHostToDevice, st));
    if (k) IPCFP_CUDA(cudaMemcpyAsync(d_in.p + 64, slots, 32 * k, cudaMemcpyHostToDevice, st));
    SlotArgs a;
    a.store = s->view; a.root_cid = d_in.p; a.slots = d_in.p + 64; a.n = k; a.found = d_found.p; a.raw_len = d_len.p; a.values = d_vals.p;
    a.wbits = wbits.p; a.err = dw; a.stats = dw + DW_STATS; a.strict_only = getenv("IPCFP_HAMT_STRICT") ? 1 : 0;
    IPCFP_CUDA(cudaMemsetAsync(dw + DW_STATS, 0, 16, st));
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_LOOKUP_BEGIN], st));
    a.per_warp = k <= 16384 ? 1 : 0;
    if (!a.per_warp) a.strict_only = 1;
    if (k) { k_read_slots<<<div_up(a.per_warp ? k * 32 : k, 128), 128, 0, st>>>(a); IPCFP_LAUNCH_CHECK(); }
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_LOOKUP_END], st));
    IPCFP_CUDA(cudaMemcpyAsync(hw, dw, 6 * 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (hw[DW_ERR] != IPCFP_NO_ERROR) throw_storage_error(hw[DW_ERR]);
    const uint64_t stat_nodes = hw[DW_STATS], stat_bytes = hw[DW_STATS + 1];
    std::unique_ptr<SlotResultBox> box(new SlotResultBox());
    memset(&box->r, 0, sizeof box->r);
    box->found = PinnedArray(s->pool, k + 8);
    box->raw_len = PinnedArray(s->pool, (k + 8) * 4);
    box->values = PinnedArray(s->pool, 32 * k + 32);
    if (k) {
        IPCFP_CUDA(cudaMemcpyAsync(box->found.p, d_found.p, k, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(box->raw_len.p, d_len.p, k * 4, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(box->values.p, d_vals.p, k * 32, cudaMemcpyDeviceToHost, st));
    }
    materialize_witness(s, wbits.p, box->wit);
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_STORAGE_END], st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    box->r.n = k; box->r.found = box->found.as<uint8_t>(); box->r.raw_len = box->raw_len.as<uint32_t>(); box->r.values = box->values.as<uint8_t>();
    box->wit.fill(box->r.witness);
    float ms;
    IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_BEGIN], s->ev[EV_STORAGE_END]));
    box->r.ms_total = ms;
    IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_LOOKUP_BEGIN], s->ev[EV_LOOKUP_END]));
    box->r.ms_lookup = ms;
    box->r.lookup_nodes = stat_nodes;
    box->r.lookup_bytes = stat_bytes + 32 * k;
    return &box.release()->r;
}
void slot_result_free(ipcfp_slot_result* r) { delete reinterpret_cast<SlotResultBox*>(r); }

struct StorageResultBox {
    ipcfp_storage_result r;
    PinnedArray proofs;
    WitnessOut wit;
    std::vector<uint64_t> spec_off;
    std::vector<uint32_t> spec_idx;
};
ipcfp_storage_result* generate_storage_proofs(Store* s, const uint8_t* child_cid, const uint8_t* state_root, const ipcfp_storage_spec* specs, uint64_t n,
                                              bool by_ref) {
    s->use();
    if (!child_cid || !state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    if (n && !specs) throw Error(IPCFP_ERR_INVALID_ARG, "null specs");
    cudaStream_t st = s->stream;
    unsigned long long* dw = s->dev_words.p;
    uint64_t* hw = s->host_words.p;
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_BEGIN], st));
    IPCFP_CUDA(cudaMemsetAsync(dw, 0xff, 8, st));
    AsyncBuf<uint8_t> d_in(128, st);
    AsyncBuf<ipcfp_storage_spec> d_specs(n + 1, st);
    AsyncBuf<ipcfp_storage_proof> d_out(n + 1, st);
    AsyncBuf<uint32_t> d_rec(n * REC_CAP + 8, st), d_recn(n + 8, st), wbits((s->n + 31) / 32 + 8, st);
    wbits.zero();
    IPCFP_CUDA(cudaMemcpyAsync(d_in.p, child_cid, 38, cudaMemcpyHostToDevice, st));
    IPCFP_CUDA(cudaMemcpyAsync(d_in.p + 64, state_root, 38, cudaMemcpyHostToDevice, st));
    if (n) IPCFP_CUDA(cudaMemcpyAsync(d_specs.p, specs, n * sizeof(ipcfp_storage_spec), cudaMemcpyHostToDevice, st));
    StorageArgs a;
    a.store = s->view; a.child_cid = d_in.p; a.state_root_json = d_in.p + 64; a.specs = d_specs.p; a.n = n; a.out = d_out.p;
    a.rec_list = d_rec.p; a.rec_n = d_recn.p; a.wbits = wbits.p; a.err = dw;
    if (n) { k_storage_proofs<<<div_up(n * 32, 128), 128, 0, st>>>(a); IPCFP_LAUNCH_CHECK(); }
    IPCFP_CUDA(cudaMemcpyAsync(hw, dw, 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (hw[DW_ERR] != IPCFP_NO_ERROR) throw_storage_error(hw[DW_ERR]);
    return storage_result_finish(s, d_out.p, d_rec.p, d_recn.p, wbits.p, n, by_ref);
}
// The result of n proofs on the device in spec order, with their recorder lists and the witness bitmap they marked: the proofs copied
// back, the witness materialised, the per-spec lists. Timed from s->ev[EV_BEGIN].
ipcfp_storage_result* storage_result_finish(Store* s, const ipcfp_storage_proof* d_out, const uint32_t* d_rec, const uint32_t* d_recn, const uint32_t* wbits,
                                            uint64_t n, bool by_ref) {
    cudaStream_t st = s->stream;
    std::unique_ptr<StorageResultBox> box(new StorageResultBox());
    memset(&box->r, 0, sizeof box->r);
    box->proofs = PinnedArray(s->pool, (n + 1) * sizeof(ipcfp_storage_proof));
    PinnedArray rec(s->pool, (n * REC_CAP + 8) * 4), recn(s->pool, (n + 8) * 4);
    if (n) {
        IPCFP_CUDA(cudaMemcpyAsync(box->proofs.p, d_out, n * sizeof(ipcfp_storage_proof), cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(rec.p, d_rec, n * REC_CAP * 4, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaMemcpyAsync(recn.p, d_recn, n * 4, cudaMemcpyDeviceToHost, st));
    }
    materialize_witness(s, wbits, box->wit, by_ref);
    // per-spec Vec<ProofBlock>: map recorded block indices to positions in the sorted union
    PinnedArray& sorted_idx = box->wit.sorted_idx;
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_STORAGE_END], st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    std::map<uint32_t, uint32_t> pos;
    for (uint64_t i = 0; i < box->wit.n; i++) pos[sorted_idx.as<uint32_t>()[i]] = (uint32_t)i;
    box->spec_off.push_back(0);
    for (uint64_t i = 0; i < n; i++) {
        uint32_t c = recn.as<uint32_t>()[i];
        std::vector<uint32_t> v;
        for (uint32_t k = 0; k < c; k++) v.push_back(pos[rec.as<uint32_t>()[i * REC_CAP + k]]);
        std::sort(v.begin(), v.end());
        box->spec_idx.insert(box->spec_idx.end(), v.begin(), v.end());
        box->spec_off.push_back(box->spec_idx.size());
    }
    box->r.n_proofs = n; box->r.proofs = box->proofs.as<ipcfp_storage_proof>();
    box->wit.fill(box->r.witness);
    box->r.spec_witness_offsets = box->spec_off.data();
    box->r.spec_witness_index = box->spec_idx.data();
    float ms;
    IPCFP_CUDA(cudaEventElapsedTime(&ms, s->ev[EV_BEGIN], s->ev[EV_STORAGE_END]));
    box->r.ms_total = ms;
    return &box.release()->r;
}
void storage_result_free(ipcfp_storage_result* r) { delete reinterpret_cast<StorageResultBox*>(r); }
const WitnessOut& storage_result_witness(const ipcfp_storage_result* r) { return reinterpret_cast<const StorageResultBox*>(r)->wit; }

}  // namespace ipcfp
