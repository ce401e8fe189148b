// verify.cu — GPU-batched verifiers over a WITNESS store (SURVEY §8 f-2).
//
//   verify_event_proofs     reference src/proofs/events/verifier.rs:51-290  (verify_event_proof → verify_single_proof per proof)
//   verify_storage_proofs   reference src/proofs/storage/verifier.rs:24-170 (verify_storage_proof per proof)
//
// The witness blocks go into an ipcfp_store first (ipcfp_store_create with IPCFP_STORE_VERIFY_CIDS): that is the Blake2b-256 check of
// EVERY witness block which the reference's load_witness_store leaves out (`put_keyed`, events/verifier.rs:79-89 — SURVEY F6).
// What the reference repeats per proof but depends on the tipset only is done once per call: header consistency (:147-181), the
// TxMeta recompute and the execution order (events/utils.rs:16-30, :64-73 — O(messages) PER PROOF in the reference). Then one warp
// per proof (lane 0 walks, see storage.cu for why) replays verify_execution_order (:184-204: exec[exec_index] == message_cid, which
// for a duplicate-free list is `position(message_cid) == exec_index`), Amtv0<Receipt>.get(exec_index) → events_root →
// Amt<StampedEvent>.get(event_index) (:207-254) and verify_event_data_matches (:257-290).
// Results are the reference's Vec<bool>; an Err of the reference (missing block, decode failure, TxMeta mismatch) fails the call
// with the index of the FIRST proof that meets it. Trust anchors (:124-144) are host-side policy closures and stay with the caller.
#include <algorithm>
#include <cstring>

#include "verify_items.cuh"   // the per-item device code (also compiled for the host by tests/host_fuzz/emu_verify.cu)

namespace ipcfp {

// once per call, one thread (verify_tipset_item)
__global__ void k_verify_tipset(VerifyTipsetArgs a) {
    if (threadIdx.x || blockIdx.x) return;
    verify_tipset_item(a);
}
__global__ void k_verify_txmeta(StoreView s, const uint8_t* txmeta_cids, uint32_t n_parents, unsigned long long* err) {
    uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_parents) return;
    verify_txmeta_item(s, txmeta_cids, k, err);
}
// one warp per proof, lane 0 walks (see storage.cu for why)
__global__ void __launch_bounds__(128) k_verify_events(VerifyEventArgs a) {
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= a.n || (threadIdx.x & 31)) return;
    verify_event_item(a, t);
}

static void throw_verify_error(uint64_t key) {
    const uint32_t code = (uint32_t)(key >> 8) & 0xff, detail = (uint32_t)key & 0xff;
    const uint64_t index = (key >> 16) & 0xFFFFFFFFFFull;
    switch (code) {
        case DC_MISSING: throw Error(IPCFP_ERR_MISSING_BLOCK, "missing block in the witness (detail " + std::to_string(detail) + ")", index);
        case DC_CID_MISMATCH: throw Error(IPCFP_ERR_CID_MISMATCH, "TxMeta mismatch: header vs recomputed (parent " + std::to_string(detail) + ")", index);
        case DC_ACTOR_NOT_FOUND: throw Error(IPCFP_ERR_ACTOR_NOT_FOUND, "actor not found", index);
        default: throw Error(IPCFP_ERR_DECODE, "decode error in the witness (detail " + std::to_string(detail) + ")", index);
    }
}

void verify_event_proofs(Store* s, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs, uint64_t n, const uint8_t* data_blob, uint64_t blob_size,
                         const ipcfp_event_spec* filter, uint8_t* results) {
    s->use();
    if (!t || !t->child_cid || (t->n_parents && !t->parent_cids)) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor has null fields");
    if (t->n_parents > 64) throw Error(IPCFP_ERR_UNSUPPORTED, "too many parent blocks");
    if (n && (!proofs || !results)) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
    if (n == 0) return;
    cudaStream_t st = s->stream;
    AsyncBuf<uint8_t> d_blob(blob_size + 16, st);
    AsyncBuf<ipcfp_event_proof> d_proofs(n, st);
    IPCFP_CUDA(cudaMemcpyAsync(d_proofs.p, proofs, n * sizeof(ipcfp_event_proof), cudaMemcpyHostToDevice, st));
    if (blob_size) IPCFP_CUDA(cudaMemcpyAsync(d_blob.p, data_blob, blob_size, cudaMemcpyHostToDevice, st));
    verify_event_proofs_dev(s, t, d_proofs.p, n, d_blob.p, blob_size, filter, results);
}

// the proofs and their data blob (blob_size bytes + 16 of padding) already on the device, on the store's device
void verify_event_proofs_dev(Store* s, const ipcfp_tipset_desc* t, const ipcfp_event_proof* d_proofs, uint64_t n, const uint8_t* d_blob, uint64_t blob_size,
                             const ipcfp_event_spec* filter, uint8_t* results) {
    if (!t || !t->child_cid || (t->n_parents && !t->parent_cids)) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor has null fields");
    if (t->n_parents > 64) throw Error(IPCFP_ERR_UNSUPPORTED, "too many parent blocks");
    if (n == 0) return;
    cudaStream_t st = s->stream;
    unsigned long long* dw = s->dev_words.p;
    uint64_t* hw = s->host_words.p;
    const uint32_t P = t->n_parents;
    IPCFP_CUDA(cudaMemsetAsync(dw, 0xff, 8, st));
    AsyncBuf<uint8_t> d_cids(38ull * (2 * P + 2) + 64, st), d_res(n + 16, st);
    AsyncBuf<uint32_t> d_flags(8, st);
    IPCFP_CUDA(cudaMemcpyAsync(d_cids.p, t->child_cid, 38, cudaMemcpyHostToDevice, st));
    if (P) IPCFP_CUDA(cudaMemcpyAsync(d_cids.p + 38, t->parent_cids, 38ull * P, cudaMemcpyHostToDevice, st));
    uint8_t* d_tx = d_cids.p + 38ull * (P + 1);
    VerifyTipsetArgs ta;
    ta.store = s->view; ta.parent_cids = d_cids.p + 38; ta.child_cid = d_cids.p; ta.n_parents = P;
    ta.parent_epoch = t->parent_epoch; ta.child_epoch = t->child_epoch;
    ta.consistent = d_flags.p; ta.receipts_root_blk = d_flags.p + 1; ta.txmeta_cids = d_tx; ta.err = dw;
    k_verify_tipset<<<1, 32, 0, st>>>(ta); IPCFP_LAUNCH_CHECK();
    std::vector<uint8_t> h_tx(38ull * P + 8);
    uint32_t h_flags[2] = {0, 0};
    if (P) IPCFP_CUDA(cudaMemcpyAsync(h_tx.data(), d_tx, 38ull * P, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaMemcpyAsync(h_flags, d_flags.p, 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaMemcpyAsync(hw, dw, 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (hw[DW_ERR] != IPCFP_NO_ERROR) throw_verify_error(hw[DW_ERR]);
    ExecOrderOut exo;
    if (h_flags[0]) {
        // collect_exec_list(verify_txmeta = true) once for the whole batch: TxMeta recompute, then the engine's own message-AMT walk
        // + first-seen dedup (the same kernels generate_event_proof uses), on the TxMeta links taken from the parent HEADERS
        k_verify_txmeta<<<div_up(P, 64), 64, 0, st>>>(s->view, d_tx, P, dw); IPCFP_LAUNCH_CHECK();
        TipsetDev td;
        td.parent_epoch = t->parent_epoch; td.child_epoch = t->child_epoch; td.n_parents = P;
        td.parent_cids.assign(t->parent_cids, t->parent_cids + 38ull * P);
        td.txmeta_cids.assign(h_tx.begin(), h_tx.begin() + 38ull * P);
        memcpy(td.child_cid, t->child_cid, 38);
        memcpy(td.receipts_root, t->child_cid, 38);   // unused in execution-order-only mode (any CID of the store)
        td.n_receipts = 0;
        td.events_roots.alloc(64);
        td.has_root.alloc(64);
        ipcfp_event_spec dummy;
        memset(&dummy, 0, sizeof dummy);
        dummy.event_signature = "";
        dummy.topic_1 = "";
        IPCFP_CUDA(cudaMemcpyAsync(hw + HW_PARKED_KEY, dw, 8, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
        const uint64_t tx_key = hw[HW_PARKED_KEY];
        try {
            (void)generate_event_proof(s, td, &dummy, IPCFP_SCAN_SKIP_TX_AMTS, false, 0, 0, nullptr, &exo);
        } catch (Error& e) {
            // collect_exec_list takes the parents in order and checks parent k's TxMeta CID before it walks parent k's two message AMTs.
            // The walk's fault key names the parent it met (eidx / 3: its TxMeta, BLS or SECP AMT); a mismatching TxMeta of an earlier
            // parent, or of the same one (its TxMeta loaded and decoded, so the fault is in one of its AMTs), is met first.
            if (tx_key != IPCFP_NO_ERROR) {
                IPCFP_CUDA(cudaMemcpyAsync(hw + DW_TX_ERR, dw + DW_TX_ERR, 8, cudaMemcpyDeviceToHost, st));
                IPCFP_CUDA(cudaStreamSynchronize(st));
                const uint64_t walk_key = hw[DW_TX_ERR];
                const uint32_t eidx = (uint32_t)(walk_key >> 56);
                if (walk_key == IPCFP_NO_ERROR || eidx == IPCFP_TX_EIDX_NONE || (uint32_t)(tx_key & 0xff) <= eidx / 3) throw_verify_error(tx_key);
            }
            e.index = 0;   // failures of the walk surface at the first proof, like everything that depends on the tipset only
            throw;
        }
        if (tx_key != IPCFP_NO_ERROR) throw_verify_error(tx_key);
        IPCFP_CUDA(cudaMemsetAsync(dw, 0xff, 8, st));
    }
    AsyncBuf<Matcher> d_filter;
    if (filter) {
        if (!filter->event_signature || !filter->topic_1) throw Error(IPCFP_ERR_INVALID_ARG, "filter spec has null fields");
        Matcher m;
        memset(&m, 0, sizeof m);
        // keccak256(signature) on the device through the batched-hash entry (K2)
        uint8_t t0[32];
        uint64_t off0 = 0;
        uint32_t len0 = (uint32_t)strlen(filter->event_signature);
        hash_batch(1, (const uint8_t*)filter->event_signature, len0, &off0, &len0, 1, s->device, t0);
        memcpy(m.t0, t0, 32);
        uint8_t t1[32];
        memset(t1, 0, 32);
        size_t n1 = strlen(filter->topic_1);
        memcpy(t1, filter->topic_1, n1 < 32 ? n1 : 32);
        memcpy(m.t1, t1, 32);
        d_filter.alloc(1, st);
        IPCFP_CUDA(cudaMemcpyAsync(d_filter.p, &m, sizeof m, cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaStreamSynchronize(st));   // m is a stack object
    }
    VerifyEventArgs va;
    va.store = s->view; va.proofs = d_proofs; va.n = n; va.blob = d_blob; va.blob_size = blob_size;
    va.consistent = d_flags.p; va.receipts_root_blk = d_flags.p + 1;
    va.exec_raw = exo.exec_raw.p; va.exec_idx = exo.exec_idx.p; va.n_exec = exo.n_exec;
    va.filter = filter ? d_filter.p : nullptr; va.results = d_res.p; va.err = dw;
    k_verify_events<<<div_up(n * 32, 128), 128, 0, st>>>(va); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaMemcpyAsync(results, d_res.p, n, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaMemcpyAsync(hw, dw, 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (hw[DW_ERR] != IPCFP_NO_ERROR) throw_verify_error(hw[DW_ERR]);
}

// ------------------------------------------------------------------------------------------ storage
__global__ void __launch_bounds__(128) k_verify_storage(VerifyStorageArgs a) {
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= a.n || (threadIdx.x & 31)) return;
    verify_storage_item(a, t);
}

void verify_storage_proofs(Store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs, uint64_t n, uint8_t* results) {
    s->use();
    if (!t || !t->child_cid || !t->child_parent_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    if (n && (!proofs || !results)) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
    if (n == 0) return;
    cudaStream_t st = s->stream;
    AsyncBuf<ipcfp_storage_proof> d_proofs(n, st);
    IPCFP_CUDA(cudaMemcpyAsync(d_proofs.p, proofs, n * sizeof(ipcfp_storage_proof), cudaMemcpyHostToDevice, st));
    verify_storage_proofs_dev(s, t, d_proofs.p, n, results);
}

// the proofs already on the device, on the store's device
void verify_storage_proofs_dev(Store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* d_proofs, uint64_t n, uint8_t* results) {
    if (!t || !t->child_cid || !t->child_parent_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    if (n == 0) return;
    cudaStream_t st = s->stream;
    unsigned long long* dw = s->dev_words.p;
    uint64_t* hw = s->host_words.p;
    IPCFP_CUDA(cudaMemsetAsync(dw, 0xff, 8, st));
    AsyncBuf<uint8_t> d_in(128, st), d_res(n + 16, st);
    IPCFP_CUDA(cudaMemcpyAsync(d_in.p, t->child_cid, 38, cudaMemcpyHostToDevice, st));
    IPCFP_CUDA(cudaMemcpyAsync(d_in.p + 64, t->child_parent_state_root, 38, cudaMemcpyHostToDevice, st));
    VerifyStorageArgs a;
    a.store = s->view; a.child_cid = d_in.p; a.state_root_json = d_in.p + 64; a.proofs = d_proofs; a.n = n; a.results = d_res.p; a.err = dw;
    k_verify_storage<<<div_up(n * 32, 128), 128, 0, st>>>(a); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaMemcpyAsync(results, d_res.p, n, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaMemcpyAsync(hw, dw, 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    if (hw[DW_ERR] != IPCFP_NO_ERROR) throw_verify_error(hw[DW_ERR]);
}

}  // namespace ipcfp
