// message_proof.cu — ipcfp_generate_message_proofs_resident: whether a message executed and how it ended (DESIGN.md §2, "Message
// proofs"). Per-request code: message_proof_items.cuh.
//   message_positions      (events.cu) the execution order with its witness bitmap (ExecOrderBuild) and each request's position in it
//                          (MsgRequests::select)
//   k_message_proofs       one request per warp, lane 0 walks (the shape of k_actor_proofs): Amtv0<Receipt>::get(position), and with
//                          IPCFP_MESSAGE_WITH_BODY the message block
//   k_message_data_gather  one CTA per proof copies its return data, then its params, into the data blob
// Every block the walks read is marked in the execution order's witness bitmap, materialised once as the call's witness.
// Host synchronisations: five when the message AMTs take the dense walk (the general walk adds its own, see EventCall) — the walk's, the
// error word with the data lengths, materialize_witness's two (witness count, witness copy), the end.
#include <algorithm>
#include <cstring>
#include <memory>

#include "engine.cuh"
#include "message_proof_items.cuh"

namespace ipcfp {

__global__ void __launch_bounds__(128) k_message_proofs(MsgProofArgs a) {
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= a.n || (threadIdx.x & 31)) return;
    ipcfp_message_proof q;
    memset(&q, 0, sizeof q);   // padding included: the proofs reach the caller byte for byte
    const uint8_t *ret, *par;
    Fail f{0, 0};
    if (!message_proof_one(a, t, q, ret, par, f)) { report_error(a.err, ST_STORAGE, t, f.code, f.detail); return; }
    a.out[t] = q;
    a.src[t] = ret; a.src[a.n + t] = par;
    a.len[t] = q.return_len; a.len[a.n + t] = q.params_len;
}

// per proof t: its return data at blob[off[t]], its params right behind
__global__ void k_message_data_gather(const uint8_t* const* src, const uint64_t* len, const uint64_t* off, uint64_t n, uint8_t* blob) {
    for (uint64_t t = blockIdx.x; t < n; t += gridDim.x) {
        uint8_t* o = blob + off[t];
        for (int k = 0; k < 2; k++) {
            const uint8_t* p = src[k * n + t];
            const uint64_t l = len[k * n + t];
            for (uint64_t i = threadIdx.x; i < l; i += blockDim.x) o[i] = p[i];
            o += l;
        }
    }
}

// ------------------------------------------------------------------------------------------ host
void message_proof_check(const uint8_t* message_cids, uint64_t n, uint32_t flags) {
    if (flags & ~(uint32_t)(IPCFP_WITNESS_BY_REFERENCE | IPCFP_MESSAGE_WITH_BODY)) throw Error(IPCFP_ERR_INVALID_ARG, "unknown flag bit for message proofs");
    if (n && !message_cids) throw Error(IPCFP_ERR_INVALID_ARG, "null message CIDs with a nonzero count");
    if (n > IPCFP_MESSAGE_MAX) throw Error(IPCFP_ERR_INVALID_ARG, "more message CIDs than IPCFP_MESSAGE_MAX");
}

[[noreturn]] static void throw_request_error(uint64_t key) {
    const uint32_t code = (uint32_t)(key >> 8) & 0xff, detail = (uint32_t)key & 0xff;
    const uint64_t index = (key >> 16) & 0xFFFFFFFFFFull;
    if (code == DC_MISSING) throw Error(IPCFP_ERR_MISSING_BLOCK, "missing block on a message proof's path (detail " + std::to_string(detail) + ")", index);
    throw Error(IPCFP_ERR_DECODE, "decode error on a message proof's path (detail " + std::to_string(detail) + ")", index);
}

struct MessageResultBox {
    ipcfp_message_result r;   // must stay first
    PinnedArray proofs, blob;
    WitnessOut wit;
};

ipcfp_message_result* generate_message_proofs(Store* s, TipsetDev& td, const uint8_t* cids, uint64_t n, uint32_t flags) {
    message_proof_check(cids, n, flags);
    const bool by_ref = (flags & IPCFP_WITNESS_BY_REFERENCE) != 0;
    if (by_ref && !s->caller_blob)
        throw Error(IPCFP_ERR_UNSUPPORTED, "IPCFP_WITNESS_BY_REFERENCE needs a store made from a caller's blob (ipcfp_store_create)");
    s->use();
    cudaStream_t st = s->stream;
    unsigned long long* dw = s->dev_words.p;
    uint64_t* hw = s->host_words.p;
    // host synchronisation 1 is the walk's; message-AMT and receipts-root faults are thrown there
    MessagePositions mp;
    message_positions(s, td, cids, n, flags, mp);
    Event ev[3];
    AsyncBuf<uint8_t> d_cids(38 * n + 16, st);
    if (n) IPCFP_CUDA(cudaMemcpyAsync(d_cids.p, cids, 38 * n, cudaMemcpyHostToDevice, st));
    AsyncBuf<ipcfp_message_proof> d_out(n + 1, st);
    AsyncBuf<const uint8_t*> d_src(2 * n + 8, st);
    AsyncBuf<uint64_t> d_len(2 * n + 8, st);
    MsgProofArgs a;
    a.store = s->view; a.cids = d_cids.p; a.exec_indices = mp.exec_indices.p; a.n = n; a.receipts_root_blk = mp.receipts_root_blk;
    a.with_body = (flags & IPCFP_MESSAGE_WITH_BODY) ? 1 : 0;
    a.out = d_out.p; a.src = d_src.p; a.len = d_len.p; a.wbits = mp.wbits.p; a.err = dw + DW_ERR;
    if (n) { k_message_proofs<<<div_up(n * 32, 128), 128, 0, st>>>(a); IPCFP_LAUNCH_CHECK(); }
    IPCFP_CUDA(cudaEventRecord(ev[0], st));
    // host synchronisation 2: the error word and the data lengths
    PinnedArray lens(s->pool, (2 * n + 1) * 8);
    IPCFP_CUDA(cudaMemcpyAsync(hw, dw, 8, cudaMemcpyDeviceToHost, st));
    if (n) IPCFP_CUDA(cudaMemcpyAsync(lens.p, d_len.p, 2 * n * 8, cudaMemcpyDeviceToHost, st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    const uint64_t n_exec = hw[DW_N_EXEC];
    if (hw[DW_ERR] != IPCFP_NO_ERROR) throw_request_error(hw[DW_ERR]);
    if (mp.missing_base) throw Error(IPCFP_ERR_MISSING_BLOCK, "missing block (base witness CID not in the store)");
    std::unique_ptr<MessageResultBox> box(new MessageResultBox());
    memset(&box->r, 0, sizeof box->r);
    // the data blob: per proof its return data, then its params (an exclusive scan over the proofs)
    const uint64_t* ln = lens.as<uint64_t>();
    PinnedArray offs(s->pool, (n + 1) * 8);
    uint64_t* off = offs.as<uint64_t>();
    uint64_t bytes = 0;
    for (uint64_t i = 0; i < n; i++) { off[i] = bytes; bytes += ln[i] + ln[n + i]; }
    box->blob = PinnedArray(s->pool, bytes + 16);
    if (bytes) {
        AsyncBuf<uint8_t> d_blob(bytes + 16, st);
        AsyncBuf<uint64_t> d_off(n + 1, st);
        IPCFP_CUDA(cudaMemcpyAsync(d_off.p, off, 8 * n, cudaMemcpyHostToDevice, st));
        k_message_data_gather<<<(unsigned)std::min<uint64_t>(n, 65535), 128, 0, st>>>(d_src.p, d_len.p, d_off.p, n, d_blob.p); IPCFP_LAUNCH_CHECK();
        IPCFP_CUDA(cudaMemcpyAsync(box->blob.p, d_blob.p, bytes, cudaMemcpyDeviceToHost, st));
    }
    IPCFP_CUDA(cudaEventRecord(ev[1], st));
    box->proofs = PinnedArray(s->pool, (n + 1) * sizeof(ipcfp_message_proof));
    if (n) IPCFP_CUDA(cudaMemcpyAsync(box->proofs.p, d_out.p, n * sizeof(ipcfp_message_proof), cudaMemcpyDeviceToHost, st));
    // host synchronisations 3 and 4
    materialize_witness(s, mp.wbits.p, box->wit, by_ref);
    IPCFP_CUDA(cudaEventRecord(ev[2], st));
    IPCFP_CUDA(cudaStreamSynchronize(st));   // 5
    ipcfp_message_proof* proofs = box->proofs.as<ipcfp_message_proof>();
    for (uint64_t i = 0; i < n; i++) {
        proofs[i].return_off = proofs[i].return_len ? off[i] : 0;
        proofs[i].params_off = proofs[i].params_len ? off[i] + proofs[i].return_len : 0;
    }
    ipcfp_message_result& r = box->r;
    r.n_proofs = n;
    r.proofs = proofs;
    r.data_blob = box->blob.as<uint8_t>();
    r.data_blob_size = bytes;
    box->wit.fill(r.witness);
    r.n_exec = n_exec;
    r.ms_total = elapsed_ms(s->ev[EV_BEGIN], ev[2]);
    r.ms_exec_order = elapsed_ms(s->ev[EV_BEGIN], s->ev[EV_EXEC_ORDER]);
    r.ms_walk = elapsed_ms(s->ev[EV_EXEC_ORDER], ev[0]);
    r.ms_gather = elapsed_ms(ev[0], ev[1]);
    r.ms_witness = elapsed_ms(ev[1], ev[2]);
    r.host_syncs = 5;
    return &box.release()->r;
}
void message_result_free(ipcfp_message_result* r) { delete reinterpret_cast<MessageResultBox*>(r); }

}  // namespace ipcfp
