// json.cu — IPCFP_RESULT_JSON: the EventProofBundle of a generate_event_proof call rendered on the device, byte for byte what
// ipcfp_event_result_to_json (csrc/bundle_json.cpp) renders from the POD result on the host. Everything the text holds is on the device
// once k_witness_emit has run: the sorted witness CIDs and each entry's block index (block bytes come straight from the store's arena,
// so IPCFP_WITNESS_BY_REFERENCE renders too), the EventProofs and their topic / data bytes, the tipset constants.
//   k_json_proof_len / k_json_block_len   exact length of every record (json_items.cuh), separator included
//   exclusive_scan_u32                    record offsets; the two totals are read back (the one host synchronisation of JSON mode)
//   k_json_proofs                         one thread per proof (+ the framing); skipped proof slots write nothing
//   k_json_blocks                         one warp per block: decimal CID bytes and base64 data split over the lanes
// The UnifiedProofBundle of ipcfp_generate_proof_bundle_resident (render_unified_json) takes the same steps over three lists: the
// StorageProofs (k_json_storage_len / k_json_storage, which writes the framing), the EventProofs of every spec, the union's blocks.
#include <algorithm>

#include "engine.cuh"
#include "json_items.cuh"
#include "prims.cuh"

namespace ipcfp {

// record lengths are scanned as u32: a longer record (a block of more than 3 GiB, GiBs of event data) raises the flag instead
__device__ __forceinline__ uint32_t json_len32(uint64_t n, unsigned long long* overflow) {
    if (n > 0xffffffffull) { atomicOr(overflow, 1ull); return 0; }
    return (uint32_t)n;
}
__global__ void __launch_bounds__(256) k_json_proof_len(const ipcfp_event_proof* __restrict__ proofs, uint64_t n, JsonProofCtx c,
                                                        const uint8_t* __restrict__ blob, uint32_t* lens, unsigned long long* overflow) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) lens[i] = json_len32(json_proof_len(c, proofs[i], blob), overflow);
}
__global__ void __launch_bounds__(256) k_json_block_len(const uint8_t* __restrict__ cids, const uint32_t* __restrict__ idx, uint64_t m, StoreView v,
                                                        uint32_t* lens, unsigned long long* overflow) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) lens[i] = json_len32(json_block_len(cids + 38 * i, __ldg(v.lengths + idx[i])), overflow);
}
__global__ void __launch_bounds__(256) k_json_storage_len(const ipcfp_storage_proof* __restrict__ proofs, uint64_t n, JsonStorageCtx c, uint32_t* lens,
                                                          unsigned long long* overflow) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) lens[i] = json_len32(json_storage_len(c, proofs[i]), overflow);
}
// list = where the proofs list starts; thread 0 also writes the EventProofBundle framing at `frame` unless it is null (the grid has at
// least one block)
__global__ void __launch_bounds__(256) k_json_proofs(const ipcfp_event_proof* __restrict__ proofs, uint64_t n, JsonProofCtx c, const uint8_t* __restrict__ blob,
                                                     const uint64_t* __restrict__ offs, char* list, char* frame, uint64_t P, uint64_t Q) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 && frame) json_frame_write(frame, P, Q);
    if (i >= n) return;
    const ipcfp_event_proof p = proofs[i];
    if (json_proof_kept(p)) json_proof_write(list + offs[i], offs[i] == 0, c, p, blob);
}
// thread 0 also writes the UnifiedProofBundle framing; the grid has at least one block
__global__ void __launch_bounds__(256) k_json_storage(const ipcfp_storage_proof* __restrict__ proofs, uint64_t n, JsonStorageCtx c,
                                                      const uint64_t* __restrict__ offs, char* out, uint64_t S, uint64_t P, uint64_t Q) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) json_u_frame_write(out, S, P, Q);
    if (i < n) json_storage_write(out + JSON_STORAGE_HEAD + offs[i], offs[i] == 0, c, proofs[i]);
}
// one warp per witness block, read from the arena by block index at any alignment (as k_witness_copy does)
__global__ void __launch_bounds__(256) k_json_blocks(const uint8_t* __restrict__ cids, const uint32_t* __restrict__ idx, uint64_t m, StoreView v,
                                                     const uint64_t* __restrict__ offs, char* out) {
    const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= m) return;
    uint32_t len;
    const uint8_t* src = store_block(v, idx[w], len);
    json_block_write(out + offs[w], offs[w] == 0, cids + 38 * w, src, len, threadIdx.x & 31, 32);
}

// The steps both renderers share. A text is made of up to three lists of records; per list the caller enqueues the record lengths into
// lens (the overflow flag is DW_JSON_OVERFLOW, cleared by the constructor), then offsets() scans every list and reads the list totals back
// in the one host synchronisation of JSON mode, and copy_out() copies the written text into pinned host memory.
// DW_JSON_TOTAL0..2: list totals → host words HW_JSON_TOTALS.
namespace {
struct JsonLists {
    static constexpr int MAXL = 3;
    Store* s;
    cudaStream_t st;
    int nl;
    uint64_t n[MAXL] = {};
    AsyncBuf<uint32_t> lens[MAXL];
    AsyncBuf<uint64_t> offs[MAXL];
    AsyncBuf<uint64_t> scratch;
    uint64_t total[MAXL] = {};
    JsonLists(Store* store, int count, const uint64_t* sizes) : s(store), st(store->stream), nl(count) {
        uint64_t mx = 0;
        for (int k = 0; k < nl; k++) {
            n[k] = sizes[k];
            lens[k].alloc(n[k] + 1, st);
            offs[k].alloc(n[k] + 1, st);
            mx = std::max(mx, n[k]);
        }
        scratch.alloc(scan_scratch_elems(mx + 1) + 8, st);
        IPCFP_CUDA(cudaMemsetAsync(overflow(), 0, 8, st));
    }
    unsigned long long* overflow() const { return s->dev_words.p + DW_JSON_OVERFLOW; }
    void offsets() {
        static const int word[MAXL] = {DW_JSON_TOTAL0, DW_JSON_TOTAL1, DW_JSON_TOTAL2};
        unsigned long long* dw = s->dev_words.p;
        for (int k = 0; k < nl; k++) exclusive_scan_u32(lens[k].p, offs[k].p, n[k], (uint64_t*)(dw + word[k]), scratch.p, st);
        publish_words(s, HW_JSON_TOTALS, HW_JSON_TOTALS_WORDS, dw + DW_JSON_TOTAL0);
        IPCFP_CUDA(cudaStreamSynchronize(st));   // the exact length of the text: JSON mode's one host synchronisation
        const uint64_t* hw = s->host_words.p;
        if (hw[HW_JSON_TOTALS + DW_JSON_OVERFLOW - DW_JSON_TOTAL0]) throw Error(IPCFP_ERR_UNSUPPORTED, "a record of the JSON bundle is longer than 4 GiB");
        for (int k = 0; k < nl; k++) total[k] = hw[HW_JSON_TOTALS + word[k] - DW_JSON_TOTAL0];
    }
    void copy_out(const char* d_text, uint64_t len, PinnedArray& out) const {
        out = PinnedArray(s->pool, len + 1);
        IPCFP_CUDA(cudaMemcpyAsync(out.p, d_text, len, cudaMemcpyDeviceToHost, st));
        out.as<char>()[len] = 0;
    }
};
}  // namespace

uint64_t render_event_json(Store* s, const JsonInputs& in, PinnedArray& out) {
    cudaStream_t st = s->stream;
    const uint64_t np = in.n_proofs, m = in.m, sizes[2] = {np, m};
    JsonProofCtx c{in.parent_epoch, in.child_epoch, in.n_parents, in.parent_cids, in.child_cid};
    JsonLists L(s, 2, sizes);
    if (np) { k_json_proof_len<<<div_up(np, 256), 256, 0, st>>>(in.proofs, np, c, in.blob, L.lens[0].p, L.overflow()); IPCFP_LAUNCH_CHECK(); }
    if (m) { k_json_block_len<<<div_up(m, 256), 256, 0, st>>>(in.cids, in.idx, m, s->view, L.lens[1].p, L.overflow()); IPCFP_LAUNCH_CHECK(); }
    L.offsets();
    const uint64_t P = L.total[0], Q = L.total[1], total = json_total_len(P, Q);
    AsyncBuf<char> d_out(total + 16, st);
    k_json_proofs<<<div_up(std::max<uint64_t>(np, 1), 256), 256, 0, st>>>(in.proofs, np, c, in.blob, L.offs[0].p, d_out.p + JSON_PROOFS_HEAD, d_out.p, P, Q);
    IPCFP_LAUNCH_CHECK();
    if (m) { k_json_blocks<<<div_up(m * 32, 256), 256, 0, st>>>(in.cids, in.idx, m, s->view, L.offs[1].p, d_out.p + json_blocks_at(P)); IPCFP_LAUNCH_CHECK(); }
    L.copy_out(d_out.p, total, out);
    return total;
}

uint64_t render_unified_json(Store* s, const UnifiedJsonInputs& in, PinnedArray& out) {
    cudaStream_t st = s->stream;
    const uint64_t ns = in.n_storage, np = in.n_proofs, m = in.m, sizes[3] = {ns, np, m};
    JsonStorageCtx sc{in.child_epoch, in.child_cid, in.state_root};
    JsonProofCtx c{in.parent_epoch, in.child_epoch, in.n_parents, in.parent_cids, in.child_cid};
    JsonLists L(s, 3, sizes);
    if (ns) { k_json_storage_len<<<div_up(ns, 256), 256, 0, st>>>(in.storage, ns, sc, L.lens[0].p, L.overflow()); IPCFP_LAUNCH_CHECK(); }
    if (np) { k_json_proof_len<<<div_up(np, 256), 256, 0, st>>>(in.proofs, np, c, in.blob, L.lens[1].p, L.overflow()); IPCFP_LAUNCH_CHECK(); }
    if (m) { k_json_block_len<<<div_up(m, 256), 256, 0, st>>>(in.cids, in.idx, m, s->view, L.lens[2].p, L.overflow()); IPCFP_LAUNCH_CHECK(); }
    L.offsets();
    const uint64_t S = L.total[0], P = L.total[1], Q = L.total[2], total = json_u_total_len(S, P, Q);
    AsyncBuf<char> d_out(total + 16, st);
    k_json_storage<<<div_up(std::max<uint64_t>(ns, 1), 256), 256, 0, st>>>(in.storage, ns, sc, L.offs[0].p, d_out.p, S, P, Q); IPCFP_LAUNCH_CHECK();
    if (np) {
        k_json_proofs<<<div_up(np, 256), 256, 0, st>>>(in.proofs, np, c, in.blob, L.offs[1].p, d_out.p + json_u_events_at(S), nullptr, P, Q);
        IPCFP_LAUNCH_CHECK();
    }
    if (m) { k_json_blocks<<<div_up(m * 32, 256), 256, 0, st>>>(in.cids, in.idx, m, s->view, L.offs[2].p, d_out.p + json_u_blocks_at(S, P)); IPCFP_LAUNCH_CHECK(); }
    L.copy_out(d_out.p, total, out);
    return total;
}

}  // namespace ipcfp
