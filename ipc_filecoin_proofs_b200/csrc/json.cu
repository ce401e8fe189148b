// json.cu — IPCFP_RESULT_JSON: the EventProofBundle of a generate_event_proof call rendered on the device, byte for byte what
// ipcfp_event_result_to_json (csrc/bundle_json.cpp) renders from the POD result on the host. Everything the text holds is on the device
// once k_witness_emit has run: the sorted witness CIDs and each entry's block index (block bytes come straight from the store's arena,
// so IPCFP_WITNESS_BY_REFERENCE renders too), the EventProofs and their topic / data bytes, the tipset constants.
//   k_json_proof_len / k_json_block_len   exact length of every record (json_items.cuh), separator included
//   exclusive_scan_u32                    record offsets; the two totals are read back (the one host synchronisation of JSON mode)
//   k_json_proofs                         one thread per proof (+ the framing); skipped proof slots write nothing
//   k_json_blocks                         one warp per block: decimal CID bytes and base64 data split over the lanes
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
// thread 0 also writes the framing; the grid has at least one block
__global__ void __launch_bounds__(256) k_json_proofs(const ipcfp_event_proof* __restrict__ proofs, uint64_t n, JsonProofCtx c, const uint8_t* __restrict__ blob,
                                                     const uint64_t* __restrict__ offs, char* out, uint64_t P, uint64_t Q) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) json_frame_write(out, P, Q);
    if (i >= n) return;
    const ipcfp_event_proof p = proofs[i];
    if (json_proof_kept(p)) json_proof_write(out + JSON_PROOFS_HEAD + offs[i], offs[i] == 0, c, p, blob);
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

uint64_t render_event_json(Store* s, const JsonInputs& in, PinnedArray& out) {
    cudaStream_t st = s->stream;
    unsigned long long* dw = s->dev_words.p;   // [24] proofs list length, [25] blocks list length, [26] overflow flag → host words 200..202
    const uint64_t* hw = s->host_words.p;
    const uint64_t np = in.n_proofs, m = in.m;
    JsonProofCtx c{in.parent_epoch, in.child_epoch, in.n_parents, in.parent_cids, in.child_cid};
    AsyncBuf<uint32_t> plen(np + 1, st), blen(m + 1, st);
    AsyncBuf<uint64_t> poff(np + 1, st), boff(m + 1, st), scratch(scan_scratch_elems(std::max(np, m) + 1) + 8, st);
    IPCFP_CUDA(cudaMemsetAsync(dw + 26, 0, 8, st));
    if (np) { k_json_proof_len<<<div_up(np, 256), 256, 0, st>>>(in.proofs, np, c, in.blob, plen.p, dw + 26); IPCFP_LAUNCH_CHECK(); }
    if (m) { k_json_block_len<<<div_up(m, 256), 256, 0, st>>>(in.cids, in.idx, m, s->view, blen.p, dw + 26); IPCFP_LAUNCH_CHECK(); }
    exclusive_scan_u32(plen.p, poff.p, np, (uint64_t*)(dw + 24), scratch.p, st);
    exclusive_scan_u32(blen.p, boff.p, m, (uint64_t*)(dw + 25), scratch.p, st);
    publish_words_from(s, dw + 24, 200, 3);
    IPCFP_CUDA(cudaStreamSynchronize(st));   // the exact length of the text: JSON mode's one host synchronisation
    if (hw[202]) throw Error(IPCFP_ERR_UNSUPPORTED, "a record of the JSON bundle is longer than 4 GiB");
    const uint64_t P = hw[200], Q = hw[201], total = json_total_len(P, Q);
    AsyncBuf<char> d_out(total + 16, st);
    k_json_proofs<<<div_up(std::max<uint64_t>(np, 1), 256), 256, 0, st>>>(in.proofs, np, c, in.blob, poff.p, d_out.p, P, Q); IPCFP_LAUNCH_CHECK();
    if (m) { k_json_blocks<<<div_up(m * 32, 256), 256, 0, st>>>(in.cids, in.idx, m, s->view, boff.p, d_out.p + json_blocks_at(P)); IPCFP_LAUNCH_CHECK(); }
    out = PinnedArray(s->pool, total + 1);
    IPCFP_CUDA(cudaMemcpyAsync(out.p, d_out.p, total, cudaMemcpyDeviceToHost, st));
    out.as<char>()[total] = 0;
    return total;
}

}  // namespace ipcfp
