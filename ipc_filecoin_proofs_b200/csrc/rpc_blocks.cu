// rpc_blocks.cu — ipcfp_store_create_rpc_json: a block store straight from Filecoin.ChainReadObj JSON-RPC responses, with canonical texts
// parsed and their base64 decoded on the device (rpc_blocks_items.cuh), straight into the new store's arena. Any input the device path
// does not accept goes through ipcfp_blocks_from_rpc_json (csrc/rpc_blocks_parse.cpp) and store_create, so results never depend on the path.
//
// Device path, all on the store's stream:
//   H2D of the texts, each followed by RB_SEP (+ JP_PAD zero bytes): texts of RB_DIRECT_BYTES or more straight from the caller's memory,
//                          the others packed into pinned staging chunks
//   k_rb_mark              one thread per 32 bytes: bit p of the bitmap = a record starts at p
//   bitmap_to_indices      record starts, ascending (prims.cu)
//   k_rb_records           one warp per record: its data run (ballots over 32 bytes), template and joints (lane 0), the base64 characters
//                          (all lanes); claims owner[id], writes the id's 16-aligned arena bytes and character count, adds the owned bytes
//   exclusive_scan_u32     arena offsets by id
//   ── host synchronisation 1: the meta words. Accepted: no defer, one record per id, every byte of the texts owned.
//   k_rb_blocks            one warp per id: offset, length, base64 decoded straight into the store's block bytes at offset
//   store_finish (store.cu)
#include <cstring>

#include "engine.cuh"
#include "prims.cuh"
#include "rpc_blocks_items.cuh"
#include "text_scan.cuh"

namespace ipcfp {

struct RbMeta {
    unsigned long long defer;   // non-zero: not canonical (or an id twice)
    unsigned long long n;       // record starts
    unsigned long long owned;   // bytes the records own
    unsigned long long b_total; // arena bytes (16-aligned blocks)
};
static_assert(sizeof(RbMeta) <= HW_PARSE_META_WORDS * 8, "the meta words fit their host words (HW_PARSE_META)");

__global__ void __launch_bounds__(256) k_rb_mark(const char* __restrict__ t, uint64_t len, uint32_t* bits, uint64_t nwords) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwords) return;
    uint32_t b = 0;
    for (uint32_t k = 0; k < 32; k++) {
        const uint64_t p = 32 * w + k;
        if (p < len && t[p] == '{' && rb_start_at(t, p)) b |= 1u << k;
    }
    bits[w] = b;
}

// one warp per record slot of [0, cap)
__global__ void __launch_bounds__(128) k_rb_records(const char* __restrict__ t, uint64_t len, const uint32_t* __restrict__ pos, uint64_t cap,
                                                    uint64_t n_ids, RbMeta* meta, uint32_t* owner, uint32_t* blen, uint32_t* nch) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= cap) return;
    const uint64_t n = meta->n;
    if (n > cap) {   // denser than any canonical text
        if (i == 0 && lane == 0) meta->defer = 1;
        return;
    }
    if (i >= n) return;
    // the data run: the first stop byte at or after the data (the buffer ends in JP_PAD zero bytes, which stop it)
    uint64_t q = (uint64_t)pos[i] + RB_HEAD_LEN;
    for (;;) {
        const uint32_t stop = __ballot_sync(0xffffffffu, rb_stop_byte(t[q + lane]));
        if (stop) { q += __ffs(stop) - 1; break; }
        q += 32;
    }
    RbRec r;
    bool ok = true;
    if (lane == 0) ok = rb_record(t, len, pos, n, i, q, n_ids, r);
    ok = __shfl_sync(0xffffffffu, ok, 0);
    if (ok) {
        JpBlock b;
        b.data_at = __shfl_sync(0xffffffffu, r.blk.data_at, 0);
        b.n_chars = __shfl_sync(0xffffffffu, r.blk.n_chars, 0);
        b.pads = __shfl_sync(0xffffffffu, r.blk.pads, 0);
        bool good = true;
        for (uint64_t k = lane; k < b.n_chars - b.pads; k += 32) good &= jp_block_char_ok(t, b, k);
        ok = __all_sync(0xffffffffu, good);
    }
    if (lane) return;
    if (!ok || atomicCAS(&owner[r.id], 0xffffffffu, (uint32_t)i) != 0xffffffffu) { meta->defer = 1; return; }
    blen[r.id] = (uint32_t)jp_align16(r.blk.len);
    nch[r.id] = (uint32_t)r.blk.n_chars;
    atomicAdd(&meta->owned, (unsigned long long)r.owned);
}

// one warp per block: block j is the record owner[j]
__global__ void __launch_bounds__(128) k_rb_blocks(const char* __restrict__ t, const uint32_t* __restrict__ pos, const uint32_t* __restrict__ owner,
                                                   const uint32_t* __restrict__ nch, uint64_t nb, const uint64_t* __restrict__ boff, uint64_t* offsets,
                                                   uint32_t* lengths, uint8_t* blob) {
    const uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (j >= nb) return;
    JpBlock b;
    b.data_at = (uint64_t)pos[owner[j]] + RB_HEAD_LEN;
    b.n_chars = nch[j];
    jp_b64_span(t, b);   // accepted by k_rb_records: sets pads and len
    if (lane == 0) { offsets[j] = boff[j]; lengths[j] = b.len; }
    uint8_t* out = blob + boff[j];
    for (uint64_t g = lane; g < b.n_chars / 4; g += 32) jp_block_group(t, b, g, out);
}

#define RB_DIRECT_BYTES (1ull << 20)   // texts this long are copied from the caller's memory; shorter ones are packed first
#define RB_STAGE_BYTES (16ull << 20)   // one pinned staging chunk (two of them alternate)

// the texts, each followed by RB_SEP, to d (len bytes in all): few large copies, however many texts there are
static void upload_texts(Store* s, const char* const* texts, const uint64_t* lens, uint64_t n_texts, char* d) {
    cudaStream_t st = s->stream;
    PinnedArray stage[2];
    Event done[2] = {Event(cudaEventDisableTiming), Event(cudaEventDisableTiming)};   // a buffer's last copy (none yet: complete)
    int cur = 0;
    uint64_t fill = 0, at = 0, chunk_at = 0;
    auto flush = [&] {
        if (!fill) return;
        IPCFP_CUDA(cudaMemcpyAsync(d + chunk_at, stage[cur].p, fill, cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaEventRecord(done[cur], st));
        cur ^= 1;
        fill = 0;
    };
    for (uint64_t k = 0; k < n_texts; k++) {
        const uint64_t L = lens[k];
        if (L >= RB_DIRECT_BYTES) {
            flush();
            IPCFP_CUDA(cudaMemcpyAsync(d + at, texts[k], L, cudaMemcpyHostToDevice, st));
            IPCFP_CUDA(cudaMemsetAsync(d + at + L, RB_SEP, 1, st));
            at += L + 1;
            continue;
        }
        if (fill + L + 1 > RB_STAGE_BYTES) flush();
        if (!fill) {   // a fresh chunk: its buffer's last copy must be done before it is written again
            if (!stage[cur].p) stage[cur] = PinnedArray(s->pool, RB_STAGE_BYTES);
            IPCFP_CUDA(cudaEventSynchronize(done[cur]));
            chunk_at = at;
        }
        char* h = stage[cur].as<char>() + fill;
        memcpy(h, texts[k], L);
        h[L] = RB_SEP;
        fill += L + 1;
        at += L + 1;
    }
    flush();
    IPCFP_CUDA(cudaStreamSynchronize(st));   // the staging buffers go back to the pool
}

// the device path; false: not canonical (the store is then discarded)
static bool blocks_on_device(Store* s, const uint8_t* cids, uint64_t nb, const char* const* texts, const uint64_t* lens, uint64_t n_texts,
                             uint32_t flags, ipcfp_store_json_info& info, Clock::time_point t0) {
    uint64_t len = 0, want_owned = 0;
    for (uint64_t k = 0; k < n_texts; k++) {
        if (!texts[k] || lens[k] == 0) return false;
        len += lens[k] + 1;
        want_owned += lens[k] == 2 && texts[k][0] == '[' && texts[k][1] == ']' ? 0 : lens[k];
        if (len >= 0xffffff00ull) return false;   // record starts are u32
    }
    if (nb && !cids) return false;
    cudaStream_t st = s->stream;
    const uint64_t cap = len / RB_MIN_RECORD + 1;
    TextScan<RbMeta> sc(s, len, len / RB_HEAD_LEN + 8, nb + 1, 0);
    AsyncBuf<uint32_t> owner(nb + 1, st), blen(nb + 1, st), nch(nb + 1, st);
    AsyncBuf<uint64_t> boff(nb + 1, st);
    upload_texts(s, texts, lens, n_texts, sc.text.p);
    IPCFP_CUDA(cudaMemsetAsync(owner.p, 0xff, (nb + 1) * 4, st));
    IPCFP_CUDA(cudaMemsetAsync(blen.p, 0, (nb + 1) * 4, st));
    Event tm[4];
    IPCFP_CUDA(cudaEventRecord(tm[0], st));
    sc.starts(k_rb_mark);
    k_rb_records<<<div_up(cap * 32, 128), 128, 0, st>>>(sc.text.p, len, sc.pos.p, cap, nb, sc.meta.p, owner.p, blen.p, nch.p); IPCFP_LAUNCH_CHECK();
    if (nb) exclusive_scan_u32(blen.p, boff.p, nb, (uint64_t*)&sc.meta.p->b_total, sc.scratch.p, st);
    IPCFP_CUDA(cudaEventRecord(tm[1], st));
    const RbMeta m = sc.read();   // host synchronisation 1
    if (m.defer || m.n != nb || m.owned != want_owned) return false;
    // the store, its blocks decoded straight into the arena
    DevBuf<uint8_t> cids_dev;
    uint8_t* blocks = store_alloc_blocks(s, nb, m.b_total, cids_dev, true);
    if (nb) IPCFP_CUDA(cudaMemcpyAsync(cids_dev.p, cids, nb * IPCFP_CID_LEN, cudaMemcpyHostToDevice, st));
    IPCFP_CUDA(cudaEventRecord(tm[2], st));
    if (nb) {
        k_rb_blocks<<<div_up(nb * 32, 128), 128, 0, st>>>(sc.text.p, sc.pos.p, owner.p, nch.p, nb, boff.p, s->offsets.p, s->lengths.p, blocks);
        IPCFP_LAUNCH_CHECK();
    }
    IPCFP_CUDA(cudaEventRecord(tm[3], st));
    IPCFP_CUDA(cudaStreamSynchronize(st));
    info.parsed_on_device = 1;
    info.ms_parse = ms_since(t0);
    info.ms_kernels = elapsed_ms(tm[0], tm[1]) + elapsed_ms(tm[2], tm[3]);
    store_finish(s, cids_dev.p, cids, cids, flags);
    return true;
}

Store* store_create_rpc_json(const uint8_t* cids, uint64_t nb, const char* const* texts, const uint64_t* lens, uint64_t n_texts, int device,
                             uint32_t flags, ipcfp_store_json_info& info) {
    // the device path needs texts to read; everything else (and every failure) is the host path's to report
    Store* s = store_create_parsed(
        device, flags, info, n_texts && texts && lens && nb < 0x7fffffffull,
        [&](Store* fresh, Clock::time_point t0) { return blocks_on_device(fresh, cids, nb, texts, lens, n_texts, flags, info, t0); },
        [&](ipcfp_parsed_blocks** pb) { return ipcfp_blocks_from_rpc_json(cids, nb, texts, lens, n_texts, pb); }, nullptr);
    s->caller_blob = false;
    return s;
}

}  // namespace ipcfp
