// rpc_json.cu — ipcfp_tipset_upload_json: a device-resident tipset straight from the Lotus JSON-RPC texts, with the receipt list parsed on
// the device when it is canonical (rpc_json_items.cuh). The two small ApiTipset texts, and any receipt list the device path does not
// accept, go through ipcfp_tipset_desc_from_json (csrc/rpc_parse.cpp) and tipset_upload, so results never depend on the path.
//
// Device path, all on the store's stream:
//   H2D of the text (+ JP_PAD zero bytes)
//   k_rj_mark              one thread per 32 text bytes: bit p of the bitmap = a record starts at p; a byte no canonical text holds
//                          sets the defer word
//   bitmap_to_indices      record starts, ascending (prims.cu)
//   ── host synchronisation 1: the record count and the defer word; they size the tipset's events_roots / has_root
//   k_rj_records           one thread per record: its template and its joints, its 38 CID bytes and flag straight into the tipset's arrays
//   ── host synchronisation 2: the defer word
#include <cstring>

#include "engine.cuh"
#include "rpc_json_items.cuh"
#include "text_scan.cuh"

namespace ipcfp {

struct RjMeta {
    unsigned long long defer;   // non-zero: not canonical
    unsigned long long n;       // record starts
};
static_assert(sizeof(RjMeta) <= HW_PARSE_META_WORDS * 8, "the meta words fit their host words (HW_PARSE_META)");

__global__ void __launch_bounds__(256) k_rj_mark(const char* __restrict__ t, uint64_t len, uint32_t* bits, uint64_t nwords, RjMeta* meta) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwords) return;
    uint32_t b = 0;
    bool foreign = false;
    for (uint32_t k = 0; k < 32; k++) {
        const uint64_t p = 32 * w + k;
        if (p >= len) break;
        const char c = t[p];
        foreign |= rj_foreign_byte(c);
        if (c == '{' && rj_start_at(t, p)) b |= 1u << k;
    }
    bits[w] = b;
    if (foreign) meta->defer = 1;
}

__global__ void __launch_bounds__(128) k_rj_records(const char* __restrict__ t, uint64_t len, const uint32_t* __restrict__ pos, uint64_t n,
                                                    uint8_t* roots, uint8_t* has, RjMeta* meta) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t h = 0;
    if (!rj_record(t, len, pos, n, i, roots + 38ull * i, h)) meta->defer = 1;
    has[i] = h;
}

// the device path for the receipt list; false: not canonical (td's receipt arrays are then to be replaced)
static bool receipts_on_device(Store* s, const char* text, uint64_t len, TipsetDev& td) {
    if (len < 2 || len >= (1ull << 32) || text[0] != '[' || text[len - 1] != ']') return false;   // record starts are u32
    if (len == 2) { td.n_receipts = 0; return true; }
    cudaStream_t st = s->stream;
    const uint64_t cap = len / RJ_MIN_RECORD + 1;
    TextScan<RjMeta> sc(s, len, len / RJ_HEAD_LEN + 8, 0, 0);
    // straight from the caller's pageable memory: the driver's own pipelined staging beat a copy through two pinned chunks of the pool
    // (8 MB each, filled by one host thread): the whole parse of the 142 MB list of 1 M receipts took 22 ms against 28 ms on an H100 host
    IPCFP_CUDA(cudaMemcpyAsync(sc.text.p, text, len, cudaMemcpyHostToDevice, st));
    Event tm[4];
    IPCFP_CUDA(cudaEventRecord(tm[0], st));
    sc.starts(k_rj_mark, sc.meta.p);
    IPCFP_CUDA(cudaEventRecord(tm[1], st));
    const RjMeta m = sc.read();   // host synchronisation 1
    const uint64_t n = m.n;
    if (m.defer || n == 0 || n > cap) return false;
    td.n_receipts = n;
    td.events_roots.alloc(n * 38 + 64);
    td.has_root.alloc(n + 64);
    IPCFP_CUDA(cudaEventRecord(tm[2], st));
    k_rj_records<<<div_up(n, 128), 128, 0, st>>>(sc.text.p, len, sc.pos.p, n, td.events_roots.p, td.has_root.p, sc.meta.p); IPCFP_LAUNCH_CHECK();
    IPCFP_CUDA(cudaEventRecord(tm[3], st));
    const bool canonical = sc.read().defer == 0;   // host synchronisation 2
    td.ms_kernels = elapsed_ms(tm[0], tm[1]) + elapsed_ms(tm[2], tm[3]);
    return canonical;
}

static void rethrow_parse(ipcfp_status st) {
    const uint64_t index = ipcfp_last_error_index();
    throw Error(st, ipcfp_last_error(), index);
}

void tipset_upload_json(Store* s, const char* parent, uint64_t parent_len, const char* child, uint64_t child_len, const char* receipts,
                        uint64_t receipts_len, TipsetDev& td) {
    s->use();
    if (!receipts && receipts_len) throw Error(IPCFP_ERR_INVALID_ARG, "null receipt list");
    // the two ApiTipset texts (with an empty list): their failures come first, as in ipcfp_tipset_desc_from_json
    ipcfp_parsed_tipset* pt = nullptr;
    ipcfp_status st = ipcfp_tipset_desc_from_json(parent, parent_len, child, child_len, "[]", 2, &pt);
    if (st != IPCFP_OK) rethrow_parse(st);
    std::unique_ptr<ipcfp_parsed_tipset, void (*)(ipcfp_parsed_tipset*)> keep(pt, ipcfp_parsed_tipset_free);
    const Clock::time_point t0 = Clock::now();
    TipsetDev dev;
    if (receipts && receipts_on_device(s, receipts, receipts_len, dev)) {
        tipset_upload(s, &pt->desc, td);   // the upload's own checks, the host fields; no receipt yet
        td.n_receipts = dev.n_receipts;
        if (dev.n_receipts) { td.events_roots = std::move(dev.events_roots); td.has_root = std::move(dev.has_root); }
        td.parsed_on_device = true;
        td.ms_kernels = dev.ms_kernels;
        td.ms_parse = ms_since(t0);
        return;
    }
    keep.reset();
    st = ipcfp_tipset_desc_from_json(parent, parent_len, child, child_len, receipts, receipts_len, &pt);
    if (st != IPCFP_OK) rethrow_parse(st);
    keep.reset(pt);
    tipset_upload(s, &pt->desc, td);
    IPCFP_CUDA(cudaStreamSynchronize(s->stream));
    td.ms_parse = ms_since(t0);
}

void tipset_describe(TipsetDev& td, bool with_roots, ipcfp_tipset_info* out) {
    memset(out, 0, sizeof *out);
    ipcfp_tipset_desc& d = out->desc;
    d.parent_epoch = td.parent_epoch;
    d.child_epoch = td.child_epoch;
    d.n_parents = td.n_parents;
    d.parent_cids = td.n_parents ? td.parent_cids.data() : nullptr;
    d.parent_txmeta_cids = td.n_parents ? td.txmeta_cids.data() : nullptr;
    d.child_cid = td.child_cid;
    d.receipts_root = td.receipts_root;
    d.child_parent_state_root = td.has_state_root ? td.child_state_root : nullptr;
    d.n_receipts = td.n_receipts;
    if (with_roots && td.n_receipts) {
        if (td.host_has.size() != td.n_receipts) {
            IPCFP_CUDA(cudaSetDevice(td.device));
            std::vector<uint8_t> roots(td.n_receipts * 38), has(td.n_receipts);
            IPCFP_CUDA(cudaMemcpy(roots.data(), td.events_roots.p, roots.size(), cudaMemcpyDeviceToHost));
            IPCFP_CUDA(cudaMemcpy(has.data(), td.has_root.p, has.size(), cudaMemcpyDeviceToHost));
            td.host_roots.swap(roots);
            td.host_has.swap(has);
        }
        d.events_roots = td.host_roots.data();
        d.has_events_root = td.host_has.data();
    }
    out->parsed_on_device = td.parsed_on_device ? 1u : 0u;
    out->ms_parse = td.ms_parse;
    out->ms_kernels = td.ms_kernels;
}

}  // namespace ipcfp
