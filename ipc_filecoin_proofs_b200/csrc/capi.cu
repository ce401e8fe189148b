// capi.cu — the extern "C" surface declared in include/ipcfp.h.
#include <atomic>
#include <cstring>

#include "engine.cuh"
#include "log_filter.cuh"

namespace ipcfp {

static thread_local std::string g_last_error;
static thread_local uint64_t g_last_index = UINT64_MAX;
static std::atomic<uint64_t> g_launches{0};

void note_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
void set_last_error(const std::string& msg, uint64_t index) { g_last_error = msg; g_last_index = index; }

template <class F> static ipcfp_status guard(F f) {
    g_last_error.clear();
    g_last_index = UINT64_MAX;
    try { f(); return IPCFP_OK; }
    catch (const Error& e) { g_last_error = e.msg; g_last_index = e.index; return e.status; }
    catch (const std::bad_alloc&) { g_last_error = "out of host memory"; return IPCFP_ERR_INVALID_ARG; }
    catch (const std::exception& e) { g_last_error = e.what(); return IPCFP_ERR_INVALID_ARG; }
}

// guard() with the prologue of every entry point that makes an object: "null argument" unless `ok` (its pointer arguments are set) and
// `out` is set, *out cleared, then *out = f()
template <class R, class F> static ipcfp_status produce(bool ok, R** out, F f) {
    return guard([&] {
        if (!ok || !out) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        *out = nullptr;
        *out = f();
    });
}

static Store* store_of(ipcfp_store* s) { return reinterpret_cast<Store*>(s); }
static TipsetDev& tipset_of(ipcfp_tipset* t) { return *reinterpret_cast<TipsetDev*>(t); }

// f(store, tipset) with the descriptor uploaded into a call-local TipsetDev, asynchronously on the store's stream (ipcfp_tipset_upload
// would add a host synchronisation)
template <class F> static auto with_uploaded_tipset(Store* st, const ipcfp_tipset_desc* t, F f) {
    TipsetDev td;
    tipset_upload(st, t, td);
    return f(st, td);
}

// produce() of a call on a tipset, *out = f(store, tipset): a resident tipset as it is, a descriptor through with_uploaded_tipset
template <class R, class F> static ipcfp_status on_tipset(ipcfp_store* s, ipcfp_tipset* t, R** out, F f) {
    return produce(s && t, out, [&] { return f(store_of(s), tipset_of(t)); });
}
template <class R, class F> static ipcfp_status on_tipset(ipcfp_store* s, const ipcfp_tipset_desc* t, R** out, F f) {
    return produce(s != nullptr, out, [&] { return with_uploaded_tipset(store_of(s), t, f); });
}

// *out = the store make() creates; a block that fails its CID check is reported with the store in *out
template <class F> static ipcfp_status make_store(ipcfp_store** out, F make) {
    return guard([&] {
        if (!out) throw Error(IPCFP_ERR_INVALID_ARG, "null out");
        *out = nullptr;
        Store* s = make();
        *out = reinterpret_cast<ipcfp_store*>(s);
        if (s->first_bad != UINT64_MAX) throw Error(IPCFP_ERR_CID_MISMATCH, "blake2b-256(block) != CID digest", s->first_bad);
    });
}
// *out = a resident tipset that upload(store, tipset) fills, complete on the device when the call returns
template <class F> static ipcfp_status make_resident(ipcfp_store* s, ipcfp_tipset** out, F upload) {
    return produce(s != nullptr, out, [&] {
        Store* st = store_of(s);
        std::unique_ptr<TipsetDev> td(new TipsetDev());
        upload(st, *td);
        IPCFP_CUDA(cudaStreamSynchronize(st->stream));
        return reinterpret_cast<ipcfp_tipset*>(td.release());
    });
}

// ------------------------------------------------------------------------------------------ bundle
struct BundleBox {
    ipcfp_bundle r;   // must stay first
    std::vector<ipcfp_event_result*> ev;
    WitnessOut wit;   // the union
    PinnedArray json;
    ~BundleBox() {
        if (r.storage) storage_result_free(r.storage);
        for (auto* e : ev) event_result_free(e);
    }
};

struct FetchPlanBox {
    ipcfp_fetch_plan r;   // must stay first
    FetchPlan plan;
};

static void plan_flags_check(uint32_t flags) {
    if (flags) throw Error(IPCFP_ERR_INVALID_ARG, "unknown flag bit for a fetch plan");
}
// the fetch plan that plan(FetchPlan&) makes, in the box ipcfp_fetch_plan_free releases
template <class F> static ipcfp_fetch_plan* make_plan(F plan) {
    std::unique_ptr<FetchPlanBox> box(new FetchPlanBox());
    FetchPlan& p = box->plan;
    plan(p);
    box->r.n_missing = p.cids.size() / 38;
    box->r.cids = p.cids.data();
    box->r.n_needed = p.n_needed;
    box->r.n_levels = p.n_levels;
    box->r.ms_total = p.ms_total;
    return &box.release()->r;
}

#define IPCFP_BUNDLE_FLAGS (IPCFP_WITNESS_BY_REFERENCE | IPCFP_RESULT_JSON)

// generate_proof_bundle (proofs/generator.rs:25-95) against a device-resident tipset: the storage specs in one batch, then event item
// 0 .. n_events - 1 in order (gen(k) makes item k's EventProofBundle: an event spec's or a log filter's), then the BTreeSet<(Cid, data)>
// union of every proof's blocks on the device (witness_union: OR of the lists' rank bits, one compaction) and, with IPCFP_RESULT_JSON,
// the UnifiedProofBundle text rendered from device memory. check() runs before any device work.
template <class Check, class Gen>
static ipcfp_bundle* generate_proof_bundle(Store* st, TipsetDev& td, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs, uint64_t n_events,
                                           uint32_t flags, Check check, Gen gen) {
    if (flags & ~(uint32_t)IPCFP_BUNDLE_FLAGS) throw Error(IPCFP_ERR_INVALID_ARG, "unknown flag bit for a proof bundle");
    if (n_sspecs && !sspecs) throw Error(IPCFP_ERR_INVALID_ARG, "null specs");
    check();
    if ((flags & IPCFP_WITNESS_BY_REFERENCE) && !st->caller_blob)
        throw Error(IPCFP_ERR_UNSUPPORTED, "IPCFP_WITNESS_BY_REFERENCE needs a store made from a caller's blob (ipcfp_store_create)");
    st->use();
    const bool by_ref = (flags & IPCFP_WITNESS_BY_REFERENCE) != 0;
    cudaStream_t stream = st->stream;
    Event t0, t1, j0, j1;
    IPCFP_CUDA(cudaEventRecord(t0, stream));
    std::unique_ptr<BundleBox> box(new BundleBox());
    memset(&box->r, 0, sizeof box->r);
    std::vector<const WitnessOut*> lists;
    if (n_sspecs) {
        if (!td.has_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
        box->r.storage = generate_storage_proofs(st, td.child_cid, td.child_state_root, sspecs, n_sspecs, by_ref);
        lists.push_back(&storage_result_witness(box->r.storage));
    }
    for (uint64_t i = 0; i < n_events; i++) {
        box->ev.push_back(gen(i));
        lists.push_back(&event_result_witness(box->ev.back()));
    }
    witness_union(st, lists, box->wit, by_ref);

    if (flags & IPCFP_RESULT_JSON) {
        IPCFP_CUDA(cudaEventRecord(j0, stream));
        // the records' inputs in ONE upload: storage proofs, every spec's EventProofs with their topics / data offsets rebased into one
        // concatenated data blob, the tipset CIDs the records repeat
        const uint64_t ns = box->r.storage ? box->r.storage->n_proofs : 0;
        uint64_t np = 0, nb = 0;
        for (auto* e : box->ev) { np += e->n_proofs; nb += e->data_blob_size; }
        auto up16 = [](uint64_t x) { return (x + 15) & ~15ull; };
        const uint64_t o_ev = up16(ns * sizeof(ipcfp_storage_proof)), o_blob = o_ev + up16(np * sizeof(ipcfp_event_proof)),
                       o_cids = o_blob + up16(nb + 16), size = o_cids + 38ull * (2 + td.n_parents);
        PinnedArray stage(st->pool, size);
        uint8_t* h = stage.as<uint8_t>();
        if (ns) memcpy(h, box->r.storage->proofs, ns * sizeof(ipcfp_storage_proof));
        ipcfp_event_proof* hp = (ipcfp_event_proof*)(h + o_ev);
        uint64_t k = 0, base = 0;
        for (auto* e : box->ev) {
            for (uint64_t q = 0; q < e->n_proofs; q++, k++) {
                hp[k] = e->proofs[q];
                hp[k].data_off += base;
                hp[k].topics_off += base;
            }
            if (e->data_blob_size) memcpy(h + o_blob + base, e->data_blob, e->data_blob_size);
            base += e->data_blob_size;
        }
        memcpy(h + o_cids, td.child_cid, 38);
        memcpy(h + o_cids + 38, td.child_state_root, 38);
        if (td.n_parents) memcpy(h + o_cids + 76, td.parent_cids.data(), 38ull * td.n_parents);
        AsyncBuf<uint8_t> d(size, stream);
        IPCFP_CUDA(cudaMemcpyAsync(d.p, h, size, cudaMemcpyHostToDevice, stream));
        UnifiedJsonInputs ji{(const ipcfp_storage_proof*)d.p, ns, (const ipcfp_event_proof*)(d.p + o_ev), np, d.p + o_blob,
                             box->wit.cids_dev.p, box->wit.idx_dev.p, box->wit.n, td.parent_epoch, td.child_epoch, td.n_parents,
                             d.p + o_cids + 76, d.p + o_cids, d.p + o_cids + 38};
        box->r.json_len = render_unified_json(st, ji, box->json);
        IPCFP_CUDA(cudaEventRecord(j1, stream));
    }
    IPCFP_CUDA(cudaEventRecord(t1, stream));
    IPCFP_CUDA(cudaStreamSynchronize(stream));
    box->r.n_event_results = box->ev.size();
    box->r.events = box->ev.data();
    box->wit.fill(box->r.witness);
    box->r.ms_total = elapsed_ms(t0, t1);
    if (flags & IPCFP_RESULT_JSON) {
        box->r.json = box->json.as<char>();
        box->r.ms_json = elapsed_ms(j0, j1);
    }
    return &box.release()->r;
}

// the bundle of event specs
static ipcfp_bundle* generate_proof_bundle(Store* st, TipsetDev& td, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                           const ipcfp_event_spec* especs, uint64_t n_especs, uint32_t flags) {
    return generate_proof_bundle(
        st, td, sspecs, n_sspecs, n_especs, flags,
        [&] { if (n_especs && !especs) throw Error(IPCFP_ERR_INVALID_ARG, "null specs"); },
        [&](uint64_t i) { return generate_event_proof(st, td, &especs[i], flags & IPCFP_WITNESS_BY_REFERENCE, false, 0, 0); });
}
// the bundle of log filters: every filter is checked before any device work
static ipcfp_bundle* generate_log_bundle(Store* st, TipsetDev& td, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                         const ipcfp_log_filter* filters, uint64_t n_filters, uint32_t flags) {
    return generate_proof_bundle(
        st, td, sspecs, n_sspecs, n_filters, flags, [&] { LogFilterSet::check(filters, n_filters); },
        [&](uint64_t k) { return generate_log_proof(st, td, &filters[k], flags & IPCFP_WITNESS_BY_REFERENCE); });
}

}  // namespace ipcfp

using namespace ipcfp;

struct ipcfp_store { Store s; };

extern "C" {

const char* ipcfp_last_error(void) { return g_last_error.c_str(); }
uint64_t ipcfp_last_error_index(void) { return g_last_index; }
const char* ipcfp_version(void) {
    return "ipcfp-b200 0.2 (sm_90a): k_verify_cids k_hash_batch k_build_index sort_by_cid k_pass1_stage k_pass2 k_amt_dense k_amt_expand k_dedup "
           "k_storage_proofs k_read_slots k_path_* k_verify_events k_verify_storage k_scan k_witness_copy k_witness_emit k_union_mark k_json_* k_jp_* k_rj_* k_rb_* k_car_* | sharded: k_xb_* k_exec_claim_seg "
           "k_exec_mark_dups k_select_positions k_fetch_positions k_part_pack k_merge_* (NCCL via dlopen)";
}
uint64_t ipcfp_kernel_launch_count(void) { return g_launches.load(); }

ipcfp_status ipcfp_host_alloc(size_t bytes, void** out) {
    return guard([&] {
        if (!out) throw Error(IPCFP_ERR_INVALID_ARG, "null out");
        int cnt = 0;
        if (cudaGetDeviceCount(&cnt) != cudaSuccess || cnt == 0) { cudaGetLastError(); throw Error(IPCFP_ERR_NO_DEVICE, "no CUDA device"); }
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
        NumaPrefer numa(dev);   // pages of the caller's staging buffers next to the GPU they feed
        IPCFP_CUDA(cudaMallocHost(out, bytes ? bytes : 1));
    });
}
void ipcfp_host_free(void* p) { if (p) cudaFreeHost(p); }

ipcfp_status ipcfp_store_create(const uint8_t* cids, const uint64_t* offsets, const uint32_t* lengths, const uint8_t* blob, uint64_t blob_size,
                                uint64_t n_blocks, int device, uint32_t flags, ipcfp_store** out) {
    return make_store(out, [&] { return store_create(cids, offsets, lengths, blob, blob_size, n_blocks, device, flags); });
}
ipcfp_status ipcfp_store_create_rpc_json(const uint8_t* cids, uint64_t n_blocks, const char* const* texts, const uint64_t* text_lens, uint64_t n_texts,
                                         int device, uint32_t flags, ipcfp_store** out, ipcfp_store_json_info* info) {
    return make_store(out, [&] {
        ipcfp_store_json_info si;
        Store* s = store_create_rpc_json(cids, n_blocks, texts, text_lens, n_texts, device, flags, si);
        if (info) *info = si;
        return s;
    });
}
ipcfp_status ipcfp_store_create_car(const uint8_t* car, uint64_t len, int device, uint32_t flags, ipcfp_store** out, ipcfp_store_json_info* info) {
    return make_store(out, [&] {
        ipcfp_store_json_info si;
        Store* s = store_create_car(car, len, device, flags, si);
        if (info) *info = si;
        return s;
    });
}
void ipcfp_store_destroy(ipcfp_store* s) { delete reinterpret_cast<Store*>(s); }
uint64_t ipcfp_store_n_blocks(const ipcfp_store* s) { return s ? reinterpret_cast<const Store*>(s)->n : 0; }
uint64_t ipcfp_store_first_bad_block(const ipcfp_store* s) { return s ? reinterpret_cast<const Store*>(s)->first_bad : UINT64_MAX; }
ipcfp_status ipcfp_store_get(ipcfp_store* s, const uint8_t cid[IPCFP_CID_LEN], uint8_t* buf, uint32_t cap, uint32_t* len, int* found) {
    return guard([&] {
        if (!s || !cid || !found) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        store_get(store_of(s), cid, buf, cap, len, found);
    });
}
ipcfp_status ipcfp_store_has(ipcfp_store* s, const uint8_t cid[IPCFP_CID_LEN], int* found) {
    return guard([&] {
        if (!s || !cid || !found) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        uint32_t len;
        store_get(store_of(s), cid, nullptr, 0, &len, found);
    });
}

ipcfp_status ipcfp_blake2b256_batch(const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets, const uint32_t* lengths, uint64_t n, int device,
                                    uint8_t* out) {
    return guard([&] { hash_batch(0, blob, blob_size, offsets, lengths, n, device, out); });
}
ipcfp_status ipcfp_keccak256_batch(const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets, const uint32_t* lengths, uint64_t n, int device,
                                   uint8_t* out) {
    return guard([&] { hash_batch(1, blob, blob_size, offsets, lengths, n, device, out); });
}
ipcfp_status ipcfp_sha256_batch(const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets, const uint32_t* lengths, uint64_t n, int device,
                                uint8_t* out) {
    return guard([&] { hash_batch(2, blob, blob_size, offsets, lengths, n, device, out); });
}
ipcfp_status ipcfp_compute_mapping_slots(const uint8_t* keys32, const uint64_t* slot_indices, uint64_t n, int device, uint8_t* out) {
    return guard([&] { mapping_slots(keys32, slot_indices, n, device, out); });
}

ipcfp_status ipcfp_generate_event_proof(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_spec* spec, uint32_t flags,
                                        ipcfp_event_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_event_proof(st, td, spec, flags, false, 0, 0); });
}
ipcfp_status ipcfp_generate_event_proof_shard(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_spec* spec, uint64_t lo, uint64_t hi,
                                              uint32_t world_size, uint32_t rank, uint32_t flags, ipcfp_event_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_event_proof(st, td, spec, flags, true, lo, hi); });
}
void ipcfp_event_result_free(ipcfp_event_result* r) { if (r) event_result_free(r); }

ipcfp_status ipcfp_tipset_upload(ipcfp_store* s, const ipcfp_tipset_desc* t, ipcfp_tipset** out) {
    return make_resident(s, out, [&](Store* st, TipsetDev& td) { tipset_upload(st, t, td); });
}
void ipcfp_tipset_free(ipcfp_tipset* t) { delete reinterpret_cast<TipsetDev*>(t); }
ipcfp_status ipcfp_tipset_upload_json(ipcfp_store* s, const char* parent, uint64_t parent_len, const char* child, uint64_t child_len,
                                      const char* receipts, uint64_t receipts_len, ipcfp_tipset** out) {
    return make_resident(s, out, [&](Store* st, TipsetDev& td) {
        tipset_upload_json(st, parent, parent_len, child, child_len, receipts, receipts_len, td);
    });
}
ipcfp_status ipcfp_tipset_describe(ipcfp_tipset* t, int with_events_roots, ipcfp_tipset_info* out) {
    return guard([&] {
        if (!t || !out) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        tipset_describe(tipset_of(t), with_events_roots != 0, out);
    });
}
ipcfp_status ipcfp_generate_event_proof_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_event_spec* spec, uint32_t flags,
                                                 ipcfp_event_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_event_proof(st, td, spec, flags, false, 0, 0); });
}
ipcfp_status ipcfp_generate_event_proof_shard_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_event_spec* spec, uint64_t lo, uint64_t hi,
                                                       uint32_t world_size, uint32_t rank, uint32_t flags, ipcfp_event_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_event_proof(st, td, spec, flags, true, lo, hi); });
}
ipcfp_status ipcfp_generate_log_proof_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_log_filter* filter, uint32_t flags,
                                               ipcfp_event_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_log_proof(st, td, filter, flags); });
}
ipcfp_status ipcfp_generate_log_proof(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_log_filter* filter, uint32_t flags,
                                      ipcfp_event_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_log_proof(st, td, filter, flags); });
}
ipcfp_status ipcfp_generate_message_log_proof_resident(ipcfp_store* s, ipcfp_tipset* t, const uint8_t* message_cids, uint64_t n,
                                                       const ipcfp_log_filter* filter, uint32_t flags, uint64_t* exec_indices, ipcfp_event_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) {
        return generate_message_log_proof(st, td, message_cids, n, filter, flags, exec_indices);
    });
}
ipcfp_status ipcfp_generate_message_log_proof(ipcfp_store* s, const ipcfp_tipset_desc* t, const uint8_t* message_cids, uint64_t n,
                                              const ipcfp_log_filter* filter, uint32_t flags, uint64_t* exec_indices, ipcfp_event_result** out) {
    return produce(s != nullptr, out, [&] {
        message_request_check(message_cids, n, filter, true, exec_indices);   // before the upload: no device work for a refused request
        return with_uploaded_tipset(store_of(s), t, [&](Store* st, TipsetDev& td) {
            return generate_message_log_proof(st, td, message_cids, n, filter, flags, exec_indices);
        });
    });
}
void* ipcfp_store_stream(ipcfp_store* s) { return s ? (void*)store_of(s)->stream : nullptr; }

ipcfp_status ipcfp_read_storage_slots(ipcfp_store* s, const uint8_t root[IPCFP_CID_LEN], const uint8_t* slots, uint64_t k, ipcfp_slot_result** out) {
    return produce(s && root && (!k || slots), out, [&] { return read_storage_slots(store_of(s), root, slots, k); });
}
void ipcfp_slot_result_free(ipcfp_slot_result* r) { if (r) slot_result_free(r); }

ipcfp_status ipcfp_generate_storage_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* specs, uint64_t n,
                                           ipcfp_storage_result** out) {
    return produce(s != nullptr, out, [&] {
        if (!t) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
        return generate_storage_proofs(store_of(s), t->child_cid, t->child_parent_state_root, specs, n);
    });
}
void ipcfp_storage_result_free(ipcfp_storage_result* r) { if (r) storage_result_free(r); }

ipcfp_status ipcfp_generate_storage_path_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_path* paths, uint64_t n, uint32_t flags,
                                                         ipcfp_path_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_storage_path_proofs(st, td, paths, n, flags); });
}
ipcfp_status ipcfp_plan_fetch_storage_paths_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_path* paths, uint64_t n, uint32_t flags,
                                                     ipcfp_fetch_plan** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) {
        plan_flags_check(flags);
        return make_plan([&](FetchPlan& p) { plan_fetch_storage_paths(st, td, paths, n, p); });
    });
}
ipcfp_status ipcfp_verify_storage_paths(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs, uint64_t n_proofs,
                                        const ipcfp_storage_path* paths, uint64_t n_paths, ipcfp_path_result** out) {
    return produce(s != nullptr, out, [&] { return verify_storage_paths(store_of(s), t, proofs, n_proofs, paths, n_paths); });
}
void ipcfp_path_result_free(ipcfp_path_result* r) { if (r) path_result_free(r); }

// generate_proof_bundle (proofs/generator.rs:25-95): the tipset uploaded, then the resident call's body without flags
ipcfp_status ipcfp_generate_proof_bundle(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                         const ipcfp_event_spec* especs, uint64_t n_especs, ipcfp_bundle** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_proof_bundle(st, td, sspecs, n_sspecs, especs, n_especs, 0); });
}
ipcfp_status ipcfp_generate_proof_bundle_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                                  const ipcfp_event_spec* especs, uint64_t n_especs, uint32_t flags, ipcfp_bundle** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_proof_bundle(st, td, sspecs, n_sspecs, especs, n_especs, flags); });
}
ipcfp_status ipcfp_generate_log_bundle_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                                const ipcfp_log_filter* filters, uint64_t n_filters, uint32_t flags, ipcfp_bundle** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_log_bundle(st, td, sspecs, n_sspecs, filters, n_filters, flags); });
}
ipcfp_status ipcfp_generate_log_bundle(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                       const ipcfp_log_filter* filters, uint64_t n_filters, uint32_t flags, ipcfp_bundle** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_log_bundle(st, td, sspecs, n_sspecs, filters, n_filters, flags); });
}
void ipcfp_bundle_free(ipcfp_bundle* b) { delete reinterpret_cast<BundleBox*>(b); }

ipcfp_status ipcfp_plan_fetch_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                       const ipcfp_event_spec* especs, uint64_t n_especs, uint32_t flags, ipcfp_fetch_plan** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) {
        plan_flags_check(flags);
        return make_plan([&](FetchPlan& p) { plan_fetch(st, td, sspecs, n_sspecs, especs, n_especs, p); });
    });
}
ipcfp_status ipcfp_plan_fetch(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                              const ipcfp_event_spec* especs, uint64_t n_especs, uint32_t flags, ipcfp_fetch_plan** out) {
    return produce(s != nullptr, out, [&] {
        plan_flags_check(flags);
        return with_uploaded_tipset(store_of(s), t, [&](Store* st, TipsetDev& td) {
            return make_plan([&](FetchPlan& p) { plan_fetch(st, td, sspecs, n_sspecs, especs, n_especs, p); });
        });
    });
}
ipcfp_status ipcfp_plan_fetch_log_bundle_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_storage_spec* sspecs, uint64_t n_sspecs,
                                                  const ipcfp_log_filter* filters, uint64_t n_filters, uint32_t flags, ipcfp_fetch_plan** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) {
        plan_flags_check(flags);
        return make_plan([&](FetchPlan& p) { plan_fetch(st, td, sspecs, n_sspecs, nullptr, 0, p, filters, n_filters); });
    });
}
// the bundle plan of one filter and no storage spec; a refused filter has no index
ipcfp_status ipcfp_plan_fetch_log_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_log_filter* filter, uint32_t flags, ipcfp_fetch_plan** out) {
    return produce(s && t && filter, out, [&] {
        plan_flags_check(flags);
        log_filter_check(filter);
        return make_plan([&](FetchPlan& p) { plan_fetch(store_of(s), tipset_of(t), nullptr, 0, nullptr, 0, p, filter, 1); });
    });
}
ipcfp_status ipcfp_plan_fetch_message_log_resident(ipcfp_store* s, ipcfp_tipset* t, const uint8_t* message_cids, uint64_t n,
                                                   const ipcfp_log_filter* filter, uint32_t flags, ipcfp_fetch_plan** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) {
        plan_flags_check(flags);
        return make_plan([&](FetchPlan& p) { plan_fetch_messages(st, td, message_cids, n, filter, p); });
    });
}
void ipcfp_fetch_plan_free(ipcfp_fetch_plan* p) { delete reinterpret_cast<FetchPlanBox*>(p); }

struct ResolveBox {
    ipcfp_resolve_result r;   // must stay first
    ResolveOut out;
};
ipcfp_status ipcfp_resolve_addresses(ipcfp_store* s, const uint8_t state_root[IPCFP_CID_LEN], const ipcfp_address* addrs, uint64_t n,
                                     ipcfp_resolve_result** out) {
    return produce(s && state_root, out, [&] {
        std::unique_ptr<ResolveBox> box(new ResolveBox());
        resolve_addresses(store_of(s), state_root, addrs, n, box->out);
        ipcfp_resolve_result& r = box->r;
        memset(&r, 0, sizeof r);
        r.n = n;
        r.actor_ids = box->out.ids.data();
        r.status = box->out.status.data();
        r.init_status = box->out.init_status;
        r.n_missing = box->out.missing.size() / 38;
        r.missing_cids = box->out.missing.data();
        box->out.wit.fill(r.witness);
        r.ms_total = box->out.ms_total;
        r.ms_lookup = box->out.ms_lookup;
        return &box.release()->r;
    });
}
void ipcfp_resolve_result_free(ipcfp_resolve_result* r) { delete reinterpret_cast<ResolveBox*>(r); }
ipcfp_status ipcfp_address_parse(const char* text, uint64_t len, ipcfp_address* out) {
    return guard([&] {
        if (!text || !out) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        address_parse(text, len, *out);
    });
}
ipcfp_status ipcfp_address_from_eth(const uint8_t eth[20], ipcfp_address* out) {
    return guard([&] {
        if (!eth || !out) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        address_from_eth(eth, *out);
    });
}

ipcfp_status ipcfp_generate_message_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const uint8_t* message_cids, uint64_t n, uint32_t flags,
                                                    ipcfp_message_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_message_proofs(st, td, message_cids, n, flags); });
}
ipcfp_status ipcfp_generate_message_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const uint8_t* message_cids, uint64_t n, uint32_t flags,
                                           ipcfp_message_result** out) {
    return produce(s != nullptr, out, [&] {
        message_proof_check(message_cids, n, flags);   // before the upload: no device work for a refused request
        return with_uploaded_tipset(store_of(s), t, [&](Store* st, TipsetDev& td) { return generate_message_proofs(st, td, message_cids, n, flags); });
    });
}
void ipcfp_message_result_free(ipcfp_message_result* r) { if (r) message_result_free(r); }
ipcfp_status ipcfp_plan_fetch_message_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const uint8_t* message_cids, uint64_t n, uint32_t flags,
                                                      ipcfp_fetch_plan** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) {
        return make_plan([&](FetchPlan& p) { plan_fetch_message_proofs(st, td, message_cids, n, flags, p); });
    });
}
ipcfp_status ipcfp_verify_message_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_message_proof* proofs, uint64_t n,
                                         const uint8_t* data_blob, uint64_t data_blob_size, uint32_t flags, uint8_t* results) {
    return guard([&] {
        if (!s) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        verify_message_proofs(store_of(s), t, proofs, n, data_blob, data_blob_size, flags, results);
    });
}

ipcfp_status ipcfp_generate_actor_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_address* addrs, uint64_t n,
                                                  const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags, ipcfp_actor_result** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) { return generate_actor_proofs(st, td, addrs, n, evm_code_cids, n_evm, flags); });
}
ipcfp_status ipcfp_generate_actor_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_address* addrs, uint64_t n,
                                         const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags, ipcfp_actor_result** out) {
    return produce(s != nullptr, out, [&] {
        actor_request_check(addrs, n, evm_code_cids, n_evm, flags);   // before the upload: no device work for a refused request
        return with_uploaded_tipset(store_of(s), t, [&](Store* st, TipsetDev& td) {
            return generate_actor_proofs(st, td, addrs, n, evm_code_cids, n_evm, flags);
        });
    });
}
void ipcfp_actor_result_free(ipcfp_actor_result* r) { if (r) actor_result_free(r); }
ipcfp_status ipcfp_plan_fetch_actor_proofs_resident(ipcfp_store* s, ipcfp_tipset* t, const ipcfp_address* addrs, uint64_t n,
                                                    const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags, ipcfp_fetch_plan** out) {
    return on_tipset(s, t, out, [&](Store* st, TipsetDev& td) {
        return make_plan([&](FetchPlan& p) { plan_fetch_actor_proofs(st, td, addrs, n, evm_code_cids, n_evm, flags, p); });
    });
}
ipcfp_status ipcfp_verify_actor_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_actor_proof* proofs, uint64_t n,
                                       const uint8_t* evm_code_cids, uint64_t n_evm, uint32_t flags, uint8_t* results) {
    return guard([&] {
        if (!s) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        verify_actor_proofs(store_of(s), t, proofs, n, evm_code_cids, n_evm, flags, results);
    });
}

ipcfp_status ipcfp_verify_event_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs, uint64_t n, const uint8_t* blob,
                                       uint64_t blob_size, const ipcfp_event_spec* filter, uint8_t* results) {
    return guard([&] {
        if (!s) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        verify_event_proofs(store_of(s), t, proofs, n, blob, blob_size, filter, results);
    });
}
// check_event = the set of one filter; a refused filter has no index
ipcfp_status ipcfp_verify_event_proofs_log(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs, uint64_t n, const uint8_t* blob,
                                           uint64_t blob_size, const ipcfp_log_filter* filter, uint8_t* results) {
    return guard([&] {
        if (!s || !filter) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        try { verify_event_proofs(store_of(s), t, proofs, n, blob, blob_size, nullptr, results, filter, 1); }
        catch (Error& e) {
            if (e.status == IPCFP_ERR_INVALID_ARG && e.index == 0) e.index = UINT64_MAX;
            throw;
        }
    });
}
ipcfp_status ipcfp_verify_event_proofs_any(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs, uint64_t n, const uint8_t* blob,
                                           uint64_t blob_size, const ipcfp_log_filter* filters, uint64_t n_filters, uint8_t* results) {
    return guard([&] {
        if (!s) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        verify_event_proofs(store_of(s), t, proofs, n, blob, blob_size, nullptr, results, filters, n_filters);
    });
}
ipcfp_status ipcfp_verify_storage_proofs(ipcfp_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs, uint64_t n, uint8_t* results) {
    return guard([&] {
        if (!s) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        verify_storage_proofs(store_of(s), t, proofs, n, results);
    });
}

ipcfp_status ipcfp_verify_bundle_json(const char* json, uint64_t len, int device, ipcfp_trusted_parent_ts_fn trusted_parent,
                                      ipcfp_trusted_child_header_fn trusted_child, void* trust_ctx, const ipcfp_event_spec* filter,
                                      ipcfp_bundle_verdict** out) {
    return produce(json != nullptr, out, [&] { return verify_bundle_json(json, len, device, trusted_parent, trusted_child, trust_ctx, filter); });
}
ipcfp_status ipcfp_verify_bundle_json_any(const char* json, uint64_t len, int device, ipcfp_trusted_parent_ts_fn trusted_parent,
                                          ipcfp_trusted_child_header_fn trusted_child, void* trust_ctx, const ipcfp_log_filter* filters,
                                          uint64_t n_filters, ipcfp_bundle_verdict** out) {
    return produce(json != nullptr, out, [&] {
        LogFilterSet::check(filters, n_filters);
        return verify_bundle_json(json, len, device, trusted_parent, trusted_child, trust_ctx, nullptr, filters, n_filters);
    });
}
void ipcfp_bundle_verdict_free(ipcfp_bundle_verdict* v) { if (v) bundle_verdict_free(v); }

ipcfp_status ipcfp_comm_unique_id(uint8_t id[IPCFP_COMM_ID_BYTES]) {
    return guard([&] {
        if (!id) throw Error(IPCFP_ERR_INVALID_ARG, "null argument");
        comm_unique_id(id);
    });
}
ipcfp_status ipcfp_comm_init(const uint8_t id[IPCFP_COMM_ID_BYTES], uint32_t world_size, uint32_t rank, int device, ipcfp_comm** out) {
    return produce(id != nullptr, out, [&] { return reinterpret_cast<ipcfp_comm*>(comm_init(id, world_size, rank, device)); });
}
void ipcfp_comm_destroy(ipcfp_comm* c) { if (c) comm_destroy(reinterpret_cast<Comm*>(c)); }
ipcfp_status ipcfp_generate_event_proof_sharded(ipcfp_comm* c, ipcfp_store* s, ipcfp_tipset* t, const ipcfp_event_spec* spec, const uint64_t* bounds,
                                                uint32_t flags, ipcfp_event_result** out) {
    return produce(c && s && t && bounds, out, [&] {
        Comm* cm = reinterpret_cast<Comm*>(c);
        const uint32_t W = comm_world(cm), r = comm_rank(cm);
        TipsetDev& td = tipset_of(t);
        for (uint32_t k = 0; k < W; k++) if (bounds[k] > bounds[k + 1]) throw Error(IPCFP_ERR_INVALID_ARG, "shard bounds must ascend");
        if (bounds[0] != 0 || bounds[W] != td.n_receipts) throw Error(IPCFP_ERR_INVALID_ARG, "shard bounds must cover [0, n_receipts)");
        return generate_event_proof(store_of(s), td, spec, flags, true, bounds[r], bounds[r + 1], cm);
    });
}

}  // extern "C"
