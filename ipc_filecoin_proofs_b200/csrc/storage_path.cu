// storage_path.cu — storage paths (DESIGN.md §3, "Storage paths"): a Solidity value named by its access path, its slots derived and
// its words proven on the device. Per-path code: storage_path_items.cuh; per-proof code: storage.cuh.
//   k_path_slots        one thread per path: chained Keccak-256 and u256 adds → the fixed specs (length words, value or header words)
//   k_path_proofs       one warp per spec, lane 0 walks (k_storage_proofs' shape): wave 1 over the fixed specs, wave 2 over the data slots
//   k_path_expand       one thread per path: status, data-slot count and value length from wave 1's words; then two scans (prims.cu)
//   k_path_place_specs  one thread per path: the expanded specs in their final positions, the data slots keccak256(slot) + j
//   k_path_place        one warp per fixed spec: wave 1's proof and recorder list moved to its final position
//   k_path_values       one thread per path: the value from the proofs (and, for the verifier, whether every spec had a good proof)
//   k_path_lookup       the verifier's wave: each spec's proof found in the caller's list (binary search over (actor_id, slot))
#include <algorithm>
#include <cstring>
#include <numeric>

#include "engine.cuh"
#include "prims.cuh"
#include "storage_path_items.cuh"

namespace ipcfp {

__global__ void __launch_bounds__(128) k_path_slots(PathsDev P, ipcfp_storage_spec* fixed, ipcfp_path_value* info) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.n) return;
    const PathDev& p = P.paths[t];
    ipcfp_path_value v;
    memset(&v, 0, sizeof v);
    path_fixed_specs(p, P.steps + p.step_off, P.keys, fixed + p.fixed_off, v.slot, v.byte_offset);
    v.valid = 1;
    info[t] = v;
}

// One spec per warp. owner / pos: the spec's path and its position in the path (a failure's index is (path << 24) | position, so that
// the smallest key is the first failing path's first failing spec in expanded order). skip_fixed (wave 2, over the final list): the
// fixed specs are not proven again. Optional outputs: rec_list / rec_n / wbits (generate), ok (1: the spec was proven), err.
__global__ void __launch_bounds__(128) k_path_proofs(StorageArgs a, const uint32_t* owner, const uint32_t* pos, const PathDev* skip_fixed, uint8_t* ok) {
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= a.n || (threadIdx.x & 31)) return;
    if (skip_fixed && pos[t] < skip_fixed[owner[t]].n_fixed) return;
    Recorder rec{a.rec_list ? a.rec_list + t * REC_CAP : nullptr, 0, a.wbits, false};
    rec.rank_of = a.store.rank_of;
    ipcfp_storage_proof q;
    memset(&q, 0, sizeof q);   // tail padding included: the proofs reach the caller byte for byte
    Fail f{0, 0};
    const uint64_t key_index = ((uint64_t)owner[t] << PATH_POS_BITS) | pos[t];
    bool good = storage_proof_one(a, t, rec, q, f);
    if (good && rec.overflow) { good = false; f = Fail{DC_UNSUPPORTED, 2}; }
    if (!good && a.err) report_error(a.err, ST_STORAGE, key_index, f.code, f.detail);
    if (a.rec_n) a.rec_n[t] = good ? rec.n : 0;
    if (ok) ok[t] = good;
    if (good) a.out[t] = q;
}

__global__ void __launch_bounds__(128) k_path_expand(PathsDev P, const ipcfp_storage_proof* fixed, const uint8_t* ok, ipcfp_path_value* info, uint32_t* cnt,
                                                     uint32_t* vlen) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.n) return;
    const PathDev& p = P.paths[t];
    const PathExpansion e = path_expand(p, P.steps + p.step_off, fixed + p.fixed_off, ok + p.fixed_off);
    info[t].status = e.status;
    cnt[t] = p.n_fixed + e.n_data;
    vlen[t] = e.value_len;
}

__global__ void __launch_bounds__(128) k_path_place_specs(PathsDev P, const ipcfp_storage_spec* fixed, const uint32_t* cnt, const uint64_t* first,
                                                          const uint32_t* vlen, const uint64_t* voff, ipcfp_path_value* info, ipcfp_storage_spec* specs,
                                                          uint32_t* owner, uint32_t* pos) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.n) return;
    const PathDev& p = P.paths[t];
    const uint64_t f = first[t];
    info[t].first_spec = f;
    info[t].n_specs = cnt[t];
    info[t].value_off = voff[t];
    info[t].value_len = vlen[t];
    for (uint32_t k = 0; k < p.n_fixed; k++) { specs[f + k] = fixed[p.fixed_off + k]; owner[f + k] = (uint32_t)t; pos[f + k] = k; }
    const uint32_t n_data = cnt[t] - p.n_fixed;
    if (!n_data) return;
    uint8_t base[32];
    keccak_key_slot(nullptr, 0, info[t].slot, base);
    for (uint32_t j = 0; j < n_data; j++) {
        ipcfp_storage_spec& sp = specs[f + p.n_fixed + j];
        sp.actor_id = p.actor_id;
        path_data_slot(base, j, sp.slot);
        owner[f + p.n_fixed + j] = (uint32_t)t;
        pos[f + p.n_fixed + j] = p.n_fixed + j;
    }
}

// wave 1's results at their final positions: one warp per fixed spec, the lanes copy the recorder list
__global__ void __launch_bounds__(128) k_path_place(const ipcfp_storage_proof* w1, const uint32_t* w1_rec, const uint32_t* w1_recn, const uint8_t* w1_ok,
                                                    uint64_t n_fixed, const uint32_t* owner, const uint32_t* pos, const ipcfp_path_value* info,
                                                    ipcfp_storage_proof* out, uint32_t* rec, uint32_t* recn, uint8_t* ok) {
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (t >= n_fixed) return;
    const uint64_t f = info[owner[t]].first_spec + pos[t];
    if (lane == 0) { out[f] = w1[t]; ok[f] = w1_ok[t]; if (recn) recn[f] = w1_recn[t]; }
    if (!rec) return;
    const uint32_t c = w1_recn[t];
    for (uint32_t k = lane; k < c; k += 32) rec[f * REC_CAP + k] = w1_rec[t * REC_CAP + k];
}

__global__ void __launch_bounds__(128) k_path_values(PathsDev P, const ipcfp_storage_proof* proofs, const uint8_t* ok, ipcfp_path_value* info, uint8_t* blob) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.n) return;
    const PathDev& p = P.paths[t];
    ipcfp_path_value& v = info[t];
    uint32_t good = 1;
    for (uint64_t k = 0; k < v.n_specs; k++) good &= ok[v.first_spec + k];
    v.valid = good;
    path_value(p, proofs + v.first_spec, (uint32_t)(v.n_specs - p.n_fixed), (uint32_t)v.value_len, blob + v.value_off);
}

// the verifier: spec t's proof from the caller's list (order: indices sorted by (actor_id, slot), verified ones first); ok = it exists
// and ipcfp_verify_storage_proofs accepted it
__global__ void __launch_bounds__(128) k_path_lookup(const ipcfp_storage_spec* specs, uint64_t n, const uint32_t* owner, const uint32_t* pos, const PathDev* skip_fixed,
                                                     const ipcfp_storage_proof* proofs, const uint32_t* order, const uint8_t* results, uint64_t n_proofs,
                                                     ipcfp_storage_proof* out, uint8_t* ok) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    if (skip_fixed && pos[t] < skip_fixed[owner[t]].n_fixed) return;
    const int64_t i = proof_find(proofs, order, n_proofs, specs[t].actor_id, specs[t].slot);
    ok[t] = i >= 0 && results[i];
    if (i >= 0) out[t] = proofs[i]; else memset(&out[t], 0, sizeof out[t]);
}

// ------------------------------------------------------------------------------------------ host
// The caller's paths, checked and gathered for one upload; owner / pos of every fixed spec
struct PathPack {
    std::vector<PathDev> paths;
    std::vector<PathStepDev> steps;
    std::vector<uint8_t> keys;
    std::vector<uint32_t> owner, pos;
    uint64_t n_fixed = 0;
};
static void path_pack(const ipcfp_storage_path* paths, uint64_t n, PathPack& pk) {
    if (n && !paths) throw Error(IPCFP_ERR_INVALID_ARG, "null paths");
    if (n > IPCFP_PATH_MAX_PATHS) throw Error(IPCFP_ERR_INVALID_ARG, "more than IPCFP_PATH_MAX_PATHS paths");
    pk.paths.resize(n);
    for (uint64_t i = 0; i < n; i++) {
        const ipcfp_storage_path& q = paths[i];
        auto refuse = [&](const char* why) { throw Error(IPCFP_ERR_INVALID_ARG, std::string("storage path: ") + why, i); };
        if (q.n_steps > IPCFP_PATH_MAX_STEPS) refuse("more than IPCFP_PATH_MAX_STEPS steps");
        if (q.n_steps && !q.steps) refuse("null steps");
        if (q.kind != IPCFP_PATH_WORDS && q.kind != IPCFP_PATH_BYTES) refuse("unknown kind");
        if (q.kind == IPCFP_PATH_WORDS && (q.n_words == 0 || q.n_words > IPCFP_PATH_MAX_WORDS)) refuse("n_words out of 1..IPCFP_PATH_MAX_WORDS");
        PathDev& p = pk.paths[i];
        memset(&p, 0, sizeof p);
        p.actor_id = q.actor_id;
        memcpy(p.base_slot, q.base_slot, 32);
        p.n_steps = q.n_steps; p.kind = q.kind; p.n_words = q.kind == IPCFP_PATH_WORDS ? q.n_words : 0;
        p.step_off = pk.steps.size();
        uint32_t n_array = 0;
        for (uint32_t j = 0; j < q.n_steps; j++) {
            const ipcfp_path_step& s = q.steps[j];
            PathStepDev d;
            memset(&d, 0, sizeof d);
            d.op = s.op;
            if (s.op == IPCFP_PATH_MAPPING) {
                if (s.key_len > IPCFP_PATH_MAX_KEY) refuse("key over IPCFP_PATH_MAX_KEY bytes");
                if (s.key_len && !s.key) refuse("null key");
                d.key_len = s.key_len;
                d.key_off = pk.keys.size();
                pk.keys.insert(pk.keys.end(), s.key, s.key + s.key_len);
            } else if (s.op == IPCFP_PATH_ARRAY || s.op == IPCFP_PATH_STATIC) {
                if (s.elem_bytes > 32) refuse("elem_bytes over 32");
                if (s.elem_slots == 0) refuse("elem_slots is 0");
                d.index = s.index; d.elem_slots = s.elem_slots; d.elem_bytes = s.elem_bytes;
                n_array += s.op == IPCFP_PATH_ARRAY;
            } else if (s.op == IPCFP_PATH_FIELD) {
                d.index = s.index;
            } else refuse("unknown step op");
            pk.steps.push_back(d);
        }
        p.n_fixed = path_n_fixed(n_array, q.kind, q.n_words);
        p.fixed_off = pk.n_fixed;
        for (uint32_t k = 0; k < p.n_fixed; k++) { pk.owner.push_back((uint32_t)i); pk.pos.push_back(k); }
        pk.n_fixed += p.n_fixed;
    }
    pk.keys.resize(pk.keys.size() + 16, 0);
}

// The pack on the device (one upload) and the buffers every call shares: the fixed specs, wave 1's proofs and ok flags, the per-path
// results; up to the expansion's scans
struct PathRun {
    Store* s;
    cudaStream_t st;
    PathsDev P{};
    uint64_t n = 0, n_fixed = 0;
    PinnedArray stage;   // the upload's pinned source, kept until the run ends (every call synchronises before that)
    AsyncBuf<uint8_t> up;
    const uint32_t *owner1 = nullptr, *pos1 = nullptr;
    AsyncBuf<ipcfp_storage_spec> fixed;
    AsyncBuf<ipcfp_storage_proof> w1;
    AsyncBuf<uint8_t> w1_ok;
    AsyncBuf<ipcfp_path_value> info;
    AsyncBuf<uint32_t> cnt, vlen;
    AsyncBuf<uint64_t> first, voff, scratch, totals;
    uint64_t n_specs = 0, value_bytes = 0;
    // the final list (after size())
    AsyncBuf<ipcfp_storage_spec> specs;
    AsyncBuf<uint32_t> owner, pos;
    AsyncBuf<ipcfp_storage_proof> out;
    AsyncBuf<uint8_t> ok, values;

    PathRun(Store* store, const PathPack& pk, const uint8_t* child_cid, const uint8_t* state_root) : s(store), st(store->stream) {
        n = pk.paths.size();
        n_fixed = pk.n_fixed;
        auto up16 = [](uint64_t x) { return (x + 15) & ~15ull; };
        const uint64_t o_steps = up16(n * sizeof(PathDev)), o_keys = o_steps + up16(pk.steps.size() * sizeof(PathStepDev)),
                       o_own = o_keys + up16(pk.keys.size()), o_pos = o_own + up16(4 * n_fixed), o_cids = o_pos + up16(4 * n_fixed),
                       size = o_cids + 128;
        stage = PinnedArray(s->pool, size);
        uint8_t* b = stage.as<uint8_t>();
        memset(b, 0, size);
        if (n) memcpy(b, pk.paths.data(), n * sizeof(PathDev));
        if (!pk.steps.empty()) memcpy(b + o_steps, pk.steps.data(), pk.steps.size() * sizeof(PathStepDev));
        memcpy(b + o_keys, pk.keys.data(), pk.keys.size());
        if (n_fixed) { memcpy(b + o_own, pk.owner.data(), 4 * n_fixed); memcpy(b + o_pos, pk.pos.data(), 4 * n_fixed); }
        if (child_cid) memcpy(b + o_cids, child_cid, 38);
        if (state_root) memcpy(b + o_cids + 64, state_root, 38);
        up.alloc(size, st);
        IPCFP_CUDA(cudaMemcpyAsync(up.p, b, size, cudaMemcpyHostToDevice, st));
        P = PathsDev{(const PathDev*)up.p, (const PathStepDev*)(up.p + o_steps), up.p + o_keys, n};
        owner1 = (const uint32_t*)(up.p + o_own);
        pos1 = (const uint32_t*)(up.p + o_pos);
        child = up.p + o_cids;
        sroot = up.p + o_cids + 64;
        fixed.alloc(n_fixed + 1, st);
        w1.alloc(n_fixed + 1, st);
        w1_ok.alloc(n_fixed + 16, st);
        w1_ok.zero();
        info.alloc(n + 1, st);
        cnt.alloc(n + 1, st); vlen.alloc(n + 1, st);
        first.alloc(n + 1, st); voff.alloc(n + 1, st);
        scratch.alloc(scan_scratch_elems(n) + 8, st);
        totals.alloc(2, st);
        totals.zero();
    }
    const uint8_t *child = nullptr, *sroot = nullptr;

    void slots() { if (n) { k_path_slots<<<div_up(n, 128), 128, 0, st>>>(P, fixed.p, info.p); IPCFP_LAUNCH_CHECK(); } }
    StorageArgs args(const ipcfp_storage_spec* sp, uint64_t m, ipcfp_storage_proof* o) const {
        StorageArgs a{};
        a.store = s->view; a.child_cid = child; a.state_root_json = sroot; a.specs = sp; a.n = m; a.out = o;
        return a;
    }
    void proofs(const StorageArgs& a, const uint32_t* own, const uint32_t* ps, bool skip_fixed, uint8_t* okp) {
        if (a.n) { k_path_proofs<<<div_up(a.n * 32, 128), 128, 0, st>>>(a, own, ps, skip_fixed ? P.paths : nullptr, okp); IPCFP_LAUNCH_CHECK(); }
    }
    // the expansion and its scans, then host synchronisation 1: the size of the final list and of the values
    void size(PinnedArray& words) {
        if (n) { k_path_expand<<<div_up(n, 128), 128, 0, st>>>(P, w1.p, w1_ok.p, info.p, cnt.p, vlen.p); IPCFP_LAUNCH_CHECK(); }
        exclusive_scan_u32(cnt.p, first.p, n, totals.p, scratch.p, st);
        exclusive_scan_u32(vlen.p, voff.p, n, totals.p + 1, scratch.p, st);
        IPCFP_CUDA(cudaMemcpyAsync(words.p, totals.p, 16, cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
        n_specs = words.as<uint64_t>()[0];
        value_bytes = words.as<uint64_t>()[1];
        specs.alloc(n_specs + 1, st);
        owner.alloc(n_specs + 1, st); pos.alloc(n_specs + 1, st);
        out.alloc(n_specs + 1, st);
        ok.alloc(n_specs + 16, st);
        ok.zero();
        values.alloc(value_bytes + 16, st);
        if (n) {
            k_path_place_specs<<<div_up(n, 128), 128, 0, st>>>(P, fixed.p, cnt.p, first.p, vlen.p, voff.p, info.p, specs.p, owner.p, pos.p);
            IPCFP_LAUNCH_CHECK();
        }
    }
    void place(const uint32_t* w1_rec, const uint32_t* w1_recn, uint32_t* rec, uint32_t* recn) {
        if (n_fixed) {
            k_path_place<<<div_up(n_fixed * 32, 128), 128, 0, st>>>(w1.p, w1_rec, w1_recn, w1_ok.p, n_fixed, owner1, pos1, info.p, out.p, rec, recn, ok.p);
            IPCFP_LAUNCH_CHECK();
        }
    }
    void values_kernel() { if (n) { k_path_values<<<div_up(n, 128), 128, 0, st>>>(P, out.p, ok.p, info.p, values.p); IPCFP_LAUNCH_CHECK(); } }
};

struct PathResultBox {
    ipcfp_path_result r;   // must stay first
    PinnedArray info, specs, values;
    ~PathResultBox() { if (r.storage) storage_result_free(r.storage); }
};
// the per-path results, the specs and the values copied back (enqueued; on the host after the next synchronisation)
static std::unique_ptr<PathResultBox> result_box(PathRun& run) {
    std::unique_ptr<PathResultBox> box(new PathResultBox());
    memset(&box->r, 0, sizeof box->r);
    Store* s = run.s;
    box->info = PinnedArray(s->pool, (run.n + 1) * sizeof(ipcfp_path_value));
    box->specs = PinnedArray(s->pool, (run.n_specs + 1) * sizeof(ipcfp_storage_spec));
    box->values = PinnedArray(s->pool, run.value_bytes + 16);
    if (run.n) IPCFP_CUDA(cudaMemcpyAsync(box->info.p, run.info.p, run.n * sizeof(ipcfp_path_value), cudaMemcpyDeviceToHost, run.st));
    if (run.n_specs) IPCFP_CUDA(cudaMemcpyAsync(box->specs.p, run.specs.p, run.n_specs * sizeof(ipcfp_storage_spec), cudaMemcpyDeviceToHost, run.st));
    if (run.value_bytes) IPCFP_CUDA(cudaMemcpyAsync(box->values.p, run.values.p, run.value_bytes, cudaMemcpyDeviceToHost, run.st));
    ipcfp_path_result& r = box->r;
    r.n_paths = run.n; r.paths = box->info.as<ipcfp_path_value>();
    r.n_specs = run.n_specs; r.specs = box->specs.as<ipcfp_storage_spec>();
    r.value_blob = box->values.as<uint8_t>(); r.value_blob_size = run.value_bytes;
    return box;
}

ipcfp_path_result* generate_storage_path_proofs(Store* s, TipsetDev& td, const ipcfp_storage_path* paths, uint64_t n, uint32_t flags) {
    if (flags & ~(uint32_t)IPCFP_WITNESS_BY_REFERENCE) throw Error(IPCFP_ERR_INVALID_ARG, "unknown flag bit for storage paths");
    PathPack pk;
    path_pack(paths, n, pk);
    if (!td.has_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    const bool by_ref = (flags & IPCFP_WITNESS_BY_REFERENCE) != 0;
    if (by_ref && !s->caller_blob)
        throw Error(IPCFP_ERR_UNSUPPORTED, "IPCFP_WITNESS_BY_REFERENCE needs a store made from a caller's blob (ipcfp_store_create)");
    s->use();
    cudaStream_t st = s->stream;
    unsigned long long* dw = s->dev_words.p;
    Event ev[4];
    PathRun run(s, pk, td.child_cid, td.child_state_root);
    IPCFP_CUDA(cudaEventRecord(s->ev[EV_BEGIN], st));
    IPCFP_CUDA(cudaMemsetAsync(dw, 0xff, 8, st));
    AsyncBuf<uint32_t> wbits((s->n + 31) / 32 + 8, st), w1_rec(run.n_fixed * REC_CAP + 8, st), w1_recn(run.n_fixed + 8, st);
    wbits.zero();
    run.slots();
    IPCFP_CUDA(cudaEventRecord(ev[0], st));
    // wave 1: the fixed specs
    StorageArgs a1 = run.args(run.fixed.p, run.n_fixed, run.w1.p);
    a1.rec_list = w1_rec.p; a1.rec_n = w1_recn.p; a1.wbits = wbits.p; a1.err = dw;
    run.proofs(a1, run.owner1, run.pos1, false, run.w1_ok.p);
    IPCFP_CUDA(cudaEventRecord(ev[1], st));
    PinnedArray words(s->pool, 16);
    run.size(words);   // host synchronisation 1
    // wave 2: the data slots, into the final list; wave 1's results join them there
    AsyncBuf<uint32_t> rec(run.n_specs * REC_CAP + 8, st), recn(run.n_specs + 8, st);
    IPCFP_CUDA(cudaEventRecord(ev[2], st));
    run.place(w1_rec.p, w1_recn.p, rec.p, recn.p);
    w1_rec.release();   // wave 1's lists are in the final ones now: freed in stream order, so a call holds one copy of them
    StorageArgs a2 = run.args(run.specs.p, run.n_specs, run.out.p);
    a2.rec_list = rec.p; a2.rec_n = recn.p; a2.wbits = wbits.p; a2.err = dw;
    run.proofs(a2, run.owner.p, run.pos.p, true, run.ok.p);
    run.values_kernel();
    IPCFP_CUDA(cudaEventRecord(ev[3], st));
    std::unique_ptr<PathResultBox> box = result_box(run);
    uint64_t* hw = s->host_words.p;
    IPCFP_CUDA(cudaMemcpyAsync(hw + DW_ERR, dw, 8, cudaMemcpyDeviceToHost, st));   // read with the witness count's synchronisation
    box->r.storage = storage_result_finish(s, run.out.p, rec.p, recn.p, wbits.p, run.n_specs, by_ref);
    if (hw[DW_ERR] != IPCFP_NO_ERROR) {
        try { throw_storage_error(hw[DW_ERR]); }
        catch (Error& e) { e.index >>= PATH_POS_BITS; throw; }   // the path of the first failing spec
    }
    ipcfp_path_result& r = box->r;
    r.ms_total = r.storage->ms_total;
    r.ms_slots = elapsed_ms(s->ev[EV_BEGIN], ev[0]);
    r.ms_wave1 = elapsed_ms(ev[0], ev[1]);
    r.ms_wave2 = elapsed_ms(ev[2], ev[3]);
    r.ms_witness = elapsed_ms(ev[3], s->ev[EV_STORAGE_END]);
    r.host_syncs = 4;   // the size, then storage_result_finish's three (witness count, witness copy, end)
    return &box.release()->r;
}

void plan_fetch_storage_paths(Store* s, TipsetDev& td, const ipcfp_storage_path* paths, uint64_t n, FetchPlan& out) {
    PathPack pk;
    path_pack(paths, n, pk);
    if (!td.has_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    s->use();
    cudaStream_t st = s->stream;
    std::vector<ipcfp_storage_spec> specs;
    {
        PathRun run(s, pk, td.child_cid, td.child_state_root);
        run.slots();
        // wave 1 as far as the store goes: a spec that cannot be proven yet (a missing block, or one the generator will refuse) has no word
        run.proofs(run.args(run.fixed.p, run.n_fixed, run.w1.p), run.owner1, run.pos1, false, run.w1_ok.p);
        PinnedArray words(s->pool, 16);
        run.size(words);   // a BYTES path's data slots only where its header word was read
        specs.resize(run.n_specs);
        if (run.n_specs) IPCFP_CUDA(cudaMemcpyAsync(specs.data(), run.specs.p, run.n_specs * sizeof(ipcfp_storage_spec), cudaMemcpyDeviceToHost, st));
        IPCFP_CUDA(cudaStreamSynchronize(st));
    }
    // rule 4 over the expanded specs known so far
    plan_fetch(s, td, specs.data(), specs.size(), nullptr, 0, out);
}

ipcfp_path_result* verify_storage_paths(Store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs, uint64_t n_proofs,
                                        const ipcfp_storage_path* paths, uint64_t n_paths) {
    if (!t || !t->child_cid || !t->child_parent_state_root) throw Error(IPCFP_ERR_INVALID_ARG, "tipset descriptor lacks child_cid / parent_state_root");
    if (n_proofs && !proofs) throw Error(IPCFP_ERR_INVALID_ARG, "null proofs");
    if (n_proofs > UINT32_MAX) throw Error(IPCFP_ERR_INVALID_ARG, "too many proofs");
    PathPack pk;
    path_pack(paths, n_paths, pk);
    s->use();
    cudaStream_t st = s->stream;
    Event ev[5];
    IPCFP_CUDA(cudaEventRecord(ev[4], st));
    // every proof replayed over the witness store (its Err fails the call)
    std::vector<uint8_t> results(n_proofs + 1, 0);
    verify_storage_proofs(s, t, proofs, n_proofs, results.data());
    std::vector<uint32_t> order(n_proofs);
    std::iota(order.begin(), order.end(), 0u);
    std::sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
        const ipcfp_storage_proof &a = proofs[x], &b = proofs[y];
        if (a.actor_id != b.actor_id) return a.actor_id < b.actor_id;
        if (const int c = memcmp(a.slot, b.slot, 32)) return c < 0;
        if (results[x] != results[y]) return results[x] > results[y];
        return x < y;
    });
    AsyncBuf<ipcfp_storage_proof> d_proofs(n_proofs + 1, st);
    AsyncBuf<uint32_t> d_order(n_proofs + 1, st);
    AsyncBuf<uint8_t> d_res(n_proofs + 16, st);
    if (n_proofs) {
        IPCFP_CUDA(cudaMemcpyAsync(d_proofs.p, proofs, n_proofs * sizeof(ipcfp_storage_proof), cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(d_order.p, order.data(), n_proofs * 4, cudaMemcpyHostToDevice, st));
        IPCFP_CUDA(cudaMemcpyAsync(d_res.p, results.data(), n_proofs, cudaMemcpyHostToDevice, st));
    }
    PathRun run(s, pk, nullptr, nullptr);
    run.slots();
    IPCFP_CUDA(cudaEventRecord(ev[0], st));
    if (run.n_fixed) {
        k_path_lookup<<<div_up(run.n_fixed, 128), 128, 0, st>>>(run.fixed.p, run.n_fixed, run.owner1, run.pos1, nullptr, d_proofs.p, d_order.p, d_res.p, n_proofs,
                                                                 run.w1.p, run.w1_ok.p);
        IPCFP_LAUNCH_CHECK();
    }
    IPCFP_CUDA(cudaEventRecord(ev[1], st));
    PinnedArray words(s->pool, 16);
    run.size(words);
    IPCFP_CUDA(cudaEventRecord(ev[2], st));
    run.place(nullptr, nullptr, nullptr, nullptr);
    if (run.n_specs) {
        k_path_lookup<<<div_up(run.n_specs, 128), 128, 0, st>>>(run.specs.p, run.n_specs, run.owner.p, run.pos.p, run.P.paths, d_proofs.p, d_order.p, d_res.p,
                                                                n_proofs, run.out.p, run.ok.p);
        IPCFP_LAUNCH_CHECK();
    }
    run.values_kernel();
    IPCFP_CUDA(cudaEventRecord(ev[3], st));
    std::unique_ptr<PathResultBox> box = result_box(run);
    IPCFP_CUDA(cudaStreamSynchronize(st));
    ipcfp_path_result& r = box->r;
    r.ms_slots = elapsed_ms(ev[4], ev[0]);
    r.ms_wave1 = elapsed_ms(ev[0], ev[1]);
    r.ms_wave2 = elapsed_ms(ev[2], ev[3]);
    r.ms_total = elapsed_ms(ev[4], ev[3]);
    return &box.release()->r;
}

void path_result_free(ipcfp_path_result* r) { delete reinterpret_cast<PathResultBox*>(r); }

}  // namespace ipcfp
