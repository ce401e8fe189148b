// emu_message_select.cu — the per-item code of ipcfp_generate_message_log_proof (csrc/msg_select_items.cuh: msg_sort_key and
// msg_select_item of the request sort / k_msg_select, msg_match_item of k_msg_match) EXECUTED ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// Mode "select" (no argument), stdin: "n_exec n_req n_receipts", then exec_raw (n_exec CIDs in hex, one per line), exec_idx (n_exec positions into exec_raw, the
// execution order exec[i] = exec_raw[exec_idx[i]]), then the n_req requested CIDs in hex. stdout: the number of selected receipts, the
// selected receipts in ascending order, then every request's execution index (UINT64_MAX: not executed). tests/test_message_proof_host.py
// checks it against the Python selection (tests/oracle_messages.select).
//
// Mode "match <file>": a block set, a receipt list and the selected receipts (binary, little-endian: n_blocks u64, then per block CID[38],
// length u32, bytes; n_receipts u64, then per receipt has_root u8, events root CID[38]; n_sel u64, then the selected receipts u32
// ascending; n_emitters u32 and the emitters u64 of an all-wildcard log filter's emitter set). msg_match_item runs on every selected
// receipt, in a shuffled order as warps would. stdout: the error word as "err <stage> <index> <code>" (or "err none"), then per selected
// receipt "<i> <matched> <events> <bytes>". tests/test_message_proof_host.py checks it against tests/oracle_messages.py.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <vector>

#include "host_shims.h"
#define atomicAdd(p, v) (*(p) += (v))   // before the device headers, as host_shims.h does for atomicMin / atomicOr

#include "../../ipc_filecoin_proofs_b200/csrc/hashes.cuh"
#include "../../ipc_filecoin_proofs_b200/csrc/walk.cuh"
#ifndef __CUDA_ARCH__
#define prefetch_l2(p) ((void)0)   // inline PTX: nothing to do on the host
#endif
#include "../../ipc_filecoin_proofs_b200/csrc/msg_select_items.cuh"
#include "host_store.h"

using namespace ipcfp;

template <class T> static T get(FILE* f) { T v; if (fread(&v, sizeof v, 1, f) != 1) exit(2); return v; }

static int run_match(const char* path) {
    FILE* f = fopen(path, "rb");
    if (!f) return 2;
    const uint64_t nb = get<uint64_t>(f);
    std::vector<uint8_t> cids(38 * nb), blob;
    std::vector<uint64_t> offs(nb);
    std::vector<uint32_t> lens(nb);
    for (uint64_t k = 0; k < nb; k++) {
        if (fread(cids.data() + 38 * k, 1, 38, f) != 38) return 2;
        lens[k] = get<uint32_t>(f);
        offs[k] = blob.size();
        blob.resize(blob.size() + lens[k]);
        if (lens[k] && fread(blob.data() + offs[k], 1, lens[k], f) != lens[k]) return 2;
        blob.resize((blob.size() + 15) & ~(size_t)15);   // 16-aligned blocks, as the store lays them out
    }
    const uint64_t nr = get<uint64_t>(f);
    // device-shaped buffers: the roots padded by 64 bytes as the tipset upload pads them, per-receipt arrays of exactly n entries
    std::vector<uint8_t> roots(38 * nr + 64, 0), has(nr);
    for (uint64_t i = 0; i < nr; i++) {
        has[i] = get<uint8_t>(f);
        if (fread(roots.data() + 38 * i, 1, 38, f) != 38) return 2;
    }
    const uint64_t ns = get<uint64_t>(f);
    std::vector<uint32_t> sel(ns);
    for (auto& x : sel) x = get<uint32_t>(f);
    const uint32_t ne = get<uint32_t>(f);
    std::vector<uint64_t> em(ne);
    for (auto& x : em) x = get<uint64_t>(f);
    fclose(f);
    HostStore hs(cids.data(), offs.data(), lens.data(), blob.data(), blob.size(), nb);
    LogFilter lf;
    memset(&lf, 0, sizeof lf);
    lf.ne = ne;
    for (uint32_t k = 0; k < ne && k < LF_INLINE; k++) lf.emit[k] = em[k];
    if (ne > LF_INLINE) return 2;   // the large-set path is the log filter's own harness's (emu_log_filter.cu)
    std::vector<uint32_t> bits((nr + 31) / 32, 0), cnt(nr, 0), nby(nr, 0);
    unsigned long long err = IPCFP_NO_ERROR, stats[2] = {0, 0}, n_sel = ns;
    MsgMatchArgsT<LogFilter> a;
    a.store = hs.view; a.store_dev = &hs.view; a.m_dev = &lf; a.events_roots = roots.data(); a.has_root = has.data();
    a.sel = sel.data(); a.n_sel = &n_sel; a.n_sel_max = ns; a.match_bits = bits.data(); a.cnt = cnt.data(); a.nbytes = nby.data();
    a.err = &err; a.stats = stats; a.per_warp = 1;
    std::vector<uint64_t> order(ns);
    for (uint64_t t = 0; t < ns; t++) order[t] = t;
    uint64_t r = 0x9E3779B97F4A7C15ull;
    for (uint64_t t = ns; t > 1; t--) { r ^= r << 13; r ^= r >> 7; r ^= r << 17; std::swap(order[t - 1], order[r % t]); }
    for (uint64_t t : order) msg_match_item(a, t);
    if (err == IPCFP_NO_ERROR) printf("err none\n");
    else printf("err %llu %llu %llu\n", err >> 56, (err >> 16) & 0xFFFFFFFFFFull, (err >> 8) & 0xff);
    for (uint32_t i : sel) printf("%u %u %u %u\n", i, (bits[i >> 5] >> (i & 31)) & 1u, cnt[i], nby[i]);
    return 0;
}

static bool read_cid(uint8_t out[38]) {
    char buf[128];
    if (scanf("%127s", buf) != 1 || strlen(buf) != 76) return false;
    for (int k = 0; k < 38; k++) { unsigned v; sscanf(buf + 2 * k, "%2x", &v); out[k] = (uint8_t)v; }
    return true;
}

int main(int argc, char** argv) {
    if (argc > 2 && !strcmp(argv[1], "match")) return run_match(argv[2]);
    unsigned long long n_exec, n_req, n_receipts;
    if (scanf("%llu %llu %llu", &n_exec, &n_req, &n_receipts) != 3) return 2;
    // exact-size buffers: an access past them is an AddressSanitizer report under `make sanitize`
    std::vector<RawCid> raw(n_exec), req(n_req), sorted(n_req);
    std::vector<uint32_t> idx(n_exec), pos(n_req);
    uint8_t c[38];
    for (auto& r : raw) { if (!read_cid(c)) return 2; r = rawcid_from_bytes(c); }
    for (auto& i : idx) if (scanf("%u", &i) != 1) return 2;
    for (auto& r : req) { if (!read_cid(c)) return 2; r = rawcid_from_bytes(c); }
    // the device's sort: stable passes over msg_sort_key's slices, least significant first, from the input order
    std::vector<uint32_t> perm(n_req);
    for (uint32_t j = 0; j < n_req; j++) perm[j] = j;
    for (uint32_t q = MSG_SORT_SLICES; q-- > 0;)
        std::stable_sort(perm.begin(), perm.end(), [&](uint32_t x, uint32_t y) { return msg_sort_key(req[x], q) < msg_sort_key(req[y], q); });
    for (uint32_t r = 0; r < n_req; r++) { sorted[r] = req[perm[r]]; pos[r] = perm[r]; }
    for (uint32_t r = 1; r < n_req; r++) {   // the binary search needs rawcid_cmp order with input-order ties
        const int c = rawcid_cmp(sorted[r - 1], sorted[r]);
        if (c > 0 || (c == 0 && pos[r - 1] > pos[r])) return 3;
    }
    std::vector<uint64_t> exec_indices(n_req, UINT64_MAX);
    std::vector<uint64_t> sel;
    for (uint64_t i = 0; i < n_exec; i++)
        if (msg_select_item(raw.data(), idx.data(), i, sorted.data(), pos.data(), (uint32_t)n_req, n_receipts, exec_indices.data())) sel.push_back(i);
    printf("%zu\n", sel.size());
    for (uint64_t i : sel) printf("%llu\n", (unsigned long long)i);
    for (uint64_t e : exec_indices) printf("%llu\n", (unsigned long long)e);
    return 0;
}
