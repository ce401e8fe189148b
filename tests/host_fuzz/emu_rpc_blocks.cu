// emu_rpc_blocks.cu — the device parser of ipcfp_store_create_rpc_json executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// The per-item functions of csrc/rpc_blocks_items.cuh (and the base64 items of json_parse_items.cuh), compiled for the host and driven as
// csrc/rpc_blocks.cu drives them — the texts joined by separators, the record starts, the data runs, the per-record template and joint
// checks in a shuffled order, the id claims, the owned-byte sum, the decode into 16-aligned slots — against ipcfp_blocks_from_rpc_json
// (csrc/rpc_blocks_parse.cpp, linked as the checker):
//   * random canonical inputs (any number of blocks, lengths 0 … 200, responses shuffled, split over batches and single-object texts,
//     empty batches): the device items must accept every one and give the host parser's offsets, lengths and bytes;
//   * byte mutations of such inputs (replace / insert / delete / duplicate a span, in one text): each must either be refused by the device
//     items (the call then defers to the host parser) or give exactly the host parser's arrays; an accept where the host parser refuses
//     is a failure.
// The buffer the device items read is an exact-size heap buffer followed by JP_PAD zero bytes, as on the device; under AddressSanitizer any
// read outside is a report.
//
//   nvcc -std=c++17 -O2 -o emu_rpc_blocks tests/host_fuzz/emu_rpc_blocks.cu ipc_filecoin_proofs_b200/csrc/rpc_blocks_parse.cpp && ./emu_rpc_blocks 2000 60000 7
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/rpc_blocks_items.cuh"

namespace ipcfp { void set_last_error(const std::string&, uint64_t) {} }   // the library's error slot (capi.cu), not linked here

using namespace ipcfp;

static uint64_t rs;
static uint64_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return rs; }

static const char B64[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
static std::string b64(const std::string& d) {
    std::string o;
    for (size_t i = 0; i < d.size(); i += 3) {
        uint32_t v = (uint8_t)d[i] << 16;
        if (i + 1 < d.size()) v |= (uint8_t)d[i + 1] << 8;
        if (i + 2 < d.size()) v |= (uint8_t)d[i + 2];
        o.push_back(B64[v >> 18]);
        o.push_back(B64[(v >> 12) & 63]);
        o.push_back(i + 1 < d.size() ? B64[(v >> 6) & 63] : '=');
        o.push_back(i + 2 < d.size() ? B64[v & 63] : '=');
    }
    return o;
}

struct Blocks { std::vector<uint64_t> offsets; std::vector<uint32_t> lengths; std::vector<uint8_t> blob; };

// a random canonical input over n random blocks; want receives their arrays
static std::vector<std::string> make_input(uint64_t n, Blocks& want) {
    std::vector<std::string> els;
    want = Blocks();
    for (uint64_t i = 0; i < n; i++) {
        std::string d(rnd() % 4 == 0 ? rnd() % 4 : rnd() % 200, '\0');
        for (auto& c : d) c = (char)rnd();
        want.offsets.push_back(want.blob.size());
        want.lengths.push_back((uint32_t)d.size());
        want.blob.insert(want.blob.end(), d.begin(), d.end());
        want.blob.resize((want.blob.size() + 15) & ~15ull, 0);
        els.push_back("{\"jsonrpc\":\"2.0\",\"result\":\"" + b64(d) + "\",\"id\":" + std::to_string(i) + "}");
    }
    for (uint64_t q = n; q > 1; q--) std::swap(els[q - 1], els[rnd() % q]);
    std::vector<std::string> texts;
    for (size_t k = 0; k < els.size() || texts.empty();) {
        if (rnd() % 8 == 0) { texts.push_back("[]"); continue; }
        if (k < els.size() && rnd() % 3 == 0) { texts.push_back(els[k++]); continue; }
        const size_t m = std::min<size_t>(els.size() - k, 1 + rnd() % 12);
        std::string t = "[";
        for (size_t j = 0; j < m; j++) t += (j ? "," : "") + els[k + j];
        texts.push_back(t + "]");
        k += m;
    }
    return texts;
}

// csrc/rpc_blocks.cu's flow with the kernels replaced by loops; false = defer
static bool device_parse(const std::vector<std::string>& texts, uint64_t nb, Blocks& out) {
    uint64_t len = 0, want_owned = 0;
    for (const auto& t : texts) {
        if (t.empty()) return false;
        len += t.size() + 1;
        want_owned += t == "[]" ? 0 : t.size();
    }
    std::vector<char> buf(len + JP_PAD, 0);   // the device copy
    uint64_t at = 0;
    for (const auto& t : texts) { memcpy(buf.data() + at, t.data(), t.size()); buf[at + t.size()] = RB_SEP; at += t.size() + 1; }
    const char* t = buf.data();
    // k_rb_mark + bitmap_to_indices
    std::vector<uint32_t> pos;
    for (uint64_t p = 0; p < len; p++) if (t[p] == '{' && rb_start_at(t, p)) pos.push_back((uint32_t)p);
    const uint64_t n = pos.size(), cap = len / RB_MIN_RECORD + 1;
    if (n > cap) return false;
    // k_rb_records, in any order
    std::vector<uint32_t> owner(nb + 1, 0xffffffffu), blen(nb + 1, 0), nch(nb + 1, 0);
    std::vector<uint64_t> order(n);
    for (uint64_t i = 0; i < n; i++) order[i] = i;
    for (uint64_t q = n; q > 1; q--) std::swap(order[q - 1], order[rnd() % q]);
    bool defer = false;
    uint64_t owned = 0;
    for (uint64_t i : order) {
        uint64_t q = (uint64_t)pos[i] + RB_HEAD_LEN;
        while (!rb_stop_byte(t[q])) q++;
        RbRec r;
        bool ok = rb_record(t, len, pos.data(), n, i, q, nb, r);
        if (ok) for (uint64_t k = 0; k < r.blk.n_chars - r.blk.pads; k++) ok &= jp_block_char_ok(t, r.blk, k);
        if (!ok || owner[r.id] != 0xffffffffu) { defer = true; continue; }
        owner[r.id] = (uint32_t)i;
        blen[r.id] = (uint32_t)jp_align16(r.blk.len);
        nch[r.id] = (uint32_t)r.blk.n_chars;
        owned += r.owned;
    }
    if (defer || n != nb || owned != want_owned) return false;
    // exclusive_scan_u32 + k_rb_blocks
    out = Blocks();
    uint64_t total = 0;
    for (uint64_t j = 0; j < nb; j++) { out.offsets.push_back(total); total += blen[j]; }
    out.blob.assign(total, 0);
    out.lengths.resize(nb);
    for (uint64_t j = 0; j < nb; j++) {
        JpBlock b;
        b.data_at = (uint64_t)pos[owner[j]] + RB_HEAD_LEN;
        b.n_chars = nch[j];
        jp_b64_span(t, b);
        out.lengths[j] = b.len;
        for (uint64_t g = 0; g < b.n_chars / 4; g++) jp_block_group(t, b, g, out.blob.data() + out.offsets[j]);
    }
    return true;
}

// the device result equals the host parser's; when the host refuses, the device must have deferred. *host_ok: the host accepted
static bool same_as_host(const std::vector<std::string>& texts, uint64_t nb, bool dev_ok, const Blocks& dev, bool* host_ok) {
    std::vector<uint8_t> cids(38 * nb + 1, 7);
    std::vector<const char*> ptrs;
    std::vector<uint64_t> lens;
    for (const auto& t : texts) { ptrs.push_back(t.data()); lens.push_back(t.size()); }
    ipcfp_parsed_blocks* pb = nullptr;
    const ipcfp_status st = ipcfp_blocks_from_rpc_json(cids.data(), nb, ptrs.data(), lens.data(), texts.size(), &pb);
    *host_ok = st == IPCFP_OK;
    auto fail = [&](const char* m) {
        fprintf(stderr, "device accepted, %s\n", m);
        for (const auto& t : texts) fprintf(stderr, "  text: %.300s\n", t.c_str());
        if (pb) ipcfp_parsed_blocks_free(pb);
        return false;
    };
    if (!dev_ok) { if (pb) ipcfp_parsed_blocks_free(pb); return true; }
    if (st != IPCFP_OK) return fail("host parser refused");
    const ipcfp_witness& w = pb->blocks;
    if (w.n_blocks != nb || w.blob_size != dev.blob.size()) return fail("block count or blob size differs");
    if (nb && (memcmp(w.offsets, dev.offsets.data(), 8 * nb) || memcmp(w.lengths, dev.lengths.data(), 4 * nb))) return fail("offsets or lengths differ");
    if (w.blob_size && memcmp(w.blob, dev.blob.data(), w.blob_size)) return fail("block bytes differ");
    ipcfp_parsed_blocks_free(pb);
    return true;
}

static std::string mutate(const std::string& s) {
    static const char ALPH[] = "{}[]\",:0123456789 \t\nabzAZ=+/\\-.enulid";
    std::string m = s;
    const int edits = 1 + (int)(rnd() % 3);
    for (int e = 0; e < edits && !m.empty(); e++) {
        const uint64_t i = rnd() % m.size();
        switch (rnd() % 5) {
            case 0: m[i] = ALPH[rnd() % (sizeof ALPH - 1)]; break;
            case 1: m.insert(m.begin() + i, ALPH[rnd() % (sizeof ALPH - 1)]); break;
            case 2: m.erase(i, 1 + rnd() % 3); break;
            case 3: { const uint64_t j = rnd() % m.size(), l = std::min<uint64_t>(1 + rnd() % 80, m.size() - j); m.insert(i, m.substr(j, l)); break; }
            default: { const uint64_t l = std::min<uint64_t>(1 + rnd() % 80, m.size() - i); m.erase(i, l); break; }
        }
    }
    return m;
}

int main(int argc, char** argv) {
    const uint64_t n_inputs = argc > 1 ? strtoull(argv[1], 0, 10) : 2000, n_mut = argc > 2 ? strtoull(argv[2], 0, 10) : 60000;
    rs = (argc > 3 ? strtoull(argv[3], 0, 10) : 7) * 0x9E3779B97F4A7C15ull | 1;
    std::vector<std::vector<std::string>> inputs;
    std::vector<uint64_t> counts;
    uint64_t blocks = 0;
    for (uint64_t k = 0; k < n_inputs; k++) {
        const uint64_t n = k % 50 == 0 ? 0 : 1 + rnd() % (rnd() % 8 == 0 ? 200 : 12);
        Blocks want, got;
        const auto texts = make_input(n, want);
        bool host_ok;
        if (!device_parse(texts, n, got)) { fprintf(stderr, "canonical input %llu deferred\n  text: %.300s\n", (unsigned long long)k, texts[0].c_str()); return 1; }
        if (got.offsets != want.offsets || got.lengths != want.lengths || got.blob != want.blob) {
            fprintf(stderr, "canonical input %llu: arrays differ from the generator's\n", (unsigned long long)k);
            return 1;
        }
        if (!same_as_host(texts, n, true, got, &host_ok)) return 1;
        blocks += n;
        inputs.push_back(texts);
        counts.push_back(n);
    }
    uint64_t dev_ok = 0, host_ok_n = 0;
    for (uint64_t k = 0; k < n_mut; k++) {
        const uint64_t w = rnd() % inputs.size();
        auto texts = inputs[w];
        auto& t = texts[rnd() % texts.size()];
        t = mutate(t);
        Blocks got;
        const bool ok = device_parse(texts, counts[w], got);
        bool host_ok;
        if (!same_as_host(texts, counts[w], ok, got, &host_ok)) return 1;
        dev_ok += ok;
        host_ok_n += host_ok;
    }
    printf("ok: device ChainReadObj parser == ipcfp_blocks_from_rpc_json on %llu canonical inputs (%llu blocks) "
           "and %llu mutants (%llu accepted by the device items, %llu by the host parser)\n",
           (unsigned long long)n_inputs, (unsigned long long)blocks, (unsigned long long)n_mut, (unsigned long long)dev_ok,
           (unsigned long long)host_ok_n);
    return 0;
}
