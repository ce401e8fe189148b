// emu_rpc_json.cu — the device receipt-list parser of ipcfp_tipset_upload_json executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// The per-item functions of csrc/rpc_json_items.cuh, compiled for the host and driven as csrc/rpc_json.cu drives them — the host's framing
// check, the per-32-byte marks with the foreign-byte defer, the record starts, the per-record template checks in a shuffled order — against
// ipcfp_tipset_desc_from_json (csrc/rpc_parse.cpp, linked as the checker):
//   * random canonical receipt lists (edge values: ExitCode 0 / u32 max, GasUsed 0 / u64 max, Return of any base64 length, EventsRoot null
//     or a random 38-byte CID): the device items must accept every one and give the host parser's events_roots / has_events_root;
//   * byte mutations of such lists (replace / insert / delete / duplicate a span): each must either be refused by the device items (the
//     call then defers to the host parser) or give exactly the host parser's arrays; an accept where the host parser refuses is a failure.
// The text the device items read is an exact-size heap buffer followed by JP_PAD zero bytes, as on the device; under AddressSanitizer any
// read outside is a report.
//
//   nvcc -std=c++17 -O2 -o emu_rpc_json tests/host_fuzz/emu_rpc_json.cu ipc_filecoin_proofs_b200/csrc/rpc_parse.cpp && ./emu_rpc_json 2000 60000 7
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/rpc_json_items.cuh"

namespace ipcfp { void set_last_error(const std::string&, uint64_t) {} }   // the library's error slot (capi.cu), not linked here

using namespace ipcfp;

static uint64_t rs;
static uint64_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return rs; }

static const char B32[] = "abcdefghijklmnopqrstuvwxyz234567";
static const char B64[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
static std::string cid_string(const uint8_t* c) {
    std::string s = "b";
    uint32_t acc = 0;
    int bits = 0;
    for (int i = 0; i < 38; i++) {
        acc = (acc << 8) | c[i];
        bits += 8;
        while (bits >= 5) { s.push_back(B32[(acc >> (bits - 5)) & 31]); bits -= 5; }
        acc &= (1u << bits) - 1;
    }
    if (bits) s.push_back(B32[(acc << (5 - bits)) & 31]);
    return s;
}
static uint64_t pick_u64(uint64_t max) {
    switch (rnd() % 4) {
        case 0: return (rnd() & 1) ? 0 : max;
        case 1: return rnd() % 1000;
        case 2: return (rnd() >> (rnd() % 64)) % (max == UINT64_MAX ? UINT64_MAX : max + 1);
        default: return max == UINT64_MAX ? rnd() : rnd() % (max + 1);
    }
}

// a random canonical list and its expected arrays
static std::string make_list(uint64_t n, std::vector<uint8_t>& roots, std::vector<uint8_t>& has) {
    std::string t = "[";
    roots.assign(38 * n, 0);
    has.assign(n, 0);
    static const uint8_t pre[6] = {1, 0x71, 0xa0, 0xe4, 2, 0x20};
    for (uint64_t i = 0; i < n; i++) {
        if (i) t += ",";
        t += "{\"ExitCode\":" + std::to_string(pick_u64(0xffffffffull)) + ",\"Return\":\"";
        const uint64_t nr = rnd() % 5 == 0 ? rnd() % 40 : 0;
        for (uint64_t k = 0; k < nr; k++) t.push_back(k + 2 >= nr && rnd() % 2 ? '=' : B64[rnd() % 64]);
        t += "\",\"GasUsed\":" + std::to_string(pick_u64(UINT64_MAX)) + ",\"EventsRoot\":";
        if (rnd() % 4) {
            uint8_t* c = roots.data() + 38 * i;
            for (int k = 0; k < 38; k++) c[k] = (uint8_t)rnd();
            if (rnd() % 4) memcpy(c, pre, 6);
            has[i] = 1;
            t += "{\"/\":\"" + cid_string(c) + "\"}";
        } else t += "null";
        t += "}";
    }
    return t + "]";
}

// csrc/rpc_json.cu's flow with the kernels replaced by loops; false = defer
static bool device_parse(const std::string& text, std::vector<uint8_t>& roots, std::vector<uint8_t>& has) {
    const uint64_t len = text.size();
    if (len < 2 || text[0] != '[' || text[len - 1] != ']') return false;
    roots.clear();
    has.clear();
    if (len == 2) return true;
    std::vector<char> padded(len + JP_PAD, 0);   // the device copy
    memcpy(padded.data(), text.data(), len);
    const char* t = padded.data();
    // k_rj_mark + bitmap_to_indices
    std::vector<uint32_t> pos;
    bool foreign = false;
    for (uint64_t p = 0; p < len; p++) {
        foreign |= rj_foreign_byte(t[p]);
        if (t[p] == '{' && rj_start_at(t, p)) pos.push_back((uint32_t)p);
    }
    const uint64_t n = pos.size(), cap = len / RJ_MIN_RECORD + 1;
    if (foreign || n == 0 || n > cap) return false;
    // k_rj_records, in any order, into exact-size arrays
    roots.assign(38 * n, 0xee);
    has.assign(n, 0xee);
    std::vector<uint64_t> order(n);
    for (uint64_t i = 0; i < n; i++) order[i] = i;
    for (uint64_t q = n; q > 1; q--) std::swap(order[q - 1], order[rnd() % q]);
    bool ok = true;
    for (uint64_t i : order) {
        uint8_t h = 0;
        ok &= rj_record(t, len, pos.data(), n, i, roots.data() + 38 * i, h);
        has[i] = h;
    }
    return ok;
}

static const char* PARENT = "{\"Cids\":[],\"Blocks\":[],\"Height\":1}";
static std::string child_text() {
    uint8_t c[38] = {1, 0x71, 0xa0, 0xe4, 2, 0x20};
    const std::string m = "{\"/\":\"" + cid_string(c) + "\"}";
    return "{\"Cids\":[" + m + "],\"Blocks\":[{\"Miner\":\"f01\",\"Parents\":[],\"ParentStateRoot\":" + m + ",\"ParentMessageReceipts\":" + m +
           ",\"Messages\":" + m + ",\"Height\":2}],\"Height\":2}";
}

// the device result equals the host parser's; when the host refuses, the device must have deferred. *host_ok: the host accepted
static bool same_as_host(const std::string& text, bool dev_ok, const std::vector<uint8_t>& roots, const std::vector<uint8_t>& has, bool* host_ok) {
    static const std::string child = child_text();
    ipcfp_parsed_tipset* pt = nullptr;
    const ipcfp_status st = ipcfp_tipset_desc_from_json(PARENT, strlen(PARENT), child.data(), child.size(), text.data(), text.size(), &pt);
    *host_ok = st == IPCFP_OK;
    auto fail = [&](const char* m) {
        fprintf(stderr, "device accepted, %s\n  text: %.400s\n", m, text.c_str());
        if (pt) ipcfp_parsed_tipset_free(pt);
        return false;
    };
    if (!dev_ok) { if (pt) ipcfp_parsed_tipset_free(pt); return true; }
    if (st != IPCFP_OK) return fail("host parser refused");
    const ipcfp_tipset_desc& d = pt->desc;
    if (d.n_receipts != has.size()) return fail("receipt count differs");
    if (d.n_receipts && (memcmp(d.events_roots, roots.data(), roots.size()) || memcmp(d.has_events_root, has.data(), has.size())))
        return fail("events roots differ");
    ipcfp_parsed_tipset_free(pt);
    return true;
}

static std::string mutate(const std::string& s) {
    static const char ALPH[] = "{}[]\",:0123456789 \t\nabzAZ=+/\\-.enul";
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
    const uint64_t n_lists = argc > 1 ? strtoull(argv[1], 0, 10) : 2000, n_mut = argc > 2 ? strtoull(argv[2], 0, 10) : 60000;
    rs = (argc > 3 ? strtoull(argv[3], 0, 10) : 7) * 0x9E3779B97F4A7C15ull | 1;
    std::vector<std::string> lists;
    uint64_t receipts = 0, with_root = 0;
    for (uint64_t k = 0; k < n_lists; k++) {
        const uint64_t n = k % 50 == 0 ? 0 : 1 + rnd() % (rnd() % 8 == 0 ? 300 : 12);
        std::vector<uint8_t> want_roots, want_has, roots, has;
        const std::string t = make_list(n, want_roots, want_has);
        bool host_ok;
        if (!device_parse(t, roots, has)) { fprintf(stderr, "canonical list %llu deferred\n  text: %.400s\n", (unsigned long long)k, t.c_str()); return 1; }
        if (roots != want_roots || has != want_has) { fprintf(stderr, "canonical list %llu: arrays differ from the generator's\n", (unsigned long long)k); return 1; }
        if (!same_as_host(t, true, roots, has, &host_ok)) return 1;
        receipts += n;
        for (uint8_t h : has) with_root += h;
        lists.push_back(t);
    }
    uint64_t dev_ok = 0, host_ok_n = 0;
    for (uint64_t k = 0; k < n_mut; k++) {
        const std::string m = mutate(lists[rnd() % lists.size()]);
        std::vector<uint8_t> roots, has;
        const bool ok = device_parse(m, roots, has);
        bool host_ok;
        if (!same_as_host(m, ok, roots, has, &host_ok)) return 1;
        dev_ok += ok;
        host_ok_n += host_ok;
    }
    printf("ok: device receipt-list parser == ipcfp_tipset_desc_from_json on %llu canonical lists (%llu receipts, %llu with an events root) "
           "and %llu mutants (%llu accepted by the device items, %llu by the host parser)\n",
           (unsigned long long)n_lists, (unsigned long long)receipts, (unsigned long long)with_root, (unsigned long long)n_mut,
           (unsigned long long)dev_ok, (unsigned long long)host_ok_n);
    return 0;
}
