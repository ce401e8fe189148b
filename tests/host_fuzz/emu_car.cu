// emu_car.cu — the device CAR parser of ipcfp_store_create_car executed ON THE CPU (TEST INFRASTRUCTURE, no GPU needed).
//
// The per-item functions of csrc/car_items.cuh, compiled for the host and driven as csrc/car.cu drives them — the header through
// car_header, the candidate bitmap (car_candidate at every position), the ascending positions, the links of every (candidate, option)
// in a shuffled order (car_link), the walk from the head (car_head), the blocks and CIDs of the chain (car_block) — against ipcfp_blocks_from_car
// (csrc/car_parse.cpp, linked as the checker):
//   * random canonical CARs (0 … 60 sections, blocks of 0 … 300 bytes, random codecs below 0x80 and three-byte multihash codes,
//     duplicates, roots): the device items must accept every one and give the host parser's CIDs, offsets and lengths;
//   * the same CARs with a forged section header inside one block: the walk must step over it and give the host parser's arrays;
//   * the same CARs with one non-minimal length varint: the device items must defer (the host parser refuses them);
//   * byte mutations (flip / insert / delete / duplicate a span): each must either be deferred or give exactly the host parser's arrays;
//     an accept where the host parser refuses is a failure.
// The buffer the device items read is an exact-size heap buffer followed by CAR_PAD zero bytes, as the arena's padding on the device;
// under AddressSanitizer any read outside is a report.
//
//   nvcc -std=c++17 -O2 -o emu_car tests/host_fuzz/emu_car.cu ipc_filecoin_proofs_b200/csrc/car_parse.cpp && ./emu_car 3000 60000 7
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/car_items.cuh"
#include "../../include/ipcfp.h"

namespace ipcfp {
void set_last_error(const std::string&, uint64_t) {}   // the library's error slot (capi.cu), not linked here
bool car_header(const uint8_t* car, uint64_t len, uint64_t& first_section);   // car_parse.cpp
}

using namespace ipcfp;
typedef std::vector<uint8_t> Bytes;

static uint64_t rs;
static uint64_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return rs; }

static void varint(Bytes& o, uint64_t v, bool nonminimal = false) {
    while (v >= 0x80) { o.push_back((uint8_t)(v | 0x80)); v >>= 7; }
    if (nonminimal) { o.push_back((uint8_t)(v | 0x80)); o.push_back(0); }
    else o.push_back((uint8_t)v);
}
static Bytes random_cid() {
    Bytes c = {0x01, (uint8_t)(rnd() % 0x80), (uint8_t)(0x80 | rnd()), (uint8_t)(0x80 | rnd()), (uint8_t)(1 + rnd() % 0x7f), 0x20};
    for (int k = 0; k < 32; k++) c.push_back((uint8_t)rnd());
    return c;
}
// {"roots": [n_roots CIDs], "version": 1}
static Bytes header(const std::vector<Bytes>& roots) {
    Bytes h = {0xa2, 0x65, 'r', 'o', 'o', 't', 's', (uint8_t)(0x80 | roots.size())};
    for (const Bytes& r : roots) { h.push_back(0xd8); h.push_back(42); h.push_back(0x58); h.push_back(39); h.push_back(0); h.insert(h.end(), r.begin(), r.end()); }
    const char* v = "\x67version\x01";
    h.insert(h.end(), v, v + 9);
    Bytes o;
    varint(o, h.size());
    o.insert(o.end(), h.begin(), h.end());
    return o;
}
// kind 0: canonical; 1: a forged section header inside one block; 2: one non-minimal length varint (a CAR of no section is canonical:
// kind is then set to 0)
static Bytes make_car(int& kind) {
    const uint64_t n = rnd() % 4 == 0 ? rnd() % 3 : rnd() % 60;
    std::vector<Bytes> cids;
    for (uint64_t i = 0; i < n; i++) cids.push_back(i && rnd() % 8 == 0 ? cids[rnd() % i] : random_cid());
    std::vector<Bytes> roots;
    for (uint64_t r = 0, nr = rnd() % 3; r < nr; r++) roots.push_back(random_cid());
    Bytes car = header(roots);
    const uint64_t odd = n ? rnd() % n : 0;
    if (!n && kind) kind = 0;
    for (uint64_t i = 0; i < n; i++) {
        Bytes blk(rnd() % 5 == 0 ? rnd() % 4 : rnd() % 300);
        for (auto& b : blk) b = (uint8_t)rnd();
        if (kind == 1 && i == odd) {   // a section header of 38 bytes: it ends inside the payload whatever follows
            const uint8_t forged[7] = {38, 0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
            const uint64_t at = blk.size() ? rnd() % blk.size() : 0;
            blk.insert(blk.begin() + at, forged, forged + 7);
            blk.resize(std::max<size_t>(blk.size(), at + 39), 0x5a);
        }
        varint(car, cids[i].size() + blk.size(), kind == 2 && i == odd);
        car.insert(car.end(), cids[i].begin(), cids[i].end());
        car.insert(car.end(), blk.begin(), blk.end());
    }
    return car;
}

struct Arrays { Bytes cids; std::vector<uint64_t> offsets; std::vector<uint32_t> lengths; };

// csrc/car.cu's flow with the kernels replaced by loops; false = defer
static bool device_parse(const Bytes& car, Arrays& out) {
    uint64_t first;
    if (!car_header(car.data(), car.size(), first)) return false;
    const uint64_t len = car.size();
    uint8_t* t = (uint8_t*)malloc(len + CAR_PAD);   // exact size + the arena's zero padding
    memcpy(t, car.data(), len);
    memset(t + len, 0, CAR_PAD);
    std::vector<uint64_t> pos;
    for (uint64_t p = 0; p < len; p++) if (car_candidate(t, len, first, p)) pos.push_back(p);
    const uint64_t n = pos.size();
    // k_car_links, its threads in a shuffled order
    std::vector<uint64_t> links(CAR_MAX_VARINT * n), order(links.size());
    for (uint64_t k = 0; k < order.size(); k++) order[k] = k;
    for (uint64_t q = order.size(); q > 1; q--) std::swap(order[q - 1], order[rnd() % q]);
    for (uint64_t k : order) links[k] = car_link(t, len, first, pos.data(), n, k / CAR_MAX_VARINT, k % CAR_MAX_VARINT + 1);
    // the host walk from the head
    std::vector<uint64_t> chain;
    bool ok = true;
    for (uint64_t cur = car_head(t, len, first, pos.data(), n); cur != CAR_LINK_TERMINAL;) {
        if (cur == CAR_LINK_NONE || chain.size() >= n) { ok = false; break; }
        chain.push_back(cur);
        cur = links[CAR_MAX_VARINT * (cur >> 3) + (cur & 7) - 1];
    }
    out = Arrays();
    if (ok) {   // k_car_gather
        for (uint64_t link : chain) {
            uint64_t off;
            uint32_t blen;
            car_block(t, pos.data(), link, off, blen);
            out.offsets.push_back(off);
            out.lengths.push_back(blen);
            out.cids.insert(out.cids.end(), t + off - 38, t + off);
        }
    }
    free(t);
    return ok;
}

static bool host_parse(const Bytes& car, Arrays& out) {
    ipcfp_parsed_blocks* pb = nullptr;
    Bytes copy(car);   // the host parser reads exactly len bytes
    if (ipcfp_blocks_from_car(copy.data(), copy.size(), &pb) != IPCFP_OK) return false;
    const ipcfp_witness& w = pb->blocks;
    out.cids.assign(w.cids, w.cids + 38 * w.n_blocks);
    out.offsets.assign(w.offsets, w.offsets + w.n_blocks);
    out.lengths.assign(w.lengths, w.lengths + w.n_blocks);
    ipcfp_parsed_blocks_free(pb);
    return true;
}

static bool same(const Arrays& a, const Arrays& b) { return a.cids == b.cids && a.offsets == b.offsets && a.lengths == b.lengths; }

static void mutate(Bytes& c) {
    const uint64_t at = c.empty() ? 0 : rnd() % c.size(), span = 1 + rnd() % 4;
    switch (rnd() % 4) {
    case 0: if (!c.empty()) c[at] ^= (uint8_t)(1 + rnd() % 255); break;
    case 1: for (uint64_t k = 0; k < span; k++) c.insert(c.begin() + at, (uint8_t)rnd()); break;
    case 2: c.erase(c.begin() + at, c.begin() + std::min<uint64_t>(c.size(), at + span)); break;
    default: { Bytes d(c.begin() + at, c.begin() + std::min<uint64_t>(c.size(), at + span)); c.insert(c.begin() + at, d.begin(), d.end()); }
    }
}

int main(int argc, char** argv) {
    const uint64_t n_inputs = argc > 1 ? strtoull(argv[1], 0, 10) : 3000, n_mutants = argc > 2 ? strtoull(argv[2], 0, 10) : 60000;
    rs = argc > 3 ? strtoull(argv[3], 0, 10) | 1 : 7;
    uint64_t n_kind[3] = {0, 0, 0};
    for (uint64_t k = 0; k < n_inputs; k++) {
        int kind = (int)(k % 3);
        const Bytes car = make_car(kind);
        n_kind[kind]++;
        Arrays d, h;
        const bool dev = device_parse(car, d), host = host_parse(car, h);
        if (kind == 0 && (!dev || !host || !same(d, h))) { printf("FAIL: canonical input %llu: device %d host %d\n", (unsigned long long)k, dev, host); return 1; }
        if (kind == 1 && (!dev || !host || !same(d, h))) { printf("FAIL: forged prefix input %llu: device %d host %d\n", (unsigned long long)k, dev, host); return 1; }
        if (kind == 2 && dev) { printf("FAIL: non-minimal varint input %llu accepted by the device items\n", (unsigned long long)k); return 1; }
    }
    uint64_t accepted = 0, host_ok = 0;
    for (uint64_t k = 0; k < n_mutants; k++) {
        int kind = 0;
        Bytes car = make_car(kind);
        for (uint64_t m = 1 + rnd() % 2; m; m--) mutate(car);
        Arrays d, h;
        const bool dev = device_parse(car, d), host = host_parse(car, h);
        accepted += dev;
        host_ok += host;
        if (dev && (!host || !same(d, h))) { printf("FAIL: mutant %llu accepted by the device items with other arrays (host %d)\n", (unsigned long long)k, host); return 1; }
    }
    printf("ok: device CAR parser == ipcfp_blocks_from_car on %llu inputs (%llu with a forged prefix, all accepted, %llu with a non-minimal varint, all deferred, "
           "as the host parser reads them) and %llu mutants (%llu accepted by the device items, %llu by the host parser)\n", (unsigned long long)n_inputs,
           (unsigned long long)n_kind[1], (unsigned long long)n_kind[2], (unsigned long long)n_mutants,
           (unsigned long long)accepted, (unsigned long long)host_ok);
    return 0;
}
