// fuzz_events.cu — HOST build of the device-side StampedEvent decoders (TEST INFRASTRUCTURE, no GPU needed).
//
// The pass-1 / pass-2 kernels decode every event with `fast_stamped_event` (register-window fast path) and fall back to
// `parse_stamped_event` (the strict DAG-CBOR decoder) on any deviation. "Results identical by construction" rests on one
// property: whenever the fast path accepts a byte string, the strict decoder accepts it too, ends at the same position and
// yields the same EvLog. This program compiles the very same headers for the host (nvcc host pass, intrinsics mapped to
// compiler builtins) and checks that property on canonical events and on millions of mutations of them.
//
// Third property: the strict device decoder + extract_evm_log (ev_finish) agree with the CPU oracle's independent
// implementation (oracle/oracle.cpp: serde-like owned structs + a HashMap per event) on every input, well-formed or not.
//
//   nvcc -std=c++17 -O2 -o fuzz_events tests/host_fuzz/fuzz_events.cu oracle/oracle.cpp -lpthread && ./fuzz_events [iterations] [seed]
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "host_shims.h"

#include "../../ipc_filecoin_proofs_b200/csrc/ipld.cuh"
#include "../../oracle/oracle.h"

using namespace ipcfp;

static uint64_t rng_state;
static uint64_t rnd() {  // SplitMix64
    uint64_t z = (rng_state += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static void put_head(std::vector<uint8_t>& o, int major, uint64_t v) {
    if (v < 24) o.push_back((uint8_t)(major << 5 | v));
    else if (v < 0x100) { o.push_back((uint8_t)(major << 5 | 24)); o.push_back((uint8_t)v); }
    else if (v < 0x10000) { o.push_back((uint8_t)(major << 5 | 25)); o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); }
    else if (v < 0x100000000ull) { o.push_back((uint8_t)(major << 5 | 26)); for (int s = 24; s >= 0; s -= 8) o.push_back((uint8_t)(v >> s)); }
    else { o.push_back((uint8_t)(major << 5 | 27)); for (int s = 56; s >= 0; s -= 8) o.push_back((uint8_t)(v >> s)); }
}
static void put_entry(std::vector<uint8_t>& o, uint64_t flags, const char* key, uint64_t codec, size_t vlen) {
    put_head(o, 4, 4);
    put_head(o, 0, flags);
    put_head(o, 3, strlen(key));
    o.insert(o.end(), key, key + strlen(key));
    put_head(o, 0, codec);
    put_head(o, 2, vlen);
    for (size_t i = 0; i < vlen; i++) o.push_back((uint8_t)rnd());
}
// one StampedEvent in one of the shapes the synthetic tipsets and FEVM produce
static std::vector<uint8_t> make_event() {
    std::vector<uint8_t> o;
    put_head(o, 4, 2);
    static const uint64_t emitters[] = {5, 23, 24, 255, 256, 1001, 65535, 65536, 1ull << 32, (1ull << 40) + 1001};
    put_head(o, 0, emitters[rnd() % 10]);
    unsigned shape = (unsigned)(rnd() % 8);
    if (shape == 0) {  // Case A
        put_head(o, 4, 2);
        put_entry(o, 3, "topics", 0x55, 32 * (rnd() % 5));
        put_entry(o, 3, "data", 0x55, rnd() % 300);
    } else {
        unsigned nt = 1 + (unsigned)(rnd() % 4);
        bool has_d = rnd() % 4 != 0;
        put_head(o, 4, nt + (has_d ? 1 : 0));
        static const char* tk[] = {"t1", "t2", "t3", "t4"};
        for (unsigned t = 0; t < nt; t++) put_entry(o, rnd() % 8 == 0 ? rnd() % 24 : 3, tk[t], rnd() % 16 == 0 ? rnd() % 24 : 0x55, rnd() % 32 == 0 ? rnd() % 40 : 32);
        if (has_d) put_entry(o, 3, "d", 0x55, rnd() % 6 == 0 ? 256 + rnd() % 200 : rnd() % 64);
    }
    return o;
}
static bool same(const EvLog& a, const EvLog& b) {
    if (a.emitter != b.emitter || a.some != b.some || a.case_a != b.case_a || a.ntopics != b.ntopics) return false;
    if (a.data_off != b.data_off || a.data_len != b.data_len) return false;
    for (int k = 0; k < 4; k++) if (a.toff[k] != b.toff[k]) return false;
    return true;
}

// ---- second property: the byte-layout check of the dense message-AMT walk vs the strict node decoder --------------------
// MIRROR of the checks in csrc/events.cu `amt_item_dense` (non-root part; the kernel inlines them between its loads): keep
// the two in step. Property: whatever this accepts, amt_node_begin + rd_cid… + amt_node_finish accept with the same
// bitmap / link count / value count (and therefore the same links at the same offsets).
static bool dense_accepts(const uint8_t* q, uint32_t nlen, uint32_t level, uint32_t n_exp, uint32_t& bm8, uint32_t& nl, uint32_t& nv) {
    if (nlen < 5) return false;
    const uint32_t exp_nl = level ? n_exp : 0u;
    const uint32_t tpos = 4u + 43u * exp_nl < nlen - 1u ? 4u + 43u * exp_nl : nlen - 1u;
    const uint32_t w = (uint32_t)load_u64_any(q);
    const uint32_t tb = q[tpos];
    bm8 = (w >> 16) & 0xffu;
    nl = (w >> 24) - 0x80u;
    if ((w & 0xffffu) != 0x4183u || nl != exp_nl || 4u + 43u * nl >= nlen) return false;
    nv = tb - 0x80u;
    if (nv > 8u || nlen != 5u + 43u * (nl + nv) || (nl && nv) || (nl && level == 0) || (nv && level != 0) || (uint32_t)__builtin_popcount(bm8) != nl + nv) return false;
    if (bm8 != (1u << n_exp) - 1u || (level ? nl : nv) != n_exp) return false;
    for (uint32_t j = 0; j < n_exp; j++) {
        uint32_t ipos = (level ? 4u : 5u) + 43u * j, cap = nlen - (nlen < 8u ? nlen : 8u);
        if (ipos > cap) ipos = cap;
        if ((load_u64_any(q + ipos) & 0xffffffffffffull) != 0x010027582ad8ull) return false;
    }
    return true;
}
static int fuzz_amt_nodes(uint64_t iters) {
    uint64_t accepted = 0, strict_ok = 0;
    std::vector<uint8_t> buf;
    for (uint64_t it = 0; it < iters; it++) {
        uint32_t level = (uint32_t)(rnd() % 3), n = (uint32_t)(rnd() % 9);
        std::vector<uint8_t> node = {0x83, 0x41, (uint8_t)((1u << n) - 1u)};
        if (rnd() % 16 == 0) node[2] = (uint8_t)rnd();                      // a sparse / wrong bitmap
        auto links = [&](uint32_t k) {
            node.push_back((uint8_t)(0x80 + k));
            for (uint32_t i = 0; i < k; i++) {
                static const uint8_t head[11] = {0xd8, 0x2a, 0x58, 0x27, 0x00, 0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
                node.insert(node.end(), head, head + 11);
                for (int b = 0; b < 32; b++) node.push_back((uint8_t)rnd());
            }
        };
        if (level) { links(n); node.push_back(0x80); } else { node.push_back(0x80); links(n); }
        unsigned nmut = it % 2 ? 1 + (unsigned)(rnd() % 2) : 0;
        for (unsigned m = 0; m < nmut; m++) {
            size_t at = rnd() % node.size();
            switch (rnd() % 4) {
                case 0: node[at] = (uint8_t)rnd(); break;
                case 1: node[at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                case 2: node.erase(node.begin() + (long)at); break;
                default: node.insert(node.begin() + (long)at, (uint8_t)rnd()); break;
            }
            if (node.empty()) node.push_back(0x83);
        }
        unsigned lead = (unsigned)(rnd() % 16);
        buf.assign(16 + lead, 0xEE);
        buf.insert(buf.end(), node.begin(), node.end());
        buf.insert(buf.end(), 48, (uint8_t)rnd());
        const uint8_t* q = buf.data() + 16 + lead;
        const uint32_t nlen = (uint32_t)node.size();
        uint32_t n_exp = rnd() % 8 == 0 ? (uint32_t)(rnd() % 9) : n;       // what the plan expects (sometimes not what is there)
        uint32_t bm8 = 0, nl = 0, nv = 0;
        bool acc = dense_accepts(q, nlen, level, n_exp, bm8, nl, nv);
        Rd r(q, nlen);
        AmtNodeHdr h;
        amt_node_begin(r, 3, h);
        uint32_t snv = rd_array(r);
        for (uint32_t v = 0; v < snv && !r.err; v++) (void)rd_cid(r);
        amt_node_finish(r, h, snv, level);
        if (!r.err) strict_ok++;
        if (!acc) continue;
        accepted++;
        if (r.err || h.nl != nl || snv != nv || (uint32_t)(h.bm.b0 & 0xff) != bm8 || h.links_off != 4) {
            fprintf(stderr, "AMT MISMATCH at iteration %llu: dense accepted (nl %u nv %u bm %02x), strict err %u nl %u nv %u\n", (unsigned long long)it, nl, nv, bm8,
                    r.err, h.nl, snv);
            return 1;
        }
    }
    printf("ok: %llu AMT nodes, dense layout check accepted %llu (all accepted identically by the strict decoder); strict decoder accepted %llu\n",
           (unsigned long long)iters, (unsigned long long)accepted, (unsigned long long)strict_ok);
    return 0;
}

// ---- fourth property: pass 1's per-receipt unit (one events-AMT v3 root block) vs the oracle ----------------------------
// Device side = the arena decode sequence of pass 1 / node_events (csrc/pass1_stage.cuh) built from the same header functions:
// amt_root_begin(v3) → amt_node_begin → values via decode_stamped_event (fast path + strict fallback) → amt_node_finish.
// Compared: status class (ok / decode error / child block missing) and, when ok, the visited (index, emitter, Some, #topics,
// data length) list — i.e. everything pass 1 and the proof emission of pass 2 derive from the block.
static std::vector<uint8_t> make_events_root() {
    std::vector<uint8_t> o;
    uint32_t bw = rnd() % 8 == 0 ? (uint32_t)(1 + rnd() % 8) : (rnd() % 2 ? 5u : 3u);
    uint32_t width = 1u << bw, nmax = width < 12 ? width : 12;
    uint32_t n = (uint32_t)(rnd() % (nmax + 1));
    std::vector<uint8_t> bm(bw <= 3 ? 1 : (1u << (bw - 3)), 0);
    for (uint32_t k = 0; k < n;) { uint32_t b = (uint32_t)(rnd() % width); if (!(bm[b / 8] >> (b % 8) & 1)) { bm[b / 8] |= (uint8_t)(1u << (b % 8)); k++; } }
    put_head(o, 4, 4);
    put_head(o, 0, bw);
    put_head(o, 0, rnd() % 16 == 0 ? rnd() % 3 : 0);       // height (mostly 0)
    put_head(o, 0, n);
    put_head(o, 4, 3);
    put_head(o, 2, bm.size());
    o.insert(o.end(), bm.begin(), bm.end());
    if (rnd() % 32 == 0) {                                    // a node with links
        uint32_t nl = 1 + (uint32_t)(rnd() % 3);
        put_head(o, 4, nl);
        for (uint32_t i = 0; i < nl; i++) {
            static const uint8_t head[11] = {0xd8, 0x2a, 0x58, 0x27, 0x00, 0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
            o.insert(o.end(), head, head + 11);
            for (int b = 0; b < 32; b++) o.push_back((uint8_t)rnd());
        }
        put_head(o, 4, 0);
        return o;
    }
    put_head(o, 4, 0);
    put_head(o, 4, n);
    for (uint32_t k = 0; k < n; k++) { std::vector<uint8_t> e = make_event(); o.insert(o.end(), e.begin(), e.end()); }
    return o;
}
static int fuzz_events_roots(uint64_t iters) {
    uint64_t ok_blocks = 0, dec_err = 0, missing = 0, events = 0;
    std::vector<uint8_t> buf;
    const uint64_t CAP = 64;
    uint64_t oidx[CAP], oem[CAP], odl[CAP];
    uint8_t osome[CAP];
    uint32_t ont[CAP];
    for (uint64_t it = 0; it < iters; it++) {
        std::vector<uint8_t> blk = make_events_root();
        unsigned nmut = it % 2 ? 1 + (unsigned)(rnd() % 2) : 0;
        for (unsigned m = 0; m < nmut; m++) {
            size_t at = rnd() % blk.size();
            switch (rnd() % 4) {
                case 0: blk[at] = (uint8_t)rnd(); break;
                case 1: blk[at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                case 2: blk.erase(blk.begin() + (long)at); break;
                default: blk.insert(blk.begin() + (long)at, (uint8_t)rnd()); break;
            }
            if (blk.empty()) blk.push_back(0x84);
        }
        unsigned lead = (unsigned)(rnd() % 16);
        buf.assign(16 + lead, 0xEE);
        buf.insert(buf.end(), blk.begin(), blk.end());
        buf.insert(buf.end(), 48, (uint8_t)rnd());
        const uint8_t* p = buf.data() + 16 + lead;
        const uint32_t len = (uint32_t)blk.size();
        // device sequence
        Rd r(p, len);
        uint32_t bw, height;
        uint64_t cnt;
        amt_root_begin(r, 3, bw, height, cnt);
        AmtNodeHdr h;
        amt_node_begin(r, bw, h);
        uint32_t nv = rd_array(r);
        uint64_t didx[CAP], dem[CAP], ddl[CAP];
        uint8_t dsome[CAP];
        uint32_t dnt[CAP];
        uint64_t dn = 0;
        for (uint32_t v = 0; v < nv && !r.err; v++) {
            EvLog ev;
            decode_stamped_event(r, ev);
            if (r.err) break;
            if (dn < CAP) { didx[dn] = bm_select(h.bm, v); dem[dn] = ev.emitter; dsome[dn] = (uint8_t)ev.some; dnt[dn] = ev.some ? ev.ntopics : 0; ddl[dn] = ev.some ? ev.data_len : 0; }
            dn++;
        }
        amt_node_finish(r, h, nv, height);
        int dstatus = r.err ? IPCFP_ERR_DECODE : (h.nl ? IPCFP_ERR_MISSING_BLOCK : IPCFP_OK);   // links: the walker's first child lookup fails
        uint64_t on = 0;
        int ostatus = (int)oracle_scan_events_block(p, len, &on, oidx, oem, osome, ont, odl, CAP);
        bool ok = dstatus == ostatus;
        if (ok && dstatus == IPCFP_OK) {
            ok = on == dn;
            for (uint64_t k = 0; ok && k < dn && k < CAP; k++) ok = didx[k] == oidx[k] && dem[k] == oem[k] && dsome[k] == osome[k] && dnt[k] == ont[k] && ddl[k] == odl[k];
        }
        if (!ok) {
            fprintf(stderr, "ROOT MISMATCH at iteration %llu: device status %d (%llu events, err %u), oracle status %d (%llu events)\nblock:", (unsigned long long)it,
                    dstatus, (unsigned long long)dn, r.err, ostatus, (unsigned long long)on);
            for (size_t k = 0; k < blk.size(); k++) fprintf(stderr, " %02x", blk[k]);
            fprintf(stderr, "\n");
            return 1;
        }
        if (dstatus == IPCFP_OK) { ok_blocks++; events += dn; } else if (dstatus == IPCFP_ERR_DECODE) dec_err++; else missing++;
    }
    printf("ok: %llu events-AMT root blocks agree with the oracle (%llu decoded with %llu events, %llu decode errors, %llu with child links)\n",
           (unsigned long long)iters, (unsigned long long)ok_blocks, (unsigned long long)events, (unsigned long long)dec_err, (unsigned long long)missing);
    return 0;
}

// ---- fifth property: one receipts-AMT node (the unit of amt_get in csrc/ipld.cuh, pass 2's path walk) vs the oracle ---
static int fuzz_receipt_nodes(uint64_t iters) {
    uint64_t okn = 0, bad = 0;
    std::vector<uint8_t> buf;
    for (uint64_t it = 0; it < iters; it++) {
        uint32_t height = (uint32_t)(rnd() % 3), n = (uint32_t)(rnd() % 9);
        std::vector<uint8_t> node;
        put_head(node, 4, 3);
        put_head(node, 2, 1);
        uint8_t bm = 0;
        for (uint32_t k = 0; k < n;) { uint32_t b = (uint32_t)(rnd() % 8); if (!(bm >> b & 1)) { bm |= (uint8_t)(1u << b); k++; } }
        node.push_back(bm);
        auto cid = [&]() {
            static const uint8_t head[11] = {0xd8, 0x2a, 0x58, 0x27, 0x00, 0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
            node.insert(node.end(), head, head + 11);
            for (int b = 0; b < 32; b++) node.push_back((uint8_t)rnd());
        };
        if (height) { put_head(node, 4, n); for (uint32_t k = 0; k < n; k++) cid(); put_head(node, 4, 0); }
        else {
            put_head(node, 4, 0);
            put_head(node, 4, n);
            for (uint32_t k = 0; k < n; k++) {
                put_head(node, 4, 4);
                put_head(node, rnd() % 32 == 0 ? 1 : 0, rnd() % 8 == 0 ? rnd() : rnd() % 40);   // exit code (sometimes negative / huge)
                size_t rl = rnd() % 8 == 0 ? rnd() % 70 : 0;
                put_head(node, 2, rl);
                for (size_t b = 0; b < rl; b++) node.push_back((uint8_t)rnd());
                put_head(node, 0, rnd() % (1ull << 33));
                if (rnd() % 4 == 0) node.push_back(0xf6); else cid();
            }
        }
        unsigned nmut = it % 2 ? 1 + (unsigned)(rnd() % 2) : 0;
        for (unsigned m = 0; m < nmut; m++) {
            size_t at = rnd() % node.size();
            switch (rnd() % 4) {
                case 0: node[at] = (uint8_t)rnd(); break;
                case 1: node[at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                case 2: node.erase(node.begin() + (long)at); break;
                default: node.insert(node.begin() + (long)at, (uint8_t)rnd()); break;
            }
            if (node.empty()) node.push_back(0x83);
        }
        unsigned lead = (unsigned)(rnd() % 16);
        buf.assign(16 + lead, 0xEE);
        buf.insert(buf.end(), node.begin(), node.end());
        buf.insert(buf.end(), 48, (uint8_t)rnd());
        const uint8_t* p = buf.data() + 16 + lead;
        const uint32_t len = (uint32_t)node.size();
        Rd r(p, len);
        AmtNodeHdr h;
        amt_node_begin(r, 3, h);
        uint32_t nv = rd_array(r);
        uint32_t root_off[8];
        for (uint32_t v = 0; v < nv && !r.err; v++) {           // the product's decoder, keeping where the events root is
            uint32_t off = parse_receipt(r);
            if (v < 8) root_off[v] = off;
        }
        amt_node_finish(r, h, nv, height);
        uint32_t onl = 0, onv = 0;
        uint8_t has[16], roots[16 * 38];
        int ost = (int)oracle_decode_receipts_node(p, len, height, &onl, &onv, has, roots, 16);
        bool ok = (ost == IPCFP_OK) == (r.err == 0);
        if (ok && !r.err) {
            ok = onl == h.nl && onv == nv;
            for (uint32_t v = 0; ok && v < nv && v < 8; v++) {
                bool dev_has = root_off[v] != 0xffffffffu;
                ok = dev_has == (has[v] != 0) && (!dev_has || memcmp(p + root_off[v], roots + 38 * v, 38) == 0);
            }
        }
        if (!ok) {
            fprintf(stderr, "RECEIPT NODE MISMATCH at iteration %llu: device err %u nl %u nv %u; oracle status %d nl %u nv %u\nnode:", (unsigned long long)it, r.err, h.nl, nv,
                    ost, onl, onv);
            for (size_t k = 0; k < node.size(); k++) fprintf(stderr, " %02x", node[k]);
            fprintf(stderr, "\n");
            return 1;
        }
        if (r.err) bad++; else okn++;
    }
    printf("ok: %llu receipts-AMT nodes agree with the oracle (%llu decoded, %llu decode errors)\n", (unsigned long long)iters, (unsigned long long)okn,
           (unsigned long long)bad);
    return 0;
}

// ---- sixth property: one HAMT node (state tree / EVM storage, csrc/storage.cu hamt_get's unit) vs the oracle --------------
static int fuzz_hamt_nodes(uint64_t iters) {
    uint64_t okn = 0, bad = 0, hits = 0, links = 0, fast_ok = 0;
    std::vector<uint8_t> buf;
    for (uint64_t it = 0; it < iters; it++) {
        int vkind = (int)(rnd() % 2);
        uint32_t np = (uint32_t)(rnd() % 6);
        // bitfield with np bits among the low 32 slots (bit width 5), big-endian, right aligned, minimal or padded
        uint32_t bits = 0;
        for (uint32_t k = 0; k < np;) { uint32_t b = (uint32_t)(rnd() % 32); if (!(bits >> b & 1)) { bits |= 1u << b; k++; } }
        std::vector<uint8_t> bf;
        for (int s = 24; s >= 0; s -= 8) if (!bf.empty() || (bits >> s) & 0xff || rnd() % 8 == 0) bf.push_back((uint8_t)(bits >> s));
        if (rnd() % 16 == 0) bf.insert(bf.begin(), (size_t)(rnd() % 30), 0);
        std::vector<uint8_t> node;
        put_head(node, 4, 2);
        put_head(node, 2, bf.size());
        node.insert(node.end(), bf.begin(), bf.end());
        put_head(node, 4, np);
        std::vector<std::vector<uint8_t>> keys;
        auto cid = [&]() {
            static const uint8_t head[11] = {0xd8, 0x2a, 0x58, 0x27, 0x00, 0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
            node.insert(node.end(), head, head + 11);
            for (int b = 0; b < 32; b++) node.push_back((uint8_t)rnd());
        };
        for (uint32_t k = 0; k < np; k++) {
            if (rnd() % 3 == 0) { cid(); continue; }
            uint32_t nk = 1 + (uint32_t)(rnd() % 3);
            put_head(node, 4, nk);
            for (uint32_t j = 0; j < nk; j++) {
                put_head(node, 4, 2);
                std::vector<uint8_t> key(vkind ? 32 : 1 + rnd() % 9);
                for (auto& b : key) b = (uint8_t)rnd();
                if (!keys.empty() && rnd() % 16 == 0) key = keys[rnd() % keys.size()];    // a repeated key: the first one wins
                keys.push_back(key);
                put_head(node, 2, key.size());
                node.insert(node.end(), key.begin(), key.end());
                if (vkind == 0) {
                    put_head(node, 4, 5);
                    cid(); cid();
                    put_head(node, 0, rnd() % 100000);
                    size_t bl = rnd() % 12;
                    put_head(node, 2, bl);
                    for (size_t b = 0; b < bl; b++) node.push_back((uint8_t)rnd());
                    if (rnd() % 2) node.push_back(0xf6); else { put_head(node, 2, 3); node.push_back(1); node.push_back(2); node.push_back(3); }
                } else {
                    size_t vl = rnd() % 34;
                    put_head(node, 4, vl);
                    for (size_t b = 0; b < vl; b++) put_head(node, 0, rnd() % 16 == 0 ? rnd() % 300 : rnd() % 256);
                }
            }
        }
        unsigned nmut = it % 2 ? 1 + (unsigned)(rnd() % 2) : 0;
        for (unsigned m = 0; m < nmut; m++) {
            size_t at = rnd() % node.size();
            switch (rnd() % 4) {
                case 0: node[at] = (uint8_t)rnd(); break;
                case 1: node[at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                case 2: node.erase(node.begin() + (long)at); break;
                default: node.insert(node.begin() + (long)at, (uint8_t)rnd()); break;
            }
            if (node.empty()) node.push_back(0x82);
        }
        std::vector<uint8_t> key = (!keys.empty() && rnd() % 4) ? keys[rnd() % keys.size()] : std::vector<uint8_t>(vkind ? 32 : 3, (uint8_t)rnd());
        uint32_t idx = rnd() % 4 ? (uint32_t)(rnd() % 32) : (uint32_t)(rnd() % 256);
        if (bits && rnd() % 2) { do idx = (uint32_t)(rnd() % 32); while (!(bits >> idx & 1)); }
        unsigned lead = (unsigned)(rnd() % 16);
        buf.assign(16 + lead, 0xEE);
        buf.insert(buf.end(), node.begin(), node.end());
        buf.insert(buf.end(), 48, (uint8_t)rnd());
        const uint8_t* p = buf.data() + 16 + lead;
        const uint32_t len = (uint32_t)node.size();
        Rd r(p, len);
        HamtHit hit;
        hamt_node_lookup(r, vkind, idx, key.data(), (uint32_t)key.size(), hit);
        {   // the fast node decoder may only accept what the strict one accepts, with the same hit
            HamtHit fh;
            if (hamt_node_lookup_fast(p, len, vkind, idx, key.data(), (uint32_t)key.size(), fh)) {
                fast_ok++;
                if (r.err || fh.kind != hit.kind || (fh.kind == 1 && fh.val_off != hit.val_off) || (fh.kind == 2 && fh.link_off != hit.link_off)) {
                    fprintf(stderr, "HAMT FAST/STRICT MISMATCH at iteration %llu: strict err %u kind %d, fast kind %d\nnode:", (unsigned long long)it, r.err, hit.kind, fh.kind);
                    for (size_t k = 0; k < node.size(); k++) fprintf(stderr, " %02x", node[k]);
                    fprintf(stderr, "\n");
                    return 1;
                }
            } else if (!r.err && nmut == 0 && bf.size() <= 32) { fprintf(stderr, "HAMT FAST: a generated, unmutated node was not taken (iteration %llu)\n", (unsigned long long)it); return 1; }
        }
        int32_t okind = 0;
        uint8_t oout[4096];
        uint64_t olen = 0;
        int ost = (int)oracle_hamt_node_lookup(p, len, vkind, idx, key.data(), (uint32_t)key.size(), &okind, oout, sizeof oout, &olen);
        bool ok = (ost == IPCFP_OK) == (r.err == 0);
        if (ok && !r.err) {
            ok = okind == hit.kind;
            if (ok && hit.kind == 2) ok = olen == 38 && memcmp(p + hit.link_off, oout, 38) == 0;
            if (ok && hit.kind == 1) {
                Rd r2(p, len);
                r2.pos = hit.val_off;
                if (vkind == 0) { uint32_t so; parse_actor_state(r2, so); ok = !r2.err && olen == 38 && memcmp(p + so, oout, 38) == 0; }
                else {
                    uint32_t fo;
                    uint32_t ne = parse_u8vec(r2, fo);
                    ok = !r2.err && ne == olen;
                    Rd r3(p, len);
                    r3.pos = fo;
                    for (uint32_t e = 0; ok && e < ne; e++) ok = rd_uint(r3) == oout[e];
                }
            }
        }
        if (!ok) {
            fprintf(stderr, "HAMT NODE MISMATCH at iteration %llu: device err %u kind %d; oracle status %d kind %d len %llu\nnode:", (unsigned long long)it, r.err, hit.kind, ost,
                    okind, (unsigned long long)olen);
            for (size_t k = 0; k < node.size(); k++) fprintf(stderr, " %02x", node[k]);
            fprintf(stderr, "\n");
            return 1;
        }
        if (r.err) bad++; else { okn++; hits += hit.kind == 1; links += hit.kind == 2; }
    }
    printf("ok: %llu HAMT nodes agree with the oracle (%llu decoded: %llu values found, %llu links; %llu decode errors; %llu taken by the fast node decoder)\n", (unsigned long long)iters,
           (unsigned long long)okn, (unsigned long long)hits, (unsigned long long)links, (unsigned long long)bad, (unsigned long long)fast_ok);
    return 0;
}

int main(int argc, char** argv) {
    uint64_t iters = argc > 1 ? strtoull(argv[1], nullptr, 10) : 2000000;
    rng_state = argc > 2 ? strtoull(argv[2], nullptr, 10) : 0x1FC0FFEEull;
    {   // the window loader gives the same 16 bytes as memcpy at every alignment
        alignas(16) uint8_t buf[128];
        for (int k = 0; k < 128; k++) buf[k] = (uint8_t)rnd();
        for (int off = 16; off < 64; off++) {
            uint64_t a0, a1;
            win_load(buf + off, a0, a1);
            uint64_t e0, e1;
            memcpy(&e0, buf + off, 8); memcpy(&e1, buf + off + 8, 8);
            if (a0 != e0 || a1 != e1) { fprintf(stderr, "WINDOW LOADER DISAGREES at offset %d\n", off); return 1; }
        }
    }
    uint64_t accepted = 0, rejected = 0, strict_ok = 0, oracle_checked = 0;
    std::vector<uint8_t> buf;
    for (uint64_t it = 0; it < iters; it++) {
        std::vector<uint8_t> ev = make_event();
        unsigned lead = (unsigned)(rnd() % 24);              // any alignment, something before and after
        buf.assign(16, 0xEE);                                 // the arena's lead padding
        for (unsigned k = 0; k < lead; k++) buf.push_back((uint8_t)rnd());
        size_t start = buf.size();
        unsigned nmut = it % 3 == 0 ? 0 : 1 + (unsigned)(rnd() % 3);
        for (unsigned m = 0; m < nmut; m++) {
            size_t at = rnd() % ev.size();
            switch (rnd() % 4) {
                case 0: ev[at] = (uint8_t)rnd(); break;
                case 1: ev[at] ^= (uint8_t)(1u << (rnd() % 8)); break;
                case 2: ev.erase(ev.begin() + (long)at); break;
                default: ev.insert(ev.begin() + (long)at, (uint8_t)rnd()); break;
            }
            if (ev.empty()) ev.push_back(0x82);
        }
        buf.insert(buf.end(), ev.begin(), ev.end());
        unsigned tail = (unsigned)(rnd() % 40);               // bytes of the "next item" the decoders must not depend on
        for (unsigned k = 0; k < tail; k++) buf.push_back((uint8_t)rnd());
        uint32_t n = (uint32_t)(lead + ev.size() + (rnd() % 2 ? tail : 0));   // block length: with or without trailing items
        buf.insert(buf.end(), 48, 0xEE);                       // the arena's tail padding
        const uint8_t* p = buf.data() + 16;
        uint32_t pos = lead;
        (void)start;
        EvLog f;
        memset(&f, 0, sizeof f);
        uint32_t np = fast_stamped_event(p, pos, n, f);
        Rd r(p, n);
        r.pos = pos;
        EvLog s;
        parse_stamped_event(r, s);
        if (!r.err) strict_ok++;
        {   // device strict decoder vs the oracle
            uint64_t consumed = 0, emitter = 0, dlen = 0;
            uint32_t some = 0, nt = 0;
            static uint8_t tbuf[32 * 64], dbuf[1 << 16];
            ipcfp_status st = oracle_decode_event(p + pos, n - pos, &consumed, &emitter, &some, &nt, tbuf, sizeof tbuf, dbuf, sizeof dbuf, &dlen);
            bool ok = (st == IPCFP_OK) == (r.err == 0);
            if (ok && st == IPCFP_OK) {
                ok = consumed == r.pos - pos && emitter == s.emitter && some == s.some && (!some || (nt == s.ntopics && dlen == s.data_len));
                for (uint32_t k = 0; ok && some && k < nt && k < 64; k++) ok = memcmp(tbuf + 32 * k, p + topic_offset(s, k), 32) == 0;
                if (ok && some && dlen) ok = memcmp(dbuf, p + s.data_off, dlen < sizeof dbuf ? dlen : sizeof dbuf) == 0;
            }
            if (!ok) {
                fprintf(stderr, "ORACLE MISMATCH at iteration %llu: oracle status %d consumed %llu some %u nt %u dlen %llu; device err %u next %u some %u nt %u dlen %u\n",
                        (unsigned long long)it, (int)st, (unsigned long long)consumed, some, nt, (unsigned long long)dlen, r.err, r.pos - pos, s.some, s.ntopics, s.data_len);
                fprintf(stderr, "event bytes:");
                for (size_t k = 0; k < ev.size(); k++) fprintf(stderr, " %02x", ev[k]);
                fprintf(stderr, "\n");
                return 1;
            }
            oracle_checked++;
        }
        if (np == FAST_FAIL) { rejected++; continue; }
        accepted++;
        if (r.err || r.pos != np || !same(f, s)) {
            fprintf(stderr, "MISMATCH at iteration %llu: fast accepted (next %u), strict err %u next %u\n", (unsigned long long)it, np, r.err, r.pos);
            fprintf(stderr, "event bytes:");
            for (size_t k = 0; k < ev.size(); k++) fprintf(stderr, " %02x", ev[k]);
            fprintf(stderr, "\n");
            return 1;
        }
    }
    if (fuzz_amt_nodes(iters / 2)) return 1;
    if (fuzz_events_roots(iters / 8)) return 1;
    if (fuzz_receipt_nodes(iters / 4)) return 1;
    if (fuzz_hamt_nodes(iters / 4)) return 1;
    printf("ok: %llu events, fast path accepted %llu (all equal to the strict decoder), declined %llu; strict decoder accepted %llu; %llu compared with the oracle\n",
           (unsigned long long)iters, (unsigned long long)accepted, (unsigned long long)rejected, (unsigned long long)strict_ok, (unsigned long long)oracle_checked);
    return 0;
}
