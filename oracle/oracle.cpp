// oracle.cpp — CPU restatement of the reference's receipt/event scan and storage-slot path.
// TEST INFRASTRUCTURE (see oracle.h header comment: parity unpinned by the reference).
//
// Orchestration follows, line by line:
//   src/proofs/events/generator.rs:23-307   EventMatcher, generate_event_proof, find_matching_events
//   src/proofs/events/utils.rs:16-94        reconstruct_execution_order / collect_exec_list
//   src/proofs/common/evm.rs:13-100         extract_evm_log, keccak helpers, left_pad_32
//   src/proofs/common/blockstore.rs:8-39    RecordingBlockStore
//   src/proofs/common/witness.rs:9-57       WitnessCollector
//   src/proofs/storage/decode.rs:9-97       read_storage_slot (shape sniffing A1..C)
//   src/proofs/storage/generator.rs:29-178  generate_storage_proof
//   src/proofs/common/decode.rs:17-124      get_actor_state, parse_evm_state, HeaderLite
//   src/proofs/generator.rs:25-95           generate_proof_bundle
//   src/proofs/events/verifier.rs:51-290, src/proofs/storage/verifier.rs:24-170   verifiers
// The crates' arithmetic ([UPSTREAM], not in the reference tree) is restated from their
// published formats: SURVEY.md Appendix A; the decode contract is written down in DESIGN.md §3.
//
// Deliberately mirrors the reference's allocation behaviour (get() clones the block, every
// event entry owns its key String and value Vec, extract_evm_log builds a map per event,
// recorders are ordered sets) so that its timing is an honest stand-in for the Rust code.
#include "oracle.h"
#include "../synth/cpu_crypto.h"

#include <algorithm>
#include <array>
#include <chrono>
#include <cstdio>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <variant>
#include <vector>

// memcpy whose source may be an empty container's data() (nullptr with n == 0 — flagged by UBSan, harmless in practice)
static inline void copy_bytes(void* dst, const void* src, size_t n) { if (n) memcpy(dst, src, n); }
namespace orc {

typedef std::vector<uint8_t> Bytes;

struct Err {
    ipcfp_status status;
    std::string msg;
    uint64_t index;
    Err(ipcfp_status s, std::string m, uint64_t i = UINT64_MAX) : status(s), msg(std::move(m)), index(i) {}
};
[[noreturn]] static void fail_decode(const char* what) { throw Err(IPCFP_ERR_DECODE, std::string("decode: ") + what); }

// ---------------------------------------------------------------------------------- Cid
struct Cid {
    std::array<uint8_t, 38> b{};
    bool operator==(const Cid& o) const { return b == o.b; }
    bool operator!=(const Cid& o) const { return !(b == o.b); }
};
static bool read_varint(const uint8_t* p, size_t n, size_t& pos, uint64_t& v) {
    v = 0;
    for (int shift = 0; shift < 64; shift += 7) {
        if (pos >= n) return false;
        uint8_t c = p[pos++];
        v |= (uint64_t)(c & 0x7f) << shift;
        if (!(c & 0x80)) return true;
    }
    return false;
}
struct CidKey { uint64_t version, codec, code, size; const uint8_t* digest; size_t dlen; };
static CidKey cid_key(const Cid& c) {
    CidKey k{0, 0, 0, 0, nullptr, 0};
    size_t pos = 0;
    read_varint(c.b.data(), 38, pos, k.version);
    read_varint(c.b.data(), 38, pos, k.codec);
    read_varint(c.b.data(), 38, pos, k.code);
    read_varint(c.b.data(), 38, pos, k.size);
    k.digest = c.b.data() + pos;
    k.dlen = 38 - pos;
    return k;
}
// `Ord` of cid::Cid: derived over (version, codec, hash); Multihash over (code, size, digest)
static bool cid_less(const Cid& a, const Cid& b) {
    CidKey x = cid_key(a), y = cid_key(b);
    if (x.version != y.version) return x.version < y.version;
    if (x.codec != y.codec) return x.codec < y.codec;
    if (x.code != y.code) return x.code < y.code;
    if (x.size != y.size) return x.size < y.size;
    size_t n = std::min(x.dlen, y.dlen);
    int c = memcmp(x.digest, y.digest, n);
    if (c) return c < 0;
    return x.dlen < y.dlen;
}
struct CidLess { bool operator()(const Cid& a, const Cid& b) const { return cid_less(a, b); } };
struct CidHash {
    size_t operator()(const Cid& c) const { uint64_t h; copy_bytes(&h, c.b.data() + 6, 8); uint64_t g; copy_bytes(&g, c.b.data() + 30, 8); return (size_t)(h ^ (g * 0x9E3779B97F4A7C15ULL)); }
};
static Cid cid_from(const uint8_t* p) { Cid c; copy_bytes(c.b.data(), p, 38); return c; }
static std::string cid_hex(const Cid& c) {
    static const char* hx = "0123456789abcdef";
    std::string s;
    for (int i = 6; i < 14; i++) { s.push_back(hx[c.b[i] >> 4]); s.push_back(hx[c.b[i] & 15]); }
    return s + "..";
}

// ---------------------------------------------------------------------------------- Blockstore
struct Blockstore {
    virtual ~Blockstore() {}
    // fvm_ipld_blockstore::Blockstore::get -> Result<Option<Vec<u8>>>: an owned copy
    virtual bool get(const Cid& k, Bytes& out) const = 0;
};
struct MemoryBlockstore : Blockstore {
    std::unordered_map<Cid, std::pair<const uint8_t*, uint32_t>, CidHash> m;
    std::vector<Bytes> owned;
    bool get(const Cid& k, Bytes& out) const override {
        auto it = m.find(k);
        if (it == m.end()) return false;
        out.assign(it->second.first, it->second.first + it->second.second);  // clone, like MemoryBlockstore::get
        return true;
    }
    void put_keyed(const Cid& k, const uint8_t* p, uint32_t n) {
        owned.emplace_back(p, p + n);
        m[k] = {owned.back().data(), n};
    }
};
// src/proofs/common/blockstore.rs:8-39
struct RecordingBlockStore : Blockstore {
    const Blockstore& inner;
    mutable std::set<Cid, CidLess> seen;
    explicit RecordingBlockStore(const Blockstore& i) : inner(i) {}
    bool get(const Cid& k, Bytes& out) const override {
        seen.insert(k);
        return inner.get(k, out);
    }
    std::vector<Cid> take_seen() const { return std::vector<Cid>(seen.begin(), seen.end()); }
};
// src/proofs/common/witness.rs:9-57
struct ProofBlock { Cid cid; Bytes data; };
struct WitnessCollector {
    std::set<Cid, CidLess> needed;
    const Blockstore& bs;
    explicit WitnessCollector(const Blockstore& b) : bs(b) {}
    void add_cid(const Cid& c) { needed.insert(c); }
    void collect_from_recording(const RecordingBlockStore& r) { for (auto& c : r.take_seen()) needed.insert(c); }
    std::vector<ProofBlock> materialize() const {
        std::vector<ProofBlock> out;
        out.reserve(needed.size());
        for (auto& c : needed) {
            ProofBlock pb;
            pb.cid = c;
            if (!bs.get(c, pb.data)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing block " + cid_hex(c));
            out.push_back(std::move(pb));
        }
        return out;
    }
};

// ---------------------------------------------------------------------------------- DAG-CBOR decoder
// Strict subset decoder (serde_ipld_dagcbor behaviour restated): definite lengths, minimal heads,
// typed positions, exact tuple lengths, tag 42 only, no trailing bytes.
struct Dec {
    const uint8_t* p;
    size_t n, pos;
    Dec(const Bytes& b) : p(b.data()), n(b.size()), pos(0) {}
    Dec(const uint8_t* q, size_t m) : p(q), n(m), pos(0) {}
    struct Head { int major; uint64_t arg; uint8_t ai; };
    Head head() {
        if (pos >= n) fail_decode("unexpected end");
        uint8_t ib = p[pos++];
        Head h;
        h.major = ib >> 5;
        h.ai = ib & 31;
        if (h.ai < 24) { h.arg = h.ai; return h; }
        if (h.ai > 27) fail_decode("indefinite/reserved additional info");
        int nb = 1 << (h.ai - 24);
        if (pos + (size_t)nb > n) fail_decode("truncated head");
        uint64_t v = 0;
        for (int i = 0; i < nb; i++) v = (v << 8) | p[pos++];
        h.arg = v;
        if (h.major != 7) {
            static const uint64_t minv[4] = {24, 0x100, 0x10000, 0x100000000ULL};
            if (v < minv[h.ai - 24]) fail_decode("non-minimal integer encoding");
        }
        return h;
    }
    int peek_major() const { if (pos >= n) fail_decode("unexpected end"); return p[pos] >> 5; }
    bool peek_null() const { return pos < n && p[pos] == 0xf6; }
    uint64_t uint() { Head h = head(); if (h.major != 0) fail_decode("expected uint"); return h.arg; }
    int64_t integer() {
        Head h = head();
        if (h.major == 0) { if (h.arg > (uint64_t)INT64_MAX) fail_decode("i64 overflow"); return (int64_t)h.arg; }
        if (h.major == 1) { if (h.arg > (uint64_t)INT64_MAX) fail_decode("i64 overflow"); return -1 - (int64_t)h.arg; }
        fail_decode("expected integer");
    }
    Bytes bytes() {
        Head h = head();
        if (h.major != 2) fail_decode("expected bytes");
        if (h.arg > n - pos) fail_decode("bytes out of bounds");
        Bytes out(p + pos, p + pos + h.arg);
        pos += h.arg;
        return out;
    }
    static bool utf8_ok(const uint8_t* s, size_t len) {
        size_t i = 0;
        while (i < len) {
            uint8_t c = s[i];
            if (c < 0x80) { i++; continue; }
            int extra; uint32_t cp;
            if ((c & 0xe0) == 0xc0) { extra = 1; cp = c & 0x1f; }
            else if ((c & 0xf0) == 0xe0) { extra = 2; cp = c & 0x0f; }
            else if ((c & 0xf8) == 0xf0) { extra = 3; cp = c & 0x07; }
            else return false;
            if ((size_t)extra > len - 1 - i) return false;
            for (int k = 1; k <= extra; k++) { uint8_t d = s[i + k]; if ((d & 0xc0) != 0x80) return false; cp = (cp << 6) | (d & 0x3f); }
            if (extra == 1 && cp < 0x80) return false;
            if (extra == 2 && (cp < 0x800 || (cp >= 0xd800 && cp <= 0xdfff))) return false;
            if (extra == 3 && (cp < 0x10000 || cp > 0x10ffff)) return false;
            i += 1 + (size_t)extra;
        }
        return true;
    }
    std::string text() {
        Head h = head();
        if (h.major != 3) fail_decode("expected text");
        if (h.arg > n - pos) fail_decode("text out of bounds");
        if (!utf8_ok(p + pos, (size_t)h.arg)) fail_decode("invalid utf-8");
        std::string s((const char*)p + pos, (size_t)h.arg);
        pos += h.arg;
        return s;
    }
    uint64_t array() { Head h = head(); if (h.major != 4) fail_decode("expected array"); return h.arg; }
    void array_exact(uint64_t k) { if (array() != k) fail_decode("tuple length mismatch"); }
    uint64_t map() { Head h = head(); if (h.major != 5) fail_decode("expected map"); return h.arg; }
    void null() { if (!peek_null()) fail_decode("expected null"); pos++; }
    Cid cid() {
        Head t = head();
        if (t.major != 6 || t.arg != 42) fail_decode("expected tag 42");
        Head h = head();
        if (h.major != 2) fail_decode("cid: expected bytes");
        if (h.arg > n - pos) fail_decode("cid out of bounds");
        if (h.arg != 39 || p[pos] != 0x00 || p[pos + 1] != 0x01) fail_decode("cid: unsupported form (need 0x00 + 38-byte CIDv1)");
        Cid c = cid_from(p + pos + 1);
        pos += 39;
        return c;
    }
    // serde IgnoredAny
    void skip_any() {
        uint64_t remaining = 1;
        while (remaining) {
            remaining--;
            Head h = head();
            switch (h.major) {
                case 0: case 1: break;
                case 2: if (h.arg > n - pos) fail_decode("bytes out of bounds"); pos += h.arg; break;
                case 3:
                    if (h.arg > n - pos) fail_decode("text out of bounds");
                    if (!utf8_ok(p + pos, (size_t)h.arg)) fail_decode("invalid utf-8");
                    pos += h.arg; break;
                case 4: if (h.arg > n - pos) fail_decode("array too long"); remaining += h.arg; break;
                case 5: if (h.arg > (n - pos) / 2 + 1) fail_decode("map too long"); remaining += 2 * h.arg; break;
                case 6: {
                    if (h.arg != 42) fail_decode("unsupported tag");
                    Head b = head();
                    if (b.major != 2 || b.arg > n - pos) fail_decode("cid: expected bytes");
                    if (b.arg < 1 || p[pos] != 0) fail_decode("cid: missing multibase prefix");
                    pos += b.arg;
                    break;
                }
                default:
                    if (h.ai == 20 || h.ai == 21 || h.ai == 22) break;  // false / true / null
                    if (h.ai == 27) break;                                // f64
                    fail_decode("unsupported simple value / float width");
            }
        }
    }
    void end() { if (pos != n) fail_decode("trailing bytes"); }
};

// ---------------------------------------------------------------------------------- typed values
struct Entry { uint64_t flags; std::string key; uint64_t codec; Bytes value; };
struct ActorEvent { std::vector<Entry> entries; };
struct StampedEvent { uint64_t emitter; ActorEvent event; };
struct Receipt { uint64_t exit_code; Bytes return_data; uint64_t gas_used; std::optional<Cid> events_root; };

template <class V> struct ValueDec;
template <> struct ValueDec<StampedEvent> {
    static StampedEvent dec(Dec& d) {
        StampedEvent se;
        d.array_exact(2);
        se.emitter = d.uint();
        uint64_t ne = d.array();
        if (ne > d.n) fail_decode("entries too long");
        se.event.entries.reserve((size_t)ne);
        for (uint64_t i = 0; i < ne; i++) {
            Entry e;
            d.array_exact(4);
            e.flags = d.uint();
            e.key = d.text();
            e.codec = d.uint();
            e.value = d.bytes();
            se.event.entries.push_back(std::move(e));
        }
        return se;
    }
};
template <> struct ValueDec<Receipt> {
    static Receipt dec(Dec& d) {
        Receipt r;
        d.array_exact(4);
        r.exit_code = d.uint();
        if (r.exit_code > 0xffffffffULL) fail_decode("exit code overflows u32");
        r.return_data = d.bytes();
        r.gas_used = d.uint();
        if (d.peek_null()) d.null(); else r.events_root = d.cid();
        return r;
    }
};
template <> struct ValueDec<Cid> { static Cid dec(Dec& d) { return d.cid(); } };

// ---------------------------------------------------------------------------------- AMT (fvm_ipld_amt restated)
static uint64_t pow_sat(uint64_t width_bits, uint64_t exp) {  // 2^(bw*exp), saturating
    uint64_t s = width_bits * exp;
    return s >= 64 ? UINT64_MAX : (1ull << s);
}
template <class V> struct AmtNode {
    std::vector<std::optional<Cid>> links;  // size width when interior
    std::vector<std::optional<V>> vals;     // size width when leaf
    bool leaf = true;
};
template <class V> static AmtNode<V> decode_amt_node(Dec& d, int bw, uint32_t height) {
    AmtNode<V> nd;
    d.array_exact(3);
    Bytes bmap = d.bytes();
    size_t want = bw <= 3 ? 1 : (size_t)1 << (bw - 3);
    if (bmap.size() != want) fail_decode("amt: bitmap length");
    const uint32_t width = 1u << bw;
    uint64_t nl = d.array();
    if (nl > d.n) fail_decode("amt: links too long");
    std::vector<Cid> links;
    links.reserve((size_t)nl);
    for (uint64_t i = 0; i < nl; i++) links.push_back(d.cid());
    uint64_t nv = d.array();
    if (nv > d.n) fail_decode("amt: values too long");
    std::vector<V> vals;
    vals.reserve((size_t)nv);
    for (uint64_t i = 0; i < nv; i++) vals.push_back(ValueDec<V>::dec(d));
    if (nl && nv) fail_decode("amt: node has both links and values");
    uint32_t pc = 0;
    for (size_t i = 0; i < bmap.size() * 8; i++)
        if (bmap[i / 8] & (1u << (i % 8))) { if (i >= width) fail_decode("amt: bit beyond width"); pc++; }
    if (nl) {
        if (height == 0) fail_decode("amt: links at height 0");
        if (pc != nl) fail_decode("amt: bitmap/links mismatch");
        nd.leaf = false;
        nd.links.resize(width);
        size_t k = 0;
        for (uint32_t i = 0; i < width; i++) if (bmap[i / 8] & (1u << (i % 8))) nd.links[i] = links[k++];
    } else {
        if (nv && height != 0) fail_decode("amt: values above height 0");
        if (pc != nv) fail_decode("amt: bitmap/values mismatch");
        nd.leaf = true;
        nd.vals.resize(width);
        size_t k = 0;
        for (uint32_t i = 0; i < width; i++) if (bmap[i / 8] & (1u << (i % 8))) nd.vals[i] = std::move(vals[k++]);
    }
    return nd;
}
template <class V> struct Amt {
    int bw = 3;
    uint32_t height = 0;
    uint64_t count = 0;
    AmtNode<V> root;
    const Blockstore* bs = nullptr;
    // version 0: Amtv0 root [height,count,node] (bw 3); version 3: Amt root [bw,height,count,node]
    static Amt load(const Cid& c, const Blockstore& store, int version) {
        Bytes raw;
        if (!store.get(c, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "amt root not found " + cid_hex(c));
        Dec d(raw);
        Amt a;
        a.bs = &store;
        if (version == 0) { d.array_exact(3); a.bw = 3; }
        else {
            d.array_exact(4);
            uint64_t bw = d.uint();
            if (bw < 1 || bw > 8) fail_decode("amt: unsupported bit width");
            a.bw = (int)bw;
        }
        uint64_t h = d.uint();
        if (h * (uint64_t)a.bw > 64) fail_decode("amt: height exceeds maximum");
        a.height = (uint32_t)h;
        a.count = d.uint();
        a.root = decode_amt_node<V>(d, a.bw, a.height);
        d.end();
        return a;
    }
    AmtNode<V> load_node(const Cid& c, uint32_t h) const {
        Bytes raw;
        if (!bs->get(c, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "amt node not found " + cid_hex(c));
        Dec d(raw);
        AmtNode<V> nd = decode_amt_node<V>(d, bw, h);
        d.end();
        return nd;
    }
    std::optional<V> get(uint64_t i) const {
        if (i >= pow_sat((uint64_t)bw, (uint64_t)height + 1)) return std::nullopt;
        const AmtNode<V>* cur = &root;
        AmtNode<V> tmp;
        for (uint32_t h = height;; h--) {
            uint64_t sub = pow_sat((uint64_t)bw, h);
            uint32_t idx = (uint32_t)((i / sub) % (1u << bw));
            if (cur->leaf) {
                if (h != 0) return std::nullopt;  // empty subtree above height 0
                if (!cur->vals[idx]) return std::nullopt;
                return cur->vals[idx];
            }
            if (!cur->links[idx]) return std::nullopt;
            tmp = load_node(*cur->links[idx], h - 1);
            cur = &tmp;
        }
    }
    void for_each_node(const AmtNode<V>& nd, uint32_t h, uint64_t base, const std::function<void(uint64_t, const V&)>& f) const {
        const uint32_t width = 1u << bw;
        if (nd.leaf) {
            for (uint32_t i = 0; i < width; i++) if (nd.vals.size() && nd.vals[i]) f(base + i, *nd.vals[i]);
            return;
        }
        uint64_t sub = pow_sat((uint64_t)bw, h);
        for (uint32_t i = 0; i < width; i++) {
            if (!nd.links[i]) continue;
            AmtNode<V> ch = load_node(*nd.links[i], h - 1);
            for_each_node(ch, h - 1, base + (uint64_t)i * sub, f);
        }
    }
    void for_each(const std::function<void(uint64_t, const V&)>& f) const { for_each_node(root, height, 0, f); }
    // range-restricted walk used by the sharded variant: visits nodes intersecting [lo,hi)
    void for_each_range_node(const AmtNode<V>& nd, uint32_t h, uint64_t base, uint64_t lo, uint64_t hi,
                             const std::function<void(uint64_t, const V&)>& f) const {
        const uint32_t width = 1u << bw;
        if (nd.leaf) {
            for (uint32_t i = 0; i < width; i++)
                if (nd.vals.size() && nd.vals[i] && base + i >= lo && base + i < hi) f(base + i, *nd.vals[i]);
            return;
        }
        uint64_t sub = pow_sat((uint64_t)bw, h);
        for (uint32_t i = 0; i < width; i++) {
            if (!nd.links[i]) continue;
            uint64_t a = base + (uint64_t)i * sub, b = (sub == UINT64_MAX) ? UINT64_MAX : a + sub;
            if (!(a < hi && b > lo)) continue;
            AmtNode<V> ch = load_node(*nd.links[i], h - 1);
            for_each_range_node(ch, h - 1, a, lo, hi, f);
        }
    }
};

// ---------------------------------------------------------------------------------- HAMT (fvm_ipld_hamt v3 restated)
struct ActorState { Cid code, state; uint64_t sequence; Bytes balance; std::optional<Bytes> delegated; };
struct RawU8Vec { Bytes v; };  // serde Vec<u8> (a CBOR array of u8, NOT a byte string — see DESIGN.md §3)
template <> struct ValueDec<ActorState> {
    static ActorState dec(Dec& d) {
        ActorState a;
        d.array_exact(5);
        a.code = d.cid(); a.state = d.cid(); a.sequence = d.uint(); a.balance = d.bytes();
        if (d.peek_null()) d.null(); else a.delegated = d.bytes();
        return a;
    }
};
template <> struct ValueDec<RawU8Vec> {
    static RawU8Vec dec(Dec& d) {
        RawU8Vec r;
        uint64_t n = d.array();
        if (n > d.n) fail_decode("value array too long");
        r.v.reserve((size_t)n);
        for (uint64_t i = 0; i < n; i++) { uint64_t x = d.uint(); if (x > 255) fail_decode("u8 overflow"); r.v.push_back((uint8_t)x); }
        return r;
    }
};
template <class V> struct HamtNode {
    uint8_t bitfield[32];  // big-endian 256-bit
    struct KV { Bytes key; V val; };
    std::vector<std::variant<Cid, std::vector<KV>>> ptrs;
    bool test(uint32_t idx) const { return bitfield[31 - idx / 8] & (1u << (idx % 8)); }
    uint32_t index_for(uint32_t idx) const {
        uint32_t c = 0;
        for (uint32_t i = 0; i < idx; i++) if (test(i)) c++;
        return c;
    }
};
template <class V> static HamtNode<V> decode_hamt_node(const Bytes& raw) {
    Dec d(raw);
    HamtNode<V> nd;
    d.array_exact(2);
    Bytes bf = d.bytes();
    if (bf.size() > 32) fail_decode("hamt: bitfield too long");
    memset(nd.bitfield, 0, 32);
    copy_bytes(nd.bitfield + 32 - bf.size(), bf.data(), bf.size());
    uint64_t np = d.array();
    if (np > d.n) fail_decode("hamt: pointers too long");
    for (uint64_t i = 0; i < np; i++) {
        int mj = d.peek_major();
        if (mj == 6) nd.ptrs.emplace_back(d.cid());
        else if (mj == 4) {
            uint64_t nk = d.array();
            if (nk > d.n) fail_decode("hamt: bucket too long");
            std::vector<typename HamtNode<V>::KV> kvs;
            for (uint64_t k = 0; k < nk; k++) {
                typename HamtNode<V>::KV kv;
                d.array_exact(2);
                kv.key = d.bytes();
                kv.val = ValueDec<V>::dec(d);
                kvs.push_back(std::move(kv));
            }
            nd.ptrs.emplace_back(std::move(kvs));
        } else fail_decode("hamt: pointer must be link or bucket");
    }
    d.end();
    uint32_t pc = 0;
    for (int i = 0; i < 32; i++) pc += (uint32_t)__builtin_popcount(nd.bitfield[i]);
    if (pc != np) fail_decode("hamt: bitfield/pointers mismatch");
    return nd;
}
template <class V> static std::optional<V> hamt_get(const Blockstore& bs, const Cid& root, uint32_t bw, const Bytes& key) {
    if (bw < 1 || bw > 8) fail_decode("hamt: unsupported bit width");
    Bytes raw;
    if (!bs.get(root, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "hamt root not found " + cid_hex(root));
    HamtNode<V> nd = decode_hamt_node<V>(raw);
    uint8_t h[32];
    cpu_crypto::sha256(key.data(), key.size(), h);
    uint32_t consumed = 0;
    for (;;) {
        if (consumed + bw > 256) fail_decode("hamt: max depth");
        uint32_t idx = 0;
        for (uint32_t k = 0; k < bw; k++) { uint32_t bit = consumed + k; idx = (idx << 1) | ((h[bit / 8] >> (7 - bit % 8)) & 1); }
        consumed += bw;
        if (!nd.test(idx)) return std::nullopt;
        auto& p = nd.ptrs[nd.index_for(idx)];
        if (std::holds_alternative<Cid>(p)) {
            Cid c = std::get<Cid>(p);
            Bytes r2;
            if (!bs.get(c, r2)) throw Err(IPCFP_ERR_MISSING_BLOCK, "hamt node not found " + cid_hex(c));
            nd = decode_hamt_node<V>(r2);
            continue;
        }
        for (auto& kv : std::get<std::vector<typename HamtNode<V>::KV>>(p))
            if (kv.key == key) return kv.val;
        return std::nullopt;
    }
}

// ---------------------------------------------------------------------------------- evm.rs
struct EvmLog { std::vector<std::array<uint8_t, 32>> topics; Bytes data; };
// src/proofs/common/evm.rs:13-59
static std::optional<EvmLog> extract_evm_log(const ActorEvent& ev) {
    std::unordered_map<std::string, const Bytes*> m;
    for (auto& e : ev.entries) m[e.key] = &e.value;  // last duplicate wins
    auto it = m.find("topics");
    if (it != m.end()) {
        const Bytes& tb = *it->second;
        if (tb.size() % 32 != 0) return std::nullopt;
        EvmLog log;
        for (size_t o = 0; o < tb.size(); o += 32) { std::array<uint8_t, 32> t; copy_bytes(t.data(), tb.data() + o, 32); log.topics.push_back(t); }
        auto dt = m.find("data");
        if (dt != m.end()) log.data = *dt->second;
        return log;
    }
    EvmLog log;
    static const char* keys[4] = {"t1", "t2", "t3", "t4"};
    for (int i = 0; i < 4; i++) {
        auto k = m.find(keys[i]);
        if (k == m.end()) break;
        if (k->second->size() != 32) return std::nullopt;
        std::array<uint8_t, 32> t;
        copy_bytes(t.data(), k->second->data(), 32);
        log.topics.push_back(t);
    }
    if (log.topics.empty()) return std::nullopt;
    auto dd = m.find("d");
    if (dd != m.end()) log.data = *dd->second;
    return log;
}
static std::array<uint8_t, 32> hash_event_signature(const char* s) {
    std::array<uint8_t, 32> r;
    cpu_crypto::keccak256((const uint8_t*)s, strlen(s), r.data());
    return r;
}
static std::array<uint8_t, 32> ascii_to_bytes32(const char* s) {
    std::array<uint8_t, 32> r{};
    size_t n = std::min<size_t>(strlen(s), 32);
    copy_bytes(r.data(), s, n);
    return r;
}
static std::array<uint8_t, 32> left_pad_32(const Bytes& v) {
    std::array<uint8_t, 32> out{};
    if (v.size() >= 32) { copy_bytes(out.data(), v.data() + v.size() - 32, 32); return out; }
    if (!v.empty()) copy_bytes(out.data() + 32 - v.size(), v.data(), v.size());
    return out;
}
// events/generator.rs:23-41
struct EventMatcher {
    std::array<uint8_t, 32> topic0, topic1;
    EventMatcher(const char* sig, const char* t1) : topic0(hash_event_signature(sig)), topic1(ascii_to_bytes32(t1)) {}
    bool matches_log(const EvmLog& l) const { return l.topics.size() >= 2 && l.topics[0] == topic0 && l.topics[1] == topic1; }
};

// ---------------------------------------------------------------------------------- chain objects (common/decode.rs)
struct HeaderLite { std::vector<Cid> parents; int64_t height; Cid parent_state_root, parent_message_receipts, messages; uint64_t timestamp, fork_signaling; };
static HeaderLite decode_header(const Bytes& raw) {
    Dec d(raw);
    HeaderLite h;
    d.array_exact(16);
    for (int i = 0; i < 5; i++) d.skip_any();
    uint64_t np = d.array();
    if (np > d.n) fail_decode("parents too long");
    for (uint64_t i = 0; i < np; i++) h.parents.push_back(d.cid());
    d.skip_any();
    h.height = d.integer();
    h.parent_state_root = d.cid();
    h.parent_message_receipts = d.cid();
    h.messages = d.cid();
    d.skip_any();
    h.timestamp = d.uint();
    d.skip_any();
    h.fork_signaling = d.uint();
    d.skip_any();
    d.end();
    return h;
}
static std::pair<Cid, Cid> decode_txmeta(const Bytes& raw) {
    Dec d(raw);
    d.array_exact(2);
    Cid a = d.cid(), b = d.cid();
    d.end();
    return {a, b};
}
static Bytes id_address_bytes(uint64_t id) {
    Bytes k;
    k.push_back(0);
    while (id >= 0x80) { k.push_back((uint8_t)(id | 0x80)); id >>= 7; }
    k.push_back((uint8_t)id);
    return k;
}
// common/decode.rs:17-42
static ActorState get_actor_state(const Blockstore& store, const Cid& state_root, uint64_t actor_id) {
    Bytes raw;
    if (!store.get(state_root, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing StateRoot " + cid_hex(state_root));
    Dec d(raw);
    d.array_exact(3);
    uint64_t version = d.uint();
    if (version > 5) fail_decode("unknown state tree version");
    Cid actors = d.cid();
    (void)d.cid();
    d.end();
    auto a = hamt_get<ActorState>(store, actors, 5, id_address_bytes(actor_id));
    if (!a) throw Err(IPCFP_ERR_ACTOR_NOT_FOUND, "actor not found");
    return *a;
}
// common/decode.rs:79-97: contract_state of a 6-field (else 5-field) EVM state
static bool try_evm_state(const Bytes& raw, int fields, Cid& contract_state) {
    try {
        Dec d(raw);
        d.array_exact((uint64_t)fields);
        (void)d.cid();
        Bytes bh = d.bytes();
        if (bh.size() != 32) fail_decode("bytecode hash length");
        contract_state = d.cid();
        if (fields == 6) { if (d.peek_null()) d.null(); else d.skip_any(); }
        (void)d.uint();
        if (d.peek_null()) d.null(); else d.skip_any();
        d.end();
        return true;
    } catch (Err& e) {
        if (e.status != IPCFP_ERR_DECODE) throw;
        return false;
    }
}
static Cid parse_evm_state(const Bytes& raw) {
    Cid cs;
    if (try_evm_state(raw, 6, cs)) return cs;
    if (try_evm_state(raw, 5, cs)) return cs;
    fail_decode("decode EVM state (5-field)");
}

// ---------------------------------------------------------------------------------- storage/decode.rs:36-97
typedef std::vector<std::pair<Bytes, Bytes>> Pairs;
static Pairs dec_small_map(Dec& d) {  // struct SmallMap { v: Vec<(ByteBuf, ByteBuf)> }
    uint64_t n = d.map();
    if (n > d.n) fail_decode("map too long");
    bool have = false;
    Pairs pairs;
    for (uint64_t i = 0; i < n; i++) {
        std::string k = d.text();
        if (k == "v") {
            if (have) fail_decode("duplicate field v");
            have = true;
            uint64_t np = d.array();
            if (np > d.n) fail_decode("pairs too long");
            for (uint64_t j = 0; j < np; j++) { d.array_exact(2); Bytes a = d.bytes(); Bytes b = d.bytes(); pairs.emplace_back(std::move(a), std::move(b)); }
        } else d.skip_any();
    }
    if (!have) fail_decode("missing field v");
    return pairs;
}
template <class F> static bool attempt(F f) {
    try { f(); return true; } catch (Err& e) { if (e.status != IPCFP_ERR_DECODE) throw; return false; }
}
static std::optional<Bytes> read_storage_slot(const Blockstore& store, const Cid& root, const uint8_t slot[32]) {
    Bytes raw;
    if (!store.get(root, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing contract_state root " + cid_hex(root));
    Bytes key(slot, slot + 32);
    auto find = [&](const Pairs& ps) -> std::optional<Bytes> {
        for (auto& kv : ps) if (kv.first == key) return kv.second;
        return std::nullopt;
    };
    {  // A1 [params, [SmallMap]]
        std::vector<Pairs> v;
        if (attempt([&] { Dec d(raw); d.array_exact(2); (void)d.bytes(); uint64_t n = d.array(); if (n > d.n) fail_decode("len"); for (uint64_t i = 0; i < n; i++) v.push_back(dec_small_map(d)); d.end(); }))
            if (!v.empty()) return find(v[0]);
    }
    {  // A2 [params, SmallMap]
        Pairs ps;
        if (attempt([&] { Dec d(raw); d.array_exact(2); (void)d.bytes(); ps = dec_small_map(d); d.end(); })) return find(ps);
    }
    {  // A3 SmallMap
        Pairs ps;
        if (attempt([&] { Dec d(raw); ps = dec_small_map(d); d.end(); })) return find(ps);
    }
    {  // B1 (root, bitwidth)
        Cid r; uint64_t bw = 0;
        if (attempt([&] { Dec d(raw); d.array_exact(2); r = d.cid(); bw = d.uint(); d.end(); })) {
            // `bw as u32` (storage/decode.rs:79,86) truncates to the low 32 bits
            auto v = hamt_get<RawU8Vec>(store, r, (uint32_t)bw, key);
            return v ? std::optional<Bytes>(v->v) : std::nullopt;
        }
    }
    {  // B2 { root, bitwidth }
        Cid r; uint64_t bw = 0;
        if (attempt([&] {
                Dec d(raw);
                uint64_t n = d.map();
                if (n > d.n) fail_decode("map too long");
                bool hr = false, hb = false;
                for (uint64_t i = 0; i < n; i++) {
                    std::string k = d.text();
                    if (k == "root") { if (hr) fail_decode("dup root"); hr = true; r = d.cid(); }
                    else if (k == "bitwidth") { if (hb) fail_decode("dup bitwidth"); hb = true; bw = d.uint(); }
                    else d.skip_any();
                }
                if (!hr || !hb) fail_decode("missing field");
                d.end();
            })) {
            // `bw as u32` (storage/decode.rs:79,86) truncates to the low 32 bits
            auto v = hamt_get<RawU8Vec>(store, r, (uint32_t)bw, key);
            return v ? std::optional<Bytes>(v->v) : std::nullopt;
        }
    }
    // C direct HAMT, HAMT_BIT_WIDTH = 5
    auto v = hamt_get<RawU8Vec>(store, root, 5, key);
    return v ? std::optional<Bytes>(v->v) : std::nullopt;
}

// ---------------------------------------------------------------------------------- events path
struct EventProofRec { uint64_t exec_index, event_index, emitter; std::vector<std::array<uint8_t, 32>> topics; Bytes data; Cid message_cid; };

struct TipsetIn {
    int64_t parent_epoch, child_epoch;
    std::vector<Cid> parent_cids, txmeta;
    Cid child_cid, receipts_root, child_state_root_json;
    uint64_t n_receipts;
    const uint8_t* events_roots;
    const uint8_t* has_root;
};
static TipsetIn tipset_in(const ipcfp_tipset_desc* t) {
    TipsetIn x;
    x.parent_epoch = t->parent_epoch; x.child_epoch = t->child_epoch;
    // a descriptor recovered from a bundle (ipcfp_bundle_from_json) carries only what the verifiers read: no TxMeta CIDs, no receipts root
    for (uint32_t i = 0; i < t->n_parents; i++) {
        x.parent_cids.push_back(cid_from(t->parent_cids + 38 * i));
        if (t->parent_txmeta_cids) x.txmeta.push_back(cid_from(t->parent_txmeta_cids + 38 * i));
    }
    if (t->child_cid) x.child_cid = cid_from(t->child_cid);
    if (t->receipts_root) x.receipts_root = cid_from(t->receipts_root);
    if (t->child_parent_state_root) x.child_state_root_json = cid_from(t->child_parent_state_root);
    x.n_receipts = t->n_receipts; x.events_roots = t->events_roots; x.has_root = t->has_events_root;
    return x;
}

// events/utils.rs:48-94 (verify_txmeta for the offline verifier)
static std::vector<Cid> collect_exec_list(const Blockstore& bs, const std::vector<Cid>& txmeta_cids, bool verify_txmeta) {
    std::vector<Cid> out;
    std::unordered_set<Cid, CidHash> seen;
    for (size_t b = 0; b < txmeta_cids.size(); b++) {
        const Cid& tx = txmeta_cids[b];
        Bytes raw;
        if (!bs.get(tx, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing TxMeta " + cid_hex(tx), b);
        auto roots = decode_txmeta(raw);
        if (verify_txmeta) {
            Bytes enc;
            enc.push_back(0x82);
            for (const Cid* c : {&roots.first, &roots.second}) { const uint8_t h[5] = {0xd8, 0x2a, 0x58, 0x27, 0x00}; enc.insert(enc.end(), h, h + 5); enc.insert(enc.end(), c->b.begin(), c->b.end()); }
            Cid re;
            const uint8_t pre[6] = {0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
            copy_bytes(re.b.data(), pre, 6);
            cpu_crypto::blake2b256(enc.data(), enc.size(), re.b.data() + 6);
            if (re != tx) throw Err(IPCFP_ERR_CID_MISMATCH, "TxMeta mismatch", b);
        }
        for (const Cid* r : {&roots.first, &roots.second}) {
            auto amt = Amt<Cid>::load(*r, bs, 0);
            amt.for_each([&](uint64_t, const Cid& c) { if (seen.insert(c).second) out.push_back(c); });
        }
    }
    return out;
}

struct EventGenOut {
    std::vector<uint64_t> matching;
    std::vector<EventProofRec> proofs;
    std::vector<ProofBlock> blocks;
    uint64_t n_exec = 0;
    double ms_total = 0, ms_pass1 = 0, ms_pass2 = 0, ms_txamt = 0, ms_witness = 0;
    uint64_t pass1_bytes = 0, pass1_nodes = 0;
};
static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// has-any-matching-event over one receipt's events AMT (pass 1 body, events/generator.rs:209-239)
static bool receipt_has_match(const Blockstore& net, const Cid& ev_root, const EventMatcher& m, bool has_filter, uint64_t filter_id) {
    RecordingBlockStore temp(net);  // discarded
    auto amt = Amt<StampedEvent>::load(ev_root, temp, 3);
    bool has = false;
    amt.for_each([&](uint64_t, const StampedEvent& se) {
        if (has_filter && se.emitter != filter_id) return;
        auto log = extract_evm_log(se.event);
        if (log && m.matches_log(*log)) has = true;
    });
    return has;
}

static EventGenOut generate_event_proof(const Blockstore& net, const TipsetIn& ts, const ipcfp_event_spec* spec, uint32_t flags,
                                        uint32_t threads, bool sharded, uint64_t lo, uint64_t hi, uint32_t world, uint32_t rank) {
    EventGenOut out;
    double t0 = now_ms();
    EventMatcher matcher(spec->event_signature, spec->topic_1);
    bool has_filter = spec->has_actor_id_filter != 0;
    uint64_t filter_id = spec->actor_id_filter;
    if (!sharded) { lo = 0; hi = ts.n_receipts; }

    WitnessCollector collector(net);
    std::vector<std::unique_ptr<RecordingBlockStore>> tx_recs;
    const bool skip_tx = (flags & IPCFP_SCAN_SKIP_TX_AMTS) != 0;
    if (!skip_tx) {
        // collect_base_witness (events/generator.rs:122-145)
        for (auto& c : ts.parent_cids) collector.add_cid(c);
        collector.add_cid(ts.child_cid);
        collector.add_cid(ts.receipts_root);
        for (auto& c : ts.txmeta) collector.add_cid(c);
        // record_transaction_amts (:148-177)
        // sharded: a rank records TxMeta, AMT roots and the nodes intersecting its share
        // [Nraw*lo/N, Nraw*hi/N) of the concatenated (raw) message list.
        uint64_t nraw = 0;
        std::vector<uint64_t> bases;
        if (sharded) {
            // geometry of the raw list (start of every AMT in it). An AMT whose TxMeta / root cannot be loaded counts as empty here —
            // the failure itself is raised by the walk below, in the reference's order (same rule as the engine: the first fault,
            // in the order of the sequential walk, among those this shard meets)
            for (size_t b = 0; b < ts.txmeta.size(); b++) {
                std::pair<Cid, Cid> roots;
                bool have = false;
                try {
                    Bytes raw;
                    if (net.get(ts.txmeta[b], raw)) { roots = decode_txmeta(raw); have = true; }
                } catch (Err&) {}
                for (int k = 0; k < 2; k++) {
                    uint64_t cnt = 0;
                    if (have) { try { cnt = Amt<Cid>::load(k ? roots.second : roots.first, net, 0).count; } catch (Err&) {} }
                    bases.push_back(nraw);
                    nraw += cnt;
                }
            }
        }
        size_t ai = 0;
        for (size_t b = 0; b < ts.txmeta.size(); b++) {
            auto rec = std::make_unique<RecordingBlockStore>(net);
            Bytes raw;
            if (!rec->get(ts.txmeta[b], raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing TxMeta " + cid_hex(ts.txmeta[b]), b);
            auto roots = decode_txmeta(raw);
            for (const Cid* r : {&roots.first, &roots.second}) {
                auto amt = Amt<Cid>::load(*r, *rec, 0);
                if (!sharded) amt.for_each([](uint64_t, const Cid&) {});
                else {
                    uint64_t glo = ts.n_receipts ? (uint64_t)((__uint128_t)nraw * lo / ts.n_receipts) : 0, ghi = ts.n_receipts ? (uint64_t)((__uint128_t)nraw * hi / ts.n_receipts) : 0;
                    (void)rank; (void)world;
                    // ownership of a share of the raw list, per AMT (same rule as the engine, DESIGN.md §6): an AMT that ends at or
                    // before the share's start contributes nothing (its right-most nodes may span indices past its count — they
                    // belong to the shard that owns its tail); the shard that reaches an AMT's end owns everything from there on
                    uint64_t base = bases[ai], end = base + amt.count;
                    uint64_t l = glo > base ? glo - base : 0, h = ghi > base ? ghi - base : 0;
                    if (glo >= end && !(end == base && glo == base)) l = h = 0;
                    else if (ghi >= end) h = UINT64_MAX;
                    if (h > l) amt.for_each_range_node(amt.root, amt.height, 0, l, h, [](uint64_t, const Cid&) {});
                }
                ai++;
            }
            tx_recs.push_back(std::move(rec));
        }
        for (auto& r : tx_recs) collector.collect_from_recording(*r);
    }
    // build_execution_order (events/utils.rs:33-45): a second walk on a fresh, un-cached store
    std::vector<Cid> exec = collect_exec_list(net, ts.txmeta, false);
    out.n_exec = exec.size();
    double t1 = now_ms();
    out.ms_txamt = t1 - t0;

    // find_matching_events (events/generator.rs:180-307)
    RecordingBlockStore rec_receipts(net);
    auto r_amt = Amt<Receipt>::load(ts.receipts_root, rec_receipts, 0);

    // PASS 1 (:206-239)
    std::vector<uint64_t>& matching = out.matching;
    auto scan_range = [&](uint64_t a, uint64_t b, std::vector<uint64_t>& dst) {
        for (uint64_t i = a; i < b; i++) {
            if (!ts.has_root[i]) continue;
            Cid ev_root = cid_from(ts.events_roots + 38 * i);
            try {
                if (receipt_has_match(net, ev_root, matcher, has_filter, filter_id)) dst.push_back(i);
            } catch (Err& e) { e.index = i; throw; }
        }
    };
    if (threads <= 1) scan_range(lo, hi, matching);
    else {
        std::vector<std::vector<uint64_t>> parts(threads);
        std::vector<std::unique_ptr<Err>> errs(threads);
        std::vector<std::thread> th;
        for (uint32_t t = 0; t < threads; t++)
            th.emplace_back([&, t]() {
                uint64_t a = lo + (hi - lo) * t / threads, b = lo + (hi - lo) * (t + 1) / threads;
                try { scan_range(a, b, parts[t]); } catch (Err& e) { errs[t] = std::make_unique<Err>(e); }
            });
        for (auto& x : th) x.join();
        for (uint32_t t = 0; t < threads; t++) { if (errs[t]) throw *errs[t]; matching.insert(matching.end(), parts[t].begin(), parts[t].end()); }
    }
    for (uint64_t i = lo; i < hi; i++) if (ts.has_root[i]) out.pass1_nodes++;
    double t2 = now_ms();
    out.ms_pass1 = t2 - t1;

    // PASS 2 (:241-301)
    std::vector<std::unique_ptr<RecordingBlockStore>> event_recs;
    for (uint64_t i : matching) {
        if (i >= exec.size()) throw Err(IPCFP_ERR_MISSING_EXEC, "Missing message at index", i);
        const Cid& msg_cid = exec[i];
        try {
            if (!r_amt.get(i)) continue;
            Cid ev_root = cid_from(ts.events_roots + 38 * i);
            auto rec_events = std::make_unique<RecordingBlockStore>(net);
            auto e_amt = Amt<StampedEvent>::load(ev_root, *rec_events, 3);
            e_amt.for_each([&](uint64_t j, const StampedEvent& se) {
                if (has_filter && se.emitter != filter_id) return;
                auto log = extract_evm_log(se.event);
                if (log && matcher.matches_log(*log)) {
                    EventProofRec p;
                    p.exec_index = i; p.event_index = j; p.emitter = se.emitter;
                    p.topics = log->topics; p.data = log->data; p.message_cid = msg_cid;
                    out.proofs.push_back(std::move(p));
                }
            });
            event_recs.push_back(std::move(rec_events));
        } catch (Err& e) { e.index = i; throw; }
    }
    double t3 = now_ms();
    out.ms_pass2 = t3 - t2;
    for (auto& r : event_recs) collector.collect_from_recording(*r);
    collector.collect_from_recording(rec_receipts);
    out.blocks = collector.materialize();
    double t4 = now_ms();
    out.ms_witness = t4 - t3;
    out.ms_total = t4 - t0;
    return out;
}

// ---------------------------------------------------------------------------------- storage path
struct StorageProofRec { uint64_t actor_id; Cid actor_state_cid, storage_root; std::array<uint8_t, 32> slot, value; bool found; uint32_t raw_len; std::vector<ProofBlock> blocks; };
// storage/generator.rs:29-67
static StorageProofRec generate_storage_proof(const Blockstore& net, const TipsetIn& ts, uint64_t actor_id, const uint8_t slot[32]) {
    // extract_and_verify_parent_state (:72-103)
    RecordingBlockStore header_recorder(net);
    Bytes hdr_raw;
    if (!header_recorder.get(ts.child_cid, hdr_raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing child header");
    HeaderLite hdr = decode_header(hdr_raw);
    if (hdr.parent_state_root != ts.child_state_root_json) throw Err(IPCFP_ERR_STATE_ROOT_MISMATCH, "ParentStateRoot mismatch");
    Cid parent_state_root = hdr.parent_state_root;
    WitnessCollector collector(net);
    collector.add_cid(ts.child_cid);
    collector.add_cid(parent_state_root);
    // load_actor_and_storage_root (:106-134)
    RecordingBlockStore state_recorder(net);
    ActorState actor = get_actor_state(state_recorder, parent_state_root, actor_id);
    Bytes evm_raw;
    if (!state_recorder.get(actor.state, evm_raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing EVM state " + cid_hex(actor.state));
    Cid storage_root = parse_evm_state(evm_raw);
    collector.add_cid(actor.state);
    collector.add_cid(storage_root);
    collector.collect_from_recording(state_recorder);
    // read_storage_value (:137-155)
    RecordingBlockStore storage_recorder(net);
    auto raw = read_storage_slot(storage_recorder, storage_root, slot);
    collector.collect_from_recording(storage_recorder);
    StorageProofRec p;
    p.actor_id = actor_id; p.actor_state_cid = actor.state; p.storage_root = storage_root;
    copy_bytes(p.slot.data(), slot, 32);
    p.found = raw.has_value();
    p.raw_len = raw ? (uint32_t)raw->size() : 0;
    p.value = left_pad_32(raw ? *raw : Bytes());
    p.blocks = collector.materialize();
    return p;
}

// ---------------------------------------------------------------------------------- result packing
struct WitnessBuf { std::vector<uint8_t> cids; std::vector<uint64_t> offsets; std::vector<uint32_t> lengths; std::vector<uint8_t> blob; };
static void pack_witness(const std::vector<ProofBlock>& blocks, WitnessBuf& wb, ipcfp_witness& w) {
    for (auto& b : blocks) {
        wb.cids.insert(wb.cids.end(), b.cid.b.begin(), b.cid.b.end());
        wb.offsets.push_back(wb.blob.size());
        wb.lengths.push_back((uint32_t)b.data.size());
        wb.blob.insert(wb.blob.end(), b.data.begin(), b.data.end());
    }
    w.n_blocks = blocks.size(); w.cids = wb.cids.data(); w.offsets = wb.offsets.data(); w.lengths = wb.lengths.data();
    w.blob = wb.blob.data(); w.blob_size = wb.blob.size();
}
struct EventResultBox {
    ipcfp_event_result r;  // must be first
    std::vector<uint64_t> matching;
    std::vector<ipcfp_event_proof> proofs;
    std::vector<uint8_t> data;
    WitnessBuf wb;
};
static ipcfp_event_result* box_event(EventGenOut& o) {
    auto* b = new EventResultBox();
    b->matching = std::move(o.matching);
    for (auto& p : o.proofs) {
        ipcfp_event_proof q;
        memset(&q, 0, sizeof q);
        q.exec_index = p.exec_index; q.event_index = p.event_index; q.emitter = p.emitter;
        q.n_topics = (uint32_t)p.topics.size();
        q.topics_off = b->data.size();
        for (auto& t : p.topics) b->data.insert(b->data.end(), t.begin(), t.end());
        q.data_off = b->data.size(); q.data_len = (uint32_t)p.data.size();
        b->data.insert(b->data.end(), p.data.begin(), p.data.end());
        copy_bytes(q.message_cid, p.message_cid.b.data(), 38);
        b->proofs.push_back(q);
    }
    memset(&b->r, 0, sizeof b->r);
    b->r.n_matching = b->matching.size(); b->r.matching_indices = b->matching.data();
    b->r.n_proofs = b->proofs.size(); b->r.proofs = b->proofs.data();
    b->r.data_blob = b->data.data(); b->r.data_blob_size = b->data.size();
    pack_witness(o.blocks, b->wb, b->r.witness);
    b->r.n_exec = o.n_exec;
    b->r.ms_total = (float)o.ms_total; b->r.ms_pass1 = (float)o.ms_pass1; b->r.ms_pass2 = (float)o.ms_pass2;
    b->r.ms_txamt = (float)o.ms_txamt; b->r.ms_witness = (float)o.ms_witness;
    b->r.pass1_bytes = o.pass1_bytes; b->r.pass1_nodes = o.pass1_nodes;
    return &b->r;
}
struct StorageResultBox {
    ipcfp_storage_result r;
    std::vector<ipcfp_storage_proof> proofs;
    WitnessBuf wb;
    std::vector<uint64_t> spec_off;
    std::vector<uint32_t> spec_idx;
};
static ipcfp_storage_result* box_storage(std::vector<StorageProofRec>& recs, double ms) {
    auto* b = new StorageResultBox();
    std::map<Cid, Bytes, CidLess> uni;
    for (auto& p : recs) for (auto& blk : p.blocks) uni.emplace(blk.cid, blk.data);
    std::vector<ProofBlock> all;
    std::map<Cid, uint32_t, CidLess> pos;
    for (auto& kv : uni) { pos[kv.first] = (uint32_t)all.size(); all.push_back({kv.first, kv.second}); }
    b->spec_off.push_back(0);
    for (auto& p : recs) {
        ipcfp_storage_proof q;
        memset(&q, 0, sizeof q);
        q.actor_id = p.actor_id;
        copy_bytes(q.actor_state_cid, p.actor_state_cid.b.data(), 38);
        copy_bytes(q.storage_root, p.storage_root.b.data(), 38);
        copy_bytes(q.slot, p.slot.data(), 32); copy_bytes(q.value, p.value.data(), 32);
        q.found = p.found; q.raw_len = p.raw_len;
        b->proofs.push_back(q);
        for (auto& blk : p.blocks) b->spec_idx.push_back(pos[blk.cid]);
        b->spec_off.push_back(b->spec_idx.size());
    }
    memset(&b->r, 0, sizeof b->r);
    b->r.n_proofs = b->proofs.size(); b->r.proofs = b->proofs.data();
    pack_witness(all, b->wb, b->r.witness);
    b->r.spec_witness_offsets = b->spec_off.data(); b->r.spec_witness_index = b->spec_idx.data();
    b->r.ms_total = (float)ms;
    return &b->r;
}
struct SlotResultBox {
    ipcfp_slot_result r;
    std::vector<uint8_t> found, values;
    std::vector<uint32_t> raw_len;
    WitnessBuf wb;
};
struct BundleBox {
    ipcfp_bundle r;
    std::vector<ipcfp_event_result*> ev;
    WitnessBuf wb;
};

static thread_local std::string g_err;
static thread_local uint64_t g_err_index = UINT64_MAX;
template <class F> static ipcfp_status guard(F f) {
    g_err.clear(); g_err_index = UINT64_MAX;
    try { f(); return IPCFP_OK; }
    catch (Err& e) { g_err = e.msg; g_err_index = e.index; return e.status; }
    catch (std::exception& e) { g_err = e.what(); return IPCFP_ERR_INVALID_ARG; }
}

}  // namespace orc

using namespace orc;

struct oracle_store { MemoryBlockstore bs; std::vector<std::pair<const uint8_t*, uint32_t>> order; std::vector<Cid> cids; };

template <class V> static void hamt_node_lookup_t(const Bytes& raw, uint32_t idx, const Bytes& key, int32_t* kind, const std::function<void(const V&)>& on_value,
                                                  const std::function<void(const Cid&)>& on_link) {
    HamtNode<V> nd = decode_hamt_node<V>(raw);
    *kind = 0;
    if (!nd.test(idx)) return;
    auto& p = nd.ptrs[nd.index_for(idx)];
    if (std::holds_alternative<Cid>(p)) { *kind = 2; on_link(std::get<Cid>(p)); return; }
    for (auto& kv : std::get<std::vector<typename HamtNode<V>::KV>>(p))
        if (kv.key == key) { *kind = 1; on_value(kv.val); return; }
}
extern "C" {

oracle_store* oracle_store_create(const uint8_t* cids, const uint64_t* offsets, const uint32_t* lengths, const uint8_t* blob,
                                  uint64_t n) {
    auto* s = new oracle_store();
    s->bs.m.reserve((size_t)n * 2);
    for (uint64_t i = 0; i < n; i++) {
        Cid c = cid_from(cids + 38 * i);
        s->bs.m.emplace(c, std::make_pair(blob + offsets[i], lengths[i]));  // first occurrence wins
        s->order.emplace_back(blob + offsets[i], lengths[i]);
        s->cids.push_back(c);
    }
    return s;
}
void oracle_store_destroy(oracle_store* s) { delete s; }

// TEST HOOK for tests/host_fuzz: the raw message list, see oracle.h
ipcfp_status oracle_message_list(const oracle_store* s, const ipcfp_tipset_desc* t, uint8_t* out38, uint64_t cap, uint64_t* n) {
    try {
        uint64_t k = 0;
        for (uint32_t b = 0; b < t->n_parents; b++) {
            Cid tx = cid_from(t->parent_txmeta_cids + 38 * b);
            Bytes raw;
            if (!s->bs.get(tx, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing TxMeta " + cid_hex(tx), b);
            auto roots = decode_txmeta(raw);
            for (const Cid* r : {&roots.first, &roots.second}) {
                auto amt = Amt<Cid>::load(*r, s->bs, 0);
                amt.for_each([&](uint64_t, const Cid& c) { if (k < cap) copy_bytes(out38 + 38 * k, c.b.data(), 38); k++; });
            }
        }
        *n = k;
        return IPCFP_OK;
    } catch (const Err& e) {
        return e.status;
    }
}

// TEST HOOK for tests/host_fuzz: one HAMT node, see oracle.h
ipcfp_status oracle_hamt_node_lookup(const uint8_t* p, uint64_t n, int vkind, uint32_t idx, const uint8_t* key, uint32_t keylen, int32_t* kind,
                                     uint8_t* out, uint64_t out_cap, uint64_t* out_len) {
    try {
        Bytes raw(p, p + n), k(key, key + keylen);
        *out_len = 0;
        auto put = [&](const uint8_t* q, size_t m) { *out_len = m; copy_bytes(out, q, std::min<size_t>(m, (size_t)out_cap)); };
        auto on_link = [&](const Cid& c) { put(c.b.data(), 38); };
        if (vkind == 0) hamt_node_lookup_t<ActorState>(raw, idx, k, kind, [&](const ActorState& a) { put(a.state.b.data(), 38); }, on_link);
        else hamt_node_lookup_t<RawU8Vec>(raw, idx, k, kind, [&](const RawU8Vec& v) { put(v.v.data(), v.v.size()); }, on_link);
        return IPCFP_OK;
    } catch (const Err& e) {
        return e.status;
    }
}

// TEST HOOK for tests/host_fuzz: one receipts-AMT node, see oracle.h
ipcfp_status oracle_decode_receipts_node(const uint8_t* p, uint64_t n, uint32_t height, uint32_t* n_links, uint32_t* n_vals, uint8_t* has_root,
                                         uint8_t* roots38, uint64_t cap) {
    try {
        Dec d(p, (size_t)n);
        AmtNode<Receipt> nd = decode_amt_node<Receipt>(d, 3, height);
        d.end();
        uint32_t nl = 0, nv = 0;
        for (auto& l : nd.links) if (l) nl++;
        for (auto& v : nd.vals) if (v) {
            if (nv < cap) {
                has_root[nv] = v->events_root ? 1 : 0;
                if (v->events_root) copy_bytes(roots38 + 38 * nv, v->events_root->b.data(), 38);
            }
            nv++;
        }
        *n_links = nl; *n_vals = nv;
        return IPCFP_OK;
    } catch (const Err& e) {
        return e.status;
    }
}

// TEST HOOK for tests/host_fuzz: pass 1 over one events-AMT root block, see oracle.h
ipcfp_status oracle_scan_events_block(const uint8_t* block, uint64_t n, uint64_t* n_events, uint64_t* idx, uint64_t* emitter, uint8_t* some,
                                      uint32_t* ntopics, uint64_t* dlen, uint64_t cap) {
    try {
        MemoryBlockstore bs;
        Cid c;
        memset(c.b.data(), 0, 38);
        static const uint8_t prefix[6] = {0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
        copy_bytes(c.b.data(), prefix, 6);
        bs.m.emplace(c, std::make_pair(block, (uint32_t)n));
        auto amt = Amt<StampedEvent>::load(c, bs, 3);
        uint64_t k = 0;
        amt.for_each([&](uint64_t j, const StampedEvent& se) {
            auto log = extract_evm_log(se.event);
            if (k < cap) {
                idx[k] = j; emitter[k] = se.emitter; some[k] = log ? 1 : 0;
                ntopics[k] = log ? (uint32_t)log->topics.size() : 0;
                dlen[k] = log ? log->data.size() : 0;
            }
            k++;
        });
        *n_events = k;
        return IPCFP_OK;
    } catch (const Err& e) {
        return e.status;
    }
}

// TEST HOOK for tests/host_fuzz: one StampedEvent item + extract_evm_log, see oracle.h
ipcfp_status oracle_decode_event(const uint8_t* p, uint64_t n, uint64_t* consumed, uint64_t* emitter, uint32_t* some, uint32_t* ntopics,
                                 uint8_t* topics_out, uint64_t topics_cap, uint8_t* data_out, uint64_t data_cap, uint64_t* data_len) {
    try {
        Dec d(p, (size_t)n);
        StampedEvent se = ValueDec<StampedEvent>::dec(d);
        *consumed = d.pos;
        *emitter = se.emitter;
        auto log = extract_evm_log(se.event);
        *some = log ? 1 : 0;
        *ntopics = 0;
        *data_len = 0;
        if (log) {
            *ntopics = (uint32_t)log->topics.size();
            for (size_t k = 0; k < log->topics.size() && 32 * (k + 1) <= topics_cap; k++) copy_bytes(topics_out + 32 * k, log->topics[k].data(), 32);
            *data_len = log->data.size();
            copy_bytes(data_out, log->data.data(), std::min<size_t>(log->data.size(), (size_t)data_cap));
        }
        return IPCFP_OK;
    } catch (const Err& e) {
        return e.status;
    }
}
uint64_t oracle_store_verify_cids(const oracle_store* s, uint32_t threads) {
    if (threads < 1) threads = 1;
    std::vector<uint64_t> bad(threads, UINT64_MAX);
    std::vector<std::thread> th;
    size_t n = s->order.size();
    for (uint32_t t = 0; t < threads; t++)
        th.emplace_back([&, t]() {
            for (size_t i = n * t / threads; i < n * (t + 1) / threads; i++) {
                uint8_t d[32];
                cpu_crypto::blake2b256(s->order[i].first, s->order[i].second, d);
                if (memcmp(d, s->cids[i].b.data() + 6, 32) != 0) { bad[t] = i; return; }
            }
        });
    for (auto& x : th) x.join();
    uint64_t r = UINT64_MAX;
    for (auto b : bad) r = std::min(r, b);
    return r;
}
const char* oracle_last_error(void) { return g_err.c_str(); }
uint64_t oracle_last_error_index(void) { return g_err_index; }

ipcfp_status oracle_generate_event_proof(const oracle_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_spec* spec,
                                         uint32_t flags, uint32_t threads, ipcfp_event_result** out) {
    return guard([&] {
        TipsetIn ts = tipset_in(t);
        EventGenOut o = generate_event_proof(s->bs, ts, spec, flags, threads, false, 0, 0, 1, 0);
        *out = box_event(o);
    });
}
ipcfp_status oracle_generate_event_proof_shard(const oracle_store* s, const ipcfp_tipset_desc* t, const ipcfp_event_spec* spec,
                                               uint64_t lo, uint64_t hi, uint32_t world, uint32_t rank, uint32_t flags,
                                               uint32_t threads, ipcfp_event_result** out) {
    return guard([&] {
        TipsetIn ts = tipset_in(t);
        EventGenOut o = generate_event_proof(s->bs, ts, spec, flags, threads, true, lo, hi, world, rank);
        *out = box_event(o);
    });
}
void oracle_event_result_free(ipcfp_event_result* r) { delete reinterpret_cast<EventResultBox*>(r); }

ipcfp_status oracle_read_storage_slots(const oracle_store* s, const uint8_t root[38], const uint8_t* slots, uint64_t k,
                                       ipcfp_slot_result** out) {
    return guard([&] {
        double t0 = now_ms();
        auto* b = new SlotResultBox();
        std::unique_ptr<SlotResultBox> hold(b);
        Cid rc = cid_from(root);
        RecordingBlockStore rec(s->bs);
        b->found.resize(k); b->raw_len.resize(k); b->values.assign(k * 32, 0);
        for (uint64_t i = 0; i < k; i++) {
            try {
                auto v = read_storage_slot(rec, rc, slots + 32 * i);
                b->found[i] = v.has_value();
                b->raw_len[i] = v ? (uint32_t)v->size() : 0;
                auto pv = left_pad_32(v ? *v : Bytes());
                copy_bytes(&b->values[32 * i], pv.data(), 32);
            } catch (Err& e) { e.index = i; throw; }
        }
        WitnessCollector col(s->bs);
        col.collect_from_recording(rec);
        auto blocks = col.materialize();
        memset(&b->r, 0, sizeof b->r);
        b->r.n = k; b->r.found = b->found.data(); b->r.raw_len = b->raw_len.data(); b->r.values = b->values.data();
        pack_witness(blocks, b->wb, b->r.witness);
        b->r.ms_total = (float)(now_ms() - t0);
        *out = &hold.release()->r;
    });
}
void oracle_slot_result_free(ipcfp_slot_result* r) { delete reinterpret_cast<SlotResultBox*>(r); }

ipcfp_status oracle_generate_storage_proofs(const oracle_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* specs,
                                            uint64_t n, ipcfp_storage_result** out) {
    return guard([&] {
        double t0 = now_ms();
        TipsetIn ts = tipset_in(t);
        std::vector<StorageProofRec> recs;
        for (uint64_t i = 0; i < n; i++) {
            try { recs.push_back(generate_storage_proof(s->bs, ts, specs[i].actor_id, specs[i].slot)); }
            catch (Err& e) { e.index = i; throw; }
        }
        *out = box_storage(recs, now_ms() - t0);
    });
}
void oracle_storage_result_free(ipcfp_storage_result* r) { delete reinterpret_cast<StorageResultBox*>(r); }

ipcfp_status oracle_generate_proof_bundle(const oracle_store* s, const ipcfp_tipset_desc* t, const ipcfp_storage_spec* ss,
                                          uint64_t ns, const ipcfp_event_spec* es, uint64_t ne, ipcfp_bundle** out) {
    return guard([&] {
        auto* b = new BundleBox();
        std::unique_ptr<BundleBox> hold(b);
        memset(&b->r, 0, sizeof b->r);
        // proofs/generator.rs:34: BTreeSet<(Cid, Vec<u8>)>
        struct KeyLess { bool operator()(const std::pair<Cid, Bytes>& a, const std::pair<Cid, Bytes>& b) const { if (a.first != b.first) return cid_less(a.first, b.first); return a.second < b.second; } };
        std::set<std::pair<Cid, Bytes>, KeyLess> all;
        TipsetIn ts = tipset_in(t);
        if (ns) {
            std::vector<StorageProofRec> recs;
            for (uint64_t i = 0; i < ns; i++) {
                try { recs.push_back(generate_storage_proof(s->bs, ts, ss[i].actor_id, ss[i].slot)); } catch (Err& e) { e.index = i; throw; }
                for (auto& blk : recs.back().blocks) all.emplace(blk.cid, blk.data);
            }
            b->r.storage = box_storage(recs, 0);
        }
        for (uint64_t i = 0; i < ne; i++) {
            EventGenOut o = generate_event_proof(s->bs, ts, &es[i], 0, 1, false, 0, 0, 1, 0);
            for (auto& blk : o.blocks) all.emplace(blk.cid, blk.data);
            b->ev.push_back(box_event(o));
        }
        b->r.n_event_results = b->ev.size(); b->r.events = b->ev.data();
        std::vector<ProofBlock> blocks;
        for (auto& kv : all) blocks.push_back({kv.first, kv.second});
        pack_witness(blocks, b->wb, b->r.witness);
        *out = &hold.release()->r;
    });
}
void oracle_bundle_free(ipcfp_bundle* r) {
    auto* b = reinterpret_cast<BundleBox*>(r);
    if (b->r.storage) oracle_storage_result_free(b->r.storage);
    for (auto* e : b->ev) oracle_event_result_free(e);
    delete b;
}

// ---------------------------------------------------------------------------------- verifiers
static void load_witness_store(const ipcfp_witness* w, MemoryBlockstore& bs) {  // events/verifier.rs:79-89 (no hash check)
    for (uint64_t i = 0; i < w->n_blocks; i++) bs.put_keyed(cid_from(w->cids + 38 * i), w->blob + w->offsets[i], w->lengths[i]);
}
ipcfp_status oracle_verify_event_proofs(const ipcfp_witness* w, const ipcfp_tipset_desc* t, const ipcfp_event_proof* proofs,
                                        uint64_t n_proofs, const uint8_t* data_blob, const ipcfp_event_spec* filter_spec,
                                        uint8_t* results) {
    return guard([&] {
        MemoryBlockstore bs;
        bs.owned.reserve(w->n_blocks);
        load_witness_store(w, bs);
        TipsetIn ts = tipset_in(t);
        std::unique_ptr<EventMatcher> filt;
        if (filter_spec) filt = std::make_unique<EventMatcher>(filter_spec->event_signature, filter_spec->topic_1);
        for (uint64_t pi = 0; pi < n_proofs; pi++) {
            const ipcfp_event_proof& p = proofs[pi];
            results[pi] = 0;
            // verify_header_consistency (:147-181)
            Bytes child_raw;
            if (!bs.get(ts.child_cid, child_raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing child header in witness", pi);
            HeaderLite child = decode_header(child_raw);
            if (child.parents != ts.parent_cids) continue;
            if (child.height != ts.child_epoch) continue;
            Bytes ph_raw;
            if (!bs.get(ts.parent_cids[0], ph_raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing parent header in witness", pi);
            HeaderLite ph = decode_header(ph_raw);
            if (ph.height != ts.parent_epoch) continue;
            // verify_execution_order (:184-204) via reconstruct_execution_order (utils.rs:16-30)
            std::vector<Cid> txm;
            for (auto& pc : ts.parent_cids) {
                Bytes raw;
                if (!bs.get(pc, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing parent header", pi);
                txm.push_back(decode_header(raw).messages);
            }
            std::vector<Cid> exec = collect_exec_list(bs, txm, true);
            Cid msg = cid_from(p.message_cid);
            auto it = std::find(exec.begin(), exec.end(), msg);
            if (it == exec.end()) continue;
            if ((uint64_t)(it - exec.begin()) != p.exec_index) continue;
            // verify_receipt_and_event (:207-254)
            auto r_amt = Amt<Receipt>::load(child.parent_message_receipts, bs, 0);
            auto rc = r_amt.get(p.exec_index);
            if (!rc) continue;
            if (!rc->events_root) continue;
            auto e_amt = Amt<StampedEvent>::load(*rc->events_root, bs, 3);
            auto se = e_amt.get(p.event_index);
            if (!se) continue;
            // verify_event_data_matches (:257-290)
            if (se->emitter != p.emitter) continue;
            auto log = extract_evm_log(se->event);
            if (!log) continue;
            if (log->topics.size() != p.n_topics) continue;
            bool ok = true;
            for (uint32_t k = 0; k < p.n_topics; k++) if (memcmp(log->topics[k].data(), data_blob + p.topics_off + 32 * k, 32) != 0) ok = false;
            if (!ok) continue;
            if (log->data.size() != p.data_len || (p.data_len && memcmp(log->data.data(), data_blob + p.data_off, p.data_len) != 0)) continue;
            if (filt) { if (!filt->matches_log(*log)) continue; }
            results[pi] = 1;
        }
    });
}
ipcfp_status oracle_verify_storage_proofs(const ipcfp_witness* w, const ipcfp_tipset_desc* t, const ipcfp_storage_proof* proofs,
                                          uint64_t n, uint8_t* results) {
    return guard([&] {
        MemoryBlockstore bs;
        bs.owned.reserve(w->n_blocks);
        load_witness_store(w, bs);
        TipsetIn ts = tipset_in(t);
        for (uint64_t i = 0; i < n; i++) {
            const ipcfp_storage_proof& p = proofs[i];
            results[i] = 0;
            Bytes hdr;
            if (!bs.get(ts.child_cid, hdr)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing child header in witness", i);
            Cid psr = decode_header(hdr).parent_state_root;  // storage/verifier.rs:98-114
            if (psr != ts.child_state_root_json) continue;
            ActorState a = get_actor_state(bs, psr, p.actor_id);  // :117-132
            if (a.state != cid_from(p.actor_state_cid)) continue;
            Bytes evm;
            if (!bs.get(a.state, evm)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing EVM state in witness", i);
            Cid sroot = parse_evm_state(evm);  // :135-150
            if (sroot != cid_from(p.storage_root)) continue;
            auto raw = read_storage_slot(bs, sroot, p.slot);  // :153-170
            auto v = left_pad_32(raw ? *raw : Bytes());
            if (memcmp(v.data(), p.value, 32) != 0) continue;
            results[i] = 1;
        }
    });
}

void oracle_keccak256(const uint8_t* in, uint64_t len, uint8_t out[32]) { cpu_crypto::keccak256(in, (size_t)len, out); }
void oracle_blake2b256(const uint8_t* in, uint64_t len, uint8_t out[32]) { cpu_crypto::blake2b256(in, (size_t)len, out); }
void oracle_sha256(const uint8_t* in, uint64_t len, uint8_t out[32]) { cpu_crypto::sha256(in, (size_t)len, out); }
void oracle_compute_mapping_slot(const uint8_t key32[32], uint64_t slot_index, uint8_t out[32]) {  // storage/utils.rs:5-12
    uint8_t buf[64];
    copy_bytes(buf, key32, 32);
    memset(buf + 32, 0, 24);
    for (int i = 0; i < 8; i++) buf[56 + i] = (uint8_t)(slot_index >> (56 - 8 * i));
    cpu_crypto::keccak256(buf, 64, out);
}
uint64_t oracle_sort_unique_cids(uint8_t* cids, uint64_t n) {
    std::set<Cid, CidLess> s;
    for (uint64_t i = 0; i < n; i++) s.insert(cid_from(cids + 38 * i));
    uint64_t k = 0;
    for (auto& c : s) { copy_bytes(cids + 38 * k, c.b.data(), 38); k++; }
    return k;
}

}  // extern "C"
