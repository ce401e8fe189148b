// Synthetic Filecoin tipset builder (see synth.h). CPU-only test/bench infrastructure.
//
// Wire formats: SURVEY.md Appendix A ([UPSTREAM] crates restated from their published
// formats): CID v1 dag-cbor blake2b-256 (38 B), DAG-CBOR with minimal heads, AMT v0/v3
// nodes [bmap, links, values], HAMT v3 nodes [bitfield, pointers], Receipt 4-tuple,
// StampedEvent [emitter, [[flags,key,codec,value]...]], TxMeta [bls,secp],
// 16-field block header, StateRoot [version, actors, info], ActorState 5-tuple,
// EVM state 6-/5-tuple.
#include "synth.h"
#include "cpu_crypto.h"

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <vector>

namespace {

typedef std::vector<uint8_t> Bytes;

struct Rng {
    uint64_t s;
    uint64_t next() {
        s += 0x9E3779B97F4A7C15ULL;
        uint64_t z = s;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
        return z ^ (z >> 31);
    }
};
enum { DOM_RECEIPT = 1, DOM_MSG = 2, DOM_STORAGE = 3, DOM_ACTOR = 4, DOM_HDR = 5 };
static Rng rng_for(uint64_t seed, uint64_t dom, uint64_t idx) {
    Rng r{seed ^ (dom * 0xA0761D6478BD642FULL) ^ (idx * 0xE7037ED1A0B428DBULL)};
    r.next();
    return r;
}

// ------------------------------------------------------------------ CBOR writer
static void cb_head(Bytes& o, int major, uint64_t v) {
    uint8_t m = (uint8_t)(major << 5);
    if (v < 24) o.push_back(m | (uint8_t)v);
    else if (v <= 0xff) { o.push_back(m | 24); o.push_back((uint8_t)v); }
    else if (v <= 0xffff) { o.push_back(m | 25); o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); }
    else if (v <= 0xffffffffULL) { o.push_back(m | 26); for (int i = 3; i >= 0; i--) o.push_back((uint8_t)(v >> (8 * i))); }
    else { o.push_back(m | 27); for (int i = 7; i >= 0; i--) o.push_back((uint8_t)(v >> (8 * i))); }
}
static void cb_uint(Bytes& o, uint64_t v) { cb_head(o, 0, v); }
static void cb_bytes(Bytes& o, const uint8_t* p, size_t n) { cb_head(o, 2, n); o.insert(o.end(), p, p + n); }
static void cb_text(Bytes& o, const char* s) { size_t n = strlen(s); cb_head(o, 3, n); o.insert(o.end(), s, s + n); }
static void cb_array(Bytes& o, uint64_t n) { cb_head(o, 4, n); }
static void cb_map(Bytes& o, uint64_t n) { cb_head(o, 5, n); }
static void cb_null(Bytes& o) { o.push_back(0xf6); }
static void cb_cid(Bytes& o, const uint8_t cid[38]) {
    o.push_back(0xd8); o.push_back(0x2a); o.push_back(0x58); o.push_back(0x27); o.push_back(0x00);
    o.insert(o.end(), cid, cid + 38);
}

struct Cid { uint8_t b[38]; };
static const uint8_t CID_PREFIX[6] = {0x01, 0x71, 0xa0, 0xe4, 0x02, 0x20};
static Cid cid_of(const uint8_t* data, size_t len) {
    Cid c;
    memcpy(c.b, CID_PREFIX, 6);
    cpu_crypto::blake2b256(data, len, c.b + 6);
    return c;
}
static Cid fake_cid(const char* tag, uint64_t n, uint64_t seed) {
    char buf[96];
    int k = snprintf(buf, sizeof buf, "fake:%s:%llu:%llu", tag, (unsigned long long)n, (unsigned long long)seed);
    return cid_of((const uint8_t*)buf, (size_t)k);
}

// ------------------------------------------------------------------ block set
struct BlockSet {
    std::vector<uint8_t> cids;
    std::vector<uint64_t> offs;
    std::vector<uint32_t> lens;
    std::vector<uint8_t> blob;
    Cid add(const Bytes& b) {
        Cid c = cid_of(b.data(), b.size());
        add_with_cid(c, b.data(), b.size());
        return c;
    }
    void add_with_cid(const Cid& c, const uint8_t* p, size_t n) {
        cids.insert(cids.end(), c.b, c.b + 38);
        offs.push_back(blob.size());
        lens.push_back((uint32_t)n);
        blob.insert(blob.end(), p, p + n);
        size_t pad = (16 - (blob.size() & 15)) & 15;
        blob.insert(blob.end(), pad, 0);
    }
    void append(const BlockSet& o) {
        uint64_t base = blob.size();
        cids.insert(cids.end(), o.cids.begin(), o.cids.end());
        for (uint64_t x : o.offs) offs.push_back(base + x);
        lens.insert(lens.end(), o.lens.begin(), o.lens.end());
        blob.insert(blob.end(), o.blob.begin(), o.blob.end());
    }
    size_t n() const { return lens.size(); }
};

// ------------------------------------------------------------------ constants
static const char* TARGET_SIG = "NewTopDownMessage(bytes32,uint256)";
static const char* TARGET_TOPIC1 = "calib-subnet-1";
static const int TARGET_TOPIC1_IDX = 1;

struct Topics {
    uint8_t t0[8][32];   // [0] = target signature hash, [1..7] = other signatures
    uint8_t t1[16][32];  // "calib-subnet-<k>" right padded
};
static Topics make_topics() {
    Topics t;
    cpu_crypto::keccak256((const uint8_t*)TARGET_SIG, strlen(TARGET_SIG), t.t0[0]);
    for (int k = 1; k < 8; k++) {
        char buf[64];
        int n = snprintf(buf, sizeof buf, "Other%d(bytes32,uint256)", k);
        cpu_crypto::keccak256((const uint8_t*)buf, (size_t)n, t.t0[k]);
    }
    for (int k = 0; k < 16; k++) {
        char buf[64];
        int n = snprintf(buf, sizeof buf, "calib-subnet-%d", k);
        memset(t.t1[k], 0, 32);
        memcpy(t.t1[k], buf, (size_t)std::min(n, 32));
    }
    return t;
}

static void be64(uint8_t* p, uint64_t v) { for (int i = 0; i < 8; i++) p[i] = (uint8_t)(v >> (56 - 8 * i)); }

// ------------------------------------------------------------------ events AMT of one receipt
struct ReceiptInfo { bool has_root; bool selected; uint32_t gas; };

// Writes the events-AMT blocks of receipt i into `out` (one root block when E <= width,
// otherwise root + interior/leaf nodes) and returns the root CID.
struct AmtSink {
    BlockSet* keep;  // may be null: hash only
};

static void amt_node_head(Bytes& o, int bw, uint32_t nchild) {
    cb_array(o, 3);
    int nb = bw <= 3 ? 1 : (1 << (bw - 3));
    uint8_t bm[512];
    memset(bm, 0, (size_t)nb);
    for (uint32_t i = 0; i < nchild; i++) bm[i / 8] |= (uint8_t)(1u << (i % 8));
    cb_bytes(o, bm, (size_t)nb);
}

// Dense AMT builder. value_fn(i, out) appends the DAG-CBOR of value i.
// keep_fn(level, node_index) decides whether a non-root node block is materialised.
// version: 0 → root [height,count,node] (bw must be 3); 3 → root [bw,height,count,node].
static Cid build_amt(uint64_t count, int bw, int version, const std::function<void(uint64_t, Bytes&)>& value_fn,
                     const std::function<bool(int, uint64_t)>& keep_fn, BlockSet* out, unsigned threads) {
    const uint64_t W = 1ull << bw;
    std::vector<Cid> cur;
    Bytes top;  // encoding of the top node (inlined into the root)
    int height = 0;
    uint64_t n0 = (count + W - 1) / W;
    if (n0 <= 1) {
        amt_node_head(top, bw, (uint32_t)count);
        cb_array(top, 0);
        cb_array(top, count);
        for (uint64_t i = 0; i < count; i++) value_fn(i, top);
    } else {
        cur.resize(n0);
        unsigned T = std::max(1u, std::min<unsigned>(threads, (unsigned)std::max<uint64_t>(1, n0 / 1024)));
        std::vector<BlockSet> tl(T);
        std::vector<std::thread> th;
        for (unsigned t = 0; t < T; t++) {
            th.emplace_back([&, t]() {
                uint64_t lo = n0 * t / T, hi = n0 * (t + 1) / T;
                Bytes nb;
                for (uint64_t k = lo; k < hi; k++) {
                    nb.clear();
                    uint64_t a = k * W, b = std::min(count, a + W);
                    amt_node_head(nb, bw, (uint32_t)(b - a));
                    cb_array(nb, 0);
                    cb_array(nb, b - a);
                    for (uint64_t i = a; i < b; i++) value_fn(i, nb);
                    Cid c = cid_of(nb.data(), nb.size());
                    cur[k] = c;
                    if (out && keep_fn(0, k)) tl[t].add_with_cid(c, nb.data(), nb.size());
                }
            });
        }
        for (auto& x : th) x.join();
        if (out) for (auto& b : tl) out->append(b);
        // interior levels
        for (;;) {
            height++;
            uint64_t n = (cur.size() + W - 1) / W;
            if (n == 1) {
                amt_node_head(top, bw, (uint32_t)cur.size());
                cb_array(top, cur.size());
                for (auto& c : cur) cb_cid(top, c.b);
                cb_array(top, 0);
                break;
            }
            std::vector<Cid> nxt(n);
            Bytes nb;
            for (uint64_t k = 0; k < n; k++) {
                nb.clear();
                uint64_t a = k * W, b = std::min<uint64_t>(cur.size(), a + W);
                amt_node_head(nb, bw, (uint32_t)(b - a));
                cb_array(nb, b - a);
                for (uint64_t i = a; i < b; i++) cb_cid(nb, cur[i].b);
                cb_array(nb, 0);
                Cid c = cid_of(nb.data(), nb.size());
                nxt[k] = c;
                if (out && keep_fn(height, k)) out->add_with_cid(c, nb.data(), nb.size());
            }
            cur.swap(nxt);
        }
    }
    Bytes root;
    if (version == 0) { cb_array(root, 3); }
    else { cb_array(root, 4); cb_uint(root, (uint64_t)bw); }
    cb_uint(root, (uint64_t)height);
    cb_uint(root, count);
    root.insert(root.end(), top.begin(), top.end());
    Cid rc = cid_of(root.data(), root.size());
    if (out) out->add_with_cid(rc, root.data(), root.size());
    return rc;
}

struct Gen {
    synth_params p;
    Topics tp;
    uint64_t target_actor;
};

static void gen_event(const Gen& g, Rng& r, uint64_t i, uint32_t j, bool forced, Bytes& o) {
    uint64_t em = 1000 + r.next() % 16;
    uint32_t t0sel = (uint32_t)(r.next() % 8);
    uint32_t t1sel = (uint32_t)(r.next() % 16);
    bool case_a = (r.next() % 1000) < g.p.case_a_permille;
    bool mal = (r.next() % 1000) < g.p.malformed_permille;
    uint64_t dword = r.next();
    if (g.p.same_topic1) t1sel = TARGET_TOPIC1_IDX;
    if (case_a) mal = false;
    if (forced) {
        if (g.p.has_actor_filter) em = g.target_actor;
        t0sel = 0; t1sel = TARGET_TOPIC1_IDX; mal = false;
    } else if (!mal && t0sel == 0 && t1sel == TARGET_TOPIC1_IDX && (!g.p.has_actor_filter || em == g.target_actor)) {
        // would be an accidental full match: deflect
        if (g.p.same_topic1) t0sel = 1 + (uint32_t)(dword % 7);
        else t1sel = 2;
    }
    uint8_t d[32];
    be64(d, dword); be64(d + 8, i); be64(d + 16, j); be64(d + 24, ~dword);
    cb_array(o, 2);
    cb_uint(o, em);
    if (case_a) {
        cb_array(o, 2);
        uint8_t tt[64];
        memcpy(tt, g.tp.t0[t0sel], 32); memcpy(tt + 32, g.tp.t1[t1sel], 32);
        cb_array(o, 4); cb_uint(o, 3); cb_text(o, "topics"); cb_uint(o, 0x55); cb_bytes(o, tt, 64);
        cb_array(o, 4); cb_uint(o, 3); cb_text(o, "data"); cb_uint(o, 0x55); cb_bytes(o, d, 32);
    } else {
        cb_array(o, 3);
        cb_array(o, 4); cb_uint(o, 3); cb_text(o, "t1"); cb_uint(o, 0x55); cb_bytes(o, g.tp.t0[t0sel], 32);
        cb_array(o, 4); cb_uint(o, 3); cb_text(o, "t2"); cb_uint(o, 0x55); cb_bytes(o, g.tp.t1[t1sel], mal ? 31 : 32);
        cb_array(o, 4); cb_uint(o, 3); cb_text(o, "d"); cb_uint(o, 0x55); cb_bytes(o, d, 32);
    }
}

// ------------------------------------------------------------------ varied event shapes (event_shapes = 1)
// One [flags, key, codec, value] entry of a StampedEvent.
struct Entry { uint64_t flags; const char* key; uint64_t codec; Bytes val; };

static Bytes rand_bytes(Rng& r, size_t n) {
    Bytes b(n);
    for (size_t k = 0; k < n; k++) b[k] = (uint8_t)r.next();
    return b;
}
static Bytes bytes_of(const uint8_t* p, size_t n) { return Bytes(p, p + n); }

// The spec's predicate on one event, restated from the reference: the emitter filter, then extract_evm_log (the last of duplicate
// keys wins; `topics` selects Case A and must be a multiple of 32 bytes; Case B takes t1, t2, ... while present, each exactly
// 32 bytes), then topic 0 == the signature hash and topic 1 == the padded topic1.
static bool shaped_event_matches(const Gen& g, uint64_t em, const std::vector<Entry>& es) {
    if (g.p.has_actor_filter && em != g.target_actor) return false;
    const uint8_t* T0 = g.tp.t0[0];
    const uint8_t* T1 = g.tp.t1[TARGET_TOPIC1_IDX];
    static const char* tk[4] = {"t1", "t2", "t3", "t4"};
    const Bytes* t[4] = {nullptr, nullptr, nullptr, nullptr};
    const Bytes* topics = nullptr;
    for (const Entry& e : es) {
        if (!strcmp(e.key, "topics")) topics = &e.val;
        for (int k = 0; k < 4; k++) if (!strcmp(e.key, tk[k])) t[k] = &e.val;
    }
    if (topics) return topics->size() % 32 == 0 && topics->size() >= 64 && !memcmp(topics->data(), T0, 32) && !memcmp(topics->data() + 32, T1, 32);
    int lead = 0;
    while (lead < 4 && t[lead]) {
        if (t[lead]->size() != 32) return false;
        lead++;
    }
    return lead >= 2 && !memcmp(t[0]->data(), T0, 32) && !memcmp(t[1]->data(), T1, 32);
}

// One event of the varied distribution. A forced event is an unambiguous match; every other event fails the spec, either as one
// of the named near misses (wrong emitter under the filter, a 31-byte t2, swapped topics, the target topics only at t3/t4, Case A
// with one topic) or as a random shape that is deflected (its effective topic 0 replaced) should it match by accident.
static void gen_event_shaped(const Gen& g, Rng& r, bool forced, Bytes& o) {
    const uint8_t* T0 = g.tp.t0[0];
    const uint8_t* T1 = g.tp.t1[TARGET_TOPIC1_IDX];
    const uint64_t ta = g.target_actor;
    // immediate, 1-, 2-, 4- and 8-byte CBOR heads
    const uint64_t emitters[8] = {5, 23, 24, 255, 1000 + r.next() % 16, 65536 + ta, (1ull << 40) + ta, ta};
    uint64_t em = emitters[r.next() % 8];
    auto topic = [&]() -> Bytes {   // a 32-byte topic from the pool the tipset's topics come from
        uint64_t k = r.next() % 24;
        return k < 8 ? bytes_of(g.tp.t0[k], 32) : bytes_of(g.tp.t1[k - 8], 32);
    };
    auto data_b = [&]() -> Bytes { return rand_bytes(r, r.next() % 3 == 0 ? 256 + r.next() % 700 : r.next() % 64); };
    std::vector<Entry> es;
    auto add = [&](const char* key, Bytes v) { es.push_back(Entry{3, key, 0x55, std::move(v)}); };
    static const char* tk[4] = {"t1", "t2", "t3", "t4"};
    if (forced) {
        if (g.p.has_actor_filter) em = ta;
        if (r.next() % 3 == 0) {
            Bytes tp = bytes_of(T0, 32);
            tp.insert(tp.end(), T1, T1 + 32);
            for (uint64_t k = r.next() % 3; k > 0; k--) { Bytes x = topic(); tp.insert(tp.end(), x.begin(), x.end()); }
            add("topics", tp);
            add("data", rand_bytes(r, r.next() % 300));
        } else {
            add("t1", bytes_of(T0, 32));
            add("t2", bytes_of(T1, 32));
            for (uint64_t k = 2, nt = 2 + r.next() % 3; k < nt; k++) add(tk[k], topic());
            if (r.next() % 4) add("d", data_b());
        }
    } else {
        unsigned kind = (unsigned)(r.next() % 16);
        if (kind == 8) {                                   // wrong emitter (a miss only under the filter; deflected otherwise)
            if (g.p.has_actor_filter && em == ta) em = ta + 1;
            add("t1", bytes_of(T0, 32)); add("t2", bytes_of(T1, 32)); add("d", data_b());
        } else if (kind == 9) {                            // 31-byte t2
            add("t1", bytes_of(T0, 32)); add("t2", bytes_of(T1, 31)); add("d", data_b());
        } else if (kind == 10) {                           // swapped topics
            add("t1", bytes_of(T1, 32)); add("t2", bytes_of(T0, 32)); add("d", data_b());
        } else if (kind == 11) {                           // the target topics only at t3 / t4
            add("t1", topic()); add("t2", topic()); add("t3", bytes_of(T0, 32)); add("t4", bytes_of(T1, 32));
        } else if (kind == 12) {                           // Case A with one topic
            add("topics", bytes_of(T0, 32)); add("data", rand_bytes(r, r.next() % 300));
        } else if (kind < 4) {                             // Case A, 0..4 topics
            Bytes tp;
            for (uint64_t k = r.next() % 5; k > 0; k--) { Bytes x = topic(); tp.insert(tp.end(), x.begin(), x.end()); }
            add("topics", tp);
            add("data", rand_bytes(r, r.next() % 300));
        } else {                                           // Case B, 1..4 topics (now and then of another length), optional d
            for (uint64_t k = 0, nt = 1 + r.next() % 4; k < nt; k++) add(tk[k], r.next() % 16 == 0 ? rand_bytes(r, r.next() % 40) : topic());
            if (r.next() % 4) add("d", data_b());
        }
    }
    // odd flags and codecs (the reference reads neither)
    static const uint64_t odd[8] = {0, 1, 7, 23, 24, 255, 300, 70000};
    for (Entry& e : es) {
        if (r.next() % 8 == 0) e.flags = odd[r.next() % 8];
        if (r.next() % 8 == 0) e.codec = odd[r.next() % 8];
    }
    // an unknown key; a duplicate placed before the entry it repeats (the later one wins, so the event's meaning is kept)
    static const char* unknown[6] = {"topic", "dat", "t5", "t0", "D", "tt1"};
    if (r.next() % 8 == 0) {
        size_t at = (size_t)(r.next() % (es.size() + 1));
        es.insert(es.begin() + (long)at, Entry{3, unknown[r.next() % 6], 0x55, rand_bytes(r, r.next() % 40)});
    }
    if (!es.empty() && r.next() % 8 == 0) {
        size_t at = (size_t)(r.next() % es.size());
        Entry dup{es[at].flags, es[at].key, es[at].codec, rand_bytes(r, r.next() % 2 ? 32 : r.next() % 40)};
        es.insert(es.begin() + (long)at, dup);
    }
    if (forced != shaped_event_matches(g, em, es)) {
        if (forced) { fprintf(stderr, "synth: a forced event does not match\n"); abort(); }
        // the effective topic 0 (of the last `topics`, else the last `t1`) becomes another signature
        bool has_topics = false;
        for (const Entry& e : es) has_topics |= !strcmp(e.key, "topics");
        for (size_t k = es.size(); k-- > 0;)
            if (!strcmp(es[k].key, has_topics ? "topics" : "t1")) { memcpy(es[k].val.data(), g.tp.t0[1], 32); break; }
    }
    cb_array(o, 2);
    cb_uint(o, em);
    cb_array(o, es.size());
    for (const Entry& e : es) {
        cb_array(o, 4);
        cb_uint(o, e.flags);
        cb_text(o, e.key);
        cb_uint(o, e.codec);
        cb_bytes(o, e.val.data(), e.val.size());
    }
}

// Receipt i of the varied mode: 0..events_per_receipt events (at least one when selected).
static ReceiptInfo gen_receipt_shaped(const Gen& g, uint64_t i, BlockSet* out, Cid* root) {
    Rng r = rng_for(g.p.seed, DOM_RECEIPT, i);
    ReceiptInfo ri;
    bool sel = (r.next() % 1000000) < g.p.match_ppm;
    int bw = (r.next() % 1000) < g.p.bw3_permille ? 3 : 5;
    bool null_root = (r.next() % 1000) < g.p.null_root_permille;
    ri.gas = (uint32_t)r.next();
    const uint32_t E = g.p.events_per_receipt;
    uint32_t n = E ? (uint32_t)(r.next() % (E + 1)) : 0;
    if (sel && n == 0) n = 1;
    ri.has_root = !null_root && E > 0;
    ri.selected = sel && ri.has_root;
    if (!ri.has_root) { memset(root->b, 0, 38); return ri; }
    uint32_t sel_pos = n ? (uint32_t)(r.next() % n) : 0;
    std::vector<Bytes> evs(n);
    for (uint32_t j = 0; j < n; j++) gen_event_shaped(g, r, sel && j == sel_pos, evs[j]);
    auto vf = [&](uint64_t k, Bytes& o) { o.insert(o.end(), evs[k].begin(), evs[k].end()); };
    auto kf = [](int, uint64_t) { return true; };
    *root = build_amt(n, bw, 3, vf, kf, out, 1);
    return ri;
}

// Generates receipt i: its events AMT blocks (into `out` when non-null) and root CID.
static ReceiptInfo gen_receipt(const Gen& g, uint64_t i, BlockSet* out, Cid* root) {
    if (g.p.event_shapes == 1) return gen_receipt_shaped(g, i, out, root);
    Rng r = rng_for(g.p.seed, DOM_RECEIPT, i);
    ReceiptInfo ri;
    bool sel = (r.next() % 1000000) < g.p.match_ppm;
    uint32_t E = g.p.events_per_receipt;
    uint32_t sel_pos = E ? (uint32_t)(r.next() % E) : 0;
    int bw = (r.next() % 1000) < g.p.bw3_permille ? 3 : 5;
    bool null_root = (r.next() % 1000) < g.p.null_root_permille;
    ri.gas = (uint32_t)r.next();
    ri.has_root = !null_root && E > 0;
    ri.selected = sel && ri.has_root;
    if (!ri.has_root) { memset(root->b, 0, 38); return ri; }
    // events are generated sequentially from the receipt stream so any E works
    std::vector<Bytes> evs(E);
    for (uint32_t j = 0; j < E; j++) gen_event(g, r, i, j, sel && j == sel_pos, evs[j]);
    auto vf = [&](uint64_t k, Bytes& o) { o.insert(o.end(), evs[k].begin(), evs[k].end()); };
    auto kf = [](int, uint64_t) { return true; };
    *root = build_amt(E, bw, 3, vf, kf, out, 1);
    return ri;
}

// ------------------------------------------------------------------ HAMT builder
struct HEntry { uint8_t h[32]; Bytes key; Bytes val; };

static uint32_t hash_bits(const uint8_t h[32], int depth, int bw) {
    uint32_t v = 0;
    int start = depth * bw;
    for (int k = 0; k < bw; k++) {
        int bit = start + k;
        v = (v << 1) | ((h[bit / 8] >> (7 - bit % 8)) & 1);
    }
    return v;
}

static void hamt_bitfield(Bytes& o, const std::vector<uint32_t>& idxs) {
    uint8_t bf[32];
    memset(bf, 0, 32);
    for (uint32_t idx : idxs) bf[31 - idx / 8] |= (uint8_t)(1u << (idx % 8));
    int lead = 0;
    while (lead < 32 && bf[lead] == 0) lead++;
    cb_bytes(o, bf + lead, (size_t)(32 - lead));
}

// entries[lo,hi) sorted by hash and sharing the first depth*bw bits
static Bytes hamt_node(std::vector<HEntry>& es, size_t lo, size_t hi, int depth, int bw, BlockSet& out) {
    std::vector<uint32_t> idxs;
    Bytes ptrs;
    uint32_t nptr = 0;
    size_t a = lo;
    while (a < hi) {
        uint32_t idx = hash_bits(es[a].h, depth, bw);
        size_t b = a;
        while (b < hi && hash_bits(es[b].h, depth, bw) == idx) b++;
        idxs.push_back(idx);
        nptr++;
        if (b - a <= 3) {
            std::vector<size_t> ord;
            for (size_t k = a; k < b; k++) ord.push_back(k);
            std::sort(ord.begin(), ord.end(), [&](size_t x, size_t y) { return es[x].key < es[y].key; });
            cb_array(ptrs, b - a);
            for (size_t k : ord) {
                cb_array(ptrs, 2);
                cb_bytes(ptrs, es[k].key.data(), es[k].key.size());
                ptrs.insert(ptrs.end(), es[k].val.begin(), es[k].val.end());
            }
        } else {
            Bytes child = hamt_node(es, a, b, depth + 1, bw, out);
            Cid c = out.add(child);
            cb_cid(ptrs, c.b);
        }
        a = b;
    }
    Bytes node;
    cb_array(node, 2);
    hamt_bitfield(node, idxs);
    cb_array(node, nptr);
    node.insert(node.end(), ptrs.begin(), ptrs.end());
    return node;
}

static Cid build_hamt(std::vector<HEntry>& es, int bw, BlockSet& out) {
    std::sort(es.begin(), es.end(), [](const HEntry& x, const HEntry& y) { return memcmp(x.h, y.h, 32) < 0; });
    Bytes root = hamt_node(es, 0, es.size(), 0, bw, out);
    return out.add(root);
}

static void uvarint(Bytes& o, uint64_t v) {
    while (v >= 0x80) { o.push_back((uint8_t)(v | 0x80)); v >>= 7; }
    o.push_back((uint8_t)v);
}

static void storage_key32(uint64_t k, uint64_t n_entries, uint8_t key32[32]) {
    memset(key32, 0, 32);
    if (k == n_entries) { memcpy(key32, TARGET_TOPIC1, strlen(TARGET_TOPIC1)); return; }
    be64(key32 + 24, k);
}
static void mapping_slot(const uint8_t key32[32], uint64_t slot_index, uint8_t out[32]) {
    uint8_t buf[64];
    memcpy(buf, key32, 32);
    memset(buf + 32, 0, 24);
    be64(buf + 56, slot_index);
    cpu_crypto::keccak256(buf, 64, out);
}
static uint32_t storage_value(uint64_t seed, uint64_t k, uint64_t n_entries, uint8_t v[32]) {
    if (k == n_entries) { v[0] = 15; return 1; }
    Rng r = rng_for(seed, DOM_STORAGE, k);
    uint32_t len = 1 + (uint32_t)(r.next() % 32);
    for (uint32_t i = 0; i < len; i += 8) {
        uint64_t w = r.next();
        for (uint32_t b = 0; b < 8 && i + b < len; b++) v[i + b] = (uint8_t)(w >> (8 * b));
    }
    if (v[0] == 0) v[0] = 1;
    return len;
}

}  // namespace

struct synth_tipset {
    synth_params p;
    BlockSet bs;
    int64_t parent_epoch, child_epoch;
    std::vector<uint8_t> parent_cids, parent_txmeta;
    Cid child_cid, receipts_root, parent_state_root, storage_root;
    std::vector<uint8_t> events_roots, has_root;
    std::vector<uint64_t> selected;
    uint64_t target_actor;
};

extern "C" {

void synth_default_params(synth_params* p) {
    memset(p, 0, sizeof *p);
    p->seed = 0x1FC0FFEEULL;
    p->n_receipts = 64;
    p->events_per_receipt = 8;
    p->match_ppm = 10000;
    p->has_actor_filter = 1;
    p->target_actor = 1001;
    p->bw3_permille = 100;
    p->case_a_permille = 10;
    p->malformed_permille = 1;
    p->null_root_permille = 0;
    p->n_parents = 2;
    p->dup_msgs = 4;
    p->with_state_tree = 0;
    p->n_actors = 2048;
    p->hamt_entries = 0;
    p->threads = 0;
    p->same_topic1 = 0;
}

synth_tipset* synth_build(const synth_params* pp) {
    synth_tipset* T = new synth_tipset();
    T->p = *pp;
    synth_params& p = T->p;
    unsigned threads = p.threads ? p.threads : std::max(1u, std::thread::hardware_concurrency());
    if (p.n_parents == 0) p.n_parents = 1;
    Gen g;
    g.p = p; g.tp = make_topics(); g.target_actor = p.target_actor;
    T->target_actor = p.target_actor;
    const uint64_t N = p.n_receipts;
    bool sharded = !(p.shard_lo == 0 && p.shard_hi == 0);
    uint64_t slo = sharded ? p.shard_lo : 0, shi = sharded ? p.shard_hi : N;
    T->parent_epoch = 2992953;
    T->child_epoch = T->parent_epoch + 1;

    // ---- 1. events AMTs (parallel over receipts)
    T->events_roots.assign(N * 38, 0);
    T->has_root.assign(N, 0);
    std::vector<uint32_t> gas(N);
    std::vector<uint8_t> selflag(N, 0);
    {
        unsigned Tn = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(threads, N / 256 + 1));
        std::vector<BlockSet> tl(Tn);
        std::vector<std::thread> th;
        for (unsigned t = 0; t < Tn; t++) {
            th.emplace_back([&, t]() {
                uint64_t lo = N * t / Tn, hi = N * (t + 1) / Tn;
                for (uint64_t i = lo; i < hi; i++) {
                    Cid root;
                    bool keep = i >= slo && i < shi;
                    ReceiptInfo ri = gen_receipt(g, i, keep ? &tl[t] : nullptr, &root);
                    gas[i] = ri.gas;
                    T->has_root[i] = ri.has_root;
                    selflag[i] = ri.selected;
                    if (ri.has_root) memcpy(&T->events_roots[i * 38], root.b, 38);
                }
            });
        }
        for (auto& x : th) x.join();
        for (auto& b : tl) { T->bs.append(b); b = BlockSet(); }
    }
    for (uint64_t i = 0; i < N; i++) if (selflag[i]) T->selected.push_back(i);

    // ---- 2. receipts AMT (Amtv0, bit width 3)
    {
        auto vf = [&](uint64_t i, Bytes& o) {
            cb_array(o, 4);
            cb_uint(o, 0);
            cb_bytes(o, nullptr, 0);
            cb_uint(o, gas[i]);
            if (T->has_root[i]) cb_cid(o, &T->events_roots[i * 38]); else cb_null(o);
        };
        auto kf = [&](int level, uint64_t k) {
            if (!sharded) return true;
            // node covers receipts [k*8^(level+1), (k+1)*8^(level+1))
            unsigned sh = 3u * (unsigned)(level + 1);
            uint64_t a = sh >= 64 ? 0 : (k << sh);
            uint64_t b = sh >= 64 ? ~0ull : ((k + 1) << sh);
            return a < shi && b > slo;
        };
        T->receipts_root = build_amt(N, 3, 0, vf, kf, &T->bs, threads);
    }

    // ---- 3. message AMTs + TxMeta + parent headers
    // exec order = for each parent block: BLS AMT values then SECP AMT values (events/utils.rs:48-94)
    const uint32_t P = p.n_parents;
    std::vector<Cid> txmeta(P), phdr(P);
    auto msg_cid = [&](uint64_t k) {
        uint8_t buf[16];
        for (int i = 0; i < 8; i++) { buf[i] = (uint8_t)(k >> (8 * i)); buf[8 + i] = (uint8_t)(p.seed >> (8 * i)); }
        return cid_of(buf, 16);
    };
    uint64_t bls0 = 0;  // size of block 0's BLS list
    uint64_t nraw_total = N, raw_base = 0;
    {
        uint64_t b0 = (N * 1 / P - N * 0 / P) * 3 / 4;
        for (uint32_t b = 1; b < P; b++) nraw_total += std::min<uint64_t>(p.dup_msgs, b0);
    }
    for (uint32_t b = 0; b < P; b++) {
        uint64_t lo = N * b / P, hi = N * (b + 1) / P;
        uint64_t nbls = (hi - lo) * 3 / 4, nsecp = (hi - lo) - nbls;
        if (b == 0) bls0 = nbls;
        uint64_t dup = (b > 0) ? std::min<uint64_t>(p.dup_msgs, bls0) : 0;
        // BLS list of block b: [dup duplicates of block 0's first messages] + its own
        auto bls_v = [&](uint64_t i, Bytes& o) {
            uint64_t k = i < dup ? i : lo + (i - dup);
            Cid c = msg_cid(k);
            cb_cid(o, c.b);
        };
        auto secp_v = [&](uint64_t i, Bytes& o) {
            Cid c = msg_cid(lo + nbls + i);
            cb_cid(o, c.b);
        };
        // sharding of message AMTs: a shard keeps the nodes that intersect its share
        // [Nraw*slo/N, Nraw*shi/N) of the concatenated ("raw") message list of all AMTs
        auto mk_keep = [&](uint64_t amt_base) {
            return [=](int level, uint64_t k) {
                if (!sharded) return true;
                uint64_t glo = (uint64_t)((__uint128_t)nraw_total * slo / N), ghi = (uint64_t)((__uint128_t)nraw_total * shi / N);
                unsigned sh = 3u * (unsigned)(level + 1);
                uint64_t a = amt_base + (sh >= 64 ? 0 : (k << sh));
                uint64_t bb = sh >= 64 ? ~0ull : amt_base + ((k + 1) << sh);
                return a < ghi && bb > glo;
            };
        };
        uint64_t base_bls = raw_base, base_secp = raw_base + nbls + dup;
        raw_base += nbls + dup + nsecp;
        Cid bls_root = build_amt(nbls + dup, 3, 0, bls_v, mk_keep(base_bls), &T->bs, threads);
        Cid secp_root = build_amt(nsecp, 3, 0, secp_v, mk_keep(base_secp), &T->bs, threads);
        Bytes tm;
        cb_array(tm, 2); cb_cid(tm, bls_root.b); cb_cid(tm, secp_root.b);
        txmeta[b] = T->bs.add(tm);
    }
    auto header = [&](uint32_t which, int64_t height, const std::vector<Cid>& parents, const Cid& state_root,
                      const Cid& receipts, const Cid& messages) {
        Rng r = rng_for(p.seed, DOM_HDR, which);
        Bytes h;
        uint8_t junk[128];
        for (int i = 0; i < 128; i += 8) { uint64_t w = r.next(); memcpy(junk + i, &w, 8); }
        cb_array(h, 16);
        { Bytes a; a.push_back(0); uvarint(a, 1000 + which); cb_bytes(h, a.data(), a.size()); }  // 0 miner
        cb_array(h, 1); cb_bytes(h, junk, 32);                                                    // 1 ticket
        cb_array(h, 2); cb_uint(h, 1); cb_bytes(h, junk + 32, 32);                                // 2 election proof
        cb_array(h, 1); cb_array(h, 2); cb_uint(h, 4000000 + which); cb_bytes(h, junk + 64, 48);  // 3 beacon entries
        cb_array(h, 1); cb_array(h, 2); cb_uint(h, 3); cb_bytes(h, junk, 32);                     // 4 winpost proof
        cb_array(h, parents.size()); for (auto& c : parents) cb_cid(h, c.b);                      // 5 parents
        { uint8_t w[5] = {0, 0x12, 0x34, 0x56, (uint8_t)which}; cb_bytes(h, w, 5); }              // 6 parent weight
        cb_uint(h, (uint64_t)height);                                                             // 7 height
        cb_cid(h, state_root.b);                                                                  // 8 parent_state_root
        cb_cid(h, receipts.b);                                                                    // 9 parent_message_receipts
        cb_cid(h, messages.b);                                                                    // 10 messages
        { uint8_t s[97]; s[0] = 2; memcpy(s + 1, junk, 96); cb_bytes(h, s, 97); }                 // 11 bls aggregate
        cb_uint(h, 1700000000ull + (uint64_t)height * 30);                                        // 12 timestamp
        { uint8_t s[97]; s[0] = 2; memcpy(s + 1, junk + 16, 96); cb_bytes(h, s, 97); }            // 13 block sig
        cb_uint(h, 0);                                                                            // 14 fork signaling
        { uint8_t f[2] = {0, 100}; cb_bytes(h, f, 2); }                                           // 15 parent base fee
        return h;
    };
    std::vector<Cid> grand{fake_cid("grandparent", 0, p.seed)};
    for (uint32_t b = 0; b < P; b++) {
        Bytes h = header(b, T->parent_epoch, grand, fake_cid("gp-state", b, p.seed), fake_cid("gp-receipts", b, p.seed), txmeta[b]);
        phdr[b] = T->bs.add(h);
    }
    for (uint32_t b = 0; b < P; b++) {
        T->parent_cids.insert(T->parent_cids.end(), phdr[b].b, phdr[b].b + 38);
        T->parent_txmeta.insert(T->parent_txmeta.end(), txmeta[b].b, txmeta[b].b + 38);
    }

    // ---- 4. state tree
    Cid state_root = fake_cid("state-root", 0, p.seed);
    memset(T->storage_root.b, 0, 38);
    if (p.with_state_tree) {
        // storage HAMT of the target EVM actor: slot -> Vec<u8> (serde seq of u8, see DESIGN.md)
        const uint64_t M = p.hamt_entries;
        std::vector<HEntry> es(M + 1);
        {
            unsigned Tn = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(threads, M / 4096 + 1));
            std::vector<std::thread> th;
            for (unsigned t = 0; t < Tn; t++) {
                th.emplace_back([&, t]() {
                    uint64_t lo = (M + 1) * t / Tn, hi = (M + 1) * (t + 1) / Tn;
                    for (uint64_t k = lo; k < hi; k++) {
                        uint8_t key32[32], slot[32], v[32];
                        storage_key32(k, M, key32);
                        mapping_slot(key32, 0, slot);
                        uint32_t vl = storage_value(p.seed, k, M, v);
                        HEntry& e = es[k];
                        e.key.assign(slot, slot + 32);
                        cpu_crypto::sha256(slot, 32, e.h);
                        cb_array(e.val, vl);
                        for (uint32_t i = 0; i < vl; i++) cb_uint(e.val, v[i]);
                    }
                });
            }
            for (auto& x : th) x.join();
        }
        Cid hamt_root = build_hamt(es, 5, T->bs);
        T->storage_root = hamt_root;
        es.clear(); es.shrink_to_fit();
        // alternative contract_state shapes (storage/decode.rs:45-89)
        auto small_pairs = [&](Bytes& o) {
            cb_map(o, 1); cb_text(o, "v"); cb_array(o, 3);
            for (uint64_t k = 0; k < 3; k++) {
                uint8_t key32[32], slot[32], v[32];
                storage_key32(k, M, key32); mapping_slot(key32, 0, slot);
                uint32_t vl = storage_value(p.seed, k, M, v);
                cb_array(o, 2); cb_bytes(o, slot, 32); cb_bytes(o, v, vl);
            }
        };
        uint8_t params[3] = {1, 2, 3};
        Bytes b1; cb_array(b1, 2); cb_cid(b1, hamt_root.b); cb_uint(b1, 5);
        Bytes a3; small_pairs(a3);
        Bytes a2; cb_array(a2, 2); cb_bytes(a2, params, 3); small_pairs(a2);
        Bytes a1; cb_array(a1, 2); cb_bytes(a1, params, 3); cb_array(a1, 1); small_pairs(a1);
        Bytes b2; cb_map(b2, 2); cb_text(b2, "root"); cb_cid(b2, hamt_root.b); cb_text(b2, "bitwidth"); cb_uint(b2, 5);
        Cid c_b1 = T->bs.add(b1), c_a3 = T->bs.add(a3), c_a2 = T->bs.add(a2), c_a1 = T->bs.add(a1), c_b2 = T->bs.add(b2);
        // actors HAMT
        std::vector<HEntry> as(p.n_actors);
        for (uint32_t a = 0; a < p.n_actors; a++) {
            uint64_t id = 1000 + a;
            Rng r = rng_for(p.seed, DOM_ACTOR, id);
            HEntry& e = as[a];
            e.key.push_back(0); uvarint(e.key, id);
            cpu_crypto::sha256(e.key.data(), e.key.size(), e.h);
            Cid state = fake_cid("actor-state", id, p.seed);
            const Cid* cs = nullptr;
            bool v5 = false;
            switch (id) {
                case 1001: cs = &hamt_root; break;
                case 1002: cs = &c_b1; v5 = true; break;
                case 1003: cs = &c_a3; break;
                case 1004: cs = &c_a2; break;
                case 1005: cs = &c_a1; break;
                case 1006: cs = &c_b2; break;
                default: break;
            }
            if (id == p.target_actor && !cs) cs = &hamt_root;
            if (cs) {
                Bytes ev;
                uint8_t bh[32];
                for (int i = 0; i < 32; i += 8) { uint64_t w = r.next(); memcpy(bh + i, &w, 8); }
                Cid bytecode = fake_cid("bytecode", id, p.seed);
                cb_array(ev, v5 ? 5 : 6);
                cb_cid(ev, bytecode.b); cb_bytes(ev, bh, 32); cb_cid(ev, cs->b);
                if (!v5) cb_null(ev);
                cb_uint(ev, 1);
                cb_null(ev);
                state = T->bs.add(ev);
            }
            Cid code = fake_cid("code", id % 7, p.seed);
            cb_array(e.val, 5);
            cb_cid(e.val, code.b); cb_cid(e.val, state.b); cb_uint(e.val, r.next() % 100000);
            { uint8_t bal[4] = {0, (uint8_t)r.next(), (uint8_t)r.next(), (uint8_t)r.next()}; cb_bytes(e.val, bal, 4); }
            if (cs) { uint8_t da[22]; da[0] = 4; da[1] = 10; for (int i = 2; i < 22; i++) da[i] = (uint8_t)r.next(); cb_bytes(e.val, da, 22); }
            else cb_null(e.val);
        }
        Cid actors_root = build_hamt(as, 5, T->bs);
        Bytes info; cb_array(info, 0);
        Cid info_cid = T->bs.add(info);
        Bytes sr; cb_array(sr, 3); cb_uint(sr, 5); cb_cid(sr, actors_root.b); cb_cid(sr, info_cid.b);
        state_root = T->bs.add(sr);
    }
    T->parent_state_root = state_root;

    // ---- 5. child header
    {
        std::vector<Cid> parents(phdr.begin(), phdr.end());
        Bytes h = header(100, T->child_epoch, parents, state_root, T->receipts_root, fake_cid("child-messages", 0, p.seed));
        T->child_cid = T->bs.add(h);
    }
    return T;
}

void synth_free(synth_tipset* t) { delete t; }

uint64_t synth_n_blocks(const synth_tipset* t) { return t->bs.n(); }
const uint8_t* synth_cids(const synth_tipset* t) { return t->bs.cids.data(); }
const uint64_t* synth_offsets(const synth_tipset* t) { return t->bs.offs.data(); }
const uint32_t* synth_lengths(const synth_tipset* t) { return t->bs.lens.data(); }
const uint8_t* synth_blob(const synth_tipset* t) { return t->bs.blob.data(); }
uint64_t synth_blob_size(const synth_tipset* t) { return t->bs.blob.size(); }

int64_t synth_parent_epoch(const synth_tipset* t) { return t->parent_epoch; }
int64_t synth_child_epoch(const synth_tipset* t) { return t->child_epoch; }
uint32_t synth_n_parents(const synth_tipset* t) { return t->p.n_parents; }
const uint8_t* synth_parent_cids(const synth_tipset* t) { return t->parent_cids.data(); }
const uint8_t* synth_parent_txmeta_cids(const synth_tipset* t) { return t->parent_txmeta.data(); }
const uint8_t* synth_child_cid(const synth_tipset* t) { return t->child_cid.b; }
const uint8_t* synth_receipts_root(const synth_tipset* t) { return t->receipts_root.b; }
const uint8_t* synth_parent_state_root(const synth_tipset* t) { return t->parent_state_root.b; }
uint64_t synth_n_receipts(const synth_tipset* t) { return t->p.n_receipts; }
const uint8_t* synth_events_roots(const synth_tipset* t) { return t->events_roots.data(); }
const uint8_t* synth_has_events_root(const synth_tipset* t) { return t->has_root.data(); }
const char* synth_event_signature(const synth_tipset*) { return TARGET_SIG; }
const char* synth_topic1(const synth_tipset*) { return TARGET_TOPIC1; }
uint64_t synth_target_actor(const synth_tipset* t) { return t->target_actor; }
uint64_t synth_n_selected(const synth_tipset* t) { return t->selected.size(); }
const uint64_t* synth_selected(const synth_tipset* t) { return t->selected.data(); }
const uint8_t* synth_storage_root(const synth_tipset* t) { return t->storage_root.b; }

uint32_t synth_storage_entry(const synth_tipset* t, uint64_t k, uint8_t key32[32], uint8_t value[32]) {
    storage_key32(k, t->p.hamt_entries, key32);
    return storage_value(t->p.seed, k, t->p.hamt_entries, value);
}
void synth_storage_absent_key(const synth_tipset*, uint64_t k, uint8_t key32[32]) {
    memset(key32, 0xff, 24);
    be64(key32 + 24, k);
}

void synth_blake2b256(const uint8_t* in, uint64_t len, uint8_t out[32]) { cpu_crypto::blake2b256(in, (size_t)len, out); }
void synth_keccak256(const uint8_t* in, uint64_t len, uint8_t out[32]) { cpu_crypto::keccak256(in, (size_t)len, out); }
void synth_sha256(const uint8_t* in, uint64_t len, uint8_t out[32]) { cpu_crypto::sha256(in, (size_t)len, out); }

}  // extern "C"
