// json_parse_items.cuh — per-item functions of the device bundle parser (ipcfp_verify_bundle_json, csrc/json_parse.cu): the CANONICAL
// text of an EventProofBundle / UnifiedProofBundle — what serde_json::to_string, csrc/bundle_json.cpp, json_items.cuh and bundle_json.py
// write — read back into the PODs csrc/bundle_parse.cpp (ipcfp_bundle_from_json) returns. They live in a header so that
// tests/host_fuzz/emu_json_parse.cu runs the very same code on the CPU against bundle_parse.cpp.
//
// Canonical means: struct field order, no whitespace, ProofBlock.cid as the 38-number byte array, CID strings of exactly 62 characters
// ("b" + 61 base32 characters whose one unused bit is zero), lower-case "0x" hex with 32-byte topics, base64 with padding and zero unused
// bits, integers without leading zeros or "-0". Any other text is refused here (the caller DEFERS to the host parser), so that "accepted
// here ⇒ the host parser accepts the same text with the same values" holds by construction: every byte of an accepted text is consumed
// by exactly one template check —
//   * a record is found by its first bytes ({"parent_epoch": / {"child_epoch": / {"cid":[; a canonical string holds no '{' or '"', so
//     these occur at record starts only), and each record is parsed by a strict template from its start;
//   * a record must end exactly one comma before the next record of its list (blocks: their span IS that gap, and every byte of the
//     data string must be base64);
//   * the list framing {"proofs":[…],"blocks":[…]} / {"storage_proofs":[…],"event_proofs":[…],"blocks":[…]} must join the lists'
//     first and last records exactly, and end at the end of the text (jp_frame_ok).
// Range checks are those of bundle_parse.cpp: u64 overflow, the i64 range, CID bytes ≤ 255, data_len ≤ u32; the fields every proof shares
// must equal the previous proof's of the same list (text equality: canonical spellings are unique), storage vs event proofs on the host.
//
// Every buffer these functions read holds the text followed by JP_PAD zero bytes (jp_kind_at looks 16 bytes ahead).
#pragma once
#include "common.cuh"

namespace ipcfp {

#define JP_FN __host__ __device__ __forceinline__
#define JP_PAD 64u
#define JP_MIN_RECORD 95u   // the shortest canonical record: a block of 38 one-digit CID bytes and no data
enum : uint32_t { JP_STORAGE = 0, JP_EVENT = 1, JP_BLOCK = 2, JP_NONE = 3 };

JP_FN bool jp_same(const char* a, const char* b, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) if (a[i] != b[i]) return false;
    return true;
}
// the record kind whose first bytes stand at p (reads at most 16 bytes from p)
JP_FN uint32_t jp_kind_at(const char* t, uint64_t p) {
    if (t[p] != '{' || t[p + 1] != '"') return JP_NONE;
    if (jp_same(t + p, "{\"cid\":[", 8)) return JP_BLOCK;
    if (jp_same(t + p, "{\"parent_epoch\":", 16)) return JP_EVENT;
    if (jp_same(t + p, "{\"child_epoch\":", 15)) return JP_STORAGE;
    return JP_NONE;
}
JP_FN int jp_b32(char c) { return c >= 'a' && c <= 'z' ? c - 'a' : c >= '2' && c <= '7' ? c - '2' + 26 : -1; }
JP_FN int jp_hex(char c) { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : -1; }
JP_FN int jp_b64(char c) {
    return c >= 'A' && c <= 'Z' ? c - 'A' : c >= 'a' && c <= 'z' ? c - 'a' + 26 : c >= '0' && c <= '9' ? c - '0' + 52 : c == '+' ? 62 : c == '/' ? 63 : -1;
}

// a template cursor over t[p, e): every read is bounds-checked against e
struct JpCur {
    const char* t;
    uint64_t p, e;
    template <int N> JP_FN bool lit(const char (&s)[N]) {
        if (e - p < (uint64_t)(N - 1)) return false;
        for (int i = 0; i < N - 1; i++) if (t[p + i] != s[i]) return false;
        p += N - 1;
        return true;
    }
    JP_FN bool peek(char c) const { return p < e && t[p] == c; }
    // canonical u64: "0" or [1-9][0-9]*, no overflow (a digit after a leading "0" fails the next literal)
    JP_FN bool u64(uint64_t& v) {
        if (p >= e || t[p] < '0' || t[p] > '9') return false;
        v = 0;
        if (t[p] == '0') { p++; return true; }
        while (p < e && t[p] >= '0' && t[p] <= '9') {
            const uint64_t d = (uint64_t)(t[p] - '0');
            if (v > (UINT64_MAX - d) / 10) return false;
            v = v * 10 + d;
            p++;
        }
        return true;
    }
    JP_FN bool i64(int64_t& v) {
        const bool neg = peek('-');
        if (neg) p++;
        uint64_t a;
        if (!u64(a)) return false;
        if (neg) { if (a == 0 || a > (uint64_t)INT64_MAX + 1) return false; v = (int64_t)(0 - a); return true; }
        if (a > (uint64_t)INT64_MAX) return false;
        v = (int64_t)a;
        return true;
    }
    // "b" + 61 base32 characters, the one unused bit zero → 38 bytes (out may be null)
    JP_FN bool cid(uint8_t* out) {
        if (e - p < 64 || t[p] != '"' || t[p + 1] != 'b' || t[p + 63] != '"') return false;
        uint32_t acc = 0;
        int bits = 0, k = 0;
        for (int i = 0; i < 61; i++) {
            const int d = jp_b32(t[p + 2 + i]);
            if (d < 0) return false;
            acc = (acc << 5) | (uint32_t)d;
            bits += 5;
            if (bits >= 8) { if (out) out[k] = (uint8_t)(acc >> (bits - 8)); k++; bits -= 8; acc &= (1u << bits) - 1; }
        }
        if (acc) return false;
        p += 64;
        return true;
    }
    // "0x" + 64 lower-case hex digits (out may be null)
    JP_FN bool hex32(uint8_t* out) {
        if (e - p < 68 || t[p] != '"' || t[p + 1] != '0' || t[p + 2] != 'x' || t[p + 67] != '"') return false;
        for (int i = 0; i < 32; i++) {
            const int h = jp_hex(t[p + 3 + 2 * i]), l = jp_hex(t[p + 4 + 2 * i]);
            if (h < 0 || l < 0) return false;
            if (out) out[i] = (uint8_t)(h * 16 + l);
        }
        p += 68;
        return true;
    }
    // "0x" + an even number of lower-case hex digits: the digits start at *at, *n bytes
    JP_FN bool hex_span(uint64_t& at, uint64_t& n) {
        if (!lit("\"0x")) return false;
        at = p;
        while (p < e && jp_hex(t[p]) >= 0) p++;
        if ((p - at) & 1) return false;
        n = (p - at) / 2;
        return lit("\"");
    }
};
JP_FN void jp_unhex(const char* s, uint64_t n, uint8_t* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = (uint8_t)(jp_hex(s[2 * i]) * 16 + jp_hex(s[2 * i + 1]));
}

// ---- EventProof (events/bundle.rs:14-23) as bundle_json.cpp::event_proofs_json writes it
struct JpEvent {
    int64_t parent_epoch, child_epoch;
    uint32_t n_parents, n_topics;
    uint64_t parents_at;   // first parent CID string (its quote); parent q at parents_at + 65·q
    uint64_t child_at, message_at, header_end;   // header = [record start, header_end): the fields every proof of the list shares
    uint64_t exec_index, event_index, emitter;
    uint64_t topics_at;    // first topic string (its quote); topic q at topics_at + 69·q
    uint64_t data_at, data_len;   // hex digits of `data`, its byte count
};
// parses the record at `at`; *end = one past its closing brace
JP_FN bool jp_event_proof(const char* t, uint64_t at, uint64_t e, JpEvent& r, uint64_t& end) {
    JpCur c{t, at, e};
    if (!c.lit("{\"parent_epoch\":") || !c.i64(r.parent_epoch) || !c.lit(",\"child_epoch\":") || !c.i64(r.child_epoch)) return false;
    if (!c.lit(",\"parent_tipset_cids\":[")) return false;
    r.parents_at = c.p;
    r.n_parents = 0;
    if (!c.peek(']')) for (;;) {
        if (!c.cid(nullptr) || ++r.n_parents > (1u << 20)) return false;
        if (!c.peek(',')) break;
        c.p++;
    }
    if (!c.lit("],\"child_block_cid\":")) return false;
    r.child_at = c.p;
    if (!c.cid(nullptr)) return false;
    r.header_end = c.p;
    if (!c.lit(",\"message_cid\":")) return false;
    r.message_at = c.p;
    if (!c.cid(nullptr)) return false;
    if (!c.lit(",\"exec_index\":") || !c.u64(r.exec_index) || !c.lit(",\"event_index\":") || !c.u64(r.event_index)) return false;
    if (!c.lit(",\"event_data\":{\"emitter\":") || !c.u64(r.emitter) || !c.lit(",\"topics\":[")) return false;
    r.topics_at = c.p;
    r.n_topics = 0;
    if (!c.peek(']')) for (;;) {
        if (!c.hex32(nullptr) || ++r.n_topics > (1u << 24)) return false;
        if (!c.peek(',')) break;
        c.p++;
    }
    if (!c.lit("],\"data\":") || !c.hex_span(r.data_at, r.data_len) || r.data_len > 0xffffffffull || !c.lit("}}")) return false;
    end = c.p;
    return true;
}
// bytes of the data blob this proof takes: topics, then data (bundle_parse.cpp::read_event_proofs)
JP_FN uint64_t jp_event_blob_len(const JpEvent& r) { return 32ull * r.n_topics + r.data_len; }
// the POD and its blob bytes (at blob + off), from a record jp_event_proof accepted
JP_FN void jp_event_write(const char* t, const JpEvent& r, uint64_t off, ipcfp_event_proof& p, uint8_t* blob) {
    for (uint32_t k = 0; k < sizeof(ipcfp_event_proof); k++) ((uint8_t*)&p)[k] = 0;
    p.exec_index = r.exec_index; p.event_index = r.event_index; p.emitter = r.emitter;
    p.n_topics = r.n_topics; p.data_len = (uint32_t)r.data_len;
    p.topics_off = off; p.data_off = off + 32ull * r.n_topics;
    JpCur c{t, r.message_at, r.message_at + 64};
    c.cid(p.message_cid);
    for (uint32_t q = 0; q < r.n_topics; q++) jp_unhex(t + r.topics_at + 69ull * q + 3, 32, blob + off + 32ull * q);
    jp_unhex(t + r.data_at, r.data_len, blob + p.data_off);
}

// ---- StorageProof (storage/bundle.rs:5-14); out (may be null) receives the POD as bundle_parse.cpp fills it
struct JpStorage {
    int64_t child_epoch;
    uint64_t child_at, root_at, header_end;   // header = [record start, header_end): child epoch, child block CID, parent state root
};
JP_FN bool jp_storage_proof(const char* t, uint64_t at, uint64_t e, JpStorage& r, uint64_t& end, ipcfp_storage_proof* out) {
    JpCur c{t, at, e};
    if (out) for (uint32_t k = 0; k < sizeof(ipcfp_storage_proof); k++) ((uint8_t*)out)[k] = 0;
    if (!c.lit("{\"child_epoch\":") || !c.i64(r.child_epoch) || !c.lit(",\"child_block_cid\":")) return false;
    r.child_at = c.p;
    if (!c.cid(nullptr) || !c.lit(",\"parent_state_root\":")) return false;
    r.root_at = c.p;
    if (!c.cid(nullptr)) return false;
    r.header_end = c.p;
    uint64_t actor;
    if (!c.lit(",\"actor_id\":") || !c.u64(actor) || !c.lit(",\"actor_state_cid\":") || !c.cid(out ? out->actor_state_cid : nullptr)) return false;
    if (!c.lit(",\"storage_root\":") || !c.cid(out ? out->storage_root : nullptr)) return false;
    if (!c.lit(",\"slot\":") || !c.hex32(out ? out->slot : nullptr) || !c.lit(",\"value\":") || !c.hex32(out ? out->value : nullptr) || !c.lit("}"))
        return false;
    if (out) { out->actor_id = actor; out->found = 1; out->raw_len = 32; }
    end = c.p;
    return true;
}

// ---- ProofBlock {"cid":[d,…,d],"data":"<base64>"}: the record is t[at, end) (end = the comma before the next block, or the list's
// closing bracket), so its data string is known before it is read
struct JpBlock {
    uint64_t data_at, n_chars;   // the base64 characters
    uint32_t pads, len;          // '=' count, decoded length
};
// the base64 string of b.n_chars characters at b.data_at: its length, padding and zero unused bits; sets pads and len. The characters
// before the padding are left to jp_block_char_ok.
JP_FN bool jp_b64_span(const char* t, JpBlock& b) {
    if (b.n_chars & 3) return false;
    const char* d = t + b.data_at;
    const uint64_t n = b.n_chars;
    b.pads = 0;
    if (n && d[n - 1] == '=') b.pads = d[n - 2] == '=' ? 2 : 1;
    else if (n && d[n - 2] == '=') return false;
    if (b.pads == 2 && (jp_b64(d[n - 3]) & 15)) return false;    // canonical: the unused bits are zero
    if (b.pads == 1 && (jp_b64(d[n - 2]) & 3)) return false;
    const uint64_t len = n / 4 * 3 - b.pads;
    if (len > 0xffffffffull) return false;
    b.len = (uint32_t)len;
    return true;
}
JP_FN bool jp_block_head(const char* t, uint64_t at, uint64_t end, JpBlock& b, uint8_t* cid_out) {
    JpCur c{t, at, end};
    if (!c.lit("{\"cid\":[")) return false;
    for (int k = 0; k < IPCFP_CID_LEN; k++) {
        uint64_t v;
        if ((k && !c.lit(",")) || !c.u64(v) || v > 255) return false;
        if (cid_out) cid_out[k] = (uint8_t)v;
    }
    if (!c.lit("],\"data\":\"") || end - c.p < 2 || t[end - 2] != '"' || t[end - 1] != '}') return false;
    b.data_at = c.p;
    b.n_chars = end - 2 - c.p;
    return jp_b64_span(t, b);
}
// data character k (k < n_chars - pads) is a base64 digit: what jp_block_head leaves to the lanes
JP_FN bool jp_block_char_ok(const char* t, const JpBlock& b, uint64_t k) { return jp_b64(t[b.data_at + k]) >= 0; }
// decoded bytes 3g .. 3g+2 (those below len) of group g
JP_FN void jp_block_group(const char* t, const JpBlock& b, uint64_t g, uint8_t* out) {
    const char* q = t + b.data_at + 4 * g;
    const uint32_t v = ((uint32_t)jp_b64(q[0]) << 18) | ((uint32_t)jp_b64(q[1]) << 12) | (q[2] == '=' ? 0u : (uint32_t)jp_b64(q[2]) << 6) |
                       (q[3] == '=' ? 0u : (uint32_t)jp_b64(q[3]));
    const uint64_t i = 3 * g;
    out[i] = (uint8_t)(v >> 16);
    if (i + 1 < b.len) out[i + 1] = (uint8_t)(v >> 8);
    if (i + 2 < b.len) out[i + 2] = (uint8_t)v;
}
JP_FN uint64_t jp_align16(uint64_t n) { return (n + 15) & ~15ull; }

// ---- record i of the n candidates at pos[] (ascending): its template check and its joints with its neighbours
struct JpRec {
    uint32_t kind;
    bool first, last;        // first / last record of its list
    uint64_t end;            // one past the record
    uint64_t blob_len;       // events: data-blob bytes; blocks: 16-aligned arena bytes
    uint32_t len;            // blocks: decoded length
    JpEvent ev;              // events
    JpBlock blk;             // blocks
};
// false: not canonical (defer). Blocks: the base64 characters are left to jp_block_char_ok.
JP_FN bool jp_record(const char* t, uint64_t len, const uint32_t* pos, uint64_t n, uint64_t i, JpRec& r) {
    const uint64_t at = pos[i];
    r.kind = jp_kind_at(t, at);
    const uint32_t prev = i ? jp_kind_at(t, pos[i - 1]) : JP_NONE, next = i + 1 < n ? jp_kind_at(t, pos[i + 1]) : JP_NONE;
    if (r.kind == JP_NONE || (i && prev > r.kind) || (i + 1 < n && next < r.kind)) return false;   // lists in S, E, B order
    r.first = prev != r.kind;
    r.last = next != r.kind;
    r.blob_len = 0;
    r.len = 0;
    uint64_t hdr = 0;
    if (r.kind == JP_BLOCK) {
        r.end = i + 1 < n ? (uint64_t)pos[i + 1] - 1 : len - 2;   // the blocks list is the last: "]}" follows its last record
        if (r.end < at || (i + 1 < n && t[r.end] != ',') || !jp_block_head(t, at, r.end, r.blk, nullptr)) return false;
        r.len = r.blk.len;
        r.blob_len = jp_align16(r.blk.len);
        return true;
    }
    if (r.kind == JP_EVENT) {
        if (!jp_event_proof(t, at, len, r.ev, r.end)) return false;
        r.blob_len = jp_event_blob_len(r.ev);
        hdr = r.ev.header_end - at;
    } else {
        JpStorage s;
        if (!jp_storage_proof(t, at, len, s, r.end, nullptr)) return false;
        hdr = s.header_end - at;
    }
    if (!r.last && (r.end >= len || t[r.end] != ',' || pos[i + 1] != r.end + 1)) return false;
    // the shared fields equal the previous proof's of this list (so, by induction, the first one's)
    if (!r.first && !jp_same(t + pos[i - 1], t + at, hdr)) return false;
    return true;
}

// the framing around the lists: cnt / first_start / last_end of each kind from the records
JP_FN bool jp_frame_ok(const char* t, uint64_t len, const uint64_t cnt[3], const uint64_t first_start[3], const uint64_t last_end[3]) {
    JpCur c{t, 0, len};
    uint32_t lists[3], nl = 0;
    if (c.lit("{\"proofs\":")) { if (cnt[JP_STORAGE]) return false; lists[nl++] = JP_EVENT; }
    else if (c.lit("{\"storage_proofs\":")) { lists[nl++] = JP_STORAGE; lists[nl++] = JP_EVENT; }
    else return false;
    lists[nl++] = JP_BLOCK;
    for (uint32_t l = 0; l < nl; l++) {
        const uint32_t k = lists[l];
        if (l == 1 && nl == 3 && !c.lit(",\"event_proofs\":")) return false;
        if (l == nl - 1 && !c.lit(",\"blocks\":")) return false;
        if (!c.lit("[")) return false;
        if (cnt[k]) {
            if (first_start[k] != c.p || last_end[k] < c.p || last_end[k] > len) return false;
            c.p = last_end[k];
        }
        if (!c.lit("]")) return false;
    }
    return c.lit("}") && c.p == len;
}

// the CID string at `at` (accepted before) → 38 bytes
JP_FN void jp_cid_at(const char* t, uint64_t at, uint8_t* out) {
    JpCur c{t, at, at + 64};
    c.cid(out);
}
// the fields every proof shares, read from the first proof of each list (the records checked that the others repeat them): what
// bundle_parse.cpp returns as ipcfp_parsed_bundle.tipset. false: the storage and event proofs disagree (bundle_parse.cpp refuses that).
struct JpTipset {
    int64_t parent_epoch = 0, child_epoch = 0;
    uint32_t n_parents = 0;
    uint64_t parents_at = 0;              // parent q: jp_cid_at(t, parents_at + 65·q)
    bool has_child = false, has_root = false;
    uint8_t child[IPCFP_CID_LEN] = {}, root[IPCFP_CID_LEN] = {};
};
JP_FN bool jp_tipset(const char* t, uint64_t len, const uint64_t cnt[3], const uint64_t first_start[3], JpTipset& ts) {
    uint64_t end;
    JpStorage s;
    JpEvent e;
    if (cnt[JP_STORAGE]) {
        if (!jp_storage_proof(t, first_start[JP_STORAGE], len, s, end, nullptr)) return false;
        ts.child_epoch = s.child_epoch;
        jp_cid_at(t, s.child_at, ts.child);
        jp_cid_at(t, s.root_at, ts.root);
        ts.has_child = ts.has_root = true;
    }
    if (cnt[JP_EVENT]) {
        if (!jp_event_proof(t, first_start[JP_EVENT], len, e, end)) return false;
        uint8_t child[IPCFP_CID_LEN];
        jp_cid_at(t, e.child_at, child);
        if (ts.has_child && (ts.child_epoch != e.child_epoch || !jp_same((const char*)child, (const char*)ts.child, IPCFP_CID_LEN))) return false;
        ts.child_epoch = e.child_epoch;
        for (int k = 0; k < IPCFP_CID_LEN; k++) ts.child[k] = child[k];
        ts.has_child = true;
        ts.parent_epoch = e.parent_epoch;
        ts.n_parents = e.n_parents;
        ts.parents_at = e.parents_at;
    }
    return true;
}

}  // namespace ipcfp
