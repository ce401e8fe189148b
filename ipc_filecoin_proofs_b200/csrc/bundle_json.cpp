// bundle_json.cpp — wire format of the reference's proof bundles behind the C ABI (SURVEY §8 f-3).
//
// ipcfp_bundle_to_json renders an ipcfp_bundle as `serde_json::to_string(&UnifiedProofBundle)` gives it in the reference
// (src/proofs/common/bundle.rs:10-45, src/proofs/events/bundle.rs:5-30, src/proofs/storage/bundle.rs:5-14); ipcfp_event_result_to_json
// renders one ipcfp_event_result as an EventProofBundle. Host-side string work only — no device, no CUDA call:
//   * struct field order, compact separators;
//   * CIDs held as String (`child_block_cid`, `message_cid`, `parent_tipset_cids`, `parent_state_root`, `actor_state_cid`,
//     `storage_root`): `Cid::to_string()` = multibase 'b' + lower-case RFC 4648 base32 without padding (events/generator.rs:289,
//     storage/generator.rs:170-174);
//   * `topics`, `data`, `slot`, `value`: "0x" + lower-case hex (events/generator.rs:279-281, storage/generator.rs:175-176);
//   * `ProofBlock.data`: standard base64 with padding (common/bundle.rs:20-26);
//   * `ProofBlock.cid` is a `cid::Cid`: cid 0.11's Serialize hands the CID bytes to the serializer, which serde_json writes as an
//     array of numbers ([UPSTREAM] behaviour restated, unpinned by the reference — same choice as bundle_json.py).
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>

#include "../../include/ipcfp.h"

namespace {

void cid_string(std::string& o, const uint8_t* c) {   // 38 raw bytes → "bafy2bzace…"
    static const char* B32 = "abcdefghijklmnopqrstuvwxyz234567";
    o.push_back('"');
    o.push_back('b');
    uint32_t acc = 0;
    int bits = 0;
    for (int i = 0; i < IPCFP_CID_LEN; i++) {
        acc = (acc << 8) | c[i];
        bits += 8;
        while (bits >= 5) { o.push_back(B32[(acc >> (bits - 5)) & 31]); bits -= 5; }
    }
    if (bits) o.push_back(B32[(acc << (5 - bits)) & 31]);
    o.push_back('"');
}
void hex0x(std::string& o, const uint8_t* p, uint64_t n) {
    static const char* H = "0123456789abcdef";
    o += "\"0x";
    for (uint64_t i = 0; i < n; i++) { o.push_back(H[p[i] >> 4]); o.push_back(H[p[i] & 15]); }
    o.push_back('"');
}
void base64(std::string& o, const uint8_t* p, uint64_t n) {
    static const char* T = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    o.push_back('"');
    uint64_t i = 0;
    for (; i + 3 <= n; i += 3) {
        uint32_t v = ((uint32_t)p[i] << 16) | ((uint32_t)p[i + 1] << 8) | p[i + 2];
        o.push_back(T[v >> 18]); o.push_back(T[(v >> 12) & 63]); o.push_back(T[(v >> 6) & 63]); o.push_back(T[v & 63]);
    }
    if (n - i == 1) { uint32_t v = (uint32_t)p[i] << 16; o.push_back(T[v >> 18]); o.push_back(T[(v >> 12) & 63]); o += "=="; }
    else if (n - i == 2) { uint32_t v = ((uint32_t)p[i] << 16) | ((uint32_t)p[i + 1] << 8); o.push_back(T[v >> 18]); o.push_back(T[(v >> 12) & 63]); o.push_back(T[(v >> 6) & 63]); o.push_back('='); }
    o.push_back('"');
}
void num(std::string& o, uint64_t v) { o += std::to_string(v); }
void snum(std::string& o, int64_t v) { o += std::to_string(v); }

void blocks_json(std::string& o, const ipcfp_witness& w) {   // Vec<ProofBlock>
    o.push_back('[');
    for (uint64_t i = 0; i < w.n_blocks; i++) {
        if (i) o.push_back(',');
        o += "{\"cid\":[";
        for (int k = 0; k < IPCFP_CID_LEN; k++) { if (k) o.push_back(','); num(o, w.cids[38 * i + k]); }
        o += "],\"data\":";
        base64(o, w.blob + w.offsets[i], w.lengths[i]);
        o.push_back('}');
    }
    o.push_back(']');
}
void event_proofs_json(std::string& o, const ipcfp_tipset_desc& t, const ipcfp_event_result& r, bool& first) {   // EventProof items (events/bundle.rs:14-23)
    for (uint64_t k = 0; k < r.n_proofs; k++) {
        const ipcfp_event_proof& p = r.proofs[k];
        if (!first) o.push_back(',');
        first = false;
        o += "{\"parent_epoch\":"; snum(o, t.parent_epoch);
        o += ",\"child_epoch\":"; snum(o, t.child_epoch);
        o += ",\"parent_tipset_cids\":[";
        for (uint32_t q = 0; q < t.n_parents; q++) { if (q) o.push_back(','); cid_string(o, t.parent_cids + 38 * q); }
        o += "],\"child_block_cid\":"; cid_string(o, t.child_cid);
        o += ",\"message_cid\":"; cid_string(o, p.message_cid);
        o += ",\"exec_index\":"; num(o, p.exec_index);
        o += ",\"event_index\":"; num(o, p.event_index);
        o += ",\"event_data\":{\"emitter\":"; num(o, p.emitter);
        o += ",\"topics\":[";
        for (uint32_t q = 0; q < p.n_topics; q++) { if (q) o.push_back(','); hex0x(o, r.data_blob + p.topics_off + 32 * q, 32); }
        o += "],\"data\":"; hex0x(o, r.data_blob + p.data_off, p.data_len);
        o += "}}";
    }
}
void storage_proofs_json(std::string& o, const ipcfp_tipset_desc& t, const ipcfp_storage_result& s) {   // StorageProof items (storage/bundle.rs:5-14)
    for (uint64_t i = 0; i < s.n_proofs; i++) {
        const ipcfp_storage_proof& p = s.proofs[i];
        if (i) o.push_back(',');
        o += "{\"child_epoch\":"; snum(o, t.child_epoch);
        o += ",\"child_block_cid\":"; cid_string(o, t.child_cid);
        o += ",\"parent_state_root\":"; cid_string(o, t.child_parent_state_root);
        o += ",\"actor_id\":"; num(o, p.actor_id);
        o += ",\"actor_state_cid\":"; cid_string(o, p.actor_state_cid);
        o += ",\"storage_root\":"; cid_string(o, p.storage_root);
        o += ",\"slot\":"; hex0x(o, p.slot, 32);
        o += ",\"value\":"; hex0x(o, p.value, 32);
        o.push_back('}');
    }
}
char* dup_out(const std::string& s, uint64_t* len) {
    char* p = (char*)malloc(s.size() + 1);
    if (!p) return nullptr;
    memcpy(p, s.data(), s.size());
    p[s.size()] = 0;
    if (len) *len = s.size();
    return p;
}

}  // namespace

extern "C" {

ipcfp_status ipcfp_bundle_to_json(const ipcfp_bundle* b, const ipcfp_tipset_desc* t, char** out, uint64_t* out_len) {
    if (!b || !t || !out || !t->child_cid || (t->n_parents && !t->parent_cids) || (b->storage && !t->child_parent_state_root)) return IPCFP_ERR_INVALID_ARG;
    std::string o;
    o.reserve(64 + b->witness.blob_size * 4 / 3 + b->witness.n_blocks * 200);
    o += "{\"storage_proofs\":[";
    if (b->storage) storage_proofs_json(o, *t, *b->storage);
    o += "],\"event_proofs\":[";
    bool first = true;
    for (uint64_t k = 0; k < b->n_event_results; k++) event_proofs_json(o, *t, *b->events[k], first);
    o += "],\"blocks\":";
    blocks_json(o, b->witness);
    o.push_back('}');
    *out = dup_out(o, out_len);
    return *out ? IPCFP_OK : IPCFP_ERR_INVALID_ARG;
}
ipcfp_status ipcfp_event_result_to_json(const ipcfp_event_result* r, const ipcfp_tipset_desc* t, char** out, uint64_t* out_len) {
    if (!r || !t || !out || !t->child_cid || (t->n_parents && !t->parent_cids)) return IPCFP_ERR_INVALID_ARG;
    if (r->witness.n_blocks && !r->witness.blob) return IPCFP_ERR_INVALID_ARG;   // a by-reference witness (IPCFP_WITNESS_BY_REFERENCE) carries no bytes to render
    std::string o;
    o.reserve(64 + r->witness.blob_size * 4 / 3 + r->witness.n_blocks * 200);
    o += "{\"proofs\":[";
    bool first = true;
    event_proofs_json(o, *t, *r, first);
    o += "],\"blocks\":";
    blocks_json(o, r->witness);
    o.push_back('}');
    *out = dup_out(o, out_len);
    return *out ? IPCFP_OK : IPCFP_ERR_INVALID_ARG;
}
void ipcfp_json_free(char* p) { free(p); }
// one Filecoin.ChainReadObj request per CID of the plan, in plan order, ids first_id + k
ipcfp_status ipcfp_fetch_plan_to_rpc_json(const ipcfp_fetch_plan* p, uint64_t first_id, char** out, uint64_t* out_len) {
    if (!p || !out || (p->n_missing && !p->cids)) return IPCFP_ERR_INVALID_ARG;
    std::string o;
    o.reserve(2 + p->n_missing * 140);
    o.push_back('[');
    for (uint64_t k = 0; k < p->n_missing; k++) {
        if (k) o.push_back(',');
        o += "{\"jsonrpc\":\"2.0\",\"method\":\"Filecoin.ChainReadObj\",\"params\":[{\"/\":";
        cid_string(o, p->cids + 38 * k);
        o += "}],\"id\":";
        num(o, first_id + k);
        o.push_back('}');
    }
    o.push_back(']');
    *out = dup_out(o, out_len);
    return *out ? IPCFP_OK : IPCFP_ERR_INVALID_ARG;
}

}  // extern "C"
