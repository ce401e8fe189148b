// json_items.cuh — per-item device functions of the EventProofBundle JSON renderer (IPCFP_RESULT_JSON, csrc/json.cu): the exact length
// and the text of one EventProof record and of one ProofBlock record, byte for byte what csrc/bundle_json.cpp writes
// (ipcfp_event_result_to_json; serde_json of src/proofs/events/bundle.rs:5-30, src/proofs/common/bundle.rs:10-26). They live in a header
// so that tests/host_fuzz/emu_json.cu runs the very same code on the CPU against bundle_json.cpp. The StorageProof record and the
// UnifiedProofBundle framing (ipcfp_generate_proof_bundle_resident with IPCFP_RESULT_JSON) are checked the same way by
// tests/host_fuzz/emu_json_unified.cu against ipcfp_bundle_to_json.
//
// The bundle is laid out as
//   {"proofs":  S P0  S P1 …  ],"blocks":  S B0  S B1 …  ]}
// where every record carries one separator byte S in front of it: '[' for the first record of its list (exclusive offset 0), ',' for the
// others. An empty list is the single '[' the framing writes. Offsets are exclusive scans of the per-item lengths (separator included),
// so every item is written independently of the others.
#pragma once
#include "common.cuh"

namespace ipcfp {

#define JSON_PROOFS_HEAD 10u   // {"proofs":
#define JSON_BLOCKS_HEAD 10u   // ,"blocks":

__device__ __forceinline__ uint32_t json_dec_len(uint64_t v) {
    uint32_t n = 1;
    while (v >= 10) { v /= 10; n++; }
    return n;
}
// decimal digits of v at o (json_dec_len(v) bytes)
__device__ __forceinline__ void json_dec_write(char* o, uint64_t v) {
    uint32_t n = json_dec_len(v);
    do { o[--n] = (char)('0' + v % 10); v /= 10; } while (n);
}
// |v| of an i64 as u64 (INT64_MIN included)
__device__ __forceinline__ uint64_t json_abs64(int64_t v) { return v < 0 ? 0ull - (uint64_t)v : (uint64_t)v; }

// `Cid::to_string()` of a 38-byte CIDv1 with its quotes: "b" + 61 base32 characters (RFC 4648 lower case, no padding)
#define JSON_CID_STR_LEN 64u
__device__ __forceinline__ void json_cid_str_write(char* o, const uint8_t* c) {
    const char* B32 = "abcdefghijklmnopqrstuvwxyz234567";
    uint32_t k = 0;
    o[k++] = '"';
    o[k++] = 'b';
    uint32_t acc = 0;
    int bits = 0;
    for (int i = 0; i < IPCFP_CID_LEN; i++) {
        acc = (acc << 8) | c[i];
        bits += 8;
        while (bits >= 5) { o[k++] = B32[(acc >> (bits - 5)) & 31]; bits -= 5; }
    }
    if (bits) o[k++] = B32[(acc << (5 - bits)) & 31];
    o[k] = '"';
}

// Output sinks: one renderer, run once to count (JsonCount) and once to write (JsonWrite), so that a record's length and its text
// cannot disagree.
struct JsonCount {
    uint64_t n = 0;
    template <int N> __device__ __forceinline__ void lit(const char (&)[N]) { n += N - 1; }
    __device__ __forceinline__ void ch(char) { n++; }
    __device__ __forceinline__ void u64(uint64_t v) { n += json_dec_len(v); }
    __device__ __forceinline__ void i64(int64_t v) { n += (v < 0) + json_dec_len(json_abs64(v)); }
    __device__ __forceinline__ void cid_str(const uint8_t*) { n += JSON_CID_STR_LEN; }
    __device__ __forceinline__ void hex0x(const uint8_t*, uint64_t len) { n += 4 + 2 * len; }
};
struct JsonWrite {
    char* o;
    template <int N> __device__ __forceinline__ void lit(const char (&s)[N]) { for (int i = 0; i < N - 1; i++) o[i] = s[i]; o += N - 1; }
    __device__ __forceinline__ void ch(char c) { *o++ = c; }
    __device__ __forceinline__ void u64(uint64_t v) { json_dec_write(o, v); o += json_dec_len(v); }
    __device__ __forceinline__ void i64(int64_t v) { if (v < 0) *o++ = '-'; u64(json_abs64(v)); }
    __device__ __forceinline__ void cid_str(const uint8_t* c) { json_cid_str_write(o, c); o += JSON_CID_STR_LEN; }
    __device__ __forceinline__ void hex0x(const uint8_t* p, uint64_t len) {   // "0x" + lower-case hex
        const char* H = "0123456789abcdef";
        *o++ = '"'; *o++ = '0'; *o++ = 'x';
        for (uint64_t i = 0; i < len; i++) { o[2 * i] = H[p[i] >> 4]; o[2 * i + 1] = H[p[i] & 15]; }
        o += 2 * len;
        *o++ = '"';
    }
};

// what every EventProof of one call shares (the tipset descriptor)
struct JsonProofCtx {
    int64_t parent_epoch, child_epoch;
    uint32_t n_parents;
    const uint8_t* parent_cids;   // n_parents*38
    const uint8_t* child_cid;     // 38
};

// Pass 2 reserves a slot for every event of a matching receipt; the slots of a receipt the receipts AMT does not hold stay
// exec_index == UINT64_MAX (events/generator.rs:249-251 `continue`) and are not part of the bundle.
__device__ __forceinline__ bool json_proof_kept(const ipcfp_event_proof& p) { return p.exec_index != UINT64_MAX; }

// one EventProof (events/bundle.rs:14-23), field order and spelling as bundle_json.cpp::event_proofs_json
template <class S> __device__ __forceinline__ void json_proof_record(S& s, const JsonProofCtx& c, const ipcfp_event_proof& p, const uint8_t* blob) {
    s.lit("{\"parent_epoch\":"); s.i64(c.parent_epoch);
    s.lit(",\"child_epoch\":"); s.i64(c.child_epoch);
    s.lit(",\"parent_tipset_cids\":[");
    for (uint32_t q = 0; q < c.n_parents; q++) { if (q) s.ch(','); s.cid_str(c.parent_cids + 38ull * q); }
    s.lit("],\"child_block_cid\":"); s.cid_str(c.child_cid);
    s.lit(",\"message_cid\":"); s.cid_str(p.message_cid);
    s.lit(",\"exec_index\":"); s.u64(p.exec_index);
    s.lit(",\"event_index\":"); s.u64(p.event_index);
    s.lit(",\"event_data\":{\"emitter\":"); s.u64(p.emitter);
    s.lit(",\"topics\":[");
    for (uint32_t q = 0; q < p.n_topics; q++) { if (q) s.ch(','); s.hex0x(blob + p.topics_off + 32ull * q, 32); }
    s.lit("],\"data\":"); s.hex0x(blob + p.data_off, p.data_len);
    s.lit("}}");
}
// length of proof slot k in the proofs list, separator included (0 for a skipped slot)
__device__ __forceinline__ uint64_t json_proof_len(const JsonProofCtx& c, const ipcfp_event_proof& p, const uint8_t* blob) {
    if (!json_proof_kept(p)) return 0;
    JsonCount n;
    json_proof_record(n, c, p, blob);
    return 1 + n.n;
}
// separator + record at o (o = the slot's place: list start + its exclusive offset); first = its exclusive offset is 0
__device__ __forceinline__ void json_proof_write(char* o, bool first, const JsonProofCtx& c, const ipcfp_event_proof& p, const uint8_t* blob) {
    JsonWrite w{o};
    w.ch(first ? '[' : ',');
    json_proof_record(w, c, p, blob);
}

// ---- one ProofBlock {"cid":[d,…,d],"data":"<standard base64, padded>"} (common/bundle.rs:11-26)
#define JSON_BLOCK_CID_HEAD 8u    // {"cid":[
#define JSON_BLOCK_DATA_HEAD 10u  // ],"data":"
__device__ __forceinline__ uint32_t json_cid_array_len(const uint8_t* cid) {   // 38 decimal numbers and 37 commas
    uint32_t n = IPCFP_CID_LEN - 1;
    for (int k = 0; k < IPCFP_CID_LEN; k++) n += json_dec_len(cid[k]);
    return n;
}
__device__ __forceinline__ uint64_t json_base64_len(uint32_t len) { return 4ull * ((len + 2ull) / 3); }
// separator included
__device__ __forceinline__ uint64_t json_block_len(const uint8_t* cid, uint32_t len) {
    return 1 + JSON_BLOCK_CID_HEAD + json_cid_array_len(cid) + JSON_BLOCK_DATA_HEAD + json_base64_len(len) + 2;
}
// Lane `lane` of `nl` cooperating lanes writes its share of the record at o: CID byte k and base64 group g belong to lane k % nl and
// g % nl. No lane reads what another writes, so the lanes may run in any order (the kernel: one warp per block, nl = 32). src: the
// block's len bytes at any alignment; no byte outside them is read.
__device__ __forceinline__ void json_block_write(char* o, bool first, const uint8_t* cid, const uint8_t* src, uint32_t len, uint32_t lane, uint32_t nl) {
    const char* T = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    if (lane == 0) { JsonWrite w{o}; w.ch(first ? '[' : ','); w.lit("{\"cid\":["); }
    char* c = o + 1 + JSON_BLOCK_CID_HEAD;
    for (uint32_t k = lane; k < IPCFP_CID_LEN; k += nl) {
        uint32_t at = 0;
        for (uint32_t j = 0; j < k; j++) at += json_dec_len(cid[j]) + 1;
        json_dec_write(c + at, cid[k]);
        if (k + 1 < IPCFP_CID_LEN) c[at + json_dec_len(cid[k])] = ',';
    }
    char* d = c + json_cid_array_len(cid);
    if (lane == 0) { JsonWrite w{d}; w.lit("],\"data\":\""); }
    d += JSON_BLOCK_DATA_HEAD;
    const uint32_t ng = (len + 2) / 3;
    for (uint32_t g = lane; g < ng; g += nl) {
        const uint32_t i = 3 * g, rem = len - i;
        const uint32_t v = ((uint32_t)src[i] << 16) | (rem > 1 ? (uint32_t)src[i + 1] << 8 : 0u) | (rem > 2 ? (uint32_t)src[i + 2] : 0u);
        char* q = d + 4 * g;
        q[0] = T[v >> 18];
        q[1] = T[(v >> 12) & 63];
        q[2] = rem > 1 ? T[(v >> 6) & 63] : '=';
        q[3] = rem > 2 ? T[v & 63] : '=';
    }
    if (lane == 0) { char* e = d + 4ull * ng; e[0] = '"'; e[1] = '}'; }
}

// ---- one StorageProof (storage/bundle.rs:5-14) of a UnifiedProofBundle, field order and spelling as bundle_json.cpp::storage_proofs_json
struct JsonStorageCtx {
    int64_t child_epoch;
    const uint8_t* child_cid;    // 38
    const uint8_t* state_root;   // 38: the child header's parent_state_root
};
template <class S> __device__ __forceinline__ void json_storage_record(S& s, const JsonStorageCtx& c, const ipcfp_storage_proof& p) {
    s.lit("{\"child_epoch\":"); s.i64(c.child_epoch);
    s.lit(",\"child_block_cid\":"); s.cid_str(c.child_cid);
    s.lit(",\"parent_state_root\":"); s.cid_str(c.state_root);
    s.lit(",\"actor_id\":"); s.u64(p.actor_id);
    s.lit(",\"actor_state_cid\":"); s.cid_str(p.actor_state_cid);
    s.lit(",\"storage_root\":"); s.cid_str(p.storage_root);
    s.lit(",\"slot\":"); s.hex0x(p.slot, 32);
    s.lit(",\"value\":"); s.hex0x(p.value, 32);
    s.ch('}');
}
// separator included
__device__ __forceinline__ uint64_t json_storage_len(const JsonStorageCtx& c, const ipcfp_storage_proof& p) {
    JsonCount n;
    json_storage_record(n, c, p);
    return 1 + n.n;
}
__device__ __forceinline__ void json_storage_write(char* o, bool first, const JsonStorageCtx& c, const ipcfp_storage_proof& p) {
    JsonWrite w{o};
    w.ch(first ? '[' : ',');
    json_storage_record(w, c, p);
}

// ---- framing. P, Q: summed lengths of the proof and block lists (separators included). Total length of the bundle:
__host__ __device__ __forceinline__ uint64_t json_total_len(uint64_t P, uint64_t Q) {
    return JSON_PROOFS_HEAD + (P ? P : 1) + 1 + JSON_BLOCKS_HEAD + (Q ? Q : 1) + 2;
}
__host__ __device__ __forceinline__ uint64_t json_blocks_at(uint64_t P) { return JSON_PROOFS_HEAD + (P ? P : 1) + 1 + JSON_BLOCKS_HEAD; }
// everything of the text that is not a record (one thread)
__device__ __forceinline__ void json_frame_write(char* o, uint64_t P, uint64_t Q) {
    JsonWrite w{o};
    w.lit("{\"proofs\":");
    if (!P) w.ch('[');
    w.o = o + JSON_PROOFS_HEAD + (P ? P : 1);
    w.lit("],\"blocks\":");
    if (!Q) w.ch('[');
    w.o = o + json_blocks_at(P) + (Q ? Q : 1);
    w.lit("]}");
}

// ---- UnifiedProofBundle framing (common/bundle.rs:37-45): {"storage_proofs": S ,"event_proofs": P ,"blocks": Q }, each list laid out as
// above. S, P, Q: summed lengths of the three lists (separators included).
#define JSON_STORAGE_HEAD 18u   // {"storage_proofs":
#define JSON_EVENTS_HEAD 16u    // ,"event_proofs":
__host__ __device__ __forceinline__ uint64_t json_u_events_at(uint64_t S) { return JSON_STORAGE_HEAD + (S ? S : 1) + 1 + JSON_EVENTS_HEAD; }
__host__ __device__ __forceinline__ uint64_t json_u_blocks_at(uint64_t S, uint64_t P) { return json_u_events_at(S) + (P ? P : 1) + 1 + JSON_BLOCKS_HEAD; }
__host__ __device__ __forceinline__ uint64_t json_u_total_len(uint64_t S, uint64_t P, uint64_t Q) { return json_u_blocks_at(S, P) + (Q ? Q : 1) + 2; }
// everything of the text that is not a record (one thread)
__device__ __forceinline__ void json_u_frame_write(char* o, uint64_t S, uint64_t P, uint64_t Q) {
    JsonWrite w{o};
    w.lit("{\"storage_proofs\":");
    if (!S) w.ch('[');
    w.o = o + JSON_STORAGE_HEAD + (S ? S : 1);
    w.lit("],\"event_proofs\":");
    if (!P) w.ch('[');
    w.o = o + json_u_events_at(S) + (P ? P : 1);
    w.lit("],\"blocks\":");
    if (!Q) w.ch('[');
    w.o = o + json_u_blocks_at(S, P) + (Q ? Q : 1);
    w.lit("]}");
}

}  // namespace ipcfp
