// rpc_json_items.cuh — per-item functions of the device receipt-list parser of ipcfp_tipset_upload_json (csrc/rpc_json.cu): the CANONICAL
// text of a Vec<ApiReceipt> (src/client/types.rs:11-19) read into the events_roots / has_events_root arrays csrc/rpc_parse.cpp
// (ipcfp_tipset_desc_from_json) returns. They live in a header so that tests/host_fuzz/emu_rpc_json.cu runs the very same code on the
// CPU against rpc_parse.cpp.
//
// Canonical means: no whitespace, every element exactly
//   {"ExitCode":<u32>,"Return":"<base64 characters and '='>","GasUsed":<u64>,"EventsRoot":null}
//   {"ExitCode":<u32>,"Return":"<base64 characters and '='>","GasUsed":<u64>,"EventsRoot":{"/":"b<61 base32 characters>"}}
// with integers without leading zeros, the CID string's one unused bit zero, the elements joined by single commas inside "[" … "]".
// Any other text is refused here (the caller DEFERS to the host parser), so that "accepted here ⇒ the host parser accepts the same text
// with the same values" holds by construction: every byte of an accepted text is consumed by exactly one template check —
//   * a record is found by its first bytes {"ExitCode": — a canonical string holds no '{' or '"', so they occur at record starts only;
//   * each record is parsed by a strict template from its start, and must end exactly one comma before the next record starts;
//   * the first record starts right after the opening "[" and the last one ends right before the closing "]", the text's last byte.
// The record's values are then the host parser's: the keys are the struct's, each once; ExitCode ≤ u32, GasUsed ≤ u64; Return is a
// string (never decoded); the CID string decodes to 38 bytes with the rule of cid_of_string.
//
// Every buffer these functions read holds the text followed by JP_PAD zero bytes (rj_start_at looks 12 bytes ahead).
#pragma once
#include "json_parse_items.cuh"

namespace ipcfp {

#define RJ_MIN_RECORD 57u   // the shortest canonical record with its comma: {"ExitCode":0,"Return":"","GasUsed":0,"EventsRoot":null},
#define RJ_HEAD_LEN 12u     // {"ExitCode":

// a record starts at p
JP_FN bool rj_start_at(const char* t, uint64_t p) { return jp_same(t + p, "{\"ExitCode\":", RJ_HEAD_LEN); }
// a byte no canonical text holds: whitespace, controls, escapes, non-ASCII (the device marks these to defer early)
JP_FN bool rj_foreign_byte(char c) { return (unsigned char)c <= 0x20 || (unsigned char)c >= 0x7f || c == '\\'; }
JP_FN bool rj_b64_or_pad(char c) { return jp_b64(c) >= 0 || c == '='; }

// record i of the n starts at pos[] (ascending) in t[0, len): its template and its joints. cid (38 bytes) / has receive its events root.
JP_FN bool rj_record(const char* t, uint64_t len, const uint32_t* pos, uint64_t n, uint64_t i, uint8_t* cid, uint8_t& has) {
    const uint64_t at = pos[i];
    if (i == 0 && at != 1) return false;   // right after the opening bracket (t[0] == '[' is checked on the host)
    const uint64_t e = i + 1 < n ? (uint64_t)pos[i + 1] : len;
    JpCur c{t, at, e};
    uint64_t v;
    if (!c.lit("{\"ExitCode\":") || !c.u64(v) || v > 0xffffffffull || !c.lit(",\"Return\":\"")) return false;
    while (c.p < e && rj_b64_or_pad(t[c.p])) c.p++;
    if (!c.lit("\",\"GasUsed\":") || !c.u64(v) || !c.lit(",\"EventsRoot\":")) return false;
    has = 0;
    if (c.lit("null")) {
        for (int k = 0; k < IPCFP_CID_LEN; k++) cid[k] = 0;
    } else {
        if (!c.lit("{\"/\":") || !c.cid(cid) || !c.lit("}")) return false;
        has = 1;
    }
    if (!c.lit("}")) return false;
    // the joint: one comma, then the next record; the last record ends right before the closing bracket, the text's last byte
    if (i + 1 < n) return c.lit(",") && c.p == e;
    return c.p + 1 == len;
}

}  // namespace ipcfp
