// rpc_blocks_items.cuh — per-item functions of the device parser of ipcfp_store_create_rpc_json (csrc/rpc_blocks.cu): Filecoin.ChainReadObj
// responses in CANONICAL form read into the block arrays csrc/rpc_blocks_parse.cpp (ipcfp_blocks_from_rpc_json) returns. They live in a
// header so that tests/host_fuzz/emu_rpc_blocks.cu runs the very same code on the CPU against rpc_blocks_parse.cpp.
//
// The device reads ONE buffer: the caller's texts, each followed by the separator RB_SEP ('\n', a byte no canonical text holds), then
// JP_PAD zero bytes. Canonical means: every text is one element or "[" elements joined by "," "]", no whitespace, every element exactly
//   {"jsonrpc":"2.0","result":"<base64 with padding and zero unused bits>","id":<decimal, no leading zeros>}
// Any other input is refused here (the caller DEFERS to the host parser), so that "accepted here ⇒ the host parser accepts the same texts
// with the same blocks" holds by construction, by an exact cover of the buffer:
//   * a record is found by its first bytes {"jsonrpc":"2.0","result":" — a canonical element holds no other '{', so they occur at record
//     starts only — and parsed by a strict template from its start;
//   * each record OWNS its bytes, its joint after it ("," right before the next record, or "]" right before a separator) and, the first of
//     a batch, the "[" in front of it; no byte can be owned twice;
//   * the host adds up what the records own and accepts only when that is every byte of the texts but the "[]" texts (empty batches):
//     a byte nobody owns (whitespace, another member, a stray comma) makes the sum fall short.
// The ids must then be 0 … n-1, each once (the caller claims them with an atomic, and counts the records).
#pragma once
#include "json_parse_items.cuh"

namespace ipcfp {

#define RB_SEP '\n'
#define RB_HEAD_LEN 27u     // {"jsonrpc":"2.0","result":"
#define RB_MIN_RECORD 36u   // the shortest canonical element: {"jsonrpc":"2.0","result":"","id":0}

// a record starts at p (reads RB_HEAD_LEN bytes from p)
JP_FN bool rb_start_at(const char* t, uint64_t p) { return jp_same(t + p, "{\"jsonrpc\":\"2.0\",\"result\":\"", RB_HEAD_LEN); }
// the byte ends the run of base64 characters and '=' that starts at the record's data (the device looks at 32 of them per step)
JP_FN bool rb_stop_byte(char c) { return jp_b64(c) < 0 && c != '='; }

struct RbRec {
    JpBlock blk;       // the base64 characters: data_at, n_chars, pads, len
    uint64_t id;
    uint64_t owned;    // bytes of the buffer this record owns
};
// record i of the n at pos[] (ascending) in t[0, len), whose data run ends at q (the first stop byte at or after pos[i] + RB_HEAD_LEN):
// its template, its joints, its id (< n_ids). The characters before the padding are left to jp_block_char_ok.
JP_FN bool rb_record(const char* t, uint64_t len, const uint32_t* pos, uint64_t n, uint64_t i, uint64_t q, uint64_t n_ids, RbRec& r) {
    const uint64_t at = pos[i];
    JpCur c{t, at, len};
    if (!c.lit("{\"jsonrpc\":\"2.0\",\"result\":\"") || q < c.p) return false;
    r.blk.data_at = c.p;
    r.blk.n_chars = q - c.p;
    if (!jp_b64_span(t, r.blk)) return false;
    c.p = q;
    if (!c.lit("\",\"id\":") || !c.u64(r.id) || r.id >= n_ids || !c.lit("}")) return false;
    const uint64_t e = c.p;
    r.owned = e - at;
    // in front: a separator (or the buffer's start) for a text of one element; "[" at a text's start, or a comma, inside a batch
    const char before = at ? t[at - 1] : RB_SEP;
    bool batch = true;
    if (before == RB_SEP) batch = false;
    else if (before == '[' && (at == 1 || t[at - 2] == RB_SEP)) r.owned++;
    else if (before != ',') return false;   // a comma is owned by the record that ends there (or by nobody: the sum falls short)
    // behind: the separator; or, in a batch, a comma right before the next record or "]" right before the separator
    if (e >= len) return false;
    const char after = t[e];
    if (!batch) return after == RB_SEP;
    if (after == ',') { r.owned++; return i + 1 < n && pos[i + 1] == e + 1; }
    r.owned++;
    return after == ']' && e + 1 < len && t[e + 1] == RB_SEP;
}

}  // namespace ipcfp
