// rpc_blocks_parse.cpp — ipcfp_blocks_from_rpc_json: the block arrays of ipcfp_store_create from Filecoin.ChainReadObj JSON-RPC responses,
// in the boundary language (plain C++, built with g++, no CUDA).
//
// The reference reads every block with Filecoin.ChainReadObj, whose result is the block as a base64 string (src/client/blockstore.rs:20-28).
// This parser defines the semantics of include/ipcfp.h for a caller's batch of such requests (request i asks for CID i with "id": i);
// the device parser of ipcfp_store_create_rpc_json (csrc/rpc_blocks.cu) accepts a subset of its inputs and must give the same store.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/ipcfp.h"
#include "json_value.h"
#include "parsed_blocks.h"

namespace ipcfp { void set_last_error(const std::string& msg, uint64_t index); }   // capi.cu

namespace {

struct AtIndex { ipcfp_status st; uint64_t index; };

// one response as it arrived: its id, and its block in the arrival blob (or an error response)
struct Response { uint64_t id, off, len; bool error; };

// a response object: "jsonrpc":"2.0", an integer id below n, exactly one of "result" (base64) / "error"; unknown members skipped,
// no member twice
void read_response(const JV& v, uint64_t n, std::vector<uint8_t>& blob, Response& r) {
    if (v.t != JV::OBJ) bad();
    std::vector<const std::string*> keys;
    for (const auto& kv : v.o) keys.push_back(&kv.first);
    std::sort(keys.begin(), keys.end(), [](const std::string* a, const std::string* b) { return *a < *b; });
    for (size_t k = 1; k < keys.size(); k++) if (*keys[k] == *keys[k - 1]) bad();
    const JV* ver = v.get("jsonrpc");
    const JV* id = v.get("id");
    const JV* res = v.get("result");
    const JV* err = v.get("error");
    if (!ver || ver->t != JV::STR || ver->s != "2.0" || !id || !res == !err) bad();
    r.id = u64_of(*id);
    if (r.id >= n) bad();
    r.error = err != nullptr;
    r.off = blob.size();
    r.len = 0;
    if (res) {
        if (res->t != JV::STR) bad();
        unbase64(res->s, blob);
        r.len = blob.size() - r.off;
        if (r.len > UINT32_MAX) bad(IPCFP_ERR_UNSUPPORTED);   // ipcfp_store_create's lengths are u32
    }
}

// one text: a batch "[…]" or, when it does not start with '[', one response; element faults carry their position `pos`
void read_text(const char* text, uint64_t len, uint64_t n, uint64_t& pos, std::vector<uint8_t>& blob, std::vector<Response>& rs) {
    if (!text && len) bad();
    Parser ps{text, text + len};
    auto element = [&] {
        try {
            JV v;
            if (!ps.value(v, 1)) bad();
            Response r;
            read_response(v, n, blob, r);
            rs.push_back(r);
        } catch (const Fail& f) {
            throw AtIndex{f.st, pos};
        }
        pos++;
    };
    ps.ws();
    if (ps.lit("[")) {
        ps.ws();
        if (!ps.lit("]"))
            for (;;) {
                element();
                ps.ws();
                if (ps.lit(",")) continue;
                if (ps.lit("]")) break;
                bad();
            }
    } else element();
    ps.ws();
    if (ps.p != ps.e) bad();   // trailing bytes
}

using ParsedBlocks = ParsedBlocksBox;

void build(ParsedBlocks& P, const uint8_t* cids, uint64_t n, const char* const* texts, const uint64_t* lens, uint64_t n_texts) {
    if ((n && !cids) || (n_texts && (!texts || !lens))) bad();
    std::vector<uint8_t> arrived;
    std::vector<Response> rs;
    uint64_t pos = 0;
    for (uint64_t k = 0; k < n_texts; k++) read_text(texts[k], lens[k], n, pos, arrived, rs);
    // every id exactly once, then no error response: the smallest offending id
    std::vector<uint32_t> count(n, 0);
    std::vector<const Response*> by_id(n, nullptr);
    for (const Response& r : rs) { if (count[r.id] < 2) count[r.id]++; by_id[r.id] = &r; }
    for (uint64_t i = 0; i < n; i++) if (count[i] != 1) throw AtIndex{IPCFP_ERR_INVALID_ARG, i};
    for (uint64_t i = 0; i < n; i++) if (by_id[i]->error) throw AtIndex{IPCFP_ERR_MISSING_BLOCK, i};
    // request order, 16-aligned blocks (the layout of ipcfp_bundle_from_json's witness arrays)
    P.cids.assign(cids, cids + IPCFP_CID_LEN * n);
    P.offsets.resize(n);
    P.lengths.resize(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; i++) { P.offsets[i] = total; P.lengths[i] = (uint32_t)by_id[i]->len; total += (by_id[i]->len + 15) & ~15ull; }
    P.blob.assign(total + 64, 0);
    for (uint64_t i = 0; i < n; i++) if (by_id[i]->len) memcpy(P.blob.data() + P.offsets[i], arrived.data() + by_id[i]->off, by_id[i]->len);
    ipcfp_witness& w = P.pub.blocks;
    w.n_blocks = n;
    w.cids = P.cids.data();
    w.offsets = P.offsets.data();
    w.lengths = P.lengths.data();
    w.blob = P.blob.data();
    w.blob_size = total;
}

}  // namespace

extern "C" {

ipcfp_status ipcfp_blocks_from_rpc_json(const uint8_t* cids, uint64_t n_blocks, const char* const* texts, const uint64_t* text_lens, uint64_t n_texts,
                                        ipcfp_parsed_blocks** out) {
    ipcfp_status st = IPCFP_OK;
    uint64_t index = UINT64_MAX;
    if (out) *out = nullptr;
    try {
        if (!out) bad();
        std::unique_ptr<ParsedBlocks> P(new ParsedBlocks());
        build(*P, cids, n_blocks, texts, text_lens, n_texts);
        *out = &P.release()->pub;
    } catch (const Fail& f) {
        st = f.st;
    } catch (const AtIndex& f) {
        st = f.st;
        index = f.index;
    } catch (const std::bad_alloc&) {
        st = IPCFP_ERR_INVALID_ARG;
    }
    ipcfp::set_last_error(st == IPCFP_OK ? "" : st == IPCFP_ERR_MISSING_BLOCK ? "ipcfp_blocks_from_rpc_json: the node answered this request with an error"
                                              : index == UINT64_MAX ? "ipcfp_blocks_from_rpc_json refused the framing of a text"
                                                                    : "ipcfp_blocks_from_rpc_json refused a response (or an id is not there exactly once)",
                          index);
    return st;
}
void ipcfp_parsed_blocks_free(ipcfp_parsed_blocks* p) { delete reinterpret_cast<ParsedBlocks*>(p); }

}  // extern "C"
