// rpc_parse.cpp — ipcfp_tipset_desc_from_json: the tipset descriptor from the Lotus JSON-RPC results, in the boundary language (plain C++,
// built with g++, no CUDA).
//
// What `serde_json::from_str::<ApiTipset>` (parent, child) and `::<Vec<ApiReceipt>>` (receipts) read in the reference
// (src/client/types.rs:11-58), turned into an ipcfp_tipset_desc as extract_child_info, collect_base_witness and find_matching_events do
// (src/proofs/events/generator.rs:112-145, :199-211). This parser defines the semantics; the device receipt-list parser of
// ipcfp_tipset_upload_json (csrc/rpc_json.cu) accepts a subset of its texts and must give the same arrays on them.
//
// serde's derive, restated: a struct is a JSON object whose known keys (PascalCase, compared after unescaping) are read in text order,
// a repeated known key is an error, unknown keys are skipped, required fields must be present, Option fields may be missing or null.
// The receipt list is read element by element, so a fault inside element i is reported with index i.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/ipcfp.h"
#include "json_value.h"

namespace ipcfp { void set_last_error(const std::string& msg, uint64_t index); }   // capi.cu

namespace {

struct AtIndex { ipcfp_status st; uint64_t index; };

// a struct position: an object; a JSON array (serde's derive would read it as the fields in order) is refused as unsupported
void struct_kind(const JV& v) {
    if (v.t == JV::ARR) bad(IPCFP_ERR_UNSUPPORTED);
    if (v.t != JV::OBJ) bad();
}
// the known keys of struct o, in text order: f(k, value) for names[k]; got[k] = its value or null
template <int N, class F> void visit_struct(const JV& o, const char* const (&names)[N], const JV* (&got)[N], F f) {
    struct_kind(o);
    for (int k = 0; k < N; k++) got[k] = nullptr;
    for (const auto& kv : o.o)
        for (int k = 0; k < N; k++) {
            if (kv.first != names[k]) continue;
            if (got[k]) bad();   // duplicate field
            got[k] = &kv.second;
            f(k, kv.second);
            break;
        }
}
template <int N> void require(const JV* const (&got)[N]) { for (int k = 0; k < N; k++) if (!got[k]) bad(); }

// serde_json gives "-0" to the visitor as a float: an i64 field refuses it
int64_t i64_field(const JV& v) {
    if (v.t == JV::NUM && v.s == "-0") bad();
    return i64_of(v);
}
// CIDMap {"/": String} (types.rs:61-65); returns the string
const std::string& cid_map(const JV& v) {
    static const char* const N[] = {"/"};
    const JV* g[1];
    visit_struct(v, N, g, [](int, const JV& x) { if (x.t != JV::STR) bad(); });
    require(g);
    return g[0]->s;
}
void cid_map_list(const JV& v) {
    if (v.t != JV::ARR) bad();
    for (const JV& c : v.a) cid_map(c);
}

// ApiTipset / ApiBlockHeader (types.rs:40-58): the structure only (the caller parses the CIDs it uses)
void read_tipset(const char* text, uint64_t len, JV& root) {
    if (!text && len) bad();
    Parser ps{text, text + len};
    if (!ps.value(root, 0)) bad();
    ps.ws();
    if (ps.p != ps.e) bad();   // trailing characters
    static const char* const T[] = {"Cids", "Blocks", "Height"};
    static const char* const B[] = {"Miner", "Parents", "ParentStateRoot", "ParentMessageReceipts", "Messages", "Height"};
    const JV* g[3];
    visit_struct(root, T, g, [](int k, const JV& v) {
        if (k == 0) cid_map_list(v);
        else if (k == 1) {
            if (v.t != JV::ARR) bad();
            for (const JV& b : v.a) {
                const JV* h[6];
                visit_struct(b, B, h, [](int j, const JV& x) {
                    if (j == 0) { if (x.t != JV::STR) bad(); }
                    else if (j == 1) cid_map_list(x);
                    else if (j == 5) i64_field(x);
                    else cid_map(x);
                });
                require(h);
            }
        } else i64_field(v);
    });
    require(g);
}
const JV& member(const JV& o, const char* k) { return *o.get(k); }   // after read_tipset: present, unique

// ApiReceipt (types.rs:11-19) → its events root (None: zero bytes, flag 0)
void read_receipt(const JV& r, uint8_t* cid, uint8_t& has) {
    static const char* const N[] = {"ExitCode", "Return", "GasUsed", "EventsRoot"};
    const JV* g[4];
    visit_struct(r, N, g, [](int k, const JV& v) {
        if (k == 0) { if (u64_of(v) > UINT32_MAX) bad(); }
        else if (k == 1) { if (v.t != JV::STR) bad(); }   // Return: a String, never decoded on this path
        else if (k == 2) u64_of(v);
        else if (v.t != JV::NUL) cid_map(v);
    });
    if (!g[0] || !g[1] || !g[2]) bad();
    has = g[3] && g[3]->t != JV::NUL;
    if (has) cid_of_string(cid_map(*g[3]), cid);   // parse_cid (events/generator.rs:210)
}
// Vec<ApiReceipt>, element by element
void read_receipts(const char* text, uint64_t len, std::vector<uint8_t>& roots, std::vector<uint8_t>& has) {
    if (!text && len) bad();
    Parser ps{text, text + len};
    ps.ws();
    if (!ps.lit("[")) bad();
    ps.ws();
    if (!ps.lit("]"))
        for (uint64_t i = 0;; i++) {
            try {
                JV v;
                if (!ps.value(v, 1)) bad();
                roots.resize(roots.size() + IPCFP_CID_LEN, 0);
                has.push_back(0);
                read_receipt(v, roots.data() + IPCFP_CID_LEN * i, has[i]);
            } catch (const Fail& f) {
                throw AtIndex{f.st, i};
            }
            ps.ws();
            if (ps.lit(",")) continue;
            if (ps.lit("]")) break;
            bad();
        }
    ps.ws();
    if (ps.p != ps.e) bad();
}

struct ParsedTipset {
    ipcfp_parsed_tipset pub;   // FIRST member: the handle is a pointer to it
    std::vector<uint8_t> parents, txmeta, roots, has;
    uint8_t child[IPCFP_CID_LEN], receipts_root[IPCFP_CID_LEN], state_root[IPCFP_CID_LEN];
};

void build(ParsedTipset& P, const char* parent, uint64_t parent_len, const char* child, uint64_t child_len, const char* receipts,
           uint64_t receipts_len) {
    ipcfp_tipset_desc& d = P.pub.desc;
    memset(&d, 0, sizeof d);
    {
        JV root;
        read_tipset(parent, parent_len, root);
        const JV& cids = member(root, "Cids");
        const JV& blocks = member(root, "Blocks");
        P.parents.resize(IPCFP_CID_LEN * cids.a.size());
        for (size_t i = 0; i < cids.a.size(); i++) cid_of_string(cid_map(cids.a[i]), P.parents.data() + IPCFP_CID_LEN * i);
        if (blocks.a.size() != cids.a.size() || cids.a.size() > UINT32_MAX) bad(IPCFP_ERR_UNSUPPORTED);
        P.txmeta.resize(IPCFP_CID_LEN * blocks.a.size());
        for (size_t i = 0; i < blocks.a.size(); i++) cid_of_string(cid_map(member(blocks.a[i], "Messages")), P.txmeta.data() + IPCFP_CID_LEN * i);
        d.parent_epoch = i64_of(member(root, "Height"));
        d.n_parents = (uint32_t)cids.a.size();
    }
    {
        JV root;
        read_tipset(child, child_len, root);
        const JV& cids = member(root, "Cids");
        const JV& blocks = member(root, "Blocks");
        if (cids.a.empty() || blocks.a.empty()) bad();   // child.cids[0] / child.blocks[0]: the reference panics
        cid_of_string(cid_map(cids.a[0]), P.child);
        cid_of_string(cid_map(member(blocks.a[0], "ParentMessageReceipts")), P.receipts_root);
        cid_of_string(cid_map(member(blocks.a[0], "ParentStateRoot")), P.state_root);
        d.child_epoch = i64_of(member(root, "Height"));
    }
    read_receipts(receipts, receipts_len, P.roots, P.has);
    d.parent_cids = P.parents.empty() ? nullptr : P.parents.data();
    d.parent_txmeta_cids = P.txmeta.empty() ? nullptr : P.txmeta.data();
    d.child_cid = P.child;
    d.receipts_root = P.receipts_root;
    d.child_parent_state_root = P.state_root;
    d.n_receipts = P.has.size();
    d.events_roots = P.roots.empty() ? nullptr : P.roots.data();
    d.has_events_root = P.has.empty() ? nullptr : P.has.data();
}

}  // namespace

extern "C" {

ipcfp_status ipcfp_tipset_desc_from_json(const char* parent, uint64_t parent_len, const char* child, uint64_t child_len, const char* receipts,
                                         uint64_t receipts_len, ipcfp_parsed_tipset** out) {
    ipcfp_status st = IPCFP_OK;
    uint64_t index = UINT64_MAX;
    if (out) *out = nullptr;
    try {
        if (!out) bad();
        std::unique_ptr<ParsedTipset> P(new ParsedTipset());
        build(*P, parent, parent_len, child, child_len, receipts, receipts_len);
        *out = &P.release()->pub;
    } catch (const Fail& f) {
        st = f.st;
    } catch (const AtIndex& f) {
        st = f.st;
        index = f.index;
    } catch (const std::bad_alloc&) {
        st = IPCFP_ERR_INVALID_ARG;
    }
    ipcfp::set_last_error(st == IPCFP_OK ? "" : index == UINT64_MAX ? "ipcfp_tipset_desc_from_json refused the tipset texts or the receipt list's framing"
                                                                    : "ipcfp_tipset_desc_from_json refused a receipt",
                          index);
    return st;
}
void ipcfp_parsed_tipset_free(ipcfp_parsed_tipset* p) { delete reinterpret_cast<ParsedTipset*>(p); }

}  // extern "C"
