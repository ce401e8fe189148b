// bundle_parse.cpp — the way back of bundle_json.cpp, in the boundary language (plain C++, built with g++, no CUDA).
//
// ipcfp_bundle_from_json reads what `serde_json::from_str::<UnifiedProofBundle>` / `::<EventProofBundle>` reads in the reference
// (src/proofs/common/bundle.rs:10-45, src/proofs/events/bundle.rs:5-30, src/proofs/storage/bundle.rs:5-14) into the PODs the
// batched verifiers take (ipcfp_verify_event_proofs / ipcfp_verify_storage_proofs) and the flat block arrays
// ipcfp_store_create takes for the witness store — so a host that holds a bundle as JSON can verify it through the C ABI alone:
//
//     ipcfp_bundle_from_json(text, len, &pb);
//     ipcfp_store_create(pb->witness.cids, pb->witness.offsets, pb->witness.lengths, pb->witness.blob, pb->witness.blob_size,
//                        pb->witness.n_blocks, device, IPCFP_STORE_VERIFY_CIDS, &ws);
//     ipcfp_verify_event_proofs(ws, &pb->tipset, pb->event_proofs, pb->n_event_proofs, pb->data_blob, pb->data_blob_size, filter, results);
//
// Accepted spellings mirror ipc_filecoin_proofs_b200/bundle_json.py: CID strings are multibase base32 ("b…"); `ProofBlock.cid` may be
// the byte array cid 0.11's Serialize emits, a {"/": "b…"} link or a plain string; hex fields carry "0x"; block data is standard
// base64 with padding. serde ignores unknown fields: so does this parser. The fields every proof of a bundle shares (epochs, parent
// tipset CIDs, child block CID, parent state root) are returned once, as an ipcfp_tipset_desc; a bundle whose proofs disagree on them
// is refused (IPCFP_ERR_UNSUPPORTED) — the C ABI's verifiers take one tipset pair per call, as the generators produce them.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/ipcfp.h"
#include "json_value.h"

namespace {

void unhex(const std::string& s, std::vector<uint8_t>& out) {
    if (s.size() < 2 || s[0] != '0' || s[1] != 'x' || (s.size() & 1)) bad();
    for (size_t i = 2; i < s.size(); i += 2) {
        auto d = [&](char c) -> uint32_t { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : 99; };
        uint32_t h = d(s[i]), l = d(s[i + 1]);
        if (h == 99 || l == 99) bad();
        out.push_back((uint8_t)(h * 16 + l));
    }
}
void cid_of_field(const JV& v, uint8_t out[IPCFP_CID_LEN]) {   // ProofBlock.cid: byte array | {"/": "b…"} | "b…"
    if (v.t == JV::ARR) {
        if (v.a.size() != IPCFP_CID_LEN) bad(IPCFP_ERR_UNSUPPORTED);
        for (int k = 0; k < IPCFP_CID_LEN; k++) { uint64_t x = u64_of(v.a[k]); if (x > 255) bad(); out[k] = (uint8_t)x; }
        return;
    }
    if (v.t == JV::OBJ) { cid_of_string(need(v, "/", JV::STR).s, out); return; }
    if (v.t == JV::STR) { cid_of_string(v.s, out); return; }
    bad();
}
struct Parsed {
    ipcfp_parsed_bundle pub;   // FIRST member: the handle is a pointer to it
    std::vector<uint8_t> parent_cids, child_cid, state_root;
    std::vector<ipcfp_storage_proof> sp;
    std::vector<ipcfp_event_proof> ep;
    std::vector<uint8_t> data_blob;
    std::vector<uint8_t> w_cids, w_blob;
    std::vector<uint64_t> w_offs;
    std::vector<uint32_t> w_lens;
    bool have_event_tipset = false, have_child = false, have_state_root = false;
    int64_t parent_epoch = 0, child_epoch = 0;
    bool have_child_epoch = false;
};

void same_or_set(std::vector<uint8_t>& have, bool& flag, const uint8_t* cid) {
    if (!flag) { have.assign(cid, cid + IPCFP_CID_LEN); flag = true; return; }
    if (memcmp(have.data(), cid, IPCFP_CID_LEN)) bad(IPCFP_ERR_UNSUPPORTED);
}
void child_epoch_is(Parsed& P, int64_t v) {
    if (!P.have_child_epoch) { P.child_epoch = v; P.have_child_epoch = true; return; }
    if (P.child_epoch != v) bad(IPCFP_ERR_UNSUPPORTED);
}

void read_event_proofs(Parsed& P, const JV& arr) {
    for (const JV& it : arr.a) {
        if (it.t != JV::OBJ) bad();
        const int64_t pe = i64_of(need(it, "parent_epoch", JV::NUM));
        child_epoch_is(P, i64_of(need(it, "child_epoch", JV::NUM)));
        const JV& ptc = need(it, "parent_tipset_cids", JV::ARR);
        std::vector<uint8_t> parents(ptc.a.size() * IPCFP_CID_LEN);
        for (size_t q = 0; q < ptc.a.size(); q++) { if (ptc.a[q].t != JV::STR) bad(); cid_of_string(ptc.a[q].s, parents.data() + IPCFP_CID_LEN * q); }
        if (!P.have_event_tipset) { P.parent_epoch = pe; P.parent_cids = parents; P.have_event_tipset = true; }
        else if (P.parent_epoch != pe || P.parent_cids != parents) bad(IPCFP_ERR_UNSUPPORTED);
        uint8_t c[IPCFP_CID_LEN];
        cid_of_string(need(it, "child_block_cid", JV::STR).s, c);
        same_or_set(P.child_cid, P.have_child, c);
        ipcfp_event_proof r;
        memset(&r, 0, sizeof r);
        cid_of_string(need(it, "message_cid", JV::STR).s, r.message_cid);
        r.exec_index = u64_of(need(it, "exec_index", JV::NUM));
        r.event_index = u64_of(need(it, "event_index", JV::NUM));
        const JV& ed = need(it, "event_data", JV::OBJ);
        r.emitter = u64_of(need(ed, "emitter", JV::NUM));
        const JV& tp = need(ed, "topics", JV::ARR);
        r.topics_off = P.data_blob.size();
        for (const JV& t : tp.a) {
            if (t.t != JV::STR) bad();
            const size_t before = P.data_blob.size();
            unhex(t.s, P.data_blob);
            if (P.data_blob.size() - before != 32) bad(IPCFP_ERR_UNSUPPORTED);   // the POD carries 32-byte topics (what the generator emits)
        }
        if (tp.a.size() > UINT32_MAX) bad();
        r.n_topics = (uint32_t)tp.a.size();
        r.data_off = P.data_blob.size();
        unhex(need(ed, "data", JV::STR).s, P.data_blob);
        const uint64_t dl = P.data_blob.size() - r.data_off;
        if (dl > UINT32_MAX) bad(IPCFP_ERR_UNSUPPORTED);
        r.data_len = (uint32_t)dl;
        P.ep.push_back(r);
    }
}
void read_storage_proofs(Parsed& P, const JV& arr) {
    for (const JV& it : arr.a) {
        if (it.t != JV::OBJ) bad();
        child_epoch_is(P, i64_of(need(it, "child_epoch", JV::NUM)));
        uint8_t c[IPCFP_CID_LEN];
        cid_of_string(need(it, "child_block_cid", JV::STR).s, c);
        same_or_set(P.child_cid, P.have_child, c);
        cid_of_string(need(it, "parent_state_root", JV::STR).s, c);
        same_or_set(P.state_root, P.have_state_root, c);
        ipcfp_storage_proof r;
        memset(&r, 0, sizeof r);
        r.actor_id = u64_of(need(it, "actor_id", JV::NUM));
        cid_of_string(need(it, "actor_state_cid", JV::STR).s, r.actor_state_cid);
        cid_of_string(need(it, "storage_root", JV::STR).s, r.storage_root);
        std::vector<uint8_t> b;
        unhex(need(it, "slot", JV::STR).s, b);
        if (b.size() != 32) bad();
        memcpy(r.slot, b.data(), 32);
        b.clear();
        unhex(need(it, "value", JV::STR).s, b);
        if (b.size() != 32) bad();
        memcpy(r.value, b.data(), 32);
        r.found = 1;       // the wire format carries the padded value only (storage/bundle.rs:5-14)
        r.raw_len = 32;
        P.sp.push_back(r);
    }
}
void read_blocks(Parsed& P, const JV& arr) {
    for (const JV& it : arr.a) {
        if (it.t != JV::OBJ) bad();
        const JV* c = it.get("cid");
        if (!c) bad();
        uint8_t cid[IPCFP_CID_LEN];
        cid_of_field(*c, cid);
        P.w_cids.insert(P.w_cids.end(), cid, cid + IPCFP_CID_LEN);
        const size_t off = P.w_blob.size();
        unbase64(need(it, "data", JV::STR).s, P.w_blob);
        const size_t len = P.w_blob.size() - off;
        if (len > UINT32_MAX) bad(IPCFP_ERR_UNSUPPORTED);
        P.w_offs.push_back(off);
        P.w_lens.push_back((uint32_t)len);
        while (P.w_blob.size() & 15) P.w_blob.push_back(0);   // 16-byte aligned blocks: the store's fast copy path
    }
}

}  // namespace

extern "C" {

ipcfp_status ipcfp_bundle_from_json(const char* json, uint64_t len, ipcfp_parsed_bundle** out) {
    if (!json || !out) return IPCFP_ERR_INVALID_ARG;
    *out = nullptr;
    try {
        Parser ps{json, json + len};
        JV root;
        if (!ps.value(root, 0)) return IPCFP_ERR_INVALID_ARG;
        ps.ws();
        if (ps.p != ps.e || root.t != JV::OBJ) return IPCFP_ERR_INVALID_ARG;   // trailing characters: serde_json refuses them too
        std::unique_ptr<Parsed> P(new Parsed());
        if (root.get("proofs")) read_event_proofs(*P, need(root, "proofs", JV::ARR));                       // EventProofBundle
        else {                                                                                              // UnifiedProofBundle
            read_storage_proofs(*P, need(root, "storage_proofs", JV::ARR));
            read_event_proofs(*P, need(root, "event_proofs", JV::ARR));
        }
        read_blocks(*P, need(root, "blocks", JV::ARR));
        P->w_blob.resize(P->w_blob.size() + 64, 0);
        P->data_blob.resize(P->data_blob.size() + 16, 0);
        ipcfp_parsed_bundle& b = P->pub;
        memset(&b, 0, sizeof b);
        b.tipset.parent_epoch = P->parent_epoch;
        b.tipset.child_epoch = P->child_epoch;
        b.tipset.n_parents = (uint32_t)(P->parent_cids.size() / IPCFP_CID_LEN);
        b.tipset.parent_cids = P->parent_cids.empty() ? nullptr : P->parent_cids.data();
        b.tipset.child_cid = P->have_child ? P->child_cid.data() : nullptr;
        b.tipset.child_parent_state_root = P->have_state_root ? P->state_root.data() : nullptr;
        b.n_storage_proofs = P->sp.size(); b.storage_proofs = P->sp.data();
        b.n_event_proofs = P->ep.size(); b.event_proofs = P->ep.data();
        b.data_blob = P->data_blob.data(); b.data_blob_size = P->data_blob.size() - 16;
        b.witness.n_blocks = P->w_lens.size();
        b.witness.cids = P->w_cids.data(); b.witness.offsets = P->w_offs.data(); b.witness.lengths = P->w_lens.data();
        b.witness.blob = P->w_blob.data(); b.witness.blob_size = P->w_blob.size() - 64;
        *out = &P.release()->pub;
        return IPCFP_OK;
    } catch (const Fail& f) {
        return f.st;
    } catch (const std::bad_alloc&) {
        return IPCFP_ERR_INVALID_ARG;
    }
}
void ipcfp_parsed_bundle_free(ipcfp_parsed_bundle* b) { delete reinterpret_cast<Parsed*>(b); }

}  // extern "C"
