// ipcfp.hpp — the HOST SIDE above the C ABI, in C++17, with the reference's own names.
//
// The reference is a Rust crate and this image has no Rust toolchain, so the host side that a Rust maintainer gets from
// integration/rust/gpu.rs exists here a second time in a language this image compiles: a header-only mirror of the reference's
// operator interface for the hot path — same type names, same field names, same argument meaning, same error behaviour — over
// nothing but the C ABI of include/ipcfp.h. A test that reads like the reference's own tests would is tests/cpp/host_mirror_test.cpp.
//
//   reference (Rust)                                              this header (namespace ipcfp::host)
//   ------------------------------------------------------------  ------------------------------------------------------------
//   cid::Cid, Cid::try_from(&str), to_string(), Ord               Cid, Cid::try_from, to_string, operator<      (common/witness.rs:60-63)
//   ApiTipset / ApiBlockHeader / ApiReceipt / CIDMap               same names and fields                          (client/types.rs:13-58)
//   ProofBlock, EventData, EventProof, EventProofBundle            same                                           (common/bundle.rs:11-18, events/bundle.rs:5-30)
//   StorageProof, UnifiedProofBundle                               same                                           (storage/bundle.rs:5-14, common/bundle.rs:38-45)
//   StorageProofSpec, EventProofSpec                               same                                           (proofs/generator.rs:12-22)
//   RpcBlockstore / CachedBlockstore: Blockstore                   GpuBlockstore: get / has / put_keyed           (client/blockstore.rs:20-37)
//   generate_event_proof(client, &store, parent, child, sig, t1, filter)   generate_event_proof(store, parent, child, receipts, sig, t1, filter)
//                                                                  — `receipts` is what the reference fetches with client.chain_get_parent_receipts (events/generator.rs:199-204)
//   generate_storage_proof(&store, parent, child, actor_id, slot)  same                                           (storage/generator.rs:29-67)
//   (README "Storage Slot Calculation": values in Solidity structures)  StoragePath, generate_storage_path_proofs, plan_fetch_storage_paths,
//                                                                  verify_storage_paths                           (storage/utils.rs:5-19)
//   read_storage_slot(&store, &root, &slot)                        same                                           (storage/decode.rs:36-97)
//   generate_proof_bundle(client, parent, child, sspecs, especs)   generate_proof_bundle(store, parent, child, receipts, sspecs, especs)   (proofs/generator.rs:25-95)
//   verify_event_proof(&bundle, &trusted_ts, &trusted_child, check_event)  same; check_event is an EventProofSpec (create_event_filter, events/verifier.rs:28-41)
//   verify_storage_proof(&proof, &blocks, &trusted_child)          same                                           (storage/verifier.rs:24-63)
//   compute_mapping_slot / calculate_storage_slot / ascii_to_bytes32 / left_pad_32   same                         (storage/utils.rs:5-19, common/evm.rs:72-100)
//   keccak256 / hash_event_signature / create_event_filter / parse_cid / parse_cids  same                         (common/evm.rs:62-88, events/verifier.rs:28-41, common/witness.rs:60-72)
//   resolve_eth_address_to_actor_id(client, eth_addr)             resolve_eth_address_to_actor_id(store, state_root, eth_addr): the state tree
//                                                                  instead of two RPC calls; resolve_addresses batches; parse_address  (common/address.rs:8-77)
//   (future work "Parallel Generation", README.md:384)             ShardedComm, generate_event_proof_sharded → ShardedEventProof
//   serde_json::to_string(&bundle) / from_str                      to_json(bundle) / bundle_from_json(text)
//   anyhow::Error                                                  ipcfp::host::Error (status, message, index)
//
// All compute happens behind the C ABI on the GPU. There is no CPU path here either: without a CUDA device every call that
// needs one throws ipcfp::host::Error with status IPCFP_ERR_NO_DEVICE.
#ifndef IPCFP_HPP
#define IPCFP_HPP

#include <array>
#include <cctype>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <optional>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "ipcfp.h"

// Everything lives in ipcfp::host. (The library's own C++ internals are in namespace ipcfp and libipcfp.so exports them: a host
// that defined, say, its own ipcfp::Error would interpose the library's — found the hard way by tests/cpp/host_mirror_test.cpp.
// Host code must not add names to namespace ipcfp itself.)
namespace ipcfp {
namespace host {

// ------------------------------------------------------------------------------------------ errors (anyhow::Error)
struct Error : std::runtime_error {
    ipcfp_status status;
    uint64_t index;   // receipt / spec / block index the failure belongs to, or UINT64_MAX
    Error(ipcfp_status st, const std::string& msg, uint64_t idx = UINT64_MAX) : std::runtime_error(msg), status(st), index(idx) {}
};
inline void check(ipcfp_status st, const char* what) {
    if (st == IPCFP_OK) return;
    const char* m = ipcfp_last_error();
    throw Error(st, std::string(what) + ": " + (m && *m ? m : "ipcfp status " + std::to_string((int)st)), ipcfp_last_error_index());
}

// ------------------------------------------------------------------------------------------ hex ("0x…", lower case) and base32
inline std::string to_hex0x(const uint8_t* p, size_t n) {
    static const char* D = "0123456789abcdef";
    std::string s = "0x";
    s.reserve(2 + 2 * n);
    for (size_t i = 0; i < n; i++) { s.push_back(D[p[i] >> 4]); s.push_back(D[p[i] & 15]); }
    return s;
}
inline std::vector<uint8_t> from_hex0x(const std::string& s) {   // hex::decode(s.trim_start_matches("0x"))
    size_t b = 0;
    while (s.compare(b, 2, "0x") == 0) b += 2;
    if ((s.size() - b) % 2) throw Error(IPCFP_ERR_INVALID_ARG, "odd number of hex digits");
    std::vector<uint8_t> out((s.size() - b) / 2);
    auto nib = [](char c) -> int { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
    for (size_t i = 0; i < out.size(); i++) {
        int h = nib(s[b + 2 * i]), l = nib(s[b + 2 * i + 1]);
        if (h < 0 || l < 0) throw Error(IPCFP_ERR_INVALID_ARG, "invalid hex digit");
        out[i] = (uint8_t)(h << 4 | l);
    }
    return out;
}
inline std::array<uint8_t, 32> from_hex32(const std::string& s) {
    auto v = from_hex0x(s);
    if (v.size() != 32) throw Error(IPCFP_ERR_INVALID_ARG, "expected 32 bytes of hex");
    std::array<uint8_t, 32> a;
    memcpy(a.data(), v.data(), 32);
    return a;
}

// ------------------------------------------------------------------------------------------ Cid (cid 0.11; the C ABI carries 38-byte CIDv1 only)
struct Cid {
    std::array<uint8_t, IPCFP_CID_LEN> bytes{};

    static Cid from_bytes(const uint8_t* p) { Cid c; memcpy(c.bytes.data(), p, IPCFP_CID_LEN); return c; }
    // Cid::try_from(&str): multibase 'b' = RFC 4648 base32, lower case, no padding ("bafy2bzace…", 62 characters for 38 bytes)
    static Cid try_from(const std::string& s) {
        if (s.size() != 62 || s[0] != 'b') throw Error(IPCFP_ERR_INVALID_ARG, "not a base32 CIDv1 of 38 bytes: " + s);
        Cid c;
        uint32_t acc = 0;
        int bits = 0;
        size_t o = 0;
        for (size_t i = 1; i < s.size(); i++) {
            const char ch = s[i];
            int v = ch >= 'a' && ch <= 'z' ? ch - 'a' : ch >= '2' && ch <= '7' ? ch - '2' + 26 : -1;
            if (v < 0) throw Error(IPCFP_ERR_INVALID_ARG, "invalid base32 character in CID: " + s);
            acc = acc << 5 | (uint32_t)v;
            bits += 5;
            if (bits >= 8) {
                bits -= 8;
                if (o == IPCFP_CID_LEN) throw Error(IPCFP_ERR_INVALID_ARG, "CID longer than 38 bytes: " + s);
                c.bytes[o++] = (uint8_t)(acc >> bits);
                acc &= (1u << bits) - 1;
            }
        }
        if (o != IPCFP_CID_LEN || acc != 0) throw Error(IPCFP_ERR_INVALID_ARG, "CID is not 38 bytes / has non-zero trailing bits: " + s);
        if (c.bytes[0] != 0x01) throw Error(IPCFP_ERR_UNSUPPORTED, "not a CIDv1: " + s);
        return c;
    }
    std::string to_string() const {
        static const char* A = "abcdefghijklmnopqrstuvwxyz234567";
        std::string s = "b";
        uint32_t acc = 0;
        int bits = 0;
        for (uint8_t b : bytes) {
            acc = acc << 8 | b;
            bits += 8;
            while (bits >= 5) { bits -= 5; s.push_back(A[(acc >> bits) & 31]); }
            acc &= (1u << bits) - 1;
        }
        if (bits) s.push_back(A[(acc << (5 - bits)) & 31]);
        return s;
    }
    bool operator==(const Cid& o) const { return bytes == o.bytes; }
    bool operator!=(const Cid& o) const { return !(*this == o); }
    // `Ord` of cid::Cid: derived over (version, codec, hash), Multihash over (code, size, digest) — drives BTreeSet<Cid>
    // (common/blockstore.rs:10, common/witness.rs:10) and hence the order of every Vec<ProofBlock>
    bool operator<(const Cid& o) const {
        uint64_t a[4], b[4];
        size_t pa = key(a), pb = o.key(b);
        for (int i = 0; i < 4; i++) if (a[i] != b[i]) return a[i] < b[i];
        const size_t na = IPCFP_CID_LEN - pa, nb = IPCFP_CID_LEN - pb;
        int c = memcmp(bytes.data() + pa, o.bytes.data() + pb, na < nb ? na : nb);
        return c != 0 ? c < 0 : na < nb;
    }

  private:
    size_t key(uint64_t out[4]) const {   // unsigned-varint fields version, codec, multihash code, digest size; returns the digest offset
        size_t pos = 0;
        for (int f = 0; f < 4; f++) {
            uint64_t v = 0;
            for (int shift = 0; shift < 64 && pos < IPCFP_CID_LEN; shift += 7) {
                uint8_t c = bytes[pos++];
                v |= (uint64_t)(c & 0x7f) << shift;
                if (!(c & 0x80)) break;
            }
            out[f] = v;
        }
        return pos;
    }
};

// ------------------------------------------------------------------------------------------ inputs that came over RPC (client/types.rs:13-58)
struct CIDMap { std::string cid; };   // {"/": "bafy…"}
struct ApiReceipt {
    uint32_t exit_code = 0;
    std::string return_data;          // base64
    uint64_t gas_used = 0;
    std::optional<CIDMap> events_root;
};
struct ApiBlockHeader {
    std::string miner;
    std::vector<CIDMap> parents;
    CIDMap parent_state_root;
    CIDMap parent_message_receipts;
    CIDMap messages;
    int64_t height = 0;
};
struct ApiTipset {
    std::vector<CIDMap> cids;
    std::vector<ApiBlockHeader> blocks;
    int64_t height = 0;
};

// ------------------------------------------------------------------------------------------ outputs (bundle.rs)
struct ProofBlock {
    Cid cid;
    std::vector<uint8_t> data;   // raw DAG-CBOR block bytes
    bool operator==(const ProofBlock& o) const { return cid == o.cid && data == o.data; }
};
struct EventData {
    uint64_t emitter = 0;
    std::vector<std::string> topics;   // "0x…" hex
    std::string data;                  // "0x…" hex
    bool operator==(const EventData& o) const { return emitter == o.emitter && topics == o.topics && data == o.data; }
};
struct EventProof {
    int64_t parent_epoch = 0;
    int64_t child_epoch = 0;
    std::vector<std::string> parent_tipset_cids;
    std::string child_block_cid;
    std::string message_cid;
    uint64_t exec_index = 0;
    uint64_t event_index = 0;
    EventData event_data;
    bool operator==(const EventProof& o) const {
        return parent_epoch == o.parent_epoch && child_epoch == o.child_epoch && parent_tipset_cids == o.parent_tipset_cids &&
               child_block_cid == o.child_block_cid && message_cid == o.message_cid && exec_index == o.exec_index &&
               event_index == o.event_index && event_data == o.event_data;
    }
};
struct EventProofBundle {
    std::vector<EventProof> proofs;
    std::vector<ProofBlock> blocks;
};
struct StorageProof {
    int64_t child_epoch = 0;
    std::string child_block_cid;
    std::string parent_state_root;
    uint64_t actor_id = 0;
    std::string actor_state_cid;
    std::string storage_root;
    std::string slot;    // 0x… 32 bytes
    std::string value;   // 0x… 32 bytes
    bool operator==(const StorageProof& o) const {
        return child_epoch == o.child_epoch && child_block_cid == o.child_block_cid && parent_state_root == o.parent_state_root &&
               actor_id == o.actor_id && actor_state_cid == o.actor_state_cid && storage_root == o.storage_root && slot == o.slot && value == o.value;
    }
};
struct UnifiedProofBundle {
    std::vector<StorageProof> storage_proofs;
    std::vector<EventProof> event_proofs;
    std::vector<ProofBlock> blocks;
};
struct UnifiedVerificationResult {
    std::vector<bool> storage_results, event_results;
    bool all_valid() const {
        for (bool v : storage_results) if (!v) return false;
        for (bool v : event_results) if (!v) return false;
        return true;
    }
};

// ------------------------------------------------------------------------------------------ specs (proofs/generator.rs:12-22)
using H256 = std::array<uint8_t, 32>;
struct StorageProofSpec {
    uint64_t actor_id = 0;
    H256 slot{};
};
struct EventProofSpec {
    std::string event_signature;   // e.g. "NewTopDownMessage(bytes32,uint256)"
    std::string topic_1;           // ASCII, right-padded to 32 bytes by the matcher
    std::optional<uint64_t> actor_id_filter;
};
// An eth_getLogs-style log filter (ipcfp_log_filter): emitters empty = any; topics[k] empty = any value at position k; topics.size()
// is n_positions (an event needs at least that many topics).
struct LogFilter {
    std::vector<uint64_t> emitters;
    std::vector<std::vector<H256>> topics;
    // the filter a spec stands for: {[actor] or any, 2 positions, [{keccak256(sig)}, {ascii_to_bytes32(topic_1)}]} (keccak on `device`)
    static LogFilter from_spec(const EventProofSpec& spec, int device = 0);
};
inline ipcfp_log_filter log_filter_c(const LogFilter& f, std::vector<std::vector<uint8_t>>& keep) {
    ipcfp_log_filter c;
    memset(&c, 0, sizeof c);
    c.n_emitters = f.emitters.size();
    c.emitters = f.emitters.empty() ? nullptr : f.emitters.data();   // borrowed: f must outlive the call
    c.n_positions = (uint32_t)f.topics.size();
    for (size_t k = 0; k < f.topics.size() && k < 4; k++) {
        if (f.topics[k].empty()) continue;
        keep.emplace_back();
        for (const H256& v : f.topics[k]) keep.back().insert(keep.back().end(), v.begin(), v.end());
        c.n_values[k] = f.topics[k].size();
        c.values[k] = keep.back().data();
    }
    return c;
}
inline ipcfp_event_spec spec_c(const std::string& sig, const std::string& topic_1, const std::optional<uint64_t>& filter) {
    ipcfp_event_spec s;
    memset(&s, 0, sizeof s);
    s.event_signature = sig.c_str();   // borrowed: the strings must outlive the call
    s.topic_1 = topic_1.c_str();
    s.has_actor_id_filter = filter ? 1 : 0;
    s.actor_id_filter = filter ? *filter : 0;
    return s;
}

// ------------------------------------------------------------------------------------------ small host helpers of common/evm.rs
inline H256 ascii_to_bytes32(const std::string& s) {   // evm.rs:72-78: right-padded with zeros, truncated to 32
    H256 a{};
    memcpy(a.data(), s.data(), s.size() < 32 ? s.size() : 32);
    return a;
}
inline H256 left_pad_32(const std::vector<uint8_t>& v) {   // evm.rs:91-100: longer than 32 keeps the LAST 32 bytes
    H256 a{};
    if (v.size() >= 32) memcpy(a.data(), v.data() + v.size() - 32, 32);
    else if (!v.empty()) memcpy(a.data() + 32 - v.size(), v.data(), v.size());
    return a;
}

// ------------------------------------------------------------------------------------------ the block store (Blockstore)
class GpuBlockstore {
  public:
    GpuBlockstore(const GpuBlockstore&) = delete;
    GpuBlockstore& operator=(const GpuBlockstore&) = delete;
    GpuBlockstore(GpuBlockstore&& o) noexcept : h_(o.h_), device_(o.device_) { o.h_ = nullptr; }
    GpuBlockstore& operator=(GpuBlockstore&& o) noexcept {
        if (this != &o) { reset(); h_ = o.h_; device_ = o.device_; o.h_ = nullptr; }
        return *this;
    }
    ~GpuBlockstore() { reset(); }

    // what CachedBlockstore holds after the RPC fetches (client/cached_blockstore.rs:53-85): (cid, bytes) pairs → flat arrays → HBM.
    // verify: Blake2b-256 of every block against its CID on the GPU (IPCFP_STORE_VERIFY_CIDS).
    template <class Blocks>   // any range of pair-likes {Cid, std::vector<uint8_t>} (or ProofBlock via from_witness)
    static GpuBlockstore ingest(const Blocks& blocks, int device = 0, bool verify = true) {
        std::vector<uint8_t> cids, blob;
        std::vector<uint64_t> offs;
        std::vector<uint32_t> lens;
        for (const auto& kv : blocks) {
            const Cid& c = std::get<0>(kv);
            const std::vector<uint8_t>& d = std::get<1>(kv);
            if (d.size() > 0xffffffffull) throw Error(IPCFP_ERR_UNSUPPORTED, "block larger than 4 GiB");
            cids.insert(cids.end(), c.bytes.begin(), c.bytes.end());
            offs.push_back(blob.size());
            lens.push_back((uint32_t)d.size());
            blob.insert(blob.end(), d.begin(), d.end());
        }
        return from_flat(cids.data(), offs.data(), lens.data(), blob.data(), blob.size(), offs.size(), device, verify);
    }
    // callers that already hold the flat arrays (ideally in memory from ipcfp_host_alloc: the copy then runs at PCIe rate)
    static GpuBlockstore from_flat(const uint8_t* cids, const uint64_t* offsets, const uint32_t* lengths, const uint8_t* blob, uint64_t blob_size,
                                   uint64_t n_blocks, int device = 0, bool verify = true) {
        ipcfp_store* h = nullptr;
        check(ipcfp_store_create(cids, offsets, lengths, blob, blob_size, n_blocks, device, verify ? IPCFP_STORE_VERIFY_CIDS : 0u, &h), "ipcfp_store_create");
        return GpuBlockstore(h, device);
    }
    // a CARv1 archive held in memory (ipcfp_store_create_car): block k is section k; by-reference offsets index `car`, which the caller
    // keeps for as long as it reads such witnesses. Pass verify for bytes from an untrusted source.
    static GpuBlockstore from_car(const uint8_t* car, uint64_t len, int device = 0, bool verify = true, ipcfp_store_json_info* info = nullptr) {
        ipcfp_store* h = nullptr;
        check(ipcfp_store_create_car(car, len, device, verify ? IPCFP_STORE_VERIFY_CIDS : 0u, &h, info), "ipcfp_store_create_car");
        return GpuBlockstore(h, device);
    }
    // load_witness_store (events/verifier.rs:78-89, storage/verifier.rs:66-77) — with the CID check `put_keyed` leaves out
    static GpuBlockstore from_witness(const std::vector<ProofBlock>& blocks, int device = 0) {
        std::vector<std::pair<Cid, std::vector<uint8_t>>> kv;
        kv.reserve(blocks.size());
        for (const auto& b : blocks) kv.emplace_back(b.cid, b.data);
        return ingest(kv, device, true);
    }

    // Blockstore::get — Ok(None) for an unknown CID
    std::optional<std::vector<uint8_t>> get(const Cid& k) const {
        uint32_t len = 0;
        int found = 0;
        check(ipcfp_store_get(h_, k.bytes.data(), nullptr, 0, &len, &found), "ipcfp_store_get");
        if (!found) return std::nullopt;
        std::vector<uint8_t> buf(len ? len : 1);
        check(ipcfp_store_get(h_, k.bytes.data(), buf.data(), len, &len, &found), "ipcfp_store_get");
        buf.resize(len);
        return buf;
    }
    bool has(const Cid& k) const {
        int found = 0;
        check(ipcfp_store_has(h_, k.bytes.data(), &found), "ipcfp_store_has");
        return found != 0;
    }
    // the store is read-only once ingested, like RpcBlockstore (`unreachable!` at client/blockstore.rs:31)
    void put_keyed(const Cid&, const std::vector<uint8_t>&) { throw std::logic_error("GpuBlockstore::put_keyed: the store is read-only (client/blockstore.rs:31)"); }

    uint64_t n_blocks() const { return ipcfp_store_n_blocks(h_); }
    ipcfp_store* raw() const { return h_; }
    int device() const { return device_; }

  private:
    GpuBlockstore(ipcfp_store* h, int device) : h_(h), device_(device) {}
    void reset() { if (h_) { ipcfp_store_destroy(h_); h_ = nullptr; } }
    ipcfp_store* h_ = nullptr;
    int device_ = 0;
};

// ------------------------------------------------------------------------------------------ (parent, child, receipts) → ipcfp_tipset_desc
class TipsetDesc {
  public:
    // extract_child_info (events/generator.rs:112-119): child.cids[0], child.blocks[0].{parent_message_receipts, parent_state_root};
    // parent.cids / parent.blocks[i].messages (events/generator.rs:148-161); ApiReceipt.events_root (:199-211)
    TipsetDesc(const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts) {
        if (child.cids.empty() || child.blocks.empty()) throw Error(IPCFP_ERR_INVALID_ARG, "child tipset has no blocks");
        if (parent.cids.size() != parent.blocks.size()) throw Error(IPCFP_ERR_INVALID_ARG, "parent tipset: cids and blocks differ in length");
        for (const auto& c : parent.cids) append(parent_cids_, Cid::try_from(c.cid));
        for (const auto& b : parent.blocks) append(txmeta_cids_, Cid::try_from(b.messages.cid));
        append(child_cid_, Cid::try_from(child.cids[0].cid));
        append(receipts_root_, Cid::try_from(child.blocks[0].parent_message_receipts.cid));
        append(state_root_, Cid::try_from(child.blocks[0].parent_state_root.cid));
        events_roots_.assign(receipts.size() * IPCFP_CID_LEN + 1, 0);
        has_root_.assign(receipts.size() + 1, 0);
        for (size_t i = 0; i < receipts.size(); i++)
            if (receipts[i].events_root) {
                Cid c = Cid::try_from(receipts[i].events_root->cid);
                memcpy(events_roots_.data() + i * IPCFP_CID_LEN, c.bytes.data(), IPCFP_CID_LEN);
                has_root_[i] = 1;
            }
        memset(&d_, 0, sizeof d_);
        d_.parent_epoch = parent.height;
        d_.child_epoch = child.height;
        d_.n_parents = (uint32_t)parent.cids.size();
        d_.n_receipts = receipts.size();
        parent_strings_.reserve(parent.cids.size());
        for (const auto& c : parent.cids) parent_strings_.push_back(c.cid);
        child_string_ = child.cids[0].cid;
        state_root_string_ = child.blocks[0].parent_state_root.cid;
    }
    TipsetDesc(const TipsetDesc&) = delete;
    TipsetDesc& operator=(const TipsetDesc&) = delete;
    const ipcfp_tipset_desc* c() {   // pointers are taken here, after every vector has its final address
        d_.parent_cids = parent_cids_.data();
        d_.parent_txmeta_cids = txmeta_cids_.data();
        d_.child_cid = child_cid_.data();
        d_.receipts_root = receipts_root_.data();
        d_.child_parent_state_root = state_root_.data();
        d_.events_roots = events_roots_.data();
        d_.has_events_root = has_root_.data();
        return &d_;
    }
    int64_t parent_epoch() const { return d_.parent_epoch; }
    int64_t child_epoch() const { return d_.child_epoch; }
    const std::vector<std::string>& parent_tipset_cids() const { return parent_strings_; }
    const std::string& child_block_cid() const { return child_string_; }
    const std::string& parent_state_root() const { return state_root_string_; }

  private:
    static void append(std::vector<uint8_t>& v, const Cid& c) { v.insert(v.end(), c.bytes.begin(), c.bytes.end()); }
    std::vector<uint8_t> parent_cids_, txmeta_cids_, child_cid_, receipts_root_, state_root_, events_roots_, has_root_;
    std::vector<std::string> parent_strings_;
    std::string child_string_, state_root_string_;
    ipcfp_tipset_desc d_;
};

// ------------------------------------------------------------------------------------------ POD results → the reference's structs
inline std::vector<ProofBlock> proof_blocks(const ipcfp_witness& w, const uint8_t* by_reference_blob = nullptr) {
    const uint8_t* blob = w.blob ? w.blob : by_reference_blob;   // IPCFP_WITNESS_BY_REFERENCE: offsets index the caller's own blob
    if (w.n_blocks && !blob) throw Error(IPCFP_ERR_INVALID_ARG, "witness carries no block bytes and no blob was given");
    std::vector<ProofBlock> out(w.n_blocks);
    for (uint64_t i = 0; i < w.n_blocks; i++) {
        out[i].cid = Cid::from_bytes(w.cids + IPCFP_CID_LEN * i);
        out[i].data.assign(blob + w.offsets[i], blob + w.offsets[i] + w.lengths[i]);
    }
    return out;
}
// the EventProof construction of events/generator.rs:276-296 (hex formatting :279-281). Slots pass 1 reserved for a receipt that is
// absent from the receipts AMT (the `continue` at :249-251) carry exec_index = UINT64_MAX and are dropped here.
inline std::vector<EventProof> event_proofs(const ipcfp_event_result& r, const TipsetDesc& t) {
    std::vector<EventProof> out;
    out.reserve(r.n_proofs);
    for (uint64_t i = 0; i < r.n_proofs; i++) {
        const ipcfp_event_proof& p = r.proofs[i];
        if (p.exec_index == UINT64_MAX) continue;
        EventProof e;
        e.parent_epoch = t.parent_epoch();
        e.child_epoch = t.child_epoch();
        e.parent_tipset_cids = t.parent_tipset_cids();
        e.child_block_cid = t.child_block_cid();
        e.message_cid = Cid::from_bytes(p.message_cid).to_string();
        e.exec_index = p.exec_index;
        e.event_index = p.event_index;
        e.event_data.emitter = p.emitter;
        for (uint32_t k = 0; k < p.n_topics; k++) e.event_data.topics.push_back(to_hex0x(r.data_blob + p.topics_off + 32ull * k, 32));
        e.event_data.data = to_hex0x(r.data_blob + p.data_off, p.data_len);
        out.push_back(std::move(e));
    }
    return out;
}
inline StorageProof storage_proof(const ipcfp_storage_proof& p, const TipsetDesc& t) {   // storage/generator.rs:165-178
    StorageProof s;
    s.child_epoch = t.child_epoch();
    s.child_block_cid = t.child_block_cid();
    s.parent_state_root = t.parent_state_root();
    s.actor_id = p.actor_id;
    s.actor_state_cid = Cid::from_bytes(p.actor_state_cid).to_string();
    s.storage_root = Cid::from_bytes(p.storage_root).to_string();
    s.slot = to_hex0x(p.slot, 32);
    s.value = to_hex0x(p.value, 32);
    return s;
}

// ------------------------------------------------------------------------------------------ generators
// generate_event_proof (events/generator.rs:60-107)
inline EventProofBundle generate_event_proof(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts,
                                             const std::string& event_signature, const std::string& topic_1, std::optional<uint64_t> actor_id_filter) {
    TipsetDesc t(parent, child, receipts);
    ipcfp_event_spec spec = spec_c(event_signature, topic_1, actor_id_filter);
    ipcfp_event_result* r = nullptr;
    check(ipcfp_generate_event_proof(store.raw(), t.c(), &spec, 0, &r), "generate_event_proof");
    EventProofBundle b;
    try {
        b.proofs = event_proofs(*r, t);
        b.blocks = proof_blocks(r->witness);
    } catch (...) { ipcfp_event_result_free(r); throw; }
    ipcfp_event_result_free(r);
    return b;
}

// generate_event_proof with a log filter as the predicate: one EventProofBundle (ipcfp_generate_log_proof). More than four topic
// positions is refused like any other invalid filter.
inline EventProofBundle generate_log_proof(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts,
                                           const LogFilter& filter) {
    if (filter.topics.size() > 4) throw Error(IPCFP_ERR_INVALID_ARG, "generate_log_proof: more than four topic positions");
    TipsetDesc t(parent, child, receipts);
    std::vector<std::vector<uint8_t>> keep;
    const ipcfp_log_filter f = log_filter_c(filter, keep);
    ipcfp_event_result* r = nullptr;
    check(ipcfp_generate_log_proof(store.raw(), t.c(), &f, 0, &r), "generate_log_proof");
    EventProofBundle b;
    try {
        b.proofs = event_proofs(*r, t);
        b.blocks = proof_blocks(r->witness);
    } catch (...) { ipcfp_event_result_free(r); throw; }
    ipcfp_event_result_free(r);
    return b;
}

// The logs of given messages (ipcfp_generate_message_log_proof): the EventProofBundle of `filter` (none: every log) restricted to the
// receipts of `message_cids`, and every message's position in the execution order (std::nullopt: the tipset did not execute it). Only
// the selected receipts' events AMTs are read. More than IPCFP_MESSAGE_MAX messages or four topic positions is refused.
struct MessageLogProof {
    EventProofBundle bundle;
    std::vector<std::optional<uint64_t>> exec_indices;
};
inline MessageLogProof generate_event_proof(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts,
                                            const std::vector<Cid>& message_cids, const std::optional<LogFilter>& filter = std::nullopt) {
    if (filter && filter->topics.size() > 4) throw Error(IPCFP_ERR_INVALID_ARG, "generate_event_proof: more than four topic positions");
    TipsetDesc t(parent, child, receipts);
    std::vector<std::vector<uint8_t>> keep;
    ipcfp_log_filter f;
    if (filter) f = log_filter_c(*filter, keep);
    std::vector<uint8_t> cids(IPCFP_CID_LEN * message_cids.size());
    for (size_t k = 0; k < message_cids.size(); k++) memcpy(cids.data() + IPCFP_CID_LEN * k, message_cids[k].bytes.data(), IPCFP_CID_LEN);
    std::vector<uint64_t> idx(message_cids.size());
    ipcfp_event_result* r = nullptr;
    check(ipcfp_generate_message_log_proof(store.raw(), t.c(), cids.empty() ? nullptr : cids.data(), message_cids.size(), filter ? &f : nullptr, 0,
                                           idx.empty() ? nullptr : idx.data(), &r),
          "generate_event_proof");
    MessageLogProof m;
    try {
        m.bundle.proofs = event_proofs(*r, t);
        m.bundle.blocks = proof_blocks(r->witness);
    } catch (...) { ipcfp_event_result_free(r); throw; }
    ipcfp_event_result_free(r);
    for (uint64_t i : idx) m.exec_indices.push_back(i == UINT64_MAX ? std::nullopt : std::optional<uint64_t>(i));
    return m;
}

// generate_storage_proof (storage/generator.rs:29-67) → (StorageProof, Vec<ProofBlock>)
inline std::pair<StorageProof, std::vector<ProofBlock>> generate_storage_proof(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child,
                                                                               uint64_t actor_id, const H256& slot) {
    TipsetDesc t(parent, child, {});
    ipcfp_storage_spec s;
    memset(&s, 0, sizeof s);
    s.actor_id = actor_id;
    memcpy(s.slot, slot.data(), 32);
    ipcfp_storage_result* r = nullptr;
    check(ipcfp_generate_storage_proofs(store.raw(), t.c(), &s, 1, &r), "generate_storage_proof");
    std::pair<StorageProof, std::vector<ProofBlock>> out;
    try {
        out.first = storage_proof(r->proofs[0], t);
        out.second = proof_blocks(r->witness);
    } catch (...) { ipcfp_storage_result_free(r); throw; }
    ipcfp_storage_result_free(r);
    return out;
}

// read_storage_slot (storage/decode.rs:36-97): Ok(None) when the key is absent. The C ABI carries the value left-padded to 32 bytes plus
// its raw length: values of up to 32 bytes come back exactly; of a longer one the last 32 bytes (what left_pad_32 keeps, evm.rs:92-96).
inline std::optional<std::vector<uint8_t>> read_storage_slot(GpuBlockstore& store, const Cid& contract_state_root, const H256& slot) {
    ipcfp_slot_result* r = nullptr;
    check(ipcfp_read_storage_slots(store.raw(), contract_state_root.bytes.data(), slot.data(), 1, &r), "read_storage_slot");
    std::optional<std::vector<uint8_t>> out;
    if (r->found[0]) {
        const uint32_t n = r->raw_len[0] < 32 ? r->raw_len[0] : 32;
        out = std::vector<uint8_t>(r->values + 32 - n, r->values + 32);
    }
    ipcfp_slot_result_free(r);
    return out;
}

// ------------------------------------------------------------------------------------------ address resolution from the state tree
// ipcfp_resolve_addresses in the reference's types. Per-address outcomes are statuses (unknown addresses are answers, not failures).
struct ResolvedAddresses {
    std::vector<uint64_t> actor_ids;     // 0 where status != IPCFP_OK
    std::vector<ipcfp_status> status;
    ipcfp_status init_status = IPCFP_OK; // StateRoot → actors HAMT → Init state
    std::vector<Cid> missing;            // blocks the walks lacked, `Cid` order: one ChainReadObj round
    std::vector<ProofBlock> witness;     // every block the walks read, `Cid` order
};
inline ResolvedAddresses resolve_addresses(GpuBlockstore& store, const Cid& state_root, const std::vector<ipcfp_address>& addrs) {
    ipcfp_resolve_result* r = nullptr;
    check(ipcfp_resolve_addresses(store.raw(), state_root.bytes.data(), addrs.data(), addrs.size(), &r), "resolve_addresses");
    ResolvedAddresses out;
    out.actor_ids.assign(r->actor_ids, r->actor_ids + r->n);
    out.status.assign(r->status, r->status + r->n);
    out.init_status = r->init_status;
    for (uint64_t i = 0; i < r->n_missing; i++) out.missing.push_back(Cid::from_bytes(r->missing_cids + IPCFP_CID_LEN * i));
    out.witness = proof_blocks(r->witness);
    ipcfp_resolve_result_free(r);
    return out;
}
// parse_address (common/address.rs:65-77): "f…" or "t…"
inline ipcfp_address parse_address(const std::string& s) {
    ipcfp_address a;
    check(ipcfp_address_parse(s.data(), s.size(), &a), ("Failed to parse address '" + s + "'").c_str());
    return a;
}
// the validation of resolve_eth_address_to_actor_id (common/address.rs:10-21) and EthAddressToFilecoinAddress
inline ipcfp_address eth_to_filecoin_address(const std::string& eth_addr) {
    size_t b = 0;
    while (eth_addr.compare(b, 2, "0x") == 0) b += 2;   // trim_start_matches("0x")
    const std::string h = eth_addr.substr(b);
    if (h.size() % 2) throw Error(IPCFP_ERR_INVALID_ARG, "Invalid hex in Ethereum address: Odd number of digits");
    for (size_t i = 0; i < h.size(); i++)
        if (!isxdigit((unsigned char)h[i])) throw Error(IPCFP_ERR_INVALID_ARG, std::string("Invalid hex in Ethereum address: Invalid character '") + h[i] +
                                                                            "' at position " + std::to_string(i));
    const std::vector<uint8_t> bytes = from_hex0x(h);
    if (bytes.size() != 20)
        throw Error(IPCFP_ERR_INVALID_ARG, "Invalid Ethereum address length: expected 20 bytes, got " + std::to_string(bytes.size()));
    ipcfp_address a;
    check(ipcfp_address_from_eth(bytes.data(), &a), "eth_to_filecoin_address");
    return a;
}
// resolve_eth_address_to_actor_id (common/address.rs:8-62) from the state tree at state_root (the child header's ParentStateRoot)
inline uint64_t resolve_eth_address_to_actor_id(GpuBlockstore& store, const Cid& state_root, const std::string& eth_addr) {
    const ResolvedAddresses r = resolve_addresses(store, state_root, {eth_to_filecoin_address(eth_addr)});
    if (r.status[0] != IPCFP_OK) throw Error(r.status[0], "Failed to lookup ID address: ipcfp status " + std::to_string((int)r.status[0]));
    return r.actor_ids[0];
}

// ipcfp_generate_actor_proofs: what the state tree under the child header's ParentStateRoot holds for each address. A proof keeps the C
// record (its fields are the account's: actor_id, sequence, balance, code, head, delegated, the EVM fields) and, with code, the bytecode.
struct ActorProof {
    ipcfp_actor_proof c;
    std::vector<uint8_t> bytecode;       // with_code, EVM actors
    std::vector<size_t> witness;         // indices into ActorProofs::blocks
};
struct ActorProofs {
    std::vector<ActorProof> proofs;
    std::vector<ProofBlock> blocks;      // the union, `Cid` order
};
namespace detail {
inline std::vector<uint8_t> cid_bytes(const std::vector<Cid>& cids) {
    std::vector<uint8_t> out;
    for (const Cid& c : cids) out.insert(out.end(), c.bytes.begin(), c.bytes.end());
    return out;
}
// the descriptor of a child block and its ParentStateRoot: the fields an actor proof reads (no receipts: the root is a placeholder)
struct ActorDesc {
    std::array<uint8_t, IPCFP_CID_LEN> receipts{};
    ipcfp_tipset_desc d;
    ActorDesc(const Cid& child, const Cid& parent_state_root) {
        memset(&d, 0, sizeof d);
        d.child_cid = child.bytes.data();
        d.child_parent_state_root = parent_state_root.bytes.data();
        d.receipts_root = receipts.data();
    }
};
}  // namespace detail
inline ActorProofs generate_actor_proofs(GpuBlockstore& store, const Cid& child, const Cid& parent_state_root, const std::vector<ipcfp_address>& addrs,
                                         const std::vector<Cid>& evm_code_cids, bool with_code) {
    detail::ActorDesc t(child, parent_state_root);
    const std::vector<uint8_t> evm = detail::cid_bytes(evm_code_cids);
    ipcfp_actor_result* r = nullptr;
    check(ipcfp_generate_actor_proofs(store.raw(), &t.d, addrs.data(), addrs.size(), evm.data(), evm_code_cids.size(),
                                      with_code ? IPCFP_ACTOR_WITH_CODE : 0u, &r), "generate_actor_proofs");
    ActorProofs out;
    for (uint64_t i = 0; i < r->n_proofs; i++) {
        ActorProof p;
        p.c = r->proofs[i];
        p.bytecode.assign(r->code_blob + p.c.code_off, r->code_blob + p.c.code_off + p.c.code_len);
        p.witness.assign(r->proof_witness_index + r->proof_witness_offsets[i], r->proof_witness_index + r->proof_witness_offsets[i + 1]);
        out.proofs.push_back(std::move(p));
    }
    out.blocks = proof_blocks(r->witness);
    ipcfp_actor_result_free(r);
    return out;
}
// ipcfp_plan_fetch_actor_proofs_resident: one fetch round (the CIDs the store lacks, `Cid` order) for generate_actor_proofs
inline std::vector<Cid> plan_fetch_actor_proofs(GpuBlockstore& store, const Cid& child, const Cid& parent_state_root, const std::vector<ipcfp_address>& addrs,
                                                const std::vector<Cid>& evm_code_cids, bool with_code) {
    detail::ActorDesc t(child, parent_state_root);
    const std::vector<uint8_t> evm = detail::cid_bytes(evm_code_cids);
    ipcfp_tipset* tip = nullptr;
    check(ipcfp_tipset_upload(store.raw(), &t.d, &tip), "ipcfp_tipset_upload");
    ipcfp_fetch_plan* p = nullptr;
    const ipcfp_status st = ipcfp_plan_fetch_actor_proofs_resident(store.raw(), tip, addrs.data(), addrs.size(), evm.data(), evm_code_cids.size(),
                                                                   with_code ? IPCFP_ACTOR_WITH_CODE : 0u, &p);
    ipcfp_tipset_free(tip);
    check(st, "plan_fetch_actor_proofs");
    std::vector<Cid> out;
    for (uint64_t k = 0; k < p->n_missing; k++) out.push_back(Cid::from_bytes(p->cids + IPCFP_CID_LEN * k));
    ipcfp_fetch_plan_free(p);
    return out;
}
// ipcfp_verify_actor_proofs over the proofs' blocks (a store of them with every block checked against its CID): one verdict per proof
inline std::vector<bool> verify_actor_proofs(const ActorProofs& ap, const Cid& child, const Cid& parent_state_root, const std::vector<Cid>& evm_code_cids,
                                             bool with_code, int device = 0) {
    GpuBlockstore store = GpuBlockstore::from_witness(ap.blocks, device);
    detail::ActorDesc t(child, parent_state_root);
    const std::vector<uint8_t> evm = detail::cid_bytes(evm_code_cids);
    std::vector<ipcfp_actor_proof> qs;
    for (const ActorProof& p : ap.proofs) qs.push_back(p.c);
    std::vector<uint8_t> res(qs.size() + 1, 0);
    check(ipcfp_verify_actor_proofs(store.raw(), &t.d, qs.data(), qs.size(), evm.data(), evm_code_cids.size(), with_code ? IPCFP_ACTOR_WITH_CODE : 0u,
                                    res.data()), "verify_actor_proofs");
    return std::vector<bool>(res.begin(), res.begin() + qs.size());
}

// ipcfp_generate_message_proofs: whether each message executed in the tipset pair and how it ended (its receipt), and with_body the
// message itself. A proof keeps the C record (status, exec_index, exit_code, gas_used, events_root, the body fields) with its return
// data and params; the witness is one union for all proofs.
struct MessageProof {
    ipcfp_message_proof c;
    std::vector<uint8_t> return_data;
    std::vector<uint8_t> params;         // with_body
};
struct MessageProofs {
    std::vector<MessageProof> proofs;
    std::vector<ProofBlock> blocks;      // the union, `Cid` order
};
inline MessageProofs generate_message_proofs(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts,
                                             const std::vector<Cid>& message_cids, bool with_body = false) {
    TipsetDesc t(parent, child, receipts);
    const std::vector<uint8_t> cids = detail::cid_bytes(message_cids);
    ipcfp_message_result* r = nullptr;
    check(ipcfp_generate_message_proofs(store.raw(), t.c(), cids.empty() ? nullptr : cids.data(), message_cids.size(),
                                        with_body ? IPCFP_MESSAGE_WITH_BODY : 0u, &r), "generate_message_proofs");
    MessageProofs out;
    for (uint64_t i = 0; i < r->n_proofs; i++) {
        MessageProof p;
        p.c = r->proofs[i];
        p.return_data.assign(r->data_blob + p.c.return_off, r->data_blob + p.c.return_off + p.c.return_len);
        p.params.assign(r->data_blob + p.c.params_off, r->data_blob + p.c.params_off + p.c.params_len);
        out.proofs.push_back(std::move(p));
    }
    out.blocks = proof_blocks(r->witness);
    ipcfp_message_result_free(r);
    return out;
}
// ipcfp_plan_fetch_message_proofs_resident: one fetch round (the CIDs the store lacks, `Cid` order) for generate_message_proofs
inline std::vector<Cid> plan_fetch_message_proofs(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts,
                                                  const std::vector<Cid>& message_cids, bool with_body = false) {
    TipsetDesc t(parent, child, receipts);
    const std::vector<uint8_t> cids = detail::cid_bytes(message_cids);
    ipcfp_tipset* tip = nullptr;
    check(ipcfp_tipset_upload(store.raw(), t.c(), &tip), "ipcfp_tipset_upload");
    ipcfp_fetch_plan* p = nullptr;
    const ipcfp_status st = ipcfp_plan_fetch_message_proofs_resident(store.raw(), tip, cids.empty() ? nullptr : cids.data(), message_cids.size(),
                                                                     with_body ? IPCFP_MESSAGE_WITH_BODY : 0u, &p);
    ipcfp_tipset_free(tip);
    check(st, "plan_fetch_message_proofs");
    std::vector<Cid> out;
    for (uint64_t k = 0; k < p->n_missing; k++) out.push_back(Cid::from_bytes(p->cids + IPCFP_CID_LEN * k));
    ipcfp_fetch_plan_free(p);
    return out;
}
// ipcfp_verify_message_proofs over the proofs' blocks (a store of them with every block checked against its CID): one verdict per proof
inline std::vector<bool> verify_message_proofs(const MessageProofs& mp, const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts,
                                               bool with_body = false, int device = 0) {
    GpuBlockstore store = GpuBlockstore::from_witness(mp.blocks, device);
    TipsetDesc t(parent, child, receipts);
    std::vector<ipcfp_message_proof> qs;
    std::vector<uint8_t> blob;   // each proof's return data, then its params, as the generator lays them out
    for (const MessageProof& p : mp.proofs) {
        ipcfp_message_proof q = p.c;
        q.return_off = p.return_data.empty() ? 0 : blob.size();
        blob.insert(blob.end(), p.return_data.begin(), p.return_data.end());
        q.params_off = p.params.empty() ? 0 : blob.size();
        blob.insert(blob.end(), p.params.begin(), p.params.end());
        qs.push_back(q);
    }
    std::vector<uint8_t> res(qs.size() + 1, 0);
    check(ipcfp_verify_message_proofs(store.raw(), t.c(), qs.data(), qs.size(), blob.empty() ? nullptr : blob.data(), blob.size(),
                                      with_body ? IPCFP_MESSAGE_WITH_BODY : 0u, res.data()), "verify_message_proofs");
    return std::vector<bool>(res.begin(), res.begin() + qs.size());
}

// the UnifiedProofBundle of an ipcfp_bundle, which it frees
inline UnifiedProofBundle unified_bundle(ipcfp_bundle* b, const TipsetDesc& t) {
    UnifiedProofBundle u;
    try {
        if (b->storage)
            for (uint64_t i = 0; i < b->storage->n_proofs; i++) u.storage_proofs.push_back(storage_proof(b->storage->proofs[i], t));
        for (uint64_t k = 0; k < b->n_event_results; k++) {
            auto ep = event_proofs(*b->events[k], t);
            u.event_proofs.insert(u.event_proofs.end(), std::make_move_iterator(ep.begin()), std::make_move_iterator(ep.end()));
        }
        u.blocks = proof_blocks(b->witness);
    } catch (...) { ipcfp_bundle_free(b); throw; }
    ipcfp_bundle_free(b);
    return u;
}
inline std::vector<ipcfp_storage_spec> storage_specs_c(const std::vector<StorageProofSpec>& storage_specs) {
    std::vector<ipcfp_storage_spec> ss(storage_specs.size());
    for (size_t i = 0; i < ss.size(); i++) {
        memset(&ss[i], 0, sizeof ss[i]);
        ss[i].actor_id = storage_specs[i].actor_id;
        memcpy(ss[i].slot, storage_specs[i].slot.data(), 32);
    }
    return ss;
}

// generate_proof_bundle (proofs/generator.rs:25-95): every spec against one store, blocks deduplicated as BTreeSet<(Cid, data)>
inline UnifiedProofBundle generate_proof_bundle(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts,
                                                const std::vector<StorageProofSpec>& storage_specs, const std::vector<EventProofSpec>& event_specs) {
    TipsetDesc t(parent, child, receipts);
    const std::vector<ipcfp_storage_spec> ss = storage_specs_c(storage_specs);
    std::vector<ipcfp_event_spec> es;
    es.reserve(event_specs.size());
    for (const auto& e : event_specs) es.push_back(spec_c(e.event_signature, e.topic_1, e.actor_id_filter));
    ipcfp_bundle* b = nullptr;
    check(ipcfp_generate_proof_bundle(store.raw(), t.c(), ss.empty() ? nullptr : ss.data(), ss.size(), es.empty() ? nullptr : es.data(), es.size(), &b),
          "generate_proof_bundle");
    return unified_bundle(b, t);
}
// the same bundle with log filters in place of event specs (ipcfp_generate_log_bundle): the storage proofs, then every filter's event
// proofs in order. The filters of LogFilter::from_spec give the spec bundle, byte for byte.
inline UnifiedProofBundle generate_proof_bundle(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<ApiReceipt>& receipts,
                                                const std::vector<StorageProofSpec>& storage_specs, const std::vector<LogFilter>& log_filters) {
    for (const auto& f : log_filters)
        if (f.topics.size() > 4) throw Error(IPCFP_ERR_INVALID_ARG, "generate_proof_bundle: more than four topic positions");
    TipsetDesc t(parent, child, receipts);
    const std::vector<ipcfp_storage_spec> ss = storage_specs_c(storage_specs);
    std::vector<std::vector<uint8_t>> keep;
    std::vector<ipcfp_log_filter> fs;
    for (const auto& f : log_filters) fs.push_back(log_filter_c(f, keep));
    ipcfp_bundle* b = nullptr;
    check(ipcfp_generate_log_bundle(store.raw(), t.c(), ss.empty() ? nullptr : ss.data(), ss.size(), fs.empty() ? nullptr : fs.data(), fs.size(), 0, &b),
          "generate_proof_bundle");
    return unified_bundle(b, t);
}

// keccak256 / hash_event_signature (common/evm.rs:62-69, :81-88), on the GPU
inline H256 keccak256(const std::vector<uint8_t>& bytes, int device = 0) {
    H256 out{};
    const uint64_t off = 0;
    const uint32_t len = (uint32_t)bytes.size();
    const uint8_t none = 0;
    check(ipcfp_keccak256_batch(bytes.empty() ? &none : bytes.data(), bytes.size(), &off, &len, 1, device, out.data()), "keccak256");
    return out;
}
inline H256 hash_event_signature(const std::string& s, int device = 0) { return keccak256(std::vector<uint8_t>(s.begin(), s.end()), device); }
inline LogFilter LogFilter::from_spec(const EventProofSpec& spec, int device) {
    LogFilter f;
    if (spec.actor_id_filter) f.emitters.push_back(*spec.actor_id_filter);
    f.topics = {{hash_event_signature(spec.event_signature, device)}, {ascii_to_bytes32(spec.topic_1)}};
    return f;
}
// create_event_filter(event_sig, subnet_id) (events/verifier.rs:28-41): the predicate verify_event_proof takes as check_event
inline EventProofSpec create_event_filter(const std::string& event_sig, const std::string& subnet_id) { return EventProofSpec{event_sig, subnet_id, std::nullopt}; }
// parse_cid / parse_cids (common/witness.rs:60-72): the error names what was being parsed
inline Cid parse_cid(const std::string& cid_str, const std::string& context) {
    try { return Cid::try_from(cid_str); } catch (const Error& e) { throw Error(e.status, "invalid " + context + " CID: " + e.what()); }
}
inline std::vector<Cid> parse_cids(const std::vector<std::string>& cid_strs, const std::string& context) {
    std::vector<Cid> out;
    out.reserve(cid_strs.size());
    for (const auto& s : cid_strs) out.push_back(parse_cid(s, context));
    return out;
}
// (RecordingBlockStore and WitnessCollector — common/blockstore.rs:8-39, common/witness.rs:9-57 — have no host-side counterpart:
// recording and materialisation happen inside the GPU call; what they produce is the `blocks` of the returned bundle, in `Cid` order.)

// compute_mapping_slot / calculate_storage_slot (storage/utils.rs:5-19): keccak256(key32 ‖ u256_be(slot_index)), on the GPU
inline H256 compute_mapping_slot(const H256& key, uint64_t slot_index, int device = 0) {
    H256 out{};
    check(ipcfp_compute_mapping_slots(key.data(), &slot_index, 1, device, out.data()), "compute_mapping_slot");
    return out;
}
inline H256 calculate_storage_slot(const std::string& subnet_ascii, uint64_t subnets_slot_index, int device = 0) {
    return compute_mapping_slot(ascii_to_bytes32(subnet_ascii), subnets_slot_index, device);
}

// ------------------------------------------------------------------------------------------ one tipset over several GPUs
// The reference's future-work "Parallel Generation" (README.md:384): one process per GPU, one communicator per process. Rank 0 makes
// the id (ShardedComm::unique_id) and hands the 128 bytes to the other ranks by any means. The cross-shard protocol (first-seen dedup of
// the execution order, message-CID fetch, union of the witness CID sets) runs inside the library over NCCL (DESIGN.md §6). Compiled
// here, not run by tests/cpp/host_mirror_test.cpp (it needs NCCL and one GPU per rank): the same C calls are exercised through ctypes by
// tests/test_parallel.py::test_sharded_call_over_nccl at world sizes 1, 2, 4, 8.
class ShardedComm {
  public:
    static std::array<uint8_t, IPCFP_COMM_ID_BYTES> unique_id() {
        std::array<uint8_t, IPCFP_COMM_ID_BYTES> id{};
        check(ipcfp_comm_unique_id(id.data()), "ipcfp_comm_unique_id");
        return id;
    }
    ShardedComm(const std::array<uint8_t, IPCFP_COMM_ID_BYTES>& id, uint32_t world, uint32_t rank, int device) : world_(world), rank_(rank) {
        check(ipcfp_comm_init(id.data(), world, rank, device, &h_), "ipcfp_comm_init");
    }
    ShardedComm(const ShardedComm&) = delete;
    ShardedComm& operator=(const ShardedComm&) = delete;
    ~ShardedComm() { if (h_) ipcfp_comm_destroy(h_); }
    ipcfp_comm* raw() const { return h_; }
    uint32_t world() const { return world_; }
    uint32_t rank() const { return rank_; }

  private:
    ipcfp_comm* h_ = nullptr;
    uint32_t world_, rank_;
};
struct ShardedEventProof {
    std::vector<EventProof> proofs;   // proofs of the receipts this rank owns; message_cid / exec_index final (execution order resolved across shards)
    std::vector<ProofBlock> blocks;   // this shard's witness blocks in `Cid` order
    std::vector<Cid> union_part;      // entries [union_first, union_first + union_part.size()) of the BTreeSet<Cid> union over ALL shards
    uint64_t union_first = 0, union_total = 0, total_matching = 0, total_proofs = 0;
};
// generate_event_proof for ONE tipset split by receipt index: rank r scans receipts bounds[r] .. bounds[r+1] out of a store that holds
// the blocks that range needs. Every rank must make the call; they succeed or fail together, naming the error the single-store call
// on the whole tipset would have named.
inline ShardedEventProof generate_event_proof_sharded(ShardedComm& comm, GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child,
                                                      const std::vector<ApiReceipt>& receipts, const std::vector<uint64_t>& bounds,
                                                      const std::string& event_signature, const std::string& topic_1, std::optional<uint64_t> actor_id_filter) {
    if (bounds.size() != (size_t)comm.world() + 1) throw Error(IPCFP_ERR_INVALID_ARG, "bounds must hold world + 1 receipt indices");
    TipsetDesc t(parent, child, receipts);
    ipcfp_event_spec spec = spec_c(event_signature, topic_1, actor_id_filter);
    ipcfp_tipset* tip = nullptr;
    check(ipcfp_tipset_upload(store.raw(), t.c(), &tip), "ipcfp_tipset_upload");
    ipcfp_event_result* r = nullptr;
    const ipcfp_status st = ipcfp_generate_event_proof_sharded(comm.raw(), store.raw(), tip, &spec, bounds.data(), IPCFP_SHARDED_UNION_TO_HOST, &r);
    ipcfp_tipset_free(tip);
    check(st, "generate_event_proof_sharded");
    ShardedEventProof out;
    try {
        out.proofs = event_proofs(*r, t);
        out.blocks = proof_blocks(r->witness);
        for (uint64_t i = 0; i < r->n_union_part; i++) out.union_part.push_back(Cid::from_bytes(r->union_cids + IPCFP_CID_LEN * i));
        out.union_first = r->union_part_first;
        out.union_total = r->n_union_cids;
        out.total_matching = r->total_matching;
        out.total_proofs = r->total_proofs;
    } catch (...) { ipcfp_event_result_free(r); throw; }
    ipcfp_event_result_free(r);
    return out;
}

// ------------------------------------------------------------------------------------------ verifiers
using TrustedParentTs = std::function<bool(int64_t, const std::vector<Cid>&)>;
using TrustedChildHeader = std::function<bool(int64_t, const Cid&)>;

// verify_event_proof (events/verifier.rs:51-74). The trust closures are host policy (:124-144) and run here; everything else of
// verify_single_proof runs on the GPU over a witness store whose every block was Blake2b-checked against its CID. `check_event` plays
// create_event_filter(event_sig, subnet_id) (:28-41): the event must satisfy matches_log of that spec.
inline std::vector<bool> verify_event_proof(const EventProofBundle& bundle, const TrustedParentTs& is_trusted_parent_ts,
                                            const TrustedChildHeader& is_trusted_child_header, const EventProofSpec* check_event = nullptr, int device = 0) {
    std::vector<bool> results(bundle.proofs.size(), false);
    if (bundle.proofs.empty()) return results;
    GpuBlockstore store = GpuBlockstore::from_witness(bundle.blocks, device);
    ipcfp_event_spec filter;
    if (check_event) filter = spec_c(check_event->event_signature, check_event->topic_1, check_event->actor_id_filter);
    // proofs of one bundle share the tipset pair; one batched call per distinct pair
    std::map<std::tuple<int64_t, int64_t, std::vector<std::string>, std::string>, std::vector<size_t>> groups;
    for (size_t i = 0; i < bundle.proofs.size(); i++) {
        const EventProof& p = bundle.proofs[i];
        groups[std::make_tuple(p.parent_epoch, p.child_epoch, p.parent_tipset_cids, p.child_block_cid)].push_back(i);
    }
    for (const auto& g : groups) {
        const int64_t parent_epoch = std::get<0>(g.first), child_epoch = std::get<1>(g.first);
        std::vector<Cid> parents;
        for (const auto& s : std::get<2>(g.first)) parents.push_back(Cid::try_from(s));
        const Cid child = Cid::try_from(std::get<3>(g.first));
        if (!is_trusted_parent_ts(parent_epoch, parents) || !is_trusted_child_header(child_epoch, child)) continue;   // verify_trust_anchors → Ok(false)
        std::vector<uint8_t> pc;
        for (const auto& c : parents) pc.insert(pc.end(), c.bytes.begin(), c.bytes.end());
        ipcfp_tipset_desc d;
        memset(&d, 0, sizeof d);
        d.parent_epoch = parent_epoch;
        d.child_epoch = child_epoch;
        d.n_parents = (uint32_t)parents.size();
        d.parent_cids = pc.data();
        d.child_cid = child.bytes.data();
        std::vector<uint8_t> blob;
        std::vector<ipcfp_event_proof> raw;
        for (size_t i : g.second) {
            const EventProof& p = bundle.proofs[i];
            ipcfp_event_proof q;
            memset(&q, 0, sizeof q);
            q.exec_index = p.exec_index;
            q.event_index = p.event_index;
            q.emitter = p.event_data.emitter;
            q.n_topics = (uint32_t)p.event_data.topics.size();
            q.topics_off = blob.size();
            for (const auto& t : p.event_data.topics) { H256 h = from_hex32(t); blob.insert(blob.end(), h.begin(), h.end()); }
            std::vector<uint8_t> data = from_hex0x(p.event_data.data);
            q.data_off = blob.size();
            q.data_len = (uint32_t)data.size();
            blob.insert(blob.end(), data.begin(), data.end());
            Cid m = Cid::try_from(p.message_cid);
            memcpy(q.message_cid, m.bytes.data(), IPCFP_CID_LEN);
            raw.push_back(q);
        }
        blob.resize(blob.size() + 16, 0);   // never hand the library a NULL blob
        std::vector<uint8_t> res(raw.size(), 0);
        check(ipcfp_verify_event_proofs(store.raw(), &d, raw.data(), raw.size(), blob.data(), blob.size() - 16, check_event ? &filter : nullptr, res.data()),
              "verify_event_proof");
        for (size_t k = 0; k < g.second.size(); k++) results[g.second[k]] = res[k] != 0;
    }
    return results;
}

// verify_storage_proof (storage/verifier.rs:24-63), one proof against its witness blocks
inline bool verify_storage_proof(const StorageProof& proof, const std::vector<ProofBlock>& blocks, const TrustedChildHeader& is_trusted_child_header, int device = 0) {
    const Cid child = Cid::try_from(proof.child_block_cid);
    if (!is_trusted_child_header(proof.child_epoch, child)) return false;   // verify_trust_anchor → Ok(false)
    GpuBlockstore store = GpuBlockstore::from_witness(blocks, device);
    const Cid psr = Cid::try_from(proof.parent_state_root);
    ipcfp_tipset_desc d;
    memset(&d, 0, sizeof d);
    d.child_epoch = proof.child_epoch;
    d.child_cid = child.bytes.data();
    d.child_parent_state_root = psr.bytes.data();
    ipcfp_storage_proof q;
    memset(&q, 0, sizeof q);
    q.actor_id = proof.actor_id;
    memcpy(q.actor_state_cid, Cid::try_from(proof.actor_state_cid).bytes.data(), IPCFP_CID_LEN);
    memcpy(q.storage_root, Cid::try_from(proof.storage_root).bytes.data(), IPCFP_CID_LEN);
    memcpy(q.slot, from_hex32(proof.slot).data(), 32);
    memcpy(q.value, from_hex32(proof.value).data(), 32);
    uint8_t res = 0;
    check(ipcfp_verify_storage_proofs(store.raw(), &d, &q, 1, &res), "verify_storage_proof");
    return res != 0;
}

// ------------------------------------------------------------------------------------------ storage paths (ipcfp.h, "Storage paths")
// A Solidity value by its access path: the declared slot, then steps, then what to read. Each builder step returns a new path:
//   StoragePath::at(actor, 0).mapping(subnet_id).field(2).bytes()            subnets[id].<string member at slot offset 2>
struct StoragePath {
    struct Step { uint32_t op; std::vector<uint8_t> key; uint64_t index; uint32_t elem_slots, elem_bytes; };
    uint64_t actor_id = 0;
    H256 base_slot{};
    std::vector<Step> steps;
    uint32_t kind = IPCFP_PATH_WORDS;
    uint32_t n_words = 1;

    static StoragePath at(uint64_t actor_id, const H256& slot) { StoragePath p; p.actor_id = actor_id; p.base_slot = slot; return p; }
    static StoragePath at(uint64_t actor_id, uint64_t slot) {
        H256 s{};
        for (int i = 0; i < 8; i++) s[31 - i] = (uint8_t)(slot >> (8 * i));
        return at(actor_id, s);
    }
    // a value-type key in its 32-byte padded form, or the raw bytes of a bytes / string key
    StoragePath mapping(const std::vector<uint8_t>& key) const { return with(Step{IPCFP_PATH_MAPPING, key, 0, 0, 0}); }
    StoragePath mapping(const H256& key) const { return mapping(std::vector<uint8_t>(key.begin(), key.end())); }
    StoragePath array(uint64_t index, uint32_t elem_slots = 1, uint32_t elem_bytes = 0) const { return with(Step{IPCFP_PATH_ARRAY, {}, index, elem_slots, elem_bytes}); }
    StoragePath static_array(uint64_t index, uint32_t elem_slots = 1, uint32_t elem_bytes = 0) const {
        return with(Step{IPCFP_PATH_STATIC, {}, index, elem_slots, elem_bytes});
    }
    StoragePath field(uint64_t offset) const { return with(Step{IPCFP_PATH_FIELD, {}, offset, 0, 0}); }
    StoragePath words(uint32_t n) const { StoragePath p = *this; p.kind = IPCFP_PATH_WORDS; p.n_words = n; return p; }
    StoragePath bytes() const { StoragePath p = *this; p.kind = IPCFP_PATH_BYTES; p.n_words = 0; return p; }

  private:
    StoragePath with(Step s) const { StoragePath p = *this; p.steps.push_back(std::move(s)); return p; }
};
// One path's outcome: its status (IPCFP_PATH_*), final slot, packed byte offset, value (the words, or the decoded bytes) and its proofs
// (the StorageProofs of its expanded specs, in expanded order). valid: the verifier's verdict (always true from the generator).
struct StoragePathValue {
    uint32_t status = IPCFP_PATH_OK;
    bool valid = true;
    H256 slot{};
    uint32_t byte_offset = 0;
    std::vector<uint8_t> value;
    std::vector<StorageProof> proofs;
};
struct StoragePathProofs {
    std::vector<StoragePathValue> paths;
    std::vector<ProofBlock> blocks;   // the witness union of every proof
};

namespace detail {
struct PathsC {
    std::vector<std::vector<ipcfp_path_step>> steps;
    std::vector<ipcfp_storage_path> c;
    explicit PathsC(const std::vector<StoragePath>& paths) {
        steps.resize(paths.size());
        for (size_t i = 0; i < paths.size(); i++) {
            const StoragePath& p = paths[i];
            for (const auto& s : p.steps)
                steps[i].push_back(ipcfp_path_step{s.op, (uint32_t)s.key.size(), s.key.empty() ? nullptr : s.key.data(), s.index, s.elem_slots, s.elem_bytes});
            ipcfp_storage_path q;
            memset(&q, 0, sizeof q);
            q.actor_id = p.actor_id;
            memcpy(q.base_slot, p.base_slot.data(), 32);
            q.n_steps = (uint32_t)p.steps.size();
            q.kind = p.kind;
            q.steps = steps[i].empty() ? nullptr : steps[i].data();
            q.n_words = p.n_words;
            c.push_back(q);
        }
    }
};
// the per-path values of a result; proofs from `proofs` (the result's own, or the caller's for the verifier) when given
inline std::vector<StoragePathValue> path_values(const ipcfp_path_result& r, const std::vector<StorageProof>* proofs) {
    std::vector<StoragePathValue> out(r.n_paths);
    for (uint64_t i = 0; i < r.n_paths; i++) {
        const ipcfp_path_value& v = r.paths[i];
        StoragePathValue& o = out[i];
        o.status = v.status;
        o.valid = v.valid != 0;
        memcpy(o.slot.data(), v.slot, 32);
        o.byte_offset = v.byte_offset;
        o.value.assign(r.value_blob + v.value_off, r.value_blob + v.value_off + v.value_len);
        if (proofs) o.proofs.assign(proofs->begin() + v.first_spec, proofs->begin() + v.first_spec + v.n_specs);
    }
    return out;
}
}  // namespace detail

// ipcfp_generate_storage_path_proofs_resident against (parent, child)'s tipset: every path's value and the StorageProofs of its
// expanded specs, as generate_storage_proof returns them, with the witness union
inline StoragePathProofs generate_storage_path_proofs(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<StoragePath>& paths) {
    TipsetDesc t(parent, child, {});
    detail::PathsC pc(paths);
    ipcfp_tipset* tip = nullptr;
    check(ipcfp_tipset_upload(store.raw(), t.c(), &tip), "ipcfp_tipset_upload");
    ipcfp_path_result* r = nullptr;
    const ipcfp_status st = ipcfp_generate_storage_path_proofs_resident(store.raw(), tip, pc.c.data(), pc.c.size(), 0, &r);
    ipcfp_tipset_free(tip);
    check(st, "generate_storage_path_proofs");
    StoragePathProofs out;
    try {
        std::vector<StorageProof> proofs;
        for (uint64_t k = 0; k < r->storage->n_proofs; k++) proofs.push_back(storage_proof(r->storage->proofs[k], t));
        out.paths = detail::path_values(*r, &proofs);
        out.blocks = proof_blocks(r->storage->witness);
    } catch (...) { ipcfp_path_result_free(r); throw; }
    ipcfp_path_result_free(r);
    return out;
}
// ipcfp_plan_fetch_storage_paths_resident: one fetch round (the CIDs the store lacks, `Cid` order) for generate_storage_path_proofs
inline std::vector<Cid> plan_fetch_storage_paths(GpuBlockstore& store, const ApiTipset& parent, const ApiTipset& child, const std::vector<StoragePath>& paths) {
    TipsetDesc t(parent, child, {});
    detail::PathsC pc(paths);
    ipcfp_tipset* tip = nullptr;
    check(ipcfp_tipset_upload(store.raw(), t.c(), &tip), "ipcfp_tipset_upload");
    ipcfp_fetch_plan* p = nullptr;
    const ipcfp_status st = ipcfp_plan_fetch_storage_paths_resident(store.raw(), tip, pc.c.data(), pc.c.size(), 0, &p);
    ipcfp_tipset_free(tip);
    check(st, "plan_fetch_storage_paths");
    std::vector<Cid> out;
    for (uint64_t k = 0; k < p->n_missing; k++) out.push_back(Cid::from_bytes(p->cids + IPCFP_CID_LEN * k));
    ipcfp_fetch_plan_free(p);
    return out;
}
// ipcfp_verify_storage_paths: the paths' claims against StorageProofs (one child block and state root, as in a bundle) and their blocks,
// after the trust anchor; per path valid, status and value (proofs left empty). An untrusted child gives every path valid = false.
inline std::vector<StoragePathValue> verify_storage_paths(const std::vector<StorageProof>& proofs, const std::vector<ProofBlock>& blocks,
                                                          const std::vector<StoragePath>& paths, const TrustedChildHeader& is_trusted_child_header, int device = 0) {
    if (proofs.empty()) throw Error(IPCFP_ERR_INVALID_ARG, "verify_storage_paths: no proofs");
    const Cid child = Cid::try_from(proofs[0].child_block_cid);
    const Cid psr = Cid::try_from(proofs[0].parent_state_root);
    std::vector<ipcfp_storage_proof> qs(proofs.size());
    for (size_t i = 0; i < proofs.size(); i++) {
        const StorageProof& p = proofs[i];
        if (p.child_block_cid != proofs[0].child_block_cid || p.parent_state_root != proofs[0].parent_state_root)
            throw Error(IPCFP_ERR_UNSUPPORTED, "verify_storage_paths: proofs of several child blocks");
        ipcfp_storage_proof& q = qs[i];
        memset(&q, 0, sizeof q);
        q.actor_id = p.actor_id;
        memcpy(q.actor_state_cid, Cid::try_from(p.actor_state_cid).bytes.data(), IPCFP_CID_LEN);
        memcpy(q.storage_root, Cid::try_from(p.storage_root).bytes.data(), IPCFP_CID_LEN);
        memcpy(q.slot, from_hex32(p.slot).data(), 32);
        memcpy(q.value, from_hex32(p.value).data(), 32);
    }
    GpuBlockstore store = GpuBlockstore::from_witness(blocks, device);
    ipcfp_tipset_desc d;
    memset(&d, 0, sizeof d);
    d.child_epoch = proofs[0].child_epoch;
    d.child_cid = child.bytes.data();
    d.child_parent_state_root = psr.bytes.data();
    detail::PathsC pc(paths);
    ipcfp_path_result* r = nullptr;
    check(ipcfp_verify_storage_paths(store.raw(), &d, qs.data(), qs.size(), pc.c.data(), pc.c.size(), &r), "verify_storage_paths");
    std::vector<StoragePathValue> out = detail::path_values(*r, nullptr);
    ipcfp_path_result_free(r);
    if (!is_trusted_child_header(proofs[0].child_epoch, child))
        for (auto& v : out) v.valid = false;
    return out;
}

// verify_proof_bundle (proofs/verifier.rs:12-60): every storage proof and every event proof of a UnifiedProofBundle against its
// blocks; the TrustPolicy of the reference arrives as the two closures it is turned into there (:21-25, :38-47)
inline UnifiedVerificationResult verify_proof_bundle(const UnifiedProofBundle& b, const TrustedParentTs& is_trusted_parent_ts,
                                                     const TrustedChildHeader& is_trusted_child_header, const EventProofSpec* check_event = nullptr, int device = 0) {
    UnifiedVerificationResult r;
    for (const auto& s : b.storage_proofs) r.storage_results.push_back(verify_storage_proof(s, b.blocks, is_trusted_child_header, device));
    EventProofBundle eb;
    eb.proofs = b.event_proofs;
    eb.blocks = b.blocks;
    r.event_results = verify_event_proof(eb, is_trusted_parent_ts, is_trusted_child_header, check_event, device);
    return r;
}

namespace detail {
// ipcfp_verify_bundle_json or its _any form: call(tp, tc, ctx, &verdict) with the closures turned into C callbacks
template <class Call>
inline UnifiedVerificationResult verify_json_with(const TrustedParentTs& is_trusted_parent_ts, const TrustedChildHeader& is_trusted_child_header, Call call) {
    struct Ctx { const TrustedParentTs* parent; const TrustedChildHeader* child; } ctx{&is_trusted_parent_ts, &is_trusted_child_header};
    auto tp = [](void* c, int64_t epoch, const uint8_t* cids, uint32_t n) -> int {
        std::vector<Cid> parents;
        for (uint32_t q = 0; q < n; q++) parents.push_back(Cid::from_bytes(cids + 38ull * q));
        return (*static_cast<Ctx*>(c)->parent)(epoch, parents) ? 1 : 0;
    };
    auto tc = [](void* c, int64_t epoch, const uint8_t* cid) -> int { return (*static_cast<Ctx*>(c)->child)(epoch, Cid::from_bytes(cid)) ? 1 : 0; };
    ipcfp_bundle_verdict* v = nullptr;
    check(call(+tp, +tc, (void*)&ctx, &v), "verify_proof_bundle_json");
    UnifiedVerificationResult r;
    for (uint64_t i = 0; i < v->n_storage_proofs; i++) r.storage_results.push_back(v->storage_results[i] != 0);
    for (uint64_t i = 0; i < v->n_event_proofs; i++) r.event_results.push_back(v->event_results[i] != 0);
    ipcfp_bundle_verdict_free(v);
    return r;
}
}  // namespace detail

// verify_proof_bundle from the bundle's JSON text (EventProofBundle or UnifiedProofBundle), through ipcfp_verify_bundle_json: parse, witness
// store and verification on the GPU (text not in serde_json's canonical form is read by the host parser, with the same results). Each
// closure is called at most once, on this thread.
inline UnifiedVerificationResult verify_proof_bundle_json(const std::string& text, const TrustedParentTs& is_trusted_parent_ts,
                                                          const TrustedChildHeader& is_trusted_child_header, const EventProofSpec* check_event = nullptr,
                                                          int device = 0) {
    ipcfp_event_spec filter;
    if (check_event) filter = spec_c(check_event->event_signature, check_event->topic_1, check_event->actor_id_filter);
    return detail::verify_json_with(is_trusted_parent_ts, is_trusted_child_header, [&](auto tp, auto tc, void* ctx, ipcfp_bundle_verdict** v) {
        return ipcfp_verify_bundle_json(text.data(), text.size(), device, tp, tc, ctx, check_event ? &filter : nullptr, v);
    });
}
// the same with a set of log filters as check_event (ipcfp_verify_bundle_json_any): an event proof is true only when its event matches
// at least one of check_any; an empty set is no check_event
inline UnifiedVerificationResult verify_proof_bundle_json(const std::string& text, const TrustedParentTs& is_trusted_parent_ts,
                                                          const TrustedChildHeader& is_trusted_child_header, const std::vector<LogFilter>& check_any,
                                                          int device = 0) {
    for (const auto& f : check_any)
        if (f.topics.size() > 4) throw Error(IPCFP_ERR_INVALID_ARG, "verify_proof_bundle_json: more than four topic positions");
    std::vector<std::vector<uint8_t>> keep;
    std::vector<ipcfp_log_filter> fs;
    for (const auto& f : check_any) fs.push_back(log_filter_c(f, keep));
    return detail::verify_json_with(is_trusted_parent_ts, is_trusted_child_header, [&](auto tp, auto tc, void* ctx, ipcfp_bundle_verdict** v) {
        return ipcfp_verify_bundle_json_any(text.data(), text.size(), device, tp, tc, ctx, fs.empty() ? nullptr : fs.data(), fs.size(), v);
    });
}

// ------------------------------------------------------------------------------------------ wire format (serde_json of the bundle structs)
// to_json: what `serde_json::to_string(&bundle)` gives in the reference (common/bundle.rs:10-45, events/bundle.rs:5-30,
// storage/bundle.rs:5-14) — struct field order, compact, ProofBlock.cid as the byte array cid 0.11's Serialize emits, block data as
// standard base64. Byte for byte what ipcfp_bundle_to_json / ipcfp_event_result_to_json render from the POD results.
namespace detail {
inline void json_string(std::string& o, const std::string& s) {   // serde_json's escaping
    static const char* H = "0123456789abcdef";
    o.push_back('"');
    for (unsigned char c : s) {
        switch (c) {
            case '"': o += "\\\""; break;
            case '\\': o += "\\\\"; break;
            case '\b': o += "\\b"; break;
            case '\f': o += "\\f"; break;
            case '\n': o += "\\n"; break;
            case '\r': o += "\\r"; break;
            case '\t': o += "\\t"; break;
            default:
                if (c < 0x20) { o += "\\u00"; o.push_back(H[c >> 4]); o.push_back(H[c & 15]); }
                else o.push_back((char)c);
        }
    }
    o.push_back('"');
}
inline void json_base64(std::string& o, const std::vector<uint8_t>& v) {   // base64::engine::general_purpose::STANDARD
    static const char* T = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    o.push_back('"');
    size_t i = 0;
    const size_t n = v.size();
    for (; i + 3 <= n; i += 3) {
        const uint32_t x = (uint32_t)v[i] << 16 | (uint32_t)v[i + 1] << 8 | v[i + 2];
        o.push_back(T[x >> 18]); o.push_back(T[(x >> 12) & 63]); o.push_back(T[(x >> 6) & 63]); o.push_back(T[x & 63]);
    }
    if (n - i == 1) { const uint32_t x = (uint32_t)v[i] << 16; o.push_back(T[x >> 18]); o.push_back(T[(x >> 12) & 63]); o += "=="; }
    else if (n - i == 2) { const uint32_t x = (uint32_t)v[i] << 16 | (uint32_t)v[i + 1] << 8; o.push_back(T[x >> 18]); o.push_back(T[(x >> 12) & 63]); o.push_back(T[(x >> 6) & 63]); o.push_back('='); }
    o.push_back('"');
}
inline void json_blocks(std::string& o, const std::vector<ProofBlock>& blocks) {
    o.push_back('[');
    for (size_t i = 0; i < blocks.size(); i++) {
        if (i) o.push_back(',');
        o += "{\"cid\":[";
        for (int k = 0; k < IPCFP_CID_LEN; k++) { if (k) o.push_back(','); o += std::to_string((unsigned)blocks[i].cid.bytes[k]); }
        o += "],\"data\":";
        json_base64(o, blocks[i].data);
        o.push_back('}');
    }
    o.push_back(']');
}
inline void json_event_proofs(std::string& o, const std::vector<EventProof>& proofs) {
    o.push_back('[');
    for (size_t i = 0; i < proofs.size(); i++) {
        const EventProof& p = proofs[i];
        if (i) o.push_back(',');
        o += "{\"parent_epoch\":" + std::to_string(p.parent_epoch) + ",\"child_epoch\":" + std::to_string(p.child_epoch) + ",\"parent_tipset_cids\":[";
        for (size_t q = 0; q < p.parent_tipset_cids.size(); q++) { if (q) o.push_back(','); json_string(o, p.parent_tipset_cids[q]); }
        o += "],\"child_block_cid\":"; json_string(o, p.child_block_cid);
        o += ",\"message_cid\":"; json_string(o, p.message_cid);
        o += ",\"exec_index\":" + std::to_string(p.exec_index) + ",\"event_index\":" + std::to_string(p.event_index);
        o += ",\"event_data\":{\"emitter\":" + std::to_string(p.event_data.emitter) + ",\"topics\":[";
        for (size_t q = 0; q < p.event_data.topics.size(); q++) { if (q) o.push_back(','); json_string(o, p.event_data.topics[q]); }
        o += "],\"data\":"; json_string(o, p.event_data.data);
        o += "}}";
    }
    o.push_back(']');
}
}  // namespace detail
inline std::string to_json(const EventProofBundle& b) {
    std::string o = "{\"proofs\":";
    detail::json_event_proofs(o, b.proofs);
    o += ",\"blocks\":";
    detail::json_blocks(o, b.blocks);
    o.push_back('}');
    return o;
}
inline std::string to_json(const UnifiedProofBundle& b) {
    std::string o = "{\"storage_proofs\":[";
    for (size_t i = 0; i < b.storage_proofs.size(); i++) {
        const StorageProof& p = b.storage_proofs[i];
        if (i) o.push_back(',');
        o += "{\"child_epoch\":" + std::to_string(p.child_epoch) + ",\"child_block_cid\":"; detail::json_string(o, p.child_block_cid);
        o += ",\"parent_state_root\":"; detail::json_string(o, p.parent_state_root);
        o += ",\"actor_id\":" + std::to_string(p.actor_id) + ",\"actor_state_cid\":"; detail::json_string(o, p.actor_state_cid);
        o += ",\"storage_root\":"; detail::json_string(o, p.storage_root);
        o += ",\"slot\":"; detail::json_string(o, p.slot);
        o += ",\"value\":"; detail::json_string(o, p.value);
        o.push_back('}');
    }
    o += "],\"event_proofs\":";
    detail::json_event_proofs(o, b.event_proofs);
    o += ",\"blocks\":";
    detail::json_blocks(o, b.blocks);
    o.push_back('}');
    return o;
}
// serde_json::from_str::<UnifiedProofBundle> / ::<EventProofBundle> through the C ABI's parser (ipcfp_bundle_from_json,
// csrc/bundle_parse.cpp: unknown fields ignored, trailing characters refused, canonical base64, the three spellings of ProofBlock.cid).
// An EventProofBundle ({"proofs": …, "blocks": …}) comes back with storage_proofs empty. The C ABI's verifiers take one tipset pair
// per call, so a bundle whose proofs disagree on the shared fields is refused (IPCFP_ERR_UNSUPPORTED), as by the C parser.
inline UnifiedProofBundle bundle_from_json(const std::string& text) {
    ipcfp_parsed_bundle* pb = nullptr;
    check(ipcfp_bundle_from_json(text.data(), text.size(), &pb), "bundle_from_json");
    UnifiedProofBundle u;
    try {
        const ipcfp_tipset_desc& t = pb->tipset;
        std::vector<std::string> parents;
        for (uint32_t i = 0; i < t.n_parents; i++) parents.push_back(Cid::from_bytes(t.parent_cids + IPCFP_CID_LEN * i).to_string());
        const std::string child = t.child_cid ? Cid::from_bytes(t.child_cid).to_string() : std::string();
        const std::string psr = t.child_parent_state_root ? Cid::from_bytes(t.child_parent_state_root).to_string() : std::string();
        for (uint64_t i = 0; i < pb->n_storage_proofs; i++) {
            const ipcfp_storage_proof& p = pb->storage_proofs[i];
            StorageProof s;
            s.child_epoch = t.child_epoch;
            s.child_block_cid = child;
            s.parent_state_root = psr;
            s.actor_id = p.actor_id;
            s.actor_state_cid = Cid::from_bytes(p.actor_state_cid).to_string();
            s.storage_root = Cid::from_bytes(p.storage_root).to_string();
            s.slot = to_hex0x(p.slot, 32);
            s.value = to_hex0x(p.value, 32);
            u.storage_proofs.push_back(std::move(s));
        }
        for (uint64_t i = 0; i < pb->n_event_proofs; i++) {
            const ipcfp_event_proof& p = pb->event_proofs[i];
            EventProof e;
            e.parent_epoch = t.parent_epoch;
            e.child_epoch = t.child_epoch;
            e.parent_tipset_cids = parents;
            e.child_block_cid = child;
            e.message_cid = Cid::from_bytes(p.message_cid).to_string();
            e.exec_index = p.exec_index;
            e.event_index = p.event_index;
            e.event_data.emitter = p.emitter;
            for (uint32_t k = 0; k < p.n_topics; k++) e.event_data.topics.push_back(to_hex0x(pb->data_blob + p.topics_off + 32ull * k, 32));
            e.event_data.data = to_hex0x(pb->data_blob + p.data_off, p.data_len);
            u.event_proofs.push_back(std::move(e));
        }
        u.blocks = proof_blocks(pb->witness);
    } catch (...) { ipcfp_parsed_bundle_free(pb); throw; }
    ipcfp_parsed_bundle_free(pb);
    return u;
}

}  // namespace host
}  // namespace ipcfp
#endif  // IPCFP_HPP
