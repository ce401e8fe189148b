// oracle_resolve.cpp — the C++ oracle of ipcfp_resolve_addresses (TEST INFRASTRUCTURE), built on oracle/oracle.cpp's own code: its strict
// DAG-CBOR decoder (`Dec`), `get_actor_state` (StateRoot → actors HAMT → ActorState, the storage path's lookup) and its HAMT walk
// (`hamt_get<V>`, `decode_hamt_node<V>`) with one more value type, the ActorID. This translation unit includes oracle.cpp, so it is built
// INSTEAD of oracle.cpp, never beside it: as a shared library (tests/oracle_resolve.py) or linked into the host harnesses
// (tests/host_fuzz/fuzz_hamt_u64.cu).
//
//   builtin-actors init/src/state.rs [UPSTREAM]   State { address_map: Cid, next_id: ActorID, network_name: String }, the Init actor is ID 1
//   fvm_shared address [UPSTREAM]                 Address::from_bytes: protocol 0 = minimal LEB128 u64; 1, 2 = 20 bytes; 3 = 48 bytes;
//                                                 4 = minimal LEB128 namespace + at most 54 bytes; the address_map key is to_bytes()
//   Lotus StateTree.LookupID [UPSTREAM]           an ID address resolves to itself without a read
#include "../oracle/oracle.cpp"

namespace orc {

struct ActorIdValue { uint64_t id; };   // the ActorID under an address_map key: one CBOR unsigned integer
template <> struct ValueDec<ActorIdValue> {
    static ActorIdValue dec(Dec& d) { return ActorIdValue{d.uint()}; }
};

// Blockstore::get through a log: the blocks found (the read set) and the last CID that was not there
struct ReadLog : Blockstore {
    const Blockstore& inner;
    mutable std::set<Cid, CidLess> read;
    mutable std::optional<Cid> missing;
    explicit ReadLog(const Blockstore& i) : inner(i) {}
    bool get(const Cid& k, Bytes& out) const override {
        if (inner.get(k, out)) { read.insert(k); return true; }
        missing = k;
        return false;
    }
};

// unsigned_varint::decode::u64 (minimal, at most 10 bytes, no overflow)
static bool leb(const uint8_t* p, size_t n, size_t& used, uint64_t& v) {
    v = 0;
    for (size_t i = 0; i < n && i < 10; i++) {
        if (i == 9 && (p[i] & 0x7f) > 1) return false;
        v |= (uint64_t)(p[i] & 0x7f) << (7 * i);
        if (!(p[i] & 0x80)) { used = i + 1; return !(i > 0 && p[i] == 0); }
    }
    return false;
}
static bool address_from_bytes(const ipcfp_address& a, bool& is_id, uint64_t& id) {
    is_id = false;
    if (a.len < 1 || a.len > IPCFP_ADDRESS_MAX) return false;
    const uint8_t* p = a.bytes + 1;
    const size_t n = a.len - 1u;
    size_t used = 0;
    uint64_t v = 0;
    switch (a.bytes[0]) {
        case 0: if (!leb(p, n, used, v) || used != n) return false; is_id = true; id = v; return true;
        case 1: case 2: return n == 20;
        case 3: return n == 48;
        case 4: return leb(p, n, used, v) && n - used <= 54;
        default: return false;
    }
}

// StateRoot → Init actor → InitState [address_map, next_id, network_name] → address_map root
static Cid init_address_map(const Blockstore& bs, const Cid& state_root) {
    const ActorState init = get_actor_state(bs, state_root, 1);
    Bytes raw;
    if (!bs.get(init.state, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing Init state " + cid_hex(init.state));
    Dec d(raw);
    d.array_exact(3);
    const Cid map = d.cid();
    (void)d.uint();
    (void)d.text();
    d.end();
    return map;
}

}  // namespace orc

extern "C" {

// The whole call: ids / status per address, the Init path's status, the missing CIDs and the read set (both unique, `Cid` order).
// missing and read are written up to their capacities; *n_missing / *n_read are the full counts.
ipcfp_status oracle_resolve_addresses(const oracle_store* s, const uint8_t* state_root, const ipcfp_address* addrs, uint64_t n, uint64_t* ids,
                                      int32_t* status, int32_t* init_status, uint8_t* missing, uint64_t missing_cap, uint64_t* n_missing,
                                      uint8_t* read, uint64_t read_cap, uint64_t* n_read) {
    ReadLog log(s->bs);
    std::set<Cid, CidLess> miss;
    Cid map;
    *init_status = IPCFP_OK;
    try {
        map = init_address_map(log, cid_from(state_root));
    } catch (const Err& e) {
        *init_status = e.status;
        if (e.status == IPCFP_ERR_MISSING_BLOCK && log.missing) miss.insert(*log.missing);
    }
    for (uint64_t i = 0; i < n; i++) {
        bool is_id;
        uint64_t id = 0;
        ids[i] = 0;
        if (!address_from_bytes(addrs[i], is_id, id)) { status[i] = IPCFP_ERR_INVALID_ARG; continue; }
        if (is_id) { status[i] = IPCFP_OK; ids[i] = id; continue; }
        if (*init_status != IPCFP_OK) { status[i] = *init_status; continue; }
        log.missing.reset();
        try {
            auto v = hamt_get<ActorIdValue>(log, map, 5, Bytes(addrs[i].bytes, addrs[i].bytes + addrs[i].len));
            status[i] = v ? IPCFP_OK : IPCFP_ERR_ACTOR_NOT_FOUND;
            if (v) ids[i] = v->id;
        } catch (const Err& e) {
            status[i] = e.status;
            if (e.status == IPCFP_ERR_MISSING_BLOCK && log.missing) miss.insert(*log.missing);
        }
    }
    uint64_t k = 0;
    for (const Cid& c : miss) { if (k < missing_cap) copy_bytes(missing + 38 * k, c.b.data(), 38); k++; }
    *n_missing = k;
    k = 0;
    for (const Cid& c : log.read) { if (k < read_cap) copy_bytes(read + 38 * k, c.b.data(), 38); k++; }
    *n_read = k;
    return IPCFP_OK;
}

// One address_map node (the ActorID value type), as oracle_hamt_node_lookup does for the other two: *kind 0 none, 1 value (*value), 2 link
// (out38); a decode failure returns IPCFP_ERR_DECODE.
ipcfp_status oracle_hamt_u64_node_lookup(const uint8_t* p, uint64_t n, uint32_t idx, const uint8_t* key, uint32_t keylen, int32_t* kind, uint64_t* value,
                                         uint8_t* out38) {
    try {
        Bytes raw(p, p + n), k(key, key + keylen);
        hamt_node_lookup_t<ActorIdValue>(raw, idx, k, kind, [&](const ActorIdValue& v) { *value = v.id; },
                                         [&](const Cid& c) { copy_bytes(out38, c.b.data(), 38); });
        return IPCFP_OK;
    } catch (const Err& e) {
        return e.status;
    }
}

}  // extern "C"
