// oracle_actors.cpp — the C++ oracle of ipcfp_generate_actor_proofs_resident (TEST INFRASTRUCTURE), built on oracle/oracle.cpp's own code:
// its strict DAG-CBOR decoder (`Dec`), `decode_header`, `get_actor_state` (StateRoot → actors HAMT → ActorState with the `ValueDec<ActorState>`
// decoder) and `hamt_get<V>`, and on tests/oracle_resolve.cpp's Init path and ActorID value type. It includes oracle_resolve.cpp (which
// includes oracle.cpp), so it is built INSTEAD of both: as a shared library (tests/oracle_actors.py).
//
//   fvm_shared ActorState [UPSTREAM]      [code, head, sequence, balance (bigint_ser), delegated_address: Option<Address>]
//   fvm_shared bigint_ser [UPSTREAM]      empty = 0; else sign byte (0 plus, 1 minus) + big-endian magnitude (this library: at most 32 bytes)
//   builtin-actors evm State [UPSTREAM]   EvmStateV6 / V5 as parse_evm_state reads them, with every field kept
#include "oracle_resolve.cpp"

namespace orc {

struct EvmFields { Cid bytecode, contract_state; Bytes hash; uint64_t nonce; };
static bool evm_fields(const Bytes& raw, int fields, EvmFields& e) {
    try {
        Dec d(raw);
        d.array_exact((uint64_t)fields);
        e.bytecode = d.cid();
        e.hash = d.bytes();
        if (e.hash.size() != 32) fail_decode("bytecode hash length");
        e.contract_state = d.cid();
        if (fields == 6) { if (d.peek_null()) d.null(); else d.skip_any(); }
        e.nonce = d.uint();
        if (d.peek_null()) d.null(); else d.skip_any();
        d.end();
        return true;
    } catch (Err& x) {
        if (x.status != IPCFP_ERR_DECODE) throw;
        return false;
    }
}

// one proof into q (zeroed by the caller); absences are statuses
static void prove_one(const Blockstore& bs, const Cid& child, const Cid& sroot, const ipcfp_address& a, const std::optional<Cid>& amap,
                      const std::optional<Err>& init_err, const std::vector<Cid>& evm, bool with_code, ipcfp_actor_proof& q, Bytes& code) {
    Bytes hdr;
    if (!bs.get(child, hdr)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing child header");
    if (decode_header(hdr).parent_state_root != sroot) throw Err(IPCFP_ERR_STATE_ROOT_MISMATCH, "ParentStateRoot mismatch");
    q.address = a;
    bool is_id;
    uint64_t id = 0;
    (void)address_from_bytes(a, is_id, id);
    if (!is_id) {
        if (init_err) throw *init_err;
        auto v = hamt_get<ActorIdValue>(bs, *amap, 5, Bytes(a.bytes, a.bytes + a.len));
        if (!v) { q.status = IPCFP_ACTOR_NO_ADDRESS; return; }
        id = v->id;
    }
    q.actor_id = id;
    ActorState st;
    try {
        st = get_actor_state(bs, sroot, id);
    } catch (const Err& x) {
        if (x.status != IPCFP_ERR_ACTOR_NOT_FOUND) throw;
        q.status = IPCFP_ACTOR_NO_ACTOR;
        return;
    }
    copy_bytes(q.code, st.code.b.data(), 38);
    copy_bytes(q.head, st.state.b.data(), 38);
    q.sequence = st.sequence;
    if (!st.balance.empty()) {
        if (st.balance[0] > 1 || st.balance.size() - 1 > 32) fail_decode("balance");
        const size_t m = st.balance.size() - 1;
        bool nonzero = false;
        for (size_t i = 0; i < m; i++) { q.balance[32 - m + i] = st.balance[1 + i]; nonzero |= st.balance[1 + i] != 0; }
        q.balance_negative = (uint8_t)(st.balance[0] == 1 && nonzero);
    }
    if (st.delegated) {
        ipcfp_address d{};
        if (st.delegated->size() > IPCFP_ADDRESS_MAX) fail_decode("delegated address");
        d.len = (uint8_t)st.delegated->size();
        copy_bytes(d.bytes, st.delegated->data(), d.len);
        bool did;
        uint64_t dv;
        if (!address_from_bytes(d, did, dv)) fail_decode("delegated address");
        q.has_delegated = 1;
        q.delegated = d;
    }
    if (std::find(evm.begin(), evm.end(), st.code) == evm.end()) { q.status = IPCFP_ACTOR_FOUND; return; }
    Bytes raw;
    if (!bs.get(st.state, raw)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing EVM state");
    EvmFields e;
    if (!evm_fields(raw, 6, e) && !evm_fields(raw, 5, e)) fail_decode("EVM state");
    q.is_evm = 1;
    q.evm_nonce = e.nonce;
    copy_bytes(q.bytecode_cid, e.bytecode.b.data(), 38);
    copy_bytes(q.contract_state, e.contract_state.b.data(), 38);
    copy_bytes(q.bytecode_hash, e.hash.data(), 32);
    if (with_code) {
        if (!bs.get(e.bytecode, code)) throw Err(IPCFP_ERR_MISSING_BLOCK, "missing bytecode");
        uint8_t h[32];
        cpu_crypto::keccak256(code.data(), code.size(), h);
        if (memcmp(h, q.bytecode_hash, 32) != 0) fail_decode("bytecode hash");
        q.code_len = code.size();
    }
    q.status = IPCFP_ACTOR_FOUND;
}

}  // namespace orc

extern "C" {

// The whole call: proofs (code_off into `code`), per-proof read sets (CIDs in `Cid` order, proof i's at reads[38 * read_off[i] ..
// 38 * read_off[i + 1])), or the failure: its status, *fail_index the first failing proof. Buffers are written up to their capacities;
// *code_size and read_off[n] are the full sizes.
ipcfp_status oracle_actor_proofs(const oracle_store* s, const uint8_t* child, const uint8_t* state_root, const ipcfp_address* addrs, uint64_t n,
                                 const uint8_t* evm_codes, uint64_t n_evm, int with_code, ipcfp_actor_proof* out, uint8_t* code, uint64_t code_cap,
                                 uint64_t* code_size, uint8_t* reads, uint64_t reads_cap, uint64_t* read_off, uint64_t* fail_index) {
    using namespace orc;
    *fail_index = UINT64_MAX;
    std::vector<Cid> evm;
    for (uint64_t k = 0; k < n_evm; k++) evm.push_back(cid_from(evm_codes + 38 * k));
    const Cid sroot = cid_from(state_root), ch = cid_from(child);
    bool any_other = false;
    for (uint64_t i = 0; i < n; i++) {
        bool is_id;
        uint64_t id;
        if (!address_from_bytes(addrs[i], is_id, id)) { *fail_index = i; return IPCFP_ERR_INVALID_ARG; }
        any_other |= !is_id;
    }
    ReadLog init_log(s->bs);
    std::optional<Cid> amap;
    std::optional<Err> init_err;
    if (any_other) {
        try { amap = init_address_map(init_log, sroot); } catch (const Err& e) { init_err = e; }
    }
    uint64_t cs = 0, r = 0;
    read_off[0] = 0;
    for (uint64_t i = 0; i < n; i++) {
        ReadLog log(s->bs);
        ipcfp_actor_proof q;
        memset(&q, 0, sizeof q);
        Bytes c;
        try {
            prove_one(log, ch, sroot, addrs[i], amap, init_err, evm, with_code != 0, q, c);
        } catch (const Err& e) {
            *fail_index = i;
            return e.status;
        }
        if (q.code_len) {
            q.code_off = cs;
            if (cs + c.size() <= code_cap) copy_bytes(code + cs, c.data(), c.size());
            cs += c.size();
        }
        out[i] = q;
        std::set<Cid, CidLess> read = log.read;
        if (addrs[i].bytes[0] != 0) read.insert(init_log.read.begin(), init_log.read.end());
        for (const Cid& x : read) { if (r < reads_cap) copy_bytes(reads + 38 * r, x.b.data(), 38); r++; }
        read_off[i + 1] = r;
    }
    *code_size = cs;
    return IPCFP_OK;
}

}  // extern "C"
