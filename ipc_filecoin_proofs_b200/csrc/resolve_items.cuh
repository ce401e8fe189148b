// resolve_items.cuh — per-item device functions of address resolution (resolve.cu holds the kernels and the host flow). They live in a
// header, as storage.cuh does, so that the same code can be compiled for the host.
//   StateRoot → actors HAMT (width 5) → Init actor (ID 1) → InitState [address_map, next_id, network_name] → address_map HAMT (width 5)
//   builtin-actors init/src/state.rs [UPSTREAM]      State { address_map: Cid, next_id: ActorID, network_name: String }, HAMT_BIT_WIDTH 5
//   fvm_shared address [UPSTREAM]                     Address::to_bytes() is the address_map key; the value is the ActorID (u64)
//   Lotus StateTree.LookupID [UPSTREAM]               ID addresses resolve to themselves without a read
#pragma once
#include "storage.cuh"

namespace ipcfp {

// unsigned_varint::decode::u64 followed by "no bytes left" (fvm_shared from_leb_bytes): at most 10 bytes, minimal, no overflow
__host__ __device__ inline bool leb_u64(const uint8_t* p, uint32_t n, uint32_t& used, uint64_t& v) {
    v = 0;
    for (uint32_t i = 0; i < n && i < 10; i++) {
        const uint64_t b = p[i] & 0x7f;
        if (i == 9 && b > 1) return false;
        v |= b << (7 * i);
        if (!(p[i] & 0x80)) {
            if (i > 0 && p[i] == 0) return false;   // a trailing zero group is not minimal
            used = i + 1;
            return true;
        }
    }
    return false;
}
// fvm_shared Address::from_bytes accepts bytes[0, len); *id = the ID of a protocol-0 address
__host__ __device__ inline bool address_bytes_valid(const uint8_t* bytes, uint32_t len, uint64_t* id) {
    if (len < 1 || len > IPCFP_ADDRESS_MAX) return false;
    const uint8_t* p = bytes + 1;
    const uint32_t n = len - 1u;
    uint32_t used = 0;
    uint64_t v = 0;
    switch (bytes[0]) {
        case 0: if (!leb_u64(p, n, used, v) || used != n) return false; if (id) *id = v; return true;
        case 1: case 2: return n == 20;
        case 3: return n == 48;
        case 4: return leb_u64(p, n, used, v) && n - used <= 54;
        default: return false;
    }
}
__host__ __device__ inline bool address_valid(const ipcfp_address& a, uint64_t* id) { return address_bytes_valid(a.bytes, a.len, id); }

// The Init path: the address_map root of the state tree at state_root (a pointer into the store's block arena). Fails as
// storage_proof_one fails on the same blocks: DC_MISSING (rec.missing names the block), DC_DECODE, DC_ACTOR_NOT_FOUND (no actor ID 1).
static __device__ bool resolve_init(const StoreView& s, Recorder& rec, const uint8_t* state_root, const uint8_t*& address_map, Fail& f) {
    address_map = nullptr;
    uint8_t key[11];
    const uint8_t* state_cid;
    if (!actor_state(s, rec, state_root, key, id_address_key(1, key), state_cid, f)) return false;
    const int32_t ib = rec_get(s, rec, state_cid);
    if (ib < 0) SFAIL(DC_MISSING, 3);
    uint32_t il;
    const uint8_t* ip = store_block(s, (uint32_t)ib, il);
    Rd r(ip, il);
    rd_array_exact(r, 3);
    const uint32_t map_off = rd_cid(r);
    (void)rd_uint(r);
    uint32_t tl;
    (void)rd_text(r, tl);
    rd_end(r);
    if (r.err) SFAIL(DC_DECODE, r.err);
    address_map = ip + map_off;
    return true;
}

// address_map.get(key): the ActorID, or DC_ACTOR_NOT_FOUND when the key is not in the map
static __device__ bool resolve_lookup(const StoreView& s, Recorder& rec, const uint8_t* address_map, const uint8_t* key, uint32_t keylen, uint64_t& id,
                                      Fail& f) {
    id = 0;
    bool found;
    ValueRef vr;
    if (!hamt_get(s, rec, address_map, 5, HV_U64, key, keylen, found, vr, f)) return false;
    if (!found) SFAIL(DC_ACTOR_NOT_FOUND, 0);
    uint32_t bl;
    const uint8_t* bp = store_block(s, vr.blk, bl);
    Rd r(bp, bl);
    r.pos = vr.off;
    id = rd_uint(r);   // the node decoder has accepted this value as one minimal major-0 integer
    return true;
}

__host__ __device__ __forceinline__ ipcfp_status resolve_status(uint32_t code) {
    return code == DC_MISSING ? IPCFP_ERR_MISSING_BLOCK : code == DC_ACTOR_NOT_FOUND ? IPCFP_ERR_ACTOR_NOT_FOUND : IPCFP_ERR_DECODE;
}

}  // namespace ipcfp
