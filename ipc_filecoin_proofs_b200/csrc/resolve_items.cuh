// resolve_items.cuh — per-item device functions of address resolution (resolve.cu holds the kernels and the host flow). They live in a
// header, as storage.cuh does, so that the same code can be compiled for the host.
//   StateRoot → actors HAMT (width 5) → Init actor (ID 1) → InitState [address_map, next_id, network_name] → address_map HAMT (width 5)
//   builtin-actors init/src/state.rs [UPSTREAM]      State { address_map: Cid, next_id: ActorID, network_name: String }, HAMT_BIT_WIDTH 5
//   fvm_shared address [UPSTREAM]                     Address::to_bytes() is the address_map key; the value is the ActorID (u64)
//   Lotus StateTree.LookupID [UPSTREAM]               ID addresses resolve to themselves without a read
#pragma once
#include "storage.cuh"

namespace ipcfp {

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
