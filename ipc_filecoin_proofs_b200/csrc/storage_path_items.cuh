// storage_path_items.cuh — per-path device functions of the storage-path calls (storage_path.cu): Solidity's storage-layout rules as
// slot arithmetic (DESIGN.md §3, "Storage paths"), the expansion of a path into its specs from the words wave 1 proved, and the value
// read back from the proofs. They live in a header so that tests/host_fuzz can run the very same code on the CPU. The proofs themselves
// are storage_proof_one's (storage.cuh); the Keccak-256 permutation is hashes.cuh's.
#pragma once
#include "storage.cuh"

namespace ipcfp {

// A path as the kernels read it: the caller's ipcfp_storage_path with its steps and keys gathered into one upload
struct PathStepDev {
    uint32_t op, key_len;
    uint64_t key_off;        // MAPPING: into the key bytes
    uint64_t index;
    uint32_t elem_slots, elem_bytes;
};
struct PathDev {
    uint64_t actor_id;
    uint8_t base_slot[32];
    uint32_t n_steps, kind, n_words;
    uint32_t n_fixed;        // its fixed specs: the ARRAY steps' length words, then the WORDS slots or the BYTES header word
    uint64_t step_off;       // into the steps
    uint64_t fixed_off;      // its fixed specs in wave 1's list: [fixed_off, fixed_off + n_fixed)
};
struct PathsDev {
    const PathDev* paths;
    const PathStepDev* steps;
    const uint8_t* keys;
    uint64_t n;
};
// The position of a spec inside its path rides in the low bits of a failure's index: (path << 24) | position
#define PATH_POS_BITS 24
static_assert(IPCFP_PATH_MAX_STEPS + IPCFP_PATH_MAX_WORDS + IPCFP_PATH_MAX_BYTES / 32 + 1 < (1u << PATH_POS_BITS), "a path's specs fit the position bits");
static_assert((uint64_t)IPCFP_PATH_MAX_PATHS << PATH_POS_BITS <= 0xFFFFFFFFFFull + 1, "the path and position fit the error key's 40-bit index");

__host__ __device__ __forceinline__ uint32_t path_n_fixed(uint32_t n_array_steps, uint32_t kind, uint32_t n_words) {
    return n_array_steps + (kind == IPCFP_PATH_WORDS ? n_words : 1u);
}

// s += v << (8 * shift), mod 2^256; s is big-endian
__device__ __forceinline__ void u256_add_at(uint8_t s[32], uint64_t v, uint32_t shift) {
    uint32_t carry = 0;
    for (uint32_t i = 0; i < 32; i++) {   // i: byte position from the low end
        const uint32_t add = (i >= shift && i - shift < 8) ? (uint32_t)(v >> (8 * (i - shift))) & 0xffu : 0u;
        const uint32_t x = (uint32_t)s[31 - i] + add + carry;
        s[31 - i] = (uint8_t)x;
        carry = x >> 8;
    }
}
// s += a * b, mod 2^256 (a * b has at most 96 bits: two 64-bit partial products)
__device__ __forceinline__ void u256_add_mul(uint8_t s[32], uint64_t a, uint32_t b) {
    u256_add_at(s, (a & 0xffffffffull) * b, 0);
    u256_add_at(s, (a >> 32) * b, 4);
}
// v > x for a big-endian u256 v
__device__ __forceinline__ bool u256_gt_u64(const uint8_t v[32], uint64_t x) {
    for (int i = 0; i < 24; i++) if (v[i]) return true;
    uint64_t lo = 0;
    for (int i = 24; i < 32; i++) lo = lo << 8 | v[i];
    return lo > x;
}

// keccak256(key ‖ slot), absorbed straight from the key bytes and the slot (no staging copy); out may alias slot
__device__ __forceinline__ void keccak_key_slot(const uint8_t* key, uint32_t key_len, const uint8_t* slot, uint8_t out[32]) {
    uint64_t st[25];
    for (int i = 0; i < 25; i++) st[i] = 0;
    const uint32_t len = key_len + 32;
    for (uint32_t off = 0;; off += 136) {
        const uint32_t take = len - off < 136 ? len - off : 136;
        for (uint32_t i = 0; i < take; i++) {
            const uint32_t g = off + i;
            const uint8_t b = g < key_len ? key[g] : slot[g - key_len];
            st[i >> 3] ^= (uint64_t)b << (8 * (i & 7));
        }
        if (take == 136) { keccak_f1600(st); continue; }
        st[take >> 3] ^= 0x01ull << (8 * (take & 7));   // Keccak (not SHA-3) padding
        st[16] ^= 0x8000000000000000ull;
        keccak_f1600(st);
        break;
    }
    for (int i = 0; i < 32; i++) out[i] = (uint8_t)(st[i >> 3] >> (8 * (i & 7)));
}

__device__ __forceinline__ uint32_t path_per_slot(const PathStepDev& s) {
    return (s.elem_slots == 1 && s.elem_bytes >= 1) ? 32u / s.elem_bytes : 1u;
}

// Slot derivation of one path: the fixed specs (the length word of every ARRAY step, then the n_words slots or the BYTES header word)
// into fixed[0 .. n_fixed), the final slot and the packed byte offset of its last step
__device__ __forceinline__ void path_fixed_specs(const PathDev& p, const PathStepDev* steps, const uint8_t* keys, ipcfp_storage_spec* fixed,
                                                 uint8_t slot[32], uint32_t& byte_offset) {
    for (int i = 0; i < 32; i++) slot[i] = p.base_slot[i];
    byte_offset = 0;
    uint32_t k = 0;
    for (uint32_t j = 0; j < p.n_steps; j++) {
        const PathStepDev& s = steps[j];
        byte_offset = 0;
        if (s.op == IPCFP_PATH_MAPPING) {
            keccak_key_slot(keys + s.key_off, s.key_len, slot, slot);
        } else if (s.op == IPCFP_PATH_FIELD) {
            u256_add_mul(slot, s.index, 1);
        } else {
            const uint32_t per = path_per_slot(s);
            if (s.op == IPCFP_PATH_ARRAY) {
                fixed[k].actor_id = p.actor_id;
                for (int i = 0; i < 32; i++) fixed[k].slot[i] = slot[i];
                k++;
                keccak_key_slot(nullptr, 0, slot, slot);
            }
            u256_add_mul(slot, s.index / per, s.elem_slots);
            if (per > 1) byte_offset = (uint32_t)(s.index % per) * s.elem_bytes;
        }
    }
    const uint32_t nv = p.kind == IPCFP_PATH_WORDS ? p.n_words : 1u;
    for (uint32_t w = 0; w < nv; w++, k++) {
        fixed[k].actor_id = p.actor_id;
        for (int i = 0; i < 32; i++) fixed[k].slot[i] = slot[i];
        u256_add_at(fixed[k].slot, w, 0);
    }
}

// The expansion of one path from its fixed words (fixed[k] = the proof of fixed spec k; ok[k] == 0: no word, the spec failed or has
// no proof): the path's status, how many data slots a BYTES value has, and the value's length
struct PathExpansion { uint32_t status, n_data, value_len; };
__device__ __forceinline__ PathExpansion path_expand(const PathDev& p, const PathStepDev* steps, const ipcfp_storage_proof* fixed, const uint8_t* ok) {
    PathExpansion e{IPCFP_PATH_OK, 0, 0};
    uint32_t k = 0;
    for (uint32_t j = 0; j < p.n_steps; j++) {
        if (steps[j].op != IPCFP_PATH_ARRAY) continue;
        if (e.status == IPCFP_PATH_OK && (!ok || ok[k]) && !u256_gt_u64(fixed[k].value, steps[j].index)) e.status = IPCFP_PATH_INDEX_OUT_OF_RANGE;
        k++;
    }
    if (p.kind == IPCFP_PATH_WORDS) { e.value_len = 32 * p.n_words; return e; }
    if (ok && !ok[k]) return e;
    const uint8_t* h = fixed[k].value;
    uint32_t bstat = IPCFP_PATH_OK;
    uint64_t len = 0;
    if (!(h[31] & 1)) {                  // short: the length in the low byte
        len = h[31] >> 1;
        if (len > 31) bstat = IPCFP_PATH_BAD_BYTES;
    } else {                             // long: (h - 1) / 2 = h >> 1 for odd h
        bool big = false;
        for (int i = 0; i < 24; i++) big |= h[i] != 0;
        for (int i = 24; i < 32; i++) len = len << 8 | h[i];
        len >>= 1;
        if (big || len > IPCFP_PATH_MAX_BYTES) bstat = IPCFP_PATH_TOO_LONG;
        else if (len < 32) bstat = IPCFP_PATH_BAD_BYTES;
        else e.n_data = (uint32_t)((len + 31) / 32);
    }
    if (bstat == IPCFP_PATH_OK) e.value_len = (uint32_t)len;
    if (e.status == IPCFP_PATH_OK) e.status = bstat;
    return e;
}

// Spec j of a BYTES path's data: keccak256(slot) + j (base = keccak256(slot))
__device__ __forceinline__ void path_data_slot(const uint8_t base[32], uint32_t j, uint8_t out[32]) {
    for (int i = 0; i < 32; i++) out[i] = base[i];
    u256_add_at(out, j, 0);
}

// The path's value from its proofs in expanded order (proofs[0 .. n_fixed + n_data)): the value words, or the decoded bytes
__device__ __forceinline__ void path_value(const PathDev& p, const ipcfp_storage_proof* proofs, uint32_t n_data, uint32_t value_len, uint8_t* out) {
    const uint32_t v0 = p.n_fixed - (p.kind == IPCFP_PATH_WORDS ? p.n_words : 1u);
    if (p.kind == IPCFP_PATH_WORDS) {
        for (uint32_t w = 0; w < p.n_words; w++)
            for (int i = 0; i < 32; i++) out[32 * w + i] = proofs[v0 + w].value[i];
        return;
    }
    if (!n_data) {   // short: the word's high-order bytes
        for (uint32_t i = 0; i < value_len; i++) out[i] = proofs[v0].value[i];
        return;
    }
    for (uint32_t i = 0; i < value_len; i++) out[i] = proofs[p.n_fixed + i / 32].value[i % 32];
}

// (actor_id, slot) order of storage proofs: the verifier's lookup
__device__ __forceinline__ int proof_key_cmp(const ipcfp_storage_proof& q, uint64_t actor, const uint8_t* slot) {
    if (q.actor_id != actor) return q.actor_id < actor ? -1 : 1;
    for (int i = 0; i < 32; i++) if (q.slot[i] != slot[i]) return q.slot[i] < slot[i] ? -1 : 1;
    return 0;
}
// The first entry of order[] (proof indices sorted by (actor_id, slot), then verified ones first) with this key, or -1
__device__ __forceinline__ int64_t proof_find(const ipcfp_storage_proof* proofs, const uint32_t* order, uint64_t n, uint64_t actor, const uint8_t* slot) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        if (proof_key_cmp(proofs[order[mid]], actor, slot) < 0) lo = mid + 1; else hi = mid;
    }
    return lo < n && proof_key_cmp(proofs[order[lo]], actor, slot) == 0 ? (int64_t)order[lo] : -1;
}

}  // namespace ipcfp
