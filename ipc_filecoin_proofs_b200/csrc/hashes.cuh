// hashes.cuh — device hash functions of the engine (sm_90a).
//   K1  Blake2b-256  (RFC 7693)    : CID verification of ingested IPLD blocks
//                                     (multihash-codetable Code::Blake2b256, reference events/utils.rs:65)
//   K2  Keccak-256   (pad 0x01)    : topic0 / storage-slot keys (reference common/evm.rs:62-88, storage/utils.rs:5-12)
//   K2b SHA-256      (FIPS 180-4)  : fvm_ipld_hamt key hashing (reference storage/decode.rs:79-96 via Hamt defaults)
// All are thread-per-message with the whole state in registers: pure 64-/32-bit integer work,
// no tensor cores. Messages are read with 8-byte aligned loads + funnel shifts, so any byte
// alignment of the block inside the arena runs at the same speed (the arena is padded by 16 B
// on both sides so the aligned over-read stays inside the allocation).
#pragma once
#include "common.cuh"

namespace ipcfp {

__device__ __forceinline__ uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int n) { return (x << n) | (x >> (64 - n)); }

// Reads 8 message bytes starting at byte offset `off` of a message whose first byte is at base[skew]
// (base 8-byte aligned). Only aligned 8-byte loads are issued.
struct AlignedMsg {
    const uint64_t* base;  // 8-byte aligned
    uint32_t shift;        // skew * 8
    __device__ __forceinline__ AlignedMsg(const uint8_t* p) {
        uintptr_t a = (uintptr_t)p;
        base = (const uint64_t*)(a & ~(uintptr_t)7);
        shift = (uint32_t)(a & 7) * 8;
    }
    // word index i = message bytes [8i, 8i+8)
    __device__ __forceinline__ uint64_t word(uint32_t i) const {
        uint64_t lo = __ldg(base + i);
        if (shift == 0) return lo;
        uint64_t hi = __ldg(base + i + 1);
        return (lo >> shift) | (hi << (64 - shift));
    }
};

__device__ __forceinline__ uint64_t mask_low_bytes(uint64_t w, uint32_t nbytes) {  // keep the first nbytes (0..8)
    if (nbytes >= 8) return w;
    if (nbytes == 0) return 0;
    return w & ((1ull << (8 * nbytes)) - 1);
}

// ------------------------------------------------------------------ Blake2b-256
__constant__ static const uint64_t B2B_IV[8] = {
    0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
    0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};

#define B2B_G(a, b, c, d, x, y)                                  \
    a = a + b + (x); d = rotr64(d ^ a, 32); c = c + d; b = rotr64(b ^ c, 24); \
    a = a + b + (y); d = rotr64(d ^ a, 16); c = c + d; b = rotr64(b ^ c, 63);

#define B2B_ROUND(s0, s1, s2, s3, s4, s5, s6, s7, s8, s9, s10, s11, s12, s13, s14, s15) \
    B2B_G(v0, v4, v8, v12, m[s0], m[s1]) B2B_G(v1, v5, v9, v13, m[s2], m[s3])           \
    B2B_G(v2, v6, v10, v14, m[s4], m[s5]) B2B_G(v3, v7, v11, v15, m[s6], m[s7])         \
    B2B_G(v0, v5, v10, v15, m[s8], m[s9]) B2B_G(v1, v6, v11, v12, m[s10], m[s11])       \
    B2B_G(v2, v7, v8, v13, m[s12], m[s13]) B2B_G(v3, v4, v9, v14, m[s14], m[s15])

__device__ __forceinline__ void b2b_compress(uint64_t h[8], const uint64_t m[16], uint64_t t, bool last) {
    uint64_t v0 = h[0], v1 = h[1], v2 = h[2], v3 = h[3], v4 = h[4], v5 = h[5], v6 = h[6], v7 = h[7];
    uint64_t v8 = 0x6a09e667f3bcc908ULL, v9 = 0xbb67ae8584caa73bULL, v10 = 0x3c6ef372fe94f82bULL, v11 = 0xa54ff53a5f1d36f1ULL;
    uint64_t v12 = 0x510e527fade682d1ULL ^ t, v13 = 0x9b05688c2b3e6c1fULL;
    uint64_t v14 = last ? ~0x1f83d9abfb41bd6bULL : 0x1f83d9abfb41bd6bULL, v15 = 0x5be0cd19137e2179ULL;
    B2B_ROUND(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
    B2B_ROUND(14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3)
    B2B_ROUND(11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4)
    B2B_ROUND(7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8)
    B2B_ROUND(9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13)
    B2B_ROUND(2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9)
    B2B_ROUND(12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11)
    B2B_ROUND(13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10)
    B2B_ROUND(6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5)
    B2B_ROUND(10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0)
    B2B_ROUND(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
    B2B_ROUND(14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3)
    h[0] ^= v0 ^ v8; h[1] ^= v1 ^ v9; h[2] ^= v2 ^ v10; h[3] ^= v3 ^ v11;
    h[4] ^= v4 ^ v12; h[5] ^= v5 ^ v13; h[6] ^= v6 ^ v14; h[7] ^= v7 ^ v15;
}

// digest of msg[0..len) into out (4 little-endian words == 32 raw bytes in memory order)
__device__ __forceinline__ void blake2b256(const uint8_t* msg, uint32_t len, Digest& out) {
    uint64_t h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = B2B_IV[i];
    h[0] ^= 0x01010020ULL;
    AlignedMsg am(msg);
    uint32_t off = 0;
    uint64_t m[16];
    while (len - off > 128) {
#pragma unroll
        for (int i = 0; i < 16; i++) m[i] = am.word(off / 8 + i);
        off += 128;
        b2b_compress(h, m, off, false);
    }
    uint32_t rem = len - off;  // 0 (only when len == 0) .. 128
#pragma unroll
    for (int i = 0; i < 16; i++) {
        uint32_t have = rem > 8u * i ? rem - 8u * i : 0;
        m[i] = have ? mask_low_bytes(am.word(off / 8 + i), have) : 0;
    }
    b2b_compress(h, m, len, true);
    out.w[0] = h[0]; out.w[1] = h[1]; out.w[2] = h[2]; out.w[3] = h[3];
}

// ------------------------------------------------------------------ Keccak-256
__constant__ static const uint64_t KECCAK_RC[24] = {
    0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL,
    0x000000000000808bULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,
    0x000000000000008aULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,
    0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL, 0x8000000000008003ULL,
    0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};

__device__ __forceinline__ void keccak_f1600(uint64_t s[25]) {
#pragma unroll 1
    for (int r = 0; r < 24; r++) {
        uint64_t c0 = s[0] ^ s[5] ^ s[10] ^ s[15] ^ s[20];
        uint64_t c1 = s[1] ^ s[6] ^ s[11] ^ s[16] ^ s[21];
        uint64_t c2 = s[2] ^ s[7] ^ s[12] ^ s[17] ^ s[22];
        uint64_t c3 = s[3] ^ s[8] ^ s[13] ^ s[18] ^ s[23];
        uint64_t c4 = s[4] ^ s[9] ^ s[14] ^ s[19] ^ s[24];
        uint64_t d0 = c4 ^ rotl64(c1, 1), d1 = c0 ^ rotl64(c2, 1), d2 = c1 ^ rotl64(c3, 1), d3 = c2 ^ rotl64(c4, 1), d4 = c3 ^ rotl64(c0, 1);
        // theta + rho + pi
        uint64_t b0 = s[0] ^ d0;
        uint64_t b10 = rotl64(s[1] ^ d1, 1), b20 = rotl64(s[2] ^ d2, 62), b5 = rotl64(s[3] ^ d3, 28), b15 = rotl64(s[4] ^ d4, 27);
        uint64_t b16 = rotl64(s[5] ^ d0, 36), b1 = rotl64(s[6] ^ d1, 44), b11 = rotl64(s[7] ^ d2, 6), b21 = rotl64(s[8] ^ d3, 55), b6 = rotl64(s[9] ^ d4, 20);
        uint64_t b7 = rotl64(s[10] ^ d0, 3), b17 = rotl64(s[11] ^ d1, 10), b2 = rotl64(s[12] ^ d2, 43), b12 = rotl64(s[13] ^ d3, 25), b22 = rotl64(s[14] ^ d4, 39);
        uint64_t b23 = rotl64(s[15] ^ d0, 41), b8 = rotl64(s[16] ^ d1, 45), b18 = rotl64(s[17] ^ d2, 15), b3 = rotl64(s[18] ^ d3, 21), b13 = rotl64(s[19] ^ d4, 8);
        uint64_t b14 = rotl64(s[20] ^ d0, 18), b24 = rotl64(s[21] ^ d1, 2), b9 = rotl64(s[22] ^ d2, 61), b19 = rotl64(s[23] ^ d3, 56), b4 = rotl64(s[24] ^ d4, 14);
        // chi
        s[0] = b0 ^ (~b1 & b2); s[1] = b1 ^ (~b2 & b3); s[2] = b2 ^ (~b3 & b4); s[3] = b3 ^ (~b4 & b0); s[4] = b4 ^ (~b0 & b1);
        s[5] = b5 ^ (~b6 & b7); s[6] = b6 ^ (~b7 & b8); s[7] = b7 ^ (~b8 & b9); s[8] = b8 ^ (~b9 & b5); s[9] = b9 ^ (~b5 & b6);
        s[10] = b10 ^ (~b11 & b12); s[11] = b11 ^ (~b12 & b13); s[12] = b12 ^ (~b13 & b14); s[13] = b13 ^ (~b14 & b10); s[14] = b14 ^ (~b10 & b11);
        s[15] = b15 ^ (~b16 & b17); s[16] = b16 ^ (~b17 & b18); s[17] = b17 ^ (~b18 & b19); s[18] = b18 ^ (~b19 & b15); s[19] = b19 ^ (~b15 & b16);
        s[20] = b20 ^ (~b21 & b22); s[21] = b21 ^ (~b22 & b23); s[22] = b22 ^ (~b23 & b24); s[23] = b23 ^ (~b24 & b20); s[24] = b24 ^ (~b20 & b21);
        s[0] ^= KECCAK_RC[r];
    }
}

__device__ __forceinline__ void keccak256(const uint8_t* msg, uint32_t len, Digest& out) {
    uint64_t s[25];
#pragma unroll
    for (int i = 0; i < 25; i++) s[i] = 0;
    AlignedMsg am(msg);
    uint32_t off = 0;
    while (len - off >= 136) {
#pragma unroll
        for (int i = 0; i < 17; i++) s[i] ^= am.word(off / 8 + i);
        keccak_f1600(s);
        off += 136;
    }
    uint32_t rem = len - off;  // 0..135
#pragma unroll
    for (int i = 0; i < 17; i++) {
        uint32_t have = rem > 8u * i ? rem - 8u * i : 0;
        uint64_t w = have ? mask_low_bytes(am.word(off / 8 + i), have) : 0;
        if (rem / 8 == (uint32_t)i) w ^= 0x01ull << (8 * (rem % 8));  // Keccak (not SHA-3) domain byte
        if (i == 16) w ^= 0x8000000000000000ULL;
        s[i] ^= w;
    }
    keccak_f1600(s);
    out.w[0] = s[0]; out.w[1] = s[1]; out.w[2] = s[2]; out.w[3] = s[3];
}

// ------------------------------------------------------------------ SHA-256
__constant__ static const uint32_t SHA256_K[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be,
    0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa,
    0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85,
    0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3,
    0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f,
    0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

__device__ __forceinline__ uint32_t rotr32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

__device__ __forceinline__ void sha256_block(uint32_t h[8], uint32_t w[16]) {
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        if (i >= 16) {
            uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
            uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
            w[i & 15] = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
        }
        uint32_t S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
        uint32_t ch = (e & f) ^ (~e & g);
        uint32_t t1 = hh + S1 + ch + SHA256_K[i] + w[i & 15];
        uint32_t S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
        uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        uint32_t t2 = S0 + mj;
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// out_be[8]: digest as eight big-endian words (bit 0 of the digest = MSB of out_be[0])
__device__ __forceinline__ void sha256(const uint8_t* msg, uint32_t len, uint32_t out_be[8]) {
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    uint32_t w[16];
    uint32_t off = 0;
    // byte-wise gather: SHA-256 messages on this path are ≤ 32-byte keys
    for (;;) {
        bool final_block = off > len || len - off < 56;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            uint32_t v = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                uint32_t idx = off + 4 * i + k;
                uint32_t byte = idx < len ? msg[idx] : (idx == len ? 0x80u : 0u);
                v = (v << 8) | byte;
            }
            w[i] = v;
        }
        if (final_block) { w[14] = (uint32_t)(((uint64_t)len * 8) >> 32); w[15] = (uint32_t)(len * 8u); }
        sha256_block(h, w);
        if (final_block) break;
        off += 64;
    }
#pragma unroll
    for (int i = 0; i < 8; i++) out_be[i] = h[i];
}

}  // namespace ipcfp
