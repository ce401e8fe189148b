// car_items.cuh — per-item functions of the device CAR parser of ipcfp_store_create_car (csrc/car.cu): the sections of a CARv1 found in
// the bytes already copied to the store's arena, giving the block arrays csrc/car_parse.cpp (ipcfp_blocks_from_car) returns. They live in
// a header so that tests/host_fuzz/emu_car.cu runs the very same code on the CPU against car_parse.cpp.
//
// A CANDIDATE is a position s of the payload where a section's CID may start:
//   * the 6 bytes at s are the prefix of a CID of the store's form: 01 | codec < 0x80 | a minimal 3-byte multihash code | 20;
//   * an OPTION of s exists: a position q in [s - 5, s) (and at or after the header's end) where a minimal varint L of at most 5 bytes
//     (a longer one would frame a block of 2^32 bytes or more) ends exactly at s, with L >= 38 and s + L inside the payload.
// Candidates are CID starts, not section starts, because one CID start can have several options: the varint byte in front of a real
// section's L (the last byte of the block before, high bit set in half of all cases) forms a longer valid varint ending at the same s.
// Every section of a CAR the host parser accepts without an error gives a candidate, with its start among the options. But raw bytes
// inside a block can form a candidate too: ordinary CBOR such as 01 18 cc 82 58 20 (an integer, then an array whose first item is a
// 32-byte string) has the form. So the candidates are not the chain; the chain is found by following LINKS:
//   * the link of option q of candidate i is where that section ends, e = s + L: TERMINAL when e is the payload's end, else (j, e) when
//     e is an option of candidate j (the first candidate after e, found by binary search), else NONE;
//   * the HEAD is the candidate whose option is the header's end.
// Following links from the head visits exactly the sections the host parser walks: each varint is read from its start, is minimal and
// ends at a CID of the store's form, and the next section starts where this one ends. Candidates inside blocks are never visited. A walk
// that meets NONE (a section whose next one is not of the candidate form: a fault, a non-minimal varint, a CID the store refuses, a
// block of 2^32 bytes or more) sends the CAR to the host parser, which reports the fault.
//
// A CID embedded in CBOR (58 27 00 01 71 …) is never a candidate: the byte before 01 is 00, and no minimal varint of 38 or more ends in 00.
//
// Every buffer these functions read holds the payload followed by at least CAR_PAD readable bytes.
#pragma once
#include "common.cuh"

namespace ipcfp {

#define CAR_FN __host__ __device__ __forceinline__
#define CAR_PAD 16u             // bytes read past a candidate's start (the 6-byte prefix), rounded up
#define CAR_MIN_SECTION 39u     // the shortest section: a one-byte varint and a 38-byte CID with an empty block
#define CAR_MAX_VARINT 5u

// the varint at t[p]: true when it is minimal and at most CAR_MAX_VARINT bytes long (reads at most 5 bytes; the caller bounds them)
CAR_FN bool car_len_at(const uint8_t* t, uint64_t p, uint32_t& vlen, uint64_t& L) {
    L = 0;
    for (uint32_t k = 0; k < CAR_MAX_VARINT; k++) {
        const uint8_t b = t[p + k];
        L |= (uint64_t)(b & 0x7f) << (7 * k);
        if (!(b & 0x80)) { vlen = k + 1; return k == 0 || b != 0; }
    }
    return false;
}

// the 6 bytes at c are the prefix of a 38-byte CID of the store's form
CAR_FN bool car_cid_prefix(const uint8_t* c) {
    return c[0] == 0x01 && c[1] < 0x80 && (c[2] & 0x80) && (c[3] & 0x80) && c[4] && c[4] < 0x80 && c[5] == 0x20;
}

// q is an option of the CID start s in the payload t[0, len): the minimal varint at q ends at s, L >= 38, s + L <= len (reads [q, s))
CAR_FN bool car_option(const uint8_t* t, uint64_t len, uint64_t q, uint64_t s, uint64_t& L) {
    uint32_t vlen;
    return car_len_at(t, q, vlen, L) && q + vlen == s && L >= IPCFP_CID_LEN && L <= len - s;
}

// the first option of s is at or after `first` (the header's end), the last at s - 1
CAR_FN uint64_t car_options_from(uint64_t first, uint64_t s) { return s - first > CAR_MAX_VARINT ? s - CAR_MAX_VARINT : first; }

// a candidate CID starts at s of the payload t[0, len) whose sections start at or after `first` (reads [s - 5, s + 6))
CAR_FN bool car_candidate(const uint8_t* t, uint64_t len, uint64_t first, uint64_t s) {
    if (s <= first || len - s < 6 || t[s] != 0x01 || t[s - 1] >= 0x80 || !car_cid_prefix(t + s)) return false;
    uint64_t L;
    for (uint64_t q = car_options_from(first, s); q < s; q++)
        if (car_option(t, len, q, s, L)) return true;
    return false;
}

#define CAR_LINK_NONE (~0ull)
#define CAR_LINK_TERMINAL (~1ull)
// a link to option q = pos[j] - d of candidate j, d in 1 … 5
CAR_FN uint64_t car_link_to(uint64_t j, uint64_t d) { return (j << 3) | d; }

// the first index of pos[0, n) (ascending) whose position is greater than e
CAR_FN uint64_t car_after(const uint64_t* pos, uint64_t n, uint64_t e) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        if (pos[mid] > e) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// the link to the section that starts at e: TERMINAL at the payload's end, (j, pos[j] - e) when e is an option of candidate j, else NONE
CAR_FN uint64_t car_link_at(const uint8_t* t, uint64_t len, const uint64_t* pos, uint64_t n, uint64_t e) {
    if (e == len) return CAR_LINK_TERMINAL;
    const uint64_t j = car_after(pos, n, e);
    uint64_t L;
    if (j >= n || pos[j] - e > CAR_MAX_VARINT || !car_option(t, len, e, pos[j], L)) return CAR_LINK_NONE;
    return car_link_to(j, pos[j] - e);
}

// the head: the link to the section at the header's end
CAR_FN uint64_t car_head(const uint8_t* t, uint64_t len, uint64_t first, const uint64_t* pos, uint64_t n) {
    return car_link_at(t, len, pos, n, first);
}

// the link of option q = pos[i] - d of candidate i (see the banner); NONE when q is no option
CAR_FN uint64_t car_link(const uint8_t* t, uint64_t len, uint64_t first, const uint64_t* pos, uint64_t n, uint64_t i, uint64_t d) {
    const uint64_t s = pos[i];
    uint64_t L;
    if (d > s - first || !car_option(t, len, s - d, s, L) || L - IPCFP_CID_LEN > 0xffffffffull) return CAR_LINK_NONE;
    return car_link_at(t, len, pos, n, s + L);
}

// the section of a link: its block t[off, off + blen) (the CID is the 38 bytes in front of it)
CAR_FN void car_block(const uint8_t* t, const uint64_t* pos, uint64_t link, uint64_t& off, uint32_t& blen) {
    const uint64_t s = pos[link >> 3];
    uint32_t vlen;
    uint64_t L;
    car_len_at(t, s - (link & 7), vlen, L);
    off = s + IPCFP_CID_LEN;
    blen = (uint32_t)(L - IPCFP_CID_LEN);
}

}  // namespace ipcfp
