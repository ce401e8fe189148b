// car_parse.cpp — ipcfp_blocks_from_car: the block arrays of ipcfp_store_create from a CARv1 archive held in memory, in the boundary
// language (plain C++, built with g++, no CUDA).
//
// CARv1 (https://ipld.io/specs/transport/car/carv1/): a varint H, a DAG-CBOR header of H bytes {"roots": [CID…], "version": 1}, then
// sections to the end of the buffer, each a varint L and L bytes: a CID followed by its block. Blocks are returned in place: the offsets
// index the caller's buffer, so the CAR itself can be the store's blob. This parser defines the semantics of include/ipcfp.h; the device
// path of ipcfp_store_create_car (csrc/car.cu) accepts a subset of its inputs and must give the same arrays on them.
//
// Strict choices: varints are minimal unsigned LEB128 below 2^63 (what multiformats/go-varint accepts), CBOR heads are minimal and of
// definite length, L = 0 is an error (not an end marker), and only version 1 is read.
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/ipcfp.h"
#include "parsed_blocks.h"

namespace ipcfp {
void set_last_error(const std::string& msg, uint64_t index);   // capi.cu

// a minimal unsigned LEB128 varint below 2^63 at p[at, end); false when it is truncated, longer than 9 bytes or not minimal
bool car_varint(const uint8_t* p, uint64_t end, uint64_t& at, uint64_t& v) {
    v = 0;
    for (uint32_t k = 0; k < 9; k++) {
        if (at >= end) return false;
        const uint8_t b = p[at++];
        v |= (uint64_t)(b & 0x7f) << (7 * k);
        if (!(b & 0x80)) return k == 0 || b != 0;
    }
    return false;
}
}  // namespace ipcfp

namespace {

using ipcfp::car_varint;

struct AtIndex { ipcfp_status st; uint64_t index; };
[[noreturn]] void fail(ipcfp_status st, uint64_t index = UINT64_MAX) { throw AtIndex{st, index}; }

// a minimal CBOR head of definite length in p[at, end): its major type and argument
struct Cbor {
    const uint8_t* p;
    uint64_t at, end;
    bool head(uint32_t& major, uint64_t& arg) {
        if (at >= end) return false;
        const uint8_t b = p[at++];
        major = b >> 5;
        const uint32_t ai = b & 31;
        if (ai < 24) { arg = ai; return true; }
        if (ai > 27) return false;   // reserved, or an indefinite length
        const uint32_t nb = 1u << (ai - 24);
        if (end - at < nb) return false;
        arg = 0;
        for (uint32_t k = 0; k < nb; k++) arg = arg << 8 | p[at++];
        static const uint64_t least[4] = {24, 1ull << 8, 1ull << 16, 1ull << 32};
        return arg >= least[ai - 24];
    }
    bool expect(uint32_t major, uint64_t& arg) { uint32_t m; return head(m, arg) && m == major; }
    bool skip(uint64_t n) { if (end - at < n) return false; at += n; return true; }
};

// the header: a varint H >= 1, then exactly one DAG-CBOR map of H bytes with the keys "roots" (an array of tag-42 byte strings whose first
// byte is 0x00) and "version" (an unsigned integer), each once, in either order. Entries are read in file order; a version other than 1
// is IPCFP_ERR_UNSUPPORTED where it is read, any other fault IPCFP_ERR_DECODE. Returns the offset of the first section.
uint64_t read_header(const uint8_t* car, uint64_t len) {
    uint64_t at = 0, h = 0;
    if (!car_varint(car, len, at, h) || h == 0 || h > len - at) fail(IPCFP_ERR_DECODE);
    Cbor c{car, at, at + h};
    uint64_t n_entries;
    if (!c.expect(5, n_entries)) fail(IPCFP_ERR_DECODE);
    bool have_roots = false, have_version = false;
    for (uint64_t e = 0; e < n_entries; e++) {
        uint64_t kl;
        if (!c.expect(3, kl) || kl > c.end - c.at) fail(IPCFP_ERR_DECODE);
        const char* key = (const char*)car + c.at;
        c.at += kl;
        if (kl == 7 && !memcmp(key, "version", 7)) {
            uint64_t v;
            if (have_version || !c.expect(0, v)) fail(IPCFP_ERR_DECODE);
            if (v != 1) fail(IPCFP_ERR_UNSUPPORTED);
            have_version = true;
        } else if (kl == 5 && !memcmp(key, "roots", 5)) {
            uint64_t n_roots;
            if (have_roots || !c.expect(4, n_roots)) fail(IPCFP_ERR_DECODE);
            for (uint64_t r = 0; r < n_roots; r++) {
                uint64_t tag, bl;
                if (!c.expect(6, tag) || tag != 42 || !c.expect(2, bl) || bl == 0 || bl > c.end - c.at || car[c.at] != 0x00) fail(IPCFP_ERR_DECODE);
                c.at += bl;
            }
            have_roots = true;
        } else fail(IPCFP_ERR_DECODE);
    }
    if (c.at != c.end || !have_roots || !have_version) fail(IPCFP_ERR_DECODE);
    return c.end;
}

// the CID at the start of section bytes s[0, L): IPCFP_ERR_DECODE when it does not decode under the CID spec, IPCFP_ERR_UNSUPPORTED when
// it is not the store's form (CIDv1 with a one-byte codec, a three-byte multihash code and a 32-byte digest: 38 bytes)
void read_cid(const uint8_t* s, uint64_t L, uint64_t k) {
    if (L >= 2 && s[0] == 0x12 && s[1] == 0x20) fail(L >= 34 ? IPCFP_ERR_UNSUPPORTED : IPCFP_ERR_DECODE, k);   // CIDv0
    uint64_t at = 0, version, codec, code, size;
    if (!car_varint(s, L, at, version) || version != 1) fail(IPCFP_ERR_DECODE, k);
    if (!car_varint(s, L, at, codec)) fail(IPCFP_ERR_DECODE, k);
    const uint64_t at_code = at;
    if (!car_varint(s, L, at, code)) fail(IPCFP_ERR_DECODE, k);
    const uint64_t code_bytes = at - at_code;
    if (!car_varint(s, L, at, size) || size > L - at) fail(IPCFP_ERR_DECODE, k);
    if (at_code != 2 || code_bytes != 3 || size != 32) fail(IPCFP_ERR_UNSUPPORTED, k);
}

using ParsedBlocks = ParsedBlocksBox;   // released by ipcfp_parsed_blocks_free (rpc_blocks_parse.cpp)

void build(ParsedBlocks& P, const uint8_t* car, uint64_t len) {
    uint64_t at = read_header(car, len);
    for (uint64_t k = 0; at < len; k++) {
        uint64_t L;
        if (!car_varint(car, len, at, L) || L == 0 || L > len - at) fail(IPCFP_ERR_DECODE, k);
        read_cid(car + at, L, k);
        if (L - IPCFP_CID_LEN > UINT32_MAX) fail(IPCFP_ERR_UNSUPPORTED, k);   // ipcfp_store_create's lengths are u32
        P.cids.insert(P.cids.end(), car + at, car + at + IPCFP_CID_LEN);
        P.offsets.push_back(at + IPCFP_CID_LEN);
        P.lengths.push_back((uint32_t)(L - IPCFP_CID_LEN));
        at += L;
    }
    ipcfp_witness& w = P.pub.blocks;
    w.n_blocks = P.lengths.size();
    w.cids = P.cids.data();
    w.offsets = P.offsets.data();
    w.lengths = P.lengths.data();
    w.blob = nullptr;
    w.blob_size = len;
}

}  // namespace

namespace ipcfp {
// the header rule of ipcfp_blocks_from_car alone (the device path of ipcfp_store_create_car decodes the header with it): true with the
// offset of the first section, false when the header is refused (ipcfp_blocks_from_car then gives the status)
bool car_header(const uint8_t* car, uint64_t len, uint64_t& first_section) {
    try { first_section = read_header(car, len); return true; }
    catch (const AtIndex&) { return false; }
}
}  // namespace ipcfp

extern "C" {

ipcfp_status ipcfp_blocks_from_car(const uint8_t* car, uint64_t len, ipcfp_parsed_blocks** out) {
    ipcfp_status st = IPCFP_OK;
    uint64_t index = UINT64_MAX;
    if (out) *out = nullptr;
    try {
        if (!out || !car) fail(IPCFP_ERR_INVALID_ARG);
        std::unique_ptr<ParsedBlocks> P(new ParsedBlocks());
        build(*P, car, len);
        *out = &P.release()->pub;
    } catch (const AtIndex& f) {
        st = f.st;
        index = f.index;
    } catch (const std::bad_alloc&) {
        st = IPCFP_ERR_INVALID_ARG;
    }
    ipcfp::set_last_error(st == IPCFP_OK ? ""
                          : st == IPCFP_ERR_INVALID_ARG ? "ipcfp_blocks_from_car: null argument (or out of host memory)"
                          : index == UINT64_MAX ? (st == IPCFP_ERR_UNSUPPORTED ? "ipcfp_blocks_from_car: not a CARv1 (header version is not 1)"
                                                                               : "ipcfp_blocks_from_car: malformed CAR header")
                          : st == IPCFP_ERR_UNSUPPORTED ? "ipcfp_blocks_from_car: a section's CID is not a 38-byte CIDv1 with a 32-byte digest, or its block is 4 GiB or more"
                                                        : "ipcfp_blocks_from_car: malformed section (length, bounds or CID)",
                          index);
    return st;
}

}  // extern "C"
