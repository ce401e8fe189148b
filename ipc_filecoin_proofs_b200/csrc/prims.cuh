// prims.cuh — small device-wide primitives written for this engine (no CUB/Thrust):
// exclusive scan, bitmap → ordered index list, stable LSD radix sort of (u32 key, u32 value), and on top of them the sort + unique
// of a list of CIDs.
// They implement what the reference gets from BTreeSet / Vec ordering on the CPU
// (common/witness.rs:10,30-32; proofs/generator.rs:34,85-88; events/utils.rs:56-91).
#pragma once
#include "common.cuh"

namespace ipcfp {

// out[i] = sum_{j<i} in[j] (u64 accumulators); *total_dev (device u64) receives the grand total.
// scratch must hold scan_scratch_elems(n) u64.
size_t scan_scratch_elems(uint64_t n);
void exclusive_scan_u32(const uint32_t* in, uint64_t* out, uint64_t n, uint64_t* total_dev, uint64_t* scratch, cudaStream_t st);

// Ordered list of set-bit positions of a bitmap of nbits bits (nbits rounded up to 32 must be allocated).
// word_prefix: u64[nwords] scratch. out: u32[≥ popcount]. *total_dev receives the count.
void bitmap_to_indices(const uint32_t* bits, uint64_t nbits, uint32_t* out, uint64_t* total_dev, uint64_t* word_prefix,
                       uint64_t* scratch, cudaStream_t st);
// The same in two steps, with 64-bit positions (bitmaps of 2^32 bits or more), so that the caller can size `out` by the count:
// bitmap_count64 sets word_prefix and *total_dev; bitmap_scatter64 then writes the positions (out: u64[total]).
void bitmap_count64(const uint32_t* bits, uint64_t nbits, uint64_t* total_dev, uint64_t* word_prefix, uint64_t* scratch, cudaStream_t st);
void bitmap_scatter64(const uint32_t* bits, uint64_t nbits, const uint64_t* word_prefix, uint64_t* out, cudaStream_t st);

// Stable radix sort of n (key,val) pairs by the `nbits` low bits of key (8-bit digits, LSD).
// keys/vals are sorted in place using the alt buffers as ping-pong space.
// hist: u32[256 * radix_blocks(n) + 256] scratch.
unsigned radix_blocks(uint64_t n);
void radix_sort_pairs(uint32_t* keys, uint32_t* vals, uint32_t* keys_alt, uint32_t* vals_alt, uint64_t n, int nbits,
                      uint32_t* hist, uint64_t* scan_tmp, uint64_t* scratch, cudaStream_t st);

// n 38-byte CIDs (device memory) ordered by digest bytes 0-3 and then all 38 bytes, duplicates removed, into out (room for n); returns
// the count and synchronises st. Among CIDs of one 6-byte prefix that is the raw byte order, which is `Cid` order; across prefixes it
// is not (the varint multihash code does not sort bytewise): *mixed = the first position whose prefix differs from entry 0's
// (UINT64_MAX: none), and such a list is then put in `Cid` order on the host with sort_cids_host.
uint64_t sort_unique_cids(cudaStream_t st, const void* cids, uint64_t n, void* out, uint64_t* mixed);
// a list of 38-byte CIDs (n*38) into `Cid` order on the host (stable)
void sort_cids_host(std::vector<uint8_t>& cids);

}  // namespace ipcfp
