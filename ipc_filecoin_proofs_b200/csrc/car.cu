// car.cu — ipcfp_store_create_car: a block store straight from a CARv1 archive, with its sections found on the device. The CAR's bytes
// ARE the store's arena: blocks are used in place, with the varints and CIDs left between them, so by-reference offsets index the caller's
// CAR. A CAR whose section chain the device does not find (every invalid CAR) goes through ipcfp_blocks_from_car (csrc/car_parse.cpp)
// instead, over the arena already on the device, so results never depend on the path.
//
// Device path, all on the store's stream unless noted:
//   header                 decoded on the host (car_header, the host parser's own rule)
//   H2D of the CAR         into the store's block bytes in CAR_CHUNK pieces on a copy stream; chunk k is marked once chunk k + 1 has landed
//                          (a candidate reads 5 bytes before it and 6 from it)
//   k_car_mark             one thread per 32 bytes: bit s of the bitmap = a candidate CID starts at s (car_items.cuh)
//   bitmap_count64         the candidate count
//   ── host synchronisation 1: the count; the position and link arrays are sized by it
//   bitmap_scatter64       candidate positions, ascending, 64-bit (prims.cu)
//   k_car_links            one thread per (candidate, option): where its section ends, as a link to the next candidate; the head
//   ── host synchronisation 2: the links. The host follows them from the head (a few words per section, no CAR byte) to the payload's end
//   k_car_gather           one thread per section of the chain: offset, length, CID
//   store_finish (store.cu)
// The scratch is sized by the candidate count and released before the index is built; when it cannot be allocated, the CAR goes through
// the host parser like any CAR the device path does not accept.
#include <algorithm>
#include <cstring>
#include <vector>

#include "car_items.cuh"
#include "engine.cuh"
#include "prims.cuh"

namespace ipcfp {

bool car_header(const uint8_t* car, uint64_t len, uint64_t& first_section);   // car_parse.cpp

struct CarMeta {
    unsigned long long n;      // candidates
    unsigned long long head;   // the link to the section at the header's end
};
static_assert(sizeof(CarMeta) <= HW_PARSE_META_WORDS * 8, "the meta words fit their host words (HW_PARSE_META)");

// words [w0, w1) of the bitmap over the payload t[0, len); sections start at or after `first`
__global__ void __launch_bounds__(256) k_car_mark(const uint8_t* __restrict__ t, uint64_t len, uint64_t first, uint64_t w0, uint64_t w1,
                                                  uint32_t* bits) {
    const uint64_t w = w0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= w1) return;
    uint32_t b = 0;
    for (uint32_t k = 0; k < 32; k++) {
        const uint64_t p = 32 * w + k;
        if (p < len && car_candidate(t, len, first, p)) b |= 1u << k;
    }
    bits[w] = b;
}

// one thread per (candidate i, option d = 1 … 5): links[5 i + d - 1]; thread 0 also finds the head
__global__ void __launch_bounds__(256) k_car_links(const uint8_t* __restrict__ t, uint64_t len, uint64_t first, const uint64_t* __restrict__ pos,
                                                   uint64_t n, uint64_t* links, CarMeta* meta) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) meta->head = car_head(t, len, first, pos, n);
    if (k >= CAR_MAX_VARINT * n) return;
    links[k] = car_link(t, len, first, pos, n, k / CAR_MAX_VARINT, k % CAR_MAX_VARINT + 1);
}

// one thread per section k of the chain (chain[k]: the link that reaches it): its offset, length and CID
__global__ void k_car_gather(const uint8_t* __restrict__ t, const uint64_t* __restrict__ pos, const uint64_t* __restrict__ chain, uint64_t m,
                             uint64_t* offsets, uint32_t* lengths, uint8_t* cids) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m) return;
    uint64_t off;
    uint32_t blen;
    car_block(t, pos, chain[k], off, blen);
    offsets[k] = off;
    lengths[k] = blen;
    const uint8_t* c = t + off - IPCFP_CID_LEN;
    for (uint32_t b = 0; b < IPCFP_CID_LEN; b++) cids[IPCFP_CID_LEN * k + b] = c[b];
}

static const uint64_t CAR_CHUNK = 64ull << 20;   // the H2D piece: ipcfp_store_create's chunk (a multiple of 32, so chunks hold whole bitmap words)

// b = count elements on `st`; false (nothing allocated) when the device is out of memory
template <class T> static bool try_alloc(AsyncBuf<T>& b, size_t count, cudaStream_t st) {
    b.release();
    const cudaError_t e = cudaMallocAsync((void**)&b.p, (count ? count : 1) * sizeof(T), st);
    if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); b.p = nullptr; return false; }
    IPCFP_CUDA(e);
    b.st = st;
    b.n = count;
    return true;
}

// the chain from the head (host): chain[k] = the link that reaches section k; false when a link is NONE
static bool walk(const uint64_t* links, uint64_t n, uint64_t head, std::vector<uint64_t>& chain) {
    for (uint64_t cur = head; cur != CAR_LINK_TERMINAL;) {
        if (cur == CAR_LINK_NONE || chain.size() >= n) return false;   // links only go forward: at most n sections
        chain.push_back(cur);
        cur = links[CAR_MAX_VARINT * (cur >> 3) + (cur & 7) - 1];
    }
    return true;
}

// the CAR in the store's arena and its blocks indexed: on the device when the links give its section chain, else with the host parser's
// arrays (whose error, if any, is thrown)
static void blocks_on_device(Store* s, const uint8_t* car, uint64_t len, uint64_t first, uint32_t flags, ipcfp_store_json_info& info,
                             Clock::time_point t0) {
    cudaStream_t st = s->stream;
    uint8_t* t = store_alloc_arena(s, len, false);
    ChunkedCopy copy;
    std::vector<Event> timed;   // a pair around every parse kernel
    auto timed_launch = [&](auto enqueue) {
        timed.emplace_back();
        IPCFP_CUDA(cudaEventRecord(timed.back(), st));
        enqueue();
        timed.emplace_back();
        IPCFP_CUDA(cudaEventRecord(timed.back(), st));
    };
    DevBuf<uint8_t> cids_dev;
    bool accepted = false;
    {   // the scratch of the device parse: gone before the index is built
        const uint64_t nwords = (len + 31) / 32;
        AsyncBuf<uint32_t> bits;
        AsyncBuf<uint64_t> word_prefix, scratch, pos, links, chain_dev;
        AsyncBuf<CarMeta> meta;
        bool room = try_alloc(bits, nwords + 1, st) && try_alloc(word_prefix, nwords + 1, st) &&
                    try_alloc(scratch, scan_scratch_elems(nwords) + 8, st) && try_alloc(meta, 1, st);
        auto mark = [&](uint64_t k, cudaEvent_t landed) {   // chunk k, once `landed` (the next chunk's copy, or the last one's) is done
            const uint64_t w0 = k * (CAR_CHUNK / 32), w1 = std::min(nwords, (k + 1) * (CAR_CHUNK / 32));
            IPCFP_CUDA(cudaStreamWaitEvent(st, landed, 0));
            timed_launch([&] { k_car_mark<<<div_up(w1 - w0, 256), 256, 0, st>>>(t, len, first, w0, w1, bits.p); IPCFP_LAUNCH_CHECK(); });
        };
        const uint64_t n_chunks = div_up(len, CAR_CHUNK);
        cudaEvent_t landed = nullptr;
        for (uint64_t k = 0; k < n_chunks; k++) {
            landed = copy.copy(t, car, k * CAR_CHUNK, std::min(len, (k + 1) * CAR_CHUNK));
            if (!room) continue;
            if (k) mark(k - 1, landed);
            if (k + 1 == n_chunks) mark(k, landed);
        }
        IPCFP_CUDA(cudaStreamWaitEvent(st, landed, 0));   // the whole CAR is in the arena, whichever path reads it
        uint64_t* hm = s->host_words.p + HW_PARSE_META;
        uint64_t n = 0;
        if (room) {
            timed_launch([&] { bitmap_count64(bits.p, len, (uint64_t*)&meta.p->n, word_prefix.p, scratch.p, st); });
            IPCFP_CUDA(cudaMemcpyAsync(hm, meta.p, sizeof(CarMeta), cudaMemcpyDeviceToHost, st));
            IPCFP_CUDA(cudaStreamSynchronize(st));   // host synchronisation 1
            n = hm[0];
            room = try_alloc(pos, n, st) && try_alloc(links, CAR_MAX_VARINT * n, st);
        }
        PinnedArray links_h;
        if (room) {
            timed_launch([&] {
                bitmap_scatter64(bits.p, len, word_prefix.p, pos.p, st);
                k_car_links<<<div_up(CAR_MAX_VARINT * n + 1, 256), 256, 0, st>>>(t, len, first, pos.p, n, links.p, meta.p); IPCFP_LAUNCH_CHECK();
            });
            bits.release();
            word_prefix.release();
            scratch.release();
            links_h = PinnedArray(s->pool, CAR_MAX_VARINT * n * 8);
            if (n) IPCFP_CUDA(cudaMemcpyAsync(links_h.p, links.p, CAR_MAX_VARINT * n * 8, cudaMemcpyDeviceToHost, st));
            IPCFP_CUDA(cudaMemcpyAsync(hm, meta.p, sizeof(CarMeta), cudaMemcpyDeviceToHost, st));
            IPCFP_CUDA(cudaStreamSynchronize(st));   // host synchronisation 2
            links.release();
            std::vector<uint64_t> chain;
            accepted = walk(links_h.as<uint64_t>(), n, hm[1], chain) && chain.size() < 0x7fffffffull &&
                       try_alloc(chain_dev, chain.size(), st);
            if (accepted) {
                const uint64_t m = chain.size();
                info.parsed_on_device = 1;
                store_alloc_index(s, m, cids_dev);
                if (m) {
                    IPCFP_CUDA(cudaMemcpyAsync(chain_dev.p, chain.data(), m * 8, cudaMemcpyHostToDevice, st));
                    timed_launch([&] {
                        k_car_gather<<<div_up(m, 256), 256, 0, st>>>(t, pos.p, chain_dev.p, m, s->offsets.p, s->lengths.p, cids_dev.p);
                        IPCFP_LAUNCH_CHECK();
                    });
                }
                IPCFP_CUDA(cudaStreamSynchronize(st));   // the chain's host copy goes away at the end of this scope
            }
        }
    }

    ipcfp_parsed_blocks* pb = nullptr;
    std::unique_ptr<ipcfp_parsed_blocks, void (*)(ipcfp_parsed_blocks*)> keep(nullptr, ipcfp_parsed_blocks_free);
    const uint8_t* first_prefix = nullptr;
    if (accepted) {
        if (s->n) {
            uint32_t vlen;
            uint64_t L;
            car_len_at(car, first, vlen, L);   // section 0's varint: the head
            first_prefix = car + first + vlen;
        }
    } else {
        // deferred: the host parser's arrays over the arena already on the device
        const ipcfp_status hs = ipcfp_blocks_from_car(car, len, &pb);
        if (hs != IPCFP_OK) throw Error(hs, ipcfp_last_error(), ipcfp_last_error_index());
        keep.reset(pb);
        const ipcfp_witness& w = pb->blocks;
        if (w.n_blocks >= 0x7fffffffull) throw Error(IPCFP_ERR_UNSUPPORTED, "more than 2^31 blocks in one store");
        store_alloc_index(s, w.n_blocks, cids_dev);
        if (w.n_blocks) {
            IPCFP_CUDA(cudaMemcpyAsync(cids_dev.p, w.cids, w.n_blocks * IPCFP_CID_LEN, cudaMemcpyHostToDevice, st));
            IPCFP_CUDA(cudaMemcpyAsync(s->offsets.p, w.offsets, w.n_blocks * 8, cudaMemcpyHostToDevice, st));
            IPCFP_CUDA(cudaMemcpyAsync(s->lengths.p, w.lengths, w.n_blocks * 4, cudaMemcpyHostToDevice, st));
            first_prefix = w.cids;
        }
    }
    IPCFP_CUDA(cudaStreamSynchronize(st));   // the host arrays go away with `keep`; the parse's times are final
    info.ms_parse = ms_since(t0);
    if (accepted)
        for (size_t k = 0; k < timed.size(); k += 2) info.ms_kernels += elapsed_ms(timed[k], timed[k + 1]);
    store_finish(s, cids_dev.p, pb ? pb->blocks.cids : nullptr, first_prefix, flags);
}

Store* store_create_car(const uint8_t* car, uint64_t len, int device, uint32_t flags, ipcfp_store_json_info& info) {
    // the device path needs a header; everything else (and every failure) is the host parser's to report
    uint64_t first = 0;
    return store_create_parsed(
        device, flags, info, car && car_header(car, len, first),
        [&](Store* s, Clock::time_point t0) { blocks_on_device(s, car, len, first, flags, info, t0); return true; },
        [&](ipcfp_parsed_blocks** pb) { return ipcfp_blocks_from_car(car, len, pb); }, car);
}

}  // namespace ipcfp
