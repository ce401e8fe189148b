// text_scan.cuh — the head of every device text parse (json_parse.cu, rpc_json.cu, rpc_blocks.cu): the text on the device with JP_PAD
// zero bytes behind it, the bitmap of record starts that the parser's mark kernel fills, the starts in ascending order, and the parse's
// meta words read back through the store's host words. The parser uploads the text and runs its own kernels on the starts.
#pragma once
#include <algorithm>
#include <cstring>
#include <type_traits>

#include "engine.cuh"
#include "json_parse_items.cuh"
#include "prims.cuh"

namespace ipcfp {

// Meta: the parse's device words, with the record count in `n`
template <class Meta> struct TextScan {
    static_assert(std::is_trivially_copyable<Meta>::value, "the meta words are read back as bytes");
    Store* s;
    const uint64_t len, nwords;
    AsyncBuf<char> text;                       // len + JP_PAD bytes, the pad zeroed
    AsyncBuf<uint32_t> bits, pos;              // the bitmap of record starts; the starts (pos_cap of them at most)
    AsyncBuf<uint64_t> word_prefix, scratch;   // scratch: scans of the bitmap's words or of scan_n elements, whichever is more
    AsyncBuf<Meta> meta;                       // every byte meta_fill
    TextScan(Store* st, uint64_t text_len, uint64_t pos_cap, uint64_t scan_n, int meta_fill)
        : s(st), len(text_len), nwords((text_len + 31) / 32), text(len + JP_PAD, s->stream), bits(nwords + 8, s->stream), pos(pos_cap, s->stream),
          word_prefix(nwords + 8, s->stream), scratch(scan_scratch_elems(std::max(nwords, scan_n)) + 8, s->stream), meta(1, s->stream) {
        IPCFP_CUDA(cudaMemsetAsync(text.p + len, 0, JP_PAD, s->stream));
        IPCFP_CUDA(cudaMemsetAsync(meta.p, meta_fill, sizeof(Meta), s->stream));
    }
    // mark(text, len, bits, nwords, extra...), one thread per bitmap word, sets bit p where a record starts at p; then pos = the starts
    // in ascending order and meta->n = their count
    template <class Kernel, class... Extra> void starts(Kernel mark, Extra... extra) {
        mark<<<div_up(nwords, 256), 256, 0, s->stream>>>(text.p, len, bits.p, nwords, extra...);
        IPCFP_LAUNCH_CHECK();
        bitmap_to_indices(bits.p, len, pos.p, (uint64_t*)&meta.p->n, word_prefix.p, scratch.p, s->stream);
    }
    // the meta words once everything enqueued so far has run: one host synchronisation
    Meta read() const {
        uint64_t* hm = s->host_words.p + HW_PARSE_META;
        IPCFP_CUDA(cudaMemcpyAsync(hm, meta.p, sizeof(Meta), cudaMemcpyDeviceToHost, s->stream));
        IPCFP_CUDA(cudaStreamSynchronize(s->stream));
        Meta m;
        memcpy(&m, hm, sizeof m);
        return m;
    }
};

}  // namespace ipcfp
