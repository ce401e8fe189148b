// parsed_blocks.h — the object behind an ipcfp_parsed_blocks handle, shared by its host parsers (rpc_blocks_parse.cpp: the blocks of
// ChainReadObj responses, in a blob of their own; car_parse.cpp: the sections of a CAR, indexing the caller's buffer, blob empty), so that
// one ipcfp_parsed_blocks_free releases either.
#pragma once
#include <cstdint>
#include <vector>

#include "../../include/ipcfp.h"

struct ParsedBlocksBox {
    ipcfp_parsed_blocks pub;   // FIRST member: the handle is a pointer to it
    std::vector<uint8_t> cids, blob;
    std::vector<uint64_t> offsets;
    std::vector<uint32_t> lengths;
};
