// CPU harness of the per-stream block sizes of the many-stream entry points (kanzi-go_b200/csrc/kz_stream_plan.h): block cutting with a
// block size per stream, and the decompression pass plan with a block size per block, for tests/test_stream_plan_sizes_host.py.
#include <cstdint>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_stream_plan.h"

extern "C" {
// Cuts ns streams, stream s into blocks of block_size[s]; out_off / out_len get the blocks (room for all of them), out_first ns + 1
// entries. Returns the number of blocks.
uint32_t cut_blocks_sizes(const uint64_t* src_off, const uint64_t* src_len, uint32_t ns, const uint32_t* block_size, uint64_t* out_off, uint32_t* out_len,
                          uint32_t* out_first) {
    const kz::BlockList L = kz::cut_blocks(src_off, src_len, ns, block_size);
    for (uint32_t b = 0; b < L.size(); b++) out_off[b] = L.off[b], out_len[b] = L.len[b];
    for (uint32_t s = 0; s <= ns; s++) out_first[s] = L.first[s];
    return L.size();
}

// The decompression passes of n blocks, block b of block size block_size[b]: out_order (n entries) the blocks pass after pass, out_first
// (passes + 1 entries) where each pass starts in it, out_stride each pass's stride. Returns the number of passes; *scratch = the plan's.
uint32_t plan_decompress_sizes(const uint32_t* block_size, uint32_t n, uint64_t budget, uint32_t* out_order, uint32_t* out_first, uint64_t* out_stride,
                               uint32_t* out_pass, uint32_t* out_slot, uint64_t* scratch) {
    const kz::PassPlan P = kz::plan_decompress_passes(std::vector<uint32_t>(block_size, block_size + n), budget);
    for (uint32_t i = 0; i < n; i++) out_order[i] = P.order[i], out_pass[i] = P.pass[i], out_slot[i] = P.slot[i];
    for (uint32_t p = 0; p <= P.npasses(); p++) out_first[p] = P.first[p];
    for (uint32_t p = 0; p < P.npasses(); p++) out_stride[p] = P.stride[p];
    *scratch = P.scratch;
    return P.npasses();
}

// The same, with one block size for all blocks through the uniform form (the plan of a group before streams of different block sizes
// could share it).
uint32_t plan_decompress_uniform(uint32_t n, uint32_t block_size, uint64_t budget, uint32_t* out_order, uint32_t* out_first, uint64_t* out_stride,
                                 uint32_t* out_pass, uint32_t* out_slot, uint64_t* scratch) {
    const kz::PassPlan P = kz::plan_decompress_passes(n, kz::decompress_slot(block_size), kz::decompress_block_cost(block_size), budget);
    for (uint32_t i = 0; i < n; i++) out_order[i] = P.order[i], out_pass[i] = P.pass[i], out_slot[i] = P.slot[i];
    for (uint32_t p = 0; p <= P.npasses(); p++) out_first[p] = P.first[p];
    for (uint32_t p = 0; p < P.npasses(); p++) out_stride[p] = P.stride[p];
    *scratch = P.scratch;
    return P.npasses();
}

uint64_t decompress_slot(uint32_t block_size) { return kz::decompress_slot(block_size); }
uint64_t decompress_cost(uint32_t block_size) { return kz::decompress_block_cost(block_size); }
}
