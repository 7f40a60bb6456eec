// TEXT transform (TextCodec, encoding 2) on the GPU — declarations (kz_text.cu). The state machine itself is kz_text_core.cuh.
// Reference: v2/transform/TextCodec.go (wrapper :549-592, textCodec2 :1137-1724).
#pragma once
#include <vector>

#include "kz_common.cuh"

namespace kz {

bool text_available();  // false when the library was built without the static dictionary (kanzi-go_b200/gen_text_dict.py)

// Every block of a batch has a hash map of its own, sized by its stream's ctx["blockSize"] bs[b]: 2^clamp(log2(bs[b] / 32), 13, 24) slots.
// The maps of a batch lie back to back: block b's starts at slot off[b] (a prefix sum) and has lg[b] bits of index. Returns the slots of all.
uint64_t text_map_layout(const uint64_t* bs, uint32_t nblocks, std::vector<uint64_t>& off, std::vector<uint32_t>& lg);

// device workspace for a batch; bs: ctx["blockSize"] of every block (host array of nblocks entries)
size_t text_workspace(const uint64_t* bs, uint32_t nblocks, uint32_t max_len);          // forward (serial + data-parallel scratch)
size_t text_workspace_serial(const uint64_t* bs, uint32_t nblocks);                     // serial walk only
size_t text_workspace_inverse(const uint64_t* bs, uint32_t nblocks, uint32_t max_len);  // inverse (serial + data-parallel scratch)

// h_blocks: host copy of d_blocks (the data-parallel path builds its own descriptors from it). *serial (when given) += the blocks the
// data-parallel path handed to the serial walk.
cudaError_t text_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, const StageBlock* h_blocks, uint32_t nblocks, uint32_t max_len,
                               const uint64_t* bs, uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream, uint64_t* launches,
                               uint64_t* serial = nullptr);
cudaError_t text_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, const StageBlock* h_blocks, uint32_t nblocks, const uint64_t* bs,
                               uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream, uint64_t* launches, uint64_t* serial = nullptr);

}  // namespace kz
