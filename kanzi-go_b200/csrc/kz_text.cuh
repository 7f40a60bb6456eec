// TEXT transform (TextCodec, encoding 2) on the GPU — declarations (kz_text.cu). The state machine itself is kz_text_core.cuh.
// Reference: v2/transform/TextCodec.go (wrapper :549-592, textCodec2 :1137-1724).
#pragma once
#include "kz_common.cuh"

namespace kz {

bool text_available();  // false when the library was built without the static dictionary (kanzi-go_b200/gen_text_dict.py)
// device workspace for a batch; stream_block_size = ctx["blockSize"] (sizes the hash map: 2^clamp(log2(bs / 32), 13, 24) slots)
size_t text_workspace(uint32_t nblocks, uint64_t stream_block_size, uint32_t max_len);  // forward (serial + data-parallel scratch)
size_t text_workspace_serial(uint32_t nblocks, uint64_t stream_block_size);          // serial walk only
size_t text_workspace_inverse(uint32_t nblocks, uint64_t stream_block_size, uint32_t max_len);  // inverse (serial + data-parallel scratch)

// h_blocks: host copy of d_blocks (the data-parallel path builds its own descriptors from it)
cudaError_t text_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, const StageBlock* h_blocks, uint32_t nblocks, uint32_t max_len,
                               uint64_t stream_block_size, uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream, uint64_t* launches);
cudaError_t text_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, const StageBlock* h_blocks, uint32_t nblocks, uint64_t stream_block_size,
                               uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream, uint64_t* launches);

}  // namespace kz
