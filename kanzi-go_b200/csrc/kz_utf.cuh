// UTF transform (UTFCodec) on the GPU — declarations (kz_utf.cu). The per-block logic is kz_utf_core.cuh.
// Reference: v2/transform/UTFCodec.go (Forward :87-262, Inverse :267-383, MaxEncodedLen :386-388).
#pragma once
#include "kz_common.cuh"

namespace kz {

size_t utf_workspace(uint32_t nblocks);
cudaError_t utf_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint8_t* ws, size_t ws_bytes, StageResult* d_res,
                              cudaStream_t stream, uint64_t* launches);
cudaError_t utf_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint8_t* ws, size_t ws_bytes, StageResult* d_res,
                              cudaStream_t stream, uint64_t* launches);

}  // namespace kz
