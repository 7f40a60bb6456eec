// MM transform (FSDCodec: fixed step delta) on the GPU — declarations (kz_fsd.cu).
// Reference: v2/transform/FSDCodec.go (MaxEncodedLen :128-130, Forward :135-312, Inverse :317-404).
#pragma once
#include "kz_common.cuh"

namespace kz {

static const uint32_t FSD_TILE = 4096;

static inline __host__ __device__ uint32_t fsd_max_encoded_len(uint32_t n) { return n + ((n >> 4) > 64 ? (n >> 4) : 64); }
size_t fsd_workspace(uint32_t nblocks, uint32_t max_len);

cudaError_t fsd_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint32_t max_len, uint8_t* ws, size_t ws_bytes,
                              StageResult* d_res, cudaStream_t stream, uint64_t* launches);
// FSDCodec.Inverse over tiles of 32 source bytes, all blocks together (h_blocks: descriptors on the host; ws of fsd_inverse_workspace bytes)
size_t fsd_inverse_workspace(uint32_t nblocks, uint64_t total_len);
cudaError_t fsd_inverse_tiles(const uint8_t* d_in, uint8_t* d_out, const StageBlock* h_blocks, uint32_t nblocks, uint8_t* ws, size_t ws_bytes, StageResult* d_res,
                              cudaStream_t stream, uint64_t* launches);

}  // namespace kz
