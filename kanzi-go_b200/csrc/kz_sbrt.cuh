// Declarations of the sort-by-rank kernels (kz_sbrt.cu).
#pragma once
#include "kz_common.cuh"

namespace kz {

static const int SBRT_SEG_BYTES = 4096;

struct SbrtBlock {
    uint64_t src_off;   // byte offsets of the block inside the source / destination buffers (16-byte aligned)
    uint64_t dst_off;
    uint32_t len;
    uint32_t seg_base;  // index of the block's first segment in the segment tables
    uint32_t active;    // 0: skip the block (COPY block / transform already skipped)
    uint32_t pad;
};

__global__ void sbrt_last2_kernel(const uint8_t* data, const SbrtBlock* blocks, int32_t* table);
__global__ void sbrt_carry_kernel(const SbrtBlock* blocks, int32_t* table);
// ranks of every segment (seg_block[s] = block of segment s); mode: 1 = MTFT, 2 = RANK; max_len = longest block of the batch (blocks up to
// 16 MiB take 32-bit keys, longer ones 64-bit keys)
void sbrt_rank_launch(const uint8_t* data, const SbrtBlock* d_blocks, int mode, const uint32_t* seg_block, uint32_t nsegs, const int32_t* table,
                      uint8_t* out, uint32_t max_len, cudaStream_t stream);
// mode: 1 = MTFT, 2 = RANK; max_len = longest block of the batch (blocks up to 16 MiB take the 4-warp kernel, longer ones the one-warp kernel)
void sbrt_inverse_launch_len(const uint8_t* data, const SbrtBlock* d_blocks, int nblocks, int mode, uint8_t* out, uint32_t max_len, cudaStream_t stream);

}  // namespace kz
