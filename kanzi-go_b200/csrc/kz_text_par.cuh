// Data-parallel TEXT forward (kz_text_par.cu); the phases are kz_text_par_core.cuh.
#pragma once
#include <vector>

#include "kz_text.cuh"

namespace kz {

// upper bound of the device workspace for nblocks blocks of at most max_len bytes; bs[b]: ctx["blockSize"] of block b (sizes its hash map)
size_t text_parallel_workspace(const uint64_t* bs, uint32_t nblocks, uint32_t max_len);
// TEXT forward of the blocks text_plan_kernel let through (d_go[b] = mode | 0x100). d_res[b] is completed for the blocks done here;
// h_fallback[b] != 0: the parallel statement does not cover the block, the serial walk has to do it. Synchronises the stream.
cudaError_t text_forward_parallel(const uint8_t* d_in, uint8_t* d_out, const std::vector<StageBlock>& tb, const uint32_t* d_go, const uint64_t* bs,
                                  const void* d_sdict, const uint8_t* d_swords, int static_n, uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream,
                                  std::vector<uint32_t>& h_fallback, uint64_t* launches);

// TEXT inverse of a batch; h_fallback[b] != 0: the block is left to the serial walk (trivial blocks and every anomaly). Synchronises.
size_t text_inverse_parallel_workspace(const uint64_t* bs, uint32_t nblocks, uint32_t max_len);
cudaError_t text_inverse_parallel(const uint8_t* d_in, uint8_t* d_out, const std::vector<StageBlock>& tb, const uint64_t* bs, const void* d_sdict,
                                  const uint8_t* d_swords, int static_n, uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream,
                                  std::vector<uint32_t>& h_fallback, uint64_t* launches);

}  // namespace kz
