// EXE transform (EXECodec) on the GPU — declarations (kz_exe.cu). The per-block logic is kz_exe_core.cuh.
#pragma once
#include "kz_common.cuh"

namespace kz {

__global__ void exe_forward_kernel(const uint8_t* in, const StageBlock* blocks, int nblocks, uint8_t* out, StageResult* res);
__global__ void exe_inverse_kernel(const uint8_t* in, const StageBlock* blocks, int nblocks, uint8_t* out, StageResult* res);

}  // namespace kz
