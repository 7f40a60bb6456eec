// ROLZ kernels (kz_rolz.cu)
#pragma once
#include "kz_common.cuh"

namespace kz {

struct RolzBlock {
    uint64_t src_off;      // input offset (forward: block data, inverse: ROLZ stream), 16-byte aligned
    uint64_t dst_off;      // output offset
    uint64_t scratch_off;  // per block scratch (rolz_scratch_bytes)
    uint32_t len;          // input length
    uint32_t cap;          // size of the destination (len(dst) of the reference call)
    int32_t data_type;     // ctx["dataType"] (internal/Global.go DataType); forward only
    uint32_t pad;
};
// result: StageResult (kz_common.cuh); forward data_type = ctx["dataType"] after the call (DetectSimpleType may set it)

// bytes of the nested rANS buffer for a ROLZ chunk of `chunk` bytes (>= the reference's max(min(2 len, 9/8 chunk), 64 KiB))
static inline __host__ __device__ size_t rolz_ans_buffer(size_t chunk) {
    const size_t c = chunk < ((size_t)4 << 20) ? chunk : ((size_t)4 << 20);
    const size_t s = 2 * c + 1024;
    return s < 65536 + 1024 ? 65536 + 1024 : s;
}
size_t rolz_scratch_bytes(size_t n);  // n = block length (forward) or destination capacity (inverse)

__global__ void rolz_forward_kernel(const uint8_t* in, const RolzBlock* blocks, int nblocks, uint8_t* scratch_all, uint8_t* out, StageResult* res);
__global__ void rolz_inverse_kernel(const uint8_t* in, const RolzBlock* blocks, int nblocks, uint8_t* scratch_all, uint8_t* out, StageResult* res);

}  // namespace kz
