// EXE transform (EXECodec, v2/transform/EXECodec.go) on the GPU: one thread per block runs the logic of kz_exe_core.cuh (header parse,
// jump statistics, then the rewrite of call / jump targets whose output position depends on every earlier escape). Blocks of a batch
// run side by side; the stage declines quickly on blocks that are not executable code.
#include "kz_exe.cuh"
#include "kz_exe_core.cuh"

namespace kz {

__global__ void __launch_bounds__(32) exe_forward_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks, uint8_t* __restrict__ out,
                                                          StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const StageBlock blk = blocks[b];
    StageResult r;
    r.status = 1;
    r.out_len = 0;
    r.data_type = blk.data_type;
    r.mode = 0;
    if (blk.len != 0) {
        int dt = blk.data_type;
        const int64_t n = exec::forward(in + blk.src_off, (int64_t)blk.len, out + blk.dst_off, (int64_t)blk.cap, &dt);
        r.data_type = dt;
        if (n >= 0) {
            r.status = 0;
            r.out_len = (uint32_t)n;
        } else if (n == -2) {
            r.status = -KZ_E_PROCESS_BLOCK;
        }
    }
    res[b] = r;
}

__global__ void __launch_bounds__(32) exe_inverse_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks, uint8_t* __restrict__ out,
                                                          StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const StageBlock blk = blocks[b];
    StageResult r;
    r.status = 0;
    r.out_len = 0;
    r.data_type = 0;
    r.mode = 0;
    if (blk.len != 0 && blk.cap != 0) {
        const int64_t n = exec::inverse(in + blk.src_off, (int64_t)blk.len, out + blk.dst_off, (int64_t)blk.cap);
        if (n < 0) r.status = -KZ_E_PROCESS_BLOCK;
        else r.out_len = (uint32_t)n;
    }
    res[b] = r;
}

}  // namespace kz
