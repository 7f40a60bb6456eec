// The incompressible-block test of kanzi's skipBlocks option (kanzi c --skip) on the GPU.
// Reference: encodingTask.encode (io/CompressedStream.go:778-800) stores a block of more than 15 bytes raw when it starts with the magic
// number of a compressed format or when ComputeFirstOrderEntropy1024 of its order-0 histogram (internal/Global.go:196-251) reaches
// entropy.INCOMPRESSIBLE_THRESHOLD. The magic number is read on the host (kz_api.cu magic_data_type) from the block heads the same
// copy brings back; these kernels give the entropy half:
//   skip_hist_kernel: one warp per tile of at most SKIP_TILE bytes, so the blocks of a batch (16 B to 1 GiB) share the GPU by size;
//     8 replicas of the 256 counters per warp in shared memory spread same-symbol atomics, then one global add per non-zero counter.
//   skip_decide_kernel: one thread per block runs the reference's integer entropy (kz_entropy_core.cuh) on the histogram.
#include "kz_entropy_core.cuh"
#include "kz_skip.cuh"

namespace kz {

__global__ void __launch_bounds__(32 * SKIP_HIST_WARPS) skip_hist_kernel(const uint8_t* __restrict__ base, const SkipTile* __restrict__ tiles,
                                                                         uint32_t ntiles, uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[SKIP_HIST_WARPS][8 * 256];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t t = blockIdx.x * SKIP_HIST_WARPS + warp;
    if (t >= ntiles) return;  // the warps of a CTA never meet
    uint32_t* H = h[warp];
    for (int i = lane; i < 8 * 256; i += 32) H[i] = 0;
    __syncwarp();
    const SkipTile T = tiles[t];
    const uint8_t* p = base + T.off;
    uint32_t* my = H + (lane & 7) * 256;
    // head bytes up to the first 16-byte boundary, then 16-byte loads, then the tail
    const uint32_t head = min(T.len, (uint32_t)((16u - ((uint32_t)(uintptr_t)p & 15u)) & 15u));
    if ((uint32_t)lane < head) atomicAdd(&my[p[lane]], 1u);
    const uint32_t n16 = (T.len - head) >> 4;
    const uint4* p4 = reinterpret_cast<const uint4*>(p + head);
    for (uint32_t i = lane; i < n16; i += 32) {
        const uint4 v = __ldg(&p4[i]);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; k++) {
            atomicAdd(&my[w[k] & 0xFF], 1u);
            atomicAdd(&my[(w[k] >> 8) & 0xFF], 1u);
            atomicAdd(&my[(w[k] >> 16) & 0xFF], 1u);
            atomicAdd(&my[w[k] >> 24], 1u);
        }
    }
    for (uint32_t i = head + (n16 << 4) + lane; i < T.len; i += 32) atomicAdd(&my[p[i]], 1u);
    __syncwarp();
    uint32_t* g = hist + (size_t)T.block * 256;
    for (int s = lane; s < 256; s += 32) {
        uint32_t c = 0;
#pragma unroll
        for (int r = 0; r < 8; r++) c += H[r * 256 + s];
        if (c) atomicAdd(&g[s], c);
    }
}

__global__ void __launch_bounds__(256) skip_decide_kernel(const uint32_t* __restrict__ hist, const uint32_t* __restrict__ len, uint32_t nblocks,
                                                          const uint32_t* __restrict__ log2tab, uint8_t* __restrict__ flag) {
    __shared__ uint32_t T[257];
    for (int i = threadIdx.x; i < 257; i += blockDim.x) T[i] = log2tab[i];
    __syncthreads();
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    flag[b] = entropy_1024(len[b], hist + (size_t)b * 256, T) >= INCOMPRESSIBLE_THRESHOLD ? 1 : 0;
}

}  // namespace kz
