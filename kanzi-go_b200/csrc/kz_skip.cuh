// Declarations of the incompressible-block test of kanzi's skipBlocks option (kz_skip.cu).
#pragma once
#include "kz_common.cuh"

namespace kz {

// One warp's share of the histogram pass: len bytes at off (any alignment) of block `block`. A block is cut into tiles of at most
// SKIP_TILE bytes, so a large block spreads over many warps and CTAs while a small one takes one warp.
struct SkipTile {
    uint64_t off;
    uint32_t len;
    uint32_t block;
};
constexpr uint32_t SKIP_TILE = 32u << 10;
constexpr int SKIP_HIST_WARPS = 4;  // warps per CTA of skip_hist_kernel

// hist[block * 256 + s] += occurrences of byte s in every tile (hist zeroed by the caller)
__global__ void skip_hist_kernel(const uint8_t* base, const SkipTile* tiles, uint32_t ntiles, uint32_t* hist);
// flag[b] = 1 when the order-0 entropy of block b (len[b] bytes, histogram hist[b * 256 ...]) reaches INCOMPRESSIBLE_THRESHOLD, else 0;
// log2tab = LOG2_4096 (257 entries)
__global__ void skip_decide_kernel(const uint32_t* hist, const uint32_t* len, uint32_t nblocks, const uint32_t* log2tab, uint8_t* flag);

}  // namespace kz
