// Order-0 entropy of a block from its histogram (internal/Global.go:175-214), host/device shared: the MM transform's distance test
// (kz_fsd.cu) and the incompressible-block test of kanzi's skipBlocks option (kz_skip.cu) run it on the device,
// tests/host/entropy_core_host.cpp on the CPU.
#pragma once
#include <stdint.h>

#include <cmath>

#if defined(__CUDACC__)
#define KZE_HD __host__ __device__ __forceinline__
#else
#define KZE_HD inline
#endif

namespace kz {

// entropy.INCOMPRESSIBLE_THRESHOLD (entropy/EntropyUtils.go:26): encodingTask.encode stores a block whose order-0 entropy reaches it
// (io/CompressedStream.go:786-798)
constexpr int INCOMPRESSIBLE_THRESHOLD = 973;

// internal/Global.go:60-93 LOG2_4096[i] = round(4096 * log2(i)) (entries 0 and 1 are 0): a data table of the reference, regenerated from
// its definition (checked entry by entry against the reference's table when this was written)
inline const uint32_t* host_log2_4096() {
    static uint32_t tab[257];
    static bool init = false;
    if (!init) {
        tab[0] = 0;
        for (int k = 1; k <= 256; k++) tab[k] = (uint32_t)(4096.0 * std::log2((double)k) + 0.5);
        init = true;
    }
    return tab;
}

// internal/Global.go:175-191 Log2ScaledBy1024
KZE_HD uint32_t log2_scaled_1024(uint32_t x, const uint32_t* T) {
    if (x < 256) return (T[x] + 2) >> 2;
#if defined(__CUDA_ARCH__)
    const uint32_t lg = 31u - (uint32_t)__clz((int)x);
#else
    const uint32_t lg = 31u - (uint32_t)__builtin_clz(x);
#endif
    if ((x & (x - 1)) == 0) return lg << 10;
    return ((lg - 7) * 1024) + ((T[x >> (lg - 7)] + 2) >> 2);
}

// internal/Global.go:196-214 ComputeFirstOrderEntropy1024
KZE_HD int entropy_1024(uint32_t block_len, const uint32_t* histo, const uint32_t* T) {
    if (block_len == 0) return 0;
    unsigned long long sum = 0;
    const uint32_t ll = log2_scaled_1024(block_len, T);
    for (int i = 0; i < 256; i++) {
        if (histo[i] == 0) continue;
        const uint32_t l = log2_scaled_1024(histo[i], T);
        sum += ((unsigned long long)histo[i] * (unsigned long long)(ll - l)) >> 3;
    }
    return (int)(sum / (unsigned long long)block_len);
}

}  // namespace kz
