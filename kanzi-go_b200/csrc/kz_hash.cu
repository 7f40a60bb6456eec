// Block checksums: XXHash32 / XXHash64 (kanzi -x 32 / -x 64) on sm_90a.
//
// Reference: hash/XXHash32.go:51-97, hash/XXHash64.go (same structure with 64-bit lanes), used by
// encodingTask.encode (io/CompressedStream.go:753-760: hash of the ORIGINAL block, seed = bitstream type "KANZ")
// and decodingTask.decode (:1990-2006: hash of the decoded block compared with the transmitted value).
//
// The hash is four independent accumulator chains over 16-byte (32-bit variant) or 32-byte (64-bit variant) stripes,
// v = rotl(v + x * P2, r) * P1: one WARP per block, lane k < 4 owns accumulator k and walks its chain with the loads of
// the next 16 stripes already in flight (two register batches); blocks are hashed concurrently. The chain is the
// format's limit: 4 MiB / 16 B = 262144 dependent rounds per block. The XXH64 round functions are kz_xxh64_core.cuh's.
#include "kz_hash.cuh"
#include "kz_xxh64_core.cuh"

namespace kz {

KZ_D uint32_t rotl32(uint32_t x, int r) { return __funnelshift_l(x, x, r); }

KZ_D uint32_t ld32le(const uint8_t* p, bool aligned) {
    if (aligned) return *reinterpret_cast<const uint32_t*>(p);
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
KZ_D uint64_t ld64le(const uint8_t* p, bool aligned) {
    if (aligned) return *reinterpret_cast<const uint64_t*>(p);
    return (uint64_t)ld32le(p, false) | ((uint64_t)ld32le(p + 4, false) << 32);
}

static const uint32_t P32_1 = 2654435761u, P32_2 = 2246822519u, P32_3 = 3266489917u, P32_4 = 668265263u, P32_5 = 374761393u;

static const int HB = 16;  // stripes per register batch

KZ_D uint32_t xxh32_block(const uint8_t* __restrict__ p, uint32_t len, uint32_t seed, int lane) {
    const bool al = (reinterpret_cast<uintptr_t>(p) & 3) == 0;
    uint32_t n = 0;
    uint32_t h;
    if (len >= 16) {
        const uint32_t stripes = len >> 4;
        uint32_t v = lane == 0 ? seed + P32_1 + P32_2 : (lane == 1 ? seed + P32_2 : (lane == 2 ? seed : seed - P32_1));
        if (lane < 4) {
            const uint8_t* q = p + 4 * lane;
            uint32_t a[HB], b[HB];
            uint32_t s = 0;
            const uint32_t full = stripes / (2 * HB) * (2 * HB);
            if (full) {
#pragma unroll
                for (int j = 0; j < HB; j++) a[j] = ld32le(q + 16 * (size_t)j, al);
                for (; s < full; s += 2 * HB) {
#pragma unroll
                    for (int j = 0; j < HB; j++) b[j] = ld32le(q + 16 * (size_t)(s + HB + j), al);
#pragma unroll
                    for (int j = 0; j < HB; j++) v = rotl32(v + a[j] * P32_2, 13) * P32_1;
                    if (s + 2 * HB < full) {
#pragma unroll
                        for (int j = 0; j < HB; j++) a[j] = ld32le(q + 16 * (size_t)(s + 2 * HB + j), al);
                    }
#pragma unroll
                    for (int j = 0; j < HB; j++) v = rotl32(v + b[j] * P32_2, 13) * P32_1;
                }
            }
            for (; s < stripes; s++) v = rotl32(v + ld32le(q + 16 * (size_t)s, al) * P32_2, 13) * P32_1;
        }
        const uint32_t v1 = __shfl_sync(0xFFFFFFFFu, v, 0), v2 = __shfl_sync(0xFFFFFFFFu, v, 1), v3 = __shfl_sync(0xFFFFFFFFu, v, 2),
                       v4 = __shfl_sync(0xFFFFFFFFu, v, 3);
        h = rotl32(v1, 1) + rotl32(v2, 7) + rotl32(v3, 12) + rotl32(v4, 18);
        n = stripes << 4;
    } else {
        h = seed + P32_5;
    }
    h += len;
    for (; n + 4 <= len; n += 4) h = rotl32(h + ld32le(p + n, al) * P32_3, 17) * P32_4;
    for (; n < len; n++) h = rotl32(h + (uint32_t)p[n] * P32_5, 11) * P32_1;
    h ^= h >> 15;
    h *= P32_2;
    h ^= h >> 13;
    h *= P32_3;
    h ^= h >> 16;
    return h;
}

KZ_D uint64_t xxh64_block(const uint8_t* __restrict__ p, uint32_t len, uint64_t seed, int lane) {
    const bool al = (reinterpret_cast<uintptr_t>(p) & 7) == 0;
    uint32_t n = 0;
    uint64_t h;
    if (len >= 32) {
        const uint32_t stripes = len >> 5;
        uint64_t v = lane == 0 ? seed + P64_1 + P64_2 : (lane == 1 ? seed + P64_2 : (lane == 2 ? seed : seed - P64_1));
        if (lane < 4) {
            const uint8_t* q = p + 8 * lane;
            uint64_t a[HB], b[HB];
            uint32_t s = 0;
            const uint32_t full = stripes / (2 * HB) * (2 * HB);
            if (full) {
#pragma unroll
                for (int j = 0; j < HB; j++) a[j] = ld64le(q + 32 * (size_t)j, al);
                for (; s < full; s += 2 * HB) {
#pragma unroll
                    for (int j = 0; j < HB; j++) b[j] = ld64le(q + 32 * (size_t)(s + HB + j), al);
#pragma unroll
                    for (int j = 0; j < HB; j++) v = xxh64_round(v, a[j]);
                    if (s + 2 * HB < full) {
#pragma unroll
                        for (int j = 0; j < HB; j++) a[j] = ld64le(q + 32 * (size_t)(s + 2 * HB + j), al);
                    }
#pragma unroll
                    for (int j = 0; j < HB; j++) v = xxh64_round(v, b[j]);
                }
            }
            for (; s < stripes; s++) v = xxh64_round(v, ld64le(q + 32 * (size_t)s, al));
        }
        const uint64_t v1 = __shfl_sync(0xFFFFFFFFu, v, 0), v2 = __shfl_sync(0xFFFFFFFFu, v, 1), v3 = __shfl_sync(0xFFFFFFFFu, v, 2),
                       v4 = __shfl_sync(0xFFFFFFFFu, v, 3);
        h = xxh64_fold(v1, v2, v3, v4);
        n = stripes << 5;
    } else {
        h = seed + P64_5;
    }
    h += (uint64_t)len;
    for (; n + 8 <= len; n += 8) h = rotl64(h ^ xxh64_round(0, ld64le(p + n, al)), 27) * P64_1 + P64_4;
    for (; n + 4 <= len; n += 4) h = rotl64(h ^ ((uint64_t)ld32le(p + n, (reinterpret_cast<uintptr_t>(p + n) & 3) == 0) * P64_1), 23) * P64_2 + P64_3;
    for (; n < len; n++) h = rotl64(h ^ ((uint64_t)p[n] * P64_5), 11) * P64_1;
    return xxh64_avalanche(h);
}

// one warp per block; bits = 32 or 64; seed = 0x4B414E5A ("KANZ", io/CompressedStream.go:272-276)
__global__ void __launch_bounds__(32) xxhash_blocks_kernel(const uint8_t* __restrict__ data, const HashJob* __restrict__ jobs, int njobs, int bits,
                                                           uint64_t* __restrict__ out) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= njobs) return;
    const HashJob j = jobs[b];
    uint64_t h;
    if (bits == 32) h = xxh32_block(data + j.off, j.len, 0x4B414E5Au, lane);
    else h = xxh64_block(data + j.off, j.len, 0x4B414E5Aull, lane);
    if (lane == 0) out[b] = h;
}

}  // namespace kz
