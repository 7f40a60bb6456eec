// The record hash of kz_xxh64_core.cuh on the device, for the keys of a cached range read: every touched record of a call in one launch,
// one warp per 4 KiB tile, then one thread per record for the root.
//
// A record starts at any bit of the stream, so a warp first realigns its tile into shared memory: each lane takes 32-bit words at
// bit-granular positions (bits_at reads two stream words and shifts) and zeroes what lies behind the record's last bit. Lanes 0..3 then
// walk the four XXH64 accumulator chains of the tile's 32-byte stripes (128 dependent rounds for a full tile) and lane 0 the tail.
#include "kz_record_hash.cuh"
#include "kz_xxh64_core.cuh"

namespace kz {

__global__ void __launch_bounds__(32 * RECORD_HASH_WARPS)
    record_hash_tiles_kernel(const uint32_t* __restrict__ words, const RecordHashJob* __restrict__ jobs, int njobs, uint64_t ntiles,
                             uint64_t* __restrict__ digest) {
    __shared__ __align__(16) uint32_t tile_s[RECORD_HASH_WARPS][RECORD_TILE / 4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t w = (uint64_t)blockIdx.x * RECORD_HASH_WARPS + warp;
    if (w >= ntiles) return;
    int lo = 0, hi = njobs - 1;  // the last job whose first tile is <= w
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (jobs[mid].tile0 <= w) lo = mid;
        else hi = mid - 1;
    }
    const RecordHashJob j = jobs[lo];
    const uint64_t t = w - j.tile0;
    const uint32_t n = record_tile_len(j.bits, t);
    const uint64_t end = j.start + j.bits;
    uint32_t* s = tile_s[warp];
    for (uint32_t i = lane; i < (n + 3) / 4; i += 32) {
        const uint64_t pos = j.start + 8 * (t * RECORD_TILE + 4 * (uint64_t)i);
        uint32_t v = bits_at(words, pos, 32);
        if (pos + 32 > end) v &= ~(0xFFFFFFFFu >> (uint32_t)(end - pos));  // keep the end - pos (< 32) leading bits
        s[i] = __byte_perm(v, 0, 0x0123);                                   // bytes in stream order, as a little-endian word
    }
    __syncwarp();
    const uint8_t* b = reinterpret_cast<const uint8_t*>(s);
    const uint64_t* q = reinterpret_cast<const uint64_t*>(s);
    uint64_t h = 0, p = 0;
    if (n >= 32) {
        const uint32_t stripes = n >> 5;
        uint64_t v = lane == 0 ? P64_1 + P64_2 : (lane == 1 ? P64_2 : (lane == 2 ? 0 : 0 - P64_1));
        if (lane < 4)
            for (uint32_t k = 0; k < stripes; k++) v = xxh64_round(v, q[4 * k + lane]);
        const uint64_t v1 = __shfl_sync(0xFFFFFFFFu, v, 0), v2 = __shfl_sync(0xFFFFFFFFu, v, 1), v3 = __shfl_sync(0xFFFFFFFFu, v, 2),
                       v4 = __shfl_sync(0xFFFFFFFFu, v, 3);
        h = xxh64_fold(v1, v2, v3, v4);
        p = (uint64_t)stripes << 5;
    } else {
        h = P64_5;
    }
    if (lane == 0) {
        auto rd = [&](uint64_t at, int k) {
            uint64_t x = 0;
            for (int i = k - 1; i >= 0; i--) x = (x << 8) | b[at + i];
            return x;
        };
        digest[w] = xxh64_tail(h + n, rd, p, n);
    }
}

__global__ void __launch_bounds__(128)
    record_hash_root_kernel(const RecordHashJob* __restrict__ jobs, int njobs, const uint64_t* __restrict__ digest, uint64_t* __restrict__ key) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= njobs) return;
    const RecordHashJob j = jobs[r];
    key[r] = record_root(digest + j.tile0, record_tiles(j.bits), j.bits);
}

}  // namespace kz
