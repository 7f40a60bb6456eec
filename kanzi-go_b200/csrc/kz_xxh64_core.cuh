// XXH64 (Yann Collet's public algorithm) and the record hash of the block cache, host/device shared: the block checksums (kz_hash.cu) take
// the round functions from here, the index blob hash (kz_read_plan.h) and the host variant of the record hash run it on the CPU, the
// record_hash kernels (kz_record_hash.cu) on the device, tests/host/block_cache_host.cpp under g++.
//
// Record hash: the key of a decoded block in the block cache (kz_block_cache.h) is the content of its record, not its place in a stream.
// A record is a bit string of `bits` bits that may start at any bit. It is realigned to bit 0 (byte j holds bits [8j, 8j + 8), MSB first,
// as the stream stores them) and zero padded to a whole byte, cut into tiles of RECORD_TILE bytes, and hashed as a tree: the XXH64 (seed 0)
// of every tile, then the XXH64 (seed 0) of the tile digests and the bit length, each a little-endian u64. The tiles are independent, so
// the device hashes them one warp each.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#if defined(__CUDACC__)
#define KZX_HD __host__ __device__ __forceinline__
#else
#define KZX_HD inline
#endif

namespace kz {

constexpr uint64_t P64_1 = 11400714785074694791ull, P64_2 = 14029467366897019727ull, P64_3 = 1609587929392839161ull, P64_4 = 9650029242287828579ull,
                   P64_5 = 2870177450012600261ull;

KZX_HD uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
KZX_HD uint64_t xxh64_round(uint64_t acc, uint64_t v) { return rotl64(acc + v * P64_2, 31) * P64_1; }
KZX_HD uint64_t xxh64_merge(uint64_t h, uint64_t v) { return (h ^ xxh64_round(0, v)) * P64_1 + P64_4; }
KZX_HD uint64_t xxh64_avalanche(uint64_t h) {
    h ^= h >> 33;
    h *= P64_2;
    h ^= h >> 29;
    h *= P64_3;
    h ^= h >> 32;
    return h;
}
// the four accumulator lanes after the stripes, folded into one value
KZX_HD uint64_t xxh64_fold(uint64_t v1, uint64_t v2, uint64_t v3, uint64_t v4) {
    uint64_t h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    return xxh64_merge(xxh64_merge(xxh64_merge(xxh64_merge(h, v1), v2), v3), v4);
}

// The part of XXH64 behind the stripes: h already holds the length, bytes [p, n) remain (fewer than 32).
template <class Rd>
KZX_HD uint64_t xxh64_tail(uint64_t h, Rd&& rd, uint64_t p, uint64_t n) {
    for (; n - p >= 8; p += 8) h = rotl64(h ^ xxh64_round(0, rd(p, 8)), 27) * P64_1 + P64_4;
    if (n - p >= 4) {
        h = rotl64(h ^ (rd(p, 4) * P64_1), 23) * P64_2 + P64_3;
        p += 4;
    }
    for (; p < n; p++) h = rotl64(h ^ (rd(p, 1) * P64_5), 11) * P64_1;
    return xxh64_avalanche(h);
}

// XXH64 of n bytes: rd(at, k) gives bytes [at, at + k) (k = 1, 4 or 8) as a little-endian value. Serial; the device hashes a tile with
// four lanes instead (kz_record_hash.cu).
template <class Rd>
KZX_HD uint64_t xxh64_with(Rd&& rd, uint64_t n, uint64_t seed) {
    uint64_t p = 0, h;
    if (n >= 32) {
        uint64_t v1 = seed + P64_1 + P64_2, v2 = seed + P64_2, v3 = seed, v4 = seed - P64_1;
        for (; n - p >= 32; p += 32) {
            v1 = xxh64_round(v1, rd(p, 8));
            v2 = xxh64_round(v2, rd(p + 8, 8));
            v3 = xxh64_round(v3, rd(p + 16, 8));
            v4 = xxh64_round(v4, rd(p + 24, 8));
        }
        h = xxh64_fold(v1, v2, v3, v4);
    } else {
        h = seed + P64_5;
    }
    return xxh64_tail(h + n, rd, p, n);
}

KZX_HD uint64_t xxh64_bytes(const uint8_t* p, uint64_t n, uint64_t seed) {
    return xxh64_with(
        [p](uint64_t at, int k) {
            uint64_t v = 0;
#if defined(__CUDA_ARCH__)
            for (int i = k - 1; i >= 0; i--) v = (v << 8) | p[at + i];
#else
            memcpy(&v, p + at, (size_t)k);  // the hosts are little endian
#endif
            return v;
        },
        n, seed);
}

// ---- the record hash ---------------------------------------------------------------------------------------------------------------
constexpr uint32_t RECORD_TILE = 4096;

KZX_HD uint64_t record_bytes(uint64_t bits) { return (bits + 7) / 8; }
KZX_HD uint64_t record_tiles(uint64_t bits) { return (record_bytes(bits) + RECORD_TILE - 1) / RECORD_TILE; }
// bytes of tile t of a record
KZX_HD uint32_t record_tile_len(uint64_t bits, uint64_t t) {
    const uint64_t left = record_bytes(bits) - t * RECORD_TILE;
    return (uint32_t)(left < RECORD_TILE ? left : RECORD_TILE);
}

// Byte j of the realigned record that starts at bit `start` of the byte string s: zero behind the record's last bit. s must be readable
// up to byte (start + bits - 1) / 8.
KZX_HD uint8_t record_byte(const uint8_t* s, uint64_t start, uint64_t bits, uint64_t j) {
    const uint64_t pos = start + 8 * j, end = start + bits;
    const uint32_t r = (uint32_t)(pos & 7);
    uint32_t v = (uint32_t)s[pos >> 3] << 8;
    if (r && ((pos >> 3) + 1) * 8 < end) v |= s[(pos >> 3) + 1];
    uint8_t b = (uint8_t)(v >> (8 - r));
    if (pos + 8 > end) b &= (uint8_t)(0xFF00u >> (end - pos));  // the last byte keeps its end - pos leading bits
    return b;
}

// The root of the tree: XXH64 of the tile digests dig[0 .. ntiles) and the bit length, as little-endian u64.
KZX_HD uint64_t record_root(const uint64_t* dig, uint64_t ntiles, uint64_t bits) {
    // every read is a whole word: the stripes and the tail of a length that is a multiple of 8
    return xxh64_with([&](uint64_t at, int) { return at / 8 < ntiles ? dig[at / 8] : bits; }, 8 * (ntiles + 1), 0);
}

// The record hash of the record at bits [start, start + bits) of the byte string s, serially (the host variant of a cached read).
inline uint64_t record_hash_host(const uint8_t* s, uint64_t start, uint64_t bits) {
    std::vector<uint64_t> dig(record_tiles(bits));
    uint8_t tile[RECORD_TILE];
    for (uint64_t t = 0; t < dig.size(); t++) {
        const uint32_t n = record_tile_len(bits, t);
        const uint8_t* q = s + start / 8 + t * RECORD_TILE;
        const uint32_t r = (uint32_t)(start & 7), fast = t + 1 < dig.size() ? n : n - 1;  // bytes whose two source bytes lie in the record
        if (r == 0) memcpy(tile, q, fast);
        else
            for (uint32_t j = 0; j < fast; j++) tile[j] = (uint8_t)((q[j] << r) | (q[j + 1] >> (8 - r)));
        if (fast < n) tile[n - 1] = record_byte(s, start, bits, t * RECORD_TILE + n - 1);
        dig[t] = xxh64_bytes(tile, n, 0);
    }
    return record_root(dig.data(), dig.size(), bits);
}

}  // namespace kz
