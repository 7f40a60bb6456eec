// Declarations of the record hash kernels (kz_record_hash.cu): the keys of a cached range read (kz_read_ranges_cached_device).
#pragma once
#include "kz_common.cuh"

namespace kz {

struct RecordHashJob {
    uint64_t start, bits;  // the record's payload: bits [start, start + bits) of the stream
    uint64_t tile0;        // index of its first tile digest; the jobs' tiles are numbered back to back
};

// one warp per tile: digest[tile] = XXH64 of the tile (kz_xxh64_core.cuh); blocks of RECORD_HASH_WARPS warps
constexpr int RECORD_HASH_WARPS = 4;
__global__ void record_hash_tiles_kernel(const uint32_t* words, const RecordHashJob* jobs, int njobs, uint64_t ntiles, uint64_t* digest);
// one thread per record: key[j] = the root of record j's tree over its tile digests
__global__ void record_hash_root_kernel(const RecordHashJob* jobs, int njobs, const uint64_t* digest, uint64_t* key);

}  // namespace kz
