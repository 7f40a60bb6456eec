// PACK / DNA transform (AliasCodec) on the GPU — declarations (kz_alias.cu).
// Reference: v2/transform/AliasCodec.go (Forward :74-273, Inverse :278-434, MaxEncodedLen :437-439).
#pragma once
#include "kz_common.cuh"

namespace kz {

static const uint32_t ALIAS_TILE = 4096;  // positions per tile of the digram parse / expansion scans

// bytes of device workspace for a batch (forward and inverse)
size_t alias_workspace(uint32_t nblocks, uint32_t max_len);

// All blocks of a batch; d_blocks / d_res are device arrays of nblocks entries. No host synchronisation inside.
cudaError_t alias_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint32_t max_len, uint8_t* ws, size_t ws_bytes,
                                StageResult* d_res, cudaStream_t stream, uint64_t* launches);
cudaError_t alias_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint32_t max_len, uint8_t* ws, size_t ws_bytes,
                                StageResult* d_res, cudaStream_t stream, uint64_t* launches);

// internal/Global.go:346-419 DetectSimpleType over a 256-bin histogram (device; header-only so that every kernel file can use it)
static __device__ __forceinline__ int detect_simple_type_dev(uint32_t count, const uint32_t* f) {
    if (count == 0) return 0;
    const char* DNA = "acgntuACGNTU";
    const char* NUM = "0123456789+-*/=,.:; ";
    const char* B64 = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    uint64_t sum = 0;
    for (int i = 0; i < 12; i++) sum += f[(uint8_t)DNA[i]];
    if (sum > (uint64_t)count - (uint64_t)count / 12) return 6;  // DT_DNA
    sum = 0;
    for (int i = 0; i < 20; i++) sum += f[(uint8_t)NUM[i]];
    if (sum == (uint64_t)count) return 4;  // DT_NUMERIC
    sum = 0;
    for (int i = 0; i < 64; i++) sum += f[(uint8_t)B64[i]];
    if (sum + f[0x3D] == (uint64_t)count) return 5;  // DT_BASE64
    sum = 0;
    for (int i = 0; i < 256; i++)
        if (f[i] > 0) sum++;
    if (sum == 256) return 7;  // DT_BIN
    if (sum <= 4) return 9;    // DT_SMALL_ALPHABET
    return 0;
}

}  // namespace kz
