// BWT entry points (kz_bwt.cu). All pointers are device pointers unless noted.
#pragma once
#include "kz_common.cuh"

namespace kz {
size_t bwt_forward_workspace(uint32_t n);
// BWTBlockCodec.Forward of one block: d_dst receives header + BWT bytes (n + 1 + chunks * index size), *d_out_len its length
cudaError_t bwt_forward_device(const uint8_t* d_src, uint32_t n, uint8_t* d_dst, uint32_t* d_out_len, uint8_t* ws, size_t ws_bytes, cudaStream_t stream,
                               uint64_t* launches);
// BWTBlockCodec.Forward of a batch of blocks sorted together (block k: n_of[k] >= 2 bytes at d_in + src_off[k] -> d_out + dst_off[k]; d_out_len[number[k]] = length)
// hook (optional): every part of every doubling round timed under "bwt_round:<r>:<part>"; wide_rounds: the 56-bit global sort in every round
// (the rounds the batches with a block above 4 MiB take), same output
size_t bwt_forward_batch_workspace(uint64_t total, uint32_t nblocks);
uint64_t bwt_forward_batch_max_total();
uint32_t bwt_forward_batch_max_blocks();
struct LzHook;
cudaError_t bwt_forward_batch(const uint8_t* d_in, uint8_t* d_out, const uint64_t* src_off, const uint64_t* dst_off, const uint32_t* n_of, const uint32_t* number,
                              uint32_t nb, uint32_t* d_out_len, uint8_t* ws, size_t ws_bytes, cudaStream_t stream, uint64_t* launches, LzHook* hook = nullptr,
                              bool wide_rounds = false);
// BWTBlockCodec.Inverse of a batch (one sort, one head list, one set of launches for all blocks); h_headers + 64 k = first 33 bytes of block k's stream.
// The shape of the walk (the output bytes never depend on it): sub-lists cut every `stride` ranks (a power of two), `stage` bytes of staging per
// sub-list (a multiple of 4).
struct IbwtShape {
    uint32_t stride = 32, stage = 128;
};
// max_len: the longest stream of the batch (it decides between 32-bit and 64-bit LF words)
size_t bwt_inverse_batch_workspace(uint64_t total, uint32_t nblocks, uint32_t max_len, const IbwtShape& shape = IbwtShape());
uint64_t bwt_inverse_batch_max_total();
uint32_t bwt_inverse_batch_max_blocks();
// hook (optional): the parts timed under "bwt_inverse:<part>" (sort, walk, doubling, copy, sync)
cudaError_t bwt_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const uint64_t* src_off, const uint64_t* dst_off, const uint32_t* len_of, const uint8_t* h_headers,
                              uint32_t nb, uint32_t cap, uint32_t* out_len, uint8_t* ws, size_t ws_bytes, cudaStream_t stream, uint64_t* launches,
                              const IbwtShape& shape = IbwtShape(), LzHook* hook = nullptr);
// BWTS.Forward / BWTS.Inverse of one block (n bytes in, n bytes out)
size_t bwts_forward_workspace(uint32_t n);
size_t bwts_inverse_workspace(uint32_t n);
cudaError_t bwts_forward_device(const uint8_t* d_src, uint32_t n, uint8_t* d_dst, uint8_t* ws, size_t ws_bytes, cudaStream_t stream, uint64_t* launches);
cudaError_t bwts_inverse_device(const uint8_t* d_src, uint32_t n, uint8_t* d_dst, uint8_t* ws, size_t ws_bytes, cudaStream_t stream, uint64_t* launches);
}  // namespace kz
