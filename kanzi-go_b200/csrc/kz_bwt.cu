// Burrows-Wheeler transform of a whole block on one GPU: suffix array by prefix doubling (forward) and sampled list
// ranking (inverse).
//
// Reference semantics reproduced bit-exactly (paths relative to the reference's v2/ directory):
//   transform/BWT.go:132-173 Forward + transform/DivSufSort.go:179-311 ComputeBWT: suffix order without sentinel (a suffix
//     that is a proper prefix of another sorts first), output dst[0] = src[n-1] followed by src[SA[r]-1] for every rank
//     r in order except the rank of suffix 0; primary index k = rank(k * ceil(n/8)) + 1 (1 index when n < 256).
//     The BWT is canonical, so the suffix array is built with a GPU algorithm instead of DivSufSort's induced sorting:
//     rank arrays are doubled (h = 7, 14, 28, ...) with one 64-bit radix sort of (rank[i], rank[i+h]) per round
//     (cub::DeviceRadixSort for the sort itself; everything else is hand written).
//   transform/BWT.go:178-358 Inverse (inverseMergeTPSI) / :361-628 (biPSIv2): both walk the permutation
//     "rank of suffix i -> rank of suffix i+1" from primaryIndex(0)-1. The format only offers 8 independent walks,
//     far too few for a GPU, so the permutation list is cut at every rank that is a multiple of 32 (plus the 8 primary
//     ranks): all sub-lists are walked in parallel once, their bytes staged per sub-list, the sub-list heads are ranked
//     with pointer doubling, and the staged bytes are copied to their final offsets.
//   transform/BWTBlockCodec.go:78-136, :141-225: block header (mode byte + big-endian primaryIndex-1 per chunk).
#include <cub/device/device_radix_sort.cuh>
#include <thrust/iterator/reverse_iterator.h>
#include <cub/device/dispatch/dispatch_three_way_partition.cuh>
#include <cub/device/dispatch/dispatch_segmented_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <cub/device/device_select.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include <algorithm>
#include <string>
#include <vector>

#include "kz_bwt.cuh"
#include "kz_bwt_core.cuh"
#include "kz_lz.cuh"

namespace kz {

namespace {

KZ_HD uint32_t bwt_chunks(uint32_t n) { return n < 256 ? 1u : 8u; }

// key of suffix i from its first 7 bytes, 9 bits per symbol (byte + 1, 0 past the end): shorter suffix sorts first
__global__ void bwt_init_keys_kernel(const uint8_t* __restrict__ src, uint32_t n, uint64_t* __restrict__ keys, uint32_t* __restrict__ idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t k = 0;
#pragma unroll
    for (int j = 0; j < 7; j++) {
        const uint32_t p = i + j;
        const uint64_t s = p < n ? (uint64_t)src[p] + 1 : 0;
        k = (k << 9) | s;
    }
    keys[i] = k;
    idx[i] = i;
}

// flags[j] = 1 when sorted position j starts a new group of equal keys
__global__ void bwt_flag_kernel(const uint64_t* __restrict__ keys, uint32_t n, uint32_t* __restrict__ head) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    head[j] = (j == 0 || keys[j] != keys[j - 1]) ? j : 0u;
}

// inclusive max-scan over `head` in place (group start index for every sorted position), three-phase block scan
__global__ void scan_max_local_kernel(uint32_t* __restrict__ v, uint32_t n, uint32_t* __restrict__ block_max) {
    __shared__ uint32_t s_warp[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t base = blockIdx.x * (blockDim.x * 8);
    uint32_t x[8];
    uint32_t run = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const uint32_t j = base + tid * 8 + q;
        x[q] = j < n ? v[j] : 0u;
        run = max(run, x[q]);
        x[q] = run;
    }
    uint32_t incl = run;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= d) incl = max(incl, t);
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < (blockDim.x >> 5) ? s_warp[lane] : 0u;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, w, d);
            if (lane >= d) w = max(w, t);
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    uint32_t prev = __shfl_up_sync(0xFFFFFFFFu, incl, 1);
    if (lane == 0) prev = 0;
    if (warp > 0) prev = max(prev, s_warp[warp - 1]);
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const uint32_t j = base + tid * 8 + q;
        if (j < n) v[j] = max(x[q], prev);
    }
    if (tid == blockDim.x - 1) block_max[blockIdx.x] = max(incl, prev);
}
__global__ void scan_max_blocks_kernel(uint32_t* __restrict__ block_max, uint32_t nblocks) {  // one CTA, serial over tiles of 1024
    __shared__ uint32_t s_carry;
    __shared__ uint32_t s_warp[32];
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t start = 0; start < nblocks; start += 1024) {
        const uint32_t i = start + threadIdx.x;
        uint32_t x = i < nblocks ? block_max[i] : 0u;
        uint32_t incl = x;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= d) incl = max(incl, t);
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = s_warp[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, w, d);
                if (lane >= d) w = max(w, t);
            }
            s_warp[lane] = w;
        }
        __syncthreads();
        uint32_t r = max(incl, s_carry);
        if (warp > 0) r = max(r, s_warp[warp - 1]);
        if (i < nblocks) block_max[i] = r;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = r;
        __syncthreads();
    }
}
// v[j] = max(v[j], prefix of previous blocks); rank[sa[j]] = v[j]; counts positions whose group has more than one member
__global__ void bwt_apply_rank_kernel(uint32_t* __restrict__ head, const uint32_t* __restrict__ block_max, const uint32_t* __restrict__ sa, uint32_t n,
                                      uint32_t* __restrict__ rank, uint32_t* __restrict__ unsorted_flag) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t blk = j / (256 * 8);
    uint32_t g = head[j];
    if (blk > 0) g = max(g, block_max[blk - 1]);
    head[j] = g;
    rank[sa[j]] = g;
    if (g != j) *unsorted_flag = 1;  // position j is not the head of its group -> some group has >= 2 members
}

__global__ void bwt_double_keys_kernel(const uint32_t* __restrict__ rank, uint32_t n, uint32_t h, uint32_t log_n, uint64_t* __restrict__ keys,
                                       uint32_t* __restrict__ idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t hi = rank[i];
    const uint64_t lo = (uint64_t)i + h < n ? (uint64_t)rank[i + h] + 1 : 0;  // <= n < 2^log_n
    keys[i] = (hi << log_n) | lo;
    idx[i] = i;
}

// BWT bytes + primary indexes from the final suffix array (ComputeBWT layout)
__global__ void bwt_emit_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ sa, const uint32_t* __restrict__ rank, uint32_t n,
                                uint8_t* __restrict__ dst /*n bytes*/, uint32_t* __restrict__ primary /*8*/) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) dst[0] = src[n - 1];
    if (r < 8) {
        const uint32_t chunks = bwt_chunks(n);
        uint32_t step = n / chunks;
        if (step * chunks != n) step++;
        primary[r] = (r < chunks && (uint64_t)r * step < n) ? rank[r * step] + 1 : 0;
    }
    if (r >= n) return;
    const uint32_t s = sa[r];
    if (s == 0) return;
    const uint32_t rank0 = rank[0];
    dst[r < rank0 ? r + 1 : r] = src[s - 1];
}

// BWTBlockCodec.Forward header (:113-133). One thread.
__global__ void bwt_header_kernel(const uint32_t* __restrict__ primary, uint32_t n, uint8_t* __restrict__ dst, uint32_t* __restrict__ out_len) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t log_bs = log2_floor(n);
    if (n & (n - 1)) log_bs++;
    const int pidx = (int)(log_bs + 7) >> 3;
    const uint32_t chunks = bwt_chunks(n);
    dst[0] = (uint8_t)((log2_floor(chunks) << 2) | (uint32_t)(pidx - 1));
    uint32_t idx = 1;
    for (uint32_t i = 0; i < chunks; i++) {
        const uint32_t p = primary[i] - 1;
        for (int shift = (pidx - 1) << 3; shift >= 0; shift -= 8) dst[idx++] = (uint8_t)(p >> shift);
    }
    *out_len = n + chunks * pidx + 1;
}

// ---------------- inverse ----------------
// Wyllie pointer doubling over the heads: after the rounds dist[j] = number of bytes from head j to the end of the list
__global__ void ibwt_jump_kernel(const uint32_t* __restrict__ succ_in, const uint64_t* __restrict__ dist_in, uint32_t nheads, uint32_t* __restrict__ succ_out,
                                 uint64_t* __restrict__ dist_out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nheads) return;
    const uint32_t s = succ_in[j];
    uint64_t d = dist_in[j];
    uint32_t s2 = s;
    if (s < nheads) {
        d += dist_in[s];
        s2 = succ_in[s];
    }
    succ_out[j] = s2;
    dist_out[j] = d;
}

}  // namespace

size_t bwt_forward_workspace(uint32_t n) {
    size_t temp = 0;
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, (int)n, 0, 64);
    // keys x2, idx x2, rank, head, block_max, flags, cub temp
    return (size_t)n * (8 * 2 + 4 * 2 + 4 + 4) + 4 * ((size_t)n / 2048 + 16) + 256 + temp + 4096;
}

// d_src: n bytes; d_dst: n + 33 bytes (header + BWT); ws: workspace of bwt_forward_workspace(n) bytes (256-byte aligned)
cudaError_t bwt_forward_device(const uint8_t* d_src, uint32_t n, uint8_t* d_dst, uint32_t* d_out_len, uint8_t* ws, size_t ws_bytes, cudaStream_t stream,
                               uint64_t* launches) {
    if (n < 2) return cudaErrorInvalidValue;
    auto align = [](size_t x) { return (x + 255) & ~size_t(255); };
    size_t off = 0;
    uint64_t* keys_a = (uint64_t*)(ws + off); off = align(off + (size_t)n * 8);
    uint64_t* keys_b = (uint64_t*)(ws + off); off = align(off + (size_t)n * 8);
    uint32_t* idx_a = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* idx_b = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* rank = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* head = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    const uint32_t nscan = (n + 2047) / 2048;
    uint32_t* block_max = (uint32_t*)(ws + off); off = align(off + (size_t)nscan * 4);
    uint32_t* flags = (uint32_t*)(ws + off); off = align(off + 64);
    uint32_t* primary = flags + 4;
    void* temp = ws + off;
    size_t temp_bytes = ws_bytes > off ? ws_bytes - off : 0;
    const uint32_t T = 256, G = (n + T - 1) / T;
    uint32_t log_n = 1;
    while ((1ull << log_n) <= n) log_n++;
    uint32_t header;
    {
        uint32_t log_bs = log2_floor(n);
        if (n & (n - 1)) log_bs++;
        const uint32_t pidx = (log_bs + 7) >> 3;
        if (pidx == 0 || pidx >= 5) return cudaErrorInvalidValue;
        header = (n < 256 ? 1u : 8u) * pidx + 1;
    }
    bwt_init_keys_kernel<<<G, T, 0, stream>>>(d_src, n, keys_a, idx_a);
    (*launches)++;
    uint32_t h = 7;
    int end_bit = 63;
    for (int round = 0; round < 40; round++) {
        cub::DoubleBuffer<uint64_t> k(keys_a, keys_b);
        cub::DoubleBuffer<uint32_t> v(idx_a, idx_b);
        size_t tb = temp_bytes;
        cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, tb, k, v, (int)n, 0, end_bit, stream);
        if (e != cudaSuccess) return e;
        (*launches) += 8;
        const uint64_t* sk = k.Current();
        const uint32_t* sa = v.Current();
        cudaMemsetAsync(flags, 0, 4, stream);
        bwt_flag_kernel<<<G, T, 0, stream>>>(sk, n, head);
        scan_max_local_kernel<<<nscan, 256, 0, stream>>>(head, n, block_max);
        scan_max_blocks_kernel<<<1, 1024, 0, stream>>>(block_max, nscan);
        bwt_apply_rank_kernel<<<G, T, 0, stream>>>(head, block_max, sa, n, rank, flags);
        (*launches) += 4;
        uint32_t unsorted = 0;
        e = cudaMemcpyAsync(&unsorted, flags, 4, cudaMemcpyDeviceToHost, stream);
        if (e != cudaSuccess) return e;
        e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) return e;
        if (!unsorted || h >= n) {
            bwt_emit_kernel<<<G, T, 0, stream>>>(d_src, sa, rank, n, d_dst + header, primary);
            bwt_header_kernel<<<1, 32, 0, stream>>>(primary, n, d_dst, d_out_len);
            (*launches) += 2;
            return cudaGetLastError();
        }
        // the sorted buffers become scratch; build the doubled keys into the "a" buffers
        bwt_double_keys_kernel<<<G, T, 0, stream>>>(rank, n, h, log_n, keys_a, idx_a);
        (*launches)++;
        h *= 2;
        end_bit = 2 * (int)log_n;
    }
    return cudaErrorUnknown;
}

// ---- forward, all blocks of a batch in one position space ------------------------------------------------------------------------------------
// A 4 MiB sort cannot fill an H100 and 48 of them one after another pay 48 x (rounds x (sort + 6 small kernels + a host sync)). Here the blocks
// are laid end to end (block b = positions [base[b], base[b] + n[b])) and sorted together: the block index is the top of the first key
// (block | 6 symbols x 9 bits), so ranks taken as global group heads fall into [base[b], base[b] + n[b]) and the doubled keys
// (rank[i] << lg | rank[i + h] + 1, 0 past the END OF THE BLOCK) never mix blocks. One sort, one flag / scan / apply pass and one host
// sync per round for the whole batch; the number of rounds is the maximum over the blocks.
namespace {
struct BwtBatchBlock {
    uint64_t src_off, dst_off;
    uint32_t base, n;
    uint32_t header, pad;
};
const int BWT_BATCH_MAX = 1024;  // 10 bits of block index above 54 bits of symbols
__device__ __forceinline__ uint32_t bwtb_find(const uint32_t* __restrict__ s_base, uint32_t nb, uint32_t i) {  // last block with base <= i
    uint32_t lo = 0, hi = nb;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s_base[mid] <= i) lo = mid;
        else hi = mid;
    }
    return lo;
}
__global__ void __launch_bounds__(256) bwtb_init_keys_kernel(const uint8_t* __restrict__ in, const BwtBatchBlock* __restrict__ blocks, uint32_t nb, uint32_t total,
                                                              uint64_t* __restrict__ keys, uint32_t* __restrict__ idx) {
    __shared__ uint32_t s_base[BWT_BATCH_MAX];
    for (uint32_t k = threadIdx.x; k < nb; k += 256) s_base[k] = blocks[k].base;
    __syncthreads();
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const uint32_t b = bwtb_find(s_base, nb, i);
    const BwtBatchBlock B = blocks[b];
    const uint8_t* src = in + B.src_off;
    const uint32_t l = i - B.base;
    uint64_t k = b;
#pragma unroll
    for (int j = 0; j < 6; j++) {
        const uint32_t p = l + j;
        const uint64_t sym = p < B.n ? (uint64_t)src[p] + 1 : 0;
        k = (k << 9) | sym;
    }
    keys[i] = k;
    idx[i] = i;
}
__global__ void __launch_bounds__(256) bwtb_double_keys_kernel(const uint32_t* __restrict__ rank, const BwtBatchBlock* __restrict__ blocks, uint32_t nb, uint32_t total,
                                                                uint32_t h, uint32_t lg, uint64_t* __restrict__ keys, uint32_t* __restrict__ idx) {
    __shared__ uint32_t s_base[BWT_BATCH_MAX];
    __shared__ uint32_t s_n[BWT_BATCH_MAX];
    for (uint32_t k = threadIdx.x; k < nb; k += 256) s_base[k] = blocks[k].base, s_n[k] = blocks[k].n;
    __syncthreads();
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const uint32_t b = bwtb_find(s_base, nb, i);
    const uint64_t end = (uint64_t)s_base[b] + s_n[b];
    const uint64_t hi = rank[i];
    const uint64_t lo = (uint64_t)i + h < end ? (uint64_t)rank[i + h] + 1 : 0;  // <= total < 2^lg
    keys[i] = (hi << lg) | lo;
    idx[i] = i;
}
__global__ void __launch_bounds__(256) bwtb_emit_kernel(const uint8_t* __restrict__ in, const BwtBatchBlock* __restrict__ blocks, uint32_t nb, uint32_t total,
                                                         const uint32_t* __restrict__ sa, const uint32_t* __restrict__ rank, uint8_t* __restrict__ out) {
    __shared__ uint32_t s_base[BWT_BATCH_MAX];
    for (uint32_t k = threadIdx.x; k < nb; k += 256) s_base[k] = blocks[k].base;
    __syncthreads();
    const uint32_t r = blockIdx.x * 256 + threadIdx.x;
    if (r >= total) return;
    const uint32_t b = bwtb_find(s_base, nb, r);  // ranks of block b are [base, base + n) as well
    const BwtBatchBlock B = blocks[b];
    const uint8_t* src = in + B.src_off;
    uint8_t* dst = out + B.dst_off + B.header;
    const uint32_t rl = r - B.base;
    if (rl == 0) dst[0] = src[B.n - 1];
    const uint32_t s = sa[r] - B.base;
    if (s == 0) return;
    const uint32_t rank0 = rank[B.base] - B.base;
    dst[rl < rank0 ? rl + 1 : rl] = src[s - 1];
}
// primary indexes + BWTBlockCodec header of every block (BWTBlockCodec.go:113-133); one thread per block
__global__ void bwtb_header_kernel(const BwtBatchBlock* __restrict__ blocks, uint32_t nb, const uint32_t* __restrict__ rank, uint8_t* __restrict__ out,
                                   uint32_t* __restrict__ out_len /* indexed by pad = caller's block number */) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const BwtBatchBlock B = blocks[b];
    const uint32_t n = B.n;
    uint8_t* dst = out + B.dst_off;
    uint32_t log_bs = log2_floor(n);
    if (n & (n - 1)) log_bs++;
    const int pidx = (int)(log_bs + 7) >> 3;
    const uint32_t chunks = bwt_chunks(n);
    uint32_t step = n / chunks;
    if (step * chunks != n) step++;
    dst[0] = (uint8_t)((log2_floor(chunks) << 2) | (uint32_t)(pidx - 1));
    uint32_t idx = 1;
    for (uint32_t i = 0; i < chunks; i++) {
        const uint32_t prim = ((uint64_t)i * step < n) ? rank[B.base + i * step] - B.base + 1 : 0;
        const uint32_t p = prim - 1;
        for (int shift = (pidx - 1) << 3; shift >= 0; shift -= 8) dst[idx++] = (uint8_t)(p >> shift);
    }
    out_len[B.pad] = n + chunks * pidx + 1;
}
// ---- rounds over the unresolved part only -----------------------------------------------------------------------------------------------------
// After a round every group of equal h-prefixes is a contiguous range of sorted positions and only groups with more than one member can
// change. The members of those groups are compacted (sorted position, suffix), sorted by (group head, rank of the suffix h further), and
// written back into the same positions: the work of a round is proportional to what is still unresolved, not to the batch.
__global__ void __launch_bounds__(256) bwtu_flags_full_kernel(const uint32_t* __restrict__ head, uint32_t total, uint8_t* __restrict__ flags) {
    const uint32_t j = blockIdx.x * 256 + threadIdx.x;
    if (j >= total) return;
    const uint32_t hj = head[j];
    flags[j] = (hj != j || (j + 1 < total && head[j + 1] == hj)) ? 1 : 0;
}
__global__ void __launch_bounds__(256) bwtu_flags_kernel(const uint32_t* __restrict__ nhead, const uint32_t* __restrict__ cpos, uint32_t m, uint8_t* __restrict__ flags) {
    const uint32_t u = blockIdx.x * 256 + threadIdx.x;
    if (u >= m) return;
    const uint32_t hu = nhead[u];
    flags[u] = (hu != cpos[u] || (u + 1 < m && nhead[u + 1] == hu)) ? 1 : 0;
}
__global__ void __launch_bounds__(256) bwtu_keys_kernel(const uint32_t* __restrict__ rank, const uint32_t* __restrict__ cval, uint32_t m,
                                                         const BwtBatchBlock* __restrict__ blocks, uint32_t nb, uint32_t h, uint32_t lg, uint64_t* __restrict__ keys) {
    __shared__ uint32_t s_base[BWT_BATCH_MAX];
    __shared__ uint32_t s_n[BWT_BATCH_MAX];
    for (uint32_t k = threadIdx.x; k < nb; k += 256) s_base[k] = blocks[k].base, s_n[k] = blocks[k].n;
    __syncthreads();
    const uint32_t u = blockIdx.x * 256 + threadIdx.x;
    if (u >= m) return;
    const uint32_t i = cval[u];
    const uint32_t b = bwtb_find(s_base, nb, i);
    const uint64_t end = (uint64_t)s_base[b] + s_n[b];
    const uint64_t hi = rank[i];
    const uint64_t lo = (uint64_t)i + h < end ? (uint64_t)rank[i + h] + 1 : 0;
    keys[u] = (hi << lg) | lo;
}
// candidate heads of the new groups: the sorted position of the first member (0 elsewhere; a max-scan spreads them)
__global__ void __launch_bounds__(256) bwtu_heads_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ cpos, uint32_t m, uint32_t* __restrict__ f) {
    const uint32_t u = blockIdx.x * 256 + threadIdx.x;
    if (u >= m) return;
    f[u] = (u == 0 || keys[u] != keys[u - 1]) ? cpos[u] : 0u;
}
__global__ void __launch_bounds__(256) bwtu_apply_kernel(uint32_t* __restrict__ f, const uint32_t* __restrict__ block_max, const uint32_t* __restrict__ cpos,
                                                          const uint32_t* __restrict__ cval, uint32_t m, uint32_t* __restrict__ sa, uint32_t* __restrict__ rank) {
    const uint32_t u = blockIdx.x * 256 + threadIdx.x;
    if (u >= m) return;
    const uint32_t blk = u / (256 * 8);
    uint32_t g = f[u];
    if (blk > 0) g = max(g, block_max[blk - 1]);
    f[u] = g;
    const uint32_t v = cval[u];
    sa[cpos[u]] = v;
    rank[v] = g;
}

// ---- narrow rounds (every block of the batch at most BWT_NARROW_MAX_N bytes) --------------------------------------------------------------
// The same rounds without a 56-bit global sort. Members u < m (cpos[u]: sorted position, ascending; groups are contiguous runs of u) get
// their suffix v = sa[cpos[u]] and a 32-bit second key (rank of v + h relative to the block's base, + 1; 0 past the end of the block: at
// most n <= 2^22, 23 bits) in one pass, before any rank changes. Then:
//  - groups of at most BWT_SMALL_GROUP members are sorted by that key inside the CTA that owns their first member (kz_bwt_core.cuh), which
//    writes sa, the new ranks and the "still unresolved" flag of every member directly;
//  - the members of the larger groups are selected and radix sorted on (ordinal of the large group << 23 | second key): the ordinal has at
//    most log2(m_large / (G + 1)) bits, so the key is 32 bits or a few passes above instead of 2 x 28 bits;
//  - one select of the sorted positions that are still unresolved gives the next round's members (their suffixes are read from sa).
const uint32_t BWT_NARROW_MAX_N = 1u << 22;
const uint32_t BWTN_G = bwtc::BWT_SMALL_GROUP;
const uint32_t BWTN_TILE = 2048;                          // members per CTA of the small-group pass
const uint32_t BWTN_ITEMS = (BWTN_TILE + 2 * BWTN_G + 2 + 255) / 256;
const uint32_t BWTN_WIN = BWTN_ITEMS * 256;               // window of a CTA: G members before its tile, G + 1 after (+ the end of the list)
const uint32_t BWTN_START = 1u << 31;                     // bit of a second key: the member heads its group
const uint16_t BWTN_NONE = 0xFFFF;

__global__ void __launch_bounds__(256) bwtn_keys_kernel(const uint32_t* __restrict__ sa, const uint32_t* __restrict__ rank, const uint32_t* __restrict__ cpos, uint32_t m,
                                                         const BwtBatchBlock* __restrict__ blocks, uint32_t nb, uint32_t h, uint32_t* __restrict__ key2,
                                                         uint32_t* __restrict__ val) {
    __shared__ uint32_t s_base[BWT_BATCH_MAX];
    __shared__ uint32_t s_n[BWT_BATCH_MAX];
    for (uint32_t k = threadIdx.x; k < nb; k += 256) s_base[k] = blocks[k].base, s_n[k] = blocks[k].n;
    __syncthreads();
    const uint32_t u = blockIdx.x * 256 + threadIdx.x;
    if (u >= m) return;
    const uint32_t p = cpos[u];
    const uint32_t v = sa[p];
    const uint32_t b = bwtb_find(s_base, nb, v);
    const uint32_t base = s_base[b];
    const uint32_t k = (uint64_t)v + h < (uint64_t)base + s_n[b] ? rank[v + h] - base + 1 : 0u;
    key2[u] = k | (rank[v] == p ? BWTN_START : 0u);
    val[u] = v;
}

// CTA t owns the groups whose first member lies in [t * TILE, (t + 1) * TILE). A member's group runs from the last start at or before it to the
// first start after it; the window (G before the tile, G + 1 after) holds both ends of every group of at most G members the CTA owns or
// touches, so big[u] (member of a group of more than G) is exact for the CTA's own members.
__global__ void __launch_bounds__(256) bwtn_small_kernel(const uint32_t* __restrict__ cpos, const uint32_t* __restrict__ key2, const uint32_t* __restrict__ val, uint32_t m,
                                                          uint32_t* __restrict__ sa, uint32_t* __restrict__ rank, uint8_t* __restrict__ keep, uint8_t* __restrict__ big) {
    using Scan = cub::BlockScan<uint32_t, 256>;
    __shared__ typename Scan::TempStorage s_scan;
    __shared__ uint32_t s_key[BWTN_WIN];
    __shared__ uint16_t s_prev[BWTN_WIN];  // window index of the last group start at or before w
    __shared__ uint16_t s_next[BWTN_WIN];  // window index of the first group start at or after w (W: the end of the list)
    const uint32_t t0 = blockIdx.x * BWTN_TILE;
    const uint32_t t1 = min(m, t0 + BWTN_TILE);
    const uint32_t lo = t0 > BWTN_G ? t0 - BWTN_G : 0u;
    const uint32_t hi = (uint32_t)min((uint64_t)m, (uint64_t)t0 + BWTN_TILE + BWTN_G + 1);
    const uint32_t W = hi - lo;
    for (uint32_t w = threadIdx.x; w < W; w += 256) s_key[w] = key2[lo + w];
    __syncthreads();
    uint32_t x[BWTN_ITEMS];
#pragma unroll
    for (uint32_t q = 0; q < BWTN_ITEMS; q++) {
        const uint32_t w = threadIdx.x * BWTN_ITEMS + q;
        x[q] = w < W && (s_key[w] & BWTN_START) ? w + 1 : 0u;
    }
    Scan(s_scan).InclusiveScan(x, x, cub::Max());
#pragma unroll
    for (uint32_t q = 0; q < BWTN_ITEMS; q++) {
        const uint32_t w = threadIdx.x * BWTN_ITEMS + q;
        if (w < W) s_prev[w] = x[q] ? (uint16_t)(x[q] - 1) : BWTN_NONE;
    }
    __syncthreads();
#pragma unroll
    for (uint32_t q = 0; q < BWTN_ITEMS; q++) {  // right to left: thread 0 takes the end of the window
        const uint32_t w = BWTN_WIN - 1 - (threadIdx.x * BWTN_ITEMS + q);
        x[q] = w < W ? ((s_key[w] & BWTN_START) ? w : BWTN_NONE) : (w == W && hi == m ? W : BWTN_NONE);
    }
    Scan(s_scan).InclusiveScan(x, x, cub::Min());
#pragma unroll
    for (uint32_t q = 0; q < BWTN_ITEMS; q++) {
        const uint32_t w = BWTN_WIN - 1 - (threadIdx.x * BWTN_ITEMS + q);
        if (w <= W) s_next[w] = (uint16_t)x[q];
    }
    __syncthreads();
    for (uint32_t w = threadIdx.x; w < W; w += 256) s_key[w] &= ~BWTN_START;
    __syncthreads();
    for (uint32_t w = threadIdx.x; w < W; w += 256) {
        const uint32_t u = lo + w;
        const uint32_t s = s_prev[w], e = s_next[w + 1];
        const bool small = s != BWTN_NONE && e != BWTN_NONE && e - s <= BWTN_G;
        if (u >= t0 && u < t1) big[u] = small ? 0 : 1;
        if (!small || lo + s < t0 || lo + s >= t1) continue;
        const bwtc::GroupRank g = bwtc::bwt_group_rank(s_key + s, e - s, w - s);
        const uint32_t gs = lo + s, head = cpos[gs], v = val[u];
        sa[head + g.r] = v;
        rank[v] = head + g.lt;
        keep[gs + g.r] = g.eq > 1 ? 1 : 0;
    }
}

// members l < mL of the large groups (lidx: their member indices, ascending): group starts, counted by a scan into ordinals
__global__ void __launch_bounds__(256) bwtn_lstart_kernel(const uint32_t* __restrict__ lidx, const uint32_t* __restrict__ key2, uint32_t mL, uint32_t* __restrict__ ord) {
    const uint32_t l = blockIdx.x * 256 + threadIdx.x;
    if (l < mL) ord[l] = key2[lidx[l]] >> 31;
}
template <typename K>
__global__ void __launch_bounds__(256) bwtn_lkeys_kernel(const uint32_t* __restrict__ lidx, const uint32_t* __restrict__ key2, const uint32_t* __restrict__ val,
                                                          const uint32_t* __restrict__ ord, uint32_t mL, uint32_t kb, K* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t l = blockIdx.x * 256 + threadIdx.x;
    if (l >= mL) return;
    const uint32_t u = lidx[l];
    keys[l] = ((K)(ord[l] - 1) << kb) | (K)(key2[u] & ~BWTN_START);
    vals[l] = val[u];
}
template <typename K>
__global__ void __launch_bounds__(256) bwtn_lheads_kernel(const K* __restrict__ keys, const uint32_t* __restrict__ lidx, const uint32_t* __restrict__ cpos, uint32_t mL,
                                                           uint32_t* __restrict__ f) {
    const uint32_t l = blockIdx.x * 256 + threadIdx.x;
    if (l >= mL) return;
    f[l] = (l == 0 || keys[l] != keys[l - 1]) ? cpos[lidx[l]] : 0u;
}
__global__ void __launch_bounds__(256) bwtn_lapply_kernel(uint32_t* __restrict__ f, const uint32_t* __restrict__ block_max, const uint32_t* __restrict__ lidx,
                                                           const uint32_t* __restrict__ cpos, const uint32_t* __restrict__ vals, uint32_t mL, uint32_t* __restrict__ sa,
                                                           uint32_t* __restrict__ rank) {
    const uint32_t l = blockIdx.x * 256 + threadIdx.x;
    if (l >= mL) return;
    const uint32_t blk = l / (256 * 8);
    uint32_t g = f[l];
    if (blk > 0) g = max(g, block_max[blk - 1]);
    f[l] = g;
    const uint32_t v = vals[l];
    sa[cpos[lidx[l]]] = v;
    rank[v] = g;
}
__global__ void __launch_bounds__(256) bwtn_lflags_kernel(const uint32_t* __restrict__ f, const uint32_t* __restrict__ lidx, const uint32_t* __restrict__ cpos, uint32_t mL,
                                                           uint8_t* __restrict__ keep) {
    const uint32_t l = blockIdx.x * 256 + threadIdx.x;
    if (l >= mL) return;
    const uint32_t g = f[l], u = lidx[l];
    keep[u] = (g != cpos[u] || (l + 1 < mL && f[l + 1] == g)) ? 1 : 0;
}
}  // namespace

size_t bwt_forward_batch_workspace(uint64_t total, uint32_t nblocks) {
    size_t temp = 0;
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, (int64_t)total, 0, 64);
    size_t temp2 = 0;
    cub::DeviceSelect::Flagged(nullptr, temp2, (const uint32_t*)nullptr, (const uint8_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)total);
    size_t temp3 = 0;  // no round runs a segmented sort, but its scratch size is still part of the workspace bound
    cub::DeviceSegmentedSort::SortPairs(nullptr, temp3, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)total,
                                        (int64_t)total, (const uint32_t*)nullptr, (const uint32_t*)nullptr);
    size_t temp4 = 0;  // ordinals of the large groups of a narrow round
    cub::DeviceScan::InclusiveSum(nullptr, temp4, (uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)total);
    // + the narrow rounds' large-group flags and member list (1 + 4 bytes per position)
    return (size_t)total * (8 * 2 + 4 * 2 + 4 + 4 + 4 * 4 + 1 + 1 + 4) + 4 * ((size_t)total / 2048 + 16) + (size_t)nblocks * sizeof(BwtBatchBlock) + 18 * 256 +
           std::max(std::max(temp, temp2), std::max(temp3, temp4)) + 4096;
}

namespace {
// the rounds after the first one of bwt_forward_batch when every block has at most BWT_NARROW_MAX_N bytes; the workspace buffers of the
// 56-bit rounds are reused (kv: 2 x 8 bytes per position for the large groups' keys, vv: 2 x 4 bytes for their suffixes)
struct NarrowBufs {
    uint32_t *sa, *rank, *cpos_a, *cpos_b, *key2, *val, *lidx, *count;
    uint8_t *keep, *big;
    uint64_t *kv_a, *kv_b;
    uint32_t *vv_a, *vv_b, *block_max;
    void* temp;
    size_t temp_bytes;
};
struct RoundScope {  // a part of round r timed through the hook, if any
    LzHook* hook;
    std::string name;  // the hook keeps the pointer until end()
    RoundScope(LzHook* h, int r, const char* part) : hook(h) {
        if (!hook) return;
        name = "bwt_round:" + std::to_string(r) + ":" + part;
        hook->begin(name.c_str());
    }
    ~RoundScope() {
        if (hook) hook->end();
    }
};

template <typename K>
cudaError_t bwtn_large(const NarrowBufs& B, uint32_t mL, uint32_t ob, uint32_t kb, cudaStream_t stream, uint64_t* launches, LzHook* hook, int round) {
    const uint32_t T = 256, GL = (mL + T - 1) / T, nscan = (mL + 2047) / 2048;
    K* keys_a = (K*)B.kv_a;
    K* keys_b = (K*)B.kv_b;
    {
        RoundScope rs(hook, round, "large");
        uint32_t* ord = (uint32_t*)B.kv_b;  // consumed before the sort writes there
        bwtn_lstart_kernel<<<GL, T, 0, stream>>>(B.lidx, B.key2, mL, ord);
        size_t tb = B.temp_bytes;
        cudaError_t e = cub::DeviceScan::InclusiveSum(B.temp, tb, ord, ord, (int64_t)mL, stream);
        if (e != cudaSuccess) return e;
        bwtn_lkeys_kernel<K><<<GL, T, 0, stream>>>(B.lidx, B.key2, B.val, ord, mL, kb, keys_a, B.vv_a);
        (*launches) += 4;
    }
    cub::DoubleBuffer<K> k(keys_a, keys_b);
    cub::DoubleBuffer<uint32_t> v(B.vv_a, B.vv_b);
    {
        RoundScope rs(hook, round, "sort");
        size_t tb = B.temp_bytes;
        const int end_bit = (int)(ob + kb);
        cudaError_t e = cub::DeviceRadixSort::SortPairs(B.temp, tb, k, v, (int64_t)mL, 0, end_bit, stream);
        if (e != cudaSuccess) return e;
        (*launches) += (end_bit + 7) / 8 + 1;
    }
    RoundScope rs(hook, round, "large");
    uint32_t* f = (uint32_t*)(k.Current() == keys_a ? keys_b : keys_a);  // the key buffer the sort left free
    bwtn_lheads_kernel<K><<<GL, T, 0, stream>>>(k.Current(), B.lidx, B.cpos_a, mL, f);
    scan_max_local_kernel<<<nscan, 256, 0, stream>>>(f, mL, B.block_max);
    scan_max_blocks_kernel<<<1, 1024, 0, stream>>>(B.block_max, nscan);
    bwtn_lapply_kernel<<<GL, T, 0, stream>>>(f, B.block_max, B.lidx, B.cpos_a, v.Current(), mL, B.sa, B.rank);
    bwtn_lflags_kernel<<<GL, T, 0, stream>>>(f, B.lidx, B.cpos_a, mL, B.keep);
    (*launches) += 5;
    return cudaSuccess;
}

// rounds h = 6, 12, 24, ... over the m members in B.cpos_a (sorted positions of the unresolved groups after round 0)
cudaError_t bwtn_rounds(NarrowBufs B, uint32_t m, const BwtBatchBlock* d_blocks, uint32_t nb, uint32_t max_n, cudaStream_t stream, uint64_t* launches,
                        LzHook* hook) {
    const uint32_t T = 256;
    const uint32_t kb = bwtc::bwt_bits_for(max_n);  // second key: 0 .. n
    uint32_t h = 6;
    for (int round = 1; round < 48 && m > 0; round++) {
        const uint32_t GM = (m + T - 1) / T, tiles = (m + BWTN_TILE - 1) / BWTN_TILE;
        {
            RoundScope rs(hook, round, "small");
            bwtn_keys_kernel<<<GM, T, 0, stream>>>(B.sa, B.rank, B.cpos_a, m, d_blocks, nb, h, B.key2, B.val);
            bwtn_small_kernel<<<tiles, T, 0, stream>>>(B.cpos_a, B.key2, B.val, m, B.sa, B.rank, B.keep, B.big);
            (*launches) += 2;
        }
        uint32_t mL = 0;
        {
            RoundScope rs(hook, round, "select");
            size_t tb = B.temp_bytes;
            cudaError_t e = cub::DeviceSelect::Flagged(B.temp, tb, cub::CountingInputIterator<uint32_t>(0), B.big, B.lidx, B.count, (int64_t)m, stream);
            if (e != cudaSuccess) return e;
            (*launches) += 2;
            if ((e = cudaMemcpyAsync(&mL, B.count, 4, cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
        }
        {
            RoundScope rs(hook, round, "gap");
            cudaError_t e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) return e;
        }
        if (mL > 0) {
            const uint32_t ob = bwtc::bwt_bits_for(mL / (BWTN_G + 1) - 1);  // ordinals 0 .. (large groups - 1), every large group has > G members
            const cudaError_t e = ob + kb <= 32 ? bwtn_large<uint32_t>(B, mL, ob, kb, stream, launches, hook, round)
                                                : bwtn_large<uint64_t>(B, mL, ob, kb, stream, launches, hook, round);
            if (e != cudaSuccess) return e;
        }
        h *= 2;
        if (h >= 2 * (uint64_t)max_n) break;  // every suffix pair has been compared past the end of its block
        {
            RoundScope rs(hook, round, "select");
            size_t tb = B.temp_bytes;
            cudaError_t e = cub::DeviceSelect::Flagged(B.temp, tb, (const uint32_t*)B.cpos_a, B.keep, B.cpos_b, B.count, (int64_t)m, stream);
            if (e != cudaSuccess) return e;
            (*launches) += 2;
            if ((e = cudaMemcpyAsync(&m, B.count, 4, cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
        }
        {
            RoundScope rs(hook, round, "gap");
            cudaError_t e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) return e;
        }
        std::swap(B.cpos_a, B.cpos_b);
    }
    return cudaSuccess;
}
}  // namespace
// at most this many positions / blocks in one call (keys: 2 * lg bits with total < 2^lg; 10 bits of block index in the first key)
uint64_t bwt_forward_batch_max_total() { return (1ull << 30) - 1; }
uint32_t bwt_forward_batch_max_blocks() { return BWT_BATCH_MAX; }

// BWTBlockCodec.Forward of blocks[k] = (src offset, dst offset, n >= 2, caller's block number): d_out_len[number] = n + header
cudaError_t bwt_forward_batch(const uint8_t* d_in, uint8_t* d_out, const uint64_t* src_off, const uint64_t* dst_off, const uint32_t* n_of, const uint32_t* number,
                              uint32_t nb, uint32_t* d_out_len, uint8_t* ws, size_t ws_bytes, cudaStream_t stream, uint64_t* launches, LzHook* hook,
                              bool wide_rounds) {
    if (nb == 0) return cudaSuccess;
    if (nb > (uint32_t)BWT_BATCH_MAX) return cudaErrorInvalidValue;
    std::vector<BwtBatchBlock> hb(nb);
    uint64_t total64 = 0;
    for (uint32_t k = 0; k < nb; k++) {
        const uint32_t n = n_of[k];
        if (n < 2) return cudaErrorInvalidValue;
        uint32_t log_bs = log2_floor(n);
        if (n & (n - 1)) log_bs++;
        const uint32_t pidx = (log_bs + 7) >> 3;
        if (pidx == 0 || pidx >= 5) return cudaErrorInvalidValue;
        hb[k].src_off = src_off[k], hb[k].dst_off = dst_off[k], hb[k].base = (uint32_t)total64, hb[k].n = n;
        hb[k].header = (n < 256 ? 1u : 8u) * pidx + 1;
        hb[k].pad = number[k];
        total64 += n;
    }
    if (total64 > bwt_forward_batch_max_total()) return cudaErrorInvalidValue;
    const uint32_t total = (uint32_t)total64;
    auto align = [](size_t x) { return (x + 255) & ~size_t(255); };
    size_t off = 0;
    uint64_t* keys_a = (uint64_t*)(ws + off); off = align(off + (size_t)total * 8);
    uint64_t* keys_b = (uint64_t*)(ws + off); off = align(off + (size_t)total * 8);
    uint32_t* idx_a = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    uint32_t* idx_b = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    uint32_t* rank = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    uint32_t* head = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    const uint32_t nscan = (total + 2047) / 2048;
    uint32_t* block_max = (uint32_t*)(ws + off); off = align(off + (size_t)nscan * 4);
    uint32_t* flags = (uint32_t*)(ws + off); off = align(off + 64);
    BwtBatchBlock* d_blocks = (BwtBatchBlock*)(ws + off); off = align(off + (size_t)nb * sizeof(BwtBatchBlock));
    uint32_t* cval_a = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    uint32_t* cval_b = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    uint32_t* cpos_a = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    uint32_t* cpos_b = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    uint8_t* uflags = ws + off; off = align(off + (size_t)total);
    uint8_t* big = ws + off; off = align(off + (size_t)total);
    uint32_t* lidx = (uint32_t*)(ws + off); off = align(off + (size_t)total * 4);
    uint32_t* d_count = flags + 8;
    void* temp = ws + off;
    if (ws_bytes < off) return cudaErrorInvalidValue;
    const size_t temp_bytes = ws_bytes - off;
    cudaError_t e = cudaMemcpyAsync(d_blocks, hb.data(), (size_t)nb * sizeof(BwtBatchBlock), cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
    const uint32_t T = 256, G = (total + T - 1) / T;
    uint32_t lg = 1;
    while ((1ull << lg) <= total) lg++;
    bwtb_init_keys_kernel<<<G, T, 0, stream>>>(d_in, d_blocks, nb, total, keys_a, idx_a);
    (*launches)++;
    uint32_t h = 6;
    int end_bit = 64;
    uint32_t max_n = 0;
    for (uint32_t k = 0; k < nb; k++) max_n = std::max(max_n, hb[k].n);
    // round 0: the whole batch
    uint32_t* sa = nullptr;
    {
        cub::DoubleBuffer<uint64_t> k(keys_a, keys_b);
        cub::DoubleBuffer<uint32_t> v(idx_a, idx_b);
        {
            RoundScope rs(hook, 0, "sort");
            size_t tb = temp_bytes;
            e = cub::DeviceRadixSort::SortPairs(temp, tb, k, v, (int64_t)total, 0, end_bit, stream);
            if (e != cudaSuccess) return e;
            (*launches) += 8;
        }
        const uint64_t* sk = k.Current();
        sa = v.Current();
        {
            RoundScope rs(hook, 0, "large");
            cudaMemsetAsync(flags, 0, 4, stream);
            bwt_flag_kernel<<<G, T, 0, stream>>>(sk, total, head);
            scan_max_local_kernel<<<nscan, 256, 0, stream>>>(head, total, block_max);
            scan_max_blocks_kernel<<<1, 1024, 0, stream>>>(block_max, nscan);
            bwt_apply_rank_kernel<<<G, T, 0, stream>>>(head, block_max, sa, total, rank, flags);
            (*launches) += 4;
        }
        uint32_t unsorted = 0;
        e = cudaMemcpyAsync(&unsorted, flags, 4, cudaMemcpyDeviceToHost, stream);
        if (e != cudaSuccess) return e;
        {
            RoundScope rs(hook, 0, "gap");
            e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) return e;
        }
        if (!unsorted || h >= max_n) {
            bwtb_emit_kernel<<<G, T, 0, stream>>>(d_in, d_blocks, nb, total, sa, rank, d_out);
            bwtb_header_kernel<<<(nb + 63) / 64, 64, 0, stream>>>(d_blocks, nb, rank, d_out, d_out_len);
            (*launches) += 2;
            return cudaGetLastError();
        }
    }
    // later rounds: the members of groups with more than one suffix only
    const bool narrow = !wide_rounds && max_n <= BWT_NARROW_MAX_N;
    uint32_t m = 0;
    {
        RoundScope rs(hook, 0, "select");
        bwtu_flags_full_kernel<<<G, T, 0, stream>>>(head, total, uflags);
        size_t tb = temp_bytes;
        e = cub::DeviceSelect::Flagged(temp, tb, cub::CountingInputIterator<uint32_t>(0), uflags, cpos_a, d_count, (int64_t)total, stream);
        if (e != cudaSuccess) return e;
        (*launches) += 3;
        if (!narrow) {  // the narrow rounds read the suffixes from sa
            tb = temp_bytes;
            e = cub::DeviceSelect::Flagged(temp, tb, (const uint32_t*)sa, uflags, cval_a, d_count, (int64_t)total, stream);
            if (e != cudaSuccess) return e;
            (*launches) += 2;
        }
        e = cudaMemcpyAsync(&m, d_count, 4, cudaMemcpyDeviceToHost, stream);
        if (e != cudaSuccess) return e;
    }
    {
        RoundScope rs(hook, 0, "gap");
        e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) return e;
    }
    if (narrow) {
        NarrowBufs B;
        B.sa = sa, B.rank = rank, B.cpos_a = cpos_a, B.cpos_b = cpos_b;
        B.key2 = sa == idx_a ? idx_b : idx_a, B.val = head, B.lidx = lidx, B.count = d_count;
        B.keep = uflags, B.big = big, B.kv_a = keys_a, B.kv_b = keys_b, B.vv_a = cval_a, B.vv_b = cval_b, B.block_max = block_max;
        B.temp = temp, B.temp_bytes = temp_bytes;
        e = bwtn_rounds(B, m, d_blocks, nb, max_n, stream, launches, hook);
        if (e != cudaSuccess) return e;
        m = 0;
    }
    end_bit = 2 * (int)lg;
    uint32_t* nhead = head;  // reused: new group heads of the compacted members
    // later rounds: 64-bit radix sorts of (group head, second key) over the compacted members
    for (int round = 1; round < 48 && m > 0; round++) {
        const uint32_t GM = (m + T - 1) / T, nscan_m = (m + 2047) / 2048;
        cub::DoubleBuffer<uint64_t> k(keys_a, keys_b);
        cub::DoubleBuffer<uint32_t> v(cval_a, cval_b);
        {
            RoundScope rs(hook, round, "large");
            bwtu_keys_kernel<<<GM, T, 0, stream>>>(rank, cval_a, m, d_blocks, nb, h, lg, keys_a);
        }
        {
            RoundScope rs(hook, round, "sort");
            size_t tb = temp_bytes;
            e = cub::DeviceRadixSort::SortPairs(temp, tb, k, v, (int64_t)m, 0, end_bit, stream);
            if (e != cudaSuccess) return e;
        }
        const uint32_t* sorted_val = v.Current();
        uint32_t* other = v.Current() == cval_a ? cval_b : cval_a;
        {
            RoundScope rs(hook, round, "large");
            bwtu_heads_kernel<<<GM, T, 0, stream>>>(k.Current(), cpos_a, m, nhead);
            scan_max_local_kernel<<<nscan_m, 256, 0, stream>>>(nhead, m, block_max);
            scan_max_blocks_kernel<<<1, 1024, 0, stream>>>(block_max, nscan_m);
            bwtu_apply_kernel<<<GM, T, 0, stream>>>(nhead, block_max, cpos_a, sorted_val, m, sa, rank);
        }
        (*launches) += 13;
        h *= 2;
        if (h >= 2 * (uint64_t)max_n) break;  // every suffix pair has been compared past the end of its block
        {
            RoundScope rs(hook, round, "select");
            bwtu_flags_kernel<<<GM, T, 0, stream>>>(nhead, cpos_a, m, uflags);
            size_t tb = temp_bytes;
            e = cub::DeviceSelect::Flagged(temp, tb, (const uint32_t*)cpos_a, uflags, cpos_b, d_count, (int64_t)m, stream);
            if (e != cudaSuccess) return e;
            tb = temp_bytes;
            e = cub::DeviceSelect::Flagged(temp, tb, sorted_val, uflags, other, d_count, (int64_t)m, stream);
            if (e != cudaSuccess) return e;
            (*launches) += 5;
            e = cudaMemcpyAsync(&m, d_count, 4, cudaMemcpyDeviceToHost, stream);
            if (e != cudaSuccess) return e;
        }
        {
            RoundScope rs(hook, round, "gap");
            e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) return e;
        }
        std::swap(cpos_a, cpos_b);
        if (other != cval_a) std::swap(cval_a, cval_b);  // the compacted suffixes are the next round's input
    }
    bwtb_emit_kernel<<<G, T, 0, stream>>>(d_in, d_blocks, nb, total, sa, rank, d_out);
    bwtb_header_kernel<<<(nb + 63) / 64, 64, 0, stream>>>(d_blocks, nb, rank, d_out, d_out_len);
    (*launches) += 2;
    return cudaGetLastError();
}

// ---- inverse, all blocks of a batch together ---------------------------------------------------------------------------------------------------
// The inverse of the file header (LF mapping by a stable sort, sub-lists cut every `stride` ranks, heads ranked by pointer doubling) in
// one position space for the batch (block b = [base, base + n)), the block index above the byte in the key of the stable sort (so the LF
// mapping of block b lands in its own range), one head list for all blocks, one set of launches: a 4 MiB block is 18 pointer-doubling
// launches of a few hundred threads each, so blocks inverted one after another would be mostly launch latency.
// The value that travels with the sort key is already the LF word the walk reads: (byte << 24) | local successor in 32 bits while every
// block has fewer than 2^24 bytes, (byte << 32) | local successor in 64 bits above that, so one random load per position gives both the
// successor and the output byte. Each head walks its sub-list once: the first `stage` bytes go to the head's staging slot in order, the
// length, the successor head and (for a longer sub-list) the node after the slot are recorded; once pointer doubling has given every head
// its output offset, the slots are copied to the output with coalesced stores and only the few sub-lists longer than their slot are walked
// again, from the recorded node on.
namespace {
struct IbwtBatchBlock {
    uint64_t src_off, dst_off;  // BWT bytes (behind the header) / output
    uint32_t base, n;
    uint32_t hbase, nstride;    // first head id of the block, heads on stride multiples (followed by the nprim primary heads)
    uint32_t nprim, pad;
    uint32_t prim[8];           // primary ranks (local), 0xFFFFFFFF when absent
};
const int IBWT_BATCH_MAX = 1024;
const uint32_t IBWT_NARROW_MAX_N = 0xFFFFFF;  // largest block of the 32-bit words: local ranks 0 .. n - 1 and the end mark in 24 bits
template <typename W>
struct IbwtWord;
template <>
struct IbwtWord<uint32_t> {
    static constexpr int SHIFT = 24;
    static constexpr uint32_t END = 0xFFFFFFu;  // successor of the last position of the block's list
};
template <>
struct IbwtWord<uint64_t> {
    static constexpr int SHIFT = 32;
    static constexpr uint32_t END = 0xFFFFFFFFu;
};
template <typename W>
__device__ __forceinline__ uint32_t ibwtb_next(W w) {
    return (uint32_t)(w & ((W(1) << IbwtWord<W>::SHIFT) - 1));
}
template <typename W>
__device__ __forceinline__ uint32_t ibwtb_byte(W w) {
    return (uint32_t)(w >> IbwtWord<W>::SHIFT);
}
__device__ __forceinline__ uint32_t ibwtb_find(const uint32_t* __restrict__ s_base, uint32_t nb, uint32_t i) {
    uint32_t lo = 0, hi = nb;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s_base[mid] <= i) lo = mid;
        else hi = mid;
    }
    return lo;
}
template <typename W>
__global__ void __launch_bounds__(256) ibwtb_init_kernel(const uint8_t* __restrict__ in, const IbwtBatchBlock* __restrict__ blocks, uint32_t nb, uint32_t total,
                                                          uint16_t* __restrict__ keys, W* __restrict__ vals) {
    __shared__ uint32_t s_base[IBWT_BATCH_MAX];
    for (uint32_t k = threadIdx.x; k < nb; k += 256) s_base[k] = blocks[k].base;
    __syncthreads();
    const uint32_t g = blockIdx.x * 256 + threadIdx.x;
    if (g >= total) return;
    const uint32_t b = ibwtb_find(s_base, nb, g);
    const IbwtBatchBlock& B = blocks[b];
    const uint32_t i = g - B.base;
    const uint32_t pidx = B.prim[0] + 1;
    const uint8_t c = in[B.src_off + i];
    keys[g] = (uint16_t)((b << 8) | c);
    vals[g] = ((W)c << IbwtWord<W>::SHIFT) | (i == 0 ? IbwtWord<W>::END : (i < pidx ? i - 1 : i));
}
__device__ __forceinline__ bool ibwtb_is_head(uint32_t t_local, const IbwtBatchBlock& B, uint32_t mask) {
    if ((t_local & mask) == 0) return true;
    for (uint32_t k = 0; k < B.nprim; k++)
        if (t_local == B.prim[k]) return true;
    return false;
}
__device__ __forceinline__ uint32_t ibwtb_head_id(uint32_t t_local, const IbwtBatchBlock& B, uint32_t shift) {
    if ((t_local & ((1u << shift) - 1)) == 0) return B.hbase + (t_local >> shift);
    for (uint32_t k = 0; k < B.nprim; k++)
        if (t_local == B.prim[k]) return B.hbase + B.nstride + k;
    return 0xFFFFFFFFu;
}
// heads j0 .. j1 - 1, one thread per head: walk the sub-list once; the first `stage` bytes into the head's slot, resume[j] = the node after them.
// CTAs are launched in head order, so the LF words of the resident threads come from a few consecutive blocks at a time.
template <typename W>
__global__ void __launch_bounds__(256) ibwtb_walk_kernel(const W* __restrict__ words, const IbwtBatchBlock* __restrict__ blocks, uint32_t nb, uint32_t nheads,
                                                          uint32_t shift, uint32_t stage, uint32_t* __restrict__ succ, uint32_t* __restrict__ len,
                                                          uint64_t* __restrict__ dist0, uint32_t* __restrict__ resume, uint8_t* __restrict__ slots,
                                                          uint32_t* __restrict__ bad) {
    __shared__ uint32_t s_hbase[IBWT_BATCH_MAX];
    for (uint32_t k = threadIdx.x; k < nb; k += 256) s_hbase[k] = blocks[k].hbase;
    __syncthreads();
    const uint32_t j = blockIdx.x * 256 + threadIdx.x;
    if (j >= nheads) return;
    const IbwtBatchBlock& B = blocks[ibwtb_find(s_hbase, nb, j)];
    const uint32_t n = B.n, hbase = B.hbase, nstride = B.nstride, nprim = B.nprim, mask = (1u << shift) - 1;
    uint32_t prim[8];
#pragma unroll
    for (int k = 0; k < 8; k++) prim[k] = B.prim[k];
    const uint32_t jl = j - hbase;
    uint32_t t = jl << shift;
#pragma unroll
    for (int k = 0; k < 8; k++)
        if (jl == nstride + k) t = prim[k];
    if (t >= n || (jl >= nstride && (t & mask) == 0)) {  // duplicate head or out of range
        succ[j] = 0xFFFFFFFEu;
        len[j] = 0;
        dist0[j] = 0;
        return;
    }
    const W* __restrict__ wb = words + B.base;
    uint32_t* __restrict__ slot = (uint32_t*)(slots + (size_t)j * stage);
    uint32_t l = 0, acc = 0, cur = t, s = 0xFFFFFFFFu;
    for (;;) {
        const W w = wb[cur];
        const uint32_t nx = ibwtb_next(w);
        if (l < stage) {
            acc |= ibwtb_byte(w) << ((l & 3) * 8);
            if ((l & 3) == 3) {
                slot[l >> 2] = acc;
                acc = 0;
            }
        }
        l++;
        if (l == stage) resume[j] = nx;
        if (nx == IbwtWord<W>::END) break;
        if (nx >= n || l > n) {  // corrupt permutation
            s = 0xFFFFFFFDu;
            *bad = 1;
            break;
        }
        if ((nx & mask) == 0) {
            s = hbase + (nx >> shift);
            break;
        }
#pragma unroll
        for (int k = 7; k >= 0; k--)  // the first of equal primary ranks owns the head
            if (k < (int)nprim && nx == prim[k]) s = hbase + nstride + k;
        if (s != 0xFFFFFFFFu) break;
        cur = nx;
    }
    if ((l & 3) != 0 && l < stage) slot[l >> 2] = acc;
    succ[j] = s;
    len[j] = l;
    dist0[j] = l;
}
// thread per head: its offset (corrupt input reported); then the warp copies the slots of its 32 heads one after another with coalesced
// loads and stores, and a head whose sub-list is longer than the slot walks on from the recorded node
template <typename W>
__global__ void __launch_bounds__(256) ibwtb_copy_kernel(const W* __restrict__ words, const IbwtBatchBlock* __restrict__ blocks, uint32_t nb, uint32_t nheads,
                                                          uint32_t shift, uint32_t stage, const uint32_t* __restrict__ succ0, const uint32_t* __restrict__ len,
                                                          const uint64_t* __restrict__ dist, const uint32_t* __restrict__ resume,
                                                          const uint8_t* __restrict__ slots, uint8_t* __restrict__ out, uint32_t* __restrict__ bad) {
    __shared__ uint32_t s_hbase[IBWT_BATCH_MAX];
    for (uint32_t k = threadIdx.x; k < nb; k += 256) s_hbase[k] = blocks[k].hbase;
    __syncthreads();
    const uint32_t j = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31;
    uint32_t m = 0, l = 0, n = 0, base = 0;
    uint64_t off = 0;
    uint8_t* dst = out;
    if (j < nheads && succ0[j] != 0xFFFFFFFEu) {
        const IbwtBatchBlock& B = blocks[ibwtb_find(s_hbase, nb, j)];
        n = B.n, base = B.base;
        const uint32_t jl = j - B.hbase;
        const uint32_t t = jl < B.nstride ? jl << shift : B.prim[jl - B.nstride];
        const uint64_t d = dist[j];
        // corrupt input: a head not on the list that ends the block (the permutation has more than one cycle), or the list that starts at
        // the first primary rank (the one rank no position points to) does not run through all n ranks
        if (d > n || (t == B.prim[0] && d != n)) {
            *bad = 1;
        } else {
            dst = out + B.dst_off;
            off = (uint64_t)n - d;
            l = len[j];
            m = min(l, stage);
        }
    }
    for (uint32_t q = 0; q < 32; q++) {
        const uint32_t mq = __shfl_sync(0xFFFFFFFFu, m, q);
        if (mq == 0) continue;
        const uint32_t nq = __shfl_sync(0xFFFFFFFFu, n, q);
        const uint64_t oq = ((uint64_t)__shfl_sync(0xFFFFFFFFu, (uint32_t)(off >> 32), q) << 32) | __shfl_sync(0xFFFFFFFFu, (uint32_t)off, q);
        uint8_t* const dq = (uint8_t*)(((uint64_t)__shfl_sync(0xFFFFFFFFu, (uint32_t)((uint64_t)dst >> 32), q) << 32) |
                                       __shfl_sync(0xFFFFFFFFu, (uint32_t)(uint64_t)dst, q));
        const uint32_t* __restrict__ slot = (const uint32_t*)(slots + (size_t)(j - lane + q) * stage);
        for (uint32_t w = lane; w * 4 < mq; w += 32) {
            const uint32_t v = slot[w];
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) {
                const uint32_t i = w * 4 + k;
                if (i < mq && oq + i < nq) dq[oq + i] = (uint8_t)(v >> (8 * k));
            }
        }
    }
    if (l <= stage) return;
    const W* __restrict__ wb = words + base;
    uint32_t cur = resume[j];
    for (uint32_t i = stage; i < l && cur < n; i++) {
        const W w = wb[cur];
        if (off + i < n) dst[off + i] = (uint8_t)ibwtb_byte(w);
        cur = ibwtb_next(w);
    }
}
bool ibwtb_wide(uint32_t max_n) { return max_n > IBWT_NARROW_MAX_N; }
size_t ibwtb_sort_temp(uint64_t total, bool wide) {
    size_t temp = 0;
    cub::DoubleBuffer<uint16_t> k(nullptr, nullptr);
    if (wide) {
        cub::DoubleBuffer<uint64_t> v(nullptr, nullptr);
        cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, (int64_t)total, 0, 16);
    } else {
        cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
        cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, (int64_t)total, 0, 16);
    }
    return temp;
}
struct IbwtBufs {
    uint16_t *keys_a, *keys_b;
    void *val_a, *val_b;
    uint32_t *succ_a, *succ_b, *succ0, *lenv, *resume, *bad;
    uint64_t *dist_a, *dist_b;
    uint8_t* slots;
    IbwtBatchBlock* blocks;
    void* temp;
    size_t temp_bytes;
};
template <typename W>
cudaError_t ibwtb_run(const uint8_t* d_in, uint8_t* d_out, const std::vector<IbwtBatchBlock>& hb, uint32_t total, uint32_t nheads, const IbwtBufs& U,
                      const IbwtShape& shape, cudaStream_t stream, uint64_t* launches, LzHook* hook) {
    const uint32_t nbb = (uint32_t)hb.size(), T = 256, G = (total + T - 1) / T, GH = (nheads + T - 1) / T;
    uint32_t shift = 0;
    while ((1u << shift) < shape.stride) shift++;
    cudaError_t e;
    const W* words;
    {
        LzHookScope hs(hook, "bwt_inverse:sort");
        ibwtb_init_kernel<W><<<G, T, 0, stream>>>(d_in, U.blocks, nbb, total, U.keys_a, (W*)U.val_a);
        cub::DoubleBuffer<uint16_t> k(U.keys_a, U.keys_b);
        cub::DoubleBuffer<W> v((W*)U.val_a, (W*)U.val_b);
        size_t tb = U.temp_bytes;
        int key_bits = 8;
        while ((1u << (key_bits - 8)) < nbb) key_bits++;
        if ((e = cub::DeviceRadixSort::SortPairs(U.temp, tb, k, v, (int64_t)total, 0, key_bits, stream)) != cudaSuccess) return e;  // stable: LF mapping per block
        words = v.Current();
        (*launches) += 5;
    }
    {
        LzHookScope hs(hook, "bwt_inverse:walk");
        ibwtb_walk_kernel<W><<<GH, T, 0, stream>>>(words, U.blocks, nbb, nheads, shift, shape.stage, U.succ0, U.lenv, U.dist_a, U.resume, U.slots, U.bad);
        (*launches)++;
    }
    uint32_t* succ_a = U.succ_a;
    uint32_t* succ_b = U.succ_b;
    uint64_t* dist_a = U.dist_a;
    uint64_t* dist_b = U.dist_b;
    {
        LzHookScope hs(hook, "bwt_inverse:doubling");
        if ((e = cudaMemcpyAsync(succ_a, U.succ0, (size_t)nheads * 4, cudaMemcpyDeviceToDevice, stream)) != cudaSuccess) return e;
        uint32_t max_heads = 1;
        for (const IbwtBatchBlock& B : hb) max_heads = std::max(max_heads, B.nstride + B.nprim);
        uint32_t rounds = 1;
        while ((1u << rounds) < max_heads) rounds++;
        for (uint32_t r = 0; r < rounds + 1; r++) {
            ibwt_jump_kernel<<<GH, T, 0, stream>>>(succ_a, dist_a, nheads, succ_b, dist_b);
            std::swap(succ_a, succ_b);
            std::swap(dist_a, dist_b);
            (*launches)++;
        }
    }
    {
        LzHookScope hs(hook, "bwt_inverse:copy");
        ibwtb_copy_kernel<W><<<GH, T, 0, stream>>>(words, U.blocks, nbb, nheads, shift, shape.stage, U.succ0, U.lenv, dist_a, U.resume, U.slots,
                                                                 d_out, U.bad);
        (*launches)++;
    }
    return cudaGetLastError();
}
}  // namespace

size_t bwt_inverse_batch_workspace(uint64_t total, uint32_t nblocks, uint32_t max_len, const IbwtShape& shape) {
    const bool wide = ibwtb_wide(max_len);
    const size_t nheads = (size_t)total / shape.stride + (size_t)nblocks * 10 + 16;
    return (size_t)total * (2 * 2 + (wide ? 8 : 4) * 2) + nheads * (4 * 5 + 8 * 2 + shape.stage) + (size_t)nblocks * sizeof(IbwtBatchBlock) + 17 * 256 +
           ibwtb_sort_temp(total, wide) + 4096;
}
uint64_t bwt_inverse_batch_max_total() { return (1ull << 31) - 1; }
uint32_t bwt_inverse_batch_max_blocks() { return 256; }  // 8 bits of block index above the byte in a 16-bit key

// BWTBlockCodec.Inverse of blocks k = 0..nb-1: stream at d_in + src_off[k] (len_of[k] bytes), h_headers + 64 k = its first 33 bytes on the host.
// out_len[k] = decoded length. cudaErrorInvalidValue: a malformed header (checked before anything is launched).
cudaError_t bwt_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const uint64_t* src_off, const uint64_t* dst_off, const uint32_t* len_of, const uint8_t* h_headers,
                              uint32_t nb, uint32_t cap, uint32_t* out_len, uint8_t* ws, size_t ws_bytes, cudaStream_t stream, uint64_t* launches,
                              const IbwtShape& shape, LzHook* hook) {
    if (nb == 0) return cudaSuccess;
    if (nb > bwt_inverse_batch_max_blocks()) return cudaErrorInvalidValue;
    if (shape.stride < 2 || (shape.stride & (shape.stride - 1)) || shape.stage < 4 || (shape.stage & 3)) return cudaErrorInvalidValue;
    std::vector<IbwtBatchBlock> hb;
    hb.reserve(nb);
    uint64_t total64 = 0, heads64 = 0;
    uint32_t max_n = 0;
    struct Tiny {
        uint64_t src, dst;
    };
    std::vector<Tiny> singles;
    for (uint32_t k = 0; k < nb; k++) {
        const uint32_t len = len_of[k];
        const uint8_t* hh = h_headers + (size_t)k * 64;
        if (len < 2) return cudaErrorInvalidValue;
        const uint8_t mode = hh[0];
        const uint32_t log_chunks = (mode >> 2) & 7;
        const int pidx_size = (int)(mode & 3) + 1;
        const uint32_t chunks = 1u << log_chunks;
        const uint32_t header = chunks * pidx_size + 1;
        if (len < header || chunks > 8) return cudaErrorInvalidValue;
        const uint32_t n = len - header;
        if (chunks != (n < 256 ? 1u : 8u)) return cudaErrorInvalidValue;
        out_len[k] = n;
        if (n == 0) continue;
        if (n > cap) return cudaErrorInvalidValue;
        IbwtBatchBlock B;
        for (uint32_t i = 0; i < 8; i++) B.prim[i] = 0xFFFFFFFFu;
        for (uint32_t i = 0, idx = 1; i < chunks; i++) {
            uint32_t p = 0;
            for (int q = 0; q < pidx_size; q++) p = (p << 8) | hh[idx++];
            const uint32_t pr = p + 1;
            if (pr == 0 || pr > n) return cudaErrorInvalidValue;
            B.prim[i] = pr - 1;
        }
        if (n == 1) {
            singles.push_back(Tiny{src_off[k] + header, dst_off[k]});
            continue;
        }
        B.src_off = src_off[k] + header, B.dst_off = dst_off[k], B.base = (uint32_t)total64, B.n = n;
        B.hbase = (uint32_t)heads64, B.nstride = (n + shape.stride - 1) / shape.stride, B.nprim = chunks, B.pad = 0;
        total64 += n;
        heads64 += B.nstride + B.nprim;
        max_n = std::max(max_n, n);
        hb.push_back(B);
    }
    cudaError_t e;
    for (const Tiny& t : singles)
        if ((e = cudaMemcpyAsync(d_out + t.dst, d_in + t.src, 1, cudaMemcpyDeviceToDevice, stream)) != cudaSuccess) return e;
    if (hb.empty()) return cudaSuccess;
    if (total64 > bwt_inverse_batch_max_total()) return cudaErrorInvalidValue;
    const bool wide = ibwtb_wide(max_n);
    const size_t wb = wide ? 8 : 4;
    const uint32_t total = (uint32_t)total64, nheads = (uint32_t)heads64, nbb = (uint32_t)hb.size();
    auto align = [](size_t x) { return (x + 255) & ~size_t(255); };
    size_t off = 0;
    IbwtBufs U;
    U.keys_a = (uint16_t*)(ws + off); off = align(off + (size_t)total * 2);
    U.keys_b = (uint16_t*)(ws + off); off = align(off + (size_t)total * 2);
    U.val_a = (void*)(ws + off); off = align(off + (size_t)total * wb);
    U.val_b = (void*)(ws + off); off = align(off + (size_t)total * wb);
    U.succ_a = (uint32_t*)(ws + off); off = align(off + (size_t)nheads * 4);
    U.succ_b = (uint32_t*)(ws + off); off = align(off + (size_t)nheads * 4);
    U.succ0 = (uint32_t*)(ws + off); off = align(off + (size_t)nheads * 4);
    U.lenv = (uint32_t*)(ws + off); off = align(off + (size_t)nheads * 4);
    U.resume = (uint32_t*)(ws + off); off = align(off + (size_t)nheads * 4);
    U.dist_a = (uint64_t*)(ws + off); off = align(off + (size_t)nheads * 8);
    U.dist_b = (uint64_t*)(ws + off); off = align(off + (size_t)nheads * 8);
    U.slots = ws + off; off = align(off + (size_t)nheads * shape.stage);
    U.blocks = (IbwtBatchBlock*)(ws + off); off = align(off + (size_t)nbb * sizeof(IbwtBatchBlock));
    U.bad = (uint32_t*)(ws + off); off = align(off + 64);
    U.temp = ws + off;
    if (ws_bytes < off) return cudaErrorInvalidValue;
    U.temp_bytes = ws_bytes - off;
    if ((e = cudaMemcpyAsync(U.blocks, hb.data(), (size_t)nbb * sizeof(IbwtBatchBlock), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(U.bad, 0, 4, stream)) != cudaSuccess) return e;
    // a corrupt payload (several cycles, a bad primary index) must not leave parts of the output unwritten: clear it first, report it afterwards
    for (const IbwtBatchBlock& B : hb)
        if ((e = cudaMemsetAsync(d_out + B.dst_off, 0, B.n, stream)) != cudaSuccess) return e;
    e = wide ? ibwtb_run<uint64_t>(d_in, d_out, hb, total, nheads, U, shape, stream, launches, hook)
             : ibwtb_run<uint32_t>(d_in, d_out, hb, total, nheads, U, shape, stream, launches, hook);
    if (e != cudaSuccess) return e;
    uint32_t h_bad = 0;
    {
        LzHookScope hs(hook, "bwt_inverse:sync");
        if ((e = cudaMemcpyAsync(&h_bad, U.bad, 4, cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    }
    if (h_bad) return cudaErrorInvalidValue;  // the permutation of some block is not one list through its n ranks
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// BWTS (bijective BWT, transform/BWTS.go:58-170 Forward, :211-288 Inverse).
//
// Forward. The reference builds the suffix array, finds the Lyndon factors (a factor starts where the rank of the
// suffix is smaller than every earlier one, :120-125) and repairs the order of the rotations factor by factor. The
// result is canonical: all rotations of all Lyndon factors sorted by their infinite periodic repetition, output byte =
// cyclic predecessor inside the factor (equal rotations of repeated factors carry equal bytes, so their mutual order
// does not matter). On the GPU: (1) suffix ranks by the same prefix doubling as the BWT, (2) factor starts by a
// prefix-minimum over the ranks, (3) a second prefix doubling in which "the position h bytes further" follows the
// cyclic successor inside the factor (succ_2h = succ_h o succ_h) until no group splits any more, (4) scatter.
// Inverse. The reference builds the LF mapping and walks its cycles, smallest unvisited index first, filling the output
// from the end. On the GPU: LF by one stable radix sort, cycle leaders (minimum index of a cycle) by pointer doubling of
// minima, distance from the leader by list ranking of the cycles cut at their leader, cycle offsets by a prefix sum.
// ------------------------------------------------------------------------------------------------------------
namespace {

__global__ void bwts_negrank_kernel(const uint32_t* __restrict__ rank, uint32_t n, uint32_t* __restrict__ v) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = n - rank[i];  // >= 1; larger = smaller rank
}
// in: v (n - rank), m = inclusive prefix maximum of v (finished with block_max). out: head position for the next scan
__global__ void bwts_heads_kernel(const uint32_t* __restrict__ v, const uint32_t* __restrict__ m, const uint32_t* __restrict__ block_max, uint32_t n,
                                  uint32_t* __restrict__ hpos) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool head = i == 0;
    if (i > 0) {
        const uint32_t j = i - 1;
        const uint32_t blk = j / 2048;
        uint32_t before = m[j];
        if (blk > 0) before = max(before, block_max[blk - 1]);
        head = v[i] > before;  // rank[i] smaller than every earlier rank
    }
    hpos[i] = head ? i : 0u;
}
// fstart = inclusive prefix maximum of hpos (local part in fs, block part in block_max): succ1 / pred inside the factor
__global__ void bwts_succ_kernel(const uint32_t* __restrict__ hpos, const uint32_t* __restrict__ fs, const uint32_t* __restrict__ block_max, uint32_t n,
                                 uint32_t* __restrict__ succ, uint32_t* __restrict__ pred) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t blk = i / 2048;
    uint32_t start = fs[i];
    if (blk > 0) start = max(start, block_max[blk - 1]);
    const bool last = i + 1 == n || hpos[i + 1] == i + 1;
    const uint32_t sx = last ? start : i + 1;
    succ[i] = sx;
    pred[sx] = i;
}
// first key: 7 bytes along the cyclic successor (8 bits each are enough: every rotation has all 7), succ7 for the doubling
__global__ void bwts_init_keys_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ succ1, uint32_t n, uint64_t* __restrict__ keys,
                                      uint32_t* __restrict__ idx, uint32_t* __restrict__ succ7) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t k = 0;
    uint32_t p = i;
#pragma unroll
    for (int j = 0; j < 7; j++) {
        k = (k << 9) | ((uint64_t)src[p] + 1);
        p = succ1[p];
    }
    keys[i] = k;
    idx[i] = i;
    succ7[i] = p;
}
__global__ void bwts_double_keys_kernel(const uint32_t* __restrict__ rank, const uint32_t* __restrict__ succ_h, uint32_t n, uint32_t log_n,
                                        uint64_t* __restrict__ keys, uint32_t* __restrict__ idx, uint32_t* __restrict__ succ_2h) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = succ_h[i];
    keys[i] = ((uint64_t)rank[i] << log_n) | (uint64_t)rank[s];
    idx[i] = i;
    succ_2h[i] = succ_h[s];
}
// counts the groups (positions that head their group) of the current order
__global__ void bwts_count_groups_kernel(const uint32_t* __restrict__ head, uint32_t n, uint32_t* __restrict__ count) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    const bool is_head = j < n && head[j] == j;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, is_head);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, (uint32_t)__popc(b));
}
__global__ void bwts_emit_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ sa, const uint32_t* __restrict__ pred, uint32_t n,
                                 uint8_t* __restrict__ dst) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) dst[j] = src[pred[sa[j]]];
}

// ---- inverse
__global__ void ibwts_init_kernel(const uint8_t* __restrict__ src, uint32_t n, uint8_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        keys[i] = src[i];
        vals[i] = i;
    }
}
// sorted position s holds original index v[s]  ->  lf[v[s]] = s ; min/jump initialisation
__global__ void ibwts_lf_kernel(const uint32_t* __restrict__ v, uint32_t n, uint32_t* __restrict__ lf) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) lf[v[s]] = s;
}
__global__ void ibwts_min_init_kernel(const uint32_t* __restrict__ lf, uint32_t n, uint32_t* __restrict__ mn, uint32_t* __restrict__ jp) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const uint32_t t = lf[i];
        mn[i] = min(i, t);
        jp[i] = t;
    }
}
__global__ void ibwts_min_jump_kernel(const uint32_t* __restrict__ mn_in, const uint32_t* __restrict__ jp_in, uint32_t n, uint32_t* __restrict__ mn_out,
                                      uint32_t* __restrict__ jp_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const uint32_t j = jp_in[i];
        mn_out[i] = min(mn_in[i], mn_in[j]);
        jp_out[i] = jp_in[j];
    }
}
// lists = cycles cut in front of their leader: nx[p] = lf[p], END when lf[p] leads its cycle; cnt[p] = 1
__global__ void ibwts_rank_init_kernel(const uint32_t* __restrict__ lf, const uint32_t* __restrict__ mn, uint32_t n, uint32_t* __restrict__ nx,
                                       uint32_t* __restrict__ cnt) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const uint32_t t = lf[i];
        nx[i] = mn[t] == t ? 0xFFFFFFFFu : t;
        cnt[i] = 1;
    }
}
__global__ void ibwts_rank_jump_kernel(const uint32_t* __restrict__ nx_in, const uint32_t* __restrict__ cnt_in, uint32_t n, uint32_t* __restrict__ nx_out,
                                       uint32_t* __restrict__ cnt_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const uint32_t j = nx_in[i];
        uint32_t c = cnt_in[i];
        uint32_t j2 = j;
        if (j != 0xFFFFFFFFu) {
            c += cnt_in[j];
            j2 = nx_in[j];
        }
        nx_out[i] = j2;
        cnt_out[i] = c;
    }
}
// cnt[p] = nodes from p to the end of its list; a leader's cnt is the cycle length
__global__ void ibwts_len_kernel(const uint32_t* __restrict__ mn, const uint32_t* __restrict__ cnt, uint32_t n, uint32_t* __restrict__ len_at) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) len_at[i] = mn[i] == i ? cnt[i] : 0u;
}
// exclusive sum over len_at: three-phase like scan_max (values fit 32 bits: total = n)
__global__ void scan_add_local_kernel(uint32_t* __restrict__ v, uint32_t n, uint32_t* __restrict__ block_sum) {
    __shared__ uint32_t s_warp[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t base = blockIdx.x * (blockDim.x * 8);
    uint32_t x[8];
    uint32_t run = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const uint32_t j = base + tid * 8 + q;
        const uint32_t a = j < n ? v[j] : 0u;
        x[q] = run;  // exclusive inside the thread
        run += a;
    }
    uint32_t incl = run;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= d) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < (blockDim.x >> 5) ? s_warp[lane] : 0u;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, w, d);
            if (lane >= d) w += t;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    uint32_t prev = incl - run;
    if (warp > 0) prev += s_warp[warp - 1];
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const uint32_t j = base + tid * 8 + q;
        if (j < n) v[j] = x[q] + prev;
    }
    if (tid == blockDim.x - 1) block_sum[blockIdx.x] = prev + run;
}
__global__ void scan_add_blocks_kernel(uint32_t* __restrict__ block_sum, uint32_t nblocks) {  // one thread: nblocks = n / 2048 is small
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t acc = 0;
    for (uint32_t i = 0; i < nblocks; i++) {
        const uint32_t t = block_sum[i];
        block_sum[i] = acc;
        acc += t;
    }
}
// dst[n - 1 - (offset of the cycle + steps from the leader)] = src[p]
__global__ void ibwts_write_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ mn, const uint32_t* __restrict__ cnt,
                                   const uint32_t* __restrict__ excl, const uint32_t* __restrict__ block_sum, uint32_t n, uint8_t* __restrict__ dst) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t leader = mn[p];
    const uint32_t len = cnt[leader];
    const uint32_t d = len - cnt[p];
    const uint32_t off = excl[leader] + block_sum[leader / 2048];
    const uint64_t pos = (uint64_t)off + d;
    if (pos < n) dst[n - 1 - (uint32_t)pos] = src[p];
}

}  // namespace

size_t bwts_forward_workspace(uint32_t n) { return bwt_forward_workspace(n) + (size_t)n * 4 * 4 + 4096; }
size_t bwts_inverse_workspace(uint32_t n) {
    size_t temp = 0;
    cub::DoubleBuffer<uint8_t> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, (int)n, 0, 8);
    return (size_t)n * (1 * 2 + 4 * 7) + 4 * ((size_t)n / 2048 + 16) + 4096 + temp + 4096;
}

// sorts keys_a/idx_a (n pairs), ranks the groups; returns the sorted order in *sa_out, group ranks in `rank`; flags[0] = 1 when some
// group has several members, flags[1] = number of groups
static cudaError_t bwt_sort_round(uint64_t* keys_a, uint64_t* keys_b, uint32_t* idx_a, uint32_t* idx_b, uint32_t n, int end_bit, void* temp,
                                  size_t temp_bytes, uint32_t* head, uint32_t* block_max, uint32_t nscan, uint32_t* rank, uint32_t* flags,
                                  const uint32_t** sa_out, bool count_groups, cudaStream_t stream, uint64_t* launches) {
    const uint32_t T = 256, G = (n + T - 1) / T;
    cub::DoubleBuffer<uint64_t> k(keys_a, keys_b);
    cub::DoubleBuffer<uint32_t> v(idx_a, idx_b);
    size_t tb = temp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, tb, k, v, (int)n, 0, end_bit, stream);
    if (e != cudaSuccess) return e;
    (*launches) += 8;
    const uint64_t* sk = k.Current();
    const uint32_t* sa = v.Current();
    cudaMemsetAsync(flags, 0, 8, stream);
    bwt_flag_kernel<<<G, T, 0, stream>>>(sk, n, head);
    scan_max_local_kernel<<<nscan, 256, 0, stream>>>(head, n, block_max);
    scan_max_blocks_kernel<<<1, 1024, 0, stream>>>(block_max, nscan);
    bwt_apply_rank_kernel<<<G, T, 0, stream>>>(head, block_max, sa, n, rank, flags);
    (*launches) += 4;
    if (count_groups) {
        bwts_count_groups_kernel<<<G, T, 0, stream>>>(head, n, flags + 1);
        (*launches)++;
    }
    *sa_out = sa;
    return cudaGetLastError();
}

// BWTS.Forward of one block: d_dst receives n bytes
cudaError_t bwts_forward_device(const uint8_t* d_src, uint32_t n, uint8_t* d_dst, uint8_t* ws, size_t ws_bytes, cudaStream_t stream, uint64_t* launches) {
    if (n < 2) return n == 1 ? cudaMemcpyAsync(d_dst, d_src, 1, cudaMemcpyDeviceToDevice, stream) : cudaSuccess;
    auto align = [](size_t x) { return (x + 255) & ~size_t(255); };
    size_t off = 0;
    uint64_t* keys_a = (uint64_t*)(ws + off); off = align(off + (size_t)n * 8);
    uint64_t* keys_b = (uint64_t*)(ws + off); off = align(off + (size_t)n * 8);
    uint32_t* idx_a = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* idx_b = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* rank = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* head = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* succ_a = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* succ_b = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* pred = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* aux = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    const uint32_t nscan = (n + 2047) / 2048;
    uint32_t* block_max = (uint32_t*)(ws + off); off = align(off + (size_t)nscan * 4);
    uint32_t* flags = (uint32_t*)(ws + off); off = align(off + 64);
    void* temp = ws + off;
    const size_t temp_bytes = ws_bytes > off ? ws_bytes - off : 0;
    const uint32_t T = 256, G = (n + T - 1) / T;
    uint32_t log_n = 1;
    while ((1ull << log_n) <= n) log_n++;
    // ---- (1) suffix ranks
    bwt_init_keys_kernel<<<G, T, 0, stream>>>(d_src, n, keys_a, idx_a);
    (*launches)++;
    uint32_t h = 7;
    int end_bit = 63;
    const uint32_t* sa = nullptr;
    bool done = false;
    for (int round = 0; round < 40 && !done; round++) {
        cudaError_t e = bwt_sort_round(keys_a, keys_b, idx_a, idx_b, n, end_bit, temp, temp_bytes, head, block_max, nscan, rank, flags, &sa, false, stream, launches);
        if (e != cudaSuccess) return e;
        uint32_t unsorted = 0;
        e = cudaMemcpyAsync(&unsorted, flags, 4, cudaMemcpyDeviceToHost, stream);
        if (e != cudaSuccess) return e;
        e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) return e;
        if (!unsorted || h >= n) {
            done = true;
            break;
        }
        bwt_double_keys_kernel<<<G, T, 0, stream>>>(rank, n, h, log_n, keys_a, idx_a);
        (*launches)++;
        h *= 2;
        end_bit = 2 * (int)log_n;
    }
    if (!done) return cudaErrorUnknown;
    // ---- (2) Lyndon factor starts: rank smaller than every earlier rank; cyclic successor / predecessor inside the factor
    bwts_negrank_kernel<<<G, T, 0, stream>>>(rank, n, aux);
    cudaMemcpyAsync(head, aux, (size_t)n * 4, cudaMemcpyDeviceToDevice, stream);
    scan_max_local_kernel<<<nscan, 256, 0, stream>>>(head, n, block_max);
    scan_max_blocks_kernel<<<1, 1024, 0, stream>>>(block_max, nscan);
    bwts_heads_kernel<<<G, T, 0, stream>>>(aux, head, block_max, n, succ_b /*hpos*/);
    cudaMemcpyAsync(head, succ_b, (size_t)n * 4, cudaMemcpyDeviceToDevice, stream);
    scan_max_local_kernel<<<nscan, 256, 0, stream>>>(head, n, block_max);
    scan_max_blocks_kernel<<<1, 1024, 0, stream>>>(block_max, nscan);
    bwts_succ_kernel<<<G, T, 0, stream>>>(succ_b /*hpos*/, head, block_max, n, aux /*succ1*/, pred);
    (*launches) += 7;
    // ---- (3) order of the rotations: doubling along the cyclic successor until no group splits
    bwts_init_keys_kernel<<<G, T, 0, stream>>>(d_src, aux, n, keys_a, idx_a, succ_a);
    (*launches)++;
    end_bit = 63;
    uint32_t prev_groups = 0;
    for (int round = 0; round < 64; round++) {
        cudaError_t e = bwt_sort_round(keys_a, keys_b, idx_a, idx_b, n, end_bit, temp, temp_bytes, head, block_max, nscan, rank, flags, &sa, true, stream, launches);
        if (e != cudaSuccess) return e;
        uint32_t fl[2] = {0, 0};
        e = cudaMemcpyAsync(fl, flags, 8, cudaMemcpyDeviceToHost, stream);
        if (e != cudaSuccess) return e;
        e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) return e;
        if (!fl[0] || fl[1] == prev_groups) {  // all distinct, or only equal rotations of repeated factors are left
            bwts_emit_kernel<<<G, T, 0, stream>>>(d_src, sa, pred, n, d_dst);
            (*launches)++;
            return cudaGetLastError();
        }
        prev_groups = fl[1];
        bwts_double_keys_kernel<<<G, T, 0, stream>>>(rank, succ_a, n, log_n, keys_a, idx_a, succ_b);
        (*launches)++;
        std::swap(succ_a, succ_b);
        end_bit = 2 * (int)log_n;
    }
    return cudaErrorUnknown;
}

// BWTS.Inverse of one block
cudaError_t bwts_inverse_device(const uint8_t* d_src, uint32_t n, uint8_t* d_dst, uint8_t* ws, size_t ws_bytes, cudaStream_t stream, uint64_t* launches) {
    if (n < 2) return n == 1 ? cudaMemcpyAsync(d_dst, d_src, 1, cudaMemcpyDeviceToDevice, stream) : cudaSuccess;
    auto align = [](size_t x) { return (x + 255) & ~size_t(255); };
    size_t off = 0;
    uint8_t* keys_a = ws + off; off = align(off + n);
    uint8_t* keys_b = ws + off; off = align(off + n);
    uint32_t* val_a = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* val_b = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* lf = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* a0 = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* a1 = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* b0 = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    uint32_t* b1 = (uint32_t*)(ws + off); off = align(off + (size_t)n * 4);
    const uint32_t nscan = (n + 2047) / 2048;
    uint32_t* block_sum = (uint32_t*)(ws + off); off = align(off + (size_t)nscan * 4);
    void* temp = ws + off;
    const size_t temp_bytes = ws_bytes > off ? ws_bytes - off : 0;
    const uint32_t T = 256, G = (n + T - 1) / T;
    ibwts_init_kernel<<<G, T, 0, stream>>>(d_src, n, keys_a, val_a);
    cub::DoubleBuffer<uint8_t> k(keys_a, keys_b);
    cub::DoubleBuffer<uint32_t> v(val_a, val_b);
    size_t tb = temp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, tb, k, v, (int)n, 0, 8, stream);  // stable: rank of i among equal bytes keeps the order
    if (e != cudaSuccess) return e;
    ibwts_lf_kernel<<<G, T, 0, stream>>>(v.Current(), n, lf);
    (*launches) += 10;
    uint32_t rounds = 1;
    while ((1ull << rounds) < n) rounds++;
    // cycle leaders: minimum index over the whole cycle. val_a / val_b are free again after the scatter
    uint32_t *mn = a0, *jp = a1, *mn2 = b0, *jp2 = b1;
    ibwts_min_init_kernel<<<G, T, 0, stream>>>(lf, n, mn, jp);
    for (uint32_t r = 0; r < rounds; r++) {
        ibwts_min_jump_kernel<<<G, T, 0, stream>>>(mn, jp, n, mn2, jp2);
        std::swap(mn, mn2);
        std::swap(jp, jp2);
    }
    (*launches) += rounds + 1;
    // distance to the end of the cut cycle: mn must stay intact -> use val_a/val_b and the free pair
    uint32_t* nx = jp;       // jump pointers are no longer needed
    uint32_t* cnt = mn2;
    uint32_t* nx2 = jp2;
    uint32_t* cnt2 = val_a;
    ibwts_rank_init_kernel<<<G, T, 0, stream>>>(lf, mn, n, nx, cnt);
    for (uint32_t r = 0; r < rounds; r++) {
        ibwts_rank_jump_kernel<<<G, T, 0, stream>>>(nx, cnt, n, nx2, cnt2);
        std::swap(nx, nx2);
        std::swap(cnt, cnt2);
    }
    (*launches) += rounds + 1;
    uint32_t* len_at = val_b;
    ibwts_len_kernel<<<G, T, 0, stream>>>(mn, cnt, n, len_at);
    scan_add_local_kernel<<<nscan, 256, 0, stream>>>(len_at, n, block_sum);
    scan_add_blocks_kernel<<<1, 32, 0, stream>>>(block_sum, nscan);
    ibwts_write_kernel<<<G, T, 0, stream>>>(d_src, mn, cnt, len_at, block_sum, n, d_dst);
    (*launches) += 4;
    return cudaGetLastError();
}

}  // namespace kz
