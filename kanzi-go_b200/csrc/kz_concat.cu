// Bit-granular concatenation of encoded segments into kanzi's bit-packed stream layout.
//
// The reference appends every chunk header, chunk payload, block header and block to an MSB-first bit stream with
// WriteBits / WriteArray (v2/bitstream/DefaultOutputBitStream.go:78-199; block commit io/CompressedStream.go:951-976),
// so nothing after the first chunk header is byte aligned. On the GPU every producer writes a byte-aligned segment
// into scratch memory together with its exact bit length; an exclusive scan gives each segment its destination bit and
// a gather kernel funnel-shifts the segments into place. Destination words fully covered by one segment are stored
// directly; the (at most two) boundary words of a segment are zeroed first and then OR-ed atomically.
#include "kz_ans.cuh"

namespace kz {

// ---- exclusive scan over segment bit lengths: one CTA, tiles of 1024 ---------------------------------------
__global__ void __launch_bounds__(1024) scan_bits_kernel(const uint64_t* __restrict__ seg_bits, uint64_t* __restrict__ seg_dst, int nsegs,
                                                          uint64_t base, uint64_t* __restrict__ total) {
    __shared__ uint64_t s_warp[32];
    __shared__ uint64_t s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = base;
    __syncthreads();
    for (int start = 0; start < nsegs; start += 1024) {
        const int i = start + tid;
        const uint64_t v = i < nsegs ? seg_bits[i] : 0;
        uint64_t incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint64_t w = s_warp[lane];
            uint64_t wi = w;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                uint64_t t = __shfl_up_sync(0xFFFFFFFFu, wi, d);
                if (lane >= d) wi += t;
            }
            s_warp[lane] = wi - w;  // exclusive prefix of the warp sums
        }
        __syncthreads();
        const uint64_t carry = s_carry;
        const uint64_t excl = carry + s_warp[warp] + incl - v;
        if (i < nsegs) seg_dst[i] = excl;
        __syncthreads();
        if (tid == 1023) s_carry = excl + v;
        __syncthreads();
    }
    if (tid == 0) total[0] = s_carry;
}

// dst bit positions relative to per-block bases (kz_encode_blocks layout) and per-block totals.
// blk_first[b] = index of block b's first segment, blk_first[nblocks] = nsegs; seg_off = exclusive scan over nsegs+1
// entries (the last one is a zero-length sentinel, so seg_off[nsegs] is the grand total).
__global__ void block_layout_kernel(const uint64_t* __restrict__ seg_off, const uint32_t* __restrict__ blk_first, int nblocks,
                                    const uint64_t* __restrict__ blk_base_bits, uint64_t* __restrict__ seg_dst, uint64_t* __restrict__ blk_bits) {
    const int b = blockIdx.x;
    if (b >= nblocks) return;
    const uint32_t first = blk_first[b], last = blk_first[b + 1];
    const uint64_t start = seg_off[first];
    if (threadIdx.x == 0) blk_bits[b] = seg_off[last] - start;
    const uint64_t base = blk_base_bits[b];
    for (uint32_t i = first + threadIdx.x; i < last; i += blockDim.x) seg_dst[i] = base + (seg_off[i] - start);
}

// Stream layout (io/CompressedStream.go:951-976): every block is preceded by 5 bits (lw-3) and lw bits (bit length).
// The prefix is segment blk_first[b] - 1 (reserved by the host with bit length 0 before the first scan).
__global__ void block_prefix_kernel(const uint64_t* __restrict__ seg_off, const uint32_t* __restrict__ blk_first, int nblocks, uint8_t* __restrict__ prefix_bytes /*8 per block, zeroed*/, uint64_t* __restrict__ seg_src,
                                    uint64_t* __restrict__ seg_bits, uint64_t* __restrict__ blk_bits) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const uint32_t first = blk_first[b];
    // block b's segments are [first, next prefix segment); the one after the last block is the end marker segment
    const uint32_t next_prefix = blk_first[b + 1] - 1;
    const uint64_t written = seg_off[next_prefix] - seg_off[first];
    blk_bits[b] = written;
    uint8_t* p = prefix_bytes + 8 * (size_t)b;
    const uint32_t nbits = write_block_prefix(p, written);
    seg_src[first - 1] = (uint64_t)(uintptr_t)p;
    seg_bits[first - 1] = nbits;
}

__global__ void concat_zero_kernel(const uint64_t* __restrict__ seg_bits, const uint64_t* __restrict__ seg_dst, int nsegs, uint32_t* __restrict__ dst_words) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nsegs) return;
    const uint64_t n = seg_bits[i];
    if (n == 0) return;
    const uint64_t d = seg_dst[i];
    dst_words[d >> 5] = 0;
    dst_words[(d + n - 1) >> 5] = 0;
}

// one CTA per segment (segments are at most a few thousand words; large raw copies are pre-split by the host). A segment word is the
// address of the segment's first byte, with the bit of that byte the segment starts at (0 .. 7, MSB first) in bits SEG_BIT_SHIFT and
// up (seg_source): a segment of whole bytes is its address as it is.
__global__ void __launch_bounds__(128) concat_copy_kernel(const uint64_t* __restrict__ seg_src, const uint64_t* __restrict__ seg_bits,
                                                           const uint64_t* __restrict__ seg_dst, int nsegs, uint32_t* __restrict__ dst_words) {
    const int i = blockIdx.x;
    if (i >= nsegs) return;
    const uint64_t n = seg_bits[i];
    if (n == 0) return;
    const uint64_t d = seg_dst[i];
    const uint64_t word = seg_src[i];
    const uintptr_t sp = (uintptr_t)(word & SEG_ADDR_MASK);
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(sp & ~(uintptr_t)3);
    const uint64_t s0 = (uint64_t)(sp & 3) * 8 + (word >> SEG_BIT_SHIFT);  // bit offset of the segment's first bit inside sw
    const uint64_t w0 = d >> 5, w1 = (d + n - 1) >> 5;
    const uint32_t o = (uint32_t)(d & 31);
    for (uint64_t w = w0 + threadIdx.x; w <= w1; w += blockDim.x) {
        if (w == w0) {
            const uint32_t take = (uint32_t)((32 - o) < n ? (32 - o) : n);
            const uint32_t v = bits_at(sw, s0, take) << (32 - o - take);
            if (o == 0 && take == 32) dst_words[w] = bswap32(v);
            else atomicOr(&dst_words[w], bswap32(v));
        } else {
            const uint64_t sbit = (w << 5) - d;  // segment-relative bit of this word's first bit
            const uint64_t remaining = n - sbit;
            if (remaining >= 32) {
                dst_words[w] = bswap32(bits_at(sw, s0 + sbit, 32));
            } else {
                const uint32_t r = (uint32_t)remaining;
                atomicOr(&dst_words[w], bswap32(bits_at(sw, s0 + sbit, r) << (32 - r)));
            }
        }
    }
}

}  // namespace kz

namespace kz {
// Inverse direction (decode of NONE-entropy / raw data): bytes starting at an arbitrary bit of the stream are copied
// to a byte-aligned destination (ReadArray semantics, v2/bitstream/DefaultInputBitStream.go:99-211).
__global__ void __launch_bounds__(256) extract_copy_kernel(const uint32_t* __restrict__ words, const ExtractJob* __restrict__ jobs, int njobs,
                                                            uint8_t* __restrict__ dst) {
    const int j = blockIdx.x;
    if (j >= njobs) return;
    const ExtractJob job = jobs[j];
    uint8_t* d = dst + job.dst_off;
    const uint32_t n = job.nbytes;
    // head bytes until the destination is 4-byte aligned
    uint32_t head = (uint32_t)((4 - ((uintptr_t)d & 3)) & 3);
    if (head > n) head = n;
    if (threadIdx.x < head) d[threadIdx.x] = (uint8_t)bits_at(words, job.src_bit + 8ull * threadIdx.x, 8);
    const uint32_t nw = (n - head) >> 2;
    uint32_t* dw = reinterpret_cast<uint32_t*>(d + head);
    const uint64_t sb = job.src_bit + 8ull * head;
    for (uint32_t i = threadIdx.x; i < nw; i += blockDim.x) dw[i] = bswap32(bits_at(words, sb + 32ull * i, 32));
    const uint32_t done = head + (nw << 2);
    if (threadIdx.x < n - done) d[done + threadIdx.x] = (uint8_t)bits_at(words, job.src_bit + 8ull * (done + threadIdx.x), 8);
}

// Device-to-device byte copies (blocks a transform stage declined, decoded blocks to their destination, streams to the caller's buffer).
// When source and destination share their alignment modulo 16, the body moves in 16-byte words; otherwise byte by byte.
__global__ void __launch_bounds__(256) batch_copy_kernel(const CopyJob* __restrict__ jobs, int njobs) {
    const int j = blockIdx.x;
    if (j >= njobs) return;
    const CopyJob job = jobs[j];
    const uint8_t* s = reinterpret_cast<const uint8_t*>(job.src);
    uint8_t* d = reinterpret_cast<uint8_t*>(job.dst);
    const uint64_t n = job.len;
    if (((job.src ^ job.dst) & 15) != 0) {
        for (uint64_t i = threadIdx.x; i < n; i += blockDim.x) d[i] = s[i];
        return;
    }
    uint64_t head = (16 - (job.dst & 15)) & 15;
    if (head > n) head = n;
    if (threadIdx.x < head) d[threadIdx.x] = s[threadIdx.x];
    const uint64_t nv = (n - head) >> 4;
    const uint4* sv = reinterpret_cast<const uint4*>(s + head);
    uint4* dv = reinterpret_cast<uint4*>(d + head);
    for (uint64_t i = threadIdx.x; i < nv; i += blockDim.x) dv[i] = sv[i];
    const uint64_t done = head + (nv << 4);
    if (threadIdx.x < n - done) d[done + threadIdx.x] = s[done + threadIdx.x];
}
}  // namespace kz
