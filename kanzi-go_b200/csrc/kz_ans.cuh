// Declarations shared between the rANS kernels and the host-side launcher.
#pragma once
#include "kz_common.cuh"

namespace kz {

// one entropy-coder chunk of a block's post-transform data (encode side)
struct ChunkIn {
    uint64_t src_off;  // byte offset inside the device input buffer (16-byte aligned)
    uint32_t len;
    uint32_t block;
};

// decode side: one block / one chunk
struct DecBlock {
    uint64_t data_bit;   // absolute bit offset of the entropy coded data inside the device stream buffer
    uint64_t end_bit;    // first bit past the block's bit string
    uint32_t pre_len;    // number of bytes to decode
    uint32_t nchunks;
    uint32_t chunk_base; // index of the block's first chunk
    uint32_t chunk_size; // bytes per chunk (0: the block has no chunk table entries to expand)
    uint64_t out_off;    // byte offset of the block's decoded bytes inside the output buffer (16-byte aligned)
};
struct DecChunk {
    uint64_t out_off;  // byte offset inside the output buffer (16-byte aligned)
    uint64_t end_bit;  // end of the owning block's bit string
    uint32_t out_len;
    uint32_t block;
};

static const int STATS_WARPS = 4;
static const int HDR_STRIDE = 512;             // bytes reserved per chunk header (max 3453 header bits + 19 bytes)
static const int PAY_STRIDE = 32768 + 64;      // per chunk rANS byte scratch: 2 bytes/symbol worst case + tail + alignment
static const int PAY_WORDS_END = 32768 + 32;   // 16-byte aligned end of the 16-bit word region; tail bytes follow
// encode: per warp (8 chunks): 256x8 symbol entries + 8 output rings of 64 words + 8 input rings of 16 words; 8 warps per CTA + 4096 reciprocals
static const int ENC_OUT_RING_WORDS = 64;
static const int ENC_WARP_WORDS = 256 * 8 + 8 * ENC_OUT_RING_WORDS + 8 * 16;
static const int ENC_CTA_CHUNKS = 64;
static const size_t ENC_SMEM = (4096 + 8 * ENC_WARP_WORDS) * sizeof(uint32_t);
// decode: per warp (8 chunks) 8 rings of 64 words (each 256-byte aligned) + 171x8 bucket words + 256x8 symbol words, padded
// to 256 bytes; 2 warps per CTA, plus 256 bytes of slack to align the rings
static const int DEC_BM_WORDS = 171;
static const int DEC_CTA_CHUNKS = 16;
static const int DEC_WARP_WORDS = ((8 * 64 + (DEC_BM_WORDS + 256) * 8) + 63) & ~63;
static const size_t DEC_SMEM = 2 * DEC_WARP_WORDS * sizeof(uint32_t) + 256;

// expands the per-block descriptors into per-chunk ones on the device (grid: (ceil(max chunks per block / 256), blocks))
__global__ void expand_chunks_kernel(const DecBlock* blocks, int nblocks, DecChunk* chunks);
__global__ void rcp_table_kernel(uint32_t* inv);
__global__ void ans0_stats_kernel(const uint8_t* in, const ChunkIn* chunks, int nchunks, uint32_t* enc_tab, uint8_t* hdr, uint32_t* hdr_bits,
                                  uint32_t* asz_out);
__global__ void ans0_encode_kernel(const uint8_t* in, const ChunkIn* chunks, int nchunks, const uint32_t* enc_tab, const uint32_t* rcp, uint8_t* hdr,
                                   const uint32_t* hdr_bits, const uint32_t* asz_in, uint8_t* pay, uint64_t* seg_src, uint64_t* seg_bits,
                                   const uint32_t* seg_index);
__global__ void ans_walk_kernel(const uint32_t* words, const DecBlock* blocks, int nblocks, int order, uint64_t* chunk_hdr_bit, uint64_t* blk_end,
                                int32_t* status);
__global__ void ans0_walk_kernel(const uint32_t* words, uint64_t words_len, const DecBlock* blocks, int nblocks, uint64_t* chunk_hdr_bit,
                                 uint64_t* blk_end, int32_t* status);
// per chunk record written by ans0_tables_kernel: 171 bucket words | 256 symbol entries | 12 words of chunk state
static const int DEC_TAB_WORDS = 440;
__global__ void ans0_tables_kernel(const uint32_t* words, uint64_t words_len, const DecChunk* chunks, int nchunks, const uint64_t* chunk_hdr_bit,
                                   uint32_t* tabs, uint8_t* out, int32_t* status);
__global__ void ans0_decode_kernel(const uint32_t* words, uint64_t words_len, const uint32_t* tabs, const DecChunk* chunks, int nchunks,
                                   const uint64_t* chunk_hdr_bit, uint8_t* out, int32_t* status);

// ---- bit-granular concatenation (kz_concat.cu)
// seg_dst[i] = absolute destination bit of segment i; copies seg_bits[i] bits from seg_src[i]: a byte address (any alignment), and in the
// top bits the bit of that byte the segment starts at (seg_source)
static const uint32_t SEG_BIT_SHIFT = 61;
static const uint64_t SEG_ADDR_MASK = (1ull << SEG_BIT_SHIFT) - 1;
inline uint64_t seg_source(const void* p, uint64_t bit) { return (uint64_t)(uintptr_t)((const uint8_t*)p + bit / 8) | ((bit % 8) << SEG_BIT_SHIFT); }
__global__ void concat_copy_kernel(const uint64_t* seg_src, const uint64_t* seg_bits, const uint64_t* seg_dst, int nsegs, uint32_t* dst_words);
// exclusive scan of seg_bits (one CTA): seg_dst[i] = base + sum_{k<i} bits[k]; total[0] = base + sum
__global__ void scan_bits_kernel(const uint64_t* seg_bits, uint64_t* seg_dst, int nsegs, uint64_t base, uint64_t* total);
__global__ void block_layout_kernel(const uint64_t* seg_off, const uint32_t* blk_first, int nblocks, const uint64_t* blk_base_bits, uint64_t* seg_dst,
                                    uint64_t* blk_bits);
__global__ void block_prefix_kernel(const uint64_t* seg_off, const uint32_t* blk_first, int nblocks, uint8_t* prefix_bytes, uint64_t* seg_src,
                                    uint64_t* seg_bits, uint64_t* blk_bits);
__global__ void concat_zero_kernel(const uint64_t* seg_bits, const uint64_t* seg_dst, int nsegs, uint32_t* dst_words);
// byte-aligned extraction of `nbytes` bytes starting at absolute bit `src_bit` of a big-endian bit string
struct ExtractJob {
    uint64_t src_bit;
    uint64_t dst_off;
    uint32_t nbytes;
    uint32_t pad;
};
__global__ void extract_copy_kernel(const uint32_t* words, const ExtractJob* jobs, int njobs, uint8_t* dst);

// A list of byte copies between device addresses, one CTA per job. The host cuts longer copies into pieces of at most COPY_PIECE bytes.
struct CopyJob {
    uint64_t src, dst;  // device addresses
    uint64_t len;
};
static const uint64_t COPY_PIECE = 64 * 1024;
__global__ void batch_copy_kernel(const CopyJob* jobs, int njobs);

}  // namespace kz
