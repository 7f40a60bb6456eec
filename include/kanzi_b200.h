/*
 * kanzi_b200.h — C ABI of the H100-native (sm_90a) block compression engine (libkanzi_b200.so).
 *
 * Drop-in boundary for the per-block encode/decode path of flanglet/kanzi-go (bitstream format version 6).
 * Every entry point names the reference interface it replaces (paths relative to the reference's v2/ directory).
 * The Go host binds these through cgo (see INTEGRATION.md); tests and bench.py bind them through ctypes.
 *
 * Conventions
 *   - plain pointers and sizes only; all buffers are HOST memory unless the name ends in _device;
 *   - return value 0 = success; negative = -(kanzi error code, Definitions.go:25-46); positive 1 from
 *     kz_transform_forward = "transform asks to be skipped" (the reference returns a non-nil error, Sequence.go:100-105);
 *   - no entry point aborts or throws; kz_last_error() gives the message of the last failure on that context;
 *   - there is NO CPU fallback: if no CUDA device is usable kz_init fails with -ERR_CREATE_COMPRESSOR.
 *   - entropy type ids (entropy/EntropyCodecFactory.go:26-35): NONE 0, HUFFMAN 1, RANGE 4, ANS0 5, ANS1 8.
 *   - threads: a context is used by ONE host thread at a time; different contexts are independent (own CUDA stream, own scratch) and may be
 *     driven by different threads (goroutines locked to OS threads or not: every call selects its device itself) on the same GPU at the same
 *     time - their kernels run side by side (tests/test_gpu_contexts.py; bench.py times the -l 3 and -l 5 round trips of a step that way);
 *   - subsets of the v6 format the decoders accept (anything else answers an error, never wrong bytes; the Go caller keeps its own path then):
 *     ANS0 / ANS1 log range <= 12 (what every kanzi encoder writes; the format allows 8..15, entropy/ANSRangeCodec.go:606-609), ROLZ
 *     logPosChecks = 4 (what `-t ROLZ` writes), TEXT encoding 2 only (entropy NONE / ANS0 / HUFFMAN / RANGE, transform/Factory.go:99-119),
 *     bitstream version 6 (in a header, and as the bsVersion of a headerless reader, kz_set_headerless_reader);
 *   - transform ids (transform/Factory.go:31-50): NONE 0, BWT 1, BWTS 2, LZ 3, ZRLT 6, MTFT 7, RANK 8, ROLZ 11, LZX 16; a "transform48"
 *     word packs up to 8 six-bit ids, first transform in the top 6 bits (Factory.go:26-54).
 */
#ifndef KANZI_B200_H
#define KANZI_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kz_ctx kz_ctx;

/* kanzi error codes (Definitions.go:25-46) */
enum {
    KZ_ERR_MISSING_PARAM = 1, KZ_ERR_BLOCK_SIZE = 2, KZ_ERR_INVALID_CODEC = 3, KZ_ERR_CREATE_COMPRESSOR = 4,
    KZ_ERR_CREATE_DECOMPRESSOR = 5, KZ_ERR_WRITE_FILE = 12, KZ_ERR_PROCESS_BLOCK = 13, KZ_ERR_CREATE_CODEC = 14,
    KZ_ERR_INVALID_FILE = 15, KZ_ERR_STREAM_VERSION = 16, KZ_ERR_INVALID_PARAM = 18, KZ_ERR_CRC_CHECK = 19,
    KZ_ERR_UNKNOWN = 127
};

enum { KZ_E_NONE = 0, KZ_E_HUFFMAN = 1, KZ_E_RANGE = 4, KZ_E_ANS0 = 5, KZ_E_ANS1 = 8 };
enum { KZ_T_NONE = 0, KZ_T_BWT = 1, KZ_T_BWTS = 2, KZ_T_LZ = 3, KZ_T_ZRLT = 6, KZ_T_MTFT = 7, KZ_T_RANK = 8, KZ_T_EXE = 9, KZ_T_TEXT = 10, KZ_T_ROLZ = 11, KZ_T_MM = 15, KZ_T_LZX = 16, KZ_T_UTF = 17, KZ_T_PACK = 18, KZ_T_DNA = 19 };

/* ---- lifetime ------------------------------------------------------------------------------------------- */
int kz_device_count(void);
/* One context per GPU (one process per GPU in multi-GPU runs). Owns streams and reusable HBM scratch. */
int kz_init(int device, kz_ctx** out);
void kz_destroy(kz_ctx* ctx);
const char* kz_last_error(kz_ctx* ctx);
/* Page-locked host buffers for the Writer/Reader block buffers (io/CompressedStream.go:384-394 allocates them
 * with make([]byte)); pinned memory lets the block path overlap PCIe copies with kernels. */
void* kz_alloc_pinned(size_t bytes);
void kz_free_pinned(void* p);
/* the context's cudaStream_t (all kernels of the context are launched on it), for event timing by the caller */
void* kz_cuda_stream(kz_ctx* ctx);
/* number of kernels launched by this context since the last call with reset != 0 (bench.py's gpu_launches) */
uint64_t kz_launch_count(kz_ctx* ctx, int reset);

/* ---- kanzi.EntropyEncoder / kanzi.EntropyDecoder (Definitions.go:154-179), one block ----------------------- */
/* Replaces EntropyEncoder.Write(block) as called by encodingTask.encode (io/CompressedStream.go:906): encodes
 * src[0:n] with the codec `type` into a fresh bit string. dst receives ceil(out_bits/8) bytes, zero padded; the Go
 * shim then does obs.WriteArray(dst, out_bits). Implementations: entropy/ANSRangeCodec.go:274 (ANS0/ANS1),
 * entropy/HuffmanCodec.go:390, entropy/RangeCodec.go:223, entropy/NullEntropyCodec.go:43. */
int kz_entropy_encode(kz_ctx* ctx, uint32_t type, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, uint64_t* out_bits);
/* Replaces EntropyDecoder.Read(block) (io/CompressedStream.go:1952): decodes exactly n bytes from the bit string
 * src (src_bytes bytes, the block-local buffer the decodingTask already holds, :1875); *consumed_bits = bits read. */
int kz_entropy_decode(kz_ctx* ctx, uint32_t type, const uint8_t* src, size_t src_bytes, uint8_t* dst, size_t n, uint64_t* consumed_bits);

/* ---- kanzi.ByteTransform (Definitions.go:78-91), one block ------------------------------------------------ */
/* Replaces ByteTransform.Forward(src,dst) for one transform id (transform/BWTBlockCodec.go:78, LZCodec.go:249 ...).
 * *data_type is ctx["dataType"] (in/out, internal/Global.go DataType). Returns 1 when the transform declines. */
int kz_transform_forward(kz_ctx* ctx, uint64_t type, int* data_type, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n);
/* Replaces ByteTransform.Inverse(src,dst) (BWTBlockCodec.go:141, LZCodec.go:621 ...). */
int kz_transform_inverse(kz_ctx* ctx, uint64_t type, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n);
/* Replaces ByteTransform.MaxEncodedLen (BWTBlockCodec.go:228, LZCodec.go:935). */
size_t kz_transform_max_encoded_len(uint64_t type, size_t n);

/* ---- block dispatch: Writer.processBlock / Reader.processBlock fan-out (io/CompressedStream.go:621-710, -------
 *      :1614-1744) handing ALL blocks of a batch to the GPU in one call ------------------------------------- */
/* Replaces the goroutine-per-block encodingTask.encode (io/CompressedStream.go:729-933, everything before the
 * ordered commit). Block b is slab[b*block_stride : +block_len[b]]. On return out[b*out_stride ...] holds block b's
 * block-local bit string (mode byte, length, optional checksum, entropy coded data), zero padded, and out_bits[b]
 * its exact bit length ("written", :914); status[b] = 0 or -(error code). The caller commits them in order with
 * the 5-bit/lw-bit prefixes (:951-976). out_stride must be >= kz_max_block_output(max block_len). */
int kz_encode_blocks(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t checksum_bits, const uint8_t* slab,
                     uint64_t block_stride, const uint32_t* block_len, uint32_t nblocks, uint8_t* out, uint64_t out_stride,
                     uint64_t* out_bits, int32_t* status);
/* Replaces the concurrent part of decodingTask.decode (io/CompressedStream.go:1873-2011). Block b's bit string is
 * in[in_off[b] : in_off[b] + ceil(in_bits[b]/8)] (byte aligned, as extracted by the serial section :1816-1852).
 * Decoded bytes go to out[b*out_stride ...], out_len[b] = decoded length. block_size = stream block size (:1896).
 * Every block is decoded as if it were alone in the call: status[b] = 0 or the code of decoding block b alone (a bad block header, a
 * failed entropy decode or inverse transform, a checksum mismatch, or -KZ_ERR_WRITE_FILE when its decoded length exceeds out_stride).
 * status[] and out_len[] are written for every block; a failed block gets out_len[b] = 0, and every other block its decoded bytes.
 * Returns 0, or the code (kz_last_error: the message) of the first failing block in index order. */
int kz_decode_blocks(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t checksum_bits, const uint8_t* in,
                     const uint64_t* in_off, const uint64_t* in_bits, uint32_t nblocks, uint32_t block_size, uint8_t* out,
                     uint64_t out_stride, uint32_t* out_len, int32_t* status);
size_t kz_max_block_output(size_t block_len);

/* ---- whole stream: io.Writer.Write+Close / io.Reader.Read (io/CompressedStream.go:216-256, :524-619, :1047-1100,
 *      :1556-1612) for an in-memory input, stream header included (:429-519 / :1316-1522). jobs has no meaning on
 *      the GPU (all blocks of the input form one batch per GPU pass). ------------------------------------------ */
int kz_compress_stream(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits,
                       int64_t input_size_hint, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n);
int kz_decompress_stream(kz_ctx* ctx, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n);
size_t kz_max_stream_output(size_t n, uint32_t block_size);

/* ---- device-resident variants (inputs and outputs already in HBM; used by multi-GPU pipelines and bench.py's
 *      kernel-only `value`). Pointers are CUDA device pointers on ctx's device. Lengths / offsets are host arrays.
 *      Every device variant runs after the work already queued on the device's legacy default stream (PyTorch's default stream), and
 *      so after the blocking streams: buffers written or allocated there need no synchronisation first. Work on a non-blocking stream
 *      of the caller's must be finished by the caller. */
/* Compresses n bytes at d_src into the complete stream at d_dst (header, blocks, end marker). *out_n = stream bytes. */
int kz_compress_stream_device(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits,
                              int64_t input_size_hint, const void* d_src, size_t n, void* d_dst, size_t cap, size_t* out_n);
/* Decompresses the complete stream of n bytes at d_src (must be followed by >= 64 readable bytes) into d_dst. */
int kz_decompress_stream_device(kz_ctx* ctx, const void* d_src, size_t n, void* d_dst, size_t cap, size_t* out_n);

/* ---- many independent streams in one call (BlockCompressor / BlockDecompressor over a directory: every file is a stream of its own,
 *      app/BlockCompressor.go:543-613). The blocks of all streams run through the stages together, so a call pays the per-batch kernels
 *      and host synchronisations once instead of once per stream. -------------------------------------------------------------------------
 * Stream s is read from src + src_off[s] (src_len[s] bytes) and written to dst + dst_off[s] (at most dst_cap[s] bytes); out_len[s] = bytes
 * written. Nothing is written outside [dst_off[s], dst_off[s] + dst_cap[s]).
 * Compress: stream s is byte for byte what kz_compress_stream(ctx, transform48, entropy, block_size, checksum_bits, input_size[s],
 *   src + src_off[s], src_len[s], ...) writes (input_size NULL = 0 for every stream). Empty streams are allowed (header and end marker), as
 *   are streams shorter than 16 bytes (COPY blocks). When stream s needs more than dst_cap[s] bytes, status[s] = -KZ_ERR_WRITE_FILE,
 *   nothing is written for it and out_len[s] = the bytes it needs.
 * Compress with a block size per stream (kz_compress_streams_bs[_device]; BlockCompressor's `-b auto`, where every file gets the block
 *   size size / jobs): block_size is an array of nstreams entries, and stream s is byte for byte what kz_compress_stream writes with
 *   block_size[s]. The blocks of all streams share every pass, whatever their block sizes. A block size kz_compress_stream refuses
 *   (outside [1024, 2^30], or not a multiple of 16) fails only its own stream: status[s] = -KZ_ERR_INVALID_PARAM, out_len[s] = 0, nothing
 *   written. A NULL block_size is a call-level error. kz_compress_streams[_device] is the same call with one block size, which is
 *   checked at call level.
 * Decompress: streams may have different headers (transform, entropy, block size, checksum). Streams whose headers differ at most in block
 *   size share their walk and decode passes; each other combination of transform, entropy and checksum runs passes of its own. Stream s
 *   decodes to dst + dst_off[s]; out_len[s] = its length.
 * Status: status[s] = 0 or -(kanzi error code). A stream with status 0 is complete and correct whatever happened to the others. These errors
 *   belong to one stream: a bad header or version, a bad block prefix or block header, an entropy-decode failure, a checksum mismatch, a
 *   failing inverse transform, and dst_cap[s] too small (-KZ_ERR_WRITE_FILE); each gets the code kz_decompress_stream gives for the same
 *   bytes. A call-level failure (a bad argument, an unsupported transform or entropy codec, a CUDA error) sets every status to its code.
 *   On the compress side a transform or entropy failure on one stream's data (EXE on a malformed executable header, an entropy coder
 *   that fails on a block: where the reference fails that stream with ERR_PROCESS_BLOCK) is also call-level; compress such a batch
 *   stream by stream to find the stream. The return value is 0 when every stream succeeded, otherwise the code of the first failing
 *   stream.
 * Memory: device scratch for the stages follows the blocks of one pass (at most STREAM_PASS_BUDGET = 1 GiB of slots and entropy
 *   tables, kanzi-go_b200/csrc/kz_stream_plan.h), but a call also holds all of its inputs and all of its outputs on the device at once:
 *   compress every input, every encoded block and every assembled stream; decompress every input and, for the host variant,
 *   sum(dst_cap) bytes of staging. Split a batch larger than the GPU's memory into several calls.
 * Device variants: src / dst are device pointers, the offset and length arrays are host arrays, src, dst and every offset are multiples
 *   of 16, and >= 64 readable bytes follow each input (the rule of kz_decompress_stream_device). */
int kz_compress_streams(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits, uint32_t nstreams,
                        const uint8_t* src, const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, uint8_t* dst,
                        const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status);
int kz_decompress_streams(kz_ctx* ctx, uint32_t nstreams, const uint8_t* src, const uint64_t* src_off, const uint64_t* src_len, uint8_t* dst,
                          const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status);
int kz_compress_streams_device(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits, uint32_t nstreams,
                               const void* d_src, const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, void* d_dst,
                               const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status);
int kz_decompress_streams_device(kz_ctx* ctx, uint32_t nstreams, const void* d_src, const uint64_t* src_off, const uint64_t* src_len, void* d_dst,
                                 const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status);
int kz_compress_streams_bs(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, const uint32_t* block_size, uint32_t checksum_bits, uint32_t nstreams,
                           const uint8_t* src, const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, uint8_t* dst,
                           const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status);
int kz_compress_streams_bs_device(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, const uint32_t* block_size, uint32_t checksum_bits,
                                  uint32_t nstreams, const void* d_src, const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size,
                                  void* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status);

/* ---- sharded streams (io.Writer / io.Reader with the blocks of ONE stream spread over several GPUs; the NCCL scatter / gather of the
 *      byte ranges is the host side's business, kanzi-go_b200/parallel.py; blocks are independent: io/CompressedStream.go:896-898) ---------- */
/* Block records (5 b | lw b | payload each, :951-976) of the n bytes at d_src: no stream header, no end marker. *out_bits = exact length. */
int kz_compress_fragment_device(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits, const void* d_src, size_t n,
                                void* d_dst, size_t cap, uint64_t* out_bits);
/* Stream header (Writer.writeHeader :429-519) as bytes (out: >= 32 bytes) + its bit length. Host only. */
int kz_stream_header(uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits, int64_t input_size_hint, uint8_t* out, uint32_t* out_bits);
/* Ordered, bit-granular commit: concatenates nseg device bit strings (4-byte aligned bases) into d_dst. */
int kz_concat_bits_device(kz_ctx* ctx, uint32_t nseg, const void* const* d_seg, const uint64_t* seg_bits, void* d_dst, size_t cap, uint64_t* total_bits);
/* Header fields and record boundaries of the complete stream at d_src: rec_bit[0 .. *nblocks] (max_blocks + 1 entries). */
int kz_stream_index_device(kz_ctx* ctx, const void* d_src, size_t n, uint32_t max_blocks, uint64_t* transform48, uint32_t* entropy, uint32_t* block_size,
                           uint32_t* checksum_bits, int64_t* input_size, uint64_t* rec_bit, uint32_t* nblocks);
/* Decodes nblocks records starting at bit start_bit of the fragment at d_src (16-byte aligned, >= 64 readable bytes behind frag_bytes). */
int kz_decompress_fragment_device(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits, const void* d_src,
                                  size_t frag_bytes, uint64_t start_bit, uint32_t nblocks, void* d_dst, size_t cap, size_t* out_n);

/* ---- instrumentation ------------------------------------------------------------------------------------- */
/* Milliseconds (CUDA events on the context's stream) spent in named kernels since the last reset; names:
 * "ans0_decode", "ans0_encode", "ans0_stats", "ans_walk", "concat", "huf_encode", "huf_decode", ...  Returns
 * the number of launches accumulated, 0 if the name is unknown. Only collected when kz_profile(ctx,1) was set. */
void kz_profile(kz_ctx* ctx, int enable);
uint32_t kz_kernel_time(kz_ctx* ctx, const char* name, double* total_ms);
void kz_profile_reset(kz_ctx* ctx);
/* Algorithmic bytes of a transform stage accumulated since the last reset: name = "stage:fwd:<transform id>" or
 * "stage:inv:<transform id>" (ids of transform/Factory.go:31-50); *bytes_in / *bytes_out = stage input / output bytes summed over
 * the blocks the stage ran on. Returns the number of batches accumulated (0 = unknown name). Only with kz_profile(ctx,1).
 * Also "kernel names" (enumeration): kz_profile_names writes up to cap bytes of newline separated names, returns the full size. */
uint32_t kz_stage_bytes(kz_ctx* ctx, const char* name, uint64_t* bytes_in, uint64_t* bytes_out);
size_t kz_profile_names(kz_ctx* ctx, char* buf, size_t cap);
/* BWT forward doubling rounds of this context (a profiling aid; the default is 0 and the output bytes never depend on it):
 * bit 0: with kz_profile(ctx,1), time every round's parts under "bwt_round:<r>:<part>" (parts: small, sort, large, select, gap);
 * bit 1: run the 56-bit global sort in every round, also where the blocks would take the small-group / narrow-key rounds. */
void kz_bwt_profile(kz_ctx* ctx, int flags);

/* ctx["blockSize"] of the stream the following kz_encode_blocks / kz_transform_forward / kz_transform_inverse calls belong to
 * (io/CompressedStream.go:220,1406). Only TEXT reads it (it sizes its hash map from it, transform/TextCodec.go:1143-1156);
 * 0 (default) = the longest block of the call. kz_decode_blocks and the stream entry points know the value themselves. */
void kz_set_stream_block_size(kz_ctx* ctx, uint64_t block_size);

/* ctx["from"] / ctx["to"] (kanzi d --from / --to): decode only a range of blocks. Block ids start at 1 with the stream's first record
 * (io/CompressedStream.go:1684); block id is skipped iff id < from_block (when from_block >= 0) or id >= to_block (when to_block >= 0)
 * (:1858-1871). So to_block is exclusive, from 0 acts as from 1, and to_block <= from_block or to_block == 1 decodes nothing. A negative value
 * means "not given"; the default (-1, -1) decodes every block. Returns 0, or -KZ_ERR_INVALID_PARAM without a context.
 * Read by kz_decompress_stream, kz_decompress_stream_device, kz_decompress_streams and kz_decompress_streams_device (the same range for every
 * stream, as BlockDecompressor applies one from / to to every file) and kz_reader_open, which captures the range when the session opens
 * (later calls do not change an open session, and the call is allowed while one is open). kz_decode_blocks, kz_decompress_fragment_device, kz_entropy_* and kz_transform_* ignore it:
 * their block numbers are not stream ids. So do kz_index_build[_device] and kz_read_ranges[_device]: an index covers every record, and a
 * read selects blocks by byte offset.
 * Semantics: every record of the stream is still walked to the end marker, so a bad record length, a record past the end or a truncated
 * stream is reported wherever it lies. A skipped block is never parsed, entropy decoded, inverse transformed or checksummed: a defect inside
 * it is not an error. The output is the decoded blocks of the range back to back (out_n / out_len = their length, 0 for an empty range). The
 * error order of the sessions (below) applies to the decoded blocks. The record count limit of the whole-stream entry points (cap / 1024 + 16
 * records) applies to the decoded blocks only; with a range set, the stream's length bounds the walk. */
int kz_set_block_range(kz_ctx* ctx, int64_t from_block, int64_t to_block);

/* Headerless streams: kanzi's NewWriter(..., headerless = true) and NewHeaderlessReader (io/CompressedStream.go:216, :1060). Both are off by
 * default. Callers that store the stream parameters once (object stores, record-level compression) use them to drop the 20 to 26 header
 * bytes each stream carries.
 * kz_set_headerless_writer(ctx, 1): kz_compress_stream[_device], kz_compress_streams[_device] and kz_writer_open write no stream header
 *   (Writer.writeHeader returns at once, :430): a stream is its block records and the end marker, byte for byte the headered stream with its
 *   first header-length bits removed. An empty input gives the 8-bit end marker alone. on = 0 brings back the headered bytes. Returns 0, or
 *   -KZ_ERR_INVALID_PARAM without a context.
 * kz_set_headerless_reader: kz_decompress_stream[_device], kz_decompress_streams[_device], kz_reader_open and kz_stream_index_device read
 *   no header: they take the transform, entropy, block size and checksum of the setting and walk the records from bit 0. Every stream of
 *   a many-stream call has these parameters. kz_stream_index_device returns the setting's fields (input_size = output_size) and
 *   rec_bit[0] = 0. The block range (kz_set_block_range) applies as it does to a headered stream, and so do the error codes and their
 *   order. The setting is checked when it is made, as Reader.validateHeaderless does (:1178-1280):
 *   bs_version > 6 -KZ_ERR_INVALID_PARAM, bs_version < 6 -KZ_ERR_STREAM_VERSION (the decoders read version 6 only); an entropy id that is
 *   no kanzi id (not 0..9, or PAQ = 3), a transform word with bits above 48 or a six-bit id that is no kanzi id (not 0..19, or SNAPPY = 4)
 *   -KZ_ERR_INVALID_PARAM; block_size outside [1024, 1 GiB] -KZ_ERR_INVALID_PARAM (the reference takes any size in that range; a bad
 *   block size in a header is -KZ_ERR_BLOCK_SIZE instead); checksum_bits not 0 / 32 / 64 -KZ_ERR_INVALID_PARAM; a kanzi chain or codec
 *   the GPU path lacks -KZ_ERR_CREATE_CODEC. A failed call leaves the previous setting in place. output_size < 0 or >= 2^48 means "not
 *   given" (0); it never changes the decoded bytes. kz_clear_headerless_reader turns the setting off.
 * Both settings are read when a call starts; kz_writer_open and kz_reader_open capture them, so later changes do not reach an open session
 * (and the calls are allowed while one is open). kz_compress_fragment_device, kz_decompress_fragment_device and the block entry points
 * ignore them: they never read or write a header. */
int kz_set_headerless_writer(kz_ctx* ctx, int on);
int kz_set_headerless_reader(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits, int64_t output_size,
                             uint32_t bs_version);
int kz_clear_headerless_reader(kz_ctx* ctx);

/* kanzi's skipBlocks option (kanzi c --skip, ctx["skipBlocks"]): store incompressible blocks raw. Off by default. With on != 0, the encodes
 * that follow (kz_encode_blocks, kz_compress_stream[_device], kz_compress_streams[_device], kz_compress_fragment_device and kz_writer_open,
 * which captures the setting when the session opens, as it does the headerless writer setting) decide for every block of more than 15
 * bytes what encodingTask.encode decides (io/CompressedStream.go:778-800): the block is stored when its first four bytes are the magic
 * number of a compressed format (IsDataCompressed(GetMagicType), internal/Magic.go:73-149: only FFD8FFE0 among the JPEG keys) or when
 * ComputeFirstOrderEntropy1024 of its order-0 histogram reaches INCOMPRESSIBLE_THRESHOLD (973 of 1024, entropy/EntropyUtils.go:26). A
 * stored block is written like a block of at most 15 bytes: COPY_BLOCK_MASK set, no transform and no entropy codec, its bytes raw and the
 * checksum of the block. No transform stage runs on it, in either direction. Blocks that are not stored, and every byte with the setting
 * off, are unchanged; a stored block differs from a plain NONE & NONE block in its mode byte. The decoders need no setting.
 * Cost: one order-0 histogram pass over the input and one device-to-host copy per batch (the block heads and entropy flags together).
 * With kz_profile(ctx,1), kz_stage_bytes("skip:magic" / "skip:entropy") gives the blocks (*bytes_in) and bytes (*bytes_out) stored for
 * each reason, and kz_kernel_time("skip_hist" / "skip_decide") the test's kernels. Returns 0, or -KZ_ERR_INVALID_PARAM without a context. */
int kz_set_skip_blocks(kz_ctx* ctx, int on);

/* ---- streaming sessions: CompressedOutputStream / CompressedInputStream (io/CompressedStream.go:524-710, :1556-1744) for a stream of any
 *      length, or one that arrives in pieces (a pipe, a socket), in memory that does not grow with the stream ------------------------------
 * A zlib-style pump. The session takes ctx over until kz_*_free: the caller makes no other call on ctx in between except kz_device_bytes,
 * kz_last_error, kz_set_block_range and the headerless settings (the one-thread-at-a-time rule; one session per context). batch_blocks =
 * blocks per GPU batch (the role of kanzi's `jobs`), 1 .. 1024; kz_reader_open also takes 0: about 256 MiB of blocks per batch, resolved
 * from the block size in the stream's header (or the headerless setting).
 * Bytes: the writer's output, concatenated, is byte for byte what kz_compress_stream writes for the concatenated input with the same
 *   parameters and input_size_hint, whatever the piece sizes, batch_blocks and output caps. The reader's output is what kz_decompress_stream
 *   gives for the same stream. Bytes after the end marker are ignored, as kz_decompress_stream ignores them.
 * Progress: every call consumes or produces at least one byte, or returns an error, except: n == 0 and cap == 0; n == 0 and nothing is in
 *   flight (all input so far waits in a partly filled slot for more input or for finish); cap == 0 while finished bytes wait to be handed
 *   out (give the call room). A call may block until the batch in flight ends; it never spins.
 * Pipeline: each session owns one worker thread (created at open, joined at finish or free), one copy stream and two pinned slots each for
 *   input and output. The caller's thread fills an input slot, copies it to the device on the copy stream and hands it to the worker, which
 *   computes on ctx's stream, copies the finished bytes into an output slot and publishes them. So the caller's I/O and the copies of batch
 *   k + 1 overlap the kernels of batch k.
 * Memory: device and pinned memory depend only on (block_size, batch_blocks, chain, entropy), never on the stream's length. With
 *   B = batch_blocks * block_size:
 *   writer: pinned 2 x B input + 2 x O output, device 2 x B input + O output, O = kz_max_stream_output(B, block_size) + 64; plus the
 *     context's scratch for one batch of batch_blocks blocks (transform ping-pong buffers, entropy tables), as kz_compress_stream of B bytes.
 *   reader: pinned 2 x B input + 2 x D output, device 2 x B input, 2 x (kz_max_block_output(block_size) + 64 + B) window (at least one
 *     maximal record plus one input slot) and D decoded bytes, D = batch_blocks x (max(block_size + max(512, block_size / 16),
 *     min(max(2048, 1.5 x block_size), 2^30)) + 64), rounded up to 16 per block; plus the context's scratch for one batch. The reader sizes
 *     its buffers from the stream header, a headerless reader from its setting when it opens.
 *   kz_device_bytes: the device bytes held by ctx's scratch and an open session's buffers (the sum of their capacities); while a session is
 *   open, the scratch as it was after the worker's last batch. The pages of ctx's block caches (kz_cache_create) are added.
 * Errors: the first failure is sticky: every later call returns the same code, and kz_last_error(ctx) gives its message. The reader gives a
 *   stream with a single defect (bad header or version, bad block prefix, bad block header, entropy failure, checksum mismatch, failing
 *   inverse transform, truncation) the code kz_decompress_stream gives for those bytes (given a cap large enough that its record count limit,
 *   cap / 1024 + 16 records, does not apply). It reports in kz_decompress_stream's order: a block-level failure (block header, entropy
 *   decode, inverse transform, checksum) is held until the walk over the record prefixes reaches the end marker, since a walk error found
 *   later (a length past the end of the stream, truncation) takes precedence; among block-level failures the earliest stage wins, then the
 *   earliest block. Truncation is reported by kz_reader_finish, because until then more input may come. Nothing is handed out after the
 *   first block-level failure; the blocks decoded before it may have been, and without checksums a corrupt record length is only found
 *   when the walk fails, so blocks decoded from the records the defect made up may have been handed out too. With checksums on, no block
 *   whose checksum fails is handed out (nor any block of its batch). A record longer than kz_max_block_output(block_size) bytes fails with
 *   -KZ_ERR_PROCESS_BLOCK when the reader meets it (the code kz_decompress_stream gives when such a length runs past the end of the stream;
 *   the reader cannot hold a longer record to find out whether it does). Writing or reading after finish fails with -KZ_ERR_INVALID_PARAM.
 *   kz_*_free is legal at any point, also with a batch in flight: it joins the worker and leaves ctx usable. kz_destroy with a session open
 *   closes the session first; its handle then answers -KZ_ERR_INVALID_PARAM and must still be given to kz_*_free. */
typedef struct kz_writer kz_writer;
typedef struct kz_reader kz_reader;
/* Checks the parameters as kz_compress_stream does (unsupported chain or codec: -KZ_ERR_CREATE_CODEC) and allocates every buffer. */
int kz_writer_open(kz_ctx* ctx, uint64_t transform48, uint32_t entropy, uint32_t block_size, uint32_t checksum_bits, uint32_t batch_blocks,
                   int64_t input_size_hint, kz_writer** out);
/* Consumes up to n bytes of src, writes up to cap finished stream bytes to dst. */
int kz_writer_write(kz_writer* w, const uint8_t* src, size_t n, size_t* consumed, uint8_t* dst, size_t cap, size_t* produced);
/* End of input: last (partial) block, end marker. 0 = every byte handed out, 1 = call again with room, < 0 = error. */
int kz_writer_finish(kz_writer* w, uint8_t* dst, size_t cap, size_t* produced);
void kz_writer_free(kz_writer* w);
int kz_reader_open(kz_ctx* ctx, uint32_t batch_blocks, kz_reader** out);
int kz_reader_read(kz_reader* r, const uint8_t* src, size_t n, size_t* consumed, uint8_t* dst, size_t cap, size_t* produced);
/* End of input. 0 = end marker seen and all output handed out, 1 = call again with room, < 0 = error (e.g. truncated stream). */
int kz_reader_finish(kz_reader* r, uint8_t* dst, size_t cap, size_t* produced);
void kz_reader_free(kz_reader* r);
size_t kz_device_bytes(kz_ctx* ctx);

/* ---- stream index and batched range reads: bytes [off, off + len) of the original data without decoding the stream (an object store
 *      serving ranges of a compressed object, record-level compression, one file out of a directory stream) -----------------------------
 * Blocks are independent and every block but the last decodes to exactly block_size bytes, so decoded byte off lives in block
 * off / block_size. An index records where every block record lies in the stream; it is built once, kept (kz_index_save) beside the
 * stream, and then serves any number of reads, each of which decodes only the blocks its requests touch, every block once per call.
 * The index: a host object. It holds the stream's header fields (or the headerless reader setting in force when it is built, as
 *   kz_reader_open captures it), the stream's byte length and first 32 bytes, and for every record the first bit and the bit length of
 *   its payload. It does not own the stream and holds no device memory. kz_index_build[_device] parses the header and walks the record
 *   prefixes (twice: once to count, once to store; no limit on the record count other than the stream's length) and decodes nothing.
 *   Errors are the codes kz_decompress_stream gives for the same bytes (bad header, version or block size, a record length past the
 *   end, truncation); a kanzi chain or codec the GPU path lacks is -KZ_ERR_CREATE_CODEC. The stream of an empty input gives an index
 *   of 0 blocks. kz_index_build_device follows the rule of kz_decompress_stream_device (16-byte aligned, >= 64 readable bytes behind n).
 *   The block range (kz_set_block_range) is ignored by the index and by the reads: their block numbers come from byte offsets.
 * Size: the decoded length of the last block is not in its record, and the header's input size is a hint the decoders never trust. So
 *   *size is -1 until a read has decoded the last block, and exact afterwards; 0 from the start for a stream of 0 blocks.
 * Blob layout (kz_index_save / kz_index_load), little endian: u32 magic "KZIX" (0x58495A4B) | u32 format version 1 | u64 transform48 |
 *   u32 entropy | u32 block_size | u32 checksum_bits | u32 header bit length (0 = headerless) | i64 input_size | u64 stream_bytes |
 *   u64 nblocks | i64 size (-1 = not known) | the stream's first 32 bytes (zero padded) | nblocks x u64 payload start bit | nblocks x
 *   u64 payload bit length | u64 XXH64 (seed 0) of every byte before it. 104 + 16 x nblocks bytes. kz_index_save returns the bytes
 *   needed and writes when cap suffices. kz_index_load needs no context and no GPU; a blob is input from outside the program, so every
 *   field is checked: -KZ_ERR_INVALID_FILE for a short blob, a wrong magic, version, length or hash, fields no stream header or
 *   headerless setting can hold, records out of order, without room for their prefixes or outside stream_bytes, a size that does not
 *   fit nblocks.
 * Reads: request i asks for decoded bytes [off[i], off[i] + len[i]) and gets them at dst + dst_off[i]; out_len[i] = the bytes delivered.
 *   Nothing is written outside [dst_off[i], dst_off[i] + len[i]). pread semantics: a request that runs past the end of the data is
 *   short, 0 bytes at or beyond the end, and that is no error. Requests may overlap, repeat, come in any order and have length 0. A
 *   request that touches the last block decodes it, which sets the index's size. src / n is the stream the index was built from: a
 *   read whose n or first 32 bytes differ from the index's fails as a whole with -KZ_ERR_INVALID_PARAM before anything is decoded.
 * Errors: status[i] = 0 or -(kanzi error code). A block that fails (block header, entropy decode, inverse transform, checksum; in that
 *   order) fails exactly the requests that touch it, with the code kz_decompress_stream gives for that block under
 *   kz_set_block_range(k, k + 1); a request on several failing blocks gets the code of the first. out_len[i] = 0 and nothing is written
 *   for a failed request; requests on other blocks succeed. With checksums in the stream every decoded block is verified. A decoded
 *   block that is not the last and not exactly block_size long (no kanzi writer produces one) makes offsets behind it meaningless: the
 *   requests that touch it or any later block fail with -KZ_ERR_INVALID_FILE. Call-level failures (a bad argument, a stale index, an
 *   open session on ctx, a CUDA or allocation error) set every status and are the return value; otherwise the return value is 0 when
 *   every request succeeded, else the first failing request's code.
 * Memory: the touched blocks are decoded in passes of at most STREAM_PASS_BUDGET (1 GiB, kanzi-go_b200/csrc/kz_stream_plan.h) of
 *   scratch, three slots per block; scratch follows a pass, never the number of requests or the stream's length. On top of it the host
 *   variant holds the requested bytes once on the device (and in pinned memory) and the record windows of one pass; the device variant
 *   stages only requests whose blocks span passes. The host variant uploads only the byte windows that hold the touched records
 *   (16-byte aligned starts, 64 bytes of slack, neighbours merged) and brings the requested bytes back in one transfer.
 * Cost: one decode of each touched block plus one copy launch per pass; no record walk. With kz_profile(ctx,1):
 *   kz_stage_bytes("read:blocks") = blocks decoded / decoded bytes, ("read:h2d") = windows / bytes uploaded by the host variant,
 *   ("read:out") = slices / bytes delivered.
 * Threads: the one-thread-per-context rule; while a session is open on ctx the calls that take ctx fail with -KZ_ERR_INVALID_PARAM.
 *   An index is used by one thread at a time (a read updates its size). */
typedef struct kz_index kz_index;
int kz_index_build(kz_ctx* ctx, const uint8_t* src, size_t n, kz_index** out);
int kz_index_build_device(kz_ctx* ctx, const void* d_src, size_t n, kz_index** out);
/* Any out pointer may be NULL. *size: decoded bytes, -1 = not known yet. */
int kz_index_info(const kz_index* ix, uint64_t* transform48, uint32_t* entropy, uint32_t* block_size, uint32_t* checksum_bits, int64_t* input_size,
                  uint64_t* nblocks, uint64_t* stream_bytes, int64_t* size);
size_t kz_index_save(const kz_index* ix, uint8_t* dst, size_t cap);
int kz_index_load(const uint8_t* blob, size_t n, kz_index** out);
void kz_index_free(kz_index* ix);
int kz_read_ranges(kz_ctx* ctx, kz_index* ix, const uint8_t* src, size_t n, uint32_t nreq, const uint64_t* off, const uint64_t* len, uint8_t* dst,
                   const uint64_t* dst_off, uint64_t* out_len, int32_t* status);
/* d_src as for kz_index_build_device; d_dst and dst_off need no alignment; the offset, length and result arrays are host arrays. */
int kz_read_ranges_device(kz_ctx* ctx, kz_index* ix, const void* d_src, size_t n, uint32_t nreq, const uint64_t* off, const uint64_t* len, void* d_dst,
                          const uint64_t* dst_off, uint64_t* out_len, int32_t* status);

/* ---- writes: byte ranges written into a compressed stream, and appends, re-encoding only the blocks they touch ------------------------
 * Blocks are independent, every block but the last decodes to exactly block_size bytes, and nothing in a record depends on its position,
 *   so a write that touches blocks k .. m re-encodes only those; everything before record k stays as it is and the records behind m are
 *   copied, moved by the change in bit length. The caller rewrites only the stream's tail: for an append, the last record and the end marker.
 * Writes: write i puts data[data_off[i] .. + len[i]) at decoded offset off[i], in array order (a later write wins where writes overlap).
 *   pwrite semantics: a write that ends past the current end grows the data, and a gap between the end and a write's offset reads as zero
 *   bytes. A zero-length write changes nothing, wherever it points. off[i] == KZ_WRITE_APPEND means the current end of the data, counting
 *   the call's earlier writes.
 * Result: the new stream is src[0 .. *keep) followed by dst[0 .. *out_n). *keep = floor(cut / 8), cut being the first bit of the prefix of
 *   the first record that changes, or the end marker's first bit when the writes only add blocks behind a full last block; dst starts with
 *   the cut % 8 bits of src[*keep] that lie before the cut. A call that changes nothing returns *keep = n and *out_n = 0.
 *   The new stream is byte for byte what kz_compress_stream writes for the new data with the stream's own transform, entropy, block size,
 *   checksum bits and header input-size hint (left as it is: readers never trust it); a headerless index gives a headerless stream whatever
 *   the headerless-writer setting. This holds when the old stream is what kz_compress_stream writes for the old data under ctx's current
 *   kz_set_skip_blocks setting. Records behind the cut that are not re-encoded are copied as they are and never verified.
 * Work: a block is re-encoded when a write of length > 0 overlaps it, a zero gap covers it, or it is the old last block and the data grows
 *   past its end. Only the re-encoded old blocks the writes do not cover completely are decoded. When the index does not know the size
 *   (kz_index_info), the old last block is decoded first if the result depends on its length: a KZ_WRITE_APPEND before the writes reach
 *   past the last block's range, or a write into that range or beyond while the writes do not cover all of it. Blocks the writes cover and
 *   new blocks are never decoded. Decode and encode run in passes within the budget of the reads.
 * Index: on success ix describes the new stream: record starts and lengths, stream_bytes, the first 32 bytes, and the size, which becomes
 *   exact once the last block has been decoded or fully written (else it keeps its value). kz_index_save gives the blob kz_index_build
 *   gives for the new stream, apart from the size where the build does not know it. On any failure ix, src and the caller's bytes are
 *   unchanged.
 * Errors: a stale index (n or the first 32 bytes differ) -KZ_ERR_INVALID_PARAM, as kz_read_ranges; a chain or codec the GPU path lacks
 *   -KZ_ERR_CREATE_CODEC; an open session on ctx, len[i] > 0 with a NULL data or data_off, or a new size whose blocks x block_size pass 2^62
 *   -KZ_ERR_INVALID_PARAM. A block that must be decoded and fails returns the code kz_read_ranges gives for that block (block header,
 *   entropy, inverse transform or checksum); a decoded block before the last that is not block_size bytes long -KZ_ERR_INVALID_FILE; an
 *   encode failure its code. cap too small: -KZ_ERR_WRITE_FILE with *out_n set to the capacity the call needs, the tail's length rounded up
 *   to a multiple of 4 bytes (the tail is written in whole 32-bit words). (n - keep) + k * kz_max_block_output(block_size) + 16 bytes, k
 *   blocks re-encoded or added, always suffice.
 * Memory: one pass's scratch, the uploaded tail (host variant: src from the first record the call reads or moves, n - keep bytes or
 *   slightly more) and write bytes, the new records and the output. Appends of unbounded length through a session opened on an index are
 *   not offered.
 * With kz_profile(ctx,1): kz_stage_bytes("write:decoded") = blocks / decoded bytes, ("write:encoded") = blocks / their input bytes,
 *   ("write:moved") = runs of old records / bits re-emitted behind the re-encoded blocks, ("write:h2d") = uploads / bytes (host variant).
 * Threads: the one-thread-per-context rule; an index is used by one thread at a time. */
#define KZ_WRITE_APPEND UINT64_MAX
int kz_write_ranges(kz_ctx* ctx, kz_index* ix, const uint8_t* src, size_t n, uint32_t nw, const uint64_t* off, const uint64_t* len, const uint8_t* data,
                    const uint64_t* data_off, uint8_t* dst, size_t cap, uint64_t* keep, size_t* out_n);
/* d_src as for kz_index_build_device (16-byte aligned, at least 64 readable bytes behind it); d_dst 16-byte aligned and not overlapping
 *   d_src; d_data + data_off[i] are device bytes with no alignment rule; off, len, data_off, keep and out_n are host memory. */
int kz_write_ranges_device(kz_ctx* ctx, kz_index* ix, const void* d_src, size_t n, uint32_t nw, const uint64_t* off, const uint64_t* len,
                           const void* d_data, const uint64_t* data_off, void* d_dst, size_t cap, uint64_t* keep, size_t* out_n);

/* ---- block cache: decoded blocks kept in HBM between range reads, so that repeated reads of the same blocks (an io.ReaderAt reading a
 *      few KiB at a time, hot objects of an object store) copy instead of decoding -----------------------------------------------------------
 * A cache is made on one context with a byte budget and is used only with that context. Its device memory is allocated once, when it is
 *   made: the budget rounded down to whole pages of 64 KiB, in one allocation; nothing is allocated per entry. An entry is one decoded
 *   block on max(1, ceil(length / 64 KiB)) pages. A budget below one page (0 included) is valid and caches nothing.
 * Lifetime: free the caches of a context before kz_destroy. kz_destroy releases the pages of any cache still open; its handle then answers
 *   -KZ_ERR_INVALID_PARAM (kz_cache_stats still answers) and must still be given to kz_cache_free.
 * Reads: kz_read_ranges_cached[_device] take the arguments of kz_read_ranges[_device] plus the cache, and return exactly what those return
 *   for the same arguments: the bytes, out_len, status, the return value and the update of the index's size. Only which blocks are decoded
 *   differs. They are the only calls that read or fill a cache: whole-stream decodes, sessions and kz_read_ranges[_device] never touch one.
 *   A call hashes every record its requests touch and looks the keys up; the blocks found (hits) are served first, by one copy launch out
 *   of their pages; the others are decoded in passes as kz_read_ranges decodes them, and every one that decodes without error is inserted
 *   behind its pass. A block that fails is never inserted, so it is decoded again, and fails with the same code, on every call. A block
 *   longer than the whole budget is served as without a cache and not inserted. Refused (-KZ_ERR_INVALID_PARAM, every status) like
 *   kz_read_ranges while a session is open on ctx, and also when the cache belongs to another context or is NULL.
 * Key: an entry belongs to the content of a record, not to a stream, so one cache serves many streams and indexes (a loaded index, a
 *   second index of the same stream, identical records in different streams share entries). The key is a 64-bit hash of the record's
 *   payload bits, the bit length, the fields that change what a record decodes to (transform48, entropy, checksum_bits, block_size) and
 *   whether the record is the stream's last. The hash: the payload realigned to bit 0 and zero padded to a whole byte, XXH64 (seed 0) of
 *   every 4 KiB tile, then XXH64 (seed 0) of the tile digests and the bit length as little-endian u64. Two distinct records with the same
 *   key collide with a probability of about 2^-64 per pair; a collision would serve the other record's bytes.
 * Eviction: least recently used first, by last use (a hit or an insert); deterministic. Entries used earlier in a call may be evicted by the
 *   call's own inserts (their bytes have already been copied).
 * Cost: the device variant hashes the touched records with one launch over 4 KiB tiles plus one for the roots and one copy of the keys
 *   back; the host variant hashes them on the CPU from src and uploads only the windows of the records it misses, so a call whose blocks
 *   are all cached uploads nothing. With kz_profile(ctx,1): kz_stage_bytes("read:cache_hit" / "read:cache_miss") = blocks / decoded
 *   bytes, ("read:cache_insert" / "read:cache_evict") = entries / bytes, kz_kernel_time("record_hash") the device hashing (its two
 *   launches), "host:record_hash" the host hashing; "read:blocks" counts the blocks actually decoded.
 * Stats (kz_cache_stats; any pointer may be NULL): entries, resident_bytes (decoded bytes held), budget_bytes (as given), and since the cache
 *   was made: hits and misses (blocks looked up), inserts, evictions, served_bytes (bytes copied out of the cache to requests).
 *   kz_cache_clear drops every entry and keeps the counters.
 * kz_device_bytes(ctx) counts the pages of ctx's caches. */
typedef struct kz_cache kz_cache;
int kz_cache_create(kz_ctx* ctx, uint64_t budget_bytes, kz_cache** out);
void kz_cache_free(kz_cache* cache);
int kz_cache_clear(kz_cache* cache);
int kz_cache_stats(const kz_cache* cache, uint64_t* entries, uint64_t* resident_bytes, uint64_t* budget_bytes, uint64_t* hits, uint64_t* misses,
                   uint64_t* inserts, uint64_t* evictions, uint64_t* served_bytes);
int kz_read_ranges_cached(kz_ctx* ctx, kz_cache* cache, kz_index* ix, const uint8_t* src, size_t n, uint32_t nreq, const uint64_t* off, const uint64_t* len,
                          uint8_t* dst, const uint64_t* dst_off, uint64_t* out_len, int32_t* status);
int kz_read_ranges_cached_device(kz_ctx* ctx, kz_cache* cache, kz_index* ix, const void* d_src, size_t n, uint32_t nreq, const uint64_t* off,
                                 const uint64_t* len, void* d_dst, const uint64_t* dst_off, uint64_t* out_len, int32_t* status);

/* ---- many streams per call: index many compressed objects, and serve a batch of range reads that touches many of them, in one call
 *      each (an object store answering a batch of GETs over thousands of small objects) ----------------------------------------------------
 * Streams use the layout of kz_decompress_streams[_device]: stream s is src + src_off[s], src_len[s] bytes. Device variants: d_src and every
 *   offset of a stream a call reads are multiples of 16, and at least 64 readable bytes follow each stream.
 * Index build: out[s] and status[s] are what kz_index_build[_device] gives for stream s alone. A failed stream has out[s] = NULL and status[s]
 *   = kz_index_build's code for those bytes (a bad header, version or block size, a record past the end, truncation, -KZ_ERR_CREATE_CODEC
 *   for a chain or codec the GPU path lacks). The headerless reader setting applies to every stream. The headers are gathered by one copy
 *   launch and brought back in one transfer; all streams are walked by the two walk launches of one kz_index_build. Call-level failures
 *   (a bad argument, misalignment, an open session, CUDA or allocation errors) set every status and every out[s] = NULL. The return value
 *   is 0, the call-level code, or the first failing stream's code. Free every index that is not NULL with kz_index_free.
 * Reads: request i reads [off[i], off[i] + len[i]) of stream req_stream[i] with index ix[req_stream[i]]; cache may be NULL (uncached). Its
 *   bytes at dst + dst_off[i], out_len[i] and status[i] are exactly what kz_read_ranges[_cached][_device] returns for it when called with
 *   that index, that stream, the same cache and only that stream's requests; each index's size is updated as that call updates it. pread
 *   semantics, guards around destinations, the unseekable rule and per-block errors apply per stream.
 *   What fails a whole kz_read_ranges call fails only one stream here: a NULL ix[s], a stale index (length or first 32 bytes differ) and
 *   a chain or codec the GPU path lacks fail the requests on stream s with the code kz_read_ranges returns; the other streams are served.
 *   Call-level failures set every status and are the return value: a bad argument, req_stream[i] >= nstreams, misalignment in the device
 *   variant, an open session, a cache of another context, CUDA and allocation failures. Otherwise the return value is 0 or the first
 *   failing request's code. Streams no request names are neither checked nor read, so a caller can pass its whole object table. The same
 *   kz_index* may sit in several slots; each slot is checked against its own bytes.
 * Work: each distinct (stream slot, block) the requests touch is decoded at most once, and not at all when the cache holds it. Blocks of
 *   streams with the same transform48, entropy, block_size and checksum_bits share decode passes; blocks of different ones never do. Kernel
 *   launches and synchronisations follow the passes, not the number of streams: the device variant gathers the first 32 bytes of every
 *   named stream with one copy launch and one transfer. Cache lookups and inserts run in plan order (group of decode fields in order of
 *   first appearance, then stream slot, then block). Memory: what a kz_read_ranges pass takes, plus in the host variant the record windows
 *   of one pass across all of its streams. With kz_profile(ctx,1) the "read:*" counters count the call once, as one kz_read_ranges. */
int kz_index_build_streams(kz_ctx* ctx, uint32_t nstreams, const uint8_t* src, const uint64_t* src_off, const uint64_t* src_len, kz_index** out,
                           int32_t* status);
int kz_index_build_streams_device(kz_ctx* ctx, uint32_t nstreams, const void* d_src, const uint64_t* src_off, const uint64_t* src_len, kz_index** out,
                                  int32_t* status);
int kz_read_ranges_streams(kz_ctx* ctx, kz_cache* cache, uint32_t nstreams, kz_index* const* ix, const uint8_t* src, const uint64_t* src_off,
                           const uint64_t* src_len, uint32_t nreq, const uint32_t* req_stream, const uint64_t* off, const uint64_t* len, uint8_t* dst,
                           const uint64_t* dst_off, uint64_t* out_len, int32_t* status);
/* d_dst and dst_off need no alignment; every array is a host array. */
int kz_read_ranges_streams_device(kz_ctx* ctx, kz_cache* cache, uint32_t nstreams, kz_index* const* ix, const void* d_src, const uint64_t* src_off,
                                  const uint64_t* src_len, uint32_t nreq, const uint32_t* req_stream, const uint64_t* off, const uint64_t* len, void* d_dst,
                                  const uint64_t* dst_off, uint64_t* out_len, int32_t* status);

#ifdef __cplusplus
}
#endif
#endif /* KANZI_B200_H */
