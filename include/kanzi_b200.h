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
 * Decoded bytes go to out[b*out_stride ...], out_len[b] = decoded length. block_size = stream block size (:1896). */
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
 *      kernel-only `value`). Pointers are CUDA device pointers on ctx's device. Lengths / offsets are host arrays. */
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
 *   are streams shorter than 16 bytes (COPY blocks). One call uses one block size: with `-b auto` every file has its own block size, and the
 *   caller groups files by block size. When stream s needs more than dst_cap[s] bytes, status[s] = -KZ_ERR_WRITE_FILE, nothing is written
 *   for it and out_len[s] = the bytes it needs.
 * Decompress: streams may have different headers (transform, entropy, block size, checksum); the library groups them. Stream s decodes to
 *   dst + dst_off[s]; out_len[s] = its length.
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
 * their block numbers are not stream ids.
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
 *   open, the scratch as it was after the worker's last batch.
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

#ifdef __cplusplus
}
#endif
#endif /* KANZI_B200_H */
