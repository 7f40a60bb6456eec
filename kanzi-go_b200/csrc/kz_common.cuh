// Shared device/host helpers for the kanzi H100 engine.
// Bit order everywhere is kanzi's: MSB first inside bytes, fields big-endian
// (reference: v2/bitstream/DefaultOutputBitStream.go:78-96, DefaultInputBitStream.go:78-94).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define KZ_HD __host__ __device__ __forceinline__
#define KZ_D __device__ __forceinline__

// kanzi error codes (v2/Definitions.go:25-46), stored negated in status words
#define KZ_E_BLOCK_SIZE 2
#define KZ_E_INVALID_CODEC 3
#define KZ_E_PROCESS_BLOCK 13
#define KZ_E_CREATE_CODEC 14
#define KZ_E_CRC 19

namespace kz {

static const int ANS_TOP = 1 << 15;           // entropy/ANSRangeCodec.go:32
static const int ANS0_CHUNK = 16384;          // :33
static const int ANS_MAX_CHUNK = 1 << 27;     // :35
static const int HUF_CHUNK = 16384;           // entropy/HuffmanCodec.go:30
static const int HUF_MAX_BITS = 12;           // :31
static const int RANGE_CHUNK = 32768;         // entropy/RangeCodec.go:34

KZ_HD uint32_t bswap32(uint32_t x) {
#ifdef __CUDA_ARCH__
    return __byte_perm(x, 0, 0x0123);
#else
    return __builtin_bswap32(x);
#endif
}

KZ_HD uint32_t log2_floor(uint32_t x) {  // internal/Global.go:156 Log2NoCheck
#ifdef __CUDA_ARCH__
    return 31u - (uint32_t)__clz((int)x);
#else
    return 31u - (uint32_t)__builtin_clz(x);
#endif
}

// Reads `n` (1..32) bits at absolute bit position `pos` of a big-endian bit string stored in 32-bit words
// (the buffer must be readable one word past the last touched bit).
KZ_HD uint32_t bits_at(const uint32_t* __restrict__ words, uint64_t pos, uint32_t n) {
    uint64_t i = pos >> 5;
    uint32_t o = (uint32_t)(pos & 31);
    uint32_t hi = bswap32(words[i]);
    uint32_t lo = bswap32(words[i + 1]);
    uint32_t v = o ? ((hi << o) | (lo >> (32 - o))) : hi;
    return v >> (32 - n);
}

// Sequential MSB-first reader over a word buffer. `end` is the first bit that must not be consumed;
// reads past it return zeros and set `overrun` (mirrors the panic of DefaultInputBitStream.pull, :268-294).
struct BitReader {
    const uint32_t* words;
    uint64_t pos;
    uint64_t end;
    bool overrun;
    KZ_HD BitReader(const uint32_t* w, uint64_t p, uint64_t e) : words(w), pos(p), end(e), overrun(false) {}
    KZ_HD uint32_t read(uint32_t n) {  // n in 1..32
        if (pos + n > end) {
            overrun = true;
            pos += n;
            return 0;
        }
        uint32_t v = bits_at(words, pos, n);
        pos += n;
        return v;
    }
    KZ_HD void skip(uint64_t n) {
        pos += n;
        if (pos > end) overrun = true;
    }
    // entropy/EntropyUtils.go:278-296
    KZ_HD uint32_t read_varint() {
        uint32_t res = 0, shift = 0;
        for (int i = 0; i < 4; i++) {
            uint32_t v = read(8);
            res |= (v & 0x7F) << shift;
            if (v < 128) return res;
            shift += 7;
        }
        uint32_t v = read(8);
        return res | ((v & 0x0F) << 28);
    }
};

// MSB-first writer into a zero-initialised, thread-private byte buffer (no atomics).
struct BitWriter {
    uint8_t* buf;
    uint32_t pos;  // bits
    KZ_HD BitWriter(uint8_t* b, uint32_t p = 0) : buf(b), pos(p) {}
    KZ_HD void write(uint32_t value, uint32_t n) {  // n in 1..32, buffer bytes beyond pos must be zero
        if (n < 32) value &= (1u << n) - 1u;
        uint32_t done = 0;
        while (done < n) {
            uint32_t byte = pos >> 3, off = pos & 7, room = 8 - off;
            uint32_t take = (n - done) < room ? (n - done) : room;
            uint32_t bits = (value >> (n - done - take)) & ((1u << take) - 1u);
            buf[byte] |= (uint8_t)(bits << (room - take));
            pos += take;
            done += take;
        }
    }
    // entropy/EntropyUtils.go:264-275
    KZ_HD void write_varint(uint32_t v) {
        while (v >= 128) {
            write(0x80 | (v & 0x7F), 8);
            v >>= 7;
        }
        write(v, 8);
    }
};

// ---- stream records (Writer.processBlock io/CompressedStream.go:951-976, Close :593-594) ----------------------------------
// Every block of a stream is preceded by 5 bits (lw - 3) and lw bits holding its bit length `written`; the stream ends with
// END_MARKER_BITS zero bits (a record of length 0). Writes the prefix into p (8 zeroed bytes) and returns its bit count. The one
// statement of the rule: block_prefix_kernel (single-stream assembly) and the many-stream assembly of kz_api.cu both call it.
static const uint32_t END_MARKER_BITS = 8;
KZ_HD uint32_t write_block_prefix(uint8_t* p, uint64_t written) {
    uint32_t lw = 3;
    if (written >= 8) lw = log2_floor((uint32_t)(written >> 3)) + 4;
    BitWriter bw(p);
    bw.write(lw - 3, 5);
    if (lw > 32) {
        bw.write((uint32_t)(written >> 32), lw - 32);
        bw.write((uint32_t)written, 32);
    } else {
        bw.write((uint32_t)written, lw);
    }
    return bw.pos;
}

// The reader's side of write_block_prefix (Reader.processBlock :1816-1852): 5 bits lw - 3, then the record's bit length on lw bits
// (0 = the end marker). A prefix that runs past br.end leaves br.overrun set. stream_walk_kernel and walk_records both read through it.
KZ_HD uint64_t read_block_prefix(BitReader& br) {
    const uint32_t lr = br.read(5) + 3;
    if (lr > 32) {
        uint64_t hi = br.read(lr - 32);
        return (hi << 32) | br.read(32);
    }
    return br.read(lr);
}

// Resumable walk over the block records of a window [start, end) of a stream that may still be incomplete (the streaming reader):
// at most max_records records that lie completely inside the window, their payload bit offsets and lengths in bit_off / bits. It stops
// cleanly before the first record whose prefix or payload is not completely inside, and at the end marker. status is an error only for
// real corruption: a length over 2^34 bits (-KZ_E_BLOCK_SIZE, as stream_walk_kernel) or over max_bits, more than any block of the
// stream can take (-KZ_E_PROCESS_BLOCK: the code a whole-stream walk gives when such a length runs past the end of the stream).
struct WalkResult {
    uint64_t next_bit;  // first bit behind the last record found (behind the end marker when ended)
    uint32_t count;     // records found
    int32_t status;     // 0 or -(error code)
    uint32_t ended;     // 1: the end marker was read
    uint32_t pad;
};
KZ_HD WalkResult walk_records(const uint32_t* words, uint64_t start, uint64_t end, uint32_t max_records, uint64_t max_bits, uint64_t* bit_off,
                              uint64_t* bits) {
    WalkResult r = {start, 0, 0, 0, 0};
    BitReader br(words, start, end);
    while (r.count < max_records) {
        const uint64_t len = read_block_prefix(br);
        if (br.overrun) break;
        if (len == 0) {
            r.ended = 1;
            r.next_bit = br.pos;
            break;
        }
        if (len > (1ull << 34)) {
            r.status = -KZ_E_BLOCK_SIZE;
            break;
        }
        if (len > max_bits) {
            r.status = -KZ_E_PROCESS_BLOCK;
            break;
        }
        if (br.pos + len > end) break;
        bit_off[r.count] = br.pos;
        bits[r.count] = len;
        r.count++;
        br.skip(len);
        r.next_bit = br.pos;
    }
    return r;
}

// A writer session's batch of total_bits bits (its leading carry included) hands out the whole bytes and carries the last total_bits mod 8
// bits into the next batch; the last batch hands out every byte, zero padded. Returns the bytes handed out.
KZ_HD uint64_t batch_bytes_out(uint64_t total_bits, bool last, uint32_t* carry_bits) {
    *carry_bits = last ? 0 : (uint32_t)(total_bits % 8);
    return last ? (total_bits + 7) / 8 : total_bits / 8;
}

// kanzi's ctx["from"] / ctx["to"] (kz_set_block_range): block ids start at 1 with the stream's first record
// (io/CompressedStream.go:1684), and a block is skipped iff id < from (from given) or id >= to (to given) (:1858-1871); a negative value is
// "not given". As 0-based record indices: the records [*lo, *hi) are decoded (*hi >= *lo; ~0 = no end).
KZ_HD void block_range_records(int64_t from, int64_t to, uint64_t* lo, uint64_t* hi) {
    *lo = from > 1 ? (uint64_t)(from - 1) : 0;
    *hi = to < 0 ? ~0ull : to > 1 ? (uint64_t)(to - 1) : 0;
    if (*hi < *lo) *hi = *lo;
}

// The records of one walk batch that are decoded: records first .. first + count - 1 of the stream (0-based) were walked; the slice
// [*lo, *hi) of the batch lies in the range (*lo == *hi: none).
KZ_HD void block_range_slice(int64_t from, int64_t to, uint64_t first, uint32_t count, uint32_t* lo, uint32_t* hi) {
    uint64_t rlo, rhi;
    block_range_records(from, to, &rlo, &rhi);
    const uint64_t end = first + count;
    const uint64_t a = rlo < first ? first : rlo > end ? end : rlo;
    const uint64_t b = rhi < a ? a : rhi > end ? end : rhi;
    *lo = (uint32_t)(a - first);
    *hi = (uint32_t)(b - first);
}

// ---- per-block descriptor and result of the transform stages TEXT, UTF, EXE, MM, PACK / DNA (ROLZ: result only) ---------
struct StageBlock {
    uint64_t src_off;   // byte offset of the block in the source buffer
    uint64_t dst_off;   // byte offset of the block in the destination buffer
    uint32_t len;       // input length (0 = inactive block)
    uint32_t cap;       // destination capacity (forward: MaxEncodedLen; inverse: len(dst) of the reference call)
    int32_t data_type;  // forward: ctx["dataType"] before the call
    uint32_t flags;     // PACK / DNA forward: 1 for the DNA flavour (Factory.go:151-153 "packOnlyDNA"); TEXT inverse (set inside
                        // text_inverse_batch): 1 = decoded by the data-parallel path
};
struct StageResult {
    int32_t status;     // forward: 0 = transformed, 1 = skip, negative = -(error code) where the reference panics (EXE);
                        // inverse: 0 = ok, negative = -(error code)
    uint32_t out_len;
    int32_t data_type;  // forward: ctx["dataType"] after the call
    uint32_t mode;      // forward, stage specific: TEXT the mode byte (CRLF / XML flags); MM 0 delta / 1 xor coding, distance in bits
                        // 8..15; PACK 0 skip, 1 one symbol, 2 four symbols, 3 sixteen symbols, 4 digram aliases
};

// ---- block framing shared by host and device (io/CompressedStream.go) --------------------------------------
struct BlockHeader {
    uint8_t mode;
    uint8_t skip_flags;
    uint32_t pre_len;       // "preTransformLength" on decode (= postTransformLength written by the encoder)
    uint64_t checksum;
    uint64_t data_bit;      // absolute bit offset of the entropy coded data
    int32_t status;         // 0 or -(error code)
    bool copy;
};

// decodingTask.decode :1878-1914
KZ_HD BlockHeader parse_block_header(const uint32_t* words, uint64_t bit_off, uint64_t bits, uint32_t checksum_bits, uint32_t block_size) {
    BlockHeader h;
    BitReader br(words, bit_off, bit_off + bits);
    h.status = 0;
    h.mode = (uint8_t)br.read(8);
    h.skip_flags = 0;
    h.copy = (h.mode & 0x80) != 0;
    if (!h.copy) {
        if (h.mode & 0x10) h.skip_flags = (uint8_t)br.read(8);
        else h.skip_flags = (uint8_t)((h.mode << 4) | 0x0F);
    }
    uint32_t data_size = 1 + ((h.mode >> 5) & 3);
    h.pre_len = br.read(8 * data_size);
    uint64_t max_len = (uint64_t)block_size + block_size / 2;
    if (max_len < 2048) max_len = 2048;
    if (max_len > (1ull << 30)) max_len = 1ull << 30;
    if (h.pre_len == 0 || h.pre_len > max_len) h.status = -KZ_E_BLOCK_SIZE;
    h.checksum = 0;
    if (checksum_bits == 32) h.checksum = br.read(32);
    else if (checksum_bits == 64) {
        uint64_t hi = br.read(32);
        h.checksum = (hi << 32) | br.read(32);
    }
    if (br.overrun) h.status = -KZ_E_PROCESS_BLOCK;
    h.data_bit = br.pos;
    return h;
}

// encodingTask.encode :836-887: mode byte, optional skip-flag byte, length, optional checksum. Returns bit count.
KZ_HD uint32_t make_block_header(uint8_t* dst /*>=14 zeroed bytes*/, bool copy, uint32_t ntransforms, uint8_t skip_flags, uint32_t post_len,
                                 uint32_t checksum_bits, uint64_t checksum) {
    uint32_t data_size = 1;
    if (post_len >= 256) data_size = (log2_floor(post_len) >> 3) + 1;
    uint8_t mode = copy ? 0x80 : 0;
    mode |= (uint8_t)(((data_size - 1) & 3) << 5);
    BitWriter bw(dst);
    if (copy || ntransforms <= 4) {
        mode |= (uint8_t)(skip_flags >> 4);
        bw.write(mode, 8);
    } else {
        mode |= 0x10;
        bw.write(mode, 8);
        bw.write(skip_flags, 8);
    }
    bw.write(post_len, 8 * data_size);
    if (checksum_bits == 32) bw.write((uint32_t)checksum, 32);
    else if (checksum_bits == 64) {
        bw.write((uint32_t)(checksum >> 32), 32);
        bw.write((uint32_t)checksum, 32);
    }
    return bw.pos;
}

}  // namespace kz
