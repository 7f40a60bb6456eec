// The stream index (kz_index_*) and the plan of a batched range read (kz_read_ranges, kz_api.cu). Pure host code: no CUDA types, so that
// tests/host/read_plan_host.cpp compiles it with g++ and checks it on the CPU, the blob parser under the sanitizers.
//
// Blocks are independent and every block but the last decodes to exactly block_size bytes, so decoded byte `off` lives in block
// off / block_size. An index keeps where every block record lies in the stream; a read decodes the distinct blocks its requests touch,
// each once, in passes cut by the decode rule of kz_stream_plan.h, and copies the requested slices out of them.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "kz_stream_plan.h"
#include "kz_xxh64_core.cuh"

namespace kz {

// ---- the index -------------------------------------------------------------------------------------------------------------------
const uint32_t INDEX_MAGIC = 0x58495A4Bu;  // "KZIX", little endian
const uint32_t INDEX_VERSION = 1;
const size_t INDEX_HEAD = 32;              // leading stream bytes kept to recognise another stream of the same length
const size_t INDEX_FIXED = 96;             // blob bytes before the record arrays

struct StreamIndex {
    uint64_t t48 = 0;
    uint32_t etype = 0, block_size = 0, checksum_bits = 0;
    uint32_t header_bits = 0;        // 0: a headerless stream
    int64_t input_size = 0;          // the header's hint (or the headerless setting's output size); never trusted
    uint64_t stream_bytes = 0;
    int64_t size = -1;               // decoded bytes; -1 until a read has decoded the last block
    uint8_t head[INDEX_HEAD] = {0};  // the stream's first min(32, stream_bytes) bytes, zero padded
    std::vector<uint64_t> start, bits;  // per record: first bit and bit length of its payload (behind the 5 + lw bit prefix)
    uint64_t nblocks() const { return start.size(); }
};

// XXH64, seed 0, of n bytes: the blob's trailing hash.
inline uint64_t index_xxh64(const uint8_t* p, size_t n) { return xxh64_bytes(p, n, 0); }

inline void index_put(uint8_t* p, uint64_t v, int nbytes) {
    for (int i = 0; i < nbytes; i++) p[i] = (uint8_t)(v >> (8 * i));
}
inline uint64_t index_get(const uint8_t* p, int nbytes) {
    uint64_t v = 0;
    for (int i = nbytes - 1; i >= 0; i--) v = (v << 8) | p[i];
    return v;
}

inline size_t index_blob_bytes(uint64_t nblocks) { return INDEX_FIXED + 16 * (size_t)nblocks + 8; }

// The blob of include/kanzi_b200.h ("Blob layout"): dst must hold index_blob_bytes(nblocks) bytes.
inline void index_save(const StreamIndex& x, uint8_t* dst) {
    const size_t nb = (size_t)x.nblocks();
    index_put(dst + 0, INDEX_MAGIC, 4);
    index_put(dst + 4, INDEX_VERSION, 4);
    index_put(dst + 8, x.t48, 8);
    index_put(dst + 16, x.etype, 4);
    index_put(dst + 20, x.block_size, 4);
    index_put(dst + 24, x.checksum_bits, 4);
    index_put(dst + 28, x.header_bits, 4);
    index_put(dst + 32, (uint64_t)x.input_size, 8);
    index_put(dst + 40, x.stream_bytes, 8);
    index_put(dst + 48, nb, 8);
    index_put(dst + 56, (uint64_t)x.size, 8);
    memcpy(dst + 64, x.head, INDEX_HEAD);
    for (size_t b = 0; b < nb; b++) index_put(dst + INDEX_FIXED + 8 * b, x.start[b], 8);
    for (size_t b = 0; b < nb; b++) index_put(dst + INDEX_FIXED + 8 * (nb + b), x.bits[b], 8);
    index_put(dst + INDEX_FIXED + 16 * nb, index_xxh64(dst, INDEX_FIXED + 16 * nb), 8);
}

// Whether the fields describe a stream the readers could have indexed: what parse_stream_header and kz_set_headerless_reader accept,
// records in order with a prefix of 8 .. 39 bits before each, an end marker of at least 8 bits behind the last, all inside
// stream_bytes, and a size that fits the block count.
inline bool index_consistent(const StreamIndex& x) {
    if (x.t48 >> 48 || x.etype > 31) return false;
    if (x.block_size < 1024 || x.block_size > (1u << 30)) return false;
    if (x.checksum_bits != 0 && x.checksum_bits != 32 && x.checksum_bits != 64) return false;
    if (x.header_bits != 0 && x.header_bits != 160 && x.header_bits != 176 && x.header_bits != 192 && x.header_bits != 208) return false;
    if (x.input_size < 0 || x.input_size >= ((int64_t)1 << 48)) return false;
    if (x.stream_bytes >= (1ull << 60) || x.start.size() != x.bits.size()) return false;
    const uint64_t end = 8 * x.stream_bytes, nb = x.nblocks();
    if (nb > (1ull << 62) / x.block_size) return false;  // decoded offsets stay inside 63 bits
    uint64_t pos = x.header_bits;  // first bit behind the previous record
    for (uint64_t b = 0; b < nb; b++) {
        if (x.start[b] < pos + 8 || x.start[b] > pos + 39) return false;
        if (x.bits[b] == 0 || x.bits[b] > (1ull << 34) || x.start[b] > end || x.bits[b] > end - x.start[b]) return false;
        pos = x.start[b] + x.bits[b];
    }
    if (pos > end || end - pos < 8) return false;
    if (nb == 0) return x.size == 0;
    if (x.size == -1) return true;
    return x.size > (int64_t)((nb - 1) * x.block_size) && x.size <= (int64_t)(nb * x.block_size);
}

// Parses a blob from outside the program. false: too short, a wrong magic, version, length or hash, or fields that are not consistent.
inline bool index_load(const uint8_t* blob, size_t n, StreamIndex& x) {
    if (!blob || n < INDEX_FIXED + 8) return false;
    if (index_get(blob, 4) != INDEX_MAGIC || index_get(blob + 4, 4) != INDEX_VERSION) return false;
    const uint64_t nb = index_get(blob + 48, 8);
    if (nb > (n - INDEX_FIXED - 8) / 16 || n != INDEX_FIXED + 16 * nb + 8) return false;
    if (index_get(blob + n - 8, 8) != index_xxh64(blob, n - 8)) return false;
    x.t48 = index_get(blob + 8, 8);
    x.etype = (uint32_t)index_get(blob + 16, 4);
    x.block_size = (uint32_t)index_get(blob + 20, 4);
    x.checksum_bits = (uint32_t)index_get(blob + 24, 4);
    x.header_bits = (uint32_t)index_get(blob + 28, 4);
    x.input_size = (int64_t)index_get(blob + 32, 8);
    x.stream_bytes = index_get(blob + 40, 8);
    x.size = (int64_t)index_get(blob + 56, 8);
    memcpy(x.head, blob + 64, INDEX_HEAD);
    x.start.resize((size_t)nb);
    x.bits.resize((size_t)nb);
    for (size_t b = 0; b < nb; b++) x.start[b] = index_get(blob + INDEX_FIXED + 8 * b, 8);
    for (size_t b = 0; b < nb; b++) x.bits[b] = index_get(blob + INDEX_FIXED + 8 * (nb + b), 8);
    return index_consistent(x);
}

// ---- the plan of one batched read -----------------------------------------------------------------------------------------------
// A read serves requests on one stream or on many (kz_read_ranges_streams). Each stream has a decode group: streams of one group share the
// fields a block decode depends on (transform48, entropy, block_size, checksum_bits), so their blocks may share a pass; blocks of different
// groups never do. The plan orders the touched (stream, block) pairs by group, then stream, then block.
struct ReadStream {
    uint64_t nblocks;
    uint32_t block_size;
    int64_t size;    // decoded bytes, -1: not known (taken as nblocks x block_size)
    uint32_t group;  // equal groups have equal block sizes
};

// One piece of a request inside one block: bytes [in_block, in_block + len) of pair `block` go to byte `at` of the request.
// The plan takes every block for block_size bytes long; the reader clips the slices of the last block to its decoded length.
struct ReadSlice {
    uint32_t req, block, in_block, len;
    uint64_t at;
};

struct ReadPlan {
    std::vector<uint32_t> stream;    // per touched pair: its stream ...
    std::vector<uint64_t> blocks;    // ... and its block; the distinct pairs the requests touch, in plan order
    std::vector<uint32_t> first;     // pass p decodes pairs first[p] .. first[p + 1] - 1
    std::vector<ReadSlice> slices;   // ordered by pair, so a pass's slices are contiguous ...
    std::vector<uint64_t> slice_of;  // ... slices[slice_of[k] .. slice_of[k + 1]) read pair k
    std::vector<uint64_t> want;      // per request: its length clipped to the data
    uint32_t npasses() const { return first.empty() ? 0 : (uint32_t)first.size() - 1; }
};

// Device bytes one block of a read pass takes: the two stage buffers of a decode (decompress_block_cost) and its slot in the arena
// the slices are copied from.
inline uint64_t read_block_cost(uint32_t block_size) { return decompress_block_cost(block_size) + decompress_slot(block_size); }

// The passes over pairs order[0 ..] (plan order, e.g. the pairs a cache lacks): runs of one group, each cut by plan_decompress_passes.
// Returns first: pass p holds order[first[p] .. first[p + 1]).
inline std::vector<uint32_t> plan_read_passes(const std::vector<ReadStream>& S, const std::vector<uint32_t>& stream_of, const std::vector<uint32_t>& order,
                                              uint64_t budget = STREAM_PASS_BUDGET) {
    std::vector<uint32_t> first;
    const uint32_t n = (uint32_t)order.size();
    for (uint32_t a = 0, e; a < n; a = e) {
        const ReadStream& g = S[stream_of[order[a]]];
        for (e = a + 1; e < n && S[stream_of[order[e]]].group == g.group;) e++;
        const PassPlan pp = plan_decompress_passes(e - a, decompress_slot(g.block_size), read_block_cost(g.block_size), budget);
        for (uint32_t p = 0; p < pp.npasses(); p++) first.push_back(a + pp.first[p]);
    }
    first.push_back(n);
    return first;
}

// Requests [off[i], off[i] + len[i]) on stream req_stream[i] (null: every request on stream 0). A request is clipped to its stream's
// data (pread); clipped to nothing it touches no block.
inline ReadPlan plan_reads_streams(const std::vector<ReadStream>& S, uint32_t nreq, const uint32_t* req_stream, const uint64_t* off, const uint64_t* len,
                                   uint64_t budget = STREAM_PASS_BUDGET) {
    ReadPlan P;
    struct Pair {
        uint32_t group, stream;
        uint64_t block;
        bool operator<(const Pair& o) const { return group != o.group ? group < o.group : stream != o.stream ? stream < o.stream : block < o.block; }
        bool operator==(const Pair& o) const { return group == o.group && stream == o.stream && block == o.block; }
    };
    auto stream_of = [&](uint32_t i) { return req_stream ? req_stream[i] : 0u; };
    std::vector<Pair> pairs;
    P.want.resize(nreq);
    for (uint32_t i = 0; i < nreq; i++) {
        const ReadStream& s = S[stream_of(i)];
        const uint64_t total = s.size >= 0 ? (uint64_t)s.size : s.nblocks * s.block_size;
        P.want[i] = off[i] < total ? std::min(len[i], total - off[i]) : 0;
        if (P.want[i]) {
            const uint64_t lo = off[i] / s.block_size, hi = (off[i] + P.want[i] - 1) / s.block_size;
            for (uint64_t b = lo; b <= hi; b++) pairs.push_back(Pair{s.group, stream_of(i), b});
        }
    }
    std::sort(pairs.begin(), pairs.end());
    pairs.erase(std::unique(pairs.begin(), pairs.end()), pairs.end());
    P.stream.resize(pairs.size());
    P.blocks.resize(pairs.size());
    for (size_t k = 0; k < pairs.size(); k++) P.stream[k] = pairs[k].stream, P.blocks[k] = pairs[k].block;
    // slices counted per pair, then placed: a counting sort by pair that keeps the requests' order inside a pair
    P.slice_of.assign(pairs.size() + 1, 0);
    auto each_slice = [&](auto&& f) {
        for (uint32_t i = 0; i < nreq; i++) {
            uint64_t pos = off[i], left = P.want[i];
            if (!left) continue;
            const uint32_t st = stream_of(i), bs = S[st].block_size;
            size_t k = std::lower_bound(pairs.begin(), pairs.end(), Pair{S[st].group, st, pos / bs}) - pairs.begin();
            for (; left; k++) {
                const uint32_t in_block = (uint32_t)(pos % bs);
                const uint32_t n = (uint32_t)std::min<uint64_t>(left, bs - in_block);
                f(ReadSlice{i, (uint32_t)k, in_block, n, pos - off[i]});
                pos += n;
                left -= n;
            }
        }
    };
    each_slice([&](const ReadSlice& s) { P.slice_of[s.block + 1]++; });
    for (size_t k = 0; k < pairs.size(); k++) P.slice_of[k + 1] += P.slice_of[k];
    P.slices.resize((size_t)P.slice_of.back());
    std::vector<uint64_t> fill(P.slice_of.begin(), P.slice_of.end() - 1);
    each_slice([&](const ReadSlice& s) { P.slices[(size_t)fill[s.block]++] = s; });
    std::vector<uint32_t> order(pairs.size());
    for (uint32_t k = 0; k < (uint32_t)order.size(); k++) order[k] = k;
    P.first = plan_read_passes(S, P.stream, order, budget);
    return P;
}

// The one-stream plan: requests on a stream of nblocks blocks of block_size bytes whose decoded size is `size` (-1: not known).
inline ReadPlan plan_reads(uint64_t nblocks, uint32_t block_size, int64_t size, uint32_t nreq, const uint64_t* off, const uint64_t* len,
                           uint64_t budget = STREAM_PASS_BUDGET) {
    return plan_reads_streams({ReadStream{nblocks, block_size, size, 0}}, nreq, nullptr, off, len, budget);
}

}  // namespace kz
