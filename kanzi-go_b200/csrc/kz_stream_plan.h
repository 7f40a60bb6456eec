// Pass planner of the many-stream entry points (kz_compress_streams / kz_decompress_streams, kz_api.cu). Pure host code: no CUDA
// types, so that tests/host/stream_plan_host.cpp compiles it with g++ and checks its bounds on the CPU.
//
// A pass is a set of blocks that run through the transform and entropy stages together. Every block of a pass gets a slot of the
// pass's stride in the device scratch buffers, so the scratch of a pass is (number of blocks) x cost(stride). The planner keeps that
// product under a fixed budget, and keeps the stride close to every member's length, so that a batch of many small files and one
// large one does not give every small file a slot as long as the large one.
#pragma once
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

namespace kz {

// Device scratch bytes one pass may take (the block costs below). A block whose own cost is larger runs alone in a pass of its own.
const uint64_t STREAM_PASS_BUDGET = 1ull << 30;

struct PassPlan {
    std::vector<uint32_t> first;       // pass p holds the blocks order[first[p] .. first[p + 1])
    std::vector<uint32_t> order;       // block indexes, pass after pass
    std::vector<uint64_t> stride;      // slot stride of each pass (a multiple of 16)
    std::vector<uint32_t> pass, slot;  // per block: its pass, and its slot inside that pass
    uint64_t scratch = 0;              // largest (blocks of a pass) x cost(stride) over the passes
    uint32_t npasses() const { return (uint32_t)stride.size(); }
};

inline uint64_t round16(uint64_t n) { return (n + 15) & ~15ull; }

// Scratch the entropy stage (encode_batch) takes per chunk of a codec: its chunk size, and fixed + per_byte x (chunk bytes) bytes of
// tables, headers, payload and histograms per chunk. NONE has no chunks (chunk = 0).
struct EntropyScratch {
    uint64_t chunk = 0, fixed = 0, per_byte = 0;
};

// Device bytes one block of a compression pass of stride s takes: its input slot, the two stage buffers of forward_stage (at most
// s + s/8 + 33 bytes per transform + 9,472 bytes each), its entropy output slot (kz_max_block_output(s)) and the entropy stage's
// per-chunk scratch. The transforms' own workspaces are not counted: they are sized per sub-batch of a fixed number of blocks
// (run_desc_stage in kz_api.cu) or per block (BWT, BWTS, LZ), not per pass.
inline uint64_t compress_block_cost(uint64_t s, const EntropyScratch& e) {
    const uint64_t stage = round16(s + s / 8 + 33 * 8 + 8192 + 1024 + 256);
    const uint64_t enc = round16(s + (s >> 3) + 1024 + 64 * (s / 16384 + 1) + 106496 * (s / (4u << 20) + 1));
    const uint64_t chunks = e.chunk ? (s + e.chunk - 1) / e.chunk : 0;
    return s + 2 * stage + enc + chunks * (e.fixed + e.per_byte * std::min(s, e.chunk));
}

// Reader.processBlock (io/CompressedStream.go:1649-1653) sizes each task buffer blockSize + max(512, blockSize >> 4); a decode slot
// holds that plus 64 bytes of slack, and a block takes one slot in each of the two buffers the inverse stages alternate between.
inline uint64_t decompress_slot(uint32_t block_size) { return round16((uint64_t)block_size + std::max<uint64_t>(512, block_size >> 4) + 64); }
inline uint64_t decompress_block_cost(uint32_t block_size) { return 2 * decompress_slot(block_size); }

// Compression: blocks of lengths len[], longest first. A pass opens with the longest block left, whose rounded length is the pass's
// stride s; it admits shorter blocks while s <= 2 x len + 16 and while (blocks + 1) x cost(s) <= budget.
template <class Cost>
PassPlan plan_compress_passes(const std::vector<uint32_t>& len, Cost cost, uint64_t budget = STREAM_PASS_BUDGET) {
    PassPlan P;
    const uint32_t n = (uint32_t)len.size();
    P.order.resize(n);
    std::iota(P.order.begin(), P.order.end(), 0u);
    std::stable_sort(P.order.begin(), P.order.end(), [&](uint32_t a, uint32_t b) { return len[a] > len[b]; });
    P.pass.assign(n, 0);
    P.slot.assign(n, 0);
    auto rlen = [&](uint32_t b) { return round16(std::max<uint64_t>(len[b], 1)); };
    for (uint32_t i = 0; i < n;) {
        const uint32_t p = P.npasses();
        const uint64_t s = rlen(P.order[i]), c = cost(s);
        P.first.push_back(i);
        P.stride.push_back(s);
        uint32_t k = 0;
        while (i < n && s <= 2 * std::max<uint64_t>(len[P.order[i]], 1) + 16 && (k == 0 || (uint64_t)(k + 1) * c <= budget)) {
            P.pass[P.order[i]] = p;
            P.slot[P.order[i]] = k++;
            i++;
        }
        P.scratch = std::max(P.scratch, (uint64_t)k * c);
    }
    P.first.push_back(n);
    return P;
}

// Decompression: a block's decoded length is only bounded by its stream's block size, so every block of a group gets the same stride
// and cost; the budget caps the number of blocks of a pass. Blocks keep their order (stream after stream).
inline PassPlan plan_decompress_passes(uint32_t n, uint64_t stride, uint64_t cost, uint64_t budget = STREAM_PASS_BUDGET) {
    PassPlan P;
    const uint32_t per = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(budget / std::max<uint64_t>(cost, 1), 0xFFFFFFFFu));
    P.order.resize(n);
    std::iota(P.order.begin(), P.order.end(), 0u);
    P.pass.resize(n);
    P.slot.resize(n);
    for (uint32_t i = 0; i < n; i += per) {
        const uint32_t p = P.npasses(), k = std::min(per, n - i);
        P.first.push_back(i);
        P.stride.push_back(stride);
        for (uint32_t j = 0; j < k; j++) {
            P.pass[i + j] = p;
            P.slot[i + j] = j;
        }
        P.scratch = std::max(P.scratch, (uint64_t)k * cost);
    }
    P.first.push_back(n);
    return P;
}

}  // namespace kz
