// CPU harness of the pass planner of the many-stream entry points, of the block cutting and per-block decisions of the encodes, and of
// the decode slot and error-order rules (kanzi-go_b200/csrc/kz_stream_plan.h), for tests/test_stream_plan_host.py.
#include <cstdint>
#include <string>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_stream_plan.h"

extern "C" {
// the per-chunk scratch of the costliest codec (ANS1: 4 MiB chunks, ~630 KB of tables and histograms + 2 bytes of payload per byte)
static const kz::EntropyScratch ENTROPY{4u << 20, 632000, 2};

// Plans the compression passes of n blocks with the library's cost function; out_pass / out_slot get each block's pass and slot,
// out_stride (n entries) each pass's stride. Returns the number of passes; *scratch = the plan's scratch bytes.
uint32_t plan_compress(const uint32_t* len, uint32_t n, uint64_t budget, uint32_t* out_pass, uint32_t* out_slot, uint64_t* out_stride,
                       uint64_t* scratch) {
    const kz::PassPlan P =
        kz::plan_compress_passes(std::vector<uint32_t>(len, len + n), [](uint64_t s) { return kz::compress_block_cost(s, ENTROPY); }, budget);
    for (uint32_t b = 0; b < n; b++) {
        out_pass[b] = P.pass[b];
        out_slot[b] = P.slot[b];
    }
    for (uint32_t p = 0; p < P.npasses(); p++) out_stride[p] = P.stride[p];
    *scratch = P.scratch;
    return P.npasses();
}
uint64_t compress_cost(uint64_t stride) { return kz::compress_block_cost(stride, ENTROPY); }

uint32_t plan_decompress(uint32_t n, uint32_t block_size, uint64_t budget, uint32_t* out_pass, uint32_t* out_slot, uint64_t* scratch) {
    const kz::PassPlan P = kz::plan_decompress_passes(n, kz::decompress_slot(block_size), kz::decompress_block_cost(block_size), budget);
    for (uint32_t b = 0; b < n; b++) {
        out_pass[b] = P.pass[b];
        out_slot[b] = P.slot[b];
    }
    *scratch = P.scratch;
    return P.npasses();
}
uint64_t decompress_cost(uint32_t block_size) { return kz::decompress_block_cost(block_size); }

// Cuts ns streams into blocks of block_size; out_off / out_len get the blocks (room for all of them), out_first ns + 1 entries. Returns the
// number of blocks.
uint32_t cut_blocks(const uint64_t* src_off, const uint64_t* src_len, uint32_t ns, uint32_t block_size, uint64_t* out_off, uint32_t* out_len,
                    uint32_t* out_first) {
    const kz::BlockList L = kz::cut_blocks(src_off, src_len, ns, block_size);
    for (uint32_t b = 0; b < L.size(); b++) out_off[b] = L.off[b], out_len[b] = L.len[b];
    for (uint32_t s = 0; s <= ns; s++) out_first[s] = L.first[s];
    return L.size();
}

int32_t magic_data_type(const uint8_t* head, uint32_t n) { return kz::magic_data_type(head, n); }

// The store rule over nb blocks (heads: 4 bytes each); counts[4] = magic blocks, magic bytes, entropy blocks, entropy bytes.
void stored_blocks(const uint8_t* heads, const uint8_t* flags, const uint32_t* len, uint32_t nb, uint8_t* store, uint64_t* counts) {
    std::vector<uint8_t> st;
    const kz::StoreCounts c = kz::stored_blocks(heads, flags, len, nb, st);
    for (uint32_t b = 0; b < nb; b++) store[b] = st[b];
    counts[0] = c.magic_blocks, counts[1] = c.magic_bytes, counts[2] = c.entropy_blocks, counts[3] = c.entropy_bytes;
}
uint64_t decode_stride(uint32_t block_size, uint32_t max_pre) { return kz::decode_stride(block_size, max_pre); }

// Notes n block failures (stage[i], code[i]) in the given order on one stream's DecodeFailure. runs_out[i] = whether stage[i] could
// still win before note i. Returns the code that decides the stream (0: none); *out_stage = its stage (STAGE_DONE: none).
int32_t note_failures(const int32_t* stage, const int32_t* code, uint32_t n, uint8_t* runs_out, int32_t* out_stage) {
    kz::DecodeFailure f;
    for (uint32_t i = 0; i < n; i++) {
        runs_out[i] = f.runs(stage[i]);
        f.note(stage[i], code[i], "failure " + std::to_string(i));
    }
    *out_stage = f.stage;
    return f.failed() ? f.code : 0;
}
}
