// CPU harness of the pass planner of the many-stream entry points and of the decode slot and error-order rules
// (kanzi-go_b200/csrc/kz_stream_plan.h), for tests/test_stream_plan_host.py.
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
