// CPU harness of the block range selection (block_range_records / block_range_slice, kanzi-go_b200/csrc/kz_common.cuh), for
// tests/test_block_range_host.py.
#include <cstdint>

#include "../../kanzi-go_b200/csrc/kz_common.cuh"

extern "C" {
void records(int64_t from, int64_t to, uint64_t* lo, uint64_t* hi) { kz::block_range_records(from, to, lo, hi); }

void slice(int64_t from, int64_t to, uint64_t first, uint32_t count, uint32_t* lo, uint32_t* hi) {
    kz::block_range_slice(from, to, first, count, lo, hi);
}
}
