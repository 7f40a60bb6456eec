// CPU harness of write_block_prefix (kanzi-go_b200/csrc/kz_common.cuh), the block record prefix both stream assemblies write,
// for tests/test_record_prefix_host.py.
#include <cstdint>
#include <cstring>

#include "../../kanzi-go_b200/csrc/kz_common.cuh"

extern "C" {
// out: 8 bytes; returns the prefix's bit count
uint32_t record_prefix(uint64_t written, uint8_t* out) {
    memset(out, 0, 8);
    return kz::write_block_prefix(out, written);
}
}
