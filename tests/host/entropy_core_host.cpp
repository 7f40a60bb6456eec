// CPU build of the entropy core the MM transform and the skipBlocks test run on the device (kanzi-go_b200/csrc/kz_entropy_core.cuh), for
// tests/test_entropy_core_host.py.
#include "../../kanzi-go_b200/csrc/kz_entropy_core.cuh"

extern "C" {

void entropy_core_log2_4096(uint32_t* out) {
    const uint32_t* t = kz::host_log2_4096();
    for (int i = 0; i <= 256; i++) out[i] = t[i];
}

uint32_t entropy_core_log2_scaled_1024(uint32_t x) { return kz::log2_scaled_1024(x, kz::host_log2_4096()); }

int entropy_core_entropy_1024(uint32_t block_len, const uint32_t* histo) { return kz::entropy_1024(block_len, histo, kz::host_log2_4096()); }

int entropy_core_incompressible(uint32_t block_len, const uint32_t* histo) {
    return kz::entropy_1024(block_len, histo, kz::host_log2_4096()) >= kz::INCOMPRESSIBLE_THRESHOLD;
}
}
