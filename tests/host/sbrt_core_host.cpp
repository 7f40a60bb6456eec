// CPU harness of the RANK / MTFT forward: runs kanzi-go_b200/csrc/kz_sbrt_core.cuh the way the kernels of kz_sbrt.cu do. A block is cut into
// segments of SBRT_SEG_BYTES, and each segment starts from the carried (last, second last) positions of every symbol. A rank is the count of
// larger keys, plus the tie terms when the key can tie. tests/test_sbrt_core_host.py compares the result with the oracle's SBRT forward.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_sbrt_core.cuh"

using namespace kz::sbrtc;

static const uint32_t SEG = 4096;  // SBRT_SEG_BYTES (kz_sbrt.cuh)

extern "C" {
// dst[0 .. n) = forward of src[0 .. n) (mode 1 = MTFT, 2 = RANK); *tie_bytes = bytes whose key could tie. Returns 0, or -1 for a block longer
// than SBRT_KEY_MAX_LEN.
int sbrt_core_forward(int mode, const uint8_t* src, uint32_t n, uint8_t* dst, uint64_t* tie_bytes) {
    *tie_bytes = 0;
    if (n > SBRT_KEY_MAX_LEN) return -1;
    const uint32_t nseg = (n + SEG - 1) / SEG;
    // sbrt_last2_kernel: the last two positions of every symbol inside each segment
    std::vector<int32_t> tab((size_t)nseg * 512, -1);
    for (uint32_t i = 0; i < n; i++) {
        int32_t* t = &tab[(size_t)(i / SEG) * 512 + 2 * src[i]];
        t[1] = t[0];
        t[0] = (int32_t)i;
    }
    // sbrt_carry_kernel: the last two positions before each segment
    for (int d = 0; d < 256; d++) {
        int32_t l1 = -1, l2 = -1;
        for (uint32_t g = 0; g < nseg; g++) {
            int32_t* t = &tab[(size_t)g * 512 + 2 * d];
            const int32_t a = t[0], b = t[1];
            t[0] = l1;
            t[1] = l2;
            sbrt_carry(l1, l2, a, b);
        }
    }
    // sbrt_rank_kernel, one segment after the other (each one only reads its own start table)
    for (uint32_t g = 0; g < nseg; g++) {
        uint32_t key[256], t[256];
        for (int d = 0; d < 256; d++) {
            const SbrtEntry e = sbrt_start(mode, tab[(size_t)g * 512 + 2 * d], tab[(size_t)g * 512 + 2 * d + 1]);
            key[d] = e.key;
            t[d] = e.t;
        }
        const uint32_t s1 = std::min(g * SEG + SEG, n);
        for (uint32_t pos = g * SEG; pos < s1; pos++) {
            const uint32_t c = src[pos], kc = key[c], tc = t[c];
            uint32_t r = 0;
            for (uint32_t d = 0; d < 256; d++) r += key[d] > kc ? 1u : 0u;
            if (sbrt_ties_possible(kc)) {
                ++*tie_bytes;
                for (uint32_t d = 0; d < 256; d++) r += sbrt_tie(key[d], t[d], d, kc, tc, c);
            }
            dst[pos] = (uint8_t)r;
            const SbrtEntry e = mode == 1 ? sbrt_coded<1>(pos, tc) : sbrt_coded<2>(pos, tc);
            key[c] = e.key;
            t[c] = e.t;
        }
    }
    return 0;
}
}
