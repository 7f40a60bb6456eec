// CPU harness of the small-group sort of the BWT forward rounds: runs kanzi-go_b200/csrc/kz_bwt_core.cuh (the code bwtn_small_kernel of
// kz_bwt.cu runs for every member of a group) on the host, so that tests/test_bwt_core_host.py can compare it with std::stable_sort.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_bwt_core.cuh"

using namespace kz::bwtc;

extern "C" {
// group key[0 .. size): order[r] = member placed at r, lt[x] / eq[x] / r[x] of every member. Returns 0.
int bwt_group_sort(const uint32_t* key, uint32_t size, uint32_t* order, uint32_t* lt, uint32_t* eq) {
    for (uint32_t x = 0; x < size; x++) {
        const GroupRank g = bwt_group_rank(key, size, x);
        order[g.r] = x;
        lt[x] = g.lt;
        eq[x] = g.eq;
    }
    return 0;
}
// the same against std::stable_sort: returns the number of members whose place, group offset or group size differs
uint32_t bwt_group_check(const uint32_t* key, uint32_t size) {
    std::vector<uint32_t> want(size), order(size), lt(size), eq(size);
    for (uint32_t x = 0; x < size; x++) want[x] = x;
    std::stable_sort(want.begin(), want.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
    bwt_group_sort(key, size, order.data(), lt.data(), eq.data());
    uint32_t bad = 0;
    for (uint32_t r = 0; r < size; r++) {
        const uint32_t x = want[r];
        uint32_t first = r, last = r;  // run of equal keys around place r in the stable order
        while (first > 0 && key[want[first - 1]] == key[x]) first--;
        while (last + 1 < size && key[want[last + 1]] == key[x]) last++;
        bad += order[r] != x || lt[x] != first || eq[x] != last - first + 1;
    }
    return bad;
}
uint32_t bwt_bits(uint64_t v) { return bwt_bits_for(v); }
uint32_t bwt_small_group() { return BWT_SMALL_GROUP; }
}
