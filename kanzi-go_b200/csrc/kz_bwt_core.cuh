// BWT forward doubling rounds, host/device shared core (kz_bwt.cu holds the kernels, tests/host/bwt_core_host.cpp runs the same code on the
// CPU against std::stable_sort).
//
// A later doubling round orders the members of every unresolved group by their second key (rank of the suffix h further on, 0 past the end
// of the block). A group of at most BWT_SMALL_GROUP members is ordered inside one CTA without a global sort: every member counts the members
// of its group with a smaller key and the members with an equal key, in shared memory. That gives
//     r  = lt + (equal keys at a smaller index)   the member's new place in the group (a stable sort by key),
//     lt                                          the offset of its new group (equal keys stay in one group) = its new rank - group head,
//     eq                                          the size of its new group (eq > 1: still unresolved).
// The work is size^2 compares per group, which is why only small groups take this route.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define KZB_HD __host__ __device__ __forceinline__
#else
#define KZB_HD inline
#endif

namespace kz {
namespace bwtc {

// groups with at most this many members are sorted on chip; the larger ones go through the global radix sort
constexpr uint32_t BWT_SMALL_GROUP = 256;

struct GroupRank {
    uint32_t lt, eq, r;
};

// place of member x (0 <= x < size) of the group key[0 .. size) in the group sorted stably by key
KZB_HD GroupRank bwt_group_rank(const uint32_t* key, uint32_t size, uint32_t x) {
    const uint32_t k = key[x];
    uint32_t lt = 0, eq = 0, eq_before = 0;
    for (uint32_t j = 0; j < size; j++) {
        const uint32_t kj = key[j];
        lt += kj < k;
        eq += kj == k;
        eq_before += (kj == k) & (j < x);
    }
    return GroupRank{lt, eq, lt + eq_before};
}

// bits of a field that holds every value 0 .. v
KZB_HD uint32_t bwt_bits_for(uint64_t v) {
    uint32_t b = 0;
    while (b < 64 && (v >> b) != 0) b++;
    return b;
}

}  // namespace bwtc
}  // namespace kz
