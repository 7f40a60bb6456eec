// RANK / MTFT forward, host/device shared core (kz_sbrt.cu holds the kernels, tests/host/sbrt_core_host.cpp runs the same code on the CPU
// against the oracle's SBRT forward).
//
// The list is ordered by (q descending, t descending), t = last position of the symbol. Symbols never seen are behind every other one, in
// symbol order (kz_sbrt.cu). In a block of at most 2^24 bytes q and t are below 2^24, so a symbol's state packs into one 32-bit key:
//     key = (q << 8) + min(t - q + 2, 256)   for a symbol seen before (t >= q, so the low byte is 2 .. 255, or 0 when clipped),
//     key = 1                                for a symbol never seen (its t is stored as 0, which is also p[c] before the first occurrence).
// Keys are ordered like (q, t) for two symbols with the same q, unless both are clipped. So for a symbol c whose low byte is 2 .. 255,
//     rank(c) = #{ d : key(d) > key(c) }
// exactly, with one 32-bit compare per symbol. Only a key whose low byte is 0 or 1 ("ties possible") can equal another symbol's key. Such a c also
// counts the symbols with an equal key that are above it (sbrt_tie). The coded symbol's new key needs no tie-break: its t is the current
// position, larger than every other t.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define KZS_HD __host__ __device__ __forceinline__
#else
#define KZS_HD inline
#endif

namespace kz {
namespace sbrtc {

// longest block whose keys fit 32 bits (q, t < 2^24)
constexpr uint32_t SBRT_KEY_MAX_LEN = 1u << 24;

struct SbrtEntry {
    uint32_t key;
    uint32_t t;
};

// key of a symbol seen before, with q and last position t (q <= t < 2^24)
KZS_HD uint32_t sbrt_key(uint32_t q, uint32_t t) {
    const uint32_t sub = t - q + 2u;
    return (q << 8) + (sub < 256u ? sub : 256u);
}

// state of a symbol at the start of a segment from its last two positions before the segment (-1 = none). mode: 1 = MTFT, 2 = RANK
KZS_HD SbrtEntry sbrt_start(int mode, int32_t l1, int32_t l2) {
    if (l1 < 0) return SbrtEntry{1u, 0u};
    const uint32_t q = mode == 1 ? (uint32_t)l1 : ((uint32_t)l1 + (uint32_t)(l2 >= 0 ? l2 : 0)) >> 1;
    return SbrtEntry{sbrt_key(q, (uint32_t)l1), (uint32_t)l1};
}

// new state of the symbol coded at pos whose stored t was tc (SBRT.go:150-153: q = (i + p[c]) >> 1, and p[c] = tc)
template <int MODE>
KZS_HD SbrtEntry sbrt_coded(uint32_t pos, uint32_t tc) {
    const uint32_t q = MODE == 1 ? pos : (pos + tc) >> 1;
    return SbrtEntry{sbrt_key(q, pos), pos};
}

KZS_HD bool sbrt_ties_possible(uint32_t kc) { return (kc & 0xFEu) == 0u; }

// 1 if symbol d is above symbol c through a tie of keys: a later t, or both never seen and d < c. Only needed when sbrt_ties_possible(kc)
KZS_HD uint32_t sbrt_tie(uint32_t kd, uint32_t td, uint32_t d, uint32_t kc, uint32_t tc, uint32_t c) {
    return (kd == kc && (td > tc || (td == tc && d < c))) ? 1u : 0u;
}

// carry over one segment (sbrt_carry_kernel): (l1, l2) = last two positions before the segment, (a, b) = last two inside it (-1 = none)
KZS_HD void sbrt_carry(int32_t& l1, int32_t& l2, int32_t a, int32_t b) {
    if (a >= 0) {
        l2 = b >= 0 ? b : l1;
        l1 = a;
    }
}

}  // namespace sbrtc
}  // namespace kz
