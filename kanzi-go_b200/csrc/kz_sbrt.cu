// Sort-by-rank transforms (kanzi RANK and MTFT) on sm_90a.
//
// Reference: transform/SBRT.go:127-172 (Forward), :177-226 (Inverse); modes :30-38, :93-111:
//   MTFT  qc = i                 (mask1 = -1, mask2 = 0,  shift 0)
//   RANK  qc = (i + p[c]) >> 1   (mask1 = -1, mask2 = -1, shift 1)        p[c] = previous position of c (0 before any)
// The reference keeps a list of the 256 symbols; coding symbol c at position i outputs c's index r in the list, sets
// q[c] = qc and moves c up past every symbol d with q[d] <= qc.
//
// Forward, restated for a GPU. qc never decreases for a given symbol (i grows, p[c] grows), so the list is always
// sorted by (q descending, time of the last update descending) and symbols never updated keep their initial order
// (by symbol value) behind every updated symbol of equal q. Hence
//     r(i) = #{ d != c : key(d) > key(c) },  key(d) = (q[d], t[d]),  t[d] = last position of d, or -1-d if none so far,
// which depends only on, per symbol, its last TWO positions before i. That makes the block cuttable: SBRT_SEG-byte
// segments are processed concurrently, each starting from the per-symbol (last, second last) positions before it:
//   1. sbrt_last2_kernel   per segment: last two positions of every symbol inside the segment (shared-memory atomics);
//   2. sbrt_carry_kernel   per block: running (last, second last) over the segments, one thread per symbol;
//   3. sbrt_rank_kernel    per segment, one warp: the keys of the 256 symbols in a shared-memory table (32-bit keys,
//                          kz_sbrt_core.cuh); per byte every lane counts the keys larger than key(c) among 8 of them, one REDUX
//                          gives r. Blocks above 16 MiB take sbrt_rank_wide_kernel (64-bit keys in registers).
// Inverse: the list itself is the decoder state (r -> c needs the list, which needs all earlier symbols), so a block is
// one serial chain: one CTA per block walks it with the list in registers (blocks run concurrently).
#include <algorithm>
#include <mutex>
#include <vector>

#include "kz_sbrt.cuh"
#include "kz_sbrt_core.cuh"

namespace kz {

static const int SBRT_SEG = 4096;

// ---- 1. last two positions of every symbol inside each segment
// grid: (segments of the block, blocks). table[(seg_base + s) * 512 + 2*sym + {0,1}] = (last, second last) block-relative, -1 = none
__global__ void __launch_bounds__(256) sbrt_last2_kernel(const uint8_t* __restrict__ data, const SbrtBlock* __restrict__ blocks,
                                                         int32_t* __restrict__ table) {
    __shared__ int s_l1[256], s_l2[256];
    const SbrtBlock blk = blocks[blockIdx.y];
    const uint32_t nseg = (blk.len + SBRT_SEG - 1) / SBRT_SEG;
    if (blockIdx.x >= nseg || !blk.active) return;
    const uint32_t s0 = blockIdx.x * SBRT_SEG;
    const uint32_t s1 = min(s0 + (uint32_t)SBRT_SEG, blk.len);
    const uint8_t* src = data + blk.src_off;
    s_l1[threadIdx.x] = -1;
    s_l2[threadIdx.x] = -1;
    __syncthreads();
    for (uint32_t i = s0 + threadIdx.x; i < s1; i += 256) atomicMax(&s_l1[src[i]], (int)i);
    __syncthreads();
    for (uint32_t i = s0 + threadIdx.x; i < s1; i += 256) {
        const uint8_t c = src[i];
        if ((int)i != s_l1[c]) atomicMax(&s_l2[c], (int)i);
    }
    __syncthreads();
    int32_t* t = table + ((size_t)blk.seg_base + blockIdx.x) * 512;
    t[2 * threadIdx.x] = s_l1[threadIdx.x];
    t[2 * threadIdx.x + 1] = s_l2[threadIdx.x];
}

// ---- 2. exclusive running (last, second last) over the segments of a block; in place. grid: blocks, 256 threads (symbols)
__global__ void __launch_bounds__(256) sbrt_carry_kernel(const SbrtBlock* __restrict__ blocks, int32_t* __restrict__ table) {
    const SbrtBlock blk = blocks[blockIdx.x];
    if (!blk.active) return;
    const uint32_t nseg = (blk.len + SBRT_SEG - 1) / SBRT_SEG;
    int32_t l1 = -1, l2 = -1;
    int32_t* t = table + (size_t)blk.seg_base * 512 + 2 * threadIdx.x;
    for (uint32_t s = 0; s < nseg; s++, t += 512) {
        const int32_t a = t[0], b = t[1];
        t[0] = l1;
        t[1] = l2;
        sbrtc::sbrt_carry(l1, l2, a, b);
    }
}

// acc + inc for every key of k above kc. Stated in PTX so that each key costs one compare and one predicated add (the C++ sum compiles to a
// compare, an add and a predicated move per key).
KZ_D uint32_t add_if_above(uint32_t acc, uint32_t kd, uint32_t kc, uint32_t inc) {
    asm("{\n\t.reg .pred p;\n\tsetp.gt.u32 p, %1, %2;\n\t@p add.u32 %0, %0, %3;\n\t}" : "+r"(acc) : "r"(kd), "r"(kc), "r"(inc));
    return acc;
}
KZ_D uint32_t count_above(uint32_t acc, uint4 k, uint32_t kc, uint32_t inc) {
    return add_if_above(add_if_above(add_if_above(add_if_above(acc, k.x, kc, inc), k.y, kc, inc), k.z, kc, inc), k.w, kc, inc);
}
// the tie terms of the 4 symbols d0 .. d0 + 3 held in k / t
KZ_D uint32_t count_ties(uint4 k, uint4 t, uint32_t d0, uint32_t kc, uint32_t tc, uint32_t c) {
    using namespace sbrtc;
    return sbrt_tie(k.x, t.x, d0, kc, tc, c) + sbrt_tie(k.y, t.y, d0 + 1, kc, tc, c) + sbrt_tie(k.z, t.z, d0 + 2, kc, tc, c) +
           sbrt_tie(k.w, t.w, d0 + 3, kc, tc, c);
}

// ---- 3. ranks of one segment by one warp, blocks of at most SBRT_KEY_MAX_LEN bytes. MODE: 1 = MTFT, 2 = RANK
// The 32-bit keys and last positions of the 256 symbols (kz_sbrt_core.cuh) sit in a per-warp table in shared memory. Per byte every lane
// reads key(c) and t(c) with one broadcast load each, and counts the larger keys among its 8 with two 16-byte loads. The tie terms are added
// only for a key that can tie (clipped, or a symbol never seen). The counts of the 4 bytes of a word share one register, one byte each, so one
// REDUX per word gives 4 ranks. Every lane then writes the same new entry: the same value to the same word, so each lane reads it back in
// program order and no warp barrier is needed between bytes.
template <int MODE>
__global__ void __launch_bounds__(128) sbrt_rank_kernel(const uint8_t* __restrict__ data, const SbrtBlock* __restrict__ blocks,
                                                        const uint32_t* __restrict__ seg_block, uint32_t nsegs_total,
                                                        const int32_t* __restrict__ table, uint8_t* __restrict__ out) {
    using namespace sbrtc;
    struct Table {
        uint32_t key[256];
        uint32_t t[256];
    };
    __shared__ __align__(16) uint8_t s_in[4][SBRT_SEG];
    __shared__ __align__(16) Table s_tab[4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t g = blockIdx.x * 4 + warp;  // global segment id
    if (g >= nsegs_total) return;
    const SbrtBlock blk = blocks[seg_block[g]];
    if (!blk.active) return;
    const uint32_t s0 = (g - blk.seg_base) * SBRT_SEG;
    const uint32_t cnt = min((uint32_t)SBRT_SEG, blk.len - s0);
    const uint8_t* src = data + blk.src_off + s0;
    uint8_t* dst = out + blk.dst_off + s0;
    // stage the segment (block offsets are 16-byte aligned, segments are multiples of 16); zeros up to the next multiple of 128, whose ranks
    // are computed and never stored
    {
        const uint32_t n16 = cnt >> 4, end = (cnt + 127) & ~127u;
        const uint4* s4 = reinterpret_cast<const uint4*>(src);
        uint4* d4 = reinterpret_cast<uint4*>(s_in[warp]);
        for (uint32_t i = lane; i < n16; i += 32) d4[i] = __ldg(&s4[i]);
        for (uint32_t i = (n16 << 4) + lane; i < end; i += 32) s_in[warp][i] = i < cnt ? src[i] : 0;
    }
    uint32_t* keys = s_tab[warp].key;
    uint32_t* ts = s_tab[warp].t;
    const int32_t* t0 = table + (size_t)g * 512;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int sym = lane + 32 * k;
        const SbrtEntry e = sbrt_start(MODE, t0[2 * sym], t0[2 * sym + 1]);
        keys[sym] = e.key;
        ts[sym] = e.t;
    }
    __syncwarp();
    // lane l counts symbols 4 l .. 4 l + 3 and 128 + 4 l .. 128 + 4 l + 3 (conflict-free 16-byte loads)
    const uint4* kv = reinterpret_cast<const uint4*>(keys);
    const uint4* tv = reinterpret_cast<const uint4*>(ts);
    const uint32_t* in4 = reinterpret_cast<const uint32_t*>(s_in[warp]);
    uint32_t pos = s0;
    for (uint32_t i0 = 0; i0 < cnt; i0 += 128) {  // 128 positions per round: lane l keeps the ranks of positions i0 + 4 l .. + 3
        uint32_t pack = 0;
#pragma unroll 2
        for (uint32_t w = 0; w < 32; w++) {
            const uint32_t word = in4[(i0 >> 2) + w];
            uint32_t larger = 0;  // this lane's count for byte m of the word in byte m
#pragma unroll
            for (int m = 0; m < 4; m++, pos++) {
                const uint32_t c = __byte_perm(word, 0u, 0x4440u + m), inc = 1u << (8 * m);
                const uint32_t kc = keys[c], tc = ts[c];
                const uint4 a = kv[lane], b = kv[32 + lane];
                larger = count_above(count_above(larger, a, kc, inc), b, kc, inc);
                if (sbrt_ties_possible(kc)) {  // the same in every lane
                    const uint4 ta = tv[lane], tb = tv[32 + lane];
                    larger += (count_ties(a, ta, 4 * lane, kc, tc, c) + count_ties(b, tb, 128 + 4 * lane, kc, tc, c)) << (8 * m);
                }
                const SbrtEntry e = sbrt_coded<MODE>(pos, tc);
                keys[c] = e.key;
                ts[c] = e.t;
            }
            const uint32_t ranks = __reduce_add_sync(0xFFFFFFFFu, larger);  // a rank is at most 255: no carry between the bytes
            pack = w == (uint32_t)lane ? ranks : pack;
        }
        const uint32_t base = i0 + 4 * lane;
        if (base + 4 <= cnt) {
            *reinterpret_cast<uint32_t*>(dst + base) = pack;
        } else {
            for (uint32_t q = 0; q < 4 && base + q < cnt; q++) dst[base + q] = (uint8_t)(pack >> (8 * q));
        }
    }
}

// ---- 3'. the same for blocks longer than SBRT_KEY_MAX_LEN (kanzi allows up to 1 GiB): 64-bit keys in registers. mode: 1 = MTFT, 2 = RANK
// key = q << 32 | (t + 2^31): unsigned 64-bit order = (q, t) order; t = -1-d for a symbol never seen
KZ_D uint64_t sbrt_key_wide(int32_t q, int32_t t) { return ((uint64_t)(uint32_t)q << 32) | (uint32_t)(t ^ 0x80000000); }

__global__ void __launch_bounds__(128) sbrt_rank_wide_kernel(const uint8_t* __restrict__ data, const SbrtBlock* __restrict__ blocks, int mode,
                                                             const uint32_t* __restrict__ seg_block, uint32_t nsegs_total,
                                                             const int32_t* __restrict__ table, uint8_t* __restrict__ out) {
    __shared__ uint8_t s_in[4][SBRT_SEG];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t g = blockIdx.x * 4 + warp;  // global segment id
    if (g >= nsegs_total) return;
    const uint32_t b = seg_block[g];
    const SbrtBlock blk = blocks[b];
    if (!blk.active) return;
    const uint32_t s = g - blk.seg_base;
    const uint32_t s0 = s * SBRT_SEG;
    const uint32_t cnt = min((uint32_t)SBRT_SEG, blk.len - s0);
    const uint8_t* src = data + blk.src_off + s0;
    uint8_t* dst = out + blk.dst_off + s0;
    // stage the segment (block offsets are 16-byte aligned, segments are multiples of 16)
    {
        const uint32_t n16 = cnt >> 4;
        const uint4* s4 = reinterpret_cast<const uint4*>(src);
        uint4* d4 = reinterpret_cast<uint4*>(s_in[warp]);
        for (uint32_t i = lane; i < n16; i += 32) d4[i] = __ldg(&s4[i]);
        for (uint32_t i = (n16 << 4) + lane; i < cnt; i += 32) s_in[warp][i] = src[i];
    }
    // keys of my 8 symbols (symbol = lane + 32 k) and their last positions
    const int32_t* t0 = table + (size_t)g * 512;
    uint64_t key[8];
    int32_t last[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int sym = lane + 32 * k;
        const int32_t l1 = t0[2 * sym], l2 = t0[2 * sym + 1];
        int32_t q = 0, t = -1 - sym;
        if (l1 >= 0) {
            t = l1;
            q = mode == 1 ? l1 : (l1 + (l2 >= 0 ? l2 : 0)) >> 1;
        }
        key[k] = sbrt_key_wide(q, t);
        last[k] = l1 >= 0 ? l1 : 0;  // p[c] (0 before the first occurrence)
    }
    __syncwarp();
    uint32_t pack = 0;  // ranks of 4 consecutive positions handled by this lane
    for (uint32_t i0 = 0; i0 < cnt; i0 += 128) {  // 128 positions per outer round: lane l keeps positions i0 + 4 l .. + 3
#pragma unroll 4
        for (uint32_t j = 0; j < 128; j++) {
            const uint32_t i = i0 + j;
            if (i >= cnt) break;
            const uint32_t c = s_in[warp][i];
            const int owner = (int)(c & 31), slot = (int)(c >> 5);
            // the owner picks key(c) and p[c]
            uint64_t kc = key[0];
            int32_t pc = last[0];
#pragma unroll
            for (int k = 1; k < 8; k++) {
                if (slot == k) {
                    kc = key[k];
                    pc = last[k];
                }
            }
            kc = __shfl_sync(0xFFFFFFFFu, kc, owner);
            pc = __shfl_sync(0xFFFFFFFFu, pc, owner);
            uint32_t larger = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) larger += key[k] > kc ? 1u : 0u;
            const uint32_t r = __reduce_add_sync(0xFFFFFFFFu, larger);
            if ((j >> 2) == (uint32_t)lane) pack |= r << (8 * (j & 3));
            // update (SBRT.go:150-153)
            const int32_t pos = (int32_t)(s0 + i);
            const int32_t qc = mode == 1 ? pos : (pos + pc) >> 1;
            if (lane == owner) {
                const uint64_t nk = sbrt_key_wide(qc, pos);
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    if (slot == k) {
                        key[k] = nk;
                        last[k] = pos;
                    }
                }
            }
        }
        // store the 128 ranks (4 per lane)
        const uint32_t base = i0 + 4 * lane;
        if (base + 4 <= cnt) {
            *reinterpret_cast<uint32_t*>(dst + base) = pack;
        } else {
            for (uint32_t q = 0; q < 4 && base + q < cnt; q++) dst[base + q] = (uint8_t)(pack >> (8 * q));
        }
        pack = 0;
    }
}

// ---- inverse for blocks > 16 MiB, warp-resident: the 256-entry list lives in the registers of one warp, lane l holds ranks 8 l .. 8 l + 7
// as (q, p << 8 | symbol). The list is always sorted by q (descending; SBRT.go:214-220 only ever moves the accessed symbol up, and its
// new q is never below its old one), so the move-up is a LOCAL decision per list position j <= r:
//     q[j] >  qc                 -> stays
//     q[j] <= qc, q[j-1] >  qc   -> receives the accessed symbol (this is the new rank)
//     q[j] <= qc, q[j-1] <= qc   -> receives the entry of rank j - 1
// i.e. one predicated register shift per lane plus one shuffle for the lane boundary (issued before qc is known): no reduction, no loop
// over ranks, a fixed short dependent chain per byte whatever the rank (after TEXT+BWT half of the ranks are >= 4 and their mean is 50).
// Ranks < 8 never leave lane 0 (no shuffle on the chain); a run of L zero ranks is one step (entry 0 keeps its place: p = i + L - 1,
// q = i + L - 2). 32 input ranks per round, one per lane, handed out by a shuffle issued one step ahead; the decoded symbols of a round
// go through 32 bytes of shared memory and leave as one coalesced store.
template <typename X_t>
__global__ void __launch_bounds__(32) sbrt_inverse_warp_kernel(const uint8_t* __restrict__ data, const SbrtBlock* __restrict__ blocks, int nblocks, int mode,
                                                                uint8_t* __restrict__ out) {
    __shared__ uint8_t s_out[32];
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const SbrtBlock blk = blocks[b];
    if (!blk.active) return;
    const uint8_t* src = data + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const uint32_t n = blk.len;
    const bool rank_mode = mode == 2;
    uint32_t Q[8];
    X_t X[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        Q[k] = 0;
        X[k] = (X_t)(8 * lane + k);
    }
    const uint32_t base = 8u * (uint32_t)lane;
    uint32_t nxt = lane < (int)n ? src[lane] : 0u;
    for (uint32_t i0 = 0; i0 < n; i0 += 32) {
        const uint32_t mine = nxt;
        nxt = i0 + 32 + lane < n ? src[i0 + 32 + lane] : 0u;  // next round's ranks in flight
        const uint32_t cnt = min(32u, n - i0);
        const uint32_t valid = cnt == 32 ? 0xFFFFFFFFu : ((1u << cnt) - 1u);
        const uint32_t zmask = __ballot_sync(0xFFFFFFFFu, mine == 0) & valid;
        uint32_t runmask = 0;  // bit j set: position j repeats the symbol of position j - 1 (inside a zero run)
        uint32_t j = 0;
        uint32_t r = __shfl_sync(0xFFFFFFFFu, mine, 0);
        while (j < cnt) {
            const uint32_t i = i0 + j;
            if (r == 0) {
                const uint32_t rest = ~(zmask >> j);  // bit 0 is clear (position j is a zero)
                const uint32_t L = rest ? (uint32_t)__ffs((int)rest) - 1u : 32u - j;
                const uint32_t jn = j + L;
                const uint32_t rn = __shfl_sync(0xFFFFFFFFu, mine, (int)(jn & 31u));
                if (lane == 0) {
                    const uint32_t sym = (uint32_t)X[0] & 0xFFu;
                    const uint32_t pl = i + L - 1;
                    s_out[j] = (uint8_t)sym;
                    Q[0] = rank_mode ? (L >= 2 ? pl - 1 : (uint32_t)(((uint64_t)i + (uint64_t)(X[0] >> 8)) >> 1)) : pl;
                    X[0] = ((X_t)pl << 8) | sym;
                }
                if (L >= 2) runmask |= (uint32_t)(((1ull << (L - 1)) - 1ull) << (j + 1));
                j = jn;
                r = rn;
                continue;
            }
            const uint32_t rn = __shfl_sync(0xFFFFFFFFu, mine, (int)((j + 1) & 31u));
            // the entry of rank r: select inside the owner lane (a tree over the three low bits of r), then one shuffle unless r < 8
            X_t x;
            {
                const X_t a0 = (r & 1) ? X[1] : X[0], a1 = (r & 1) ? X[3] : X[2], a2 = (r & 1) ? X[5] : X[4], a3 = (r & 1) ? X[7] : X[6];
                const X_t b0 = (r & 2) ? a1 : a0, b1 = (r & 2) ? a3 : a2;
                x = (r & 4) ? b1 : b0;
            }
            if (r < 8) {
                if (lane == 0) {
                    const uint32_t sym = (uint32_t)x & 0xFFu;
                    const uint32_t qc = rank_mode ? (uint32_t)(((uint64_t)i + (uint64_t)(x >> 8)) >> 1) : i;
                    const X_t fresh = ((X_t)i << 8) | sym;
                    s_out[j] = (uint8_t)sym;
                    bool g[8];
#pragma unroll
                    for (int k = 0; k < 8; k++) g[k] = Q[k] > qc;
#pragma unroll
                    for (int k = 7; k >= 1; k--) {
                        if ((uint32_t)k <= r && !g[k]) {
                            Q[k] = g[k - 1] ? qc : Q[k - 1];
                            X[k] = g[k - 1] ? fresh : X[k - 1];
                        }
                    }
                    if (!g[0]) {
                        Q[0] = qc;
                        X[0] = fresh;
                    }
                }
            } else {
                const uint32_t up_q = __shfl_up_sync(0xFFFFFFFFu, Q[7], 1);
                const X_t up_x = __shfl_up_sync(0xFFFFFFFFu, X[7], 1);
                x = __shfl_sync(0xFFFFFFFFu, x, (int)(r >> 3));
                const uint32_t sym = (uint32_t)x & 0xFFu;
                const uint32_t qc = rank_mode ? (uint32_t)(((uint64_t)i + (uint64_t)(x >> 8)) >> 1) : i;
                const X_t fresh = ((X_t)i << 8) | sym;
                if (lane == 0) s_out[j] = (uint8_t)sym;
                bool g[8];
#pragma unroll
                for (int k = 0; k < 8; k++) g[k] = Q[k] > qc;
                const bool g_up = lane == 0 ? true : up_q > qc;
#pragma unroll
                for (int k = 7; k >= 1; k--) {
                    if (base + (uint32_t)k <= r && !g[k]) {
                        Q[k] = g[k - 1] ? qc : Q[k - 1];
                        X[k] = g[k - 1] ? fresh : X[k - 1];
                    }
                }
                if (base <= r && !g[0]) {
                    Q[0] = g_up ? qc : up_q;
                    X[0] = g_up ? fresh : up_x;
                }
            }
            j++;
            r = rn;
        }
        __syncwarp();
        if ((uint32_t)lane < cnt) {
            const uint32_t own = ~runmask & (lane == 31 ? 0xFFFFFFFFu : ((2u << lane) - 1u));  // positions <= lane that hold a symbol of their own
            dst[i0 + lane] = s_out[31 - __clz((int)own)];
        }
        __syncwarp();
    }
}

// ---- inverse for blocks <= 16 MiB: the list in the registers of 4 warps, mirrored in shared memory ---------------------------------------------
// With the list only in registers, every instruction of a step sits on the dependent chain: look-up of the entry of rank r -> qc -> move-up
// -> next step's look-up. Here the registers keep the list for the move-up, and a copy in shared memory serves the look-ups: after step j - 1
// has stored its entries, the candidates for the rank r2 of step j + 1 are loaded from the state BEFORE step j — entry r2 and entry r2 - 1 —
// and step j decides with two compares which one (or its own fresh entry) stands at rank r2 afterwards (the move-up rule applied to that one
// position). The chain per rank is qc -> 2 compares -> 2 selects -> next qc; the move-up, the stores and the loads for the step after next
// overlap it. On one warp this is bound by the ALU pipe of its scheduler (~50 integer / predicate instructions per rank), and with every
// look-up served by the mirror nothing but the lane boundary ties the lanes together, so the 256 entries are spread over 4 warps (2 entries
// per lane) that sit on different schedulers: every warp takes the same decision about the next entry from the same shared-memory
// candidates, moves its own part of the list, stores it, and one CTA barrier per rank publishes the stores.
// With one warp per scheduler nothing hides a step's latency, so a step spends as few instructions as it can (DESIGN.md §4.3):
//   - an entry is (q, x = p << 8 | symbol) in one 8-byte word of the mirror: one load fetches a candidate or the entry above a warp's first
//     one, and one 16-byte store publishes a thread's two entries;
//   - both copies have a sentinel slot above position 0 (a q larger than any qc), so that the candidate r2 - 1 for r2 = 0 and the entry
//     above thread 0 are plain loads, with no test for position 0;
//   - warp 0 stages the ranks of a round in shared memory a round ahead and every thread holds them as 8 words: a step takes its rank r3
//     out of a register with one byte extract, and its r / r2 are the r2 / r3 of the two steps before.
// But what lies between one barrier and the next counts as well: the entry above a thread's first one is a shuffle inside a warp and a
// mirror load on lane 0 only. Loading it from the mirror on every lane, and packing a round's symbols into words for one store, each took
// instructions out of the step but made the chain slower (§4.3).
template <bool RANK_MODE>
__global__ void __launch_bounds__(128) sbrt_inverse_multi_kernel(const uint8_t* __restrict__ data, const SbrtBlock* __restrict__ blocks, int nblocks,
                                                                 uint8_t* __restrict__ out) {
    constexpr int S = 2;  // entries per lane
    // two copies, written alternately: a warp that runs ahead stores step j + 1 while another still reads the state after step j - 1 / j.
    // Position k of a copy is slot k + 2: slot 1 is the sentinel above position 0, slot 0 keeps the threads' 16-byte stores aligned.
    __shared__ __align__(16) uint2 s_e[2][258];
    __shared__ __align__(16) uint32_t s_rk[2][8];  // the 32 ranks of round k in s_rk[k & 1], 0 past the end of the block
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (b >= nblocks) return;
    const SbrtBlock blk = blocks[b];
    if (!blk.active) return;
    const uint8_t* src = data + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const uint32_t n = blk.len;
    if (n == 0) return;
    uint8_t* const rk8 = reinterpret_cast<uint8_t*>(s_rk);
    uint32_t Q[S], X[S];
    const uint32_t base = (uint32_t)(S * tid);
#pragma unroll
    for (int k = 0; k < S; k++) {
        Q[k] = 0;
        X[k] = base + k;
        s_e[0][2 + base + k] = s_e[1][2 + base + k] = make_uint2(0u, base + k);
    }
    if (tid < 2) s_e[tid][1] = make_uint2(0xFFFFFFFFu, 0u);
    if (warp == 0) {
        rk8[lane] = (uint32_t)lane < n ? src[lane] : 0u;
        rk8[32 + lane] = 32u + lane < n ? src[32 + lane] : 0u;
    }
    __syncthreads();
    uint2 ca, cb;  // candidates: entries r2 and r2 - 1 of the state before the current step
    auto load_candidates = [&](uint32_t r2, int par) {  // from the copy step `par` wrote
        ca = s_e[par][2 + r2];
        cb = s_e[par][1 + r2];
    };
    // par = parity of the step: it reads the copy of parity par ^ 1 (the state before it) and writes the copy of parity par.
    // x: the entry at rank r (the same in every thread), replaced by the entry at rank r2 after the step. Returns the entry at rank r.
    auto step = [&](uint32_t r, uint32_t r2, uint32_t i, int par, uint32_t& x) -> uint32_t {
        // the entry above this thread's first one (state before the step): a shuffle inside the warp, the mirror on lane 0
        uint2 up = make_uint2(__shfl_up_sync(0xFFFFFFFFu, Q[S - 1], 1), __shfl_up_sync(0xFFFFFFFFu, X[S - 1], 1));
        if (lane == 0) up = s_e[par ^ 1][1 + base];
        const uint32_t e = x;
        const uint32_t qc = RANK_MODE ? (i + (e >> 8)) >> 1 : i;  // i, p < 2^24
        const uint32_t fresh = __byte_perm(e, i, 0x6540u);  // i << 8 | symbol
        {  // the entry at rank r2 after this step (every warp computes the same)
            const bool mv = r2 <= r && !(ca.x > qc);
            x = mv ? (cb.x > qc ? fresh : cb.y) : ca.y;
        }
        bool gk = Q[S - 1] > qc;
#pragma unroll
        for (int k = S - 1; k >= 1; k--) {
            const bool gk1 = Q[k - 1] > qc;
            const bool mv = r >= base + k && !gk;
            const uint32_t xin = gk1 ? fresh : X[k - 1];
            Q[k] = mv ? min(Q[k - 1], qc) : Q[k];
            X[k] = mv ? xin : X[k];
            gk = gk1;
        }
        {
            const bool mv = r >= base && !gk;
            Q[0] = mv ? min(up.x, qc) : Q[0];  // up.x > qc: the fresh entry lands here
            X[0] = mv ? (up.x > qc ? fresh : up.y) : X[0];
        }
        reinterpret_cast<uint4*>(&s_e[par][2])[tid] = make_uint4(Q[0], X[0], Q[1], X[1]);
        __syncthreads();
        return e;
    };
    uint32_t r = rk8[0], r2 = rk8[1];
    uint32_t x = s_e[1][2 + r].y;
    load_candidates(r2, 1);
    uint32_t i0 = 0;
    for (; i0 + 32 <= n; i0 += 32) {
        const int rb = (int)(i0 >> 5) & 1;
        const uint4 m0 = reinterpret_cast<const uint4*>(s_rk[rb])[0], m1 = reinterpret_cast<const uint4*>(s_rk[rb])[1];
        const uint32_t M[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
        const uint32_t M8 = s_rk[rb ^ 1][0];  // the first ranks of the next round
        // the ranks of round k + 2, stored into s_rk[k & 1] at step 30: as late as the barrier of step 31 still publishes them to round k + 1,
        // so that the global load has a round's steps to arrive in
        const uint32_t nn = warp == 0 && i0 + 64 + lane < n ? src[i0 + 64 + lane] : 0u;
        uint32_t ob = 0;
#pragma unroll
        for (int j = 0; j < 32; j++) {
            const uint32_t r3 = __byte_perm(j < 30 ? M[(j + 2) >> 2] : M8, 0u, 0x4440u | ((j + 2) & 3));
            const uint32_t e = step(r, r2, i0 + (uint32_t)j, j & 1, x);  // i0 is a multiple of 32
            load_candidates(r3, j & 1);
            ob = lane == j ? e : ob;
            if (j == 30 && warp == 0) rk8[32 * rb + lane] = (uint8_t)nn;
            r = r2;
            r2 = r3;
        }
        if (warp == 0) dst[i0 + lane] = (uint8_t)ob;
    }
    if (i0 < n) {
        const uint8_t* rt = rk8 + 32 * ((i0 >> 5) & 1);
        uint32_t ob = 0;
        for (uint32_t j = 0; i0 + j < n; j++) {
            const uint32_t r3 = j < 30 ? rt[j + 2] : 0u;
            const uint32_t e = step(r, r2, i0 + j, (int)(j & 1), x);
            load_candidates(r3, (int)(j & 1));
            ob = (uint32_t)lane == j ? e : ob;
            r = r2;
            r2 = r3;
        }
        if (warp == 0 && i0 + lane < n) dst[i0 + lane] = (uint8_t)ob;
    }
}

// A chain is serial and latency-bound: a CTA that shares its SM with another chain's CTA runs at a fraction of its speed for the whole launch, and
// the block scheduler does pack CTAs (six per SM were seen: 1.6 s instead of 0.26 s) when kernels of other streams occupy the GPU at launch time.
// Dynamic shared memory that nobody touches caps the chains per SM at ceil(nblocks / SMs): the chains spread over the GPU whatever runs beside them.
// The chains of an SM take all of its shared memory, so that no CTA of another kernel shares their schedulers either: with room left for one
// (half an SM per chain), a chain beside the -l 3 round trip of another context took 256 ms instead of the 224 ms it takes alone.
// The kernel's dynamic shared memory cap is one setting of the process for each device, and contexts launch from several host threads at
// once: it is raised once per device to the most any launch asks for, so that no thread lowers it between another thread's size and launch.
template <bool RANK_MODE>
static size_t spread_chains(int nblocks) {
    const auto kernel = sbrt_inverse_multi_kernel<RANK_MODE>;
    int dev = 0, sms = 0, sm_bytes = 0, block_max = 0, reserved = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0 ||
        cudaDeviceGetAttribute(&sm_bytes, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&block_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev) != cudaSuccess)
        return 0;
    const int per = (nblocks + sms - 1) / sms;
    if (per > 5) return 0;  // small blocks in large numbers: several chains per SM overlap their latencies, no cap
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, kernel) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    static std::mutex mu;
    static std::vector<int8_t> capped;  // per device: 0 not set yet, 1 set to block_max - static, -1 setting it failed
    {
        std::lock_guard<std::mutex> lock(mu);
        if ((int)capped.size() <= dev) capped.resize(dev + 1, 0);
        if (capped[dev] == 0) {
            capped[dev] = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, block_max - (int)fa.sharedSizeBytes) == cudaSuccess ? 1 : -1;
            if (capped[dev] < 0) cudaGetLastError();
        }
        if (capped[dev] < 0) return 0;
    }
    const size_t room = (size_t)sm_bytes / (size_t)per, fixed = (size_t)reserved + fa.sharedSizeBytes;
    if (room <= fixed) return 0;
    return std::min(room - fixed, (size_t)block_max - fa.sharedSizeBytes);
}

void sbrt_rank_launch(const uint8_t* data, const SbrtBlock* d_blocks, int mode, const uint32_t* seg_block, uint32_t nsegs, const int32_t* table,
                      uint8_t* out, uint32_t max_len, cudaStream_t stream) {
    const unsigned grid = (nsegs + 3) / 4;
    if (max_len > sbrtc::SBRT_KEY_MAX_LEN) sbrt_rank_wide_kernel<<<grid, 128, 0, stream>>>(data, d_blocks, mode, seg_block, nsegs, table, out);
    else if (mode == 2) sbrt_rank_kernel<2><<<grid, 128, 0, stream>>>(data, d_blocks, seg_block, nsegs, table, out);
    else sbrt_rank_kernel<1><<<grid, 128, 0, stream>>>(data, d_blocks, seg_block, nsegs, table, out);
}

void sbrt_inverse_launch_len(const uint8_t* data, const SbrtBlock* d_blocks, int nblocks, int mode, uint8_t* out, uint32_t max_len, cudaStream_t stream) {
    if (max_len > (1u << 24)) sbrt_inverse_warp_kernel<uint64_t><<<nblocks, 32, 0, stream>>>(data, d_blocks, nblocks, mode, out);
    else if (mode == 2) sbrt_inverse_multi_kernel<true><<<nblocks, 128, spread_chains<true>(nblocks), stream>>>(data, d_blocks, nblocks, out);
    else sbrt_inverse_multi_kernel<false><<<nblocks, 128, spread_chains<false>(nblocks), stream>>>(data, d_blocks, nblocks, out);
}

}  // namespace kz
