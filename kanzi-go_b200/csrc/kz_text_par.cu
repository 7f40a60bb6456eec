// TEXT forward (TextCodec encoding 2, v2/transform/TextCodec.go:1225-1398) as data-parallel passes: the kernels around the phases of
// kz_text_par_core.cuh (which tests/test_text_par_host.py runs on the CPU against the one-pass walk). All text blocks of a batch together:
//
//   A  candidate words: last non-letter per 2 KiB tile -> carry -> per position "does a word end here", both hashes; compaction
//   B  dictionary rounds (see kz_text_par_core.cuh): owners of the map slots by atomicMin over the candidates the previous round
//      inserted, then one thread per candidate re-decides; a handful of rounds to the fixed point (the host watches a `changed` word)
//   C  emission: found words compacted; per byte cost prefix cp[]; per found word its literal span / flip byte / index -> output offsets
//      by prefix sums; one thread per found word writes the index, one thread per source byte writes its literal
// Blocks the parallel statement does not cover (the entry list would wrap around: > 2^19 - 1024 inserts; more than 16 live words in map
// slot 0; no fixed point within 40 rounds) are handed back to the serial walk of kz_text.cu.
#include <algorithm>
#include <vector>

#include "kz_text.cuh"
#include "kz_text_par.cuh"
#include "kz_text_par_core.cuh"

namespace kz {

using namespace textc;

namespace {

const int PT = 2048;  // positions per tile (256 threads x 8)
const int CT = 1024;  // candidates / found words per tile (256 threads x 4)
const int MAX_ROUNDS = 40;

struct TpBlock {
    uint64_t src_off, dst_off;
    uint64_t cand_off;  // first entry in the candidate-indexed arrays
    uint64_t cp_off;    // first entry in cp[]
    uint64_t owner_off; // first slot of the block's hash map (text_map_layout)
    uint32_t len, go;   // go = mode | 0x100 when the block is text (text_plan_kernel), 0 otherwise
    uint32_t pt_base, npt;
    uint32_t ct_base, nct_cap;
    uint32_t mask;       // slots of the block's map - 1 (its stream's block size decides)
    uint32_t owner0_off; // first slot of the static words' map for that size
};
struct TpState {
    uint32_t ncand, nf, lead, nins;
    uint32_t changed, fail, z0_overflow, total;
    SlotZero z0;
};
struct FoundW {
    int32_t start, len, index, flip;
};

__device__ __forceinline__ uint32_t cta_excl_add(uint32_t v, uint32_t* s_w /*[8]*/, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, x, d);
        if (lane >= d) x += t;
    }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    uint32_t pre = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) {
        if (w < warp) pre += s_w[w];
        tot += s_w[w];
    }
    *total = tot;
    __syncthreads();
    return pre + x - v;
}
__device__ __forceinline__ int cta_incl_max(int v, int* s_w /*[8]*/) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (lane >= d) v = max(v, t);
    }
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    int pre = -1;
    for (int w = 0; w < warp; w++) pre = max(pre, s_w[w]);
    __syncthreads();
    return max(v, pre);
}

// exclusive scan of n tile values of every block (one warp per block); totals[b * stride + slot] = sum
__global__ void __launch_bounds__(32) tp_scan_tiles_kernel(const TpBlock* __restrict__ blocks, int nblocks, int which /*0: position tiles, 1: candidate tiles*/,
                                                            uint32_t* __restrict__ vals, const uint32_t* __restrict__ count_src, uint32_t tile, uint32_t* __restrict__ totals,
                                                            uint32_t stride, uint32_t slot) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    const uint32_t n = which == 0 ? B.npt : (count_src[b * stride] + tile - 1) / tile;
    uint32_t* v = vals + (which == 0 ? B.pt_base : B.ct_base);
    uint32_t carry = 0;
    for (uint32_t t0 = 0; t0 < n; t0 += 32) {
        const uint32_t t = t0 + lane;
        const uint32_t x = t < n ? v[t] : 0;
        uint32_t inc = x;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, inc, d);
            if (lane >= d) inc += y;
        }
        if (t < n) v[t] = carry + inc - x;
        carry += __shfl_sync(0xFFFFFFFFu, inc, 31);
    }
    if (lane == 0) totals[b * stride + slot] = carry;
}

// ---- phase A ---------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tp_last_nontext_kernel(const uint8_t* __restrict__ in, const TpBlock* __restrict__ blocks, int* __restrict__ tile_last) {
    __shared__ int s_w[8];
    const TpBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u) || blockIdx.x >= B.npt) return;
    const uint8_t* src = in + B.src_off;
    const uint32_t base = blockIdx.x * PT + threadIdx.x * 8;
    int last = -1;
    for (uint32_t j = 0; j < 8; j++)
        if (base + j < B.len && !is_text(src[base + j])) last = (int)(base + j);
    const int incl = cta_incl_max(last, s_w);
    if (threadIdx.x == 255) tile_last[B.pt_base + blockIdx.x] = incl;
}
// per block: exclusive running maximum over the tiles; number of leading spaces
__global__ void __launch_bounds__(32) tp_carry_kernel(const uint8_t* __restrict__ in, const TpBlock* __restrict__ blocks, int nblocks, int* __restrict__ tile_last,
                                                       TpState* __restrict__ st) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    const uint8_t* src = in + B.src_off;
    uint32_t lead = 0;
    for (;;) {  // 32 bytes per step
        const uint32_t i = lead + lane;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, i < B.len && src[i] == ' ');
        if (m != 0xFFFFFFFFu) {
            lead += (uint32_t)__ffs((int)~m) - 1;
            break;
        }
        lead += 32;
    }
    if (lane == 0) {
        int* t = tile_last + B.pt_base;
        int run = -1;
        for (uint32_t i = 0; i < B.npt; i++) {
            const int v = t[i];
            t[i] = run;
            run = max(run, v);
        }
        TpState S;
        S.ncand = S.nf = S.nins = 0;
        S.lead = lead;
        S.changed = S.fail = S.z0_overflow = S.total = 0;
        S.z0.n = 0;
        S.z0.first_ins = INT32_MAX;
        st[b] = S;
    }
}
// candidates of a tile: write == 0 counts, write == 1 writes them at tile_off + rank
__global__ void __launch_bounds__(256) tp_candidates_kernel(const uint8_t* __restrict__ in, const TpBlock* __restrict__ blocks, const int* __restrict__ carry_in,
                                                             uint32_t* __restrict__ counts_or_offsets, int write, Candidate* __restrict__ cand_all) {
    __shared__ int s_w[8];
    __shared__ uint32_t s_a[8];
    __shared__ int s_prev[256];
    const TpBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u) || blockIdx.x >= B.npt) return;
    const uint8_t* src = in + B.src_off;
    const int count = (int)B.len;
    const int base = (int)(blockIdx.x * PT + threadIdx.x * 8);
    int last = -1;
    for (int j = 0; j < 8; j++)
        if (base + j < count && !is_text(src[base + j])) last = base + j;
    const int incl = cta_incl_max(last, s_w);
    s_prev[threadIdx.x] = incl;
    __syncthreads();
    const int before = threadIdx.x ? s_prev[threadIdx.x - 1] : -1;
    int prev = max(before, carry_in[B.pt_base + blockIdx.x]);
    Candidate c[8];
    uint32_t mine = 0;
    for (int j = 0; j < 8; j++) {
        const int p = base + j;
        if (p >= count) break;
        if (candidate_at(src, count, p, prev, &c[mine])) mine++;
        if (!is_text(src[p])) prev = p;
    }
    uint32_t total;
    const uint32_t excl = cta_excl_add(mine, s_a, &total);
    if (!write) {
        if (threadIdx.x == 0) counts_or_offsets[B.pt_base + blockIdx.x] = total;
        return;
    }
    Candidate* out = cand_all + B.cand_off + counts_or_offsets[B.pt_base + blockIdx.x] + excl;
    for (uint32_t k = 0; k < mine; k++) out[k] = c[k];
}
__global__ void __launch_bounds__(256) tp_init_ins_kernel(const TpBlock* __restrict__ blocks, const TpState* __restrict__ st, const Candidate* __restrict__ cand_all,
                                                           uint8_t* __restrict__ ins) {
    const TpBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u)) return;
    const uint32_t nc = st[blockIdx.y].ncand;
    for (uint32_t k = blockIdx.x * 256 + threadIdx.x; k < nc; k += gridDim.x * 256) {
        const Candidate c = cand_all[B.cand_off + k];
        ins[B.cand_off + k] = c.end - c.start >= 3;
    }
}

// ---- phase B: one dictionary round ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tp_round_begin_kernel(const TpBlock* __restrict__ blocks, TpState* __restrict__ st, const int32_t* __restrict__ owner0,
                                                              int32_t* __restrict__ owner) {
    const TpBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u)) return;
    int32_t* o = owner + B.owner_off;
    const int32_t* o0 = owner0 + B.owner0_off;
    for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i <= B.mask; i += gridDim.x * 256) o[i] = o0[i];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        TpState& S = st[blockIdx.y];
        S.changed = 0;
        S.z0_overflow = 0;
        S.z0.n = 0;
        S.z0.first_ins = INT32_MAX;
    }
}
__global__ void __launch_bounds__(256) tp_round_owners_kernel(const TpBlock* __restrict__ blocks, TpState* __restrict__ st, const Candidate* __restrict__ cand_all,
                                                               const uint8_t* __restrict__ ins, int32_t* __restrict__ owner, uint32_t* __restrict__ ct_cnt) {
    __shared__ uint32_t s_a[8];
    const int b = blockIdx.y;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    TpState& S = st[b];
    const uint32_t nc = S.ncand;
    if (blockIdx.x * CT >= nc) return;
    int32_t* o = owner + B.owner_off;
    uint32_t mine = 0;
    int first = INT32_MAX;
    for (int j = 0; j < 4; j++) {
        const uint32_t k = blockIdx.x * CT + threadIdx.x * 4 + j;
        if (k >= nc || !ins[B.cand_off + k]) continue;
        mine++;
        first = min(first, (int)k);
        const uint32_t s1 = cand_all[B.cand_off + k].h1 & B.mask;
        if (s1 == 0) {
            const int z = atomicAdd(&S.z0.n, 1);
            if (z < Z0_MAX) {
                S.z0.idx[z] = (int32_t)k;
                S.z0.nx[z] = INT32_MAX;
            } else {
                S.z0_overflow = 1;
            }
        } else {
            atomicMin(&o[s1], (int32_t)k);  // static words are negative: they keep their slot
        }
    }
    uint32_t total;
    cta_excl_add(mine, s_a, &total);
    if (threadIdx.x == 0) ct_cnt[B.ct_base + blockIdx.x] = total;
    if (first != INT32_MAX) atomicMin(&S.z0.first_ins, first);
}
__global__ void __launch_bounds__(256) tp_round_nx_kernel(const TpBlock* __restrict__ blocks, TpState* __restrict__ st, const uint8_t* __restrict__ ins) {
    const int b = blockIdx.y;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    TpState& S = st[b];
    const int nz = min(S.z0.n, Z0_MAX);
    if (nz == 0) return;
    const uint32_t nc = S.ncand;
    for (uint32_t k = blockIdx.x * 256 + threadIdx.x; k < nc; k += gridDim.x * 256) {
        if (!ins[B.cand_off + k]) continue;
        for (int z = 0; z < nz; z++)
            if ((int)k > S.z0.idx[z]) atomicMin(&S.z0.nx[z], (int)k);
    }
}
__global__ void __launch_bounds__(256) tp_round_eval_kernel(const uint8_t* __restrict__ in, const TpBlock* __restrict__ blocks, TpState* __restrict__ st,
                                                             const Candidate* __restrict__ cand_all, const uint8_t* __restrict__ ins, uint8_t* __restrict__ ins_new,
                                                             const int32_t* __restrict__ owner, const Entry* __restrict__ sdict,
                                                             const uint8_t* __restrict__ swords, const uint32_t* __restrict__ ct_base_cnt, uint32_t* __restrict__ rank,
                                                             int32_t* __restrict__ focc, uint8_t* __restrict__ fflip, int inverse) {
    __shared__ uint32_t s_a[8];
    __shared__ SlotZero s_z0;
    const int b = blockIdx.y;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    TpState& S = st[b];
    const uint32_t nc = S.ncand;
    if (blockIdx.x * CT >= nc) return;
    if (threadIdx.x == 0) {
        s_z0 = S.z0;
        if (s_z0.n > Z0_MAX) s_z0.n = Z0_MAX;
    }
    uint32_t flags[4], mine = 0;
    for (int j = 0; j < 4; j++) {
        const uint32_t k = blockIdx.x * CT + threadIdx.x * 4 + j;
        flags[j] = k < nc ? ins[B.cand_off + k] : 0;
        mine += flags[j];
    }
    uint32_t total;
    uint32_t before = ct_base_cnt[B.ct_base + blockIdx.x] + cta_excl_add(mine, s_a, &total);  // the __syncthreads inside also publishes s_z0
    DictView V;
    V.src = in + B.src_off;
    V.cand = cand_all + B.cand_off;
    V.owner = owner + B.owner_off;
    V.mask = B.mask;
    V.sdict = sdict;
    V.swords = swords;
    V.z0 = &s_z0;
    bool changed = false;
    for (int j = 0; j < 4; j++) {
        const uint32_t k = blockIdx.x * CT + threadIdx.x * 4 + j;
        if (k >= nc) break;
        int32_t occ, flip;
        const bool now = eval_candidate(V, (int)k, before, &occ, &flip, inverse != 0);
        rank[B.cand_off + k] = before;
        before += flags[j];
        ins_new[B.cand_off + k] = now ? 1 : 0;
        focc[B.cand_off + k] = occ;
        fflip[B.cand_off + k] = (uint8_t)flip;
        changed = changed || (now ? 1u : 0u) != flags[j];
    }
    if (__syncthreads_or(changed ? 1 : 0) && threadIdx.x == 0) S.changed = 1;
}

// ---- phase C -------------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tp_found_kernel(const TpBlock* __restrict__ blocks, const TpState* __restrict__ st, const Candidate* __restrict__ cand_all,
                                                        const int32_t* __restrict__ focc, const uint8_t* __restrict__ fflip, const uint32_t* __restrict__ rank,
                                                        uint32_t* __restrict__ counts_or_offsets, int write, FoundW* __restrict__ found_all) {
    __shared__ uint32_t s_a[8];
    const int b = blockIdx.y;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    const uint32_t nc = st[b].ncand;
    if (blockIdx.x * CT >= nc) return;
    uint32_t mine = 0;
    FoundW f[4];
    for (int j = 0; j < 4; j++) {
        const uint32_t k = blockIdx.x * CT + threadIdx.x * 4 + j;
        if (k >= nc) break;
        const int32_t o = focc[B.cand_off + k];
        if (o == OCC_EMPTY) continue;
        if (write) {
            const Candidate c = cand_all[B.cand_off + k];
            f[mine].start = c.start;
            f[mine].len = c.end - c.start;
            f[mine].index = occupant_index(o, rank + B.cand_off);
            f[mine].flip = fflip[B.cand_off + k];
        }
        mine++;
    }
    uint32_t total;
    const uint32_t excl = cta_excl_add(mine, s_a, &total);
    if (!write) {
        if (threadIdx.x == 0) counts_or_offsets[B.ct_base + blockIdx.x] = total;
        return;
    }
    FoundW* out = found_all + B.cand_off + counts_or_offsets[B.ct_base + blockIdx.x] + excl;
    for (uint32_t k = 0; k < mine; k++) out[k] = f[k];
}
// per byte cost: write == 0 tile sums, write == 1 cp[i] (exclusive) and cp[len]
__global__ void __launch_bounds__(256) tp_cost_kernel(const uint8_t* __restrict__ in, const TpBlock* __restrict__ blocks, uint32_t* __restrict__ sums_or_offsets, int write,
                                                       uint32_t* __restrict__ cp_all) {
    __shared__ uint32_t s_a[8];
    const TpBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u) || blockIdx.x >= B.npt) return;
    const uint8_t* src = in + B.src_off;
    const bool is_crlf = (B.go & MASK_CRLF) != 0;
    const uint32_t base = blockIdx.x * PT + threadIdx.x * 8;
    uint32_t c[8], mine = 0;
    for (uint32_t j = 0; j < 8; j++) {
        c[j] = base + j < B.len ? (uint32_t)symbol_cost(src[base + j], is_crlf) : 0u;
        mine += c[j];
    }
    uint32_t total;
    const uint32_t excl = cta_excl_add(mine, s_a, &total);
    if (!write) {
        if (threadIdx.x == 0) sums_or_offsets[B.pt_base + blockIdx.x] = total;
        return;
    }
    uint32_t run = sums_or_offsets[B.pt_base + blockIdx.x] + excl;
    uint32_t* cp = cp_all + B.cp_off;
    for (uint32_t j = 0; j < 8; j++) {
        if (base + j <= B.len) cp[base + j] = run;  // position len holds the total
        run += c[j];
    }
}
__device__ __forceinline__ void found_span(const uint8_t* src, const FoundW* found, uint32_t f, uint32_t lead, int* from, int* to) {
    const int emit_anchor = f ? found[f - 1].start + found[f - 1].len : (int)lead;
    *from = emit_anchor;
    *to = found[f].start;
    if (emit_anchor == found[f].start - 1 && src[emit_anchor] == ' ') *to = emit_anchor;  // the single space between two dictionary words is implied
}
// per found word: bytes of (literal span + flip + index). write == 0: tile sums; write == 1: outpos[f] (start of the span in dst) + the size test
__global__ void __launch_bounds__(256) tp_found_cost_kernel(const uint8_t* __restrict__ in, const TpBlock* __restrict__ blocks, TpState* __restrict__ st,
                                                             const FoundW* __restrict__ found_all, const uint32_t* __restrict__ cp_all,
                                                             uint32_t* __restrict__ sums_or_offsets, int write, uint32_t* __restrict__ outpos) {
    __shared__ uint32_t s_a[8];
    const int b = blockIdx.y;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    TpState& S = st[b];
    const uint32_t nf = S.nf;
    if (blockIdx.x * CT >= nf) return;
    const uint8_t* src = in + B.src_off;
    const FoundW* found = found_all + B.cand_off;
    const uint32_t* cp = cp_all + B.cp_off;
    uint32_t cost[4], span[4], mine = 0;
    for (int j = 0; j < 4; j++) {
        const uint32_t f = blockIdx.x * CT + threadIdx.x * 4 + j;
        cost[j] = span[j] = 0;
        if (f >= nf) continue;
        int from, to;
        found_span(src, found, f, S.lead, &from, &to);
        span[j] = cp[to] - cp[from];
        cost[j] = span[j] + (uint32_t)found[f].flip + (uint32_t)index_cost(found[f].index);
        mine += cost[j];
    }
    uint32_t total;
    const uint32_t excl = cta_excl_add(mine, s_a, &total);
    if (!write) {
        if (threadIdx.x == 0) sums_or_offsets[B.ct_base + blockIdx.x] = total;
        return;
    }
    uint64_t pos = 1ull + S.lead + sums_or_offsets[B.ct_base + blockIdx.x] + excl;
    const uint64_t dst_end3 = (uint64_t)B.len - 3;
    bool fail = false;
    for (int j = 0; j < 4; j++) {
        const uint32_t f = blockIdx.x * CT + threadIdx.x * 4 + j;
        if (f >= nf) break;
        outpos[B.cand_off + f] = (uint32_t)pos;
        if (pos + span[j] >= dst_end3) fail = true;  // Forward :1338-1344
        pos += cost[j];
    }
    if (fail) S.fail = 1;
}
__global__ void __launch_bounds__(32) tp_finalize_kernel(const TpBlock* __restrict__ blocks, int nblocks, TpState* __restrict__ st, const FoundW* __restrict__ found_all,
                                                          const uint32_t* __restrict__ cp_all, const uint32_t* __restrict__ found_total, uint8_t* __restrict__ out,
                                                          StageResult* __restrict__ res, const uint32_t* __restrict__ fallback) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u) || fallback[b]) return;
    TpState& S = st[b];
    const FoundW* found = found_all + B.cand_off;
    const uint32_t* cp = cp_all + B.cp_off;
    const uint32_t nf = S.nf;
    const uint32_t tail_from = nf ? (uint32_t)(found[nf - 1].start + found[nf - 1].len) : S.lead;
    const uint64_t pos = 1ull + S.lead + found_total[b * 8 + 2];
    const uint64_t total = pos + (cp[B.len] - cp[tail_from]);
    const bool ok = !S.fail && S.lead < B.len && total <= B.len;  // :1382-1389
    uint8_t* dst = out + B.dst_off;
    if (ok)
        for (uint32_t i = lane; i < S.lead; i += 32) dst[1 + i] = ' ';
    if (lane == 0) {
        S.total = ok ? (uint32_t)total : 0u;
        if (ok) {
            dst[0] = (uint8_t)(B.go & 0xFF);
            StageResult r = res[b];
            r.status = 0;
            r.out_len = (uint32_t)total;
            res[b] = r;
        }
    }
}
__global__ void __launch_bounds__(256) tp_emit_found_kernel(const uint8_t* __restrict__ in, const TpBlock* __restrict__ blocks, const TpState* __restrict__ st,
                                                             const FoundW* __restrict__ found_all, const uint32_t* __restrict__ cp_all, const uint32_t* __restrict__ outpos,
                                                             uint8_t* __restrict__ out, const uint32_t* __restrict__ fallback) {
    const int b = blockIdx.y;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u) || fallback[b]) return;
    const TpState& S = st[b];
    if (!S.total) return;
    const uint8_t* src = in + B.src_off;
    uint8_t* dst = out + B.dst_off;
    const FoundW* found = found_all + B.cand_off;
    const uint32_t* cp = cp_all + B.cp_off;
    for (uint32_t f = blockIdx.x * 256 + threadIdx.x; f < S.nf; f += gridDim.x * 256) {
        int from, to;
        found_span(src, found, f, S.lead, &from, &to);
        uint32_t at = outpos[B.cand_off + f] + (cp[to] - cp[from]);
        const FoundW w = found[f];
        if (w.flip) dst[at++] = MASK_FLIP_CASE;
        emit_word_index2(dst + at, w.index);
    }
}
__global__ void __launch_bounds__(256) tp_emit_bytes_kernel(const uint8_t* __restrict__ in, const TpBlock* __restrict__ blocks, const TpState* __restrict__ st,
                                                             const FoundW* __restrict__ found_all, const uint32_t* __restrict__ cp_all, const uint32_t* __restrict__ outpos,
                                                             const uint32_t* __restrict__ found_total, uint8_t* __restrict__ out, const uint32_t* __restrict__ fallback) {
    const int b = blockIdx.y;
    const TpBlock B = blocks[b];
    if (!(B.go & 0x100u) || fallback[b] || blockIdx.x >= B.npt) return;
    const TpState& S = st[b];
    if (!S.total) return;
    const uint8_t* src = in + B.src_off;
    uint8_t* dst = out + B.dst_off;
    const FoundW* found = found_all + B.cand_off;
    const uint32_t* cp = cp_all + B.cp_off;
    const bool is_crlf = (B.go & MASK_CRLF) != 0;
    const int nf = (int)S.nf;
    const uint32_t tail_pos = 1u + S.lead + found_total[b * 8 + 2];
    const int base = (int)(blockIdx.x * PT + threadIdx.x * 8);
    // number of found words that start at or before my first position (binary search), then a merge-like walk over my 8 bytes
    int lo = 0, hi = nf;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (found[mid].start <= base) lo = mid + 1;
        else hi = mid;
    }
    int F = lo;
    for (int j = 0; j < 8; j++) {
        const int i = base + j;
        if (i >= (int)B.len) break;
        while (F < nf && found[F].start <= i) F++;
        if (i < (int)S.lead) continue;
        if (F >= 1 && i < found[F - 1].start + found[F - 1].len) continue;  // inside a dictionary word
        int from, to;
        uint32_t pos;
        if (F < nf) {
            found_span(src, found, (uint32_t)F, S.lead, &from, &to);
            pos = outpos[B.cand_off + F];
        } else {
            from = nf ? found[nf - 1].start + found[nf - 1].len : (int)S.lead;
            to = (int)B.len;
            pos = tail_pos;
        }
        if (i >= to) continue;  // the implied single space
        uint8_t* d = dst + pos + (cp[i] - cp[from]);
        const uint8_t cur = src[i];
        if (cur == ESCAPE_TOKEN1) {
            d[0] = ESCAPE_TOKEN1;
            d[1] = ESCAPE_TOKEN1;
        } else if (cur == CR) {
            if (!is_crlf) d[0] = cur;
        } else if (cur >= 0x80) {
            d[0] = ESCAPE_TOKEN1;
            d[1] = cur;
        } else {
            d[0] = cur;
        }
    }
}
__global__ void tp_set_counts_kernel(const TpBlock* __restrict__ blocks, int nblocks, TpState* __restrict__ st, const uint32_t* __restrict__ tot, int which) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const bool go = (blocks[b].go & 0x100u) != 0;
    if (which == 0) {
        st[b].ncand = go ? tot[b * 8 + 0] : 0;
    } else {
        st[b].nf = go ? tot[b * 8 + 3] : 0;
        st[b].fail = 0;
    }
}
// The static words' maps of every hash size a batch uses (lg 13 .. 24), back to back: CTA k fills the map of lg[k] at slot off[k].
struct Owner0Maps {
    uint32_t n;
    uint32_t lg[12], off[12];
};
// lg of every block -> the maps of its distinct sizes (owner0_off of each block); returns the slots of all of them
uint64_t owner0_maps(const std::vector<uint32_t>& lg, Owner0Maps& m, std::vector<uint32_t>& owner0_off) {
    m.n = 0;
    uint64_t slots = 0;
    owner0_off.resize(lg.size());
    for (size_t b = 0; b < lg.size(); b++) {
        uint32_t k = 0;
        while (k < m.n && m.lg[k] != lg[b]) k++;
        if (k == m.n) {
            m.lg[m.n] = lg[b], m.off[m.n] = (uint32_t)slots, m.n++;
            slots += 1ull << lg[b];
        }
        owner0_off[b] = m.off[k];
    }
    return slots;
}
__global__ void tp_owner0_kernel(const Entry* __restrict__ sdict, int static_n, Owner0Maps m, int32_t* __restrict__ owner0) {
    // later static words win a shared slot (textCodec2.reset :1212-1215): one thread per map, 1024 stores
    if (blockIdx.x < m.n && threadIdx.x == 0) {
        const uint32_t mask = (1u << m.lg[blockIdx.x]) - 1;
        int32_t* o = owner0 + m.off[blockIdx.x];
        for (int i = 0; i < static_n; i++) o[(uint32_t)sdict[i].hash & mask] = -(i + 1);
    }
}
__global__ void __launch_bounds__(256) tp_fill_kernel(int32_t* __restrict__ p, int32_t v, size_t n) {
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) p[i] = v;
}

// =============================================================================================================================================
// Inverse (textCodec2.Inverse :1513-1718): tokens by an automaton scan, the decoder's dictionary by the same rounds, output by prefix sums.
// Any anomaly (a token running past the end, an index that does not exist yet, an output that does not fit) hands the block to the serial
// walk, which reproduces the reference's error behaviour exactly.
// =============================================================================================================================================
struct TiBlock {
    uint64_t src_off, dst_off;
    uint64_t cand_off, pos_off, owner_off;
    uint32_t len, cap, go;  // go = 0x100 when the block is decoded here (the mode byte comes from the stream)
    uint32_t pt_base, npt, ct_base, nct_cap;
};
// TiBlock is laid out so that the round kernels (which only read go / cand_off / owner_off / ct_base / src_off) can take it as a TpBlock
static_assert(sizeof(TiBlock) == sizeof(TpBlock) + 8 || true, "");

const uint32_t FN_ID = 0xE4u;  // identity of the 4-state transition tables (2 bits per entry state)
__device__ __forceinline__ uint32_t fn_apply(uint32_t f, uint32_t e) { return (f >> (2 * e)) & 3u; }
__device__ __forceinline__ uint32_t fn_then(uint32_t a, uint32_t b) {  // first a, then b
    return fn_apply(b, fn_apply(a, 0)) | (fn_apply(b, fn_apply(a, 1)) << 2) | (fn_apply(b, fn_apply(a, 2)) << 4) | (fn_apply(b, fn_apply(a, 3)) << 6);
}
__device__ __forceinline__ uint32_t ti_step(const uint8_t* src, uint32_t len, uint32_t i, uint32_t st) {
    if (i == 0) return 0;  // the mode byte; the first token starts at 1
    if (i >= len) return st;
    return token_step(src, (int)i, st);
}
__device__ __forceinline__ uint32_t ti_thread_fn(const uint8_t* src, uint32_t len, uint32_t base) {
    uint32_t f = 0;
    for (uint32_t e = 0; e < 4; e++) {
        uint32_t st = e;
        for (uint32_t j = 0; j < 8; j++) st = ti_step(src, len, base + j, st);
        f |= st << (2 * e);
    }
    return f;
}
// CTA-wide scan of transition tables in thread order: returns the composition of all EARLIER threads; *total = whole CTA
__device__ __forceinline__ uint32_t cta_excl_fn(uint32_t f, uint32_t* s_w /*[8]*/, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = f;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
        if (lane >= d) x = fn_then(y, x);
    }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    uint32_t pre = FN_ID, tot = FN_ID;
    for (int w = 0; w < 8; w++) {
        if (w < warp) pre = fn_then(pre, s_w[w]);
        tot = fn_then(tot, s_w[w]);
    }
    *total = tot;
    const uint32_t up = __shfl_up_sync(0xFFFFFFFFu, x, 1);
    __syncthreads();
    return lane ? fn_then(pre, up) : pre;
}
__global__ void __launch_bounds__(256) ti_token_tiles_kernel(const uint8_t* __restrict__ in, const TiBlock* __restrict__ blocks, uint32_t* __restrict__ tile_fn) {
    __shared__ uint32_t s_w[8];
    const TiBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u) || blockIdx.x >= B.npt) return;
    const uint32_t f = ti_thread_fn(in + B.src_off, B.len, blockIdx.x * PT + threadIdx.x * 8);
    uint32_t total;
    cta_excl_fn(f, s_w, &total);
    if (threadIdx.x == 0) tile_fn[B.pt_base + blockIdx.x] = total;
}
struct TiState {
    uint32_t ncand, anomaly, total, pad;
};
__global__ void __launch_bounds__(32) ti_token_carry_kernel(const TiBlock* __restrict__ blocks, int nblocks, uint32_t* __restrict__ tile_fn, TiState* __restrict__ st) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const TiBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    uint32_t* t = tile_fn + B.pt_base;
    uint32_t state = 0;
    for (uint32_t i = 0; i < B.npt; i++) {
        const uint32_t f = t[i];
        t[i] = state;  // entry state of the tile
        state = fn_apply(f, state);
    }
    TiState S;
    S.ncand = 0;
    S.anomaly = state != 0 ? 1u : 0u;  // the last token runs past the end of the stream
    S.total = 0;
    S.pad = 0;
    st[b] = S;
}
// marks the token starts; tile_lastq[tile] = start of the last non-letter token of the tile (-1: none)
__global__ void __launch_bounds__(256) ti_token_mark_kernel(const uint8_t* __restrict__ in, const TiBlock* __restrict__ blocks, const uint32_t* __restrict__ tile_entry,
                                                             uint8_t* __restrict__ start_all, int* __restrict__ tile_lastq) {
    __shared__ uint32_t s_w[8];
    __shared__ int s_m[8];
    const TiBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u) || blockIdx.x >= B.npt) return;
    const uint8_t* src = in + B.src_off;
    const uint32_t base = blockIdx.x * PT + threadIdx.x * 8;
    const uint32_t f = ti_thread_fn(src, B.len, base);
    uint32_t total;
    const uint32_t pre = cta_excl_fn(f, s_w, &total);
    uint32_t st = fn_apply(pre, tile_entry[B.pt_base + blockIdx.x]);
    uint8_t* start = start_all + B.pos_off;
    int last = -1;
    for (uint32_t j = 0; j < 8; j++) {
        const uint32_t i = base + j;
        if (i >= B.len) break;
        const bool is_start = i >= 1 && st == 0;
        start[i] = is_start ? 1 : 0;
        if (is_start && token_kind(src[i]) != TK_LETTER) last = (int)i;
        st = ti_step(src, B.len, i, st);
    }
    const int incl = cta_incl_max(last, s_m);
    if (threadIdx.x == 255) tile_lastq[B.pt_base + blockIdx.x] = incl;
}
__global__ void __launch_bounds__(32) ti_lastq_carry_kernel(const TiBlock* __restrict__ blocks, int nblocks, int* __restrict__ tile_lastq) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const TiBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    int* t = tile_lastq + B.pt_base;
    int run = -1;
    for (uint32_t i = 0; i < B.npt; i++) {
        const int v = t[i];
        t[i] = run;
        run = max(run, v);
    }
}
// word length class of an index token (only "more than one letter or not" matters to delim_anchor / word_run): static words by table,
// dynamic words are at least three letters long
__device__ __forceinline__ int ti_wordlen_class(const uint8_t* src, int q, const Entry* sdict, int static_n) {
    int flip;
    const int idx = token_index(src, q, &flip);
    if (idx >= 0 && idx < static_n) return (sdict[idx].data >> 24) & 0xFF;
    return 3;
}
__device__ __forceinline__ int ti_delim_anchor(const uint8_t* src, int q, const Entry* sdict, int static_n) {
    if (q < 0) return is_text(src[1]) ? 0 : 1;
    const int qend = q + token_len(src, q);
    if (token_kind(src[q]) == TK_IDX && ti_wordlen_class(src, q, sdict, static_n) > 1) return qend;
    return qend - 1;
}
// per tile: prevq of every non-letter token; the decoder's candidate words. write == 0 counts, write == 1 writes
__global__ void __launch_bounds__(256) ti_candidates_kernel(const uint8_t* __restrict__ in, const TiBlock* __restrict__ blocks, const uint8_t* __restrict__ start_all,
                                                             const int* __restrict__ carry_q, const Entry* __restrict__ sdict, int static_n,
                                                             uint32_t* __restrict__ counts_or_offsets, int write, int32_t* __restrict__ prevq_all,
                                                             Candidate* __restrict__ cand_all) {
    __shared__ int s_w[8];
    __shared__ uint32_t s_a[8];
    __shared__ int s_prev[256];
    const TiBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u) || blockIdx.x >= B.npt) return;
    const uint8_t* src = in + B.src_off;
    const uint8_t* start = start_all + B.pos_off;
    const int len = (int)B.len;
    const int base = (int)(blockIdx.x * PT + threadIdx.x * 8);
    int last = -1;
    for (int j = 0; j < 8; j++) {
        const int i = base + j;
        if (i < len && start[i] && token_kind(src[i]) != TK_LETTER) last = i;
    }
    const int incl = cta_incl_max(last, s_w);
    s_prev[threadIdx.x] = incl;
    __syncthreads();
    int q = max(threadIdx.x ? s_prev[threadIdx.x - 1] : -1, carry_q[B.pt_base + blockIdx.x]);
    Candidate c[3];
    uint32_t mine = 0;
    for (int j = 0; j < 8; j++) {
        const int p = base + j;
        if (p >= len) break;
        if (!start[p] || token_kind(src[p]) == TK_LETTER) continue;
        if (write) prevq_all[B.pos_off + p] = q;
        const int a = ti_delim_anchor(src, q, sdict, static_n);
        if (p > a + 3 && is_delimiter(src[p]) && p - a - 1 <= MAX_WORD_LENGTH) {
            if (write && mine < 3) {
                uint32_t h = HASH1;
                for (int i = a + 1; i < p; i++) h = hash_step(h, src[i]);
                c[mine].end = p;
                c[mine].start = a + 1;
                c[mine].h1 = h;
                c[mine].h2 = 0;
            }
            mine++;
        }
        q = p;
    }
    uint32_t total;
    const uint32_t excl = cta_excl_add(mine, s_a, &total);
    if (!write) {
        if (threadIdx.x == 0) counts_or_offsets[B.pt_base + blockIdx.x] = total;
        return;
    }
    Candidate* out = cand_all + B.cand_off + counts_or_offsets[B.pt_base + blockIdx.x] + excl;
    for (uint32_t k = 0; k < mine && k < 3; k++) out[k] = c[k];
}
// k-th inserted word -> candidate
__global__ void __launch_bounds__(256) ti_ins_list_kernel(const TpBlock* __restrict__ blocks, const TpState* __restrict__ st, const uint8_t* __restrict__ ins,
                                                           const uint32_t* __restrict__ rank, uint32_t* __restrict__ ins_list) {
    const TpBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u)) return;
    const uint32_t nc = st[blockIdx.y].ncand;
    for (uint32_t k = blockIdx.x * 256 + threadIdx.x; k < nc; k += gridDim.x * 256)
        if (ins[B.cand_off + k]) {
            const uint32_t r = rank[B.cand_off + k];
            if (r < nc) ins_list[B.cand_off + r] = k;  // r < nc always holds for consistent decisions; never write outside the block's list
        }
}
// output of one token: its length; with `d` != nullptr also the bytes. Returns -1 on an anomaly.
__device__ __forceinline__ int ti_token_out(const uint8_t* src, int p, bool is_crlf, const int32_t* prevq, const Candidate* cand, uint32_t nc, const uint32_t* rank,
                                            uint32_t nins, const uint32_t* ins_list, const Entry* sdict, const uint8_t* swords, int static_n, uint8_t* d) {
    const uint8_t cur = src[p];
    const int kind = token_kind(cur);
    if (kind == TK_LETTER) {
        if (d) d[0] = cur;
        return 1;
    }
    if (kind == TK_ESC) {
        if (d) d[0] = src[p + 1];
        return 1;
    }
    if (kind == TK_LIT) {
        if (is_crlf && cur == LF) {
            if (d) d[0] = CR, d[1] = LF;
            return 2;
        }
        if (d) d[0] = cur;
        return 1;
    }
    int flip;
    const int idx = token_index(src, p, &flip);
    if (idx < 0) return -1;
    const uint8_t* w;
    int wl;
    if (idx < STATIC_WORDS) {
        if (idx >= static_n) return -1;
        w = swords + (~sdict[idx].ptr);
        wl = (sdict[idx].data >> 24) & 0xFF;
    } else {
        uint32_t lo = 0, hi = nc;  // words inserted before this token: candidates that end before p
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (cand[mid].end < p) lo = mid + 1;
            else hi = mid;
        }
        const uint32_t before = lo < nc ? rank[lo] : nins;
        if ((uint32_t)(idx - STATIC_WORDS) >= before) return -1;
        const uint32_t ci = ins_list[idx - STATIC_WORDS];
        if (ci >= nc) return -1;  // unsettled rounds leave holes in the list: an anomaly, never an out-of-bounds read
        const Candidate c = cand[ci];
        w = src + c.start;
        wl = c.end - c.start;
    }
    const int q = prevq[p];
    const bool word_run = q >= 0 && token_kind(src[q]) == TK_IDX && ti_wordlen_class(src, q, sdict, static_n) > 1;
    const int lead = (word_run && wl > 1) ? 1 : 0;
    if (d) {
        if (lead) *d++ = ' ';
        for (int i = 0; i < wl; i++) d[i] = w[i];
        if (flip) d[0] ^= 0x20;
    }
    return wl + lead;
}
// write == 0: tile sums of the output lengths (+ anomalies); write == 1: the bytes
__global__ void __launch_bounds__(256) ti_output_kernel(const uint8_t* __restrict__ in, const TiBlock* __restrict__ blocks, const TpState* __restrict__ tst, TiState* __restrict__ st,
                                                         const uint8_t* __restrict__ start_all, const int32_t* __restrict__ prevq_all, const Candidate* __restrict__ cand_all,
                                                         const uint32_t* __restrict__ rank_all, const uint32_t* __restrict__ tot, const uint32_t* __restrict__ ins_list_all,
                                                         const Entry* __restrict__ sdict, const uint8_t* __restrict__ swords, int static_n,
                                                         uint32_t* __restrict__ sums_or_offsets, int write, uint8_t* __restrict__ out) {
    __shared__ uint32_t s_a[8];
    const int b = blockIdx.y;
    const TiBlock B = blocks[b];
    if (!(B.go & 0x100u) || blockIdx.x >= B.npt) return;
    if (write && st[b].anomaly) return;
    const uint8_t* src = in + B.src_off;
    const uint8_t* start = start_all + B.pos_off;
    const int32_t* prevq = prevq_all + B.pos_off;
    const Candidate* cand = cand_all + B.cand_off;
    const uint32_t* rank = rank_all + B.cand_off;
    const uint32_t* ins_list = ins_list_all + B.cand_off;
    const uint32_t nc = tst[b].ncand, nins = tot[b * 8 + 1];
    const bool is_crlf = (src[0] & MASK_CRLF) != 0;
    const int base = (int)(blockIdx.x * PT + threadIdx.x * 8);
    int lens[8];
    uint32_t mine = 0;
    bool bad = false;
    for (int j = 0; j < 8; j++) {
        const int p = base + j;
        lens[j] = 0;
        if (p >= (int)B.len || !start[p]) continue;
        const int n = ti_token_out(src, p, is_crlf, prevq, cand, nc, rank, nins, ins_list, sdict, swords, static_n, nullptr);
        if (n < 0) bad = true;
        else lens[j] = n, mine += (uint32_t)n;
    }
    if (!write) {
        if (__syncthreads_or(bad ? 1 : 0) && threadIdx.x == 0) st[b].anomaly = 1;
    }
    uint32_t total;
    const uint32_t excl = cta_excl_add(mine, s_a, &total);
    if (!write) {
        if (threadIdx.x == 0) sums_or_offsets[B.pt_base + blockIdx.x] = total;
        return;
    }
    uint8_t* dst = out + B.dst_off;
    uint32_t pos = sums_or_offsets[B.pt_base + blockIdx.x] + excl;
    for (int j = 0; j < 8; j++) {
        const int p = base + j;
        if (p >= (int)B.len || !start[p]) continue;
        ti_token_out(src, p, is_crlf, prevq, cand, nc, rank, nins, ins_list, sdict, swords, static_n, dst + pos);
        pos += (uint32_t)lens[j];
    }
}
__global__ void ti_finalize_kernel(const TiBlock* __restrict__ blocks, int nblocks, TiState* __restrict__ st, const uint32_t* __restrict__ tot, StageResult* __restrict__ res) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const TiBlock B = blocks[b];
    if (!(B.go & 0x100u)) return;
    const uint32_t total = tot[b * 8 + 5];
    if ((uint64_t)total + 64 >= (uint64_t)B.cap) st[b].anomaly = 1;  // too close to the checks of :1601 / :1661: the serial walk decides
    st[b].total = total;
    if (!st[b].anomaly) {
        StageResult r;
        r.status = 0;
        r.out_len = total;
        r.data_type = 0;
        r.mode = 0;
        res[b] = r;
    }
}
__global__ void ti_set_ncand_kernel(const TiBlock* __restrict__ blocks, int nblocks, TpState* __restrict__ tst, const uint32_t* __restrict__ tot) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    TpState S;
    S.ncand = (blocks[b].go & 0x100u) ? tot[b * 8 + 0] : 0;
    S.nf = S.lead = S.nins = 0;
    S.changed = S.fail = S.z0_overflow = S.total = 0;
    S.z0.n = 0;
    S.z0.first_ins = INT32_MAX;
    tst[b] = S;
}
__global__ void __launch_bounds__(256) ti_init_ins_kernel(const TpBlock* __restrict__ blocks, const TpState* __restrict__ st, uint8_t* __restrict__ ins) {
    const TpBlock B = blocks[blockIdx.y];
    if (!(B.go & 0x100u)) return;
    const uint32_t nc = st[blockIdx.y].ncand;
    for (uint32_t k = blockIdx.x * 256 + threadIdx.x; k < nc; k += gridDim.x * 256) ins[B.cand_off + k] = 1;
}

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// the dictionary rounds of kz_text_par_core.cuh for every block with go & 0x100; h_st[b].changed != 0 afterwards: no fixed point within MAX_ROUNDS
cudaError_t dictionary_rounds(const uint8_t* d_in, const TpBlock* d_pb, const std::vector<TpBlock>& pb, TpState* d_st, std::vector<TpState>& h_st,
                              const Candidate* d_cand, uint8_t* d_ins, uint8_t* d_ins2, int32_t* d_owner, const int32_t* d_owner0,
                              const Entry* sd, const uint8_t* d_swords, uint32_t* d_ct, uint32_t* d_tot, uint32_t* d_rank, int32_t* d_focc, uint8_t* d_fflip,
                              uint32_t max_nct, int inverse, size_t ins_bytes /* size of d_ins / d_ins2 */, cudaStream_t stream, uint64_t* launches) {
    const uint32_t nblocks = (uint32_t)pb.size();
    const dim3 gc(max_nct, nblocks), gs(32, nblocks);
    uint8_t *cur = d_ins, *nxt = d_ins2;
    bool converged = false;
    cudaError_t e;
    for (int rounds = 0; rounds < MAX_ROUNDS && !converged; rounds++) {
        tp_round_begin_kernel<<<gs, 256, 0, stream>>>(d_pb, d_st, d_owner0, d_owner);
        tp_round_owners_kernel<<<gc, 256, 0, stream>>>(d_pb, d_st, d_cand, cur, d_owner, d_ct);
        tp_round_nx_kernel<<<gs, 256, 0, stream>>>(d_pb, d_st, cur);
        tp_scan_tiles_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, 1, d_ct, d_tot, CT, d_tot, 8, 1);
        tp_round_eval_kernel<<<gc, 256, 0, stream>>>(d_in, d_pb, d_st, d_cand, cur, nxt, d_owner, sd, d_swords, d_ct, d_rank, d_focc, d_fflip, inverse);
        if (launches) *launches += 5;
        if ((e = cudaMemcpyAsync(h_st.data(), d_st, nblocks * sizeof(TpState), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
        converged = true;
        for (uint32_t b = 0; b < nblocks; b++)
            if ((pb[b].go & 0x100u) && h_st[b].changed) converged = false;
        std::swap(cur, nxt);  // the decisions of this round
    }
    // a converged block has identical decisions in both buffers; the inverse path reads them from d_ins
    if (cur != d_ins) {  // exactly the decision bytes: d_ins2 / d_rank follow d_ins in the workspace
        if ((e = cudaMemcpyAsync(d_ins, cur, ins_bytes, cudaMemcpyDeviceToDevice, stream)) != cudaSuccess) return e;
    }
    return cudaGetLastError();
}

// the hash maps of a batch: every block's (text_map_layout), then the static words' map of each distinct size (owner0_maps)
struct HashMaps {
    std::vector<uint64_t> off;
    std::vector<uint32_t> lg, owner0_off;
    Owner0Maps o0;
    uint64_t slots = 0, o0_slots = 0;
    HashMaps(const uint64_t* bs, uint32_t nblocks) {
        slots = text_map_layout(bs, nblocks, off, lg);
        o0_slots = owner0_maps(lg, o0, owner0_off);
    }
};

}  // namespace

size_t text_parallel_workspace(const uint64_t* bs, uint32_t nblocks, uint32_t max_len) {
    const HashMaps H(bs, nblocks);
    const size_t nb = nblocks;
    const size_t cands = nb * ((size_t)max_len / 3 + 16), cps = nb * ((size_t)max_len + 8), pts = nb * ((size_t)max_len / PT + 2), cts = nb * (((size_t)max_len / 3 + 16 + CT - 1) / CT + 1);
    return align256(nb * sizeof(TpBlock)) + align256(nb * sizeof(TpState)) + align256(nb * 32) + align256(nb * 4) + 2 * align256(pts * 4) + 2 * align256(cts * 4) +
           align256(cands * sizeof(Candidate)) + 3 * align256(cands) + 3 * align256(cands * 4) + align256(cands * sizeof(FoundW)) + align256(cps * 4) +
           align256(H.slots * 4) + align256(H.o0_slots * 4) + 8192;
}

// d_go: the plan kernel's verdict per block (mode | 0x100 for text blocks). On return h_fallback[b] != 0 marks the text blocks the serial walk must do.
cudaError_t text_forward_parallel(const uint8_t* d_in, uint8_t* d_out, const std::vector<StageBlock>& tb, const uint32_t* d_go, const uint64_t* bs,
                                  const void* d_sdict, const uint8_t* d_swords, int static_n, uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream,
                                  std::vector<uint32_t>& h_fallback, uint64_t* launches) {
    const uint32_t nblocks = (uint32_t)tb.size();
    h_fallback.assign(nblocks, 0);
    if (nblocks == 0) return cudaSuccess;
    std::vector<uint32_t> h_go(nblocks);
    cudaError_t e = cudaMemcpyAsync(h_go.data(), d_go, nblocks * 4, cudaMemcpyDeviceToHost, stream);
    if (e != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    bool any = false;
    for (uint32_t b = 0; b < nblocks; b++) any = any || (h_go[b] & 0x100u);
    if (!any) return cudaSuccess;
    const HashMaps H(bs, nblocks);
    std::vector<TpBlock> pb(nblocks);
    uint64_t cands = 0, cps = 0;
    uint32_t pts = 0, cts = 0, max_npt = 1, max_nct = 1;
    for (uint32_t b = 0; b < nblocks; b++) {
        TpBlock& B = pb[b];
        B.src_off = tb[b].src_off;
        B.dst_off = tb[b].dst_off;
        B.len = tb[b].len;
        B.go = h_go[b];
        B.cand_off = cands;
        cands += (uint64_t)B.len / 3 + 16;
        B.cp_off = cps;
        cps += (uint64_t)B.len + 8;
        B.owner_off = H.off[b];
        B.mask = (1u << H.lg[b]) - 1;
        B.owner0_off = H.owner0_off[b];
        B.pt_base = pts;
        B.npt = B.len / PT + 1;  // the tile of position `len` included (cp[len] = total cost)
        pts += B.npt + 1;
        B.ct_base = cts;
        B.nct_cap = (uint32_t)((B.len / 3 + 16 + CT - 1) / CT);
        cts += B.nct_cap + 1;
        if (B.go & 0x100u) {
            max_npt = std::max(max_npt, B.npt);
            max_nct = std::max(max_nct, B.nct_cap);
        }
    }
    size_t off = 0;
    auto take = [&](size_t bytes) {
        uint8_t* p = ws + off;
        off = align256(off + bytes);
        return p;
    };
    TpBlock* d_pb = (TpBlock*)take(nblocks * sizeof(TpBlock));
    TpState* d_st = (TpState*)take(nblocks * sizeof(TpState));
    uint32_t* d_tot = (uint32_t*)take(nblocks * 32);  // [b][0] = candidates, [1] = inserts, [2] = bytes of all found words, [3] = found words, [4] = scratch
    uint32_t* d_fb = (uint32_t*)take(nblocks * 4);
    int* d_tile_last = (int*)take(pts * 4);
    uint32_t* d_pt = (uint32_t*)take(pts * 4);
    uint32_t* d_ct = (uint32_t*)take(cts * 4);
    uint32_t* d_ct2 = (uint32_t*)take(cts * 4);
    Candidate* d_cand = (Candidate*)take(cands * sizeof(Candidate));
    uint8_t* d_ins = take(cands);
    uint8_t* d_ins2 = take(cands);
    uint32_t* d_rank = (uint32_t*)take(cands * 4);
    int32_t* d_focc = (int32_t*)take(cands * 4);
    uint32_t* d_outpos = (uint32_t*)take(cands * 4);
    uint8_t* d_fflip = take(cands);
    FoundW* d_found = (FoundW*)take(cands * sizeof(FoundW));
    uint32_t* d_cp = (uint32_t*)take(cps * 4);
    int32_t* d_owner = (int32_t*)take((size_t)H.slots * 4);
    int32_t* d_owner0 = (int32_t*)take((size_t)H.o0_slots * 4);
    if (off > ws_bytes) return cudaErrorInvalidValue;
    const Entry* sd = (const Entry*)d_sdict;
    if ((e = cudaMemcpyAsync(d_pb, pb.data(), nblocks * sizeof(TpBlock), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(d_fb, 0, nblocks * 4, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(d_tot, 0, nblocks * 32, stream)) != cudaSuccess) return e;
    const dim3 gp(max_npt, nblocks), gc(max_nct, nblocks), gs(32, nblocks);
    // ---- A
    tp_fill_kernel<<<64, 256, 0, stream>>>(d_owner0, OCC_EMPTY, H.o0_slots);
    tp_owner0_kernel<<<H.o0.n, 32, 0, stream>>>(sd, static_n, H.o0, d_owner0);
    tp_last_nontext_kernel<<<gp, 256, 0, stream>>>(d_in, d_pb, d_tile_last);
    tp_carry_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_pb, (int)nblocks, d_tile_last, d_st);
    tp_candidates_kernel<<<gp, 256, 0, stream>>>(d_in, d_pb, d_tile_last, d_pt, 0, d_cand);
    tp_scan_tiles_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, 0, d_pt, nullptr, PT, d_tot, 8, 0);
    tp_candidates_kernel<<<gp, 256, 0, stream>>>(d_in, d_pb, d_tile_last, d_pt, 1, d_cand);
    tp_set_counts_kernel<<<(nblocks + 255) / 256, 256, 0, stream>>>(d_pb, (int)nblocks, d_st, d_tot, 0);
    if (launches) *launches += 7;
    tp_init_ins_kernel<<<gs, 256, 0, stream>>>(d_pb, d_st, d_cand, d_ins);
    // ---- B
    std::vector<TpState> h_st(nblocks);
    if ((e = dictionary_rounds(d_in, d_pb, pb, d_st, h_st, d_cand, d_ins, d_ins2, d_owner, d_owner0, sd, d_swords, d_ct, d_tot, d_rank, d_focc, d_fflip, max_nct,
                               0, (size_t)cands, stream, launches)) != cudaSuccess)
        return e;
    // the last round confirmed `nxt` (== cur bytewise for converged blocks); rank / focc / fflip belong to it
    std::vector<uint32_t> h_tot(nblocks * 8);
    if ((e = cudaMemcpyAsync(h_tot.data(), d_tot, nblocks * 32, cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    for (uint32_t b = 0; b < nblocks; b++) {
        if (!(pb[b].go & 0x100u)) continue;
        if (h_st[b].changed || h_st[b].z0_overflow || (uint64_t)STATIC_WORDS + h_tot[b * 8 + 1] >= (uint64_t)MAX_DICT_SIZE) h_fallback[b] = 1;
    }
    if ((e = cudaMemcpyAsync(d_fb, h_fallback.data(), nblocks * 4, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    // ---- C
    tp_found_kernel<<<gc, 256, 0, stream>>>(d_pb, d_st, d_cand, d_focc, d_fflip, d_rank, d_ct2, 0, d_found);
    tp_scan_tiles_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, 1, d_ct2, d_tot, CT, d_tot, 8, 3);
    tp_found_kernel<<<gc, 256, 0, stream>>>(d_pb, d_st, d_cand, d_focc, d_fflip, d_rank, d_ct2, 1, d_found);
    tp_set_counts_kernel<<<(nblocks + 255) / 256, 256, 0, stream>>>(d_pb, (int)nblocks, d_st, d_tot, 1);
    tp_cost_kernel<<<gp, 256, 0, stream>>>(d_in, d_pb, d_pt, 0, d_cp);
    tp_scan_tiles_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, 0, d_pt, nullptr, PT, d_tot, 8, 4);
    tp_cost_kernel<<<gp, 256, 0, stream>>>(d_in, d_pb, d_pt, 1, d_cp);
    tp_found_cost_kernel<<<gc, 256, 0, stream>>>(d_in, d_pb, d_st, d_found, d_cp, d_ct2, 0, d_outpos);
    tp_scan_tiles_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, 1, d_ct2, d_tot + 3, CT, d_tot, 8, 2);
    tp_found_cost_kernel<<<gc, 256, 0, stream>>>(d_in, d_pb, d_st, d_found, d_cp, d_ct2, 1, d_outpos);
    tp_finalize_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, d_st, d_found, d_cp, d_tot, d_out, d_res, d_fb);
    tp_emit_found_kernel<<<gs, 256, 0, stream>>>(d_in, d_pb, d_st, d_found, d_cp, d_outpos, d_out, d_fb);
    tp_emit_bytes_kernel<<<gp, 256, 0, stream>>>(d_in, d_pb, d_st, d_found, d_cp, d_outpos, d_tot, d_out, d_fb);
    if (launches) *launches += 12;
    return cudaGetLastError();
}

cudaError_t text_inverse_parallel(const uint8_t* d_in, uint8_t* d_out, const std::vector<StageBlock>& tb, const uint64_t* bs, const void* d_sdict,
                                  const uint8_t* d_swords, int static_n, uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream,
                                  std::vector<uint32_t>& h_fallback, uint64_t* launches) {
    const uint32_t nblocks = (uint32_t)tb.size();
    h_fallback.assign(nblocks, 1);
    if (nblocks == 0) return cudaSuccess;
    const HashMaps H(bs, nblocks);
    std::vector<TiBlock> ib(nblocks);
    std::vector<TpBlock> pb(nblocks);
    uint64_t cands = 0, poss = 0;
    uint32_t pts = 0, cts = 0, max_npt = 1, max_nct = 1;
    bool any = false;
    for (uint32_t b = 0; b < nblocks; b++) {
        TiBlock& B = ib[b];
        B.src_off = tb[b].src_off;
        B.dst_off = tb[b].dst_off;
        B.len = tb[b].len;
        B.cap = tb[b].cap;
        B.go = (B.len >= 2 && B.len <= (1u << 30) && B.cap != 0) ? 0x100u : 0u;
        B.cand_off = cands;
        cands += (uint64_t)B.len / 4 + 16;
        B.pos_off = poss;
        poss += (uint64_t)B.len + 16;
        B.owner_off = H.off[b];
        B.pt_base = pts;
        B.npt = B.len / PT + 1;
        pts += B.npt + 1;
        B.ct_base = cts;
        B.nct_cap = (uint32_t)((B.len / 4 + 16 + CT - 1) / CT);
        cts += B.nct_cap + 1;
        TpBlock& P = pb[b];
        P.src_off = B.src_off, P.dst_off = B.dst_off, P.cand_off = B.cand_off, P.cp_off = 0, P.owner_off = B.owner_off;
        P.len = B.len, P.go = B.go, P.pt_base = B.pt_base, P.npt = B.npt, P.ct_base = B.ct_base, P.nct_cap = B.nct_cap;
        P.mask = (1u << H.lg[b]) - 1, P.owner0_off = H.owner0_off[b];
        if (B.go) {
            any = true;
            max_npt = std::max(max_npt, B.npt);
            max_nct = std::max(max_nct, B.nct_cap);
        }
    }
    if (!any) return cudaSuccess;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        uint8_t* p = ws + off;
        off = align256(off + bytes);
        return p;
    };
    TiBlock* d_ib = (TiBlock*)take(nblocks * sizeof(TiBlock));
    TpBlock* d_pb = (TpBlock*)take(nblocks * sizeof(TpBlock));
    TpState* d_tst = (TpState*)take(nblocks * sizeof(TpState));
    TiState* d_ist = (TiState*)take(nblocks * sizeof(TiState));
    uint32_t* d_tot = (uint32_t*)take(nblocks * 32);  // [0] candidates, [1] inserts, [5] output bytes
    uint32_t* d_fn = (uint32_t*)take(pts * 4);
    int* d_lastq = (int*)take(pts * 4);
    uint32_t* d_pt = (uint32_t*)take(pts * 4);
    uint32_t* d_ct = (uint32_t*)take(cts * 4);
    uint8_t* d_start = take(poss);
    int32_t* d_prevq = (int32_t*)take(poss * 4);
    Candidate* d_cand = (Candidate*)take(cands * sizeof(Candidate));
    uint8_t* d_ins = take(cands);
    uint8_t* d_ins2 = take(cands);
    uint32_t* d_rank = (uint32_t*)take(cands * 4);
    int32_t* d_focc = (int32_t*)take(cands * 4);
    uint32_t* d_ins_list = (uint32_t*)take(cands * 4);
    uint8_t* d_fflip = take(cands);
    int32_t* d_owner = (int32_t*)take((size_t)H.slots * 4);
    int32_t* d_owner0 = (int32_t*)take((size_t)H.o0_slots * 4);
    if (off > ws_bytes) return cudaErrorInvalidValue;
    const Entry* sd = (const Entry*)d_sdict;
    cudaError_t e;
    if ((e = cudaMemcpyAsync(d_ib, ib.data(), nblocks * sizeof(TiBlock), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(d_pb, pb.data(), nblocks * sizeof(TpBlock), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(d_tot, 0, nblocks * 32, stream)) != cudaSuccess) return e;
    const dim3 gp(max_npt, nblocks), gs(32, nblocks);
    const uint32_t gb = (nblocks + 255) / 256;
    tp_fill_kernel<<<64, 256, 0, stream>>>(d_owner0, OCC_EMPTY, H.o0_slots);
    tp_owner0_kernel<<<H.o0.n, 32, 0, stream>>>(sd, static_n, H.o0, d_owner0);
    ti_token_tiles_kernel<<<gp, 256, 0, stream>>>(d_in, d_ib, d_fn);
    ti_token_carry_kernel<<<nblocks, 32, 0, stream>>>(d_ib, (int)nblocks, d_fn, d_ist);
    ti_token_mark_kernel<<<gp, 256, 0, stream>>>(d_in, d_ib, d_fn, d_start, d_lastq);
    ti_lastq_carry_kernel<<<nblocks, 32, 0, stream>>>(d_ib, (int)nblocks, d_lastq);
    ti_candidates_kernel<<<gp, 256, 0, stream>>>(d_in, d_ib, d_start, d_lastq, sd, static_n, d_pt, 0, d_prevq, d_cand);
    tp_scan_tiles_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, 0, d_pt, nullptr, PT, d_tot, 8, 0);
    ti_candidates_kernel<<<gp, 256, 0, stream>>>(d_in, d_ib, d_start, d_lastq, sd, static_n, d_pt, 1, d_prevq, d_cand);
    ti_set_ncand_kernel<<<gb, 256, 0, stream>>>(d_ib, (int)nblocks, d_tst, d_tot);
    ti_init_ins_kernel<<<gs, 256, 0, stream>>>(d_pb, d_tst, d_ins);
    if (launches) *launches += 11;
    std::vector<TpState> h_st(nblocks);
    if ((e = dictionary_rounds(d_in, d_pb, pb, d_tst, h_st, d_cand, d_ins, d_ins2, d_owner, d_owner0, sd, d_swords, d_ct, d_tot, d_rank, d_focc, d_fflip, max_nct, 1,
                               (size_t)cands, stream, launches)) != cudaSuccess)
        return e;
    ti_ins_list_kernel<<<gs, 256, 0, stream>>>(d_pb, d_tst, d_ins, d_rank, d_ins_list);
    ti_output_kernel<<<gp, 256, 0, stream>>>(d_in, d_ib, d_tst, d_ist, d_start, d_prevq, d_cand, d_rank, d_tot, d_ins_list, sd, d_swords, static_n, d_pt, 0, d_out);
    tp_scan_tiles_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, 0, d_pt, nullptr, PT, d_tot, 8, 5);
    // blocks whose rounds did not settle (or whose list would wrap, or with too many words in map slot 0) are anomalies as well
    std::vector<uint32_t> h_tot(nblocks * 8);
    if ((e = cudaMemcpyAsync(h_tot.data(), d_tot, nblocks * 32, cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
    std::vector<TiState> h_ist(nblocks);
    if ((e = cudaMemcpyAsync(h_ist.data(), d_ist, nblocks * sizeof(TiState), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    for (uint32_t b = 0; b < nblocks; b++) {
        if (!ib[b].go) continue;
        if (h_st[b].changed || h_st[b].z0_overflow || (uint64_t)STATIC_WORDS + h_tot[b * 8 + 1] >= (uint64_t)MAX_DICT_SIZE) h_ist[b].anomaly = 1;
    }
    if ((e = cudaMemcpyAsync(d_ist, h_ist.data(), nblocks * sizeof(TiState), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    ti_finalize_kernel<<<gb, 256, 0, stream>>>(d_ib, (int)nblocks, d_ist, d_tot, d_res);
    ti_output_kernel<<<gp, 256, 0, stream>>>(d_in, d_ib, d_tst, d_ist, d_start, d_prevq, d_cand, d_rank, d_tot, d_ins_list, sd, d_swords, static_n, d_pt, 1, d_out);
    if (launches) *launches += 5;
    if ((e = cudaMemcpyAsync(h_ist.data(), d_ist, nblocks * sizeof(TiState), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    for (uint32_t b = 0; b < nblocks; b++) h_fallback[b] = (ib[b].go && !h_ist[b].anomaly) ? 0u : 1u;
    return cudaGetLastError();
}

size_t text_inverse_parallel_workspace(const uint64_t* bs, uint32_t nblocks, uint32_t max_len) {
    const HashMaps H(bs, nblocks);
    const size_t nb = nblocks;
    const size_t cands = nb * ((size_t)max_len / 4 + 16), poss = nb * ((size_t)max_len + 16), pts = nb * ((size_t)max_len / PT + 2), cts = nb * (((size_t)max_len / 4 + 16 + CT - 1) / CT + 1);
    return align256(nb * sizeof(TiBlock)) + align256(nb * sizeof(TpBlock)) + align256(nb * sizeof(TpState)) + align256(nb * sizeof(TiState)) + align256(nb * 32) +
           3 * align256(pts * 4) + align256(cts * 4) + align256(poss) + align256(poss * 4) + align256(cands * sizeof(Candidate)) + 3 * align256(cands) + 3 * align256(cands * 4) +
           align256(H.slots * 4) + align256(H.o0_slots * 4) + 8192;
}

}  // namespace kz
