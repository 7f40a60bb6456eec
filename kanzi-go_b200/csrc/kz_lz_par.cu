// Data-parallel LZ / LZX forward transform on sm_90a (the parse logic itself is kz_lz_par_core.cuh, shared with the CPU harness
// tests/host/lz_par_host.cpp). Reference: v2/transform/LZCodec.go:249-591. Passes, all blocks of a batch together:
//
//   hash      position -> (block << hash_bits | hash) key                                   [streaming, 8-byte loads]
//   sort      stable radix sort of (key, position) pairs by key (cub::DeviceRadixSort — the one library call of this path)
//   link      neighbours of the sorted order with equal keys -> prev[] per position           [scatter]
//   info      common prefix / suffix lengths of (i, prev[i]), saturated at 255               [streaming compares]
//   rounds to the fixed point of the table membership vf[] (kz_lz_par_core.cuh, 3.; two rounds for ordinary blocks):
//     filter    candidates under the previous round's vf (round 0: as linked)
//     spec      one warp per 1 KiB segment (the lanes take the next 32 probes of a literal run): speculative parse from a guessed state ->
//               match log of the segment
//     junction  one warp per segment: from the state the segment's log stopped in, the parse until it meets the log of the segment it is in
//     walk      one CTA per block: junction records staged in shared memory, one thread follows them -> piece list of the match list
//     stitch    (only blocks with a live junction that hit its cap) one lane per block: the serial stitch of kz_lz_par_core.cuh
//     flatten   pieces -> contiguous match list
//     derive    per position: vf' from the match list (closed form for the probe pattern of a literal run); changed?
//   sizes / tilescan / emit   per match token, distance bytes, length bytes, literal run: sizes, block-wide exclusive scans, final bytes
//   literals  warp-wide copies of the literal runs
#include <cub/device/device_radix_sort.cuh>

#include <vector>

#include "kz_lz.cuh"
#include "kz_lz_par_core.cuh"

namespace kz {

using namespace lzp;

namespace {

const int SEG = 1024;                // bytes per speculative segment (one warp each)
const int SEG_CAP = SEG / 4 + 8;     // log entries per segment (a match is at least 4 bytes long)
const int JCAP = 64;                 // fix-up matches per junction before it gives up (a live one that does sends the block to the serial stitch)
const int PROBE_CAP = 32;            // bytes a lane follows a match on its own before the warp takes over (a multiple of 8)
const int WALK_WIN = 4096;
const int WALKP_MAX_SERIAL_FROM = 4096;  // blocks with more segments than this take the windowed serial walk (= WALKP_MAX)           // junction records staged in shared memory per window of the walk
const int MAX_ROUNDS = 96;
const int TILE = 1024;               // matches per emission tile
const uint32_t LONG_RUN = 4096;      // literal runs above this length are copied by all warps of the block's CTAs together

struct PBlock {  // device descriptor of one block of the batch
    uint64_t src_off, dst_off;
    uint64_t pos_off;    // first entry of the block in rec[] / next[] and (bit index) in the bitmaps; a multiple of 64
    uint64_t match_off;  // first entry of the block in fix[] / ml[] / runs[]
    uint32_t count, src_end, npos;
    int32_t max_dist, min_match;
    uint32_t seg_base, nsegs;
    uint32_t piece_off;  // first entry in pieces[]
    uint32_t tile_base, ntiles_cap;
    uint32_t active, flags;
    uint32_t long_off, pad;  // first entry of the block in the list of long literal runs
};
struct PState {  // per block results of the stitch / scan passes
    uint32_t np, fix_n, nmatch;
    int32_t final_anchor;
    uint32_t m_total, mlen_total, lit_total, too_many;
};

__device__ __forceinline__ Params make_params(const uint8_t* in, const PBlock& B, int extra, const Rec* rec) {
    Params P;
    P.src = in + B.src_off;
    P.count = (int)B.count;
    P.src_end = (int)B.src_end;
    P.max_dist = B.max_dist;
    P.min_match = B.min_match;
    P.extra = extra;
    P.rec = rec + B.pos_off;
    P.seg_size = SEG;
    return P;
}

// ---- pass 0 --------------------------------------------------------------------------------------------------------------------------
// one thread per position of the concatenated position space; blk_of_tile gives the block of each 1024-position tile
__global__ void __launch_bounds__(256) lzp_hash_kernel(const uint8_t* __restrict__ in, const PBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_chunk,
                                                        int extra, int hash_bits, uint32_t nblocks, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                        uint64_t total) {
    const uint64_t g = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (g >= total) return;
    const uint32_t b = blk_of_chunk[g >> 10];
    const PBlock& B = blocks[b];
    const uint32_t i = (uint32_t)(g - B.pos_off);
    // positions >= npos (and the padding up to the next multiple of 1024) carry the block index `nblocks`: they sort behind every real key
    uint32_t key = nblocks << hash_bits;
    if (B.active && i < B.npos) key = (b << hash_bits) | lz_hash(ld64(in + B.src_off + i), extra != 0);
    keys[g] = key;
    vals[g] = i;
}
__global__ void __launch_bounds__(256) lzp_link_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, const PBlock* __restrict__ blocks, int hash_bits,
                                                        uint32_t nblocks, Rec* __restrict__ rec, uint64_t total) {
    const uint64_t g = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (g >= total) return;
    const uint32_t key = keys[g];
    const uint32_t b = key >> hash_bits;
    if (b >= nblocks) return;
    const uint64_t base = blocks[b].pos_off;
    const uint32_t i = vals[g];
    const bool has_prev = g > 0 && keys[g - 1] == key;
    rec[base + i].prev = has_prev ? vals[g - 1] : NONE;
}
__global__ void __launch_bounds__(256) lzp_info_kernel(const uint8_t* __restrict__ in, const PBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_chunk,
                                                        Rec* __restrict__ rec, uint64_t total) {
    const uint64_t g = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (g >= total) return;
    const uint32_t b = blk_of_chunk[g >> 10];
    const PBlock& B = blocks[b];
    const uint32_t i = (uint32_t)(g - B.pos_off);
    if (!B.active || i >= B.npos) {  // never probed: no candidate
        rec[g].prev = NONE;
        rec[g].info = 0;
        return;
    }
    rec[g].info = make_info(in + B.src_off, (int)B.count, (int)i, rec[g].prev);
}
// candidates of a round: the first position of the prev[] chain that is in the table (vf) when the position is probed
__global__ void __launch_bounds__(256) lzp_filter_kernel(const uint8_t* __restrict__ in, const PBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_chunk,
                                                          const uint32_t* __restrict__ act_chunks, const Rec* __restrict__ rec0, const uint32_t* __restrict__ vf,
                                                          Rec* __restrict__ rec, uint64_t total, int first_filter, uint32_t* __restrict__ dirty) {
    const uint64_t g = (uint64_t)act_chunks[blockIdx.x >> 2] * 1024 + (blockIdx.x & 3) * 256 + threadIdx.x;  // only chunks of unfinished blocks are launched
    if (g >= total) return;
    const uint32_t b = blk_of_chunk[g >> 10];
    const PBlock& B = blocks[b];
    const uint32_t i = (uint32_t)(g - B.pos_off);
    if (!B.active || i >= B.npos) {
        rec[g] = rec0[g];
        return;
    }
    const Rec r_new = filter_candidate(in + B.src_off, (int)B.count, rec0 + B.pos_off, vf + B.pos_off, (int)i);
    const Rec r_old = first_filter ? rec0[g] : rec[g];  // what the previous round's parse saw at this position
    if (r_new.prev != r_old.prev || r_new.info != r_old.info) dirty[B.seg_base + i / SEG] = 1;  // "changed": lzp_dirty_kernel spreads it
    rec[g] = r_new;
}
// A segment's speculative parse reads the candidates from its first byte up to the end of its last match (it only stops behind a match
// that ends at or behind the segment, however far the literal run before that match reaches): dirty[k] = a candidate changed anywhere in
// the segments [k, segment of the last byte it read]. desc[] is the previous round's.
__global__ void __launch_bounds__(128) lzp_dirty_kernel(const PBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_seg, const uint32_t* __restrict__ act_segs,
                                                         uint32_t n_act, const SegDesc* __restrict__ desc, const uint32_t* __restrict__ changed,
                                                         uint32_t* __restrict__ dirty) {
    const uint32_t t = blockIdx.x * 128 + threadIdx.x;
    if (t >= n_act) return;
    const uint32_t s = act_segs[t];
    const PBlock& B = blocks[blk_of_seg[s]];
    const SegDesc d = desc[s];
    const uint32_t last = B.seg_base + B.nsegs - 1;
    uint32_t k_end = last;
    if (d.end != END_BLOCK) k_end = min(last, B.seg_base + (uint32_t)(max(d.fin.anchor, 1) - 1) / SEG);
    uint32_t any = 0;
    for (uint32_t k = s; k <= k_end && !any; k++) any = changed[k];
    dirty[s] = any;
}
// vf' of every position from the block's match list; changed[b] |= (vf' != vf)
__global__ void __launch_bounds__(256) lzp_derive_kernel(const PBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_chunk, const uint32_t* __restrict__ act_chunks,
                                                          const PState* __restrict__ pst, const Match* __restrict__ ml_all, const uint32_t* __restrict__ vf,
                                                          uint32_t* __restrict__ vf2, uint32_t* __restrict__ changed, uint64_t total) {
    // one CTA per chunk of 1024 positions, four consecutive positions per thread: one search in the match list, then it only moves forward
    const uint64_t g0 = (uint64_t)act_chunks[blockIdx.x] * 1024 + threadIdx.x * 4;
    const uint32_t b = blk_of_chunk[act_chunks[blockIdx.x]];
    const PBlock& B = blocks[b];
    bool diff = false;
    if (g0 < total) {  // total is a multiple of 1024
        const Match* ml = ml_all + B.match_off;
        const uint32_t nm = pst[b].nmatch;
        const uint32_t i0 = (uint32_t)(g0 - B.pos_off);
        uint32_t v[4] = {0, 0, 0, 0};
        if (B.active && i0 < B.count) {
            uint32_t t = matches_ended(ml, nm, (int)i0);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t i = i0 + k;
                if (i >= B.count) break;
                while (t < nm && (int)(ml[t].start + ml[t].len) <= (int)i) t++;
                v[k] = derive_vf_at(ml, nm, (int)B.src_end, (int)i, t);
            }
        }
        const uint4 old = *reinterpret_cast<const uint4*>(vf + g0);
        *reinterpret_cast<uint4*>(vf2 + g0) = make_uint4(v[0], v[1], v[2], v[3]);
        diff = v[0] != old.x || v[1] != old.y || v[2] != old.z || v[3] != old.w;
    }
    if (__syncthreads_or(diff ? 1 : 0) && threadIdx.x == 0) atomicOr(&changed[b], 1u);
}

// ---- warp-cooperative parse: the 32 lanes evaluate the next 32 probes of the literal run at once ------------------------------------------------
// probe_first is a pure function of (position, the two repeat distances, candidates); the positions of the next probes follow from the run
// counter (stride 1 + (src_inc >> 6)), so the lanes take one probe each, the lowest lane with a match wins and every lane then runs the
// (uniform) second stage on the winner's values. One memory round trip per 32 probes of a literal run, and per match on compressible data.
// All lanes hold the same `st` / `m` on entry and exit.
__device__ __forceinline__ int parse_one_warp(const Params& P, State& st, Match& m) {
    const int lane = threadIdx.x & 31;
    for (;;) {
        if (st.src_idx >= P.src_end) return R_END;
        const int step = 1 + ((st.src_inc + lane) >> 6);
        int incl = step;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= d) incl += y;
        }
        const int pos = st.src_idx + incl - step;
        const bool valid = pos < P.src_end;
        int best_len = 0, ref = 0, kind = 0, b = 0, ext = 0;
        bool hit = false;
        Rec r1, r2;
        r1.prev = r2.prev = NONE, r1.info = r2.info = 0;
        if (valid) {
            // probe_first of kz_lz_par_core.cuh with every load issued before the first decision: one memory round trip per round
            const bool swapped = lane == 0 && st.repd_idx != 0;
            const int rf = swapped ? st.repd1 : st.repd0, rs = swapped ? st.repd0 : st.repd1;
            const uint8_t* src = P.src;
            const int pos1 = pos + 1;
            const int max_match = imin(P.src_end - pos1, MAX_MATCH);
            const int min_ref = imax(pos - P.max_dist, 0);
            const int ref_a = pos1 - rf, ref_b = pos1 - rs;
            const uint64_t p = ld64(src + pos);
            const Rec r0 = P.rec[pos];
            r1 = P.rec[pos + 1];
            r2 = P.rec[pos + 2];
            const uint32_t wa = ref_a > min_ref ? ld32(src + ref_a) : 0u, wb = ref_b > min_ref ? ld32(src + ref_b) : 0u;
            const uint32_t p4 = (uint32_t)(p >> 8);
            // lengths are followed for PROBE_CAP bytes only here (enough for the decision); the winner's match is extended by the whole warp
            const int capped = imin(max_match, PROBE_CAP);
            ref = ref_a;
            bool rep_probe = false;
            if (ref_a > min_ref && p4 == wa) {
                best_len = find_match(src, pos1, ref_a, capped);
                rep_probe = true;
            } else {
                ref = ref_b;
                if (ref_b > min_ref && p4 == wb) best_len = find_match(src, pos1, ref_b, capped), rep_probe = true;
            }
            if (rep_probe && capped < max_match && best_len == (capped & ~7)) ext = 1;  // no mismatch inside the cap
            if (best_len >= P.min_match) {
                hit = true;
            } else {
                ext = 0;
                int cand, t;
                unpack_rec(r0, cand, t, b);
                if (cand > min_ref && t >= 4) {
                    const int m8 = imin(P.src_end - pos, MAX_MATCH) & ~7;
                    if (t < T_CAP || m8 <= T_CAP) best_len = t < m8 ? t : m8;  // match_len without the long compare
                    else best_len = T_CAP, ext = 2;                              // saturated: at least T_CAP, the winner finds out
                    if (best_len >= P.min_match) ref = cand, kind = 1, hit = true;
                    else ext = 0;
                }
            }
        }
        const uint32_t hits = __ballot_sync(0xFFFFFFFFu, hit), vmask = __ballot_sync(0xFFFFFFFFu, valid);
        if (hits == 0) {
            const int nvalid = __popc(vmask);  // the valid lanes are a prefix
            st.src_inc += nvalid;
            st.repd_idx = 0;
            if (nvalid < 32) {
                st.src_idx = __shfl_sync(0xFFFFFFFFu, pos, nvalid);
                return R_END;
            }
            st.src_idx = __shfl_sync(0xFFFFFFFFu, pos + step, 31);
            continue;
        }
        const int w = __ffs((int)hits) - 1;
        if (w > 0) st.repd_idx = 0;
        st.src_inc += w;
        st.src_idx = __shfl_sync(0xFFFFFFFFu, pos, w);
        best_len = __shfl_sync(0xFFFFFFFFu, best_len, w);
        ref = __shfl_sync(0xFFFFFFFFu, ref, w);
        kind = __shfl_sync(0xFFFFFFFFu, kind, w);
        b = __shfl_sync(0xFFFFFFFFu, b, w);
        r1.prev = __shfl_sync(0xFFFFFFFFu, r1.prev, w), r1.info = __shfl_sync(0xFFFFFFFFu, r1.info, w);
        r2.prev = __shfl_sync(0xFFFFFFFFu, r2.prev, w), r2.info = __shfl_sync(0xFFFFFFFFu, r2.info, w);
        ext = __shfl_sync(0xFFFFFFFFu, ext, w);
        if (ext == 1) {  // repeat-distance match longer than the cap (findMatchLZX from the probe's successor)
            best_len = find_match_w(P.src, st.src_idx + 1, ref, PROBE_CAP & ~7, imin(P.src_end - (st.src_idx + 1), MAX_MATCH));
        } else if (ext == 2) {  // table match with a saturated prefix length
            const int m8 = imin(P.src_end - st.src_idx, MAX_MATCH) & ~7;
            const int tt = common_prefix_w(P.src, P.count, st.src_idx, ref, T_CAP & ~7, m8 + 8);
            best_len = tt < m8 ? tt : m8;
        }
        probe_finish<true>(P, st, best_len, ref, kind, b, r1, r2, m);
        return R_MATCH;
    }
}

// ---- pass 1: speculative segment parses (one warp per segment; act_segs lists the segments of the unfinished blocks) ---------------------
__global__ void __launch_bounds__(128) lzp_spec_kernel(const uint8_t* __restrict__ in, const PBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_seg, int extra,
                                                        const uint32_t* __restrict__ act_segs, uint32_t n_act, const Rec* __restrict__ rec, Match* __restrict__ logs,
                                                        SegDesc* __restrict__ desc, const uint32_t* __restrict__ dirty) {
    const uint32_t t = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (t >= n_act) return;
    const int lane = threadIdx.x & 31;
    const uint32_t s = act_segs[t];
    if (!dirty[s]) return;  // same candidates as in the previous round: same log
    const uint32_t b = blk_of_seg[s];
    const PBlock& B = blocks[b];
    const uint32_t k = s - B.seg_base;
    const Params P = make_params(in, B, extra, rec);
    const int s0 = (int)(k * SEG);
    const int s1 = k == B.nsegs - 1 ? 0x7FFFFFFF : s0 + SEG;
    Match* log = logs + (size_t)s * SEG_CAP;
    State st = initial_state(P.count, s0);  // spec_parse_segment of kz_lz_par_core.cuh with the warp-cooperative parse
    uint32_t n = 0, end = END_BLOCK;
    for (;;) {
        Match m;
        if (parse_one_warp(P, st, m) == R_END) break;
        if (lane == 0) log[n] = m;
        n++;
        if (st.anchor >= s1) {
            end = END_POST_MATCH;
            break;
        }
    }
    if (lane == 0) {
        SegDesc d;
        d.n = n, d.end = end, d.fin = st;
        desc[s] = d;
    }
}

// ---- pass 2: junctions (one warp per segment), the walk over them (one CTA per block), the serial stitch for what the walk could not do ---------
struct SegLogAt {
    const Match* base;
    __device__ const Match* operator()(int k) const { return base + (size_t)k * SEG_CAP; }
};
// junction_parse of kz_lz_par_core.cuh with the warp-cooperative parse; the log of the segment the cursor is in is searched 32 entries at a time
__global__ void __launch_bounds__(128) lzp_junction_kernel(const uint8_t* __restrict__ in, const PBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_seg, int extra,
                                                            const uint32_t* __restrict__ act_segs, uint32_t n_act, const Rec* __restrict__ rec, const Match* __restrict__ logs,
                                                            const SegDesc* __restrict__ desc_all, Match* __restrict__ jfix, Junction* __restrict__ junc,
                                                            const uint32_t* __restrict__ dirty, int first_round) {
    const uint32_t t = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (t >= n_act) return;
    const int lane = threadIdx.x & 31;
    const uint32_t s = act_segs[t];
    const uint32_t b = blk_of_seg[s];
    const PBlock& B = blocks[b];
    if (!first_round) {
        // the junction read the state its segment stopped in, the logs and the candidates of the segments up to the one it joined: when none
        // of those segments is dirty its record stands
        const Junction old = junc[s];
        if (old.status == J_JOINED) {
            const uint32_t k_end = min(B.seg_base + old.seg, B.seg_base + B.nsegs - 1);
            bool any = false;
            for (uint32_t k = s + lane; k <= k_end; k += 32) any = any || dirty[k] != 0;
            if (!__any_sync(0xFFFFFFFFu, any)) return;
        }
    }
    const Params P = make_params(in, B, extra, rec);
    const SegDesc* desc = desc_all + B.seg_base;
    const Match* lbase = logs + (size_t)B.seg_base * SEG_CAP;
    const int k0 = (int)(s - B.seg_base), nsegs = (int)B.nsegs;
    Match* fix = jfix + (size_t)s * JCAP;
    State st = desc[k0].fin;
    Junction J;
    J.status = J_TERMINAL, J.fix_n = 0, J.seg = 0, J.idx = 0, J.anchor = st.anchor;
    if (desc[k0].end != END_BLOCK) {
        uint32_t fn = 0;
        int cur_seg = -1;
        uint32_t cursor = 0, dn = 0;
        const Match* lg = lbase;
        bool finished = false;
        while (st.src_idx < P.src_end) {
            const int k = imin(st.src_idx / SEG, nsegs - 1);
            if (k != cur_seg) {
                cur_seg = k;
                cursor = 0;
                dn = desc[k].n;
                lg = lbase + (size_t)k * SEG_CAP;
            }
            // first entry at or behind the cursor that ends at or behind the anchor
            while (cursor < dn) {
                const uint32_t i = cursor + lane;
                const bool ge = i < dn && (int)(lg[i].start + lg[i].len) >= st.anchor;
                const uint32_t mk = __ballot_sync(0xFFFFFFFFu, ge);
                if (mk) {
                    cursor += (uint32_t)__ffs((int)mk) - 1u;
                    break;
                }
                cursor = min(cursor + 32u, dn);
            }
            if (cursor >= 1 && cursor < dn) {
                const Match c = lg[cursor], pm = lg[cursor - 1];
                if ((int)(c.start + c.len) == st.anchor && (int)c.dist == st.repd0 && (int)pm.dist == st.repd1) {
                    J.status = J_JOINED, J.fix_n = fn, J.seg = (uint32_t)k, J.idx = cursor;
                    finished = true;
                    break;
                }
            }
            if (fn >= (uint32_t)JCAP) {
                J.status = J_OVERFLOW, J.fix_n = fn;
                finished = true;
                break;
            }
            Match m;
            if (parse_one_warp(P, st, m) == R_END) break;
            if (lane == 0) fix[fn] = m;
            fn++;
        }
        if (!finished) J.status = J_TERMINAL, J.fix_n = fn, J.anchor = st.anchor;
    }
    if (lane == 0) junc[s] = J;
}
// packed junction record of the walk: n (9 bits) | END_BLOCK << 9 | status << 10 | fix_n << 12 | idx << 19; second word: joined segment
__global__ void __launch_bounds__(256) lzp_walk_kernel(const PBlock* __restrict__ blocks, const uint32_t* __restrict__ act_blocks, const SegDesc* __restrict__ desc_all,
                                                        const Junction* __restrict__ junc_all, Piece* __restrict__ pieces, uint32_t* __restrict__ piece_start,
                                                        PState* __restrict__ pst) {
    __shared__ uint32_t s_w0[WALK_WIN], s_w1[WALK_WIN];
    __shared__ int s_k, s_stop;
    const uint32_t b = act_blocks[blockIdx.x];
    const PBlock B = blocks[b];
    if (!B.active) {
        if (threadIdx.x == 0) {
            PState S;
            S.np = S.fix_n = S.nmatch = 0, S.final_anchor = 0, S.m_total = S.mlen_total = S.lit_total = S.too_many = 0;
            pst[b] = S;
        }
        return;
    }
    if (B.nsegs <= (uint32_t)WALKP_MAX_SERIAL_FROM) return;  // lzp_walk_par_kernel does these
    const SegDesc* desc = desc_all + B.seg_base;
    const Junction* junc = junc_all + B.seg_base;
    Piece* pc = pieces + B.piece_off;
    uint32_t* ps = piece_start + B.piece_off;
    uint32_t np = 0, total = 0, begin = 0;  // thread 0's walk state
    int32_t final_anchor = 0;
    bool overflow = false;
    if (threadIdx.x == 0) s_k = 0, s_stop = 0;
    __syncthreads();
    for (;;) {
        const int base = s_k;
        for (int i = threadIdx.x; i < WALK_WIN && base + i < (int)B.nsegs; i += 256) {
            const SegDesc d = desc[base + i];
            const Junction J = junc[base + i];
            s_w0[i] = d.n | (d.end == END_BLOCK ? 1u << 9 : 0u) | (J.status << 10) | (J.fix_n << 12) | (J.idx << 19);
            s_w1[i] = J.seg;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int k = base;
            while (k < base + WALK_WIN) {
                const uint32_t w0 = s_w0[k - base];
                const uint32_t n = w0 & 0x1FFu, status = (w0 >> 10) & 3u, fix_n = (w0 >> 12) & 0x7Fu;
                if (n > begin) {
                    Piece p;
                    p.spec = 1, p.seg = (uint32_t)k, p.begin = begin, p.end = n;
                    pc[np] = p;
                    ps[np] = total;
                    np++;
                    total += n - begin;
                }
                if (w0 & (1u << 9)) {
                    final_anchor = desc[k].fin.anchor;
                    s_stop = 1;
                    break;
                }
                if (status == J_OVERFLOW) {
                    overflow = true;
                    s_stop = 1;
                    break;
                }
                if (fix_n) {
                    Piece p;
                    p.spec = 2, p.seg = (uint32_t)k, p.begin = 0, p.end = fix_n;
                    pc[np] = p;
                    ps[np] = total;
                    np++;
                    total += fix_n;
                }
                if (status == J_TERMINAL) {
                    final_anchor = junc[k].anchor;
                    s_stop = 1;
                    break;
                }
                k = (int)s_w1[k - base];
                begin = (w0 >> 19) + 1;
            }
            s_k = k;
        }
        __syncthreads();
        if (s_stop) break;
    }
    if (threadIdx.x == 0) {
        PState S;
        S.np = overflow ? 0xFFFFFFFFu : np;
        S.fix_n = 0;
        S.nmatch = total;
        S.final_anchor = final_anchor;
        S.m_total = S.mlen_total = S.lit_total = S.too_many = 0;
        ps[np] = total;
        pst[b] = S;
    }
}
// The same walk for blocks of up to WALKP_MAX segments without the serial loop: the junction records are a linked list next[k] > k from
// segment 0; the live segments are marked by pointer doubling (13 rounds over shared memory), every live segment then knows where its log
// is entered (one scatter), and its pieces and match counts are placed by a block-wide scan in segment order — which is list order.
const int WALKP_MAX = 4096;
__global__ void __launch_bounds__(256) lzp_walk_par_kernel(const PBlock* __restrict__ blocks, const uint32_t* __restrict__ act_blocks, const SegDesc* __restrict__ desc_all,
                                                            const Junction* __restrict__ junc_all, Piece* __restrict__ pieces, uint32_t* __restrict__ piece_start,
                                                            PState* __restrict__ pst) {
    __shared__ uint16_t s_next[WALKP_MAX], s_ja[WALKP_MAX], s_jb[WALKP_MAX], s_begin[WALKP_MAX];
    __shared__ uint8_t s_ma[WALKP_MAX], s_mb[WALKP_MAX];
    __shared__ uint32_t s_wp[8], s_wm[8];
    __shared__ uint32_t s_over, s_anchor;
    const uint32_t b = act_blocks[blockIdx.x];
    const PBlock B = blocks[b];
    if (!B.active || B.nsegs > (uint32_t)WALKP_MAX) return;  // larger blocks: lzp_walk_kernel
    const int n = (int)B.nsegs, tid = threadIdx.x;
    const SegDesc* desc = desc_all + B.seg_base;
    const Junction* junc = junc_all + B.seg_base;
    const uint16_t TERM = 0xFFFF;
    if (tid == 0) s_over = 0, s_anchor = 0;
    for (int k = tid; k < n; k += 256) {
        const bool last = desc[k].end == END_BLOCK;
        const uint32_t st = last ? (uint32_t)J_TERMINAL : junc[k].status;
        s_next[k] = st == J_JOINED ? (uint16_t)junc[k].seg : TERM;
        s_ja[k] = s_next[k];
        s_ma[k] = k == 0 ? 1 : 0;
        s_mb[k] = k == 0 ? 1 : 0;
        s_begin[k] = 0;
    }
    __syncthreads();
    // live[k]: k is on the list from 0. Round d: every marked k marks jump[k] (2^d links ahead), then jump doubles.
    uint16_t *ja = s_ja, *jb = s_jb;
    uint8_t *ma = s_ma, *mb = s_mb;
    for (int d = 0; (1 << d) < n; d++) {
        for (int k = tid; k < n; k += 256) {
            const uint16_t j = ja[k];
            if (ma[k]) {
                mb[k] = 1;
                if (j != TERM) mb[j] = 1;
            }
            jb[k] = j == TERM ? TERM : ja[j];
        }
        __syncthreads();
        uint16_t* tj = ja; ja = jb; jb = tj;
        uint8_t* tm = ma; ma = mb; mb = tm;
        for (int k = tid; k < n; k += 256) mb[k] = ma[k];  // the other copy catches up (marks only grow)
        __syncthreads();
    }
    // where a live segment's log is entered: behind the entry its predecessor joined
    for (int k = tid; k < n; k += 256)
        if (ma[k] && s_next[k] != TERM) s_begin[s_next[k]] = (uint16_t)(junc[k].idx + 1);
    __syncthreads();
    // pieces and match counts per live segment, 16 consecutive segments per thread, block-wide exclusive scan
    uint32_t cp = 0, cm = 0;
    const int k0 = tid * 16;
    for (int k = k0; k < min(k0 + 16, n); k++) {
        if (!ma[k]) continue;
        const uint32_t nk = desc[k].n, bg = s_begin[k];
        if (nk > bg) cp++, cm += nk - bg;
        if (desc[k].end == END_BLOCK) continue;
        const Junction J = junc[k];
        if (J.status == J_OVERFLOW) {
            s_over = 1;
            continue;
        }
        if (J.fix_n) cp++, cm += J.fix_n;
    }
    uint32_t ip = cp, im = cm;
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t yp = __shfl_up_sync(0xFFFFFFFFu, ip, d), ym = __shfl_up_sync(0xFFFFFFFFu, im, d);
        if (lane >= d) ip += yp, im += ym;
    }
    if (lane == 31) s_wp[warp] = ip, s_wm[warp] = im;
    __syncthreads();
    uint32_t op = 0, om = 0, tp = 0, tm2 = 0;
    for (int w = 0; w < 8; w++) {
        if (w < warp) op += s_wp[w], om += s_wm[w];
        tp += s_wp[w], tm2 += s_wm[w];
    }
    uint32_t at = op + ip - cp, total = om + im - cm;  // first piece index / first match index of this thread's segments
    Piece* pc = pieces + B.piece_off;
    uint32_t* ps = piece_start + B.piece_off;
    for (int k = k0; k < min(k0 + 16, n); k++) {
        if (!ma[k]) continue;
        const uint32_t nk = desc[k].n, bg = s_begin[k];
        if (nk > bg) {
            Piece p;
            p.spec = 1, p.seg = (uint32_t)k, p.begin = bg, p.end = nk;
            pc[at] = p;
            ps[at] = total;
            at++;
            total += nk - bg;
        }
        if (desc[k].end == END_BLOCK) {
            s_anchor = (uint32_t)desc[k].fin.anchor;  // the list ends here
            continue;
        }
        const Junction J = junc[k];
        if (J.status == J_OVERFLOW) continue;
        if (J.fix_n) {
            Piece p;
            p.spec = 2, p.seg = (uint32_t)k, p.begin = 0, p.end = J.fix_n;
            pc[at] = p;
            ps[at] = total;
            at++;
            total += J.fix_n;
        }
        if (J.status == J_TERMINAL) s_anchor = (uint32_t)J.anchor;
    }
    __syncthreads();
    if (tid == 0) {
        PState S;
        S.np = s_over ? 0xFFFFFFFFu : tp;
        S.fix_n = 0;
        S.nmatch = tm2;
        S.final_anchor = (int32_t)s_anchor;
        S.m_total = S.mlen_total = S.lit_total = S.too_many = 0;
        ps[tp] = tm2;
        pst[b] = S;
    }
}
__global__ void __launch_bounds__(32) lzp_stitch_kernel(const uint8_t* __restrict__ in, const PBlock* __restrict__ blocks, const uint32_t* __restrict__ act_blocks, int extra,
                                                         const Rec* __restrict__ rec, const Match* __restrict__ logs, const SegDesc* __restrict__ desc, Match* __restrict__ fix,
                                                         Piece* __restrict__ pieces, uint32_t* __restrict__ piece_start, PState* __restrict__ pst) {
    const uint32_t b = act_blocks[blockIdx.x];
    if (threadIdx.x != 0 || pst[b].np != 0xFFFFFFFFu) return;  // only blocks the walk gave up on
    const PBlock B = blocks[b];
    PState S;
    S.np = S.fix_n = S.nmatch = 0;
    S.final_anchor = 0;
    S.m_total = S.mlen_total = S.lit_total = S.too_many = 0;
    const Params P = make_params(in, B, extra, rec);
    SegLogAt sl;
    sl.base = logs + (size_t)B.seg_base * SEG_CAP;
    Piece* pc = pieces + B.piece_off;
    S.np = stitch_block(P, (int)B.nsegs, desc + B.seg_base, sl, fix + B.match_off, pc, &S.fix_n, &S.final_anchor);
    uint32_t acc = 0;
    for (uint32_t p = 0; p < S.np; p++) {
        piece_start[B.piece_off + p] = acc;
        acc += pc[p].end - pc[p].begin;
    }
    piece_start[B.piece_off + S.np] = acc;
    S.nmatch = acc;
    pst[b] = S;
}

// ---- pass 3: flatten the pieces into the block's match list -------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) lzp_flatten_kernel(const PBlock* __restrict__ blocks, const uint32_t* __restrict__ act_blocks, const PState* __restrict__ pst,
                                                           const Piece* __restrict__ pieces, const uint32_t* __restrict__ piece_start, const Match* __restrict__ logs,
                                                           const Match* __restrict__ jfix, const Match* __restrict__ fix, Match* __restrict__ ml) {
    const uint32_t b = act_blocks[blockIdx.y];
    const PBlock& B = blocks[b];
    const PState& S = pst[b];
    const Piece* pc = pieces + B.piece_off;
    const uint32_t* ps = piece_start + B.piece_off;
    for (uint32_t t = blockIdx.x * 256 + threadIdx.x; t < S.nmatch; t += gridDim.x * 256) {
        uint32_t lo = 0, hi = S.np;  // last piece with start <= t
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (ps[mid] <= t) lo = mid;
            else hi = mid;
        }
        const Piece p = pc[lo];
        const uint32_t e = p.begin + (t - ps[lo]);
        ml[B.match_off + t] = p.spec == 1 ? logs[(size_t)(B.seg_base + p.seg) * SEG_CAP + e] : p.spec == 2 ? jfix[(size_t)(B.seg_base + p.seg) * JCAP + e] : fix[B.match_off + e];
    }
}

// ---- pass 4: emission -------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void match_context(const Match* __restrict__ ml, uint32_t t, int count, int& prev_anchor, int& r0, int& r1) {
    if (t >= 1) {
        const Match a = ml[t - 1];
        prev_anchor = (int)(a.start + a.len);
        r0 = (int)a.dist;
    } else {
        prev_anchor = 0;
        r0 = count;
    }
    r1 = t >= 2 ? (int)ml[t - 2].dist : count;
}
// block-wide exclusive scan of three 32-bit values over TILE threads; returns the tile totals through tot[]
__device__ __forceinline__ void tile_scan3(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t* sm /* 3 * 32 */, uint32_t tot[3]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t ia = a, ib = b, ic = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t xa = __shfl_up_sync(0xFFFFFFFFu, ia, d), xb = __shfl_up_sync(0xFFFFFFFFu, ib, d), xc = __shfl_up_sync(0xFFFFFFFFu, ic, d);
        if (lane >= d) ia += xa, ib += xb, ic += xc;
    }
    if (lane == 31) sm[warp] = ia, sm[32 + warp] = ib, sm[64 + warp] = ic;
    __syncthreads();
    if (warp == 0) {
        uint32_t wa = sm[lane], wb = sm[32 + lane], wc = sm[64 + lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t xa = __shfl_up_sync(0xFFFFFFFFu, wa, d), xb = __shfl_up_sync(0xFFFFFFFFu, wb, d), xc = __shfl_up_sync(0xFFFFFFFFu, wc, d);
            if (lane >= d) wa += xa, wb += xb, wc += xc;
        }
        sm[lane] = wa, sm[32 + lane] = wb, sm[64 + lane] = wc;
    }
    __syncthreads();
    const uint32_t oa = warp ? sm[warp - 1] : 0, ob = warp ? sm[32 + warp - 1] : 0, oc = warp ? sm[64 + warp - 1] : 0;
    tot[0] = sm[31], tot[1] = sm[63], tot[2] = sm[95];
    a = oa + ia - a;
    b = ob + ib - b;
    c = oc + ic - c;
    __syncthreads();
}
__global__ void __launch_bounds__(TILE) lzp_sizes_kernel(const PBlock* __restrict__ blocks, const PState* __restrict__ pst, const Match* __restrict__ ml_all,
                                                          uint32_t* __restrict__ tile_sums /* 4 per tile */) {
    __shared__ uint32_t sm[96];
    const int b = blockIdx.y;
    const PBlock& B = blocks[b];
    const uint32_t nm = pst[b].nmatch;
    if (blockIdx.x * TILE >= nm && blockIdx.x > 0) return;
    const Match* ml = ml_all + B.match_off;
    const uint32_t t = blockIdx.x * TILE + threadIdx.x;
    uint32_t a = 0, bb = 0, c = 0;
    bool too_many = false;
    if (t < nm) {
        int pa, r0, r1;
        match_context(ml, t, (int)B.count, pa, r0, r1);
        Sizes s;
        match_sizes(ml[t], pa, r0, r1, B.min_match, s, too_many);
        a = s.m_bytes, bb = s.mlen_bytes, c = s.lit_bytes;
    }
    const int any_too_many = __syncthreads_or(too_many ? 1 : 0);
    uint32_t tot[3];
    tile_scan3(a, bb, c, sm, tot);
    if (threadIdx.x == 0) {
        uint32_t* ts = tile_sums + 4 * (size_t)(B.tile_base + blockIdx.x);
        ts[0] = tot[0], ts[1] = tot[1], ts[2] = tot[2], ts[3] = (uint32_t)any_too_many;
    }
}
// one warp per block: exclusive scan of the tile sums, totals, the reference's two "no compression" tests, header
__global__ void __launch_bounds__(32) lzp_tilescan_kernel(const PBlock* __restrict__ blocks, int nblocks, const uint32_t* __restrict__ done, PState* __restrict__ pst,
                                                           uint32_t* __restrict__ tile_sums, uint8_t* __restrict__ out, LzResult* __restrict__ res) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const PBlock B = blocks[b];
    PState S = pst[b];
    LzResult r;
    r.status = 1;
    r.out_len = r.n_runs = r.lit_end = r.tk_n = r.m_n = r.mlen_n = 0;
    if (!B.active || !done[b]) {
        if (B.active) r.status = 3;  // no fixed point within MAX_ROUNDS: the caller parses this block serially
        if (lane == 0) res[b] = r;
        return;
    }
    const uint32_t ntiles = (S.nmatch + TILE - 1) / TILE;
    uint32_t ca = 0, cb = 0, cc = 0, bad = 0;
    for (uint32_t t0 = 0; t0 < ntiles; t0 += 32) {
        const uint32_t t = t0 + lane;
        uint32_t* ts = tile_sums + 4 * (size_t)(B.tile_base + t);
        uint32_t a = 0, bb = 0, c = 0;
        if (t < ntiles) a = ts[0], bb = ts[1], c = ts[2], bad |= ts[3];
        uint32_t ia = a, ib = bb, ic = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t xa = __shfl_up_sync(0xFFFFFFFFu, ia, d), xb = __shfl_up_sync(0xFFFFFFFFu, ib, d), xc = __shfl_up_sync(0xFFFFFFFFu, ic, d);
            if (lane >= d) ia += xa, ib += xb, ic += xc;
        }
        if (t < ntiles) ts[0] = ca + ia - a, ts[1] = cb + ib - bb, ts[2] = cc + ic - c;
        ca += __shfl_sync(0xFFFFFFFFu, ia, 31);
        cb += __shfl_sync(0xFFFFFFFFu, ib, 31);
        cc += __shfl_sync(0xFFFFFFFFu, ic, 31);
    }
    bad = __reduce_or_sync(0xFFFFFFFFu, bad);
    if (lane != 0) return;
    S.m_total = ca, S.mlen_total = cb, S.lit_total = cc, S.too_many = bad;
    const uint32_t count = B.count;
    const int lit_len = (int)count - S.final_anchor;
    const uint64_t dst_idx = 13ull + cc, tk_idx = S.nmatch, m_idx = ca;
    const uint64_t lit_end = dst_idx + (uint64_t)lit_len + (lit_len >= 7 ? (uint64_t)length_bytes(lit_len - 7) : 0ull);
    const uint64_t total = lit_end + (tk_idx + 1) + m_idx + cb;
    if (!bad && dst_idx + (uint64_t)lit_len + tk_idx + m_idx < count && total <= count - count / 100) {
        uint8_t* dst = out + B.dst_off;
        const uint32_t a = (uint32_t)lit_end, bb = (uint32_t)(tk_idx + 1), c = (uint32_t)m_idx;
        for (int i = 0; i < 4; i++) {
            dst[i] = (uint8_t)(a >> (8 * i));
            dst[4 + i] = (uint8_t)(bb >> (8 * i));
            dst[8 + i] = (uint8_t)(c >> (8 * i));
        }
        dst[12] = (uint8_t)B.flags;
        r.lit_end = a, r.tk_n = bb, r.m_n = c, r.mlen_n = cb;
        r.n_runs = S.nmatch + 1;
        if (total <= count - count / 100) {  // otherwise the reference declines after writing (:582-588): nothing is emitted here
            r.status = 0;
            r.out_len = (uint32_t)total;
        }
    }
    pst[b] = S;
    res[b] = r;
}
__global__ void __launch_bounds__(TILE) lzp_emit_kernel(const uint8_t* __restrict__ in, const PBlock* __restrict__ blocks, const PState* __restrict__ pst,
                                                         const Match* __restrict__ ml_all, const uint32_t* __restrict__ tile_sums, const LzResult* __restrict__ res,
                                                         uint8_t* __restrict__ out, LzRun* __restrict__ runs_all, uint32_t* __restrict__ long_runs,
                                                         uint32_t* __restrict__ long_n) {
    __shared__ uint32_t sm[96];
    const int b = blockIdx.y;
    const PBlock& B = blocks[b];
    const PState& S = pst[b];
    const LzResult R = res[b];
    if (R.status != 0) return;
    const uint32_t nm = S.nmatch;
    if (blockIdx.x * TILE > nm) return;  // tile blockIdx.x holds matches [x * TILE, ...) and, behind the last match, the final literals
    const Match* ml = ml_all + B.match_off;
    LzRun* runs = runs_all + B.match_off;
    uint8_t* dst = out + B.dst_off;
    const uint32_t t = blockIdx.x * TILE + threadIdx.x;
    uint32_t a = 0, bb = 0, c = 0;
    int pa = 0, r0 = 0, r1 = 0;
    Match m;
    m.start = m.len = m.dist = m.probe = 0;
    Sizes s;
    s.m_bytes = s.mlen_bytes = s.lit_bytes = 0;
    if (t < nm) {
        match_context(ml, t, (int)B.count, pa, r0, r1);
        m = ml[t];
        bool tm;
        match_sizes(m, pa, r0, r1, B.min_match, s, tm);
        a = s.m_bytes, bb = s.mlen_bytes, c = s.lit_bytes;
    }
    uint32_t tot[3];
    tile_scan3(a, bb, c, sm, tot);
    const uint32_t* ts = tile_sums + 4 * (size_t)(B.tile_base + blockIdx.x);
    const uint32_t has_tile = blockIdx.x * TILE < nm;
    const uint32_t m_at = (has_tile ? ts[0] : S.m_total) + a, mlen_at = (has_tile ? ts[1] : S.mlen_total) + bb, lit_at = 13u + (has_tile ? ts[2] : S.lit_total) + c;
    uint8_t* tk = dst + R.lit_end;
    uint8_t* mb = tk + R.tk_n;
    uint8_t* mlenb = mb + R.m_n;
    if (t < nm) {
        match_emit(m, pa, r0, r1, B.min_match, tk + t, mb + m_at, mlenb + mlen_at, dst + lit_at);
        const uint32_t lit_len = m.start - (uint32_t)pa;
        runs[t].src = (uint32_t)pa;
        runs[t].dst = lit_at + (s.lit_bytes - lit_len);
        runs[t].len = lit_len;
        if (lit_len > LONG_RUN) long_runs[B.long_off + atomicAdd(&long_n[b], 1u)] = t;
    } else if (t == nm) {  // final literals (:538-551)
        const int lit_len = (int)B.count - S.final_anchor;
        uint32_t at = lit_at;
        if (lit_len >= 7) {
            tk[t] = (uint8_t)(7 << 5);
            at += (uint32_t)emit_length(dst + at, lit_len - 7);
        } else {
            tk[t] = (uint8_t)(lit_len << 5);
        }
        runs[t].src = (uint32_t)S.final_anchor;
        runs[t].dst = at;
        runs[t].len = (uint32_t)lit_len;
        if ((uint32_t)lit_len > LONG_RUN) long_runs[B.long_off + atomicAdd(&long_n[b], 1u)] = t;
    }
}
// literal runs: warps of grid.x CTAs per block take runs round robin; long runs are cut into 4 KiB pieces over all warps
__global__ void __launch_bounds__(256) lzp_literals_kernel(const uint8_t* __restrict__ in, const PBlock* __restrict__ blocks, const LzResult* __restrict__ res,
                                                            const LzRun* __restrict__ runs_all, const uint32_t* __restrict__ long_runs,
                                                            const uint32_t* __restrict__ long_n, uint8_t* __restrict__ out) {
    const int b = blockIdx.y;
    const LzResult R = res[b];
    if (R.status != 0) return;
    const PBlock& B = blocks[b];
    const uint8_t* src = in + B.src_off;
    uint8_t* dst = out + B.dst_off;
    const LzRun* runs = runs_all + B.match_off;
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * 256 + threadIdx.x) >> 5, nwarps = (gridDim.x * 256) >> 5;
    for (uint32_t i = warp; i < R.n_runs; i += nwarps) {
        const LzRun run = runs[i];
        if (run.len > LONG_RUN) continue;  // long runs: second loop
        for (uint32_t k = lane; k < run.len; k += 32) dst[run.dst + k] = src[run.src + k];
    }
    const uint32_t nl = long_n[b];
    for (uint32_t i = 0; i < nl; i++) {
        const LzRun run = runs[long_runs[B.long_off + i]];
        for (uint32_t k0 = warp * 4096u; k0 < run.len; k0 += nwarps * 4096u) {
            const uint32_t k1 = min(k0 + 4096u, run.len);
            for (uint32_t k = k0 + lane; k < k1; k += 32) dst[run.dst + k] = src[run.src + k];
        }
    }
}

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

}  // namespace

cudaError_t lz_forward_parallel_sub(const uint8_t* d_in, uint8_t* d_out, const LzBlock* lb, uint32_t nblocks, bool extra, LzWorkspace& W, cudaStream_t stream,
                                    LzResult* res, LzHook* hook) {
    const int hash_bits = extra ? 19 : 16;
    std::vector<PBlock> pb(nblocks);
    std::vector<uint32_t> blk_of_chunk, blk_of_seg;
    uint64_t pos = 0, matches = 0;
    uint32_t segs = 0, pieces = 0, tiles = 0, longs = 0;
    for (uint32_t b = 0; b < nblocks; b++) {
        PBlock& B = pb[b];
        const uint32_t count = lb[b].len;
        B.src_off = lb[b].src_off;
        B.dst_off = lb[b].dst_off;
        B.count = count;
        B.active = count >= (uint32_t)MIN_BLOCK && lb[b].data_type != 9 /*DT_SMALL_ALPHABET*/;
        B.src_end = B.active ? count - 16 - 2 : 0;
        B.max_dist = MAX_DISTANCE2;
        B.flags = 1;
        if ((int)B.src_end < 4 * MAX_DISTANCE1) {
            B.max_dist = MAX_DISTANCE1;
            B.flags = 0;
        }
        B.min_match = lb[b].data_type == 6 /*DT_DNA*/ ? 6 : 4;
        B.flags |= (uint32_t)(((B.min_match - 2) & 7) << 1);
        B.npos = B.active ? (uint32_t)std::min<int64_t>((int64_t)count - 8, (int64_t)B.src_end + 2) : 0;
        B.pos_off = pos;
        const uint64_t padded = ((uint64_t)count + 1023) & ~1023ull;
        for (uint64_t c = 0; c < padded; c += 1024) blk_of_chunk.push_back(b);
        pos += padded;
        B.match_off = matches;
        matches += (uint64_t)count / 4 + 32;
        B.seg_base = segs;
        B.nsegs = B.active ? std::max<uint32_t>(1, (B.src_end + SEG - 1) / SEG) : 0;
        for (uint32_t k = 0; k < B.nsegs; k++) blk_of_seg.push_back(b);
        segs += B.nsegs;
        B.piece_off = pieces;
        pieces += 2 * B.nsegs + 8;
        B.tile_base = tiles;
        B.ntiles_cap = (uint32_t)((count / 4 + 32 + TILE - 1) / TILE) + 1;
        tiles += B.ntiles_cap;
        B.long_off = longs;
        B.pad = 0;
        longs += count / LONG_RUN + 2;
    }
    const uint64_t total = pos;
    if (total == 0 || segs == 0) {
        for (uint32_t b = 0; b < nblocks; b++) res[b] = LzResult{1, 0, 0, 0, 0, 0, 0};
        return cudaSuccess;
    }
    // ---- workspace layout
    size_t off = 0;
    auto take = [&](size_t bytes) {
        const size_t at = off;
        off = align256(off + bytes);
        return at;
    };
    const size_t o_pb = take(nblocks * sizeof(PBlock)), o_boc = take(blk_of_chunk.size() * 4), o_bos = take(blk_of_seg.size() * 4);
    const size_t o_keys_a = take(total * 4), o_keys_b = take(total * 4), o_vals_a = take(total * 4), o_vals_b = take(total * 4);
    const size_t o_rec = take(total * sizeof(Rec)), o_rec2 = take(total * sizeof(Rec)), o_vf = take(total * 4), o_vf2 = take(total * 4);
    const size_t o_done = take((size_t)nblocks * 4), o_changed = take((size_t)nblocks * 4), o_longn = take((size_t)nblocks * 4), o_long = take((size_t)longs * 4), o_logs = take((size_t)segs * SEG_CAP * sizeof(Match)), o_desc = take((size_t)segs * sizeof(SegDesc));
    const size_t o_fix = take(matches * sizeof(Match)), o_ml = take(matches * sizeof(Match)), o_runs = take(matches * sizeof(LzRun));
    const size_t o_pieces = take((size_t)pieces * sizeof(Piece)), o_pstart = take((size_t)pieces * 4), o_pst = take(nblocks * sizeof(PState));
    const size_t o_junc = take((size_t)segs * sizeof(Junction)), o_jfix = take((size_t)segs * JCAP * sizeof(Match));
    const size_t o_actc = take(blk_of_chunk.size() * 4), o_acts = take((size_t)segs * 4), o_actb = take((size_t)nblocks * 4), o_dirty = take((size_t)segs * 4), o_changed_seg = take((size_t)segs * 4);
    const size_t o_tiles = take((size_t)tiles * 16), o_res = take(nblocks * sizeof(LzResult));
    size_t cub_bytes = 0;
    {
        cub::DoubleBuffer<uint32_t> k(nullptr, nullptr), v(nullptr, nullptr);
        cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, k, v, (int)total, 0, 32);
    }
    const size_t o_cub = take(cub_bytes + 256);
    uint8_t* ws = W.ensure(off + 4096);
    if (!ws) return cudaErrorMemoryAllocation;
    // ---- host tables
    std::vector<uint8_t> host(o_keys_a);
    memcpy(host.data() + o_pb, pb.data(), nblocks * sizeof(PBlock));
    memcpy(host.data() + o_boc, blk_of_chunk.data(), blk_of_chunk.size() * 4);
    memcpy(host.data() + o_bos, blk_of_seg.data(), blk_of_seg.size() * 4);
    cudaError_t e = cudaMemcpyAsync(ws, host.data(), host.size(), cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
    e = cudaStreamSynchronize(stream);  // `host` goes out of scope at return; the copy is small
    if (e != cudaSuccess) return e;
    const PBlock* d_pb = (const PBlock*)(ws + o_pb);
    const uint32_t* d_boc = (const uint32_t*)(ws + o_boc);
    const uint32_t* d_bos = (const uint32_t*)(ws + o_bos);
    uint32_t *keys_a = (uint32_t*)(ws + o_keys_a), *keys_b = (uint32_t*)(ws + o_keys_b), *vals_a = (uint32_t*)(ws + o_vals_a), *vals_b = (uint32_t*)(ws + o_vals_b);
    Rec *d_rec = (Rec*)(ws + o_rec), *d_rec2 = (Rec*)(ws + o_rec2);
    uint32_t *d_vf = (uint32_t*)(ws + o_vf), *d_vf2 = (uint32_t*)(ws + o_vf2), *d_done = (uint32_t*)(ws + o_done), *d_changed = (uint32_t*)(ws + o_changed);
    Match *d_logs = (Match*)(ws + o_logs), *d_fix = (Match*)(ws + o_fix), *d_ml = (Match*)(ws + o_ml);
    SegDesc* d_desc = (SegDesc*)(ws + o_desc);
    LzRun* d_runs = (LzRun*)(ws + o_runs);
    Piece* d_pieces = (Piece*)(ws + o_pieces);
    uint32_t* d_pstart = (uint32_t*)(ws + o_pstart);
    PState* d_pst = (PState*)(ws + o_pst);
    uint32_t* d_tiles = (uint32_t*)(ws + o_tiles);
    uint32_t *d_longn = (uint32_t*)(ws + o_longn), *d_long = (uint32_t*)(ws + o_long);
    LzResult* d_res = (LzResult*)(ws + o_res);
    const uint32_t G = (uint32_t)((total + 255) / 256);
    int key_bits = hash_bits;
    while ((1u << (key_bits - hash_bits)) <= nblocks) key_bits++;  // block indices 0 .. nblocks (the last one: padding)
    // ---- passes
    cudaMemsetAsync(d_vf, 0, total * 4, stream);
    cudaMemsetAsync(ws + o_done, 0, o_longn + (size_t)nblocks * 4 - o_done, stream);  // done, changed, long run counters
    {
        LzHookScope hs(hook, "lz_hash");
        lzp_hash_kernel<<<G, 256, 0, stream>>>(d_in, d_pb, d_boc, extra ? 1 : 0, hash_bits, nblocks, keys_a, vals_a, total);
    }
    cub::DoubleBuffer<uint32_t> dk(keys_a, keys_b), dv(vals_a, vals_b);
    {
        LzHookScope hs(hook, "lz_sort");
        size_t tb = cub_bytes;
        e = cub::DeviceRadixSort::SortPairs(ws + o_cub, tb, dk, dv, (int)total, 0, std::min(32, key_bits), stream);
        if (e != cudaSuccess) return e;
    }
    {
        LzHookScope hs(hook, "lz_link");
        lzp_link_kernel<<<G, 256, 0, stream>>>(dk.Current(), dv.Current(), d_pb, hash_bits, nblocks, d_rec, total);
        lzp_info_kernel<<<G, 256, 0, stream>>>(d_in, d_pb, d_boc, d_rec, total);
    }
    Junction* d_junc = (Junction*)(ws + o_junc);
    Match* d_jfix = (Match*)(ws + o_jfix);
    uint32_t *d_actc = (uint32_t*)(ws + o_actc), *d_acts = (uint32_t*)(ws + o_acts), *d_actb = (uint32_t*)(ws + o_actb), *d_dirty = (uint32_t*)(ws + o_dirty), *d_chseg = (uint32_t*)(ws + o_changed_seg);
    cudaMemsetAsync(d_pst, 0, nblocks * sizeof(PState), stream);
    std::vector<uint32_t> h_changed(nblocks), h_done(nblocks, 0);
    // the passes of a round run over the chunks / segments / blocks that have not reached their fixed point yet
    std::vector<uint32_t> act_c, act_s, act_b;
    bool lists_stale = true;
    for (uint32_t b = 0; b < nblocks; b++)
        if (!pb[b].active) h_done[b] = 1;
    for (int round = 0; round < MAX_ROUNDS; round++) {
        if (lists_stale) {
            act_c.clear(), act_s.clear(), act_b.clear();
            for (uint32_t b = 0; b < nblocks; b++) {
                if (h_done[b]) continue;
                act_b.push_back(b);
                for (uint64_t c = pb[b].pos_off >> 10, ce = (pb[b].pos_off + pb[b].count + 1023) >> 10; c < ce; c++) act_c.push_back((uint32_t)c);
                for (uint32_t k = 0; k < pb[b].nsegs; k++) act_s.push_back(pb[b].seg_base + k);
            }
            if (act_b.empty()) break;
            // pageable source: the copies are staged before the call returns, the vectors may change afterwards
            if ((e = cudaMemcpyAsync(d_actc, act_c.data(), act_c.size() * 4, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
            if ((e = cudaMemcpyAsync(d_acts, act_s.data(), act_s.size() * 4, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
            if ((e = cudaMemcpyAsync(d_actb, act_b.data(), act_b.size() * 4, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
            lists_stale = false;
        }
        const uint32_t GA = (uint32_t)act_c.size() * 4, NS = (uint32_t)act_s.size(), NB = (uint32_t)act_b.size();
        const Rec* rec_r = d_rec;
        // dirty[s]: the candidates a segment's parse reads differ from the previous round's (round 0: everything is new)
        if (round == 0) cudaMemsetAsync(d_dirty, 0xFF, (size_t)segs * 4, stream);
        if (round > 0) {
            LzHookScope hs(hook, "lz_filter");
            cudaMemsetAsync(d_chseg, 0, (size_t)segs * 4, stream);
            lzp_filter_kernel<<<GA, 256, 0, stream>>>(d_in, d_pb, d_boc, d_actc, d_rec, d_vf, d_rec2, total, round == 1 ? 1 : 0, d_chseg);
            lzp_dirty_kernel<<<(NS + 127) / 128, 128, 0, stream>>>(d_pb, d_bos, d_acts, NS, d_desc, d_chseg, d_dirty);
            rec_r = d_rec2;
        }
        {
            LzHookScope hs(hook, round == 0 ? "lz_spec_r0" : (round == 1 ? "lz_spec_r1" : "lz_spec"));
            lzp_spec_kernel<<<(NS + 3) / 4, 128, 0, stream>>>(d_in, d_pb, d_bos, extra ? 1 : 0, d_acts, NS, rec_r, d_logs, d_desc, d_dirty);
        }
        {
            LzHookScope hs(hook, round == 0 ? "lz_stitch_r0" : (round == 1 ? "lz_stitch_r1" : "lz_stitch"));
            lzp_junction_kernel<<<(NS + 3) / 4, 128, 0, stream>>>(d_in, d_pb, d_bos, extra ? 1 : 0, d_acts, NS, rec_r, d_logs, d_desc, d_jfix, d_junc, d_dirty, round == 0 ? 1 : 0);
            lzp_walk_par_kernel<<<NB, 256, 0, stream>>>(d_pb, d_actb, d_desc, d_junc, d_pieces, d_pstart, d_pst);
            lzp_walk_kernel<<<NB, 256, 0, stream>>>(d_pb, d_actb, d_desc, d_junc, d_pieces, d_pstart, d_pst);
            lzp_stitch_kernel<<<NB, 32, 0, stream>>>(d_in, d_pb, d_actb, extra ? 1 : 0, rec_r, d_logs, d_desc, d_fix, d_pieces, d_pstart, d_pst);
        }
        {
            LzHookScope hs(hook, round == 0 ? "lz_derive_r0" : (round == 1 ? "lz_derive_r1" : "lz_derive"));
            lzp_flatten_kernel<<<dim3(64, NB), 256, 0, stream>>>(d_pb, d_actb, d_pst, d_pieces, d_pstart, d_logs, d_jfix, d_fix, d_ml);
            cudaMemsetAsync(d_changed, 0, (size_t)nblocks * 4, stream);
            lzp_derive_kernel<<<GA / 4, 256, 0, stream>>>(d_pb, d_boc, d_actc, d_pst, d_ml, d_vf, d_vf2, d_changed, total);
        }
        e = cudaMemcpyAsync(h_changed.data(), d_changed, (size_t)nblocks * 4, cudaMemcpyDeviceToHost, stream);
        if (e != cudaSuccess) return e;
        e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) return e;
        bool all = true;
        for (uint32_t b = 0; b < nblocks; b++) {
            if (!h_done[b] && !h_changed[b]) h_done[b] = 1, lists_stale = true;  // vf' == vf: this round's match list is the parse
            all = all && h_done[b];
        }
        if (all) break;
        std::swap(d_vf, d_vf2);
    }
    e = cudaMemcpyAsync(d_done, h_done.data(), (size_t)nblocks * 4, cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
    uint32_t max_tiles = 1;
    for (uint32_t b = 0; b < nblocks; b++) max_tiles = std::max(max_tiles, pb[b].ntiles_cap);
    {
        LzHookScope hs(hook, "lz_emit");
        lzp_sizes_kernel<<<dim3(max_tiles, nblocks), TILE, 0, stream>>>(d_pb, d_pst, d_ml, d_tiles);
        lzp_tilescan_kernel<<<nblocks, 32, 0, stream>>>(d_pb, (int)nblocks, d_done, d_pst, d_tiles, d_out, d_res);
        lzp_emit_kernel<<<dim3(max_tiles, nblocks), TILE, 0, stream>>>(d_in, d_pb, d_pst, d_ml, d_tiles, d_res, d_out, d_runs, d_long, d_longn);
        lzp_literals_kernel<<<dim3(16, nblocks), 256, 0, stream>>>(d_in, d_pb, d_res, d_runs, d_long, d_longn, d_out);
    }
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    e = cudaMemcpyAsync(res, d_res, nblocks * sizeof(LzResult), cudaMemcpyDeviceToHost, stream);
    if (e != cudaSuccess) return e;
    e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return e;
    return cudaSuccess;
}

// Host entry: LZ / LZX forward of a batch. blocks[b].len == 0 -> the block is skipped (status 1). res[b] as lz_parse_kernel + lz_gather_kernel
// leave it (status 0: transformed, out_len bytes at dst_off). ws / ws_bytes: device workspace, grown through `grow` (returns the new base).
cudaError_t lz_forward_parallel(const uint8_t* d_in, uint8_t* d_out, const std::vector<LzBlock>& lb, bool extra, LzWorkspace& W, cudaStream_t stream,
                                std::vector<LzResult>& res, LzHook* hook) {
    const uint32_t nblocks = (uint32_t)lb.size();
    res.assign(nblocks, LzResult{1, 0, 0, 0, 0, 0, 0});
    if (nblocks == 0) return cudaSuccess;
    const int hash_bits = extra ? 19 : 16;
    cudaError_t e = cudaSuccess;
    for (uint32_t b0 = 0; b0 < nblocks && e == cudaSuccess;) {  // sub-batches: block index bits + hash bits fit a 32-bit key, position space < 2^31
        uint32_t nb = 0;
        uint64_t total = 0;
        while (b0 + nb < nblocks && nb < (1u << (31 - hash_bits)) - 1) {
            const uint64_t add = ((uint64_t)lb[b0 + nb].len + 1023) & ~1023ull;
            if (nb > 0 && total + add > (1ull << 30)) break;
            total += add;
            nb++;
        }
        e = lz_forward_parallel_sub(d_in, d_out, lb.data() + b0, nb, extra, W, stream, res.data() + b0, hook);
        b0 += nb;
    }
    return e;
}


}  // namespace kz
