// Static rANS (kanzi "ANS0", order 0) on sm_90a: statistics + header, interleaved-state encode, header walk, decode.
//
// Reference semantics reproduced bit-exactly (paths relative to the reference's v2/ directory):
//   entropy/ANSRangeCodec.go:274-311  Write (chunking, <=32 byte raw rule handled by the caller)
//   entropy/ANSRangeCodec.go:408-427  rebuildStatistics      -> ans0_stats_kernel (histogram)
//   entropy/EntropyUtils.go:123-260   NormalizeFrequencies   -> ans0_stats_kernel (warp-parallel restatement)
//   entropy/ANSRangeCodec.go:171-270  updateFrequencies / encodeHeader + EntropyUtils.go:38-67 EncodeAlphabet
//   entropy/ANSRangeCodec.go:446-468  encSymbol.reset        -> packed 8-byte table entries
//   entropy/ANSRangeCodec.go:313-405  encodeSymbol / encodeChunk -> ans0_encode_kernel
//   entropy/ANSRangeCodec.go:605-710  decodeHeader           -> ans0_walk_kernel (skim) + ans0_tables_kernel (full)
//   entropy/ANSRangeCodec.go:846-957  decodeSymbol / decodeChunkV2 -> ans0_decode_kernel
//
// Parallel decomposition (the wire format pins it): the unit of independent work is one 16 KiB chunk whose four
// interleaved rANS states share one byte cursor. One THREAD owns one chunk (4-way ILP over the states, the cursor
// coupling is resolved with a prefix count of the four renormalisation flags), 32 chunks per warp, per-chunk tables
// in shared memory laid out bank-interleaved (lane l only ever touches bank l -> conflict free for arbitrary indices).
// Compressed bytes are read / written 16 bytes at a time per thread so that the L1 line throughput of the inherently
// uncoalesced per-chunk streams stays below the dependent-chain latency.
#include "kz_ans.cuh"
#include "kz_warp.cuh"

namespace kz {

// ------------------------------------------------------------------------------------------------------------
// statistics: one warp per chunk
// ------------------------------------------------------------------------------------------------------------

// encSymbol.reset (ANSRangeCodec.go:446-468). The per-symbol entry keeps only what depends on the chunk:
//   freq (13 bits, clamped to 2^lr - 1) | (invShift - 32) << 13 | bias << 17
//   (bias = cum, or cum + 2^lr - 1 when freq < 2; invShift - 32 = ceil(log2 freq) - 1, 0..11)
// The reciprocal invFreq depends on freq alone and comes from one table shared by all chunks (rcp_table_kernel).
// freq sits in the low bits so that e << (31 - lr + ...) style shifts drop the other fields for free.
static __device__ __forceinline__ uint32_t make_enc_entry(uint32_t cum, uint32_t freq, uint32_t lr) {
    const uint32_t fr = freq < (1u << lr) - 1u ? freq : (1u << lr) - 1u;
    const uint32_t bias = fr < 2 ? cum + (1u << lr) - 1u : cum;
    const uint32_t sh = 31u - (uint32_t)__clz((int)((fr - 1u) | 1u));
    return fr | (sh << 13) | (bias << 17);
}

__global__ void expand_chunks_kernel(const DecBlock* __restrict__ blocks, int nblocks, DecChunk* __restrict__ chunks) {
    const int b = blockIdx.y;
    if (b >= nblocks) return;
    const DecBlock blk = blocks[b];
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (blk.chunk_size == 0 || k >= blk.nchunks) return;
    DecChunk c;
    const uint64_t o = (uint64_t)k * blk.chunk_size;
    c.out_off = blk.out_off + o;
    c.end_bit = blk.end_bit;
    const uint64_t left = (uint64_t)blk.pre_len - o;
    c.out_len = left < blk.chunk_size ? (uint32_t)left : blk.chunk_size;
    c.block = (uint32_t)b;
    chunks[blk.chunk_base + k] = c;
}

// inv[f] for f in [0, 4096): the 32-bit fixed point reciprocal of :452-466 (Alverson)
__global__ void rcp_table_kernel(uint32_t* __restrict__ inv) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= 4096) return;
    uint32_t v = 0xFFFFFFFFu;
    if (f >= 2) {
        const uint32_t shift = 32u - (uint32_t)__clz((int)(f - 1));  // smallest shift with f <= 1 << shift
        v = (uint32_t)((((uint64_t)1 << (shift + 31)) + (uint64_t)(f - 1)) / (uint64_t)f);
    }
    inv[f] = v;
}

// grid: ceil(nchunks / STATS_WARPS) CTAs of STATS_WARPS warps
__global__ void __launch_bounds__(STATS_WARPS * 32) ans0_stats_kernel(const uint8_t* __restrict__ in, const ChunkIn* __restrict__ chunks, int nchunks,
                                                                       uint32_t* __restrict__ enc_tab, uint8_t* __restrict__ hdr,
                                                                       uint32_t* __restrict__ hdr_bits, uint32_t* __restrict__ asz_out) {
    __shared__ uint32_t s_hist[STATS_WARPS][8][256];  // 8 replicas per warp to spread same-address atomics
    __shared__ uint32_t s_hdr[STATS_WARPS][HDR_STRIDE / 4];
    __shared__ uint16_t s_rank[STATS_WARPS][256];  // freq-1 by alphabet rank
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * STATS_WARPS + warp;
    if (c >= nchunks) return;
    const ChunkIn ck = chunks[c];
    const uint8_t* src = in + ck.src_off;
    const uint32_t len = ck.len;
    for (int i = lane; i < HDR_STRIDE / 4; i += 32) s_hdr[warp][i] = 0;
    uint32_t f[8];
    warp_histogram(src, len, &s_hist[warp][0][0], lane, f);  // chunk starts are 16-byte aligned
    const uint32_t lr = 12;
    const int asz = warp_normalize(f, len, lr, lane);
    // cumulative frequencies in symbol order + table entries (updateFrequencies :187-203)
    uint32_t carry = 0;
    int rank_base = 0;
    uint32_t last_sym = 0;
    uint32_t* tab = enc_tab + (size_t)c * 256;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        uint32_t incl = warp_incl_scan(f[j], lane);
        uint32_t cum = carry + incl - f[j];
        uint32_t b = __ballot_sync(0xFFFFFFFFu, f[j] != 0);
        int rank = rank_base + __popc(b & ((1u << lane) - 1u));
        if (f[j] != 0) {
            tab[lane + 32 * j] = make_enc_entry(cum, f[j], lr);
            s_rank[warp][rank] = (uint16_t)(f[j] - 1);
        } else {
            tab[lane + 32 * j] = 0;
        }
        if (b) last_sym = 32u * j + (31u - (uint32_t)__clz((int)b));
        carry += __shfl_sync(0xFFFFFFFFu, incl, 31);
        rank_base += __popc(b);
    }
    __syncwarp();
    // header: 3 bits lr-8, alphabet, frequency groups (encodeHeader :216-270, EncodeAlphabet EntropyUtils.go:38-67)
    uint32_t* hw = s_hdr[warp];
    uint32_t pos = 0;
    if (lane == 0) smem_put_bits(hw, 0, lr - 8, 3);
    pos = 3;
    if (asz == 256) {
        pos += 2;  // '0','0'
    } else if (asz == 0) {
        if (lane == 0) smem_put_bits(hw, pos + 1, 1, 1);  // '0','1'
        pos += 2;
    } else {
        const uint32_t last_mask = last_sym >> 3;
        if (lane == 0) {
            smem_put_bits(hw, pos, 1, 1);
            smem_put_bits(hw, pos + 1, last_mask, 5);
        }
        pos += 6;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (f[j] != 0) {
                uint32_t s = (uint32_t)lane + 32u * j;
                smem_put_bits(hw, pos + 8 * (s >> 3) + (7 - (s & 7)), 1, 1);
            }
        }
        pos += 8 * (last_mask + 1);
    }
    if (asz > 1) {
        const int gs = asz < 64 ? 6 : 8;
        uint32_t llr = 3;
        while ((1u << llr) <= lr) llr++;
        const int ngroups = (asz - 1 + gs - 1) / gs;  // <= 32
        uint32_t log_max = 0, glen = 0;
        int first = 1 + lane * gs, count = 0;
        if (lane < ngroups) {
            count = asz - first < gs ? asz - first : gs;
            uint32_t mx = 0;
            for (int k = 0; k < count; k++) mx = max(mx, (uint32_t)s_rank[warp][first + k]);
            log_max = mx ? 32u - (uint32_t)__clz((int)mx) : 0u;
            glen = llr + (uint32_t)count * log_max;
        }
        uint32_t gincl = warp_incl_scan(glen, lane);
        uint32_t goff = pos + gincl - glen;
        if (lane < ngroups) {
            smem_put_bits(hw, goff, log_max, llr);
            if (log_max) {
                uint32_t p = goff + llr;
                for (int k = 0; k < count; k++, p += log_max) smem_put_bits(hw, p, s_rank[warp][first + k], log_max);
            }
        }
        pos += __shfl_sync(0xFFFFFFFFu, gincl, 31);
    }
    __syncwarp();
    uint32_t* gh = reinterpret_cast<uint32_t*>(hdr + (size_t)c * HDR_STRIDE);
    for (int i = lane; i < HDR_STRIDE / 4; i += 32) gh[i] = bswap32(hw[i]);
    if (lane == 0) {
        hdr_bits[c] = pos;
        asz_out[c] = (uint32_t)asz;
    }
}

// ------------------------------------------------------------------------------------------------------------
// encode (v2): FOUR lanes per chunk (lane k owns rANS state k), 8 chunks per warp, 64 chunks per 256-thread CTA.
//
// v1 (one thread per chunk) ran one warp per scheduler.
// Reference loop (ANSRangeCodec.go:347-352): the chunk is walked backwards four bytes at a time, state k takes byte
// 4g + 3 - k, a state that reaches xMax first emits its low 16 bits (low byte at buffer[n], high byte at buffer[n-1]);
// the states emit in the order st0, st1, st2, st3 towards lower addresses. Here
//   * the backward write cursor is resolved with one __ballot_sync per step (prefix count over the lower-numbered
//     states); every lane stores its 16-bit word into a 256-byte per-chunk ring in shared memory and complete
//     64-byte blocks are flushed to the chunk's scratch area with one 16-byte store per lane;
//   * input bytes arrive through a 64-byte per-chunk ring filled with cp.async three iterations ahead;
//   * per-chunk tables hold 4 bytes per symbol (freq, bias); the reciprocals come from one 16 KiB table per CTA.
// 64 chunks x 1344 bytes + 16 KiB = 100 KiB per CTA -> 2 CTAs = 128 chunks per SM (one wave for 64 x 4 MiB).
// ------------------------------------------------------------------------------------------------------------
struct EncLane {
    uint32_t st;
    uint32_t emitted;  // 16-bit words emitted so far by the whole group
};

// The table entry and the reciprocal of a symbol do not depend on the rANS state: the caller loads them for the four
// symbols of an iteration up front (enc_fetch), so that the state chain of a step is compare / select / multiply only and
// never waits on shared memory (v2 loaded them inside the step, behind the ring store's compiler barrier).
KZ_D void enc_fetch(uint32_t sym, const uint32_t* tab, const uint32_t* rcp, uint32_t& e, uint32_t& inv) {
    e = tab[sym * 8];
    inv = rcp[e & 0x1FFFu];
}

template <bool ALL_ACTIVE>
KZ_D void enc_step(EncLane& L, uint32_t e, uint32_t inv, uint32_t out_ring, uint32_t lr, uint32_t lo_mask, uint32_t grp_mask, bool active) {
    const uint32_t freq = e & 0x1FFFu;
    const uint32_t sh = (e >> 13) & 15u;  // invShift - 32
    bool emit = L.st >= (freq << (31u - lr));                             // xMax = ((ANS_TOP >> lr) << 16) * freq
    if (!ALL_ACTIVE) emit = emit && active;
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, emit);
    // word index counted from the end of the stream: states with a lower index emit first (higher addresses)
    const uint32_t u = L.emitted + __popc(bal & lo_mask);
    const uint32_t addr = out_ring + ((0u - 2u * (u + 1u)) & (4 * ENC_OUT_RING_WORDS - 1));
    const uint32_t w16 = __byte_perm(L.st, 0, 0x4401);  // memory order [hi, lo] (:322-326)
    // predicated store: no divergent branch inside the step, so the four states stay converged for the ballot
    asm volatile("{ .reg .pred p; setp.ne.u32 p, %2, 0; @p st.shared.u16 [%0], %1; }" ::"r"(addr), "r"(w16), "r"((uint32_t)emit) : "memory");
    const uint32_t x = emit ? (L.st >> 16) : L.st;
    const uint32_t q = __umulhi(x, inv) >> sh;  // (st * invFreq) >> invShift
    const uint32_t nst = x + (e >> 17) + q * ((1u << lr) - freq);
    if (ALL_ACTIVE || active) {
        L.st = nst;
        L.emitted += __popc(bal & grp_mask);
    }
}

__global__ void __launch_bounds__(256, 2) ans0_encode_kernel(const uint8_t* __restrict__ in, const ChunkIn* __restrict__ chunks, int nchunks,
                                                             const uint32_t* __restrict__ enc_tab, const uint32_t* __restrict__ rcp_g,
                                                             uint8_t* __restrict__ hdr, const uint32_t* __restrict__ hdr_bits,
                                                             const uint32_t* __restrict__ asz_in, uint8_t* __restrict__ pay,
                                                             uint64_t* __restrict__ seg_src, uint64_t* __restrict__ seg_bits,
                                                             const uint32_t* __restrict__ seg_index) {
    extern __shared__ uint32_t s_enc[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, k = lane & 3;
    uint32_t* rcp = s_enc;                                  // 4096 words
    uint32_t* wbase = s_enc + 4096 + warp * ENC_WARP_WORDS;
    uint32_t* tab = wbase + g;                              // entry of symbol s at tab[s*8]
    uint32_t* oring = wbase + 256 * 8 + g * ENC_OUT_RING_WORDS;
    uint32_t* iring = wbase + 256 * 8 + 8 * ENC_OUT_RING_WORDS + g * 16;
    for (int i = tid; i < 4096; i += 256) rcp[i] = __ldg(rcp_g + i);
    const int cbase = blockIdx.x * ENC_CTA_CHUNKS + warp * 8;
    for (int cc = 0; cc < 8; cc++) {  // cooperative, coalesced table load
        const int c2 = cbase + cc;
        if (c2 >= nchunks) break;
        const uint32_t* t = enc_tab + (size_t)c2 * 256;
#pragma unroll
        for (int j = 0; j < 8; j++) wbase[(lane + 32 * j) * 8 + cc] = __ldg(t + lane + 32 * j);
    }
    __syncthreads();
    const int c = cbase + g;
    const uint32_t grp_mask = 0xFu << (lane & ~3);
    const uint32_t lo_mask = grp_mask & ((1u << lane) - 1u);  // lanes of my group with a lower state index (they emit first)
    const uint32_t lr = 12;
    // ---- per chunk set-up
    uint32_t len = 0, end4 = 0, asz = 0, hb = 0, si = 0;
    const uint8_t* src = in;
    uint8_t* e_words = pay;
    uint8_t* my_hdr = hdr;
    bool mode = false;
    if (c < nchunks) {
        const ChunkIn ck = chunks[c];
        src = in + ck.src_off;
        len = ck.len;
        end4 = len & ~3u;
        asz = asz_in[c];
        hb = hdr_bits[c];
        si = seg_index[c];
        my_hdr = hdr + (size_t)c * HDR_STRIDE;
        e_words = pay + (size_t)c * PAY_STRIDE + PAY_WORDS_END;
        mode = asz > 1;
        if (k == 0) {
            seg_src[si] = (uint64_t)(uintptr_t)my_hdr;
            if (!mode) {  // Write :303: chunk not encoded, header only
                seg_bits[si] = hb;
                seg_src[si + 1] = 0;
                seg_bits[si + 1] = 0;
            } else {
                for (uint32_t i = end4; i < len; i++) e_words[i - end4] = src[i];  // tail bytes go last in the stream (:339-342)
            }
        }
    }
    EncLane L;
    L.st = ANS_TOP;
    L.emitted = 0;
    uint32_t ngroups = mode ? (end4 >> 2) : 0;  // groups of 4 bytes, processed from the last to the first
    const uint32_t oring_a = smem_u32(oring), iring_a = smem_u32(iring);
    // ---- leading groups so that the rest is a whole number of 16-byte units (only tail chunks of a block)
    {
        uint32_t lead = ngroups & 3;
        uint32_t lead_max = lead;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) lead_max = max(lead_max, __shfl_xor_sync(0xFFFFFFFFu, lead_max, d));
        for (uint32_t r = 0; r < lead_max; r++) {
            const bool active = r < lead;
            uint32_t sym = 0;
            if (active) sym = src[(size_t)(ngroups - 1 - r) * 4 + (3 - k)];
            uint32_t e, inv;
            enc_fetch(sym, tab, rcp, e, inv);
            enc_step<false>(L, e, inv, oring_a, lr, lo_mask, grp_mask, active);
        }
        ngroups -= lead;
    }
    const uint32_t units = ngroups >> 2;  // 16-byte units still to encode: units-1 down to 0
    uint32_t max_units = units, min_units = units;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        max_units = max(max_units, __shfl_xor_sync(0xFFFFFFFFu, max_units, d));
        min_units = min(min_units, __shfl_xor_sync(0xFFFFFFFFu, min_units, d));
    }
    // input ring: unit q lives in slot q & 3; lane k copies 4 of its 16 bytes
    auto fetch = [&](int64_t q) {
        const bool ok = mode && q >= 0 && q < (int64_t)units;
        const uint8_t* p = src + (ok ? (size_t)q * 16 + 4 * k : 0);
        const uint32_t a = iring_a + (((uint32_t)q & 3u) << 4) + 4u * k;
        if (ok) asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(a), "l"(p) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    uint32_t flushed = 0;  // 64-byte blocks already written to the scratch area
    auto flush = [&]() {   // every 4 steps (at most 32 new bytes): write out a completed 64-byte block of the ring
        __syncwarp();
        if (mode && 2u * L.emitted >= 64u * (flushed + 1u)) {
            const uint32_t ro = (0u - 64u * (flushed + 1u)) & (4 * ENC_OUT_RING_WORDS - 1);
            const uint4 v = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(oring) + ro + 16 * k);
            *reinterpret_cast<uint4*>(e_words - 64 * (size_t)(flushed + 1) + 16 * k) = v;
            flushed++;
        }
        __syncwarp();
    };
    fetch((int64_t)units - 1);
    fetch((int64_t)units - 2);
    fetch((int64_t)units - 3);
    uint32_t it = 0;
    for (; it < max_units; it++) {
        const int64_t q = (int64_t)units - 1 - it;  // negative for groups that have finished
        const bool active = q >= 0;
        asm volatile("cp.async.wait_group 2;" ::: "memory");
        __syncwarp();
        const uint32_t slot = iring_a + (((uint32_t)q & 3u) << 4) + (3u - k);
        uint32_t s3, s2, s1, s0;
        asm volatile("ld.shared.u8 %0, [%1+12];" : "=r"(s3) : "r"(slot));
        asm volatile("ld.shared.u8 %0, [%1+8];" : "=r"(s2) : "r"(slot));
        asm volatile("ld.shared.u8 %0, [%1+4];" : "=r"(s1) : "r"(slot));
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(s0) : "r"(slot));
        uint32_t e3, e2, e1, e0, i3, i2, i1, i0;
        enc_fetch(s3 & 0xFF, tab, rcp, e3, i3);
        enc_fetch(s2 & 0xFF, tab, rcp, e2, i2);
        enc_fetch(s1 & 0xFF, tab, rcp, e1, i1);
        enc_fetch(s0 & 0xFF, tab, rcp, e0, i0);
        if (it < min_units) {
            enc_step<true>(L, e3, i3, oring_a, lr, lo_mask, grp_mask, true);
            enc_step<true>(L, e2, i2, oring_a, lr, lo_mask, grp_mask, true);
            enc_step<true>(L, e1, i1, oring_a, lr, lo_mask, grp_mask, true);
            enc_step<true>(L, e0, i0, oring_a, lr, lo_mask, grp_mask, true);
        } else {
            enc_step<false>(L, e3, i3, oring_a, lr, lo_mask, grp_mask, active);
            enc_step<false>(L, e2, i2, oring_a, lr, lo_mask, grp_mask, active);
            enc_step<false>(L, e1, i1, oring_a, lr, lo_mask, grp_mask, active);
            enc_step<false>(L, e0, i0, oring_a, lr, lo_mask, grp_mask, active);
        }
        flush();
        fetch(q - 3);
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    // ---- epilogue: the bytes not yet flushed (< 64), chunk size, final states (:390-404)
    const uint32_t total = 2u * L.emitted;  // bytes of 16-bit words
    if (mode) {
        const uint32_t done = 64u * flushed;
        const uint8_t* rb = reinterpret_cast<const uint8_t*>(oring);
        for (uint32_t o = done + k; o < total; o += 4) e_words[-(int64_t)o - 1] = rb[(0u - (o + 1u)) & (4 * ENC_OUT_RING_WORDS - 1)];
    }
    const uint32_t s0 = __shfl_sync(0xFFFFFFFFu, L.st, lane & ~3);
    const uint32_t s1 = __shfl_sync(0xFFFFFFFFu, L.st, (lane & ~3) + 1);
    const uint32_t s2 = __shfl_sync(0xFFFFFFFFu, L.st, (lane & ~3) + 2);
    const uint32_t s3 = __shfl_sync(0xFFFFFFFFu, L.st, (lane & ~3) + 3);
    if (mode && k == 0) {
        const uint32_t sz = total + (len - end4);
        BitWriter bw(my_hdr, hb);
        bw.write_varint(sz);
        bw.write(s0, 32);
        bw.write(s1, 32);
        bw.write(s2, 32);
        bw.write(s3, 32);
        seg_bits[si] = bw.pos;
        seg_src[si + 1] = (uint64_t)(uintptr_t)(e_words - total);
        seg_bits[si + 1] = 8ull * sz;
    }
}

// ------------------------------------------------------------------------------------------------------------
// decode side: header walk (one thread per block) and chunk decode (one thread per chunk)
// ------------------------------------------------------------------------------------------------------------
// Skims one alphabet + frequency table (decodeHeader :626-680 without storing anything). Returns alphabet size,
// or -1 on malformed input.
KZ_D int skim_one_table(BitReader& br, uint32_t lr, uint32_t llr) {
    int asz;
    if (br.read(1) == 0) {
        asz = br.read(1) ? 0 : 256;
    } else {
        uint32_t last = br.read(5);
        asz = 0;
        for (uint32_t i = 0; i <= last; i++) asz += __popc(br.read(8));
    }
    if (asz <= 1) return asz;
    const int gs = asz < 64 ? 6 : 8;
    for (int i = 1; i < asz; i += gs) {
        uint32_t log_max = br.read(llr);
        if ((1u << log_max) > (1u << lr)) return -1;
        int n = asz - i < gs ? asz - i : gs;
        br.skip((uint64_t)n * log_max);
    }
    return asz;
}

__global__ void ans_walk_kernel(const uint32_t* __restrict__ words, const DecBlock* __restrict__ blocks, int nblocks, int order,
                                uint64_t* __restrict__ chunk_hdr_bit, uint64_t* __restrict__ blk_end, int32_t* __restrict__ status) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const DecBlock blk = blocks[b];
    if (blk.nchunks == 0) return;
    const uint32_t chunk_size = order ? (ANS0_CHUNK << 8) : ANS0_CHUNK;
    BitReader br(words, blk.data_bit, blk.end_bit);
    uint32_t remaining = blk.pre_len;
    int32_t st = 0;
    for (uint32_t k = 0; k < blk.nchunks; k++) {
        chunk_hdr_bit[blk.chunk_base + k] = br.pos;
        if (st) continue;  // descriptors of the remaining chunks point at the failure position; decode is skipped
        const uint32_t clen = remaining < chunk_size ? remaining : chunk_size;
        remaining -= clen;
        const uint32_t lr = 8 + br.read(3);
        uint32_t llr = 3;
        while ((1u << llr) <= lr) llr++;
        int total = 0;
        const int dim = order ? 256 : 1;
        for (int ctx = 0; ctx < dim; ctx++) {
            int a = skim_one_table(br, lr, llr);
            if (a < 0) {
                st = -KZ_E_PROCESS_BLOCK;
                break;
            }
            total += a;
        }
        if (st == 0 && total == 0) st = -KZ_E_PROCESS_BLOCK;
        if (st == 0 && lr > (order ? 11u : 12u)) st = -KZ_E_INVALID_CODEC;  // tables sized for the encoder's fixed ranges
        if (st == 0 && (order == 1 || total > 1)) {
            uint32_t sz = br.read_varint();
            if (sz >= (uint32_t)ANS_MAX_CHUNK) st = -KZ_E_PROCESS_BLOCK;
            br.skip(128 + 8ull * sz);
        }
        if (br.overrun && st == 0) st = -KZ_E_PROCESS_BLOCK;
    }
    blk_end[b] = br.pos;
    if (st) status[b] = st;
}

// ------------------------------------------------------------------------------------------------------------
// header walk v3 (order 0): one WARP per block. The chunk headers of a block form a serial chain (chunk k+1 starts
// where chunk k's payload ends, at an arbitrary bit), so the walk is latency bound: 256 links per 4 MiB block.
//   v2 staged a 512-byte window per link with a register load + byte swap (29 % of the samples waited on that load)
//   and chased the <= 32 frequency-group length fields with ~20 instructions and two data-dependent branches each.
//   v3 * keeps two 2 KiB windows of RAW stream bytes in shared memory, filled by cp.async (no register staging): while
//        link k is parsed, the window around the PREDICTED start of link k+1 (start of k + length of k-1) is already
//        in flight; only a misprediction (> ~700 bytes off) pays a synchronous load;
//      * chases the group lengths branch free (error flags accumulate, trip count known up front, unrolled);
//      * counts the alphabet with one popc per lane + redux.
// A header is at most 3+6+256 + 32*(4+8*15) = 4233 bits (lr <= 15 on corrupt input) + 5 varint bytes: a link that
// starts no later than WALK_WIN - WALK_NEED bytes into a window never reads outside it.
// ------------------------------------------------------------------------------------------------------------
static const int WALK_WIN = 2048;   // bytes per window
static const int WALK_NEED = 560;   // bytes a header can span (incl. read slack)
static const int WALK_BACK = 736;   // bytes kept before the predicted position

KZ_D void walk_fetch(uint32_t smem_base, const uint8_t* bytes, uint64_t nbytes, uint64_t base, int lane) {
    const uint32_t o = (uint32_t)lane * 16u;
    const uint8_t* src = bytes + base + o;
    if (base + WALK_WIN <= nbytes) {  // uniform: whole window readable
#pragma unroll
        for (int j = 0; j < WALK_WIN / 512; j++)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_base + o + 512u * j), "l"(src + 512 * j) : "memory");
    } else {  // end of the stream: 16-byte units that are not entirely readable are zero filled
#pragma unroll
        for (int j = 0; j < WALK_WIN / 512; j++) {
            const bool ok = base + o + 512u * j + 16u <= nbytes;
            const uint32_t sz = ok ? 16u : 0u;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_base + o + 512u * j), "l"(ok ? src + 512 * j : bytes), "r"(sz)
                         : "memory");
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

__global__ void __launch_bounds__(32) ans0_walk_kernel(const uint32_t* __restrict__ words, uint64_t words_len, const DecBlock* __restrict__ blocks,
                                                        int nblocks, uint64_t* __restrict__ chunk_hdr_bit, uint64_t* __restrict__ blk_end,
                                                        int32_t* __restrict__ status) {
    __shared__ __align__(16) uint32_t s_win[2][WALK_WIN / 4 + 4];
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const DecBlock blk = blocks[b];
    if (blk.nchunks == 0) return;
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(words);
    const uint64_t nbytes = words_len * 4;
    if (lane < 8) s_win[lane >> 2][WALK_WIN / 4 + (lane & 3)] = 0;
    uint64_t pos = blk.data_bit;
    uint32_t remaining = blk.pre_len;
    int32_t st = 0;
    uint64_t prev_bits = 0;
    // window `c` is the candidate for the current link, window `o` receives the prefetch for the next one
    uint32_t* win = s_win[0];
    uint32_t* win_o = s_win[1];
    uint64_t base_c = (pos >> 3) & ~15ull, base_o = ~0ull >> 1;  // byte offset of each window (multiple of 16)
    walk_fetch(smem_u32(win), bytes, nbytes, base_c, lane);
    for (uint32_t k = 0; k < blk.nchunks; k++) {
        if (lane == 0) chunk_hdr_bit[blk.chunk_base + k] = pos;
        if (st) continue;
        const uint32_t clen = remaining < (uint32_t)ANS0_CHUNK ? remaining : (uint32_t)ANS0_CHUNK;
        remaining -= clen;
        // ---- make sure a window covers this link
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();
        const uint64_t pbyte = pos >> 3;
        if (!(pbyte >= base_c && pbyte - base_c <= (uint64_t)(WALK_WIN - WALK_NEED))) {
            base_c = pbyte & ~15ull;
            walk_fetch(smem_u32(win), bytes, nbytes, base_c, lane);
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncwarp();
        }
        // ---- start fetching the window of the next link at its predicted position
        if (prev_bits && k + 1 < blk.nchunks) {
            const uint64_t pred = (pos + prev_bits) >> 3;
            base_o = (pred > (uint64_t)WALK_BACK ? pred - WALK_BACK : 0) & ~15ull;
            walk_fetch(smem_u32(win_o), bytes, nbytes, base_o, lane);
        }
        uint32_t q = (uint32_t)(pos - (base_c << 3));
        auto sbits = [&](uint32_t at, uint32_t n) -> uint32_t {  // n in 1..32, window relative bit position
            const uint32_t w = at >> 5, o = at & 31;
            return __funnelshift_l(bswap32(win[w + 1]), bswap32(win[w]), o) >> (32 - n);
        };
        const uint32_t h = sbits(q, 10);
        const uint32_t lr = 8 + (h >> 7);
        const uint32_t llr = 32u - (uint32_t)__clz((int)lr);  // smallest llr >= 3 with (1 << llr) > lr, lr in 8..15
        q += 3;
        int asz;
        if (((h >> 6) & 1) == 0) {
            asz = ((h >> 5) & 1) ? 0 : 256;
            q += 2;
        } else {
            const uint32_t last = (h >> 1) & 31;
            q += 6;
            const uint32_t cnt = (uint32_t)lane <= last ? (uint32_t)__popc(sbits(q + 8 * lane, 8)) : 0u;
            asz = (int)__reduce_add_sync(0xFFFFFFFFu, cnt);
            q += 8 * (last + 1);
        }
        if (asz == 0) st = -KZ_E_PROCESS_BLOCK;
        if (st == 0 && lr > 12) st = -KZ_E_INVALID_CODEC;  // decode tables are sized for the encoder's fixed range (<= 12)
        if (st == 0 && asz > 1) {
            const uint32_t gs = asz < 64 ? 6 : 8;
            const uint32_t ngroups = ((uint32_t)asz - 2u + gs) / gs;  // >= 1
            const uint32_t last_n = (uint32_t)asz - 1u - (ngroups - 1u) * gs;
            uint32_t max_log = 0;
#pragma unroll 4
            for (uint32_t i = 0; i + 1 < ngroups; i++) {
                const uint32_t log_max = sbits(q, llr);
                max_log = max(max_log, log_max);
                q += llr + gs * log_max;
            }
            {
                const uint32_t log_max = sbits(q, llr);
                max_log = max(max_log, log_max);
                q += llr + last_n * log_max;
            }
            if (max_log > lr) st = -KZ_E_PROCESS_BLOCK;
            // varint (EntropyUtils.go:278-296): at most 5 bytes
            const uint32_t v4 = sbits(q, 32), v1 = sbits(q + 32, 8);
            uint32_t sz = (v4 >> 24) & 0x7F, nb = 1;
            if (v4 & 0x80000000u) {
                sz |= ((v4 >> 16) & 0x7F) << 7, nb = 2;
                if (v4 & 0x00800000u) {
                    sz |= ((v4 >> 8) & 0x7F) << 14, nb = 3;
                    if (v4 & 0x00008000u) {
                        sz |= (v4 & 0x7F) << 21, nb = 4;
                        if (v4 & 0x00000080u) sz |= (v1 & 0x0F) << 28, nb = 5;
                    }
                }
            }
            q += 8 * nb;
            if (st == 0) {
                if (sz >= (uint32_t)ANS_MAX_CHUNK) st = -KZ_E_PROCESS_BLOCK;
                const uint64_t next = (base_c << 3) + q + 128 + 8ull * sz;
                prev_bits = next - pos;
                pos = next;
            }
        } else if (st == 0) {
            const uint64_t next = (base_c << 3) + q;
            prev_bits = next - pos;
            pos = next;
        }
        if (st == 0 && pos > blk.end_bit) st = -KZ_E_PROCESS_BLOCK;
        {  // the prefetched window (if any) is the candidate for the next link
            uint32_t* t = win;
            win = win_o;
            win_o = t;
            const uint64_t tb = base_c;
            base_c = base_o;
            base_o = tb;
        }
        __syncwarp();
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    if (lane == 0) {
        blk_end[b] = pos;
        if (st) status[b] = st;
    }
}

// ------------------------------------------------------------------------------------------------------------
// decode: ans0_walk_kernel locates the chunk headers, ans0_tables_kernel turns each header into a table record, and
// ans0_decode_kernel runs the rANS chains. FOUR lanes per chunk (lane k owns rANS state k), 8 chunks per warp, 16 chunks
// per 64-thread CTA, 7 CTAs x 16 = 112 chunks per SM: the 16384 chunks of 64 x 4 MiB need 147 SMs for a single wave
// (H100: 132, so a short second wave).
//   * bucket word = start flags of 24 slots in bits 0..23 | (symbols started before the bucket - 1) << 24, bucket 0
//     stores its flags without slot 0: symbol index = (b >> 24) + popc(b & ((2 << r) - 1)) needs no masking and the
//     byte address of the symbol entry is one IMAD after the POPC; the bucket index is one IMAD.HI
//     (slot / 24 = umulhi(slot, ceil(2^32 / 24)));
//   * symbol entry = freq << 20 | cum << 8 | sym: the frequency is one shift away from the multiply;
//   * table word w of chunk g lives at (w * 8 + g): the 8 chunks of a warp own disjoint groups of 4 banks;
//   * every chunk's 256-byte payload ring is 256-byte aligned in the shared window: ring addresses are one LOP3
//     ((pos & 0xFE) | base);
//   * the shared byte cursor is resolved with one __ballot_sync per step (order st3, st2, st1, st0,
//     ANSRangeCodec.go:904-917) and the renormalisation word is read with two ld.shared.u16, branch free;
//   * the ring is refilled with cp.async (no register destination) and a round is consumed one iteration after it was
//     issued, so no step waits on a load issued in the same iteration;
//   * the decoded bytes are transposed across the 4 lanes with two shuffles per 4 steps, 16 bytes stored per chunk.
// Warp region (bytes): 8 rings x 256 | 171 x 8 bucket words | 256 x 8 symbol words | pad to a multiple of 256.
// ------------------------------------------------------------------------------------------------------------
static const int RING_WORDS = 64;  // 32-bit words per chunk ring (256 bytes)

struct DecLane {
    uint32_t st;      // rANS state of this lane
    uint32_t cur2;    // byte offset of the cursor inside the (unwrapped) ring coordinate system, always even
    uint32_t acc;     // last 4 decoded symbols of this state
};

// The ring holds RAW stream bytes (filled with cp.async, no register staging); the payload starts s16 bits into the
// 16-bit unit at ring byte 0 + cur2, so a renormalisation word is the 16 bits at bit offset s16 of the 4 bytes at cur2.
template <bool ALL_ACTIVE>
KZ_D void dec_step(DecLane& L, uint32_t bm_base, uint32_t sym_base, uint32_t ring_base, uint32_t mask, uint32_t lr, uint32_t rsh, uint32_t hi_mask,
                   uint32_t grp_mask, bool active) {
    const uint32_t st = L.st;
    const uint32_t slot = st & mask;
    const uint32_t w = __umulhi(slot, 178956971u);  // slot / 24, exact for slot < 2^16
    uint32_t b, e;
    asm("ld.shared.u32 %0, [%1];" : "=r"(b) : "r"(bm_base + w * 32u));
    const uint32_t r = slot - 24u * w;
    const uint32_t p = (uint32_t)__popc(b & ((2u << r) - 1u));
    const uint32_t ea = (b >> 24) * 32u + sym_base;
    asm("ld.shared.u32 %0, [%1];" : "=r"(e) : "r"(ea + p * 32u));
    const uint32_t nst = (e >> 20) * (st >> lr) + (slot - ((e >> 8) & 0xFFFu));  // D(x) (ANSRangeCodec.go:849)
    bool need = nst < (uint32_t)ANS_TOP;
    if (!ALL_ACTIVE) need = need && active;
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, need);
    const uint32_t t2 = L.cur2 + 2u * (uint32_t)__popc(bal & hi_mask);
    uint32_t va, vb;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(va) : "r"((t2 & 0xFEu) | ring_base));
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(vb) : "r"(((t2 + 2u) & 0xFEu) | ring_base));
    const uint32_t x = __byte_perm(va, vb, 0x0145) >> rsh;  // big-endian 32 bits at t2, renormalisation word in the low 16 bits
    const uint32_t nst2 = __byte_perm(x, nst, 0x5410);      // (nst << 16) | (x & 0xFFFF)
    if (ALL_ACTIVE || active) {
        L.st = need ? nst2 : nst;
        L.cur2 += 2u * (uint32_t)__popc(bal & grp_mask);
    }
    L.acc = __byte_perm(L.acc, e, 0x4321);  // acc = (acc >> 8) | (sym << 24)
}

// ------------------------------------------------------------------------------------------------------------
// decode tables: one WARP per chunk parses the header from a shared-memory window (alphabet by popc/prefix sums, group
// lengths chased by lane 0, frequencies extracted group-parallel, cumulative frequencies by a warp scan, start flags by
// shared-memory atomics) and writes a DEC_TAB_WORDS record per chunk: 171 bucket words | 256 symbol entries | lr, mode, steps, tail, payload begin /
// end bit, 4 states. ans0_decode_kernel only copies the records (cp.async) into its interleaved layout.
// Chunks whose alphabet has a single symbol are filled here (Read :737-741) and need no decode.
// ------------------------------------------------------------------------------------------------------------
static const int TAB_WIN_WORDS = 160;  // 3 + 6 + 256 + 32 x 124 bits of header + 40 bits varint + 128 bits states + slack

__global__ void __launch_bounds__(128) ans0_tables_kernel(const uint32_t* __restrict__ words, uint64_t words_len, const DecChunk* __restrict__ chunks,
                                                          int nchunks, const uint64_t* __restrict__ chunk_hdr_bit, uint32_t* __restrict__ tabs,
                                                          uint8_t* __restrict__ out, int32_t* __restrict__ status) {
    __shared__ uint32_t s_win[4][TAB_WIN_WORDS + 2];
    __shared__ uint32_t s_bm[4][192];
    __shared__ uint16_t s_freq[4][256];
    __shared__ uint8_t s_sym[4][256];
    __shared__ uint16_t s_goff[4][32];
    __shared__ uint8_t s_glog[4][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * 4 + warp;
    if (c >= nchunks) return;
    uint32_t* rec = tabs + (size_t)c * DEC_TAB_WORDS;
    uint32_t* meta = rec + DEC_BM_WORDS + 256;
    const DecChunk ck = chunks[c];
    if (lane == 0) meta[1] = 0;  // mode: nothing to decode unless everything below checks out
    if (status[ck.block] != 0) return;
    const uint64_t hbit = chunk_hdr_bit[c];
    const uint64_t w0 = hbit >> 5;
    uint32_t* win = s_win[warp];
    for (int i = lane; i < TAB_WIN_WORDS + 2; i += 32) win[i] = w0 + i < words_len ? bswap32(__ldg(words + w0 + i)) : 0u;
    for (int i = lane; i < 192; i += 32) s_bm[warp][i] = 0;
    __syncwarp();
    auto rd = [&](uint32_t at, uint32_t n) -> uint32_t {  // n in 1..32 bits at window relative position `at`
        const uint32_t w = at >> 5, o = at & 31;
        return __funnelshift_l(win[w + 1], win[w], o) >> (32 - n);
    };
    const uint64_t room = ck.end_bit > hbit ? ck.end_bit - hbit : 0;  // bits of the block that follow the header start
    uint32_t q = (uint32_t)(hbit & 31);
    const uint32_t q0 = q;
    const uint32_t lr = 8 + rd(q, 3);
    q += 3;
    const uint32_t scale = 1u << lr;
    const uint32_t llr = 32u - (uint32_t)__clz((int)lr);  // smallest llr >= 3 with (1 << llr) > lr, lr in 8..15
    int asz = 0;
    if (rd(q, 1) == 0) {
        asz = rd(q + 1, 1) ? 0 : 256;
        q += 2;
        for (int i = lane; i < 256; i += 32) s_sym[warp][i] = (uint8_t)i;
    } else {
        const uint32_t last = rd(q + 1, 5);
        q += 6;
        const uint32_t m = (uint32_t)lane <= last ? rd(q + 8 * lane, 8) : 0u;
        const uint32_t pc = (uint32_t)__popc(m);
        uint32_t incl = pc;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= d) incl += t;
        }
        uint32_t r = incl - pc, mm = m;
        while (mm) {
            const int j = __ffs((int)mm) - 1;
            mm &= mm - 1;
            s_sym[warp][r++] = (uint8_t)(8 * lane + j);
        }
        asz = (int)__shfl_sync(0xFFFFFFFFu, incl, 31);
        q += 8 * (last + 1);
    }
    __syncwarp();
    if (asz == 0 || lr > 12) {
        if (lane == 0) atomicCAS(&status[ck.block], 0, asz == 0 ? -KZ_E_PROCESS_BLOCK : -KZ_E_INVALID_CODEC);
        return;
    }
    if (asz == 1) {  // Read :737-741: the chunk is one repeated symbol, nothing else is read
        if ((uint64_t)(q - q0) > room) {
            if (lane == 0) atomicCAS(&status[ck.block], 0, -KZ_E_PROCESS_BLOCK);
            return;
        }
        const uint32_t v = s_sym[warp][0] * 0x01010101u;
        uint8_t* dst = out + ck.out_off;  // 16-byte aligned
        const uint32_t n16 = ck.out_len >> 4;
        for (uint32_t i = lane; i < n16; i += 32) reinterpret_cast<uint4*>(dst)[i] = make_uint4(v, v, v, v);
        for (uint32_t i = (n16 << 4) + lane; i < ck.out_len; i += 32) dst[i] = (uint8_t)v;
        return;
    }
    // ---- frequency groups: lane 0 chases the group offsets (serial by format), every lane extracts one group
    const uint32_t gs = asz < 64 ? 6 : 8;
    const uint32_t ngroups = ((uint32_t)asz - 2u + gs) / gs;  // 1..32
    uint32_t bad = 0;
    if (lane == 0) {
        uint32_t p = q;
        for (uint32_t g = 0; g < ngroups; g++) {
            const uint32_t log_max = rd(p, llr);
            const uint32_t cnt = min(gs, (uint32_t)asz - 1u - g * gs);
            s_goff[warp][g] = (uint16_t)(p + llr);
            s_glog[warp][g] = (uint8_t)log_max;
            if ((1u << log_max) > scale) bad = 1;
            p += llr + cnt * log_max;
        }
        q = p;
    }
    q = __shfl_sync(0xFFFFFFFFu, q, 0);
    __syncwarp();
    uint32_t part = 0;
    if ((uint32_t)lane < ngroups) {
        const uint32_t log_max = s_glog[warp][lane];
        const uint32_t first = 1 + lane * gs;
        const uint32_t cnt = min(gs, (uint32_t)asz - first);
        uint32_t p = s_goff[warp][lane];
        for (uint32_t k2 = 0; k2 < cnt; k2++, p += log_max) {
            uint32_t f = 1;
            if (log_max > 0 && log_max <= 15) {
                f = 1 + rd(p, log_max);
                if (f >= scale) bad = 1;
            }
            s_freq[warp][first + k2] = (uint16_t)f;
            part += f;
        }
    }
    const uint32_t sum = __reduce_add_sync(0xFFFFFFFFu, part);
    if (scale <= sum) bad = 1;
    // size of the payload and the four states (ANSRangeCodec.go:726-733, :866-886)
    uint32_t sz = 0, nb = 0;
    {
        const uint32_t v4 = rd(q, 32), v1 = rd(q + 32, 8);
        sz = (v4 >> 24) & 0x7F, nb = 1;
        if (v4 & 0x80000000u) {
            sz |= ((v4 >> 16) & 0x7F) << 7, nb = 2;
            if (v4 & 0x00800000u) {
                sz |= ((v4 >> 8) & 0x7F) << 14, nb = 3;
                if (v4 & 0x00008000u) {
                    sz |= (v4 & 0x7F) << 21, nb = 4;
                    if (v4 & 0x00000080u) sz |= (v1 & 0x0F) << 28, nb = 5;
                }
            }
        }
    }
    q += 8 * nb;
    const uint32_t st_k = rd(q + 32 * (lane & 3), 32);
    q += 128;
    if (sz >= (uint32_t)ANS_MAX_CHUNK || (uint64_t)(q - q0) + 8ull * sz > room) bad = 1;
    bad = __ballot_sync(0xFFFFFFFFu, bad != 0) ? 1u : 0u;
    if (bad) {
        if (lane == 0) atomicCAS(&status[ck.block], 0, -KZ_E_PROCESS_BLOCK);
        return;
    }
    if (lane == 0) s_freq[warp][0] = (uint16_t)(scale - sum);
    __syncwarp();
    // ---- cumulative frequencies (lane l owns ranks 8 l .. 8 l + 7), symbol entries, start flags
    uint32_t f8[8], tot = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int r = lane * 8 + j;
        f8[j] = r < asz ? s_freq[warp][r] : 0u;
        tot += f8[j];
    }
    uint32_t incl = tot;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= d) incl += t;
    }
    uint32_t cum = incl - tot;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int r = lane * 8 + j;
        uint32_t e = 0;
        if (r < asz) {
            e = (f8[j] << 20) | (cum << 8) | s_sym[warp][r];
            if (cum) atomicOr(&s_bm[warp][cum / 24], 1u << (cum % 24));  // slot 0 always starts symbol 0: its flag is implied
        }
        rec[DEC_BM_WORDS + r] = e;
        cum += f8[j];
    }
    __syncwarp();
    // symbols started before each bucket, minus one (6 buckets per lane)
    uint32_t b6[6], pc6 = 0;
#pragma unroll
    for (int j = 0; j < 6; j++) {
        b6[j] = s_bm[warp][lane * 6 + j];
        pc6 += (uint32_t)__popc(b6[j]);
    }
    uint32_t inc2 = pc6;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, inc2, d);
        if (lane >= d) inc2 += t;
    }
    uint32_t running = inc2 - pc6;
#pragma unroll
    for (int j = 0; j < 6; j++) {
        const int w = lane * 6 + j;
        if (w < DEC_BM_WORDS) rec[w] = b6[j] | (running << 24);
        running += (uint32_t)__popc(b6[j]);
    }
    // ---- meta
    const uint64_t pb = hbit + (q - q0);
    const uint64_t pe = pb + 8ull * sz;
    if (lane < 4) meta[8 + lane] = st_k;
    if (lane == 0) {
        meta[0] = lr;
        meta[2] = ck.out_len >> 2;
        meta[3] = ck.out_len & 3;
        meta[4] = (uint32_t)pb;
        meta[5] = (uint32_t)(pb >> 32);
        meta[6] = (uint32_t)pe;
        meta[7] = (uint32_t)(pe >> 32);
        __threadfence_block();
        meta[1] = 1;
    }
}

__global__ void __launch_bounds__(64, 7) ans0_decode_kernel(const uint32_t* __restrict__ words, uint64_t words_len /*in 32-bit words*/, const uint32_t* __restrict__ tabs,
                                                             const DecChunk* __restrict__ chunks, int nchunks,
                                                             const uint64_t* __restrict__ chunk_hdr_bit, uint8_t* __restrict__ out,
                                                             int32_t* __restrict__ status) {
    extern __shared__ __align__(256) uint32_t s_dec[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, k = lane & 3;  // chunk slot inside the warp, state index
    // the rings must be 256-byte aligned in the shared window (DEC_SMEM carries 256 bytes of slack for this)
    uint32_t* s_al = s_dec + (((0u - smem_u32(s_dec)) & 255u) >> 2);
    uint32_t* wbase = s_al + warp * DEC_WARP_WORDS;
    uint32_t* ring = wbase + g * RING_WORDS;
    uint32_t* bm = wbase + 8 * RING_WORDS + g;                       // bucket w at bm[w*8]
    uint32_t* symtab = wbase + 8 * RING_WORDS + DEC_BM_WORDS * 8 + g;  // entry i at symtab[i*8]
    const int c = blockIdx.x * DEC_CTA_CHUNKS + warp * 8 + g;
    const uint32_t grp_mask = 0xFu << (lane & ~3);
    const uint32_t hi_mask = grp_mask & ~((2u << lane) - 1u);  // lanes of my group with a higher state index (they read first)

    // ---- per-chunk set-up: the tables were built by ans0_tables_kernel; the warp copies its 8 records into the
    // interleaved shared-memory layout (lane l moves word (l >> 3) + 4 j of chunk l & 7: conflict-free stores)
    {
        const int cg = blockIdx.x * DEC_CTA_CHUNKS + warp * 8 + (lane & 7);
        if (cg < nchunks) {
            const uint32_t* rec = tabs + (size_t)cg * DEC_TAB_WORDS;
            const uint32_t dst0 = smem_u32(wbase + 8 * RING_WORDS) + 4u * (uint32_t)(lane & 7);
            for (int i = lane >> 3; i < DEC_BM_WORDS + 256; i += 4)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst0 + 32u * (uint32_t)i), "l"(rec + i) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    uint32_t lr = 12, nsteps = 0, tail = 0;
    uint64_t pb = 0, pe = 0;
    uint8_t* dst = nullptr;
    int mode = 0;  // 0 = nothing to do, 1 = rANS decode
    DecLane L;
    L.st = 0;
    L.acc = 0;
    if (c < nchunks) {
        const uint32_t* meta = tabs + (size_t)c * DEC_TAB_WORDS + DEC_BM_WORDS + 256;
        mode = (int)__ldg(meta + 1);
        if (mode) {
            lr = __ldg(meta);
            nsteps = __ldg(meta + 2);
            tail = __ldg(meta + 3);
            pb = (uint64_t)__ldg(meta + 4) | ((uint64_t)__ldg(meta + 5) << 32);
            pe = (uint64_t)__ldg(meta + 6) | ((uint64_t)__ldg(meta + 7) << 32);
            L.st = __ldg(meta + 8 + k);
            dst = out + chunks[c].out_off;
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    uint32_t max_steps = nsteps, min_steps = nsteps;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        max_steps = max(max_steps, __shfl_xor_sync(0xFFFFFFFFu, max_steps, d));
        min_steps = min(min_steps, __shfl_xor_sync(0xFFFFFFFFu, min_steps, d));
    }
    if (max_steps == 0) return;

    // ---- payload ring: raw copy of the stream starting at the 16-byte aligned block that holds the first payload bit.
    // Ring byte r <-> source byte base_b + r. Round n copies source bytes [base_b + 64 n, +64): lane k its 16-byte unit.
    // A unit is copied when it starts before the end of the payload and lies inside the stream buffer, otherwise it is
    // zero filled (the guard past the payload, :888-893): the first `left` rounds of this lane copy, the others fill.
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(words);
    const uint64_t base_b = (pb >> 3) & ~15ull;            // source byte of ring byte 0
    const uint32_t rel = (uint32_t)(pb - 8 * base_b);      // payload bit offset inside the ring, 0..134
    const uint32_t rsh = 16u - (rel & 15u);                // see dec_step
    const uint64_t end_b = (pe + 7) >> 3;                  // first source byte past the payload
    const uint64_t lim_b = words_len * 4;
    const uint64_t lim_u = lim_b >= 15 ? lim_b - 15 : 0;   // units must start below this to be entirely readable
    const uint64_t stop_b = end_b < lim_u ? end_b : lim_u;
    const uint64_t first_u = base_b + 16u * k;
    int32_t left = (mode && stop_b > first_u) ? (int32_t)((stop_b - first_u + 63) >> 6) : 0;
    const uint8_t* src = bytes + first_u;
    const uint32_t ring_base = smem_u32(ring);
    const uint32_t unit_base = ring_base | (16u * k);
    uint32_t fill = 0;  // ring byte offset (unwrapped, multiple of 64) of the next refill round
    L.cur2 = 2u * (rel >> 4);
    auto issue = [&]() {
        const bool ok = left > 0;
        const uint8_t* s = ok ? src : bytes;
        const uint32_t src_size = ok ? 16u : 0u;  // src-size 0 zero-fills
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(unit_base | (fill & 0xC0u)), "l"(s), "r"(src_size) : "memory");
        src += 64;
        fill += 64;
        left--;
    };
    if (mode) {
#pragma unroll 1
        for (int r = 0; r < 4; r++) issue();  // initial fill: the whole ring
    } else {
        fill = 0x40000000u;  // never refills
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    const uint32_t mask = (1u << lr) - 1u;
    const uint32_t bm_base = smem_u32(bm), sym_base = smem_u32(symtab);

    // 4x4 byte transpose inside the group: after 4 steps lane k holds [a_k0 a_k1 a_k2 a_k3] (a_kj = symbol of state k in
    // step j, output position 4j + 3 - k); lane j stores the word of step j: [a_3j a_2j a_1j a_0j].
    auto transpose = [&](uint32_t acc) -> uint32_t {
        const uint32_t o2 = __shfl_xor_sync(0xFFFFFFFFu, acc, 2);
        const uint32_t t1 = (k & 2) ? __byte_perm(acc, o2, 0x3276) : __byte_perm(acc, o2, 0x5410);
        const uint32_t o1 = __shfl_xor_sync(0xFFFFFFFFu, t1, 1);
        return (k & 1) ? __byte_perm(t1, o1, 0x5173) : __byte_perm(t1, o1, 0x0426);
    };
    auto maintain = [&]() {  // every 4 steps, uniform for the warp
        asm volatile("cp.async.wait_group 0;" ::: "memory");  // the round issued one iteration ago has landed
        __syncwarp();
        // refill when at most 160 bytes are buffered ahead of the cursor: the new 64-byte round then only overwrites
        // consumed bytes (4 steps consume at most 32 bytes) and at least 128 buffered bytes remain while it is in flight
        if ((int32_t)(fill - L.cur2) <= (4 * RING_WORDS - 64 - 32)) issue();
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    const uint32_t fast_iters = min_steps >> 2;  // iterations in which every group of the warp is active
    uint32_t it = 0;
    uint8_t* dptr = dst + 4 * k;
    // 8 steps per ring check while every group is active. A check sees a gap (buffered bytes ahead of the cursor) g >= 66:
    // it starts at >= 240, drops by at most 64 per check while above 128, and never drops once it is refilled every time.
    // 8 steps consume at most 64 bytes and a consuming lane reads at most 4 bytes past its word: always inside landed data.
    for (; it + 2 <= fast_iters; it += 2) {
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        *reinterpret_cast<uint32_t*>(dptr) = transpose(L.acc);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        *reinterpret_cast<uint32_t*>(dptr + 16) = transpose(L.acc);
        dptr += 32;
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();
        if ((int32_t)(fill - L.cur2) <= 128) issue();
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    for (; it < fast_iters; it++) {
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        dec_step<true>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, true);
        *reinterpret_cast<uint32_t*>(dptr) = transpose(L.acc);
        dptr += 16;
        maintain();
    }
    const uint32_t all_iters = max_steps >> 2;
    for (; it < all_iters; it++) {  // groups with fewer steps idle here
        const bool active = (it * 4 + 3) < nsteps;
        dec_step<false>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, active);
        dec_step<false>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, active);
        dec_step<false>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, active);
        dec_step<false>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, active);
        const uint32_t w = transpose(L.acc);
        if (active) *reinterpret_cast<uint32_t*>(dptr) = w;
        dptr += 16;
        maintain();
    }
    {  // remaining 0..3 steps of a group (only the last chunk of a block can have nsteps % 4 != 0)
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();
        const uint32_t done = nsteps & ~3u;
        uint32_t rem_max = nsteps - done;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) rem_max = max(rem_max, __shfl_xor_sync(0xFFFFFFFFu, rem_max, d));
        for (uint32_t r = 0; r < rem_max; r++) {
            const bool active = done + r < nsteps;
            dec_step<false>(L, bm_base, sym_base, ring_base, mask, lr, rsh, hi_mask, grp_mask, active);
            if (active) dst[(size_t)(done + r) * 4 + (3 - k)] = (uint8_t)(L.acc >> 24);
        }
    }
    // tail bytes follow the consumed words (:951-954)
    if (mode && k == 0 && tail) {
        uint64_t pos = 8 * (base_b + L.cur2) + (rel & 15u);  // bit position of the cursor in the stream
        for (uint32_t j = 0; j < tail; j++, pos += 8) dst[(size_t)nsteps * 4 + j] = pos + 8 <= pe ? (uint8_t)bits_at(words, pos, 8) : 0;
    }
}

}  // namespace kz
