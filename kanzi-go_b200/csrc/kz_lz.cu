// LZ / LZX (kanzi's LZ77 with two repeat distances) on sm_90a — first correct CUDA path.
//
// Reference semantics reproduced bit-exactly (paths relative to the reference's v2/ directory):
//   transform/LZCodec.go:249-591 LZXCodec.Forward (hash :238-244, findMatchLZX :593-608, emitLengthLZ :193-213)
//   transform/LZCodec.go:621-778 inverseV6 (readLengthLZ :215-232), MaxEncodedLen :935-941
// `extra` selects LZX (19-bit hash table, lazy check at position + 2) versus LZ (16-bit table).
//
// The reference parse is a sequential greedy state machine (hash table contents, two repeat distances, the srcInc skip
// acceleration, lazy +1/+2 checks, backward extension): bit-exact output means replaying it exactly, so there is ONE
// serial chain per block and the only parallelism is across blocks. v1: lane 0 of one warp per block runs the parse
// against a per-block hash table in HBM/L2 and records tokens, distances, length bytes and one (source, destination,
// length) triple per literal run; the literal bytes and the final layout are then copied by all lanes / a wide kernel.
// Decode: lane 0 parses the token stream, all 32 lanes copy literals and matches (match byte i = dst[ref + i % dist]).
#include "kz_lz.cuh"

namespace kz {

namespace {

const uint64_t LZ_HASH_SEED = 0x1E35A7BDull;
const int LZ_MAX_DISTANCE1 = (1 << 16) - 2;
const int LZ_MAX_DISTANCE2 = (1 << 24) - 2;
const int LZ_MAX_MATCH = 65535 + 254 + 4;
const int LZ_MIN_BLOCK = 24;

// little-endian 64/32-bit loads at any byte offset of an 8-byte aligned buffer (the buffer has >= 16 bytes of slack)
KZ_D uint64_t ld64(const uint64_t* __restrict__ w, int p) {
    const int i = p >> 3, s = (p & 7) << 3;
    const uint64_t a = w[i];
    if (s == 0) return a;
    return (a >> s) | (w[i + 1] << (64 - s));
}
KZ_D uint32_t ld32(const uint64_t* __restrict__ w, int p) { return (uint32_t)ld64(w, p); }
KZ_D uint32_t lz_hash(uint64_t v, bool extra) {
    return extra ? (uint32_t)(((v << 24) * LZ_HASH_SEED) >> (64 - 19)) : (uint32_t)(((v << 24) * LZ_HASH_SEED) >> (64 - 16));
}
KZ_D int emit_length(uint8_t* block, int length) {
    if (length < 254) {
        block[0] = (uint8_t)length;
        return 1;
    }
    if (length < 65536 + 254) {
        length -= 254;
        block[0] = 254;
        block[1] = (uint8_t)(length >> 8);
        block[2] = (uint8_t)length;
        return 3;
    }
    length -= 255;
    block[0] = 255;
    block[1] = (uint8_t)(length >> 16);
    block[2] = (uint8_t)(length >> 8);
    block[3] = (uint8_t)length;
    return 4;
}
KZ_D int find_match(const uint64_t* __restrict__ w, int src_idx, int ref, int max_match) {
    int best = 0;
    while (best + 8 <= max_match) {
        const uint64_t diff = ld64(w, src_idx + best) ^ ld64(w, ref + best);
        if (diff != 0) {
            best += (__ffsll((long long)diff) - 1) >> 3;
            break;
        }
        best += 8;
    }
    return best;
}

}  // namespace

// One warp per block; lane 0 parses. res[b] = {status (0 ok / 1 skip), out_len, n_runs, lit_end, tk_n, m_n, mlen_n}
__global__ void __launch_bounds__(32) lz_parse_kernel(const uint8_t* __restrict__ in, const LzBlock* __restrict__ blocks, int nblocks, int extra,
                                                       int32_t* __restrict__ hashes_all, uint8_t* __restrict__ scratch_all, uint8_t* __restrict__ out,
                                                       LzResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const LzBlock blk = blocks[b];
    LzResult r;
    r.status = 1;
    r.out_len = 0;
    r.n_runs = 0;
    r.lit_end = 0;
    r.tk_n = r.m_n = r.mlen_n = 0;
    const int count = (int)blk.len;
    if (count < LZ_MIN_BLOCK || blk.data_type == 9 /*DT_SMALL_ALPHABET*/) {
        res[b] = r;
        return;
    }
    const uint8_t* src = in + blk.src_off;
    const uint64_t* w = reinterpret_cast<const uint64_t*>(src);
    uint8_t* dst = out + blk.dst_off;
    int32_t* hashes = hashes_all + ((size_t)b << (extra ? 19 : 16));
    uint8_t* scratch = scratch_all + blk.scratch_off;
    // scratch layout: tokens [count/4 + 64] | distances [3*count/4 + 64] | match length bytes [count + 64] | runs (12 bytes each)
    uint8_t* tk_buf = scratch;
    uint8_t* m_buf = tk_buf + (count / 4 + 64);
    uint8_t* mlen_buf = m_buf + (3 * (count / 4) + 64);
    LzRun* runs = reinterpret_cast<LzRun*>(scratch + (((size_t)(count / 4 + 64) + (3 * (size_t)(count / 4) + 64) + ((size_t)count + 64) + 15) & ~(size_t)15));
    const int src_end = count - 16 - 2;
    int max_dist = LZ_MAX_DISTANCE2;
    uint8_t flags = 1;
    if (src_end < 4 * LZ_MAX_DISTANCE1) {
        max_dist = LZ_MAX_DISTANCE1;
        flags = 0;
    }
    const int min_match = blk.data_type == 6 /*DT_DNA*/ ? 6 : 4;
    flags |= (uint8_t)(((min_match - 2) & 7) << 1);
    dst[12] = flags;
    const bool ex = extra != 0;
    int src_idx = 0, dst_idx = 13, anchor = 0, mlen_idx = 0, m_idx = 0, tk_idx = 0, n_runs = 0;
    int repd0 = count, repd1 = count, repd_idx = 0, src_inc = 0;
    bool too_many = false;
    while (src_idx < src_end) {
        int best_len = 0;
        const uint64_t p = ld64(w, src_idx);
        const uint32_t h0 = lz_hash(p, ex);
        const int ref0 = hashes[h0];
        hashes[h0] = src_idx;
        const int src_idx1 = src_idx + 1;
        const int max_match = min(src_end - src_idx1, LZ_MAX_MATCH);
        int ref = src_idx1 - (repd_idx ? repd1 : repd0);
        const int min_ref = max(src_idx - max_dist, 0);
        if (ref > min_ref && (uint32_t)(p >> 8) == ld32(w, ref)) {
            best_len = find_match(w, src_idx1, ref, max_match);
        } else {
            ref = src_idx1 - (repd_idx ? repd0 : repd1);
            if (ref > min_ref && (uint32_t)(p >> 8) == ld32(w, ref)) best_len = find_match(w, src_idx1, ref, max_match);
        }
        if (best_len < min_match) {
            ref = ref0;
            bool found = false;
            if (ref > min_ref && (uint32_t)p == ld32(w, ref)) {
                best_len = find_match(w, src_idx, ref, min(src_end - src_idx, LZ_MAX_MATCH));
                found = best_len >= min_match;
            }
            if (!found) {
                src_idx = src_idx1 + (src_inc >> 6);
                src_inc++;
                repd_idx = 0;
                continue;
            }
            if (ref != src_idx - repd0 && ref != src_idx - repd1) {
                const uint32_t h1 = lz_hash(ld64(w, src_idx1), ex);
                const int ref1 = hashes[h1];
                hashes[h1] = src_idx1;
                if (ref1 > min_ref + 1 && ld32(w, src_idx1 + best_len - 3) == ld32(w, ref1 + best_len - 3)) {
                    const int bl1 = find_match(w, src_idx1, ref1, max_match);
                    if (bl1 >= best_len) {
                        ref = ref1;
                        best_len = bl1;
                        src_idx = src_idx1;
                    }
                }
                if (ex) {
                    const int src_idx2 = src_idx1 + 1;
                    const uint32_t h2 = lz_hash(ld64(w, src_idx2), ex);
                    const int ref2 = hashes[h2];
                    hashes[h2] = src_idx2;
                    if (ref2 > min_ref + 2 && ld32(w, src_idx2 + best_len - 3) == ld32(w, ref2 + best_len - 3)) {
                        const int bl2 = find_match(w, src_idx2, ref2, min(src_end - src_idx2, LZ_MAX_MATCH));
                        if (bl2 >= best_len) {
                            ref = ref2;
                            best_len = bl2;
                            src_idx = src_idx2;
                        }
                    }
                }
            }
            while (src_idx > anchor && ref > min_ref && src[src_idx - 1] == src[ref - 1]) {
                best_len++;
                ref--;
                src_idx--;
            }
            if (best_len > LZ_MAX_MATCH) {
                src_idx += best_len - LZ_MAX_MATCH;
                ref += best_len - LZ_MAX_MATCH;
                best_len = LZ_MAX_MATCH;
            }
        } else {
            if (src[src_idx] == src[ref - 1] && best_len < LZ_MAX_MATCH) {
                best_len++;
                ref--;
            } else {
                src_idx++;
                hashes[lz_hash(ld64(w, src_idx), ex)] = src_idx;
            }
        }
        src_inc = 0;
        const int dist = src_idx - ref;
        const int m_len = best_len - min_match;
        int token, m_len_th;
        if (dist == repd0) {
            token = 0x00;
            m_len_th = 3;
        } else if (dist == repd1) {
            token = 0x04;
            m_len_th = 3;
        } else {
            m_len_th = 7;
            if (dist >= 256) {
                if (dist >= 65536) {
                    m_buf[m_idx] = (uint8_t)(dist >> 16);
                    m_buf[m_idx + 1] = (uint8_t)(dist >> 8);
                    m_idx += 2;
                    token = 0x18;
                } else {
                    m_buf[m_idx++] = (uint8_t)(dist >> 8);
                    token = 0x10;
                }
            } else {
                token = 0x08;
            }
            m_buf[m_idx++] = (uint8_t)dist;
        }
        if (m_len >= m_len_th) {
            token += m_len_th;
            mlen_idx += emit_length(mlen_buf + mlen_idx, m_len - m_len_th);
        } else {
            token += m_len;
        }
        repd1 = repd0;
        repd0 = dist;
        repd_idx = 1;
        const int lit_len = src_idx - anchor;
        if (lit_len == 0) {
            tk_buf[tk_idx++] = (uint8_t)token;
        } else {
            if (lit_len >= 7) {
                if (lit_len >= (1 << 24)) {
                    too_many = true;
                    break;
                }
                tk_buf[tk_idx++] = (uint8_t)((7 << 5) | token);
                dst_idx += emit_length(dst + dst_idx, lit_len - 7);
            } else {
                tk_buf[tk_idx++] = (uint8_t)((lit_len << 5) | token);
            }
            runs[n_runs].src = (uint32_t)anchor;
            runs[n_runs].dst = (uint32_t)dst_idx;
            runs[n_runs].len = (uint32_t)lit_len;
            n_runs++;
            dst_idx += lit_len;
        }
        anchor = src_idx + best_len;
        src_idx++;
        while (src_idx < anchor) {
            hashes[lz_hash(ld64(w, src_idx), ex)] = src_idx;
            src_idx++;
        }
    }
    if (!too_many) {
        const int lit_len = count - anchor;
        if (dst_idx + lit_len + tk_idx + m_idx < count) {
            if (lit_len >= 7) {
                tk_buf[tk_idx++] = (uint8_t)(7 << 5);
                dst_idx += emit_length(dst + dst_idx, lit_len - 7);
            } else {
                tk_buf[tk_idx++] = (uint8_t)(lit_len << 5);
            }
            runs[n_runs].src = (uint32_t)anchor;
            runs[n_runs].dst = (uint32_t)dst_idx;
            runs[n_runs].len = (uint32_t)lit_len;
            n_runs++;
            dst_idx += lit_len;
            const uint32_t a = (uint32_t)dst_idx, bb = (uint32_t)tk_idx, c = (uint32_t)m_idx;
            for (int i = 0; i < 4; i++) {
                dst[i] = (uint8_t)(a >> (8 * i));
                dst[4 + i] = (uint8_t)(bb >> (8 * i));
                dst[8 + i] = (uint8_t)(c >> (8 * i));
            }
            const int total = dst_idx + tk_idx + m_idx + mlen_idx;
            if (total <= count - count / 100) {
                r.status = 0;
                r.out_len = (uint32_t)total;
            }
            r.n_runs = (uint32_t)n_runs;
            r.lit_end = (uint32_t)dst_idx;
            r.tk_n = (uint32_t)tk_idx;
            r.m_n = (uint32_t)m_idx;
            r.mlen_n = (uint32_t)mlen_idx;
        }
    }
    res[b] = r;
}

// grid (nblocks, GATHER_CTAS): copies the literal runs and appends tokens | distances | length bytes
__global__ void __launch_bounds__(256) lz_gather_kernel(const uint8_t* __restrict__ in, const LzBlock* __restrict__ blocks, int nblocks,
                                                         const uint8_t* __restrict__ scratch_all, const LzResult* __restrict__ res, uint8_t* __restrict__ out) {
    const int b = blockIdx.x;
    if (b >= nblocks) return;
    const LzResult r = res[b];
    if (r.status != 0) return;
    const LzBlock blk = blocks[b];
    const int count = (int)blk.len;
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const uint8_t* scratch = scratch_all + blk.scratch_off;
    const uint8_t* tk_buf = scratch;
    const uint8_t* m_buf = tk_buf + (count / 4 + 64);
    const uint8_t* mlen_buf = m_buf + (3 * (count / 4) + 64);
    const LzRun* runs = reinterpret_cast<const LzRun*>(scratch + (((size_t)(count / 4 + 64) + (3 * (size_t)(count / 4) + 64) + ((size_t)count + 64) + 15) & ~(size_t)15));
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.y * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.y * blockDim.x) >> 5;
    for (uint32_t i = warp; i < r.n_runs; i += nwarps) {
        const LzRun run = runs[i];
        for (uint32_t k = lane; k < run.len; k += 32) dst[run.dst + k] = src[run.src + k];
    }
    const int tid = blockIdx.y * blockDim.x + threadIdx.x, nthreads = gridDim.y * blockDim.x;
    uint8_t* d2 = dst + r.lit_end;
    for (uint32_t i = tid; i < r.tk_n; i += nthreads) d2[i] = tk_buf[i];
    d2 += r.tk_n;
    for (uint32_t i = tid; i < r.m_n; i += nthreads) d2[i] = m_buf[i];
    d2 += r.m_n;
    for (uint32_t i = tid; i < r.mlen_n; i += nthreads) d2[i] = mlen_buf[i];
}

// One warp per block (inverseV6 :621-778). out_len[b] = decoded bytes, status[b] = 0 / -13.
__global__ void __launch_bounds__(32) lz_inverse_kernel(const uint8_t* __restrict__ in, const LzBlock* __restrict__ blocks, int nblocks, uint8_t* __restrict__ out,
                                                         uint32_t* __restrict__ out_len, int32_t* __restrict__ status) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const LzBlock blk = blocks[b];
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const long long count = blk.len, cap = blk.cap;
    int fail = 0;
    if (count < 13) fail = 1;
    long long tk_idx = 0, m_idx = 0, mlen_idx = 0, src_end = 0, src_idx = 13, dst_idx = 0;
    long long max_dist = 0, min_match = 0, repd0 = count, repd1 = count;
    if (!fail) {
        tk_idx = (uint32_t)src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24);
        m_idx = (uint32_t)src[4] | ((uint32_t)src[5] << 8) | ((uint32_t)src[6] << 16) | ((uint32_t)src[7] << 24);
        mlen_idx = (uint32_t)src[8] | ((uint32_t)src[9] << 8) | ((uint32_t)src[10] << 16) | ((uint32_t)src[11] << 24);
        m_idx += tk_idx;
        mlen_idx += m_idx;
        if (tk_idx > count || m_idx > count || mlen_idx > count) fail = 1;
        src_end = tk_idx - 13;
        max_dist = (src[12] & 1) ? LZ_MAX_DISTANCE2 : LZ_MAX_DISTANCE1;
        min_match = ((src[12] >> 1) & 7) + 2;
    }
    const long long dst_end = cap - 16;
    bool done = fail != 0;
    while (!done) {
        // ---- lane 0 parses one token
        long long lit_len = 0, lit_src = 0, m_len = 0, dist = 0;
        int st = 0;  // 0 = token with match, 1 = last token (literals only), 2 = failure
        if (lane == 0) {
            if (tk_idx >= count) {
                st = 2;
            } else {
                const int token = src[tk_idx++];
                bool brk = false;
                if (token >= 32) {
                    if (token >= 0xE0) {
                        long long v = -1;
                        if (src_idx < count) {
                            v = src[src_idx];
                            if (v < 254) src_idx += 1;
                            else if (v == 254 && src_idx + 3 <= count) { v += ((long long)src[src_idx + 1] << 8) + src[src_idx + 2]; src_idx += 3; }
                            else if (v == 255 && src_idx + 4 <= count) { v += ((long long)src[src_idx + 1] << 16) + ((long long)src[src_idx + 2] << 8) + src[src_idx + 3]; src_idx += 4; }
                            else v = -1;
                        }
                        if (v < 0) st = 2;
                        lit_len = 7 + v;
                    } else {
                        lit_len = token >> 5;
                    }
                    if (st == 0 && (src_idx + lit_len > count || dst_idx + lit_len > cap)) st = 2;
                    lit_src = src_idx;
                    if (st == 0) {
                        src_idx += lit_len;
                        if (src_idx >= src_end) brk = true;
                    }
                }
                if (st == 0 && brk) st = 1;
                if (st == 0) {
                    const int f = token & 0x18;
                    long long ml;
                    const bool rep = f == 0;
                    ml = rep ? (token & 3) : (token & 7);
                    if (ml == (rep ? 3 : 7)) {
                        long long v = -1;
                        if (mlen_idx < count) {
                            v = src[mlen_idx];
                            if (v < 254) mlen_idx += 1;
                            else if (v == 254 && mlen_idx + 3 <= count) { v += ((long long)src[mlen_idx + 1] << 8) + src[mlen_idx + 2]; mlen_idx += 3; }
                            else if (v == 255 && mlen_idx + 4 <= count) { v += ((long long)src[mlen_idx + 1] << 16) + ((long long)src[mlen_idx + 2] << 8) + src[mlen_idx + 3]; mlen_idx += 4; }
                            else v = -1;
                        }
                        if (v < 0) st = 2;
                        ml += min_match + v;
                    } else {
                        ml += min_match;
                    }
                    if (rep) {
                        dist = (token & 4) == 0 ? repd0 : repd1;
                    } else {
                        const int nb = f == 0x18 ? 3 : (f == 0x10 ? 2 : 1);
                        if (m_idx + nb > count) {
                            st = 2;
                        } else {
                            dist = src[m_idx++];
                            if (f >= 0x10) {
                                dist = (dist << 8) | src[m_idx++];
                                if (f == 0x18) dist = (dist << 8) | src[m_idx++];
                            }
                        }
                    }
                    repd1 = repd0;
                    repd0 = dist;
                    m_len = ml;
                    const long long m_end = dst_idx + lit_len + m_len;
                    const long long ref = dst_idx + lit_len - dist;
                    if (st == 0 && (ref < 0 || dist > max_dist || m_end > dst_end)) st = 2;  // dist 0 passes, as in the reference
                }
            }
        }
        st = __shfl_sync(0xFFFFFFFFu, st, 0);
        lit_len = __shfl_sync(0xFFFFFFFFu, lit_len, 0);
        lit_src = __shfl_sync(0xFFFFFFFFu, lit_src, 0);
        m_len = __shfl_sync(0xFFFFFFFFu, m_len, 0);
        dist = __shfl_sync(0xFFFFFFFFu, dist, 0);
        dst_idx = __shfl_sync(0xFFFFFFFFu, dst_idx, 0);
        if (st == 2) {
            fail = 1;
            break;
        }
        for (long long k = lane; k < lit_len; k += 32) dst[dst_idx + k] = src[lit_src + k];
        dst_idx += lit_len;
        if (st == 1) break;
        __syncwarp();
        const long long ref = dst_idx - dist;
        if (dist == 0) {
            // the reference copies every byte onto itself (LZCodec.go:762-764): the match keeps what the destination held
        } else if (dist >= m_len || dist >= 32) {
            // rounds of 32 bytes; a round only reads bytes written by earlier rounds when dist >= 32
            for (long long k0 = 0; k0 < m_len; k0 += 32) {
                const long long k = k0 + lane;
                uint8_t v = 0;
                if (k < m_len) v = dst[ref + k];
                __syncwarp();
                if (k < m_len) dst[dst_idx + k] = v;
                __syncwarp();
            }
        } else {
            for (long long k = lane; k < m_len; k += 32) dst[dst_idx + k] = dst[ref + (k % dist)];
        }
        dst_idx += m_len;
        __syncwarp();
    }
    if (lane == 0) {
        if (!fail && src_idx != src_end + 13) fail = 1;
        out_len[b] = fail ? 0u : (uint32_t)dst_idx;
        status[b] = fail ? -KZ_E_PROCESS_BLOCK : 0;
    }
}

}  // namespace kz
