// Zero run length transform (kanzi ZRLT) on sm_90a.
//
// Reference: transform/ZRLT.go:58-141 (Forward), :146-225 (Inverse).
//   forward: a run of z zeros becomes the binary digits of z + 1 without the leading one, one digit per byte (values 0/1);
//            any other byte b becomes b + 1, except 0xFE/0xFF which become 0xFF, b - 0xFE. The output may not be longer
//            than the input (the transform then fails and the sequence skips it).
//   inverse: a maximal group of bytes <= 1 (that are not the second byte of an 0xFF pair) is a run length, 0xFF x is
//            0xFE + x, any other byte b is b - 1.
// Both directions are scans: per byte "how many output bytes do I produce" -> exclusive prefix sum -> scatter. One CTA
// per block walks the block in 8 KiB tiles (512 threads x 16 bytes) carrying the few scalars that cross a tile
// boundary (last non-zero position / last non-0xFF position / open digit group / output offset); blocks of a batch run
// concurrently. The inverse never writes zeros: the destination is cleared beforehand, a run only advances the offset.
#include "kz_zrlt.cuh"

namespace kz {

static const int ZT = 512;           // threads per CTA
static const int ZB = 16;            // bytes per thread
static const int ZTILE = ZT * ZB;    // bytes per tile

// inclusive scans over the CTA (<= 1024 threads); s_w = 32 words of scratch
KZ_D int64_t cta_scan_max(int64_t v, int64_t* s_w) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t t = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (lane >= d) v = max(v, t);
    }
    __syncthreads();
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    if (warp == 0) {
        int64_t w = s_w[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t t = __shfl_up_sync(0xFFFFFFFFu, w, d);
            if (lane >= d) w = max(w, t);
        }
        s_w[lane] = w;
    }
    __syncthreads();
    if (warp > 0) v = max(v, s_w[warp - 1]);
    return v;
}
KZ_D uint64_t cta_scan_add(uint64_t v, uint64_t* s_w) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t t = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (lane >= d) v += t;
    }
    __syncthreads();
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    if (warp == 0) {
        uint64_t w = s_w[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t t = __shfl_up_sync(0xFFFFFFFFu, w, d);
            if (lane >= d) w += t;
        }
        s_w[lane] = w;
    }
    __syncthreads();
    if (warp > 0) v += s_w[warp - 1];
    return v;
}

// ---- forward. status: 0 ok, 1 = output would not fit (transform skipped, ZRLT.go:93-96,109-121,136-138)
__global__ void __launch_bounds__(ZT) zrlt_forward_kernel(const uint8_t* __restrict__ data, const ZrltBlock* __restrict__ blocks, int nblocks,
                                                          uint8_t* __restrict__ out, uint32_t* __restrict__ out_len, int32_t* __restrict__ status) {
    __shared__ int64_t s_scan[32];
    __shared__ uint8_t s_first[ZT + 1];
    __shared__ int64_t s_carry_nz;
    __shared__ uint64_t s_carry_off;
    __shared__ int s_fail;
    const ZrltBlock blk = blocks[blockIdx.x];
    if (!blk.active) return;
    const uint8_t* src = data + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const uint64_t n = blk.len;
    const uint64_t dst_end = n;  // "do not expand"
    const int tid = threadIdx.x;
    if (tid == 0) {
        s_carry_nz = -1;  // position of the last non-zero byte before the tile
        s_carry_off = 0;
        s_fail = 0;
    }
    __syncthreads();
    for (uint64_t base = 0; base < n; base += ZTILE) {
        const uint64_t p0 = base + (uint64_t)tid * ZB;
        uint8_t b[ZB];
        int cnt = 0;
        if (p0 + ZB <= n) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + p0));
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < ZB; k++) b[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
            cnt = ZB;
        } else {
#pragma unroll
            for (int k = 0; k < ZB; k++) {
                b[k] = p0 + k < n ? src[p0 + k] : 1;
                if (p0 + k < n) cnt = k + 1;
            }
        }
        s_first[tid] = b[0];
        if (tid == ZT - 1) s_first[ZT] = base + ZTILE < n ? src[base + ZTILE] : 1;  // the byte after the tile (1 = "not zero")
        // last non-zero position at or before each byte
        int64_t lnz = -2;  // none inside my bytes
#pragma unroll
        for (int k = 0; k < ZB; k++)
            if (k < cnt && b[k] != 0) lnz = (int64_t)(p0 + k);
        const int64_t carry_nz = s_carry_nz;
        const int64_t incl = cta_scan_max(lnz, s_scan);  // also a barrier: s_first is visible afterwards
        int64_t before = __shfl_up_sync(0xFFFFFFFFu, incl, 1);
        if ((tid & 31) == 0) before = tid ? s_scan[(tid >> 5) - 1] : -2;
        if (before < -1) before = carry_nz;  // nothing in the tile before me
        // output bytes per input byte
        uint32_t len[ZB];
        uint32_t mine = 0;
        int64_t run_nz = before;
#pragma unroll
        for (int k = 0; k < ZB; k++) {
            uint32_t l = 0;
            if (k < cnt) {
                if (b[k] == 0) {
                    const uint8_t nxt = k + 1 < ZB ? (k + 1 < cnt ? b[k + 1] : (uint8_t)1) : s_first[tid + 1];
                    const bool last_of_run = nxt != 0 || p0 + k + 1 >= n;
                    if (last_of_run) {
                        const uint64_t run_length = (p0 + k) - (uint64_t)(run_nz + 1) + 2;  // zeros + 1
                        l = 31u - (uint32_t)__clz((int)(uint32_t)run_length);
                        if (run_length >> 32) l = 32;  // cannot happen for blocks <= 1 GiB
                    }
                } else {
                    run_nz = (int64_t)(p0 + k);
                    l = b[k] >= 0xFE ? 2u : 1u;
                }
            }
            len[k] = l;
            mine += l;
        }
        const uint64_t carry_off = s_carry_off;
        const uint64_t incl_off = cta_scan_add(mine, reinterpret_cast<uint64_t*>(s_scan));
        uint64_t o = carry_off + incl_off - mine;
        bool fail = false;
        run_nz = before;
#pragma unroll
        for (int k = 0; k < ZB; k++) {
            if (k < cnt) {
                const uint32_t l = len[k];
                if (b[k] == 0) {
                    if (l) {
                        if (o + l >= dst_end) fail = true;  // dstIdx >= dstEnd - log2
                        const uint64_t run_length = (p0 + k) - (uint64_t)(run_nz + 1) + 2;
                        if (!fail)
                            for (uint32_t d = 0; d < l; d++) dst[o + d] = (uint8_t)((run_length >> (l - 1 - d)) & 1);
                    }
                } else {
                    run_nz = (int64_t)(p0 + k);
                    if (l == 2) {
                        if (o + 1 >= dst_end) fail = true;  // dstIdx >= dstEnd - 1
                        if (!fail) {
                            dst[o] = 0xFF;
                            dst[o + 1] = (uint8_t)(b[k] - 0xFE);
                        }
                    } else {
                        if (o >= dst_end) fail = true;
                        if (!fail) dst[o] = (uint8_t)(b[k] + 1);
                    }
                }
                o += l;
            }
        }
        if (fail) s_fail = 1;
        __syncthreads();
        if (tid == ZT - 1) {
            s_carry_off = carry_off + incl_off;
            s_carry_nz = incl < -1 ? carry_nz : incl;
        }
        __syncthreads();
        if (s_fail) break;
    }
    if (tid == 0) {
        out_len[blockIdx.x] = (uint32_t)s_carry_off;
        status[blockIdx.x] = s_fail ? 1 : 0;
    }
}

// The run length of a digit group as ZRLT.go:159-170 computes it: runLength = 1, then runLength = 2 * runLength + digit per digit, in
// a 64-bit uint. head = the value of the group's digits before these nd (1: none), digits = the last nd digits, nd <= 64. Past 64
// digits the leading ones have left the word, so the result is the group's value modulo 2^64, as in the reference.
KZ_D uint64_t zrlt_group_value(uint64_t head, uint64_t digits, uint32_t nd) { return nd >= 64 ? digits : (head << nd) | digits; }

// ---- inverse. The destination block [dst_off, dst_off + cap) must be zero filled by the caller.
// status: 0 ok, -KZ_E_PROCESS_BLOCK where the reference returns an error (ZRLT.go:172-173, :204-222): a run of zeros longer than the
// room left, output past cap, or bytes left over once the output is full. The last one decides only when the block's last item writes
// nothing (a trailing escape with no second byte, or a final group whose value is 0 or 1 modulo 2^64): the reference stops on the
// full output before it reads that item, and every other last item needs room of its own.
__global__ void __launch_bounds__(ZT) zrlt_inverse_kernel(const uint8_t* __restrict__ data, const ZrltBlock* __restrict__ blocks, int nblocks,
                                                          uint8_t* __restrict__ out, uint32_t* __restrict__ out_len, int32_t* __restrict__ status) {
    __shared__ int64_t s_scan[32];
    __shared__ uint8_t s_cls[ZTILE + 16];  // per byte of the tile: 0 regular, 1 digit 0, 2 digit 1, 3 escape, 4 follower
    __shared__ uint8_t s_first[ZT + 1];
    __shared__ int64_t s_carry_ff;   // position of the last byte != 0xFF before the tile (-1: none)
    __shared__ uint64_t s_carry_val; // value of the digit group that is open at the tile start (modulo 2^64)
    __shared__ int s_carry_open;     // 1: a digit group is open at the tile start
    __shared__ uint64_t s_carry_off;
    __shared__ int s_bad, s_last_empty;
    const ZrltBlock blk = blocks[blockIdx.x];
    if (!blk.active) return;
    const uint8_t* src = data + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const uint64_t n = blk.len, cap = blk.cap;
    const int tid = threadIdx.x;
    if (tid == 0) {
        s_carry_ff = -1;
        s_carry_val = 0;
        s_carry_open = 0;
        s_carry_off = 0;
        s_bad = 0;
        s_last_empty = 0;
    }
    __syncthreads();
    for (uint64_t base = 0; base < n; base += ZTILE) {
        const uint64_t p0 = base + (uint64_t)tid * ZB;
        uint8_t b[ZB];
        int cnt = 0;
        if (p0 + ZB <= n) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + p0));
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < ZB; k++) b[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
            cnt = ZB;
        } else {
#pragma unroll
            for (int k = 0; k < ZB; k++) {
                b[k] = p0 + k < n ? src[p0 + k] : 2;
                if (p0 + k < n) cnt = k + 1;
            }
        }
        // ---- roles of the 0xFF bytes: inside a run of 0xFF the bytes alternate escape / second byte, starting with escape
        int64_t lff = -2;
#pragma unroll
        for (int k = 0; k < ZB; k++)
            if (k < cnt && b[k] != 0xFF) lff = (int64_t)(p0 + k);
        const int64_t carry_ff = s_carry_ff;
        const int64_t incl_ff = cta_scan_max(lff, s_scan);
        int64_t bef = __shfl_up_sync(0xFFFFFFFFu, incl_ff, 1);
        if ((tid & 31) == 0) bef = tid ? s_scan[(tid >> 5) - 1] : -2;
        if (bef < -1) bef = carry_ff;
        uint8_t cls[ZB];
        int64_t lnf = bef;  // last non-0xFF position before the current byte
#pragma unroll
        for (int k = 0; k < ZB; k++) {
            uint8_t c = 0;
            if (k < cnt) {
                const uint64_t i = p0 + k;
                // the previous byte is an escape when it is 0xFF at an even index inside its run
                const bool prev_ff = i > 0 && (int64_t)(i - 1) > lnf;               // byte i-1 is 0xFF
                const bool follower = prev_ff && (((i - 1) - (uint64_t)(lnf + 1)) & 1) == 0;
                if (follower) c = 4;
                else if (b[k] == 0xFF) c = 3;
                else if (b[k] <= 1) c = (uint8_t)(1 + b[k]);
                if (b[k] != 0xFF) lnf = (int64_t)i;
            }
            cls[k] = c;
            s_cls[tid * ZB + k] = c;
        }
        if (tid == ZT - 1) {  // class of the byte after the tile only matters as "digit or not": peek
            uint8_t nc = 0;
            const uint64_t i = base + ZTILE;
            if (i < n) {
                const uint8_t nb = src[i];
                const bool prev_ff = (int64_t)(i - 1) > lnf;
                const bool follower = prev_ff && (((i - 1) - (uint64_t)(lnf + 1)) & 1) == 0;
                nc = follower ? 4 : (nb == 0xFF ? 3 : (nb <= 1 ? 1 + nb : 0));
            }
            s_cls[ZTILE] = nc;
        }
        __syncthreads();
        // ---- output bytes per input byte: followers and regular bytes 1; the last digit of a group: value - 1 zeros
        const uint64_t carry_val = s_carry_val;
        const bool carry_open = s_carry_open != 0;
        uint64_t adv[ZB];
        uint64_t mine = 0;
        bool bad = false;
#pragma unroll
        for (int k = 0; k < ZB; k++) {
            uint64_t a = 0;
            if (k < cnt) {
                const uint8_t c = cls[k];
                if (c == 0 || c == 4) {
                    a = 1;
                } else if (c == 1 || c == 2) {
                    const uint32_t t = tid * ZB + k;
                    const uint8_t nc = s_cls[t + 1];
                    const bool last = !(nc == 1 || nc == 2) || p0 + k + 1 >= n;
                    if (last) {  // gather the digits of the group (backwards); it may continue the group open at the tile start
                        uint64_t digits = 0;
                        uint32_t nd = 0;
                        int32_t j = (int32_t)t;
                        while (j >= 0 && (s_cls[j] == 1 || s_cls[j] == 2) && nd < 64) {
                            digits |= (uint64_t)(s_cls[j] - 1) << nd;
                            nd++;
                            j--;
                        }
                        const uint64_t head = j < 0 && carry_open ? carry_val : 1;
                        const uint64_t v = zrlt_group_value(head, digits, nd);
                        // value 0: inside the stream runLength-- wraps to 2^64 - 1 (:170-173); at its end the group is skipped (:205)
                        a = v == 0 && p0 + k + 1 == n ? 0 : v - 1;
                        if (a > cap) {
                            bad = true;  // more zeros than the block holds
                            a = 0;
                        }
                    }
                }
                if (p0 + k + 1 == n && (c == 3 || ((c == 1 || c == 2) && a == 0))) s_last_empty = 1;
            }
            adv[k] = a;
            mine += a;
        }
        const uint64_t carry_off = s_carry_off;
        const uint64_t incl_off = cta_scan_add(mine, reinterpret_cast<uint64_t*>(s_scan));
        uint64_t o = carry_off + incl_off - mine;
#pragma unroll
        for (int k = 0; k < ZB; k++) {
            if (k < cnt) {
                const uint8_t c = cls[k];
                if (c == 0) {
                    if (o < cap) dst[o] = (uint8_t)(b[k] - 1);
                } else if (c == 4) {
                    if (o < cap) dst[o] = (uint8_t)(0xFE + b[k]);
                }
                o += adv[k];
            }
        }
        if (bad) s_bad = 1;
        __syncthreads();
        if (tid == ZT - 1) {
            s_carry_off = carry_off + incl_off;
            s_carry_ff = incl_ff < -1 ? carry_ff : incl_ff;
            // digit group still open at the end of the tile?
            uint64_t open = 0;
            int is_open = 0;
            const uint8_t lc = s_cls[ZTILE - 1];
            if (base + ZTILE < n && (lc == 1 || lc == 2) && (s_cls[ZTILE] == 1 || s_cls[ZTILE] == 2)) {
                uint64_t digits = 0;
                uint32_t nd = 0;
                int32_t j = ZTILE - 1;
                while (j >= 0 && (s_cls[j] == 1 || s_cls[j] == 2) && nd < 64) {
                    digits |= (uint64_t)(s_cls[j] - 1) << nd;
                    nd++;
                    j--;
                }
                open = zrlt_group_value(j < 0 && carry_open ? carry_val : 1, digits, nd);
                is_open = 1;
            }
            s_carry_val = open;
            s_carry_open = is_open;
        }
        __syncthreads();
    }
    if (tid == 0) {
        const uint64_t total = s_carry_off;
        const bool fail = s_bad || total > cap || (s_last_empty && total >= cap);
        status[blockIdx.x] = fail ? -KZ_E_PROCESS_BLOCK : 0;
        out_len[blockIdx.x] = (uint32_t)(total > cap ? cap : total);
    }
}

}  // namespace kz
