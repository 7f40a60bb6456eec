// PACK / DNA transform (AliasCodec) on the GPU.
// Reference: v2/transform/AliasCodec.go — Forward :74-273 (small alphabets are bit packed :145-207, otherwise the most frequent
// digrams are replaced by unused byte values :208-287), Inverse :278-434. Everything is decided on the device; the host only
// launches the fixed kernel sequence below over the whole batch and reads the per-block results once.
//
// Forward: hist0 (byte histogram) -> plan (mode, header, byte map) -> pack (modes 2/3: 4 or 2 symbols per byte)
//          -> hist1 (digram histogram) -> select (the n0 most frequent digrams, header, alias map)
//          -> dg_tiles / dg_scan / dg_emit: the greedy left-to-right parse "alias the pair at i if it has one, else copy byte i"
//             is a two-state machine (state = is position i the start of a symbol?); each tile of 4096 positions reduces to a
//             function {start, skip} -> {start, skip} plus the number of symbols it emits for either entering state, a serial
//             pass over the tile functions gives every tile its entering state and output offset, and the tiles emit in parallel.
// Inverse: plan (header) -> fill (modes 1-3) -> tiles / scan / emit (mode 4: every byte expands to 1 or 2 bytes).
#include "kz_alias.cuh"

namespace kz {

namespace {

const int DT_UNDEFINED = 0, DT_MULTIMEDIA = 2, DT_EXE = 3, DT_DNA = 6, DT_BIN = 7, DT_UTF8 = 8;
const uint32_t HIST_SLICES = 32;

struct AliasInfo {  // per block, in the workspace
    uint32_t mode;     // 0 skip, 1 one symbol, 2 four symbols, 3 sixteen symbols, 4 digram
    uint32_t n0;       // free byte values (forward) / number of symbols or aliases (inverse)
    uint32_t hdr_len;  // bytes of header in front of the packed / aliased data
    uint32_t out_len;
    int32_t status;
    int32_t data_type;
    uint32_t src_end;  // inverse: end of the aliased data
    uint32_t adjust;   // inverse: src[1] (digram) or the adjust byte (packed)
    uint8_t absent[256];
    uint8_t map8[256];  // forward: symbol -> index; inverse (modes 2/3): index -> symbol in [0..16)
    uint32_t map32[256];  // inverse mode 4: byte -> (length << 16) | first | second << 8
};

struct Ws {
    uint32_t* hist0;   // [nblocks][256]
    AliasInfo* info;   // [nblocks]
    uint32_t* hist1;   // [nblocks][65536]
    uint16_t* map16;   // [nblocks][65536]  0 = no alias, else 0x100 | alias
    uint32_t* tile_fn; // [nblocks][ntiles]
    uint32_t* tile_in; // [nblocks][ntiles] entering state (forward) / unused
    uint32_t* tile_off;// [nblocks][ntiles] output offset of the tile
    uint32_t ntiles;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

Ws carve(uint8_t* ws, uint32_t nblocks, uint32_t max_len) {
    Ws w;
    w.ntiles = (max_len + ALIAS_TILE - 1) / ALIAS_TILE + 1;
    uint8_t* p = ws;
    w.hist0 = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 256 * 4);
    w.info = reinterpret_cast<AliasInfo*>(p);
    p += align256((size_t)nblocks * sizeof(AliasInfo));
    w.hist1 = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 65536 * 4);
    w.map16 = reinterpret_cast<uint16_t*>(p);
    p += align256((size_t)nblocks * 65536 * 2);
    w.tile_fn = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * w.ntiles * 4);
    w.tile_in = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * w.ntiles * 4);
    w.tile_off = reinterpret_cast<uint32_t*>(p);
    return w;
}

// ---- two-state parse functions: cnt0 | cnt1 << 13 | img0 << 26 | img1 << 27 (state 0 = start of a symbol, 1 = second byte of a pair)
KZ_D uint32_t fn_make(uint32_t img0, uint32_t cnt0, uint32_t img1, uint32_t cnt1) { return cnt0 | (cnt1 << 13) | (img0 << 26) | (img1 << 27); }
KZ_D uint32_t fn_img(uint32_t f, uint32_t s) { return (f >> (26 + s)) & 1u; }
KZ_D uint32_t fn_cnt(uint32_t f, uint32_t s) { return (f >> (13 * s)) & 0x1FFFu; }
KZ_D uint32_t fn_identity() { return fn_make(0, 0, 1, 0); }
KZ_D uint32_t fn_compose(uint32_t a, uint32_t b) {  // a first, then b
    const uint32_t i0 = fn_img(a, 0), i1 = fn_img(a, 1);
    return fn_make(fn_img(b, i0), fn_cnt(a, 0) + fn_cnt(b, i0), fn_img(b, i1), fn_cnt(a, 1) + fn_cnt(b, i1));
}

// inclusive scan of the per-thread functions of a 256-thread CTA in thread order; returns the exclusive prefix of the calling thread and
// leaves the CTA total in *total (valid for all threads after the call)
KZ_D uint32_t cta_scan_fn(uint32_t f, uint32_t* s_warp /*[8]*/, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = f;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= d) incl = fn_compose(o, incl);
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t pre = fn_identity();
    for (int w = 0; w < warp; w++) pre = fn_compose(pre, s_warp[w]);
    uint32_t tot = fn_identity();
    for (int w = 0; w < 8; w++) tot = fn_compose(tot, s_warp[w]);
    *total = tot;
    uint32_t excl = __shfl_up_sync(0xFFFFFFFFu, incl, 1);
    if (lane == 0) excl = fn_identity();
    __syncthreads();
    return fn_compose(pre, excl);
}

// the 16 positions of a thread: pair mask (bit j: positions base+j, base+j+1 have an alias) and number of valid positions
KZ_D void dg_thread_positions(const uint8_t* src, uint32_t count, const uint16_t* map16, uint32_t base, uint32_t& pm, uint32_t& nv, uint8_t (&by)[17]) {
    pm = 0;
    nv = base < count ? min(16u, count - base) : 0u;
    for (uint32_t j = 0; j < 17; j++) by[j] = (base + j < count) ? src[base + j] : 0;
    for (uint32_t j = 0; j < nv; j++) {
        const uint32_t i = base + j;
        if (i + 1 < count && map16[((uint32_t)by[j] << 8) | by[j + 1]] != 0) pm |= 1u << j;
    }
}
KZ_D uint32_t dg_thread_fn(uint32_t pm, uint32_t nv) {
    uint32_t img[2], cnt[2];
    for (uint32_t s0 = 0; s0 < 2; s0++) {
        uint32_t s = s0, c = 0;
        for (uint32_t j = 0; j < nv; j++) {
            if (s == 0) {
                c++;
                s = (pm >> j) & 1u;
            } else {
                s = 0;
            }
        }
        img[s0] = s;
        cnt[s0] = c;
    }
    return fn_make(img[0], cnt[0], img[1], cnt[1]);
}

}  // namespace

namespace {

// ------------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) alias_hist0_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, uint32_t* __restrict__ hist0) {
    __shared__ uint32_t h[256];
    const int b = blockIdx.y;
    const StageBlock blk = blocks[b];
    if (blk.len < 1024) return;
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint8_t* src = in + blk.src_off;
    const uint32_t per = ((blk.len + HIST_SLICES - 1) / HIST_SLICES + 3) & ~3u;
    const uint32_t lo = blockIdx.x * per, hi = min(blk.len, lo + per);
    for (uint32_t i = lo + 4 * threadIdx.x; i < hi; i += 1024) {
        if (i + 4 <= hi) {
            const uint32_t v = *reinterpret_cast<const uint32_t*>(src + i);  // src_off and lo are multiples of 4
            atomicAdd(&h[v & 0xFF], 1u);
            atomicAdd(&h[(v >> 8) & 0xFF], 1u);
            atomicAdd(&h[(v >> 16) & 0xFF], 1u);
            atomicAdd(&h[v >> 24], 1u);
        } else {
            for (uint32_t k = i; k < hi; k++) atomicAdd(&h[src[k]], 1u);
        }
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist0[(size_t)b * 256 + threadIdx.x], h[threadIdx.x]);
}

// one warp per block, lane 0: AliasCodec.Forward :83-207 up to the choice of the coding mode
__global__ void __launch_bounds__(32) alias_plan_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                         const uint32_t* __restrict__ hist0, AliasInfo* __restrict__ infos, uint8_t* __restrict__ out,
                                                         StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const StageBlock blk = blocks[b];
    AliasInfo& I = infos[b];
    StageResult r;
    r.status = 1;
    r.out_len = 0;
    r.data_type = blk.data_type;
    r.mode = 0;
    I.mode = 0;
    I.status = 1;
    I.out_len = 0;
    I.hdr_len = 0;
    I.n0 = 0;
    const uint32_t count = blk.len;
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    bool go = count >= 1024 && (uint64_t)blk.cap >= (uint64_t)count + 1024;  // _ALIAS_MIN_BLOCKSIZE :87, MaxEncodedLen :83
    int dt = blk.data_type;
    if (dt == DT_MULTIMEDIA || dt == DT_UTF8 || dt == DT_EXE || dt == DT_BIN) go = false;       // :98-104
    if (blk.flags && dt != DT_UNDEFINED && dt != DT_DNA) go = false;                          // :106-108
    if (go) {
        const uint32_t* f = hist0 + (size_t)b * 256;
        uint32_t n0 = 0;
        for (int i = 0; i < 256; i++)
            if (f[i] == 0) I.absent[n0++] = (uint8_t)i;
        if (n0 < 16) go = false;  // :125-127
        if (go && dt == DT_UNDEFINED) {  // :129-139
            dt = detect_simple_type_dev(count, f);
            if (dt != DT_UNDEFINED) r.data_type = dt;
            if (dt != DT_DNA && blk.flags) go = false;
        }
        if (go) {
            I.n0 = n0;
            if (n0 >= 240) {
                dst[0] = (uint8_t)n0;
                if (n0 == 255) {  // one symbol :149-155
                    dst[1] = src[0];
                    dst[2] = (uint8_t)count;
                    dst[3] = (uint8_t)(count >> 8);
                    dst[4] = (uint8_t)(count >> 16);
                    dst[5] = (uint8_t)(count >> 24);
                    I.mode = 1;
                    I.out_len = 6;
                } else {
                    uint32_t di = 1, j = 0;
                    for (int i = 0; i < 256; i++) {
                        I.map8[i] = 0;
                        if (f[i] != 0) {
                            dst[di++] = (uint8_t)i;
                            I.map8[i] = (uint8_t)j++;
                        }
                    }
                    if (n0 >= 252) {  // 4 symbols or less :170-185
                        const uint32_t c3 = count & 3;
                        dst[di++] = (uint8_t)c3;
                        for (uint32_t k = 0; k < c3; k++) dst[di++] = src[k];
                        I.mode = 2;
                        I.hdr_len = di;
                        I.out_len = di + (count - c3) / 4;
                    } else {  // 16 symbols or less :186-203
                        const uint32_t odd = count & 1;
                        dst[di++] = (uint8_t)odd;
                        if (odd) dst[di++] = src[0];
                        I.mode = 3;
                        I.hdr_len = di;
                        I.out_len = di + (count - odd) / 2;
                    }
                }
                if (I.out_len >= count) I.mode = 0;  // :289-291
                if (I.mode != 0) {
                    I.status = 0;
                    r.status = 0;
                    r.out_len = I.out_len;
                    r.mode = I.mode;
                }
            } else {
                I.mode = 4;  // decided by the digram kernels
            }
        }
    }
    I.data_type = r.data_type;
    res[b] = r;
}

// modes 2 / 3: every thread packs 4 (or 2) symbols into one byte
__global__ void __launch_bounds__(256) alias_pack_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const AliasInfo* __restrict__ infos,
                                                          uint8_t* __restrict__ out) {
    const int b = blockIdx.y;
    const AliasInfo& I = infos[b];
    if (I.mode != 2 && I.mode != 3) return;
    __shared__ uint8_t m[256];
    m[threadIdx.x] = I.map8[threadIdx.x];
    __syncthreads();
    const StageBlock blk = blocks[b];
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off + I.hdr_len;
    const uint32_t count = blk.len;
    if (I.mode == 2) {
        const uint32_t c3 = count & 3, nout = (count - c3) / 4;
        for (uint32_t k = blockIdx.x * 256 + threadIdx.x; k < nout; k += gridDim.x * 256) {
            const uint8_t* p = src + c3 + 4 * (size_t)k;
            dst[k] = (uint8_t)((m[p[0]] << 6) | (m[p[1]] << 4) | (m[p[2]] << 2) | m[p[3]]);
        }
    } else {
        const uint32_t odd = count & 1, nout = (count - odd) / 2;
        for (uint32_t k = blockIdx.x * 256 + threadIdx.x; k < nout; k += gridDim.x * 256) {
            const uint8_t* p = src + odd + 2 * (size_t)k;
            dst[k] = (uint8_t)((m[p[0]] << 4) | m[p[1]]);
        }
    }
}

// mode 4: histogram of (previous byte, byte) pairs, previous = 0 for the first byte (ComputeHistogram order 1, internal/Global.go:305-341)
__global__ void __launch_bounds__(256) alias_hist1_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const AliasInfo* __restrict__ infos,
                                                           uint32_t* __restrict__ hist1) {
    const int b = blockIdx.y;
    if (infos[b].mode != 4) return;
    const StageBlock blk = blocks[b];
    const uint8_t* src = in + blk.src_off;
    uint32_t* h = hist1 + (size_t)b * 65536;
    for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i < blk.len; i += gridDim.x * 256) {
        const uint32_t prv = i ? src[i - 1] : 0u;
        atomicAdd(&h[(prv << 8) | src[i]], 1u);
    }
}

// mode 4: the n0 most frequent digrams, by decreasing (frequency, value) (:233-240), get the free byte values in increasing order
__global__ void __launch_bounds__(1024) alias_select_kernel(const StageBlock* __restrict__ blocks, AliasInfo* __restrict__ infos, const uint32_t* __restrict__ hist1,
                                                             uint16_t* __restrict__ map16_all, uint8_t* __restrict__ out, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    AliasInfo& I = infos[b];
    if (I.mode != 4) return;
    __shared__ unsigned long long s_red[32];
    __shared__ unsigned long long s_best;
    __shared__ uint32_t s_cnt[32];
    __shared__ uint32_t s_n0;
    const StageBlock blk = blocks[b];
    const uint32_t* h = hist1 + (size_t)b * 65536;
    uint16_t* map16 = map16_all + (size_t)b * 65536;
    uint8_t* dst = out + blk.dst_off;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t f[64];
    uint32_t nz = 0;
#pragma unroll
    for (int j = 0; j < 64; j++) {
        f[j] = h[tid + 1024 * j];
        nz += f[j] != 0;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) nz += __shfl_xor_sync(0xFFFFFFFFu, nz, d);
    if (lane == 0) s_cnt[warp] = nz;
    __syncthreads();
    if (tid == 0) {
        uint32_t n1 = 0;
        for (int w = 0; w < 32; w++) n1 += s_cnt[w];
        uint32_t n0 = I.n0;
        if (n0 > n1) n0 = n1;  // :222-229
        s_n0 = n0;
    }
    __syncthreads();
    const uint32_t n0 = s_n0;
    if (n0 < 16) {
        if (tid == 0) {
            I.mode = 0;
            I.status = 1;
        }
        return;
    }
    unsigned long long best = 0;
    bool dirty = true;
    uint64_t savings = 0;
    for (uint32_t k = 0; k < n0; k++) {
        if (dirty) {
            best = 0;
#pragma unroll
            for (int j = 0; j < 64; j++) {
                const unsigned long long key = ((unsigned long long)f[j] << 16) | (unsigned long long)(tid + 1024 * j);
                if (f[j] != 0 && key > best) best = key;
            }
            dirty = false;
        }
        unsigned long long m = best;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, m, d);
            m = o > m ? o : m;
        }
        if (lane == 0) s_red[warp] = m;
        __syncthreads();
        if (warp == 0) {
            unsigned long long v = s_red[lane];
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) {
                const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, v, d);
                v = o > v ? o : v;
            }
            if (lane == 0) s_best = v;
        }
        __syncthreads();
        const unsigned long long win = s_best;
        const uint32_t val = (uint32_t)(win & 0xFFFF);
        if ((val & 1023u) == (uint32_t)tid) {
            const uint32_t jj = val >> 10;
#pragma unroll
            for (int j = 0; j < 64; j++)
                if ((uint32_t)j == jj) f[j] = 0;
            dirty = true;
        }
        if (tid == 0) {
            const uint8_t alias = I.absent[k];
            savings += win >> 16;
            map16[val] = (uint16_t)(0x100u | alias);
            dst[2 + 3 * k] = (uint8_t)(val >> 8);
            dst[3 + 3 * k] = (uint8_t)val;
            dst[4 + 3 * k] = alias;
        }
        __syncthreads();
    }
    if (tid == 0) {
        I.n0 = n0;
        dst[0] = (uint8_t)n0;
        dst[1] = 0;
        I.hdr_len = 2 + 3 * n0;
        if (savings < (uint64_t)(blk.len / 20)) {  // :259-261
            I.mode = 0;
            I.status = 1;
        }
    }
}

__global__ void __launch_bounds__(256) alias_dg_tiles_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const AliasInfo* __restrict__ infos,
                                                              const uint16_t* __restrict__ map16_all, uint32_t* __restrict__ tile_fn, uint32_t ntiles) {
    const int b = blockIdx.y;
    if (infos[b].mode != 4) return;
    const StageBlock blk = blocks[b];
    if ((uint64_t)blockIdx.x * ALIAS_TILE >= blk.len) return;
    __shared__ uint32_t s_warp[8];
    uint32_t pm, nv;
    uint8_t by[17];
    dg_thread_positions(in + blk.src_off, blk.len, map16_all + (size_t)b * 65536, blockIdx.x * ALIAS_TILE + threadIdx.x * 16, pm, nv, by);
    uint32_t total;
    cta_scan_fn(dg_thread_fn(pm, nv), s_warp, &total);
    if (threadIdx.x == 0) tile_fn[(size_t)b * ntiles + blockIdx.x] = total;
}

// serial pass over the tile functions of a block: entering state and output offset of every tile, total size, final decision
__global__ void __launch_bounds__(32) alias_dg_scan_kernel(const StageBlock* __restrict__ blocks, int nblocks, AliasInfo* __restrict__ infos,
                                                            const uint32_t* __restrict__ tile_fn, uint32_t* __restrict__ tile_in, uint32_t* __restrict__ tile_off,
                                                            uint32_t ntiles, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    AliasInfo& I = infos[b];
    if (I.mode != 4) return;
    const StageBlock blk = blocks[b];
    const uint32_t nt = (blk.len + ALIAS_TILE - 1) / ALIAS_TILE;
    uint32_t state = 0, off = I.hdr_len;
    for (uint32_t t = 0; t < nt; t++) {
        const uint32_t f = tile_fn[(size_t)b * ntiles + t];
        tile_in[(size_t)b * ntiles + t] = state;
        tile_off[(size_t)b * ntiles + t] = off;
        off += fn_cnt(f, state);
        state = fn_img(f, state);
    }
    I.out_len = off;
    if (off >= blk.len) {  // :289-291
        I.status = 1;
        return;  // mode stays 4: the emit kernel still runs, its output is ignored
    }
    I.status = 0;
    StageResult r = res[b];
    r.status = 0;
    r.out_len = off;
    r.mode = 4;
    res[b] = r;
}

__global__ void __launch_bounds__(256) alias_dg_emit_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const AliasInfo* __restrict__ infos,
                                                             const uint16_t* __restrict__ map16_all, const uint32_t* __restrict__ tile_in,
                                                             const uint32_t* __restrict__ tile_off, uint32_t ntiles, uint8_t* __restrict__ out) {
    const int b = blockIdx.y;
    const AliasInfo& I = infos[b];
    if (I.mode != 4 || I.status != 0) return;
    const StageBlock blk = blocks[b];
    if ((uint64_t)blockIdx.x * ALIAS_TILE >= blk.len) return;
    __shared__ uint32_t s_warp[8];
    const uint16_t* map16 = map16_all + (size_t)b * 65536;
    const uint32_t base = blockIdx.x * ALIAS_TILE + threadIdx.x * 16;
    uint32_t pm, nv;
    uint8_t by[17];
    dg_thread_positions(in + blk.src_off, blk.len, map16, base, pm, nv, by);
    uint32_t total;
    const uint32_t excl = cta_scan_fn(dg_thread_fn(pm, nv), s_warp, &total);
    const uint32_t s_in = tile_in[(size_t)b * ntiles + blockIdx.x];
    uint32_t s = fn_img(excl, s_in);
    uint8_t* dst = out + blk.dst_off;
    uint32_t o = tile_off[(size_t)b * ntiles + blockIdx.x] + fn_cnt(excl, s_in);
    for (uint32_t j = 0; j < nv; j++) {
        if (s == 0) {
            if ((pm >> j) & 1u) {
                dst[o++] = (uint8_t)map16[((uint32_t)by[j] << 8) | by[j + 1]];
                s = 1;
            } else {
                dst[o++] = by[j];
                if (base + j == blk.len - 1) dst[1] = 1;  // :279-283 the last byte was not consumed by a pair
            }
        } else {
            s = 0;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// inverse
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) alias_inv_plan_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                             AliasInfo* __restrict__ infos, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const StageBlock blk = blocks[b];
    AliasInfo& I = infos[b];
    StageResult r;
    r.status = 0;
    r.out_len = 0;
    r.data_type = 0;
    r.mode = 0;
    I.mode = 0;
    I.status = 0;
    const uint32_t len = blk.len;
    const uint8_t* src = in + blk.src_off;
    if (len == 0) {  // inactive block or empty input (:279-281)
        res[b] = r;
        return;
    }
    int err = 0;
    if (len < 2) err = 1;
    uint32_t n = err ? 0 : src[0];
    if (!err && n < 16) err = 1;
    if (!err) {
        if (n >= 240) {
            n = 256 - n;
            if (n == 1) {  // :304-318
                if (len < 6) {
                    err = 1;
                } else {
                    const uint32_t osize = (uint32_t)src[2] | ((uint32_t)src[3] << 8) | ((uint32_t)src[4] << 16) | ((uint32_t)src[5] << 24);
                    if (osize > blk.cap) err = 1;
                    I.mode = 1;
                    I.out_len = osize;
                    I.map8[0] = src[1];
                }
            } else {
                if (1 + n + 1 > len) err = 1;
                if (!err) {
                    for (uint32_t i = 0; i < 16; i++) I.map8[i] = i < n ? src[1 + i] : 0;
                    const uint32_t adjust = src[1 + n];
                    uint32_t si = 2 + n;
                    if (adjust > 3) err = 1;
                    I.adjust = adjust;
                    if (!err && n <= 4) {  // :336-362
                        if (si + adjust > len) err = 1;
                        if (!err) {
                            const uint64_t o = (uint64_t)adjust + 4ull * (len - si - adjust);
                            if (o > blk.cap) err = 1;
                            I.mode = 2;
                            I.hdr_len = si;
                            I.out_len = (uint32_t)o;
                        }
                    } else if (!err) {  // :363-386
                        const uint32_t a = adjust != 0 ? 1 : 0;
                        if (si + a > len) err = 1;
                        if (!err) {
                            const uint64_t o = (uint64_t)a + 2ull * (len - si - a);
                            if (o > blk.cap) err = 1;
                            I.mode = 3;
                            I.hdr_len = si;
                            I.out_len = (uint32_t)o;
                        }
                    }
                }
            }
        } else {  // :388-415 digram aliases
            const uint32_t tail = src[1];
            if (tail > len || 2 + 3 * n > len - tail) err = 1;
            if (!err) {
                for (uint32_t i = 0; i < 256; i++) I.map32[i] = 0x10000u | i;
                uint32_t si = 2;
                for (uint32_t i = 0; i < n; i++) {
                    I.map32[src[si + 2]] = 0x20000u | (uint32_t)src[si] | ((uint32_t)src[si + 1] << 8);
                    si += 3;
                }
                I.mode = 4;
                I.hdr_len = si;
                I.src_end = len - tail;
                I.adjust = tail;
            }
        }
    }
    if (err) {
        I.mode = 0;
        I.status = -KZ_E_PROCESS_BLOCK;
        r.status = -KZ_E_PROCESS_BLOCK;
    } else if (I.mode != 4) {
        r.out_len = I.out_len;
        r.mode = I.mode;
    }
    res[b] = r;
}

__global__ void __launch_bounds__(256) alias_inv_fill_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const AliasInfo* __restrict__ infos,
                                                              uint8_t* __restrict__ out) {
    const int b = blockIdx.y;
    const AliasInfo& I = infos[b];
    if (I.mode < 1 || I.mode > 3) return;
    const StageBlock blk = blocks[b];
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    __shared__ uint8_t sym[16];
    if (threadIdx.x < 16) sym[threadIdx.x] = I.map8[threadIdx.x];
    __syncthreads();
    const uint32_t stride = gridDim.x * 256, t0 = blockIdx.x * 256 + threadIdx.x;
    if (I.mode == 1) {
        for (uint32_t i = t0; i < I.out_len; i += stride) dst[i] = sym[0];
    } else if (I.mode == 2) {
        const uint32_t adj = I.adjust, si = I.hdr_len + adj, n = blk.len - si;
        if (t0 < adj) dst[t0] = src[I.hdr_len + t0];
        for (uint32_t k = t0; k < n; k += stride) {
            const uint32_t v = src[si + k];
            uint8_t* d = dst + adj + 4 * (size_t)k;
            d[0] = sym[(v >> 6) & 3];
            d[1] = sym[(v >> 4) & 3];
            d[2] = sym[(v >> 2) & 3];
            d[3] = sym[v & 3];
        }
    } else {
        const uint32_t adj = I.adjust != 0 ? 1 : 0, si = I.hdr_len + adj, n = blk.len - si;
        if (t0 < adj) dst[t0] = src[I.hdr_len + t0];
        for (uint32_t k = t0; k < n; k += stride) {
            const uint32_t v = src[si + k];
            uint8_t* d = dst + adj + 2 * (size_t)k;
            d[0] = sym[v >> 4];
            d[1] = sym[v & 15];
        }
    }
}

// mode 4: bytes of output produced by every tile of 4096 input bytes
__global__ void __launch_bounds__(256) alias_inv_tiles_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const AliasInfo* __restrict__ infos,
                                                               uint32_t* __restrict__ tile_fn, uint32_t ntiles) {
    const int b = blockIdx.y;
    const AliasInfo& I = infos[b];
    if (I.mode != 4) return;
    const uint32_t n = I.src_end - I.hdr_len;
    if ((uint64_t)blockIdx.x * ALIAS_TILE >= n) return;
    __shared__ uint32_t s_sum[8];
    const uint8_t* src = in + blocks[b].src_off + I.hdr_len;
    const uint32_t base = blockIdx.x * ALIAS_TILE + threadIdx.x * 16;
    uint32_t s = 0;
    for (uint32_t j = 0; j < 16; j++)
        if (base + j < n) s += I.map32[src[base + j]] >> 16;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, d);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < 8; w++) t += s_sum[w];
        tile_fn[(size_t)b * ntiles + blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(32) alias_inv_scan_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                             AliasInfo* __restrict__ infos, const uint32_t* __restrict__ tile_fn, uint32_t* __restrict__ tile_off,
                                                             uint32_t ntiles, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    AliasInfo& I = infos[b];
    if (I.mode != 4) return;
    const StageBlock blk = blocks[b];
    const uint8_t* src = in + blk.src_off;
    const uint32_t n = I.src_end - I.hdr_len;
    const uint32_t nt = (n + ALIAS_TILE - 1) / ALIAS_TILE;
    uint64_t off = 0;
    for (uint32_t t = 0; t < nt; t++) {
        tile_off[(size_t)b * ntiles + t] = (uint32_t)off;
        off += tile_fn[(size_t)b * ntiles + t];
    }
    // the reference stores two bytes for every alias, even a one byte one (:405-411): the last store must fit
    bool bad = false;
    if (n > 0) {
        const uint32_t last = I.map32[src[I.src_end - 1]] >> 16;
        if (off - last + 2 > blk.cap) bad = true;
    }
    if (I.adjust != 0) {  // :413-417 one trailing literal
        if (I.src_end >= blk.len || off >= blk.cap) bad = true;
        off += 1;
    }
    StageResult r = res[b];
    if (bad || off > 0xFFFFFFFFull) {
        I.status = -KZ_E_PROCESS_BLOCK;
        r.status = -KZ_E_PROCESS_BLOCK;
    } else {
        I.out_len = (uint32_t)off;
        r.out_len = (uint32_t)off;
        r.mode = 4;
    }
    res[b] = r;
}

__global__ void __launch_bounds__(256) alias_inv_emit_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const AliasInfo* __restrict__ infos,
                                                              const uint32_t* __restrict__ tile_off, uint32_t ntiles, uint8_t* __restrict__ out) {
    const int b = blockIdx.y;
    const AliasInfo& I = infos[b];
    if (I.mode != 4 || I.status != 0) return;
    const uint32_t n = I.src_end - I.hdr_len;
    const StageBlock blk = blocks[b];
    uint8_t* dst = out + blk.dst_off;
    if (blockIdx.x == 0 && threadIdx.x == 0 && I.adjust != 0) dst[I.out_len - 1] = in[blk.src_off + I.src_end];
    if ((uint64_t)blockIdx.x * ALIAS_TILE >= n) return;
    __shared__ uint32_t s_sum[8];
    const uint8_t* src = in + blk.src_off + I.hdr_len;
    const uint32_t base = blockIdx.x * ALIAS_TILE + threadIdx.x * 16;
    uint32_t v[16];
    uint32_t s = 0;
    for (uint32_t j = 0; j < 16; j++) {
        v[j] = base + j < n ? I.map32[src[base + j]] : 0u;
        s += v[j] >> 16;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= d) incl += o;
    }
    if (lane == 31) s_sum[warp] = incl;
    __syncthreads();
    uint32_t pre = 0;
    for (int w = 0; w < warp; w++) pre += s_sum[w];
    uint32_t o = tile_off[(size_t)b * ntiles + blockIdx.x] + pre + incl - s;
    for (uint32_t j = 0; j < 16; j++) {
        const uint32_t l = v[j] >> 16;
        if (l >= 1) dst[o] = (uint8_t)v[j];
        if (l == 2) dst[o + 1] = (uint8_t)(v[j] >> 8);
        o += l;
    }
}

}  // namespace

size_t alias_workspace(uint32_t nblocks, uint32_t max_len) {
    const size_t ntiles = (max_len + ALIAS_TILE - 1) / ALIAS_TILE + 1;
    return align256((size_t)nblocks * 256 * 4) + align256((size_t)nblocks * sizeof(AliasInfo)) + align256((size_t)nblocks * 65536 * 4) +
           align256((size_t)nblocks * 65536 * 2) + 3 * align256((size_t)nblocks * ntiles * 4) + 256;
}

cudaError_t alias_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint32_t max_len, uint8_t* ws, size_t ws_bytes,
                                StageResult* d_res, cudaStream_t stream, uint64_t* launches) {
    if (nblocks == 0) return cudaSuccess;
    if (ws_bytes < alias_workspace(nblocks, max_len)) return cudaErrorInvalidValue;
    const Ws w = carve(ws, nblocks, max_len);
    cudaError_t e;
    if ((e = cudaMemsetAsync(w.hist0, 0, (size_t)nblocks * 256 * 4, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(w.hist1, 0, (size_t)nblocks * 65536 * 4, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(w.map16, 0, (size_t)nblocks * 65536 * 2, stream)) != cudaSuccess) return e;
    const uint32_t ntiles_grid = (max_len + ALIAS_TILE - 1) / ALIAS_TILE;
    const uint32_t gx = ntiles_grid < 1 ? 1 : ntiles_grid;
    const uint32_t px = gx < 64 ? gx : 64;
    alias_hist0_kernel<<<dim3(HIST_SLICES, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.hist0);
    alias_plan_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.hist0, w.info, d_out, d_res);
    alias_pack_kernel<<<dim3(px, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, d_out);
    alias_hist1_kernel<<<dim3(px, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, w.hist1);
    alias_select_kernel<<<nblocks, 1024, 0, stream>>>(d_blocks, w.info, w.hist1, w.map16, d_out, d_res);
    alias_dg_tiles_kernel<<<dim3(gx, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, w.map16, w.tile_fn, w.ntiles);
    alias_dg_scan_kernel<<<nblocks, 32, 0, stream>>>(d_blocks, (int)nblocks, w.info, w.tile_fn, w.tile_in, w.tile_off, w.ntiles, d_res);
    alias_dg_emit_kernel<<<dim3(gx, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, w.map16, w.tile_in, w.tile_off, w.ntiles, d_out);
    if (launches) *launches += 8;
    return cudaGetLastError();
}

cudaError_t alias_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint32_t max_len, uint8_t* ws, size_t ws_bytes,
                                StageResult* d_res, cudaStream_t stream, uint64_t* launches) {
    if (nblocks == 0) return cudaSuccess;
    if (ws_bytes < alias_workspace(nblocks, max_len)) return cudaErrorInvalidValue;
    const Ws w = carve(ws, nblocks, max_len);
    const uint32_t ntiles_grid = (max_len + ALIAS_TILE - 1) / ALIAS_TILE;
    const uint32_t gx = ntiles_grid < 1 ? 1 : ntiles_grid;
    const uint32_t px = gx < 64 ? gx : 64;
    alias_inv_plan_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.info, d_res);
    alias_inv_fill_kernel<<<dim3(px, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, d_out);
    alias_inv_tiles_kernel<<<dim3(gx, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, w.tile_fn, w.ntiles);
    alias_inv_scan_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.info, w.tile_fn, w.tile_off, w.ntiles, d_res);
    alias_inv_emit_kernel<<<dim3(gx, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, w.tile_off, w.ntiles, d_out);
    if (launches) *launches += 5;
    return cudaGetLastError();
}

}  // namespace kz
