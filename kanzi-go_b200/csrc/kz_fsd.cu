// MM transform (FSDCodec: fixed step delta) on the GPU.
// Reference: v2/transform/FSDCodec.go — Forward :135-312 samples three sub-blocks, compares the order-0 entropy of the bytes with that
// of the xor against the byte 1, 2, 3, 4, 8 or 16 positions back (internal.ComputeFirstOrderEntropy1024, internal/Global.go:196-214),
// and when a distance wins codes the block as zig-zag deltas (escape 0xFF + xor for deltas outside [-127, 127]) or plain xors;
// Inverse :317-404.
//
// Forward kernels (whole batch, no host synchronisation): sample (7 histograms) -> plan (checks, entropies, distance, coding mode,
// header) -> tiles (bytes produced per 4096 positions) -> scan (tile offsets, completion test) -> emit -> post_hist -> final
// (the "does it still look better" test of :296-310). Inverse: one thread per block walks the tokens (a block's bytes form `dist`
// dependent chains and escapes change the operation, so there is little to share inside a block; blocks run side by side).
#include <algorithm>
#include <cmath>

#include "kz_alias.cuh"
#include <vector>

#include "kz_fsd.cuh"

namespace kz {

namespace {

const int DT_UNDEFINED = 0, DT_MULTIMEDIA = 2, DT_BIN = 7;
const uint32_t SAMPLE_SLICES = 16;

struct FsdInfo {
    uint32_t go;       // 1 while the block is still a candidate
    uint32_t mode;     // 0 delta, 1 xor
    uint32_t dist;
    int32_t ent0;
    uint32_t out_len;
    uint32_t pad[3];
};

struct Ws {
    uint32_t* log2tab;  // [257] LOG2_4096
    uint32_t* hist7;    // [nblocks][7][256]
    uint32_t* hpost;    // [nblocks][256]
    FsdInfo* info;      // [nblocks]
    uint32_t* tile_sum; // [nblocks][ntiles]
    uint32_t* tile_off; // [nblocks][ntiles]
    uint32_t ntiles;
};
size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
Ws carve(uint8_t* ws, uint32_t nblocks, uint32_t max_len) {
    Ws w;
    w.ntiles = (max_len + FSD_TILE - 1) / FSD_TILE + 1;
    uint8_t* p = ws;
    w.log2tab = reinterpret_cast<uint32_t*>(p);
    p += align256(257 * 4);
    w.hist7 = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 7 * 256 * 4);
    w.hpost = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 256 * 4);
    w.info = reinterpret_cast<FsdInfo*>(p);
    p += align256((size_t)nblocks * sizeof(FsdInfo));
    w.tile_sum = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * w.ntiles * 4);
    w.tile_off = reinterpret_cast<uint32_t*>(p);
    return w;
}

// internal/Global.go:60-93 LOG2_4096[i] = round(4096 * log2(i)) (entries 0 and 1 are 0): a data table of the reference, regenerated from
// its definition (checked entry by entry against the reference's table when this was written)
const uint32_t* host_log2_4096() {
    static uint32_t tab[257];
    static bool init = false;
    if (!init) {
        tab[0] = 0;
        for (int k = 1; k <= 256; k++) tab[k] = (uint32_t)(4096.0 * std::log2((double)k) + 0.5);
        init = true;
    }
    return tab;
}

// internal/Global.go:175-191 Log2ScaledBy1024
KZ_D uint32_t log2_scaled_1024(uint32_t x, const uint32_t* T) {
    if (x < 256) return (T[x] + 2) >> 2;
    const uint32_t lg = 31u - (uint32_t)__clz((int)x);
    if ((x & (x - 1)) == 0) return lg << 10;
    return ((lg - 7) * 1024) + ((T[x >> (lg - 7)] + 2) >> 2);
}
// internal/Global.go:196-214 ComputeFirstOrderEntropy1024
KZ_D int entropy_1024(uint32_t block_len, const uint32_t* histo, const uint32_t* T) {
    if (block_len == 0) return 0;
    unsigned long long sum = 0;
    const uint32_t ll = log2_scaled_1024(block_len, T);
    for (int i = 0; i < 256; i++) {
        if (histo[i] == 0) continue;
        const uint32_t l = log2_scaled_1024(histo[i], T);
        sum += ((unsigned long long)histo[i] * (unsigned long long)(ll - l)) >> 3;
    }
    return (int)(sum / (unsigned long long)block_len);
}

// internal/Magic.go:73-112 GetMagicType reduced to what FSDCodec.Forward :170-187 asks: no magic, or BMP / RIFF / PBM / PGM / PPM
KZ_D bool magic_allows_fsd(const uint8_t* p, uint32_t n) {
    if (n < 4) return true;
    const uint32_t key = ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
    if ((key & ~0x0Fu) == 0xFFD8FFE0u) return false;                       // JPEG
    if ((key >> 8) == 0x425A68u || (key >> 8) == 0x494433u) return false;  // bzip2, ID3
    const uint32_t k32[18] = {0x47494638u, 0x25504446u, 0x504B0304u, 0x377ABCAFu, 0x89504E47u, 0x7F454C46u, 0xFEEDFACEu, 0xCEFAEDFEu, 0xFEEDFACFu,
                              0xCFFAEDFEu, 0x28B52FFDu, 0x81CFB2CEu, 0x4D534346u, 0x52494646u, 0x664C6143u, 0xFD377A58u, 0x4B414E5Au, 0x52617221u};
    for (int i = 0; i < 18; i++)
        if (key == k32[i]) return key == 0x52494646u;  // RIFF is a candidate, the others are not
    const uint32_t k16 = key >> 16;
    if (k16 == 0x1F8Bu || k16 == 0x4D5Au) return false;  // gzip, MZ
    return true;                                          // BMP, binary PBM / PGM / PPM, or no magic at all
}

KZ_D uint32_t fsd_dist(uint32_t idx) { return idx < 5 ? idx : (idx == 5 ? 8u : 16u); }  // distances {0, 1, 2, 3, 4, 8, 16}

__global__ void __launch_bounds__(256) fsd_sample_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, uint32_t* __restrict__ hist7) {
    __shared__ uint32_t h[7 * 256];
    const int b = blockIdx.y;
    const StageBlock blk = blocks[b];
    if (blk.len < 1024) return;
    for (int i = threadIdx.x; i < 7 * 256; i += 256) h[i] = 0;
    __syncthreads();
    const uint32_t count10 = blk.len / 10, count5 = 2 * count10;
    const uint8_t* src = in + blk.src_off;
    for (uint32_t k = blockIdx.x * 256 + threadIdx.x; k < count10; k += gridDim.x * 256) {
        const uint32_t i = count10 + k;
#pragma unroll
        for (uint32_t sb = 0; sb < 3; sb++) {
            const uint8_t* p = src + 2 * sb * count5 + i;
            const uint32_t v = p[0];
            atomicAdd(&h[v], 1u);
            atomicAdd(&h[1 * 256 + (v ^ *(p - 1))], 1u);
            atomicAdd(&h[2 * 256 + (v ^ *(p - 2))], 1u);
            atomicAdd(&h[3 * 256 + (v ^ *(p - 3))], 1u);
            atomicAdd(&h[4 * 256 + (v ^ *(p - 4))], 1u);
            atomicAdd(&h[5 * 256 + (v ^ *(p - 8))], 1u);
            atomicAdd(&h[6 * 256 + (v ^ *(p - 16))], 1u);
        }
    }
    __syncthreads();
    uint32_t* g = hist7 + (size_t)b * 7 * 256;
    for (int i = threadIdx.x; i < 7 * 256; i += 256)
        if (h[i]) atomicAdd(&g[i], h[i]);
}

__global__ void __launch_bounds__(32) fsd_plan_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                       const uint32_t* __restrict__ hist7, const uint32_t* __restrict__ T, FsdInfo* __restrict__ infos,
                                                       uint8_t* __restrict__ out, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks) return;
    const int lane = threadIdx.x;
    const StageBlock blk = blocks[b];
    FsdInfo& I = infos[b];
    const uint32_t count = blk.len;
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const uint32_t count10 = count / 10, count5 = 2 * count10;
    uint32_t go = 0, dist = 0;
    int32_t dt_out = blk.data_type;
    int ent0 = 0;
    if (lane == 0) {
        go = count >= 1024 && blk.cap >= fsd_max_encoded_len(count);                                          // :145-153
        if (blk.data_type != DT_UNDEFINED && blk.data_type != DT_MULTIMEDIA && blk.data_type != DT_BIN) go = 0;  // :155-163
        if (go && !magic_allows_fsd(src, count)) go = 0;                                                        // :165-187
        if (go) {
            const uint32_t* h = hist7 + (size_t)b * 7 * 256;
            int ent[7];
            int min_idx = 0;
            for (int i = 0; i < 7; i++) {
                ent[i] = entropy_1024(3 * count10, h + i * 256, T);
                if (ent[i] < ent[min_idx]) min_idx = i;
            }
            ent0 = ent[0];
            if (ent[min_idx] >= ent[0]) {  // :236-243 the context gets whatever DetectSimpleType says, UNDEFINED included
                dt_out = detect_simple_type_dev(3 * count10, h);
                go = 0;
            } else {
                dt_out = DT_MULTIMEDIA;
                dist = fsd_dist((uint32_t)min_idx);
            }
        }
    }
    go = __shfl_sync(0xFFFFFFFFu, go, 0);
    dist = __shfl_sync(0xFFFFFFFFu, dist, 0);
    uint32_t mode = 0;
    if (go) {  // :253-268 xor coding when more than ~3 % of a sample are large deltas
        uint32_t large = 0;
        for (uint32_t i = 2 * count5 + lane; i < 3 * count5; i += 32) {
            const int delta = (int)src[i] - (int)src[i - dist];
            if (delta < -127 || delta > 127) large++;
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) large += __shfl_xor_sync(0xFFFFFFFFu, large, d);
        mode = large > (count5 >> 5) ? 1u : 0u;
    }
    if (lane == 0) {
        I.go = go;
        I.mode = mode;
        I.dist = dist;
        I.ent0 = ent0;
        I.out_len = 0;
        if (go) {
            dst[0] = (uint8_t)mode;
            dst[1] = (uint8_t)dist;
            for (uint32_t i = 0; i < dist; i++) dst[2 + i] = src[i];
        }
        StageResult r;
        r.status = 1;
        r.out_len = 0;
        r.data_type = dt_out;
        r.mode = mode | (dist << 8);
        res[b] = r;
    }
}

KZ_D uint32_t fsd_token_len(const uint8_t* src, uint32_t i, uint32_t dist) {
    const int d = (int)src[i] - (int)src[i - dist];
    return (d >= -127 && d <= 127) ? 1u : 2u;
}

// delta mode: bytes produced by every tile of 4096 positions (position p codes byte dist + p)
__global__ void __launch_bounds__(256) fsd_tiles_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const FsdInfo* __restrict__ infos,
                                                         uint32_t* __restrict__ tile_sum, uint32_t ntiles) {
    const int b = blockIdx.y;
    const FsdInfo& I = infos[b];
    if (!I.go || I.mode != 0) return;
    const StageBlock blk = blocks[b];
    const uint32_t npos = blk.len - I.dist;
    if ((uint64_t)blockIdx.x * FSD_TILE >= npos) return;
    __shared__ uint32_t s_sum[8];
    const uint8_t* src = in + blk.src_off;
    const uint32_t base = blockIdx.x * FSD_TILE + threadIdx.x * 16;
    uint32_t s = 0;
    for (uint32_t j = 0; j < 16; j++)
        if (base + j < npos) s += fsd_token_len(src, I.dist + base + j, I.dist);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, d);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < 8; w++) t += s_sum[w];
        tile_sum[(size_t)b * ntiles + blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(32) fsd_scan_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks, FsdInfo* __restrict__ infos,
                                                       const uint32_t* __restrict__ tile_sum, uint32_t* __restrict__ tile_off, uint32_t ntiles) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    FsdInfo& I = infos[b];
    if (!I.go) return;
    const StageBlock blk = blocks[b];
    const uint32_t count = blk.len, dist = I.dist;
    if (I.mode == 1) {  // xor coding: one byte per byte, the loop has no bound test (:287-293)
        I.out_len = count + 2;
        return;
    }
    const uint32_t npos = count - dist;
    const uint32_t nt = (npos + FSD_TILE - 1) / FSD_TILE;
    uint64_t off = 2 + dist;
    for (uint32_t t = 0; t < nt; t++) {
        tile_off[(size_t)b * ntiles + t] = (uint32_t)off;
        off += tile_sum[(size_t)b * ntiles + t];
    }
    // :271-286 the loop stops at dstIdx >= dstEnd - 1; it completes iff the last token starts below that bound
    const uint32_t dst_end = fsd_max_encoded_len(count);
    const uint32_t last = fsd_token_len(in + blk.src_off, count - 1, dist);
    if (off - last >= (uint64_t)dst_end - 1) {
        I.go = 0;  // :295-297 "output buffer too small": skip
        return;
    }
    I.out_len = (uint32_t)off;
}

__global__ void __launch_bounds__(256) fsd_emit_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, const FsdInfo* __restrict__ infos,
                                                        const uint32_t* __restrict__ tile_off, uint32_t ntiles, uint8_t* __restrict__ out) {
    const int b = blockIdx.y;
    const FsdInfo& I = infos[b];
    if (!I.go) return;
    const StageBlock blk = blocks[b];
    const uint32_t dist = I.dist, npos = blk.len - dist;
    if ((uint64_t)blockIdx.x * FSD_TILE >= npos) return;
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const uint32_t base = blockIdx.x * FSD_TILE + threadIdx.x * 16;
    if (I.mode == 1) {
        for (uint32_t j = 0; j < 16; j++) {
            const uint32_t p = base + j;
            if (p < npos) dst[2 + dist + p] = src[dist + p] ^ src[p];
        }
        return;
    }
    __shared__ uint32_t s_sum[8];
    uint32_t lens = 0, s = 0;  // bit j of lens: token j is an escape
    for (uint32_t j = 0; j < 16; j++)
        if (base + j < npos) {
            const uint32_t l = fsd_token_len(src, dist + base + j, dist);
            lens |= (l - 1) << j;
            s += l;
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
        const uint32_t p = base + j;
        if (p >= npos) break;
        const uint32_t cur = src[dist + p], prv = src[p];
        if ((lens >> j) & 1u) {
            dst[o] = 0xFF;  // _FSD_ESCAPE_TOKEN
            dst[o + 1] = (uint8_t)(cur ^ prv);
            o += 2;
        } else {
            const int d = (int)cur - (int)prv;  // _FSD_ZIGZAG1[127 + d]
            dst[o++] = (uint8_t)(d < 0 ? -2 * d - 1 : 2 * d);
        }
    }
}

// :296-310 histogram of two sub-ranges of the output
__global__ void __launch_bounds__(256) fsd_post_hist_kernel(const StageBlock* __restrict__ blocks, const FsdInfo* __restrict__ infos, const uint8_t* __restrict__ out,
                                                             uint32_t* __restrict__ hpost) {
    __shared__ uint32_t h[256];
    const int b = blockIdx.y;
    const FsdInfo& I = infos[b];
    if (!I.go) return;
    h[threadIdx.x] = 0;
    __syncthreads();
    const StageBlock blk = blocks[b];
    const uint32_t count10 = blk.len / 10, count5 = 2 * count10;
    const uint8_t* dst = out + blk.dst_off;
    for (uint32_t k = blockIdx.x * 256 + threadIdx.x; k < count10; k += gridDim.x * 256) {
        atomicAdd(&h[dst[count5 + k]], 1u);
        atomicAdd(&h[dst[3 * count5 + k]], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hpost[(size_t)b * 256 + threadIdx.x], h[threadIdx.x]);
}

__global__ void __launch_bounds__(32) fsd_final_kernel(const StageBlock* __restrict__ blocks, int nblocks, const FsdInfo* __restrict__ infos,
                                                        const uint32_t* __restrict__ hpost, const uint32_t* __restrict__ T, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const FsdInfo& I = infos[b];
    if (!I.go) return;
    const uint32_t count10 = blocks[b].len / 10, count5 = 2 * count10;
    if (entropy_1024(count5, hpost + (size_t)b * 256, T) >= I.ent0) return;  // "no improvement": skip
    StageResult r = res[b];
    r.status = 0;
    r.out_len = I.out_len;
    res[b] = r;
}

}  // namespace

size_t fsd_workspace(uint32_t nblocks, uint32_t max_len) {
    const size_t ntiles = (max_len + FSD_TILE - 1) / FSD_TILE + 1;
    return align256(257 * 4) + align256((size_t)nblocks * 7 * 256 * 4) + align256((size_t)nblocks * 256 * 4) + align256((size_t)nblocks * sizeof(FsdInfo)) +
           2 * align256((size_t)nblocks * ntiles * 4) + 256;
}

cudaError_t fsd_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint32_t max_len, uint8_t* ws, size_t ws_bytes,
                              StageResult* d_res, cudaStream_t stream, uint64_t* launches) {
    if (nblocks == 0) return cudaSuccess;
    if (ws_bytes < fsd_workspace(nblocks, max_len)) return cudaErrorInvalidValue;
    const Ws w = carve(ws, nblocks, max_len);
    cudaError_t e;
    if ((e = cudaMemcpyAsync(w.log2tab, host_log2_4096(), 257 * 4, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(w.hist7, 0, (size_t)nblocks * 7 * 256 * 4, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(w.hpost, 0, (size_t)nblocks * 256 * 4, stream)) != cudaSuccess) return e;
    const uint32_t gx = std::max<uint32_t>(1, (max_len + FSD_TILE - 1) / FSD_TILE);
    fsd_sample_kernel<<<dim3(SAMPLE_SLICES, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.hist7);
    fsd_plan_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.hist7, w.log2tab, w.info, d_out, d_res);
    fsd_tiles_kernel<<<dim3(gx, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, w.tile_sum, w.ntiles);
    fsd_scan_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.info, w.tile_sum, w.tile_off, w.ntiles);
    fsd_emit_kernel<<<dim3(gx, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.info, w.tile_off, w.ntiles, d_out);
    fsd_post_hist_kernel<<<dim3(SAMPLE_SLICES, nblocks), 256, 0, stream>>>(d_blocks, w.info, d_out, w.hpost);
    fsd_final_kernel<<<nblocks, 32, 0, stream>>>(d_blocks, (int)nblocks, w.info, w.hpost, w.log2tab, d_res);
    if (launches) *launches += 7;
    return cudaGetLastError();
}

// ---- inverse over tiles of 32 source bytes, all tiles of all blocks at once (FSDCodec.go:317-401) ---------------------------------------------
// out[o] = f(out[o - dist]) is `dist` interleaved chains; along a chain the delta tokens are a prefix sum (mod 256) and the rare escape
// tokens (0xFF + payload: out = payload ^ previous) cut it. A round of 32 source bytes, one per lane:
//   * which 0xFF bytes are escape markers is a parity question inside runs of 0xFF (a marker's successor is a payload, whatever its value),
//     answered with one ballot and a clz per lane;
//   * every byte that is not a marker is one output token; the k-th token moves to lane k;
//   * token values: inclusive shuffle scan with stride `dist` over the deltas (escape tokens count as 0) on top of the chain's value when
//     the round starts, then one correction per escape token of the round, in order: E = payload ^ value before it; every later token of
//     its chain moves by E - tentative value. XOR coding is the same scan with xor and no escapes.
// What a round carries into the next one is (a) whether its last byte was an escape marker, (b) the output offset, (c) the last value of
// each of the `dist` chains. (a) and (b) are decided by a scan over tiles: a tile's marker pattern depends on the
// incoming marker bit only through its leading run of 0xFF, so every tile is classified under both hypotheses (K1) and one warp per block
// chains them (K2). (c): along a chain the deltas are a prefix sum and every escape replaces the value by payload ^ previous, which is not
// a sum — but the escapes are few: each tile computes its chain totals and the list of its escapes with the delta sum in front of each
// (K3); the chain totals are scanned over the tiles (K3b), the escapes are compacted into one list per block (K3c) and one warp per block (lane =
// chain) walks that list only: corr = (payload ^ (linear value before + corr)) - linear value before (K4e). K5 is the round above with all
// three carries given.
namespace {
const int FSD_ESC_SLOTS = 17;  // escapes of a tile: marker + payload take two bytes, plus one whose marker ended the tile before
struct FsdiBlock {
    uint64_t src_off, dst_off;
    uint64_t tile_base;  // first tile of the block
    uint32_t len, cap;
    uint32_t ntiles, active;
};
struct FsdiState {  // per block, written by K2
    uint32_t bad, total, ntiles_ok, pad;
};
__device__ __forceinline__ bool fsdi_header(const uint8_t* src, uint32_t len, uint32_t cap, uint32_t& mode, uint32_t& dist) {
    if (len < 2) return false;
    mode = src[0];
    dist = src[1];
    if (dist < 1 || (dist > 4 && dist != 8 && dist != 16)) return false;
    if (len - 2 < dist || cap < dist || mode > 1) return false;
    return true;
}
// marker / payload / token masks of a tile (lane = source byte) under an incoming marker bit
__device__ __forceinline__ void fsdi_classify(uint32_t t, uint32_t cnt, uint32_t mode, uint32_t pending, uint32_t& marker, uint32_t& payload, uint32_t& tokens) {
    const int lane = threadIdx.x & 31;
    const uint32_t valid = cnt == 32 ? 0xFFFFFFFFu : ((1u << cnt) - 1u);
    marker = 0;
    if (mode == 0) {
        const uint32_t below = (1u << lane) - 1u;
        const uint32_t ff = __ballot_sync(0xFFFFFFFFu, t == 0xFFu) & valid;
        const uint32_t nz = ~ff & below;
        const uint32_t s = nz ? 32u - (uint32_t)__clz((int)nz) : 0u;
        const uint32_t par = (s == 0 && pending) ? 1u : 0u;
        const bool is_marker = ((ff >> lane) & 1u) && ((((uint32_t)lane - s) & 1u) == par);
        marker = __ballot_sync(0xFFFFFFFFu, is_marker);
    }
    payload = ((marker << 1) | pending) & valid;
    tokens = valid & ~marker;
}
// K1: one warp per tile: token count and outgoing marker bit under both hypotheses
__global__ void __launch_bounds__(128) fsdi_k1_kernel(const uint8_t* __restrict__ in, const FsdiBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_group,
                                                       uint32_t* __restrict__ rec) {
    const uint32_t gw = blockIdx.x * 4 + (threadIdx.x >> 5);  // global tile index; groups of 4 tiles never straddle blocks (tile_base % 4 == 0)
    const int lane = threadIdx.x & 31;
    const FsdiBlock& B = blocks[blk_of_group[blockIdx.x]];
    const uint32_t tl = gw - (uint32_t)B.tile_base;
    if (!B.active || tl >= B.ntiles) return;
    const uint8_t* src = in + B.src_off;
    uint32_t mode, dist;
    if (!fsdi_header(src, B.len, B.cap, mode, dist)) return;
    const uint32_t si = 2 + dist + 32 * tl;
    if (si >= B.len) return;
    const uint32_t cnt = min(32u, B.len - si);
    const uint32_t t = (uint32_t)lane < cnt ? src[si + lane] : 0u;
    uint32_t m0, p0, k0, m1, p1, k1;
    fsdi_classify(t, cnt, mode, 0, m0, p0, k0);
    fsdi_classify(t, cnt, mode, 1, m1, p1, k1);
    if (lane == 0) rec[gw] = (uint32_t)__popc(k0) | ((uint32_t)__popc(k1) << 8) | (((m0 >> (cnt - 1)) & 1u) << 16) | (((m1 >> (cnt - 1)) & 1u) << 17);
}
// K2: one CTA per block chains the tiles: a tile maps the incoming marker bit p to (outgoing bit, tokens) — a function with two cases,
// closed under composition — so the chain is a scan over those functions, 256 tiles per step. start[t] = output offset | p << 31.
struct FsdiFn {
    uint32_t po;      // bit p = outgoing marker bit for incoming bit p
    uint32_t c0, c1;  // tokens for incoming bit 0 / 1
};
__device__ __forceinline__ FsdiFn fsdi_then(const FsdiFn& a, const FsdiFn& b) {  // first a, then b
    FsdiFn r;
    const uint32_t a0 = a.po & 1u, a1 = (a.po >> 1) & 1u;
    r.po = ((b.po >> a0) & 1u) | (((b.po >> a1) & 1u) << 1);
    r.c0 = a.c0 + (a0 ? b.c1 : b.c0);
    r.c1 = a.c1 + (a1 ? b.c1 : b.c0);
    return r;
}
__global__ void __launch_bounds__(256) fsdi_k2_kernel(const uint8_t* __restrict__ in, const FsdiBlock* __restrict__ blocks, int nblocks, const uint32_t* __restrict__ rec,
                                                       uint32_t* __restrict__ start, FsdiState* __restrict__ st, uint8_t* __restrict__ out) {
    __shared__ FsdiFn s_w[8];
    __shared__ uint32_t s_ok;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (b >= nblocks) return;
    const FsdiBlock B = blocks[b];
    FsdiState S;
    S.bad = 0, S.total = 0, S.ntiles_ok = 0, S.pad = 0;
    if (!B.active) {
        if (tid == 0) st[b] = S;
        return;
    }
    const uint8_t* src = in + B.src_off;
    uint32_t mode, dist;
    if (!fsdi_header(src, B.len, B.cap, mode, dist)) {
        S.bad = 1;
        if (tid == 0) st[b] = S;
        return;
    }
    if ((uint32_t)tid < dist) out[B.dst_off + tid] = src[2 + tid];  // the first `dist` bytes are copied (:355-359)
    const uint32_t nt = (B.len - 2 - dist + 31) / 32;
    const uint32_t* r = rec + B.tile_base;
    uint32_t* sp = start + B.tile_base;
    if (tid == 0) s_ok = 0xFFFFFFFFu;
    FsdiFn carry;
    carry.po = 2u, carry.c0 = 0, carry.c1 = 0;  // identity
    __syncthreads();
    for (uint32_t t0 = 0; t0 < nt; t0 += 256) {
        const uint32_t t = t0 + tid;
        FsdiFn f;
        f.po = 2u, f.c0 = 0, f.c1 = 0;
        if (t < nt) {
            const uint32_t w = r[t];
            f.po = (w >> 16) & 3u, f.c0 = w & 0xFFu, f.c1 = (w >> 8) & 0xFFu;
        }
        FsdiFn inc = f;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            FsdiFn y;
            y.po = __shfl_up_sync(0xFFFFFFFFu, inc.po, d), y.c0 = __shfl_up_sync(0xFFFFFFFFu, inc.c0, d), y.c1 = __shfl_up_sync(0xFFFFFFFFu, inc.c1, d);
            if (lane >= d) inc = fsdi_then(y, inc);
        }
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        FsdiFn pre = carry, tot = carry;
        for (int w = 0; w < 8; w++) {
            if (w < warp) pre = fsdi_then(pre, s_w[w]);
            tot = fsdi_then(tot, s_w[w]);
        }
        FsdiFn ex;
        ex.po = __shfl_up_sync(0xFFFFFFFFu, inc.po, 1), ex.c0 = __shfl_up_sync(0xFFFFFFFFu, inc.c0, 1), ex.c1 = __shfl_up_sync(0xFFFFFFFFu, inc.c1, 1);
        if (lane == 0) ex.po = 2u, ex.c0 = 0, ex.c1 = 0;
        const FsdiFn before = fsdi_then(pre, ex);  // everything before this tile, from the block's start (incoming bit 0)
        if (t < nt) {
            const uint32_t p = before.po & 1u, di = dist + before.c0;
            sp[t] = di | (p << 31);
            const uint32_t tok = p ? f.c1 : f.c0;
            if ((uint64_t)di + tok > B.cap) atomicMin(&s_ok, t);  // the reference stops at dstEnd with source bytes left: an error (:398-400)
        }
        __syncthreads();
        carry = tot;
    }
    if (tid == 0) {
        const bool over = s_ok != 0xFFFFFFFFu;
        const bool bad = over || (carry.po & 1u);  // ... or a marker was the last source byte (:380-383)
        S.bad = bad ? 1u : 0u;
        S.total = over ? (sp[s_ok] & 0x7FFFFFFFu) : dist + carry.c0;
        S.ntiles_ok = over ? s_ok : nt;
        st[b] = S;
    }
}
// tokens of a tile in output order: lane k = token k (tk, is_esc) and its chain prefix (deltas on its chain inside the tile, escapes count 0)
__device__ __forceinline__ uint32_t fsdi_tokens(uint32_t t, uint32_t cnt, uint32_t mode, uint32_t dist, uint32_t pending, uint16_t* s_tok, uint32_t& tk, bool& is_esc,
                                                 uint32_t& prefix) {
    const int lane = threadIdx.x & 31;
    uint32_t marker, payload, tokens;
    fsdi_classify(t, cnt, mode, pending, marker, payload, tokens);
    const uint32_t m = (uint32_t)__popc(tokens);
    const uint32_t below = (1u << lane) - 1u;
    if ((tokens >> lane) & 1u) s_tok[__popc(tokens & below)] = (uint16_t)(t | (((payload >> lane) & 1u) << 8));
    __syncwarp();
    const uint32_t tw = (uint32_t)lane < m ? s_tok[lane] : 0u;
    __syncwarp();
    tk = tw & 0xFFu;
    is_esc = (tw >> 8) != 0;
    uint32_t v;
    if (mode == 0) v = is_esc ? 0u : ((tk & 1u) ? (0u - ((tk + 1u) >> 1)) : (tk >> 1));  // _FSD_ZIGZAG2
    else v = tk;
    if ((uint32_t)lane >= m) v = 0;
    for (uint32_t d = dist; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if ((uint32_t)lane >= d) v = mode == 0 ? v + y : v ^ y;
    }
    prefix = v & 0xFFu;
    return m;
}
// K3: chain totals and escape list of every tile
__global__ void __launch_bounds__(128) fsdi_k3_kernel(const uint8_t* __restrict__ in, const FsdiBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_group,
                                                       const FsdiState* __restrict__ st, const uint32_t* __restrict__ start, uint8_t* __restrict__ totals /*16 per tile*/,
                                                       uint32_t* __restrict__ esc /*FSD_ESC_SLOTS per tile*/, uint8_t* __restrict__ nesc) {
    __shared__ uint16_t s_tok_all[4][32];
    const uint32_t gw = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const uint32_t bi = blk_of_group[blockIdx.x];
    const FsdiBlock& B = blocks[bi];
    const uint32_t tl = gw - (uint32_t)B.tile_base;
    if (!B.active || tl >= st[bi].ntiles_ok) return;
    const uint8_t* src = in + B.src_off;
    const uint32_t mode = src[0], dist = src[1];
    const uint32_t si = 2 + dist + 32 * tl;
    const uint32_t cnt = min(32u, B.len - si);
    const uint32_t t = (uint32_t)lane < cnt ? src[si + lane] : 0u;
    const uint32_t sw = start[gw];
    uint32_t tk, prefix;
    bool is_esc;
    const uint32_t m = fsdi_tokens(t, cnt, mode, dist, sw >> 31, s_tok_all[threadIdx.x >> 5], tk, is_esc, prefix);
    const uint32_t di0 = sw & 0x7FFFFFFFu;
    // totals: the last token of each chain holds the chain's sum; chains without a token in the tile: 0
    if (lane < 16) totals[(size_t)gw * 16 + lane] = 0;
    __syncwarp();
    if ((uint32_t)lane < m && (uint32_t)lane + dist >= m) totals[(size_t)gw * 16 + (di0 + lane) % dist] = (uint8_t)prefix;
    const uint32_t em = __ballot_sync(0xFFFFFFFFu, is_esc);
    if (is_esc) esc[(size_t)gw * FSD_ESC_SLOTS + __popc(em & ((1u << lane) - 1u))] = ((di0 + lane) % dist) | (tk << 8) | (prefix << 16);  // chain, payload, deltas before it
    if (lane == 0) nesc[gw] = (uint8_t)__popc(em);
}
// K3b: per block, exclusive prefix over the tiles of (a) the escape counts and (b) the 16 chain totals (bytes: add modulo 256, or xor) — one CTA
// per block, 256 tiles per step, the 16 bytes of a tile scanned as four words of four byte lanes
__device__ __forceinline__ uint32_t fsdi_add4(uint32_t a, uint32_t b) {  // four independent byte additions
    return ((a & 0x7F7F7F7Fu) + (b & 0x7F7F7F7Fu)) ^ ((a ^ b) & 0x80808080u);
}
__global__ void __launch_bounds__(256) fsdi_k3b_kernel(const uint8_t* __restrict__ in, const FsdiBlock* __restrict__ blocks, int nblocks, const FsdiState* __restrict__ st,
                                                        const uint8_t* __restrict__ totals, const uint8_t* __restrict__ nesc, uint8_t* __restrict__ ptile /*16 per tile*/,
                                                        uint32_t* __restrict__ esc_base, uint32_t* __restrict__ esc_total) {
    __shared__ uint4 s_w[8];
    __shared__ uint32_t s_c[8];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (b >= nblocks) return;
    const FsdiBlock B = blocks[b];
    const uint32_t nt = st[b].ntiles_ok;
    if (!B.active || nt == 0) {
        if (tid == 0) esc_total[b] = 0;
        return;
    }
    const bool is_xor = in[B.src_off] != 0;
    const size_t tb = B.tile_base;
    uint4 carry = make_uint4(0, 0, 0, 0);
    uint32_t ccount = 0;
    auto comb = [&](uint4 a, uint4 c) {
        return is_xor ? make_uint4(a.x ^ c.x, a.y ^ c.y, a.z ^ c.z, a.w ^ c.w) : make_uint4(fsdi_add4(a.x, c.x), fsdi_add4(a.y, c.y), fsdi_add4(a.z, c.z), fsdi_add4(a.w, c.w));
    };
    for (uint32_t t0 = 0; t0 < nt; t0 += 256) {
        const uint32_t t = t0 + tid;
        uint4 v = make_uint4(0, 0, 0, 0);
        uint32_t c = 0;
        if (t < nt) {
            v = *reinterpret_cast<const uint4*>(totals + (tb + t) * 16);
            c = nesc[tb + t];
        }
        uint4 iv = v;
        uint32_t ic = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint4 y;
            y.x = __shfl_up_sync(0xFFFFFFFFu, iv.x, d), y.y = __shfl_up_sync(0xFFFFFFFFu, iv.y, d), y.z = __shfl_up_sync(0xFFFFFFFFu, iv.z, d), y.w = __shfl_up_sync(0xFFFFFFFFu, iv.w, d);
            const uint32_t yc = __shfl_up_sync(0xFFFFFFFFu, ic, d);
            if (lane >= d) iv = comb(iv, y), ic += yc;
        }
        if (lane == 31) s_w[warp] = iv, s_c[warp] = ic;
        __syncthreads();
        uint4 pre = carry;
        uint32_t prec = ccount;
        uint4 tot = carry;
        uint32_t totc = ccount;
        for (int w = 0; w < 8; w++) {
            if (w < warp) pre = comb(pre, s_w[w]), prec += s_c[w];
            tot = comb(tot, s_w[w]), totc += s_c[w];
        }
        // exclusive: everything before this tile
        uint4 ev;
        ev.x = __shfl_up_sync(0xFFFFFFFFu, iv.x, 1), ev.y = __shfl_up_sync(0xFFFFFFFFu, iv.y, 1), ev.z = __shfl_up_sync(0xFFFFFFFFu, iv.z, 1), ev.w = __shfl_up_sync(0xFFFFFFFFu, iv.w, 1);
        uint32_t ec = __shfl_up_sync(0xFFFFFFFFu, ic, 1);
        if (lane == 0) ev = make_uint4(0, 0, 0, 0), ec = 0;
        if (t < nt) {
            *reinterpret_cast<uint4*>(ptile + (tb + t) * 16) = comb(pre, ev);
            esc_base[tb + t] = prec + ec;
        }
        __syncthreads();
        carry = tot;
        ccount = totc;
    }
    if (tid == 0) esc_total[b] = ccount;
}
// K3c: the escapes of every tile into the block's flat list (two words: chain | payload << 8 | deltas before << 16, tile)
__global__ void __launch_bounds__(256) fsdi_k3c_kernel(const FsdiBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_group, const FsdiState* __restrict__ st,
                                                        const uint32_t* __restrict__ esc, const uint8_t* __restrict__ nesc, const uint32_t* __restrict__ esc_base,
                                                        uint2* __restrict__ flat) {
    const uint32_t gt = blockIdx.x * 4 + (threadIdx.x >> 6);  // 64 threads per tile slot group: thread j < nesc copies escape j
    const int j = threadIdx.x & 63;
    const uint32_t bi = blk_of_group[blockIdx.x];
    const FsdiBlock& B = blocks[bi];
    const uint32_t tl = gt - (uint32_t)B.tile_base;
    if (!B.active || tl >= st[bi].ntiles_ok) return;
    if (j < (int)nesc[gt]) flat[(size_t)B.tile_base * FSD_ESC_SLOTS + esc_base[gt] + j] = make_uint2(esc[(size_t)gt * FSD_ESC_SLOTS + j], tl);
}
// K4 (escape list version): one warp per block walks the block's ESCAPES only; corr[c] = what has to be added to
// (first value of chain c + chain prefix) behind the escapes so far. After every escape the 16 corrections are stored.
__global__ void __launch_bounds__(32) fsdi_k4e_kernel(const uint8_t* __restrict__ in, const FsdiBlock* __restrict__ blocks, int nblocks, const FsdiState* __restrict__ st,
                                                       const uint2* __restrict__ flat, const uint32_t* __restrict__ esc_total, const uint8_t* __restrict__ ptile,
                                                       uint8_t* __restrict__ corrvec /*16 per escape*/) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const FsdiBlock B = blocks[b];
    const uint32_t ne = esc_total[b];
    if (!B.active || st[b].ntiles_ok == 0 || ne == 0) return;
    const uint8_t* src = in + B.src_off;
    const uint32_t dist = src[1];
    const uint32_t c = (uint32_t)lane & 15u;
    const uint32_t r0 = c < dist ? src[2 + c] : 0u;
    const size_t tb = B.tile_base, eb0 = (size_t)B.tile_base * FSD_ESC_SLOTS;  // first tile / first escape slot of the block
    uint32_t corr = 0;
    auto fetch = [&](uint32_t e0, uint32_t& w, uint32_t& pt) {
        w = 0, pt = 0;
        if (e0 + lane < ne) {
            const uint2 f = flat[eb0 + e0 + lane];
            w = f.x;
            pt = ptile[(tb + f.y) * 16 + (f.x & 0xFFu)];
        }
    };
    uint32_t wn, ptn;
    fetch(0, wn, ptn);
    for (uint32_t e0 = 0; e0 < ne; e0 += 32) {
        const uint32_t wc = wn, ptc = ptn;
        fetch(e0 + 32, wn, ptn);  // next 32 escapes in flight
        const uint32_t n = min(32u, ne - e0);
        for (uint32_t j = 0; j < n; j++) {
            const uint32_t w = __shfl_sync(0xFFFFFFFFu, wc, (int)j), pt = __shfl_sync(0xFFFFFFFFu, ptc, (int)j);
            const uint32_t pay = (w >> 8) & 0xFFu, pl = (w >> 16) & 0xFFu;
            if ((w & 0xFFu) == c) {
                const uint32_t lin = (r0 + pt + pl) & 0xFFu;           // value before the escape without corrections
                corr = ((pay ^ ((lin + corr) & 0xFFu)) - lin) & 0xFFu;  // the escape's value is payload ^ (value before it)
            }
            if (lane < 16) corrvec[(eb0 + e0 + j) * 16 + lane] = (uint8_t)corr;
        }
    }
}

// K5: the bytes of every tile
__global__ void __launch_bounds__(128) fsdi_k5_kernel(const uint8_t* __restrict__ in, const FsdiBlock* __restrict__ blocks, const uint32_t* __restrict__ blk_of_group,
                                                       const FsdiState* __restrict__ st, const uint32_t* __restrict__ start, const uint8_t* __restrict__ ptile,
                                                       const uint32_t* __restrict__ esc_base, const uint8_t* __restrict__ corrvec, uint8_t* __restrict__ out) {
    __shared__ uint16_t s_tok_all[4][32];
    const uint32_t gw = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const uint32_t bi = blk_of_group[blockIdx.x];
    const FsdiBlock& B = blocks[bi];
    const uint32_t tl = gw - (uint32_t)B.tile_base;
    if (!B.active || st[bi].bad || tl >= st[bi].ntiles_ok) return;
    const uint8_t* src = in + B.src_off;
    const uint32_t mode = src[0], dist = src[1];
    const uint32_t si = 2 + dist + 32 * tl;
    const uint32_t cnt = min(32u, B.len - si);
    const uint32_t t = (uint32_t)lane < cnt ? src[si + lane] : 0u;
    const uint32_t sw = start[gw];
    uint32_t tk, prefix;
    bool is_esc;
    const uint32_t m = fsdi_tokens(t, cnt, mode, dist, sw >> 31, s_tok_all[threadIdx.x >> 5], tk, is_esc, prefix);
    const uint32_t di0 = sw & 0x7FFFFFFFu;
    // the chain's value when the tile starts: first value of the chain, chain totals of the tiles before, corrections of the escapes before
    const uint32_t ch = (di0 + lane) % dist;
    const uint32_t pt = ptile[(size_t)gw * 16 + ch];
    const uint32_t eb = esc_base[gw];
    const uint32_t cr = eb ? corrvec[((size_t)B.tile_base * FSD_ESC_SLOTS + eb - 1) * 16 + ch] : 0u;
    const uint32_t base = mode == 0 ? (src[2 + ch] + pt + cr) & 0xFFu : (src[2 + ch] ^ pt);
    uint32_t v = (mode == 0 ? prefix + base : prefix ^ base) & 0xFFu;
    if (mode == 0) {
        uint32_t em = __ballot_sync(0xFFFFFFFFu, is_esc);
        while (em) {  // escapes of the tile in order
            const int e = __ffs((int)em) - 1;
            em &= em - 1;
            const uint32_t prev_in = __shfl_sync(0xFFFFFFFFu, v, e >= (int)dist ? e - (int)dist : 0);
            const uint32_t prev_old = __shfl_sync(0xFFFFFFFFu, base, e);  // lane e's chain value at the tile start
            const uint32_t prev = e >= (int)dist ? prev_in : prev_old;
            const uint32_t tent = __shfl_sync(0xFFFFFFFFu, v, e);
            const uint32_t pay = __shfl_sync(0xFFFFFFFFu, tk, e);
            const uint32_t delta = ((pay ^ prev) - tent) & 0xFFu;
            if (lane >= e && ((uint32_t)(lane - e) % dist) == 0) v = (v + delta) & 0xFFu;
        }
    }
    if ((uint32_t)lane < m) out[B.dst_off + di0 + lane] = (uint8_t)v;
}
__global__ void fsdi_result_kernel(const FsdiBlock* __restrict__ blocks, int nblocks, const FsdiState* __restrict__ st, StageResult* __restrict__ res) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    StageResult r;
    r.status = 0, r.out_len = 0, r.data_type = 0, r.mode = 0;
    if (blocks[b].active) {
        r.out_len = st[b].total;
        if (st[b].bad) r.status = -KZ_E_PROCESS_BLOCK;
    }
    res[b] = r;
}
}  // namespace

size_t fsd_inverse_workspace(uint32_t nblocks, uint64_t total_len) {
    const size_t tiles = (size_t)total_len / 32 + 8 * (size_t)nblocks + 8;
    return tiles * (4 + 4 + 16 + 16 + 1 + 4 * FSD_ESC_SLOTS + 1 + 4 + (8 + 16) * FSD_ESC_SLOTS) + (size_t)nblocks * (sizeof(FsdiBlock) + sizeof(FsdiState) + 4) + 24 * 256 + 4096;
}

// FSDCodec.Inverse of a batch over tiles (kernels above); h_blocks: the descriptors on the host.
cudaError_t fsd_inverse_tiles(const uint8_t* d_in, uint8_t* d_out, const StageBlock* h_blocks, uint32_t nblocks, uint8_t* ws, size_t ws_bytes, StageResult* d_res,
                              cudaStream_t stream, uint64_t* launches) {
    if (nblocks == 0) return cudaSuccess;
    std::vector<FsdiBlock> hb(nblocks);
    std::vector<uint32_t> blk_of_group;
    uint64_t tiles = 0;
    for (uint32_t b = 0; b < nblocks; b++) {
        FsdiBlock& B = hb[b];
        B.src_off = h_blocks[b].src_off, B.dst_off = h_blocks[b].dst_off, B.len = h_blocks[b].len, B.cap = h_blocks[b].cap;
        B.active = (h_blocks[b].len != 0 && h_blocks[b].cap != 0) ? 1u : 0u;
        B.ntiles = B.active ? (B.len + 31) / 32 : 0;  // upper bound (the header and the first `dist` bytes are not tiled)
        B.tile_base = tiles;
        const uint32_t groups = (B.ntiles + 3) / 4;
        for (uint32_t g = 0; g < groups; g++) blk_of_group.push_back(b);
        tiles += (uint64_t)groups * 4;
    }
    auto align = [](size_t x) { return (x + 255) & ~size_t(255); };
    size_t off = 0;
    FsdiBlock* d_b = (FsdiBlock*)(ws + off); off = align(off + nblocks * sizeof(FsdiBlock));
    FsdiState* d_st = (FsdiState*)(ws + off); off = align(off + nblocks * sizeof(FsdiState));
    uint32_t* d_bog = (uint32_t*)(ws + off); off = align(off + (blk_of_group.size() + 1) * 4);
    uint32_t* d_rec = (uint32_t*)(ws + off); off = align(off + (tiles + 4) * 4);
    uint32_t* d_start = (uint32_t*)(ws + off); off = align(off + (tiles + 4) * 4);
    uint8_t* d_tot = ws + off; off = align(off + (tiles + 4) * 16);
    uint8_t* d_snap = ws + off; off = align(off + (tiles + 4) * 16);
    uint8_t* d_nesc = ws + off; off = align(off + (tiles + 4));
    uint32_t* d_esc = (uint32_t*)(ws + off); off = align(off + (tiles + 4) * 4 * FSD_ESC_SLOTS);
    uint32_t* d_ebase = (uint32_t*)(ws + off); off = align(off + (tiles + 4) * 4);
    uint32_t* d_etot = (uint32_t*)(ws + off); off = align(off + (size_t)nblocks * 4 + 64);
    uint2* d_flat = (uint2*)(ws + off); off = align(off + (tiles + 4) * 8 * FSD_ESC_SLOTS);
    uint8_t* d_corr = ws + off; off = align(off + (tiles + 4) * 16 * FSD_ESC_SLOTS);
    if (off > ws_bytes) return cudaErrorInvalidValue;
    cudaError_t e;
    if ((e = cudaMemcpyAsync(d_b, hb.data(), nblocks * sizeof(FsdiBlock), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    const uint32_t groups = (uint32_t)blk_of_group.size();
    if (groups) {
        if ((e = cudaMemcpyAsync(d_bog, blk_of_group.data(), (size_t)groups * 4, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
        fsdi_k1_kernel<<<groups, 128, 0, stream>>>(d_in, d_b, d_bog, d_rec);
    }
    fsdi_k2_kernel<<<nblocks, 256, 0, stream>>>(d_in, d_b, (int)nblocks, d_rec, d_start, d_st, d_out);
    if (groups) {
        fsdi_k3_kernel<<<groups, 128, 0, stream>>>(d_in, d_b, d_bog, d_st, d_start, d_tot, d_esc, d_nesc);
        fsdi_k3b_kernel<<<nblocks, 256, 0, stream>>>(d_in, d_b, (int)nblocks, d_st, d_tot, d_nesc, d_snap /* = chain prefixes per tile */, d_ebase, d_etot);
        fsdi_k3c_kernel<<<groups, 256, 0, stream>>>(d_b, d_bog, d_st, d_esc, d_nesc, d_ebase, d_flat);
        fsdi_k4e_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_b, (int)nblocks, d_st, d_flat, d_etot, d_snap, d_corr);
        fsdi_k5_kernel<<<groups, 128, 0, stream>>>(d_in, d_b, d_bog, d_st, d_start, d_snap, d_ebase, d_corr, d_out);
    }
    fsdi_result_kernel<<<(nblocks + 127) / 128, 128, 0, stream>>>(d_b, (int)nblocks, d_st, d_res);
    if (launches) *launches += 8;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;  // hb / blk_of_group go out of scope
    return cudaGetLastError();
}

}  // namespace kz
