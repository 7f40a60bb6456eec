// UTF transform (UTFCodec) on the GPU. The validation (byte and digram histograms of the block, transform/UTFCodec.go:393-515) runs in
// parallel and settles most blocks: anything that is not UTF-8 with enough multi-byte sequences is declined there. Blocks that go on are
// walked by one thread each with the logic of kz_utf_core.cuh (code point counts in a 2^22-entry map, ranks by frequency, alias
// emission): the rank of a code point depends on the counts of the whole block, and the parse is a chain of 1..4 byte steps.
#include <algorithm>

#include "kz_utf.cuh"
#include "kz_utf_core.cuh"

namespace kz {

using namespace utfc;

namespace {

const int DT_UNDEFINED = 0, DT_UTF8 = 8;
const uint32_t HIST_SLICES = 32, ZERO_SLICES = 64;

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct Ws {
    uint32_t* hist0;    // [nblocks][256]
    uint32_t* hist1;    // [nblocks][65536]
    uint32_t* forb;     // [nblocks] forbidden bytes inside the window validateUTF checks
    uint32_t* go;       // [nblocks] 0x100 | start when the walk has to run
    int32_t* alias_map; // [nblocks][1 << 22]
    uint64_t* keys;     // [nblocks][32768]
};
Ws carve(uint8_t* ws, uint32_t nblocks) {
    Ws w;
    uint8_t* p = ws;
    w.hist0 = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 256 * 4);
    w.hist1 = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 65536 * 4);
    w.forb = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 4);
    w.go = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 4);
    w.alias_map = reinterpret_cast<int32_t*>(p);
    p += align256((size_t)nblocks * ALIAS_MAP_SIZE * 4);
    w.keys = reinterpret_cast<uint64_t*>(p);
    return w;
}

KZ_D bool forward_candidate(const StageBlock& blk) {  // :92-114
    if (blk.len < (uint32_t)MIN_BLOCKSIZE || (uint64_t)blk.cap < (uint64_t)blk.len + 8192) return false;
    return blk.data_type == DT_UNDEFINED || blk.data_type == DT_UTF8;
}

// histograms of block = src[start : count - 4] for validateUTF (only needed when the data type is not already UTF-8)
__global__ void __launch_bounds__(256) utf_hist_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, uint32_t* __restrict__ hist0,
                                                        uint32_t* __restrict__ hist1, uint32_t* __restrict__ forb) {
    __shared__ uint32_t h[256];
    __shared__ uint32_t s_forb;
    const int b = blockIdx.y;
    const StageBlock blk = blocks[b];
    if (!forward_candidate(blk) || blk.data_type == DT_UTF8) return;
    h[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_forb = 0;
    __syncthreads();
    const uint8_t* src = in + blk.src_off;
    const int start = utf_start(src);
    const uint8_t* p = src + start;
    const uint32_t len = blk.len - 4 - (uint32_t)start;
    const uint32_t checked = validate_checked_len(len);
    uint32_t* h1 = hist1 + (size_t)b * 65536;
    const uint32_t per = (len + HIST_SLICES - 1) / HIST_SLICES;
    const uint32_t lo = blockIdx.x * per, hi = min(len, lo + per);
    uint32_t f = 0;
    for (uint32_t i = lo + threadIdx.x; i < hi; i += 256) {
        const uint32_t cur = p[i], prv = i ? p[i - 1] : 0u;
        atomicAdd(&h[cur], 1u);
        // validate_utf reads only the rows of the lead bytes C2..F4: the other digrams are not counted
        if (prv >= 0xC2u) atomicAdd(&h1[(prv << 8) | cur], 1u);
        if (i < checked && forbidden_byte((uint8_t)cur)) f++;
    }
    if (f) atomicAdd(&s_forb, f);
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist0[(size_t)b * 256 + threadIdx.x], h[threadIdx.x]);
    if (threadIdx.x == 0 && s_forb) atomicAdd(&forb[b], s_forb);
}

__global__ void __launch_bounds__(32) utf_plan_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                       const uint32_t* __restrict__ hist0, const uint32_t* __restrict__ hist1, const uint32_t* __restrict__ forb,
                                                       uint32_t* __restrict__ go, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const StageBlock blk = blocks[b];
    StageResult r;
    r.status = 1;
    r.out_len = 0;
    r.data_type = blk.data_type;
    r.mode = 0;
    go[b] = 0;
    if (forward_candidate(blk)) {
        const int start = utf_start(in + blk.src_off);
        bool ok = true;
        if (blk.data_type != DT_UTF8)
            ok = validate_utf(hist0 + (size_t)b * 256, hist1 + (size_t)b * 65536, blk.len - 4 - (uint32_t)start, forb[b]);
        if (ok) {
            r.data_type = DT_UTF8;  // :133-135
            go[b] = 0x100u | (uint32_t)start;
        }
    }
    res[b] = r;
}

__global__ void __launch_bounds__(256) utf_zero_kernel(const uint32_t* __restrict__ go, int32_t* __restrict__ alias_all) {
    const int b = blockIdx.y;
    if (!(go[b] & 0x100u)) return;
    int4* m = reinterpret_cast<int4*>(alias_all + (size_t)b * ALIAS_MAP_SIZE);
    for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i < ALIAS_MAP_SIZE / 4; i += gridDim.x * 256) m[i] = make_int4(0, 0, 0, 0);
}

__global__ void __launch_bounds__(32) utf_forward_walk_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                               const uint32_t* __restrict__ go, int32_t* __restrict__ alias_all, uint64_t* __restrict__ keys_all,
                                                               uint8_t* __restrict__ out, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    if (!(go[b] & 0x100u)) return;
    const StageBlock blk = blocks[b];
    const int64_t n = forward_walk(in + blk.src_off, (int)blk.len, (int)(go[b] & 0xFF), out + blk.dst_off, alias_all + (size_t)b * ALIAS_MAP_SIZE,
                                   keys_all + (size_t)b * MAX_SYMBOLS);
    if (n >= 0) {
        StageResult r = res[b];
        r.status = 0;
        r.out_len = (uint32_t)n;
        res[b] = r;
    }
}

__global__ void __launch_bounds__(32) utf_inverse_walk_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                               uint64_t* __restrict__ scratch_all, uint8_t* __restrict__ out, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const StageBlock blk = blocks[b];
    StageResult r;
    r.status = 0;
    r.out_len = 0;
    r.data_type = 0;
    r.mode = 0;
    if (blk.len != 0 && blk.cap != 0) {
        Sym* m = reinterpret_cast<Sym*>(scratch_all + (size_t)b * MAX_SYMBOLS);  // 8 bytes per entry, like the keys
        const int64_t n = inverse_walk(in + blk.src_off, (int)blk.len, out + blk.dst_off, (int64_t)blk.cap, m);
        if (n < 0) r.status = -KZ_E_PROCESS_BLOCK;
        else r.out_len = (uint32_t)n;
    }
    res[b] = r;
}

}  // namespace

size_t utf_workspace(uint32_t nblocks) {
    return align256((size_t)nblocks * 256 * 4) + align256((size_t)nblocks * 65536 * 4) + 2 * align256((size_t)nblocks * 4) +
           align256((size_t)nblocks * ALIAS_MAP_SIZE * 4) + align256((size_t)nblocks * MAX_SYMBOLS * 8) + 256;
}

cudaError_t utf_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint8_t* ws, size_t ws_bytes, StageResult* d_res,
                              cudaStream_t stream, uint64_t* launches) {
    static_assert(sizeof(Sym) == 8, "inverse scratch shares the key array");
    if (nblocks == 0) return cudaSuccess;
    if (ws_bytes < utf_workspace(nblocks)) return cudaErrorInvalidValue;
    const Ws w = carve(ws, nblocks);
    cudaError_t e;
    if ((e = cudaMemsetAsync(w.hist0, 0, (size_t)nblocks * 256 * 4, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(w.hist1, 0, (size_t)nblocks * 65536 * 4, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(w.forb, 0, (size_t)nblocks * 4, stream)) != cudaSuccess) return e;
    utf_hist_kernel<<<dim3(HIST_SLICES, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.hist0, w.hist1, w.forb);
    utf_plan_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.hist0, w.hist1, w.forb, w.go, d_res);
    utf_zero_kernel<<<dim3(ZERO_SLICES, nblocks), 256, 0, stream>>>(w.go, w.alias_map);
    utf_forward_walk_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.go, w.alias_map, w.keys, d_out, d_res);
    if (launches) *launches += 4;
    return cudaGetLastError();
}

cudaError_t utf_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, uint32_t nblocks, uint8_t* ws, size_t ws_bytes, StageResult* d_res,
                              cudaStream_t stream, uint64_t* launches) {
    if (nblocks == 0) return cudaSuccess;
    if (ws_bytes < utf_workspace(nblocks)) return cudaErrorInvalidValue;
    const Ws w = carve(ws, nblocks);
    utf_inverse_walk_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.keys, d_out, d_res);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace kz
