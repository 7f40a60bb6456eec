// TEXT transform (TextCodec, encoding 2) on the GPU: statistics and dictionary set-up in parallel, then one thread per block walks the
// words with the state machine of kz_text_core.cuh (the dictionary — which words were seen, at which index, which entries were recycled —
// is the state of that walk: every decision depends on all earlier words of the block). Blocks of a batch run side by side.
// Reference: v2/transform/TextCodec.go (see kz_text_core.cuh for the line map).
#include <algorithm>
#include <vector>

#include "kz_text.cuh"
#include "kz_text_core.cuh"
#include "kz_text_par.cuh"

#if __has_include("_gen/kz_text_dict.inc")
#include "_gen/kz_text_dict.inc"
#define KZ_HAVE_TEXT_DICT 1
#else
#define KZ_HAVE_TEXT_DICT 0
#endif

namespace kz {

using namespace textc;

bool text_available() { return KZ_HAVE_TEXT_DICT != 0; }

namespace {

const int DT_UNDEFINED = 0, DT_TEXT = 1, DT_BIN = 7;
const uint32_t HIST_SLICES = 32, INIT_SLICES = 32;
const uint32_t SWORDS_BYTES = 8192;  // room for the letters of the static dictionary (5487)

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// block b's hash map: 1 << log slots at map + off (text_map_layout)
struct MapSlice {
    uint64_t off;
    uint32_t log, pad;
};

struct Ws {
    Entry* sdict;      // [1024] static entries
    uint8_t* swords;   // lower-cased letters
    uint32_t* hist0;   // [nblocks][256]
    uint32_t* hist1;   // [nblocks][65536]
    uint32_t* go;      // [nblocks] mode byte | 0x100 when the walk has to run
    MapSlice* slice;   // [nblocks] where each block's map lies (uploaded only when a serial walk runs)
    int32_t* map;      // the maps of all blocks, back to back
    Entry* list;       // [nblocks][MAX_DICT_SIZE]
    std::vector<MapSlice> h_slice;
};
Ws carve(uint8_t* ws, uint32_t nblocks, const uint64_t* bs) {
    Ws w;
    std::vector<uint64_t> off;
    std::vector<uint32_t> lg;
    const uint64_t slots = text_map_layout(bs, nblocks, off, lg);
    w.h_slice.resize(nblocks);
    for (uint32_t b = 0; b < nblocks; b++) w.h_slice[b] = MapSlice{off[b], lg[b], 0};
    uint8_t* p = ws;
    w.sdict = reinterpret_cast<Entry*>(p);
    p += align256(sizeof(Entry) * STATIC_WORDS);
    w.swords = p;
    p += align256(SWORDS_BYTES);
    w.hist0 = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 256 * 4);
    w.hist1 = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 65536 * 4);
    w.go = reinterpret_cast<uint32_t*>(p);
    p += align256((size_t)nblocks * 4);
    w.slice = reinterpret_cast<MapSlice*>(p);
    p += align256((size_t)nblocks * sizeof(MapSlice));
    w.map = reinterpret_cast<int32_t*>(p);
    p += align256((size_t)slots * 4);
    w.list = reinterpret_cast<Entry*>(p);
    return w;
}

#if KZ_HAVE_TEXT_DICT
struct HostStatic {
    std::vector<uint8_t> words;
    std::vector<Entry> entries;
    int n = 0;
    HostStatic() {
        const int len = (int)sizeof(KZ_TC_DICT_EN_1024) - 1;
        words.assign(KZ_TC_DICT_EN_1024, KZ_TC_DICT_EN_1024 + len);
        words.resize(SWORDS_BYTES, 0);
        entries.resize(STATIC_WORDS);
        n = create_static_dictionary(words.data(), len, entries.data());
    }
};
const HostStatic& host_static() {
    static const HostStatic s;
    return s;
}
#endif

// internal/Magic.go:73-112: does GetMagicType recognise the first four bytes?
KZ_D bool has_magic(const uint8_t* p, uint32_t n) {
    if (n < 4) return false;
    const uint32_t key = ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
    if ((key & ~0x0Fu) == 0xFFD8FFE0u) return true;
    if ((key >> 8) == 0x425A68u || (key >> 8) == 0x494433u) return true;
    const uint32_t k32[18] = {0x47494638u, 0x25504446u, 0x504B0304u, 0x377ABCAFu, 0x89504E47u, 0x7F454C46u, 0xFEEDFACEu, 0xCEFAEDFEu, 0xFEEDFACFu,
                              0xCFFAEDFEu, 0x28B52FFDu, 0x81CFB2CEu, 0x4D534346u, 0x52494646u, 0x664C6143u, 0xFD377A58u, 0x4B414E5Au, 0x52617221u};
    for (int i = 0; i < 18; i++)
        if (key == k32[i]) return true;
    const uint32_t k16 = key >> 16;
    if (k16 == 0x1F8Bu || k16 == 0x424Du || k16 == 0x4D5Au) return true;
    if (k16 == 0x5034u || k16 == 0x5035u || k16 == 0x5036u) {
        const uint32_t sub = (key >> 8) & 0xFF;
        if (sub == 0x07 || sub == 0x0A || sub == 0x0D || sub == 0x20) return true;
    }
    return false;
}

KZ_D bool forward_candidate(const StageBlock& blk) {  // wrapper :549-560, Forward :1228-1241
    if (blk.len < 1024 || blk.len > (1u << 30) || blk.cap < blk.len) return false;
    return blk.data_type == DT_UNDEFINED || blk.data_type == DT_TEXT || blk.data_type == DT_BIN;
}

// byte histogram (shared memory) and the read part of the (previous byte, byte) histogram (L2 atomics), previous = 0 for the first byte (:196-222)
__global__ void __launch_bounds__(256) text_hist_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, uint32_t* __restrict__ hist0,
                                                         uint32_t* __restrict__ hist1) {
    __shared__ uint32_t h[256];
    const int b = blockIdx.y;
    const StageBlock blk = blocks[b];
    if (!forward_candidate(blk)) return;
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint8_t* src = in + blk.src_off;
    uint32_t* h1 = hist1 + (size_t)b * 65536;
    const uint32_t per = (blk.len + HIST_SLICES - 1) / HIST_SLICES;
    const uint32_t lo = blockIdx.x * per, hi = min(blk.len, lo + per);
    for (uint32_t i = lo + threadIdx.x; i < hi; i += 256) {
        const uint32_t cur = src[i], prv = i ? src[i - 1] : 0u;
        atomicAdd(&h[cur], 1u);
        // the statistics read four families of digram counters only (kz_text_core.cuh: text_stats_mode / detect_text_type): row '&' (XML entities),
        // row CR and column LF (line ends), rows 0xC2..0xF4 (UTF-8 lead bytes). The frequent digrams of a text ('e ', ' t', ...) are none of
        // these: counting them cost milliseconds per 200 MB in contended L2 atomics and nobody read the result.
        if (prv == 0x26u || prv == 0x0Du || cur == 0x0Au || prv >= 0xC2u) atomicAdd(&h1[(prv << 8) | cur], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist0[(size_t)b * 256 + threadIdx.x], h[threadIdx.x]);
}

__global__ void __launch_bounds__(32) text_plan_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                        const uint32_t* __restrict__ hist0, const uint32_t* __restrict__ hist1, uint32_t* __restrict__ go,
                                                        StageResult* __restrict__ res) {
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
        const uint8_t mode = text_stats_mode(hist0 + (size_t)b * 256, hist1 + (size_t)b * 65536, (int)blk.len, has_magic(in + blk.src_off, blk.len));
        if (mode & MASK_NOT_TEXT) {
            r.data_type = mode & MASK_DT;  // :1247-1251
        } else {
            r.data_type = DT_TEXT;
            r.mode = mode;
            go[b] = 0x100u | mode;
        }
    }
    res[b] = r;
}

// dictionary set-up of the blocks that go on: empty map, list = static entries followed by {hash 0, data i, no word} (reset :1190-1223)
__global__ void __launch_bounds__(256) text_init_kernel(const uint32_t* __restrict__ go, const Entry* __restrict__ sdict, int static_n, int32_t* __restrict__ map_all,
                                                         const MapSlice* __restrict__ slice, Entry* __restrict__ list_all) {
    const int b = blockIdx.y;
    if (go && !(go[b] & 0x100u)) return;
    int32_t* map = map_all + slice[b].off;
    const uint32_t log = slice[b].log;
    Entry* list = list_all + (size_t)b * MAX_DICT_SIZE;
    const uint32_t stride = gridDim.x * 256, t0 = blockIdx.x * 256 + threadIdx.x;
    for (uint32_t i = t0; i < (1u << log); i += stride) map[i] = -1;
    for (uint32_t i = t0; i < (uint32_t)MAX_DICT_SIZE; i += stride) {
        Entry e;
        if ((int)i < static_n) {
            e = sdict[i];
        } else {
            e.hash = 0;
            e.data = (int32_t)i;
            e.ptr = NIL;
        }
        list[i] = e;
    }
}

KZ_D Dict make_dict(int32_t* map, uint32_t log, Entry* list, int static_n, const uint8_t* swords, int count_for_size) {
    Dict D;
    D.map = map;
    D.hash_mask = (1u << log) - 1;
    D.list = list;
    D.dict_size = initial_dict_size(count_for_size);
    D.static_size = static_n;
    D.swords = swords;
    for (int i = 0; i < static_n; i++) D.map[(uint32_t)list[i].hash & D.hash_mask] = i;  // in index order: later words win a shared slot (:1212-1215)
    return D;
}

__global__ void __launch_bounds__(32) text_forward_walk_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks,
                                                                const uint32_t* __restrict__ go, int static_n, const uint8_t* __restrict__ swords,
                                                                int32_t* __restrict__ map_all, const MapSlice* __restrict__ slice, Entry* __restrict__ list_all,
                                                                uint8_t* __restrict__ out, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    if (!(go[b] & 0x100u)) return;
    const StageBlock blk = blocks[b];
    Dict D = make_dict(map_all + slice[b].off, slice[b].log, list_all + (size_t)b * MAX_DICT_SIZE, static_n, swords, (int)blk.len);
    const int n = forward_walk(in + blk.src_off, (int)blk.len, out + blk.dst_off, (uint8_t)(go[b] & 0xFF), D);
    if (n >= 0) {
        StageResult r = res[b];
        r.status = 0;
        r.out_len = (uint32_t)n;
        res[b] = r;
    }
}

__global__ void __launch_bounds__(32) text_inverse_walk_kernel(const uint8_t* __restrict__ in, const StageBlock* __restrict__ blocks, int nblocks, int static_n,
                                                                const uint8_t* __restrict__ swords, int32_t* __restrict__ map_all, const MapSlice* __restrict__ slice,
                                                                Entry* __restrict__ list_all, uint8_t* __restrict__ out, StageResult* __restrict__ res) {
    const int b = blockIdx.x;
    if (b >= nblocks || threadIdx.x != 0) return;
    const StageBlock blk = blocks[b];
    if (blk.flags == 1) return;  // decoded by the data-parallel path
    StageResult r;
    r.status = 0;
    r.out_len = 0;
    r.data_type = 0;
    r.mode = 0;
    if (blk.len != 0 && blk.cap != 0) {  // wrapper :573-575
        int64_t n = -1;
        if (blk.len >= 2 && blk.len <= (1u << 30)) {
            Dict D = make_dict(map_all + slice[b].off, slice[b].log, list_all + (size_t)b * MAX_DICT_SIZE, static_n, swords, (int)min(blk.cap, 0x7FFFFFFFu));
            n = inverse_walk(in + blk.src_off, (int)blk.len, out + blk.dst_off, (int64_t)blk.cap, D);
        }
        if (n < 0) r.status = -KZ_E_PROCESS_BLOCK;
        else r.out_len = (uint32_t)n;
    }
    res[b] = r;
}

}  // namespace

uint64_t text_map_layout(const uint64_t* bs, uint32_t nblocks, std::vector<uint64_t>& off, std::vector<uint32_t>& lg) {
    off.resize(nblocks);
    lg.resize(nblocks);
    uint64_t slots = 0;
    for (uint32_t b = 0; b < nblocks; b++) {
        lg[b] = log_hash_size(bs[b]);
        off[b] = slots;
        slots += 1ull << lg[b];
    }
    return slots;
}

size_t text_workspace_serial(const uint64_t* bs, uint32_t nblocks) {
    std::vector<uint64_t> off;
    std::vector<uint32_t> lg;
    const uint64_t slots = text_map_layout(bs, nblocks, off, lg);
    return align256(sizeof(Entry) * STATIC_WORDS) + align256(SWORDS_BYTES) + align256((size_t)nblocks * 256 * 4) + align256((size_t)nblocks * 65536 * 4) +
           align256((size_t)nblocks * 4) + align256((size_t)nblocks * sizeof(MapSlice)) + align256((size_t)slots * 4) +
           align256((size_t)nblocks * MAX_DICT_SIZE * sizeof(Entry)) + 256;
}
size_t text_workspace(const uint64_t* bs, uint32_t nblocks, uint32_t max_len) {
    return align256(text_workspace_serial(bs, nblocks)) + text_parallel_workspace(bs, nblocks, max_len) + 256;
}
size_t text_workspace_inverse(const uint64_t* bs, uint32_t nblocks, uint32_t max_len) {
    return align256(text_workspace_serial(bs, nblocks)) + text_inverse_parallel_workspace(bs, nblocks, max_len) + 256;
}

cudaError_t text_forward_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, const StageBlock* h_blocks, uint32_t nblocks, uint32_t max_len,
                               const uint64_t* bs, uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream, uint64_t* launches,
                               uint64_t* serial) {
#if !KZ_HAVE_TEXT_DICT
    (void)serial; (void)d_in; (void)d_out; (void)d_blocks; (void)h_blocks; (void)nblocks; (void)max_len; (void)bs; (void)ws; (void)ws_bytes; (void)d_res; (void)stream; (void)launches;
    return cudaErrorNotSupported;
#else
    if (nblocks == 0) return cudaSuccess;
    if (ws_bytes < text_workspace(bs, nblocks, max_len)) return cudaErrorInvalidValue;
    const Ws w = carve(ws, nblocks, bs);
    const HostStatic& S = host_static();
    cudaError_t e;
    if ((e = cudaMemcpyAsync(w.sdict, S.entries.data(), sizeof(Entry) * STATIC_WORDS, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(w.swords, S.words.data(), SWORDS_BYTES, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(w.hist0, 0, (size_t)nblocks * 256 * 4, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(w.hist1, 0, (size_t)nblocks * 65536 * 4, stream)) != cudaSuccess) return e;
    text_hist_kernel<<<dim3(HIST_SLICES, nblocks), 256, 0, stream>>>(d_in, d_blocks, w.hist0, w.hist1);
    text_plan_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.hist0, w.hist1, w.go, d_res);
    // data-parallel path (kz_text_par.cu); blocks it does not cover come back in `fallback` and take the serial walk below
    uint8_t* pws = ws + align256(text_workspace_serial(bs, nblocks));
    const size_t pws_bytes = ws_bytes - align256(text_workspace_serial(bs, nblocks));
    std::vector<StageBlock> tb(h_blocks, h_blocks + nblocks);
    std::vector<uint32_t> fallback;
    if ((e = text_forward_parallel(d_in, d_out, tb, w.go, bs, w.sdict, w.swords, S.n, pws, pws_bytes, d_res, stream, fallback, launches)) != cudaSuccess)
        return e;
    bool any = false;
    for (uint32_t b = 0; b < nblocks; b++) {
        any = any || fallback[b];
        if (serial && fallback[b] && h_blocks[b].len) ++*serial;  // a block of data the serial walk decodes
    }
    if (!any) return cudaGetLastError();
    std::vector<uint32_t> go(nblocks);
    // on the context's own (non-blocking) stream: a plain cudaMemcpy would neither wait for it nor leave other contexts alone
    if ((e = cudaMemcpyAsync(go.data(), w.go, nblocks * 4, cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    for (uint32_t b = 0; b < nblocks; b++)
        if (!fallback[b]) go[b] = 0;
    if ((e = cudaMemcpyAsync(w.go, go.data(), nblocks * 4, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(w.slice, w.h_slice.data(), nblocks * sizeof(MapSlice), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;  // `go` and the slices are locals
    text_init_kernel<<<dim3(INIT_SLICES, nblocks), 256, 0, stream>>>(w.go, w.sdict, S.n, w.map, w.slice, w.list);
    text_forward_walk_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_blocks, (int)nblocks, w.go, S.n, w.swords, w.map, w.slice, w.list, d_out, d_res);
    if (launches) *launches += 4;
    return cudaGetLastError();
#endif
}

cudaError_t text_inverse_batch(const uint8_t* d_in, uint8_t* d_out, const StageBlock* d_blocks, const StageBlock* h_blocks, uint32_t nblocks, const uint64_t* bs,
                               uint8_t* ws, size_t ws_bytes, StageResult* d_res, cudaStream_t stream, uint64_t* launches, uint64_t* serial) {
#if !KZ_HAVE_TEXT_DICT
    (void)serial; (void)d_in; (void)d_out; (void)d_blocks; (void)h_blocks; (void)nblocks; (void)bs; (void)ws; (void)ws_bytes; (void)d_res; (void)stream; (void)launches;
    return cudaErrorNotSupported;
#else
    if (nblocks == 0) return cudaSuccess;
    if (ws_bytes < text_workspace_serial(bs, nblocks)) return cudaErrorInvalidValue;
    const Ws w = carve(ws, nblocks, bs);
    const HostStatic& S = host_static();
    cudaError_t e;
    if ((e = cudaMemcpyAsync(w.sdict, S.entries.data(), sizeof(Entry) * STATIC_WORDS, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(w.swords, S.words.data(), SWORDS_BYTES, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    // data-parallel path (kz_text_par.cu); trivial blocks and every anomaly come back in `fallback` and take the serial walk below
    const size_t used = align256(text_workspace_serial(bs, nblocks));
    std::vector<StageBlock> tb(h_blocks, h_blocks + nblocks);
    std::vector<uint32_t> fallback;
    if ((e = text_inverse_parallel(d_in, d_out, tb, bs, w.sdict, w.swords, S.n, ws + used, ws_bytes - used, d_res, stream, fallback, launches)) != cudaSuccess)
        return e;
    bool any = false;
    for (uint32_t b = 0; b < nblocks; b++) {
        any = any || fallback[b];
        if (serial && fallback[b] && h_blocks[b].len) ++*serial;  // a block of data the serial walk decodes
    }
    if (!any) return cudaGetLastError();
    // the serial kernel writes res[b] for every block: give it a descriptor list in which the finished blocks are marked
    for (uint32_t b = 0; b < nblocks; b++)
        if (!fallback[b]) tb[b].flags = 1;
    StageBlock* d_tmp = reinterpret_cast<StageBlock*>(w.hist1);  // the forward-only histogram area is free here
    if ((e = cudaMemcpyAsync(d_tmp, tb.data(), nblocks * sizeof(StageBlock), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(w.slice, w.h_slice.data(), nblocks * sizeof(MapSlice), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    text_init_kernel<<<dim3(INIT_SLICES, nblocks), 256, 0, stream>>>(nullptr, w.sdict, S.n, w.map, w.slice, w.list);
    text_inverse_walk_kernel<<<nblocks, 32, 0, stream>>>(d_in, d_tmp, (int)nblocks, S.n, w.swords, w.map, w.slice, w.list, d_out, d_res);
    if (launches) *launches += 2;
    return cudaGetLastError();
#endif
}

}  // namespace kz
