// C ABI of the H100 engine (include/kanzi_b200.h) and the host-side orchestration of the per-block path.
//
// Host-side restatements (tiny, serial, run once per call) cite the reference next to each function; all per-byte
// work happens in the CUDA kernels (kz_ans.cu, kz_huffman.cu, kz_concat.cu, ...). There is deliberately NO CPU code
// path for any codec here: if the CUDA runtime is unusable every entry point fails.
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>

#include "../../include/kanzi_b200.h"
#include "kz_ans1.cuh"
#include "kz_engine.cuh"
#include "kz_bwt.cuh"
#include "kz_huffman.cuh"
#include "kz_lz.cuh"
#include "kz_range.cuh"
#include "kz_hash.cuh"
#include "kz_sbrt.cuh"
#include "kz_zrlt.cuh"
#include "kz_rolz.cuh"
#include "kz_alias.cuh"
#include "kz_fsd.cuh"
#include "kz_text.cuh"
#include "kz_utf.cuh"
#include "kz_exe.cuh"
#include "kz_entropy_core.cuh"
#include "kz_skip.cuh"
#include "kz_stream_plan.h"
#include "kz_read_plan.h"
#include "kz_write_plan.h"
#include "kz_block_cache.h"
#include "kz_record_hash.cuh"
#include "kz_xxh64_core.cuh"

#include <condition_variable>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <tuple>

using namespace kz;

#define CK(x)                                                 \
    do {                                                      \
        cudaError_t e_ = (x);                                 \
        if (e_ != cudaSuccess) return ctx->cuda_fail(e_, #x); \
    } while (0)

// A block cache (kz_cache_create): the bookkeeping of kz_block_cache.h over one device allocation of pages. ctx is null once kz_destroy has
// released the pages of a cache its caller did not free first.
struct kz_cache {
    kz_ctx* ctx;
    kz::PageCache pc;
    void* d_pages = nullptr;
    kz_cache(kz_ctx* c, uint64_t budget) : ctx(c), pc(budget) {}
    size_t device_bytes() const { return d_pages ? (size_t)pc.npages() * kz::CACHE_PAGE : 0; }
};

namespace {

const uint32_t BS_TYPE = 0x4B414E5A;  // io/CompressedStream.go:43
const uint32_t BS_VERSION = 6;        // :44
const size_t RAW_PIECE = 64 * 1024;   // raw segments are cut so that one CTA never copies more than this

cudaEvent_t get_event(kz_ctx* ctx) {
    if (!ctx->event_pool.empty()) {
        cudaEvent_t e = ctx->event_pool.back();
        ctx->event_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}

// host-side phase timer (only when profiling): accumulates wall milliseconds under "host:<name>"
struct HostScope {
    kz_ctx* ctx;
    const char* name;
    std::chrono::steady_clock::time_point t0;
    HostScope(kz_ctx* c, const char* n) : ctx(c), name(n), t0(std::chrono::steady_clock::now()) {}
    ~HostScope() {
        if (ctx->profile) {
            auto& e = ctx->prof[std::string("host:") + name];
            e.ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            e.launches++;
        }
    }
};

struct LaunchScope {
    kz_ctx* ctx;
    cudaEvent_t a = nullptr, b = nullptr;
    const char* name;
    LaunchScope(kz_ctx* c, const char* n) : ctx(c), name(n) {
        ctx->launches++;
        if (ctx->profile) {
            a = get_event(ctx);
            b = get_event(ctx);
            cudaEventRecord(a, ctx->stream);
        }
    }
    ~LaunchScope() {
        if (ctx->profile) {
            cudaEventRecord(b, ctx->stream);
            ctx->pending.push_back({name, a, b});
        }
    }
};

// algorithmic bytes of one transform stage over a batch (SURVEY 8d: stage input + stage output), kept under "stage:fwd:<id>" / "stage:inv:<id>"
void note_stage_bytes(kz_ctx* ctx, const char* dir, uint64_t id, uint64_t bytes_in, uint64_t bytes_out) {
    if (!ctx->profile) return;
    auto& e = ctx->prof[std::string("stage:") + dir + ":" + std::to_string((unsigned long long)id)];
    e.bytes_in += bytes_in;
    e.bytes_out += bytes_out;
    e.launches++;
}

void drain_profile(kz_ctx* ctx) {
    if (ctx->pending.empty()) return;
    cudaStreamSynchronize(ctx->stream);
    for (auto& p : ctx->pending) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) {
            auto& e = ctx->prof[p.name];
            e.ms += ms;
            e.launches++;
        }
        ctx->event_pool.push_back(p.a);
        ctx->event_pool.push_back(p.b);
    }
    ctx->pending.clear();
}

// adaptors for the data-parallel LZ forward path (kz_lz_par.cu): scratch from ctx->d_ws, every pass timed under its own name
struct CtxLzWorkspace : LzWorkspace {
    kz_ctx* ctx;
    explicit CtxLzWorkspace(kz_ctx* c) : ctx(c) {}
    uint8_t* ensure(size_t bytes) override { return ctx->d_ws.ensure(bytes) == cudaSuccess ? ctx->d_ws.as<uint8_t>() : nullptr; }
};
struct CtxLzHook : LzHook {
    kz_ctx* ctx;
    LaunchScope* cur = nullptr;
    explicit CtxLzHook(kz_ctx* c) : ctx(c) {}
    void begin(const char* name) override { cur = new LaunchScope(ctx, name); }
    void end() override {
        delete cur;
        cur = nullptr;
    }
};
// LZ / LZX forward of a batch: the data-parallel path (kz_lz_par.cu); blocks it hands back (status 3: no fixed point of the table
// membership within its round limit) go through the serial parse of kz_lz.cu.
int upload(kz_ctx* ctx, Packer& pk);
int lz_forward_batch(kz_ctx* ctx, const uint8_t* d_in, uint8_t* d_out, std::vector<LzBlock>& lb, bool extra, std::vector<LzResult>& hres) {
    const uint32_t nblocks = (uint32_t)lb.size();
    hres.assign(nblocks, LzResult{1, 0, 0, 0, 0, 0, 0});
    {
        CtxLzWorkspace W(ctx);
        CtxLzHook H(ctx);
        CK(lz_forward_parallel(d_in, d_out, lb, extra, W, ctx->stream, hres, &H));
        bool serial = false;
        for (uint32_t b = 0; b < nblocks; b++) serial = serial || hres[b].status == 3;
        if (!serial) return 0;
    }
    uint32_t max_len = 0;
    std::vector<LzBlock> sb(lb);
    for (uint32_t b = 0; b < nblocks; b++) {
        if (hres[b].status != 3) sb[b].len = 0;  // done by the parallel path
        max_len = std::max(max_len, sb[b].len);
    }
    const uint64_t sstride = (lz_scratch_bytes(max_len) + 255) & ~size_t(255);
    const size_t hbytes = ((size_t)nblocks << (extra ? 19 : 16)) * 4;
    for (uint32_t b = 0; b < nblocks; b++) sb[b].scratch_off = (uint64_t)b * sstride;
    CK(ctx->d_ws.ensure(sstride * nblocks + hbytes + 4096));
    CK(ctx->d_lens.ensure((size_t)nblocks * sizeof(LzResult) + 64));
    Packer pk;
    const size_t o_lb = pk.add(sb.data(), sb.size() * sizeof(LzBlock));
    int rc = upload(ctx, pk);
    if (rc) return rc;
    uint8_t* ws = ctx->d_ws.as<uint8_t>();
    int32_t* d_hash = (int32_t*)(ws + sstride * nblocks);
    CK(cudaMemsetAsync(d_hash, 0, hbytes, ctx->stream));
    LzBlock* d_lb = (LzBlock*)(ctx->d_tables.as<uint8_t>() + o_lb);
    LzResult* d_res = ctx->d_lens.as<LzResult>();
    {
        LaunchScope ls(ctx, "lz_parse");
        lz_parse_kernel<<<nblocks, 32, 0, ctx->stream>>>(d_in, d_lb, (int)nblocks, extra ? 1 : 0, d_hash, ws, d_out, d_res);
    }
    {
        LaunchScope ls(ctx, "lz_gather");
        lz_gather_kernel<<<dim3(nblocks, 8), 256, 0, ctx->stream>>>(d_in, d_lb, (int)nblocks, ws, d_res, d_out);
    }
    CK(cudaGetLastError());
    std::vector<LzResult> sres(nblocks);
    CK(cudaMemcpyAsync(sres.data(), d_res, (size_t)nblocks * sizeof(LzResult), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (uint32_t b = 0; b < nblocks; b++)
        if (hres[b].status == 3) hres[b] = sres[b];
    return 0;
}

int upload(kz_ctx* ctx, Packer& pk) {
    CK(ctx->h_stage.ensure(pk.bytes.size() + 256));
    CK(ctx->d_tables.ensure(pk.bytes.size() + 256));
    memcpy(ctx->h_stage.p, pk.bytes.data(), pk.bytes.size());
    CK(cudaMemcpyAsync(ctx->d_tables.p, ctx->h_stage.p, pk.bytes.size(), cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

// Device-to-device copies collected on the host and run by one batch_copy_kernel launch.
struct CopyList {
    std::vector<CopyJob> jobs;
    void add(const void* src, void* dst, uint64_t len) {
        for (uint64_t o = 0; o < len; o += COPY_PIECE)
            jobs.push_back({(uint64_t)(uintptr_t)src + o, (uint64_t)(uintptr_t)dst + o, std::min<uint64_t>(COPY_PIECE, len - o)});
    }
};
int run_copies(kz_ctx* ctx, const CopyList& cl) {
    if (cl.jobs.empty()) return 0;
    const size_t bytes = cl.jobs.size() * sizeof(CopyJob);
    CK(ctx->d_copy.ensure(bytes));
    // from pageable memory: the runtime has taken the list when the call returns, and the copy is ordered behind earlier kernels
    CK(cudaMemcpyAsync(ctx->d_copy.p, cl.jobs.data(), bytes, cudaMemcpyHostToDevice, ctx->stream));
    {
        LaunchScope ls(ctx, "batch_copy");
        batch_copy_kernel<<<(int)cl.jobs.size(), 256, 0, ctx->stream>>>(ctx->d_copy.as<CopyJob>(), (int)cl.jobs.size());
    }
    CK(cudaGetLastError());
    return 0;
}

// The first w bytes of n device ranges (range i: len[i] bytes at d_base + off[i]) to out, w bytes per range and zero padded, and the
// n_extra bytes at d_extra to extra, behind one synchronisation (none when there is nothing to copy). One range is one copy. Evenly
// spaced ranges, such as the blocks of one stream, are one cudaMemcpy2DAsync and one copy of a short last range. Other ranges are
// gathered into ctx->d_asm by one copy launch and come back in one transfer.
template <class Len>
int gather_heads(kz_ctx* ctx, const uint8_t* d_base, const uint64_t* off, const Len* len, size_t n, uint32_t w, uint8_t* out,
                 const uint8_t* d_extra = nullptr, size_t n_extra = 0, uint8_t* extra = nullptr) {
    const uint64_t MAX_PITCH = 1u << 30;  // the largest block size: a source pitch cudaMemcpy2DAsync takes
    auto head = [&](size_t i) { return (size_t)std::min<uint64_t>(len[i], w); };
    memset(out, 0, n * w);
    bool any = n_extra > 0;
    for (size_t i = 0; i < n && !any; i++) any = head(i) > 0;
    if (!any) return 0;
    const uint64_t pitch = n > 1 ? off[1] - off[0] : 0;
    bool even = n > 1 && off[1] > off[0] && pitch >= w && pitch <= MAX_PITCH;
    for (size_t i = 0; i < n && even; i++) even = off[i] == off[0] + i * pitch && (i + 1 == n || len[i] >= w);
    if (n == 1 || even) {
        if (n > 1) CK(cudaMemcpy2DAsync(out, w, d_base + off[0], pitch, w, n - 1, cudaMemcpyDeviceToHost, ctx->stream));
        if (head(n - 1)) CK(cudaMemcpyAsync(out + (n - 1) * w, d_base + off[n - 1], head(n - 1), cudaMemcpyDeviceToHost, ctx->stream));
    } else if (n) {
        CK(ctx->d_asm.ensure(n * w));
        CopyList cl;
        for (size_t i = 0; i < n; i++) cl.add(d_base + off[i], ctx->d_asm.as<uint8_t>() + i * w, head(i));
        int rc = run_copies(ctx, cl);
        if (rc) return rc;
        CK(cudaMemcpyAsync(out, ctx->d_asm.p, n * w, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (n_extra) CK(cudaMemcpyAsync(extra, d_extra, n_extra, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < n; i++) memset(out + i * w + head(i), 0, w - head(i));  // a gather leaves the bytes behind a short head as they were
    return 0;
}

// The first INDEX_HEAD bytes of n streams (stream i: len[i] bytes at base + off[i]) to out, INDEX_HEAD bytes per stream and zero padded:
// copied on the host, or gathered from device memory.
int read_heads(kz_ctx* ctx, const uint8_t* base, bool device, const uint64_t* off, const uint64_t* len, size_t n, uint8_t* out) {
    if (device) return gather_heads(ctx, base, off, len, n, INDEX_HEAD, out);
    memset(out, 0, n * INDEX_HEAD);
    for (size_t i = 0; i < n; i++) memcpy(out + i * INDEX_HEAD, base + off[i], std::min<uint64_t>(len[i], INDEX_HEAD));
    return 0;
}

// Host bytes staged through ctx->h_io. An upload piece copies `copy` bytes from src into a slot of `slot` >= copy bytes; the slots lie at
// 16-byte aligned offsets of ctx->d_in, and the bytes of a slot behind its copy are zero. A download piece copies len bytes at offset `at`
// of a device staging area to dst.
struct UploadPiece {
    const uint8_t* src;
    uint64_t copy, slot;
};
struct DownloadPiece {
    uint8_t* dst;
    uint64_t at, len;
};

// The pieces packed into ctx->h_io and moved to ctx->d_in in one transfer; at[i]: piece i's offset in d_in, *total: the bytes moved.
int upload_pieces(kz_ctx* ctx, const std::vector<UploadPiece>& pieces, std::vector<uint64_t>& at, uint64_t* total) {
    at.resize(pieces.size());
    uint64_t t = 0;
    for (size_t i = 0; i < pieces.size(); i++) at[i] = t, t += round16(pieces[i].slot);
    CK(ctx->h_io.ensure(t + 64));
    CK(ctx->d_in.ensure(t + 64));
    uint8_t* h = (uint8_t*)ctx->h_io.p;
    for (size_t i = 0; i < pieces.size(); i++) {
        const UploadPiece& pc = pieces[i];
        if (pc.copy) memcpy(h + at[i], pc.src, pc.copy);
        memset(h + at[i] + pc.copy, 0, round16(pc.slot) - pc.copy);
    }
    if (t) CK(cudaMemcpyAsync(ctx->d_in.p, h, t, cudaMemcpyHostToDevice, ctx->stream));
    *total = t;
    return 0;
}

// Bytes [0, total) of d_stage moved into ctx->h_io in one transfer, then each piece copied out to the caller's memory.
int download_pieces(kz_ctx* ctx, const uint8_t* d_stage, uint64_t total, const std::vector<DownloadPiece>& pieces) {
    CK(ctx->h_io.ensure(total + 64));
    if (total) CK(cudaMemcpyAsync(ctx->h_io.p, d_stage, total, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (const DownloadPiece& pc : pieces) memcpy(pc.dst, (const uint8_t*)ctx->h_io.p + pc.at, pc.len);
    return 0;
}

// XXHash32/64 of a set of blocks (hash/XXHash32.go, XXHash64.go; seed "KANZ", io/CompressedStream.go:354-356). Synchronous.
int hash_blocks(kz_ctx* ctx, const uint8_t* d_base, const std::vector<uint64_t>& off, const std::vector<uint32_t>& len, uint32_t bits,
                std::vector<uint64_t>& out) {
    const size_t nb = off.size();
    out.assign(nb, 0);
    if (nb == 0) return 0;
    std::vector<HashJob> hj(nb);
    for (size_t b = 0; b < nb; b++) {
        hj[b].off = off[b];
        hj[b].len = len[b];
        hj[b].pad = 0;
    }
    Packer pk;
    const size_t o_j = pk.add(hj.data(), hj.size() * sizeof(HashJob));
    const size_t o_h = pk.reserve(nb * 8);
    int rc = upload(ctx, pk);
    if (rc) return rc;
    uint8_t* T = ctx->d_tables.as<uint8_t>();
    {
        LaunchScope ls(ctx, "xxhash");
        xxhash_blocks_kernel<<<(int)nb, 32, 0, ctx->stream>>>(d_base, (const HashJob*)(T + o_j), (int)nb, (int)bits, (uint64_t*)(T + o_h));
    }
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out.data(), T + o_h, nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (bits == 32)
        for (auto& h : out) h &= 0xFFFFFFFFull;
    return 0;
}

// decodingTask.decode :1990-2006: hash of the decoded block against the transmitted checksum
const char* const CHECKSUM_MISMATCH = "Corrupted bitstream: block checksum mismatch";

bool etype_supported(uint32_t e) { return e == KZ_E_NONE || e == KZ_E_ANS0 || e == KZ_E_HUFFMAN || e == KZ_E_ANS1 || e == KZ_E_RANGE; }

// The block sizes a stream-level encode accepts
bool block_size_ok(uint32_t block_size) { return block_size >= 1024 && block_size <= (1u << 30) && !(block_size & 15); }
int check_checksum_bits(kz_ctx* ctx, uint32_t checksum_bits) {
    if (checksum_bits != 0 && checksum_bits != 32 && checksum_bits != 64) return ctx->fail(KZ_ERR_INVALID_PARAM, "checksum must be 0, 32 or 64 bits");
    return 0;
}
// The block size and checksum width of every stream-level encode (whole stream, many streams, writer session)
int check_encode_args(kz_ctx* ctx, uint32_t block_size, uint32_t checksum_bits) {
    if (!block_size_ok(block_size)) return ctx->fail(KZ_ERR_INVALID_PARAM, "Invalid block size");
    return check_checksum_bits(ctx, checksum_bits);
}

// The spans of a many-stream argument, span i being len[i] bytes at base + off[i]: no offset + length overflows, a buffer lies under
// spans that reach past its first byte, and in device memory (device) the base and every offset are multiples of 16.
int check_spans(kz_ctx* ctx, const void* base, const uint64_t* off, const uint64_t* len, size_t n, bool device) {
    uint64_t end = 0;
    for (size_t i = 0; i < n; i++) {
        if (off[i] + len[i] < off[i]) return ctx->fail(KZ_ERR_INVALID_PARAM, "offset + length overflows");
        if (device && (off[i] & 15)) return ctx->fail(KZ_ERR_INVALID_PARAM, "device offsets must be multiples of 16");
        end = std::max(end, off[i] + len[i]);
    }
    if (end && !base) return ctx->fail(KZ_ERR_INVALID_PARAM, "null buffer");
    if (device && ((uintptr_t)base & 15)) return ctx->fail(KZ_ERR_INVALID_PARAM, "device buffers must be 16-byte aligned");
    return 0;
}

// The gather of every bit-granular output (kz_concat.cu): segment i, seg_bits[i] bits at address seg_src[i], lands at bit seg_dst[i] of
// d_out. The three tables are device arrays. encode_batch and SegmentList write through it.
int concat_segments(kz_ctx* ctx, const uint64_t* d_seg_src, const uint64_t* d_seg_bits, const uint64_t* d_seg_dst, int nsegs, uint8_t* d_out) {
    if (nsegs <= 0) return 0;
    {
        LaunchScope ls(ctx, "concat_zero");
        concat_zero_kernel<<<(nsegs + 255) / 256, 256, 0, ctx->stream>>>(d_seg_bits, d_seg_dst, nsegs, (uint32_t*)d_out);
    }
    {
        LaunchScope ls(ctx, "concat");
        concat_copy_kernel<<<nsegs, 128, 0, ctx->stream>>>(d_seg_src, d_seg_bits, d_seg_dst, nsegs, (uint32_t*)d_out);
    }
    CK(cudaGetLastError());
    return 0;
}

// The segments of one concat_segments call, laid out on the host: each lands behind the previous one, from the bit at() names. Device bit
// strings (from any bit) are cut into RAW_PIECE pieces; short strings built on the host (a stream header, a record prefix, the end marker)
// travel with the segment table.
struct SegmentList {
    std::vector<uint64_t> src, bits, dst;
    std::vector<size_t> host_seg;  // segments whose src is an offset into `host` until write() knows where it lands
    std::vector<uint8_t> host;
    uint64_t next = 0;

    void at(uint64_t bit) { next = bit; }
    void add_device(const uint8_t* p, uint64_t bit, uint64_t nbits) {
        for (uint64_t o = 0; o < nbits; o += 8 * RAW_PIECE) push(seg_source(p, bit + o), std::min<uint64_t>(8 * RAW_PIECE, nbits - o));
    }
    void add_host(const uint8_t* bytes, uint64_t nbits) {
        if (!nbits) return;
        const size_t o = host.size();
        host.resize(o + (nbits + 63) / 64 * 8, 0);
        memcpy(&host[o], bytes, (nbits + 7) / 8);
        host_seg.push_back(src.size());
        push(o, nbits);
    }
    void add_end_marker() {
        const uint8_t zero[8] = {0};
        add_host(zero, END_MARKER_BITS);
    }
    void push(uint64_t s, uint64_t n) {
        src.push_back(s), bits.push_back(n), dst.push_back(next);
        next += n;
    }
    // the host strings, then the three tables, in one upload; the concat; one synchronisation (the tables live in ctx->d_tables)
    int write(kz_ctx* ctx, uint8_t* d_out) {
        if (src.empty()) return 0;
        Packer pk;
        const size_t o_host = pk.add(host.data(), host.size());
        const size_t o_src = pk.add(src.data(), src.size() * 8);
        const size_t o_bits = pk.add(bits.data(), bits.size() * 8);
        const size_t o_dst = pk.add(dst.data(), dst.size() * 8);
        CK(ctx->d_tables.ensure(pk.bytes.size() + 256));  // what upload() ensures: the host strings' addresses are final from here
        const uint64_t h = (uint64_t)(uintptr_t)(ctx->d_tables.as<uint8_t>() + o_host);
        for (size_t i : host_seg) ((uint64_t*)(pk.bytes.data() + o_src))[i] += h;
        int rc = upload(ctx, pk);
        if (rc) return rc;
        const uint8_t* T = ctx->d_tables.as<uint8_t>();
        rc = concat_segments(ctx, (const uint64_t*)(T + o_src), (const uint64_t*)(T + o_bits), (const uint64_t*)(T + o_dst), (int)src.size(), d_out);
        if (rc) return rc;
        CK(cudaStreamSynchronize(ctx->stream));
        return 0;
    }
};

// The per-chunk scratch encode_batch allocates for codec e (d_enc_tab, d_hdr, d_pay, d_hist), for the pass planner (kz_stream_plan.h)
EntropyScratch entropy_scratch(uint32_t e) {
    EntropyScratch s;
    if (e == KZ_E_ANS1) s = {ANS1_CHUNK, 65536 * 4 + 256 * ANS1_CTX_HDR_STRIDE + 32 + 112 + ANS1_HIST_WORDS * 4 + 256 * 4, 2};
    else if (e == KZ_E_RANGE) s = {RANGE_CHUNK, RC_OUT_STRIDE, 0};
    else if (e == KZ_E_HUFFMAN) s = {HUF_CHUNK, 256 * 2 + HUF_HDR_STRIDE + HUF_FRAG_STRIDE * 4, 0};
    else if (e == KZ_E_ANS0) s = {ANS0_CHUNK, 256 * 4 + HDR_STRIDE + PAY_STRIDE, 0};
    return s;
}

// ------------------------------------------------------------------------------------------------------------
// entropy encode of a batch of blocks + bit-granular assembly
// ------------------------------------------------------------------------------------------------------------
struct EncResult {
    uint64_t total_bits = 0;          // LAYOUT_STREAM: bits of the complete stream
    std::vector<uint64_t> blk_bits;   // per block "written"
    std::vector<int32_t> status;      // per block 0 / -(error code)
};

// LAYOUT_STREAM: stream_hdr (stream_hdr_bits bits) leads, and the end marker closes the stream unless `fragment` (the records of one rank of
// a sharded compression, or a writer session's batch before its last). volatile_lead: the leading segment is a writer session's header or
// carry, which changes from batch to batch.
int encode_batch(kz_ctx* ctx, EncLayout layout, uint32_t etype, uint32_t checksum_bits, const uint8_t* d_data, const std::vector<EncJob>& jobs,
                 const std::vector<uint8_t>& stream_hdr, uint64_t stream_hdr_bits, bool fragment, bool volatile_lead, uint8_t* d_dst, size_t dst_cap,
                 const std::vector<uint64_t>& blk_base_bits, EncResult& res) {
    const int nblocks = (int)jobs.size();
    if (!etype_supported(etype)) return ctx->fail(KZ_ERR_CREATE_CODEC, "entropy codec not available on the GPU path");
    HostScope hs_all(ctx, "encode_batch");
    std::unique_ptr<HostScope> hs_tab(new HostScope(ctx, "enc_tables"));
    // ---- host: segment and chunk tables. They are a pure function of the batch description (layout, codec, block
    // lengths and flags, buffer addresses), and a stream of equal-sized blocks repeats the same description batch after
    // batch (Writer.processBlock is called once per `jobs` blocks): the packed tables of the last batch are kept and
    // reused when the description is byte-identical (it costs host work per batch otherwise).
    const size_t small_hdr_off = 0;
    const size_t small_blk_off = 64;
    const size_t small_prefix_off = small_blk_off + 16 * (size_t)nblocks;
    const size_t small_zero_off = small_prefix_off + 8 * (size_t)nblocks;
    const size_t small_lr1_off = small_zero_off + 8;  // 3 bits "lr - 8" of the order-1 chunks: 11 - 8 = 0b011
    const size_t small_size = small_zero_off + 16;
    CK(ctx->d_small.ensure(small_size));
    uint8_t* d_small = ctx->d_small.as<uint8_t>();
    std::vector<uint8_t> key;
    // a streaming writer's leading segment (header, then the carry) changes from batch to batch: it stays out of the key and is
    // written into the kept tables below
    const bool lead = volatile_lead && layout == LAYOUT_STREAM;
    {
        auto put = [&](const void* p, size_t n) {
            const uint8_t* q = (const uint8_t*)p;
            key.insert(key.end(), q, q + n);
        };
        const uint64_t scal[8] = {(uint64_t)layout | (fragment ? 0x100u : 0u) | (lead ? 0x200u : 0u), etype, checksum_bits, (uint64_t)(uintptr_t)d_data,
                                  (uint64_t)(uintptr_t)d_small, (uint64_t)nblocks, lead ? 0 : stream_hdr_bits, (uint64_t)stream_hdr.size()};
        key.reserve(sizeof(scal) + stream_hdr.size() + jobs.size() * 40 + blk_base_bits.size() * 8);
        put(scal, sizeof(scal));
        if (!lead) put(stream_hdr.data(), stream_hdr.size());
        for (const EncJob& j : jobs) {
            const uint64_t f[4] = {j.data_off, ((uint64_t)j.post_len << 32) | j.ntransforms, ((uint64_t)j.skip_flags << 8) | (j.copy ? 1u : 0u), j.checksum};
            put(f, sizeof(f));
        }
        put(blk_base_bits.data(), blk_base_bits.size() * 8);
    }
    EncPlan& plan = ctx->enc_plan;
    if (!(plan.valid && plan.key == key)) {
        plan.valid = false;
        plan.build(key, [&](EncPlan& P) {
            std::vector<uint8_t> small(small_size, 0);
            if (!stream_hdr.empty()) memcpy(&small[small_hdr_off], stream_hdr.data(), stream_hdr.size());
            small[small_lr1_off] = 0x60;

            std::vector<uint64_t> seg_src, seg_bits;
            std::vector<uint32_t> blk_first(nblocks + 1);
            std::vector<ChunkIn> chunks;
            std::vector<uint32_t> chunk_seg;
            auto add_seg = [&](uint64_t src, uint64_t bits) {
                seg_src.push_back(src);
                seg_bits.push_back(bits);
            };
            auto add_raw = [&](const uint8_t* p, uint64_t nbytes) {
                for (uint64_t o = 0; o < nbytes; o += RAW_PIECE) add_seg((uint64_t)(uintptr_t)(p + o), 8 * std::min<uint64_t>(RAW_PIECE, nbytes - o));
            };
            if (layout == LAYOUT_STREAM) add_seg((uint64_t)(uintptr_t)(d_small + small_hdr_off), stream_hdr_bits);
            for (int b = 0; b < nblocks; b++) {
                const EncJob& j = jobs[b];
                if (layout == LAYOUT_STREAM) add_seg(0, 0);  // block prefix, filled by block_prefix_kernel
                blk_first[b] = (uint32_t)seg_src.size();
                const uint32_t et = j.copy ? (uint32_t)KZ_E_NONE : etype;
                if (layout != LAYOUT_RAW) {
                    uint8_t* hb = &small[small_blk_off + 16 * (size_t)b];
                    uint32_t hbits = make_block_header(hb, j.copy, j.ntransforms, j.skip_flags, j.post_len, checksum_bits, j.checksum);
                    add_seg((uint64_t)(uintptr_t)(d_small + small_blk_off + 16 * (size_t)b), hbits);
                }
                const uint8_t* data = d_data + j.data_off;
                if (et == KZ_E_NONE || ((et == KZ_E_ANS0 || et == KZ_E_ANS1) && j.post_len <= 32)) {  // NullEntropyCodec.go:43-61 / ANSRangeCodec.go:279-282
                    add_raw(data, j.post_len);
                } else if (et == KZ_E_ANS1) {
                    for (uint32_t o = 0; o < j.post_len; o += ANS1_CHUNK) {
                        ChunkIn c;
                        c.src_off = j.data_off + o;
                        c.len = std::min<uint32_t>(ANS1_CHUNK, j.post_len - o);
                        c.block = (uint32_t)b;
                        chunks.push_back(c);
                        add_seg((uint64_t)(uintptr_t)(d_small + small_lr1_off), 3);  // lr - 8 (updateFrequencies :174)
                        chunk_seg.push_back((uint32_t)seg_src.size());
                        for (int q = 0; q < ANS1_SEGS - 1; q++) add_seg(0, 0);  // 256 context tables, size + states, payload
                    }
                } else if (et == KZ_E_ANS0) {
                    for (uint32_t o = 0; o < j.post_len; o += ANS0_CHUNK) {
                        ChunkIn c;
                        c.src_off = j.data_off + o;
                        c.len = std::min<uint32_t>(ANS0_CHUNK, j.post_len - o);
                        c.block = (uint32_t)b;
                        chunks.push_back(c);
                        chunk_seg.push_back((uint32_t)seg_src.size());
                        add_seg(0, 0);  // A: chunk header + varint + states
                        add_seg(0, 0);  // B: rANS bytes
                    }
                } else if (et == KZ_E_RANGE) {  // RangeCodec.go:233-272: one bit string per 32 KiB chunk
                    for (uint32_t o = 0; o < j.post_len; o += RANGE_CHUNK) {
                        ChunkIn c;
                        c.src_off = j.data_off + o;
                        c.len = std::min<uint32_t>(RANGE_CHUNK, j.post_len - o);
                        c.block = (uint32_t)b;
                        chunks.push_back(c);
                        chunk_seg.push_back((uint32_t)seg_src.size());
                        add_seg(0, 0);
                    }
                } else if (et == KZ_E_HUFFMAN) {  // HuffmanCodec.go:408-430
                    for (uint32_t o = 0; o < j.post_len; o += HUF_CHUNK) {
                        const uint32_t clen = std::min<uint32_t>(HUF_CHUNK, j.post_len - o);
                        if (clen < 32) {
                            add_raw(data + o, clen);
                            continue;
                        }
                        ChunkIn c;
                        c.src_off = j.data_off + o;
                        c.len = clen;
                        c.block = (uint32_t)b;
                        chunks.push_back(c);
                        chunk_seg.push_back((uint32_t)seg_src.size());
                        for (int q = 0; q < 6; q++) add_seg(0, 0);  // header+sizes, 4 fragments, chunk last bytes
                    }
                }
            }
            if (layout == LAYOUT_STREAM) {
                add_seg((uint64_t)(uintptr_t)(d_small + small_zero_off), fragment ? 0 : END_MARKER_BITS);  // end marker (Close :593-594); none behind a fragment
                blk_first[nblocks] = (uint32_t)seg_src.size();
            } else {
                blk_first[nblocks] = (uint32_t)seg_src.size();
            }
            P.nsegs = (int)seg_src.size();
            add_seg(0, 0);  // sentinel for the scan
            P.nchunks = (int)chunks.size();
            P.max_chunk = 0;
            for (auto& c : chunks) P.max_chunk = std::max(P.max_chunk, c.len);

            Packer& pk = P.pk;
            pk.bytes.clear();
            P.o_small = pk.add(small.data(), small.size());
            P.o_src = pk.add(seg_src.data(), seg_src.size() * 8);
            P.o_bits = pk.add(seg_bits.data(), seg_bits.size() * 8);
            P.o_first = pk.add(blk_first.data(), blk_first.size() * 4);
            P.o_chunks = pk.add(chunks.data(), chunks.size() * sizeof(ChunkIn));
            P.o_cseg = pk.add(chunk_seg.data(), chunk_seg.size() * 4);
            P.o_base = pk.add(blk_base_bits.data(), blk_base_bits.size() * 8);
            P.o_off = pk.reserve(seg_src.size() * 8);
            P.o_dst = pk.reserve(seg_src.size() * 8);
            P.o_blkbits = pk.reserve((size_t)(nblocks + 1) * 8);
            P.o_total = pk.reserve(16);
            P.o_hbits = pk.reserve((size_t)P.nchunks * 4 + 4);
            P.o_asz = pk.reserve((size_t)P.nchunks * 4 + 4);
            P.o_estatus = pk.reserve((size_t)nblocks * 4 + 4);
        });
    }
    Packer& pk = plan.pk;
    if (lead) {  // segment 0 is the leading segment; its bytes sit at the start of the small strings
        memcpy(pk.bytes.data() + plan.o_small + small_hdr_off, stream_hdr.data(), std::min<size_t>(stream_hdr.size(), small_blk_off));
        memcpy(pk.bytes.data() + plan.o_bits, &stream_hdr_bits, 8);
    }
    const int nsegs = plan.nsegs, nchunks = plan.nchunks;
    const size_t o_small = plan.o_small, o_src = plan.o_src, o_bits = plan.o_bits, o_first = plan.o_first, o_chunks = plan.o_chunks, o_cseg = plan.o_cseg,
                 o_base = plan.o_base, o_off = plan.o_off, o_dst = plan.o_dst, o_blkbits = plan.o_blkbits, o_total = plan.o_total, o_hbits = plan.o_hbits,
                 o_asz = plan.o_asz, o_estatus = plan.o_estatus;
    int rc = upload(ctx, pk);
    if (rc) return rc;
    uint8_t* T = ctx->d_tables.as<uint8_t>();
    // the small byte strings must live at the addresses baked into the segment table
    CK(cudaMemcpyAsync(d_small, T + o_small, small_size, cudaMemcpyDeviceToDevice, ctx->stream));
    uint64_t* d_seg_src = (uint64_t*)(T + o_src);
    uint64_t* d_seg_bits = (uint64_t*)(T + o_bits);
    uint32_t* d_blk_first = (uint32_t*)(T + o_first);
    ChunkIn* d_chunks = (ChunkIn*)(T + o_chunks);
    uint32_t* d_cseg = (uint32_t*)(T + o_cseg);
    uint64_t* d_base = (uint64_t*)(T + o_base);
    uint64_t* d_seg_off = (uint64_t*)(T + o_off);
    uint64_t* d_seg_dst = (uint64_t*)(T + o_dst);
    uint64_t* d_blk_bits = (uint64_t*)(T + o_blkbits);
    uint64_t* d_total = (uint64_t*)(T + o_total);
    uint32_t* d_hbits = (uint32_t*)(T + o_hbits);
    uint32_t* d_asz = (uint32_t*)(T + o_asz);
    int32_t* d_estatus = (int32_t*)(T + o_estatus);
    hs_tab.reset();

    // ---- entropy kernels
    if (nchunks > 0 && etype == KZ_E_ANS1) {
        const uint32_t max_chunk = plan.max_chunk;
        const uint64_t pay_stride = (2ull * max_chunk + 96 + 15) & ~15ull;
        CK(ctx->d_enc_tab.ensure((size_t)nchunks * 65536 * sizeof(uint32_t)));
        CK(ctx->d_hdr.ensure((size_t)nchunks * 256 * ANS1_CTX_HDR_STRIDE + (size_t)nchunks * 32 + 256));
        CK(ctx->d_pay.ensure((size_t)nchunks * pay_stride));
        CK(ctx->d_hist.ensure((size_t)nchunks * ANS1_HIST_WORDS * 4 + (size_t)nchunks * 256 * 4 + 256));
        if (!ctx->d_rcp.p) {
            CK(ctx->d_rcp.ensure(4096 * sizeof(uint32_t)));
            LaunchScope ls(ctx, "rcp_table");
            rcp_table_kernel<<<16, 256, 0, ctx->stream>>>(ctx->d_rcp.as<uint32_t>());
        }
        uint32_t* d_hist = ctx->d_hist.as<uint32_t>();
        uint32_t* d_ctx_bits = d_hist + (size_t)nchunks * ANS1_HIST_WORDS;
        uint8_t* d_ctx_hdr = ctx->d_hdr.as<uint8_t>();
        uint8_t* d_tail_hdr = d_ctx_hdr + (size_t)nchunks * 256 * ANS1_CTX_HDR_STRIDE;
        CK(cudaMemsetAsync(d_hist, 0, (size_t)nchunks * ANS1_HIST_WORDS * 4, ctx->stream));
        {
            LaunchScope ls(ctx, "ans1_hist");
            ans1_hist_kernel<<<dim3(nchunks, 32), 256, 0, ctx->stream>>>(d_data, d_chunks, nchunks, d_hist);
        }
        {
            LaunchScope ls(ctx, "ans1_stats");
            ans1_stats_kernel<<<(nchunks * 256 + 3) / 4, 128, 0, ctx->stream>>>(d_hist, nchunks, ctx->d_enc_tab.as<uint32_t>(), d_ctx_hdr, d_ctx_bits);
        }
        {
            LaunchScope ls(ctx, "ans1_encode");
            ans1_encode_kernel<<<nchunks, 32, 0, ctx->stream>>>(d_data, d_chunks, nchunks, ctx->d_enc_tab.as<uint32_t>(), ctx->d_rcp.as<uint32_t>(), d_ctx_hdr,
                                                                d_ctx_bits, d_tail_hdr, ctx->d_pay.as<uint8_t>(), pay_stride, d_seg_src, d_seg_bits, d_cseg,
                                                                d_estatus);
        }
    } else if (nchunks > 0 && etype == KZ_E_RANGE) {
        CK(ctx->d_pay.ensure((size_t)nchunks * RC_OUT_STRIDE));
        LaunchScope ls(ctx, "range_encode");
        range_encode_kernel<<<(nchunks + RC_ENC_WARPS - 1) / RC_ENC_WARPS, RC_ENC_WARPS * 32, 0, ctx->stream>>>(
            d_data, d_chunks, nchunks, ctx->d_pay.as<uint8_t>(), d_seg_src, d_seg_bits, d_cseg, d_estatus);
    } else if (nchunks > 0 && etype == KZ_E_HUFFMAN) {
        CK(ctx->d_enc_tab.ensure((size_t)nchunks * 256 * sizeof(uint16_t)));
        CK(ctx->d_hdr.ensure((size_t)nchunks * HUF_HDR_STRIDE));
        CK(ctx->d_pay.ensure((size_t)nchunks * HUF_FRAG_STRIDE * 4));
        {
            LaunchScope ls(ctx, "huf_stats");
            huf_stats_kernel<<<(nchunks + HUF_STATS_WARPS - 1) / HUF_STATS_WARPS, HUF_STATS_WARPS * 32, 0, ctx->stream>>>(
                d_data, d_chunks, nchunks, ctx->d_enc_tab.as<uint16_t>(), ctx->d_hdr.as<uint8_t>(), d_hbits, d_asz);
        }
        {
            LaunchScope ls(ctx, "huf_encode");
            huf_encode_kernel<<<(nchunks + HUF_ENC_WARPS - 1) / HUF_ENC_WARPS, HUF_ENC_WARPS * 32, 0, ctx->stream>>>(
                d_data, d_chunks, nchunks, ctx->d_enc_tab.as<uint16_t>(), ctx->d_hdr.as<uint8_t>(), d_hbits, d_asz, ctx->d_pay.as<uint8_t>(),
                d_seg_src, d_seg_bits, d_cseg);
        }
    } else if (nchunks > 0) {
        CK(ctx->d_enc_tab.ensure((size_t)nchunks * 256 * sizeof(uint32_t)));
        if (!ctx->d_rcp.p) {
            CK(ctx->d_rcp.ensure(4096 * sizeof(uint32_t)));
            LaunchScope ls(ctx, "rcp_table");
            rcp_table_kernel<<<16, 256, 0, ctx->stream>>>(ctx->d_rcp.as<uint32_t>());
        }
        CK(ctx->d_hdr.ensure((size_t)nchunks * HDR_STRIDE));
        CK(ctx->d_pay.ensure((size_t)nchunks * PAY_STRIDE));
        {
            LaunchScope ls(ctx, "ans0_stats");
            ans0_stats_kernel<<<(nchunks + STATS_WARPS - 1) / STATS_WARPS, STATS_WARPS * 32, 0, ctx->stream>>>(
                d_data, d_chunks, nchunks, ctx->d_enc_tab.as<uint32_t>(), ctx->d_hdr.as<uint8_t>(), d_hbits, d_asz);
        }
        {
            LaunchScope ls(ctx, "ans0_encode");
            ans0_encode_kernel<<<(nchunks + ENC_CTA_CHUNKS - 1) / ENC_CTA_CHUNKS, 256, ENC_SMEM, ctx->stream>>>(
                d_data, d_chunks, nchunks, ctx->d_enc_tab.as<uint32_t>(), ctx->d_rcp.as<uint32_t>(), ctx->d_hdr.as<uint8_t>(), d_hbits, d_asz,
                ctx->d_pay.as<uint8_t>(), d_seg_src, d_seg_bits, d_cseg);
        }
    }
    // ---- layout + gather
    {
        LaunchScope ls(ctx, "scan");
        scan_bits_kernel<<<1, 1024, 0, ctx->stream>>>(d_seg_bits, d_seg_off, nsegs + 1, 0, d_total);
    }
    if (layout == LAYOUT_STREAM) {
        if (nblocks > 0) {
            LaunchScope ls(ctx, "block_prefix");
            block_prefix_kernel<<<(nblocks + 127) / 128, 128, 0, ctx->stream>>>(d_seg_off, d_blk_first, nblocks, d_small + small_prefix_off, d_seg_src,
                                                                                d_seg_bits, d_blk_bits);
        }
        LaunchScope ls(ctx, "scan");
        scan_bits_kernel<<<1, 1024, 0, ctx->stream>>>(d_seg_bits, d_seg_dst, nsegs + 1, 0, d_total);
    } else if (nblocks > 0) {
        LaunchScope ls(ctx, "block_layout");
        block_layout_kernel<<<nblocks, 128, 0, ctx->stream>>>(d_seg_off, d_blk_first, nblocks, d_base, d_seg_dst, d_blk_bits);
    }
    // results needed on the host before the gather can be bounds-checked
    CK(ctx->h_dl.ensure((size_t)(nblocks + 4) * 8 + (size_t)nblocks * 4 + 64));
    uint64_t* h = (uint64_t*)ctx->h_dl.p;
    int32_t* hst = (int32_t*)(h + nblocks + 4);
    CK(cudaMemcpyAsync(h, d_blk_bits, (size_t)nblocks * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h + nblocks, d_total, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(hst, d_estatus, (size_t)nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
    {
        HostScope hs_sync(ctx, "enc_sync");
        CK(cudaStreamSynchronize(ctx->stream));
    }
    res.blk_bits.assign(h, h + nblocks);
    res.total_bits = h[nblocks];
    res.status.assign(hst, hst + nblocks);
    for (int b = 0; b < nblocks; b++)
        if (res.status[b]) return ctx->fail(-res.status[b], "entropy encoding failed (the reference fails with ERR_PROCESS_BLOCK on this input)");
    if (layout == LAYOUT_STREAM) {
        if ((res.total_bits + 7) / 8 + 8 > dst_cap) return ctx->fail(KZ_ERR_WRITE_FILE, "output buffer too small");
    } else {
        for (int b = 0; b < nblocks; b++) {
            uint64_t lim = (b + 1 < nblocks ? blk_base_bits[b + 1] : 8 * (uint64_t)dst_cap);
            if (blk_base_bits[b] + res.blk_bits[b] + 64 > lim) return ctx->fail(KZ_ERR_WRITE_FILE, "output buffer too small");
        }
    }
    rc = concat_segments(ctx, d_seg_src, d_seg_bits, d_seg_dst, nsegs, d_dst);
    if (rc) return rc;
    CK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------------------
// entropy decode of a batch of blocks
// ------------------------------------------------------------------------------------------------------------
__global__ void block_header_kernel(const uint32_t* __restrict__ words, const uint64_t* __restrict__ bit_off, const uint64_t* __restrict__ bits, int nblocks,
                                    uint32_t checksum_bits, const uint32_t* __restrict__ block_size, BlockHeader* __restrict__ out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    out[b] = parse_block_header(words, bit_off[b], bits[b], checksum_bits, block_size[b]);
}

// The block records of one stream for stream_walk_kernel: bits [start_bit, end_bit) of the word buffer, found records go to entries
// out .. out + max_blocks - 1 of bit_off / bits. stop_after != 0: a fragment of that many block records (no end marker behind them).
// Only records keep_lo .. keep_hi - 1 (0-based) are stored, record r at entry out + r - keep_lo (a block range, kz_set_block_range); the
// others are walked all the same.
struct WalkJob {
    uint64_t start_bit, end_bit, out;
    uint32_t max_blocks, stop_after;
    uint64_t keep_lo = 0, keep_hi = ~0ull;
};

// Serial walk over the block length prefixes of complete streams (decodingTask.decode :1816-1852), one thread per stream: jobs[s], or
// `one` when jobs is null. count_status[2s] = records found, count_status[2s + 1] = 0 or -(error code).
__global__ void stream_walk_kernel(const uint32_t* __restrict__ words, const WalkJob* __restrict__ jobs, WalkJob one, int nstreams,
                                   uint64_t* __restrict__ bit_off_all, uint64_t* __restrict__ bits_all, uint32_t* __restrict__ count_status) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nstreams) return;
    const WalkJob job = jobs ? jobs[s] : one;
    const uint32_t max_blocks = job.max_blocks, stop_after = job.stop_after;
    uint64_t* bit_off = bit_off_all + job.out;
    uint64_t* bits = bits_all + job.out;
    BitReader br(words, job.start_bit, job.end_bit);
    uint32_t n = 0;
    int32_t st = 0;
    for (;;) {
        if (stop_after && n == stop_after) break;
        const uint64_t len = read_block_prefix(br);
        if (br.overrun) {
            st = -KZ_E_PROCESS_BLOCK;
            break;
        }
        if (len == 0) break;
        if (len > (1ull << 34)) {
            st = -KZ_E_BLOCK_SIZE;
            break;
        }
        if (n >= max_blocks) {
            st = -KZ_E_BLOCK_SIZE;
            break;
        }
        if (n >= job.keep_lo && n < job.keep_hi) {
            bit_off[n - job.keep_lo] = br.pos;
            bits[n - job.keep_lo] = len;
        }
        n++;
        br.skip(len);
        if (br.overrun) {
            st = -KZ_E_PROCESS_BLOCK;
            break;
        }
    }
    count_status[2 * s] = n;
    count_status[2 * s + 1] = (uint32_t)st;
}

// The streaming reader's walk over its window (walk_records), one thread.
__global__ void record_walk_kernel(const uint32_t* __restrict__ words, uint64_t start, uint64_t end, uint32_t max_records, uint64_t max_bits,
                                   uint64_t* __restrict__ bit_off, uint64_t* __restrict__ bits, WalkResult* __restrict__ out) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *out = walk_records(words, start, end, max_records, max_bits, bit_off, bits);
}

// What walk_streams found in one stream: n records walked, status 0 or -(error code), overflow = the block range holds more records
// than could be stored; bit_off / bits = the stored records, records first .. first + size - 1 of the stream.
struct Walked {
    uint64_t n = 0, first = 0;
    int32_t status = 0;
    bool overflow = false;
    std::vector<uint64_t> bit_off, bits;
    // appends the stored records as DecJobs of `own`, a stream of block_size; last[b]: the record is the stream's last
    void append(uint32_t own, uint32_t block_size, std::vector<DecJob>& jobs, std::vector<uint32_t>& owner, std::vector<uint8_t>& last) const {
        for (size_t r = 0; r < bit_off.size(); r++) {
            DecJob j = DecJob();
            j.bit_off = bit_off[r];
            j.bits = bits[r];
            j.block_size = block_size;
            jobs.push_back(j);
            owner.push_back(own);
            last.push_back(first + r + 1 == n);
        }
    }
};

// Walks the complete streams of jobs (start_bit, end_bit, stop_after and max_blocks set: at most max_blocks records are stored) with
// stream_walk_kernel, one thread per stream. Only the records of the block range from / to (kz_set_block_range, -1 = not given) are
// stored. Without a range max_blocks also bounds the walk; with one the walk goes over every record to the end marker, so that a walk
// error behind the range is still found, and only the stream's bytes bound it (a record takes at least 9 bits). The counts and the first
// min(slots, 1024) records come back in one round trip; the rest only when more were stored.
int walk_streams(kz_ctx* ctx, const uint32_t* d_words, std::vector<WalkJob>& jobs, int64_t from, int64_t to, std::vector<Walked>& out) {
    const uint32_t ns = (uint32_t)jobs.size();
    const bool ranged = from >= 0 || to >= 0;
    uint64_t keep_lo = 0, keep_hi = ~0ull, slots = 0;
    if (ranged) block_range_records(from, to, &keep_lo, &keep_hi);
    for (WalkJob& j : jobs) {
        const uint64_t k = std::min<uint64_t>(j.max_blocks, keep_hi - keep_lo);
        if (ranged) j.max_blocks = 0xFFFFFFFFu;
        j.out = slots;
        j.keep_lo = keep_lo;
        j.keep_hi = keep_lo + k;
        slots += k;
    }
    CK(ctx->d_dl.ensure((size_t)slots * 16 + (size_t)ns * 8 + 64));
    uint64_t* d_boff = ctx->d_dl.as<uint64_t>();
    uint64_t* d_bbits = d_boff + slots;
    uint32_t* d_cnt = (uint32_t*)(d_bbits + slots);
    const WalkJob* d_jobs = nullptr;  // one stream: its job goes as a kernel parameter
    if (ns > 1) {
        Packer pk;
        const size_t o_wj = pk.add(jobs.data(), jobs.size() * sizeof(WalkJob));
        int rc = upload(ctx, pk);
        if (rc) return rc;
        d_jobs = (const WalkJob*)(ctx->d_tables.as<uint8_t>() + o_wj);
    }
    {
        LaunchScope ls(ctx, "stream_walk");
        stream_walk_kernel<<<(ns + 127) / 128, 128, 0, ctx->stream>>>(d_words, d_jobs, jobs[0], (int)ns, d_boff, d_bbits, d_cnt);
    }
    CK(cudaGetLastError());
    const uint64_t spec = std::min<uint64_t>(slots, 1024);
    const size_t cs_bytes = round16((uint64_t)ns * 8);
    CK(ctx->h_dl.ensure(cs_bytes + (size_t)spec * 16 + 64));
    const uint32_t* cs = (uint32_t*)ctx->h_dl.p;
    uint64_t* h_boff = (uint64_t*)((uint8_t*)ctx->h_dl.p + cs_bytes);
    uint64_t* h_bbits = h_boff + spec;
    CK(cudaMemcpyAsync(ctx->h_dl.p, d_cnt, (size_t)ns * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h_boff, d_boff, (size_t)spec * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h_bbits, d_bbits, (size_t)spec * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    out.assign(ns, Walked());
    uint64_t used = 0;  // entries up to the last stored record
    for (uint32_t s = 0; s < ns; s++) {
        Walked& w = out[s];
        w.n = cs[2 * s];
        w.first = keep_lo;
        w.status = (int32_t)cs[2 * s + 1];
        const uint64_t in_range = std::min(w.n, keep_hi) - std::min(w.n, keep_lo), k = jobs[s].keep_hi - keep_lo;
        w.overflow = in_range > k;
        if (w.status || w.overflow) continue;
        w.bit_off.resize(in_range);
        w.bits.resize(in_range);
        used = std::max(used, jobs[s].out + in_range);
    }
    if (used > spec) {  // the counts are read: h_dl now takes all stored records
        CK(ctx->h_dl.ensure((size_t)used * 16 + 64));
        h_boff = (uint64_t*)ctx->h_dl.p;
        h_bbits = h_boff + used;
        CK(cudaMemcpyAsync(h_boff, d_boff, (size_t)used * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(h_bbits, d_bbits, (size_t)used * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    for (uint32_t s = 0; s < ns; s++) {
        Walked& w = out[s];
        std::copy(h_boff + jobs[s].out, h_boff + jobs[s].out + w.bit_off.size(), w.bit_off.begin());
        std::copy(h_bbits + jobs[s].out, h_bbits + jobs[s].out + w.bits.size(), w.bits.begin());
    }
    return 0;
}

// jobs[b].bit_off / bits / block_size must be set; fills pre_len, mode, ..., status. d_words = device stream buffer.
int decode_parse_headers(kz_ctx* ctx, const uint32_t* d_words, std::vector<DecJob>& jobs, uint32_t checksum_bits) {
    const int nblocks = (int)jobs.size();
    if (nblocks == 0) return 0;
    std::vector<uint64_t> off(nblocks), bits(nblocks);
    std::vector<uint32_t> bs(nblocks);
    for (int b = 0; b < nblocks; b++) {
        off[b] = jobs[b].bit_off;
        bits[b] = jobs[b].bits;
        bs[b] = jobs[b].block_size;
    }
    Packer pk;
    const size_t o_off = pk.add(off.data(), off.size() * 8);
    const size_t o_bits = pk.add(bits.data(), bits.size() * 8);
    const size_t o_bs = pk.add(bs.data(), bs.size() * 4);
    const size_t o_out = pk.reserve(sizeof(BlockHeader) * (size_t)nblocks);
    int rc = upload(ctx, pk);
    if (rc) return rc;
    uint8_t* T = ctx->d_tables.as<uint8_t>();
    {
        LaunchScope ls(ctx, "block_header");
        block_header_kernel<<<(nblocks + 127) / 128, 128, 0, ctx->stream>>>(d_words, (uint64_t*)(T + o_off), (uint64_t*)(T + o_bits), nblocks, checksum_bits,
                                                                            (const uint32_t*)(T + o_bs), (BlockHeader*)(T + o_out));
    }
    CK(ctx->h_dl.ensure(sizeof(BlockHeader) * (size_t)nblocks));
    CK(cudaMemcpyAsync(ctx->h_dl.p, T + o_out, sizeof(BlockHeader) * (size_t)nblocks, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const BlockHeader* h = (const BlockHeader*)ctx->h_dl.p;
    for (int b = 0; b < nblocks; b++) {
        jobs[b].pre_len = h[b].pre_len;
        jobs[b].mode = h[b].mode;
        jobs[b].skip_flags = h[b].skip_flags;
        jobs[b].copy = h[b].copy;
        jobs[b].checksum = h[b].checksum;
        jobs[b].data_bit = h[b].data_bit;
        jobs[b].status = h[b].status;
    }
    return 0;
}

// Decodes the entropy data of every job (data_bit, pre_len must be valid) to d_out + out_off. with_end: fetch end_pos.
int decode_batch(kz_ctx* ctx, uint32_t etype, const uint32_t* d_words, uint64_t words_len, std::vector<DecJob>& jobs, uint8_t* d_out) {
    const int nblocks = (int)jobs.size();
    if (nblocks == 0) return 0;
    if (!etype_supported(etype)) return ctx->fail(KZ_ERR_INVALID_CODEC, "entropy codec not available on the GPU path");
    std::vector<DecBlock> dblocks(nblocks);
    std::vector<ExtractJob> xjobs;
    std::vector<int32_t> status(nblocks, 0);
    uint32_t nchunks_total = 0, max_chunks = 0;
    for (int b = 0; b < nblocks; b++) {
        DecJob& j = jobs[b];
        DecBlock& db = dblocks[b];
        db.data_bit = j.data_bit;
        db.end_bit = j.bit_off + j.bits;
        db.pre_len = j.pre_len;
        db.nchunks = 0;
        db.chunk_base = nchunks_total;
        db.chunk_size = 0;
        db.out_off = j.out_off;
        status[b] = j.status;
        if (j.status) continue;
        const uint32_t et = j.copy ? (uint32_t)KZ_E_NONE : etype;
        if (et == KZ_E_NONE || ((et == KZ_E_ANS0 || et == KZ_E_ANS1) && j.pre_len <= 32)) {
            if (j.data_bit + 8ull * j.pre_len > db.end_bit) {
                status[b] = j.status = -KZ_ERR_PROCESS_BLOCK;
                continue;
            }
            for (uint64_t o = 0; o < j.pre_len; o += RAW_PIECE) {
                ExtractJob x;
                x.src_bit = j.data_bit + 8 * o;
                x.dst_off = j.out_off + o;
                x.nbytes = (uint32_t)std::min<uint64_t>(RAW_PIECE, j.pre_len - o);
                x.pad = 0;
                xjobs.push_back(x);
            }
            j.end_pos = j.data_bit + 8ull * j.pre_len;
        } else {
            // the chunk descriptors are expanded on the device (expand_chunks_kernel); Range blocks are one serial chain: one entry
            const uint32_t cs = et == KZ_E_ANS0 ? (uint32_t)ANS0_CHUNK : et == KZ_E_ANS1 ? (uint32_t)ANS1_CHUNK : et == KZ_E_HUFFMAN ? (uint32_t)HUF_CHUNK
                                                                                                                                     : 0xFFFFFFFFu;
            db.chunk_size = cs;
            db.nchunks = cs == 0xFFFFFFFFu ? 1u : (uint32_t)(((uint64_t)j.pre_len + cs - 1) / cs);
            nchunks_total += db.nchunks;
            max_chunks = std::max(max_chunks, db.nchunks);
        }
    }
    const int nchunks = (int)nchunks_total;
    Packer pk;
    const size_t o_blocks = pk.add(dblocks.data(), dblocks.size() * sizeof(DecBlock));
    const size_t o_x = pk.add(xjobs.data(), xjobs.size() * sizeof(ExtractJob));
    const size_t o_status = pk.add(status.data(), status.size() * 4);
    const size_t o_hbit = pk.reserve((size_t)nchunks * 8 + 8);
    const size_t o_end = pk.reserve((size_t)nblocks * 8 + 8);
    int rc = upload(ctx, pk);
    if (rc) return rc;
    uint8_t* T = ctx->d_tables.as<uint8_t>();
    int32_t* d_status = (int32_t*)(T + o_status);
    CK(ctx->d_chunks.ensure((size_t)nchunks * sizeof(DecChunk) + 64));
    DecChunk* d_dchunks = ctx->d_chunks.as<DecChunk>();
    if (nchunks > 0) {
        LaunchScope ls(ctx, "expand_chunks");
        expand_chunks_kernel<<<dim3((max_chunks + 255) / 256, nblocks), 256, 0, ctx->stream>>>((DecBlock*)(T + o_blocks), nblocks, d_dchunks);
    }
    if (nchunks > 0 && etype == KZ_E_ANS1) {
        CK(ctx->d_enc_tab.ensure((size_t)nchunks * 65536 * sizeof(uint32_t)));
        CK(ctx->d_hist.ensure((size_t)nchunks * 256 * 2048 + 256));
        {
            LaunchScope ls(ctx, "ans_walk");
            ans_walk_kernel<<<(nblocks + 31) / 32, 32, 0, ctx->stream>>>(d_words, (DecBlock*)(T + o_blocks), nblocks, 1, (uint64_t*)(T + o_hbit),
                                                                         (uint64_t*)(T + o_end), d_status);
        }
        LaunchScope ls(ctx, "ans1_decode");
        ans1_decode_kernel<<<nchunks, 32, 0, ctx->stream>>>(d_words, words_len, d_dchunks, nchunks, (uint64_t*)(T + o_hbit),
                                                            ctx->d_hist.as<uint8_t>(), ctx->d_enc_tab.as<uint32_t>(), d_out, d_status);
    } else if (nchunks > 0 && etype == KZ_E_RANGE) {
        LaunchScope ls(ctx, "range_decode");
        range_decode_kernel<<<nblocks, 32, 0, ctx->stream>>>(d_words, (DecBlock*)(T + o_blocks), d_dchunks, nblocks, d_out,
                                                             (uint64_t*)(T + o_end), d_status);
    } else if (nchunks > 0 && etype == KZ_E_HUFFMAN) {
        {
            LaunchScope ls(ctx, "huf_walk");
            huf_walk_kernel<<<nblocks, 32, 0, ctx->stream>>>(d_words, words_len, (DecBlock*)(T + o_blocks), nblocks, (uint64_t*)(T + o_hbit),
                                                             (uint64_t*)(T + o_end), d_status);
        }
        LaunchScope ls(ctx, "huf_decode");
        huf_decode_kernel<<<(nchunks + HUF_DEC_CTA_CHUNKS - 1) / HUF_DEC_CTA_CHUNKS, HUF_DEC_CTA_CHUNKS * 4, HUF_DEC_SMEM, ctx->stream>>>(
            d_words, words_len, d_dchunks, nchunks, (uint64_t*)(T + o_hbit), d_out, d_status);
    } else if (nchunks > 0) {
        {
            LaunchScope ls(ctx, "ans_walk");
            ans0_walk_kernel<<<nblocks, 32, 0, ctx->stream>>>(d_words, words_len, (DecBlock*)(T + o_blocks), nblocks, (uint64_t*)(T + o_hbit),
                                                              (uint64_t*)(T + o_end), d_status);
        }
        {
            CK(ctx->d_enc_tab.ensure((size_t)nchunks * DEC_TAB_WORDS * sizeof(uint32_t) + 256));
            LaunchScope ls(ctx, "ans0_tables");
            ans0_tables_kernel<<<(nchunks + 3) / 4, 128, 0, ctx->stream>>>(d_words, words_len, d_dchunks, nchunks, (uint64_t*)(T + o_hbit),
                                                                        ctx->d_enc_tab.as<uint32_t>(), d_out, d_status);
        }
        LaunchScope ls(ctx, "ans0_decode");
        ans0_decode_kernel<<<(nchunks + DEC_CTA_CHUNKS - 1) / DEC_CTA_CHUNKS, 64, DEC_SMEM, ctx->stream>>>(
            d_words, words_len, ctx->d_enc_tab.as<uint32_t>(), d_dchunks, nchunks, (uint64_t*)(T + o_hbit), d_out, d_status);
    }
    if (!xjobs.empty()) {
        LaunchScope ls(ctx, "extract");
        extract_copy_kernel<<<(int)xjobs.size(), 256, 0, ctx->stream>>>(d_words, (ExtractJob*)(T + o_x), (int)xjobs.size(), d_out);
    }
    CK(cudaGetLastError());
    CK(ctx->h_dl.ensure((size_t)nblocks * 16 + 64));
    int32_t* hs = (int32_t*)ctx->h_dl.p;
    uint64_t* he = (uint64_t*)((uint8_t*)ctx->h_dl.p + (((size_t)nblocks * 4 + 15) & ~size_t(15)));
    CK(cudaMemcpyAsync(hs, d_status, (size_t)nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(he, T + o_end, (size_t)nblocks * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < nblocks; b++) {
        jobs[b].status = hs[b];
        if (dblocks[b].nchunks) jobs[b].end_pos = he[b];
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------------------
// stream header (Writer.writeHeader io/CompressedStream.go:429-519, Reader.readHeader :1316-1460)
// ------------------------------------------------------------------------------------------------------------
uint32_t header_checksum(uint32_t ck_size, uint32_t etype, uint64_t t48, uint32_t block_size, uint32_t sz_mask, int64_t input_size) {
    const uint32_t HASH = 0x1E35A7BDu;
    uint32_t ck = HASH * (0x01030507u * BS_VERSION);
    ck ^= HASH * ~ck_size;
    ck ^= HASH * ~etype;
    ck ^= HASH * (uint32_t)((~t48) >> 32);
    ck ^= HASH * (uint32_t)(~t48);
    ck ^= HASH * ~block_size;
    if (sz_mask > 0) {
        ck ^= HASH * (uint32_t)(((uint64_t)~input_size) >> 32);
        ck ^= HASH * (uint32_t)(~input_size);
    }
    return ((ck >> 23) ^ (ck >> 3)) & 0xFFFFFFu;
}

uint32_t build_stream_header(std::vector<uint8_t>& out, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, int64_t input_size) {
    out.assign(64, 0);
    BitWriter bw(out.data());
    const uint32_t ck_size = checksum_bits == 32 ? 1 : (checksum_bits == 64 ? 2 : 0);
    bw.write(BS_TYPE, 32);
    bw.write(BS_VERSION, 4);
    bw.write(ck_size, 2);
    bw.write(etype, 5);
    bw.write((uint32_t)(t48 >> 32), 16);
    bw.write((uint32_t)t48, 32);
    bw.write(block_size >> 4, 28);
    uint32_t sz_mask;
    if (input_size <= 0 || input_size >= ((int64_t)1 << 48)) sz_mask = 0;
    else if (input_size >= ((int64_t)1 << 32)) sz_mask = 3;
    else if (input_size >= ((int64_t)1 << 16)) sz_mask = 2;
    else sz_mask = 1;
    bw.write(sz_mask, 2);
    if (sz_mask == 3) bw.write((uint32_t)((uint64_t)input_size >> 32), 16);
    if (sz_mask >= 2) bw.write((uint32_t)input_size, 32);
    if (sz_mask == 1) bw.write((uint32_t)input_size, 16);
    bw.write(0, 15);
    bw.write(header_checksum(ck_size, etype, t48, block_size, sz_mask, sz_mask ? input_size : 0), 24);
    return bw.pos;
}

struct StreamHeader {
    uint64_t t48;
    uint32_t etype, block_size, checksum_bits;
    int64_t input_size;
    uint64_t bits;  // header length
};

int parse_stream_header(kz_ctx* ctx, const uint8_t* bytes, size_t n, StreamHeader& h) {
    uint32_t tmp[20];
    memset(tmp, 0, sizeof(tmp));
    memcpy(tmp, bytes, std::min<size_t>(n, 64));
    BitReader br(tmp, 0, 8ull * std::min<size_t>(n, 64));
    if (br.read(32) != BS_TYPE) return ctx->fail(KZ_ERR_INVALID_FILE, "Invalid stream type");
    uint32_t ver = br.read(4);
    if (ver != BS_VERSION) return ctx->fail(KZ_ERR_STREAM_VERSION, "Only bitstream version 6 is supported");
    uint32_t ck_size = br.read(2);
    if (ck_size == 3) return ctx->fail(KZ_ERR_INVALID_CODEC, "Invalid bitstream, incorrect checksum size");
    h.checksum_bits = 32 * ck_size;
    h.etype = br.read(5);
    uint64_t hi = br.read(16);
    h.t48 = (hi << 32) | br.read(32);
    h.block_size = br.read(28) << 4;
    if (h.block_size < 1024 || h.block_size > (1u << 30)) return ctx->fail(KZ_ERR_BLOCK_SIZE, "Invalid bitstream, incorrect block size");
    uint32_t sz_mask = br.read(2);
    h.input_size = 0;
    if (sz_mask == 3) h.input_size = (int64_t)br.read(16) << 32;
    if (sz_mask >= 2) h.input_size |= br.read(32);
    if (sz_mask == 1) h.input_size = br.read(16);
    br.read(15);
    uint32_t ck1 = br.read(24);
    if (br.overrun) return ctx->fail(KZ_ERR_INVALID_FILE, "Invalid bitstream: truncated header");
    if (ck1 != header_checksum(ck_size, h.etype, h.t48, h.block_size, sz_mask, h.input_size))
        return ctx->fail(KZ_ERR_CRC_CHECK, "Invalid bitstream: checksum mismatch");
    h.bits = br.pos;
    return 0;
}

// A headerless stream (kz_set_headerless_reader, NewHeaderlessReader io/CompressedStream.go:1060) has no header to parse (readHeader is
// skipped, :1317): its fields are the setting's, and its first record starts at bit 0.
StreamHeader headerless_header(const kz_ctx* ctx) {
    const kz_ctx::Headerless& s = ctx->headerless_reader;
    StreamHeader h;
    h.t48 = s.t48;
    h.etype = s.etype;
    h.block_size = s.block_size;
    h.checksum_bits = s.checksum_bits;
    h.input_size = s.output_size;
    h.bits = 0;
    return h;
}

// The header of a stream of n bytes whose first min(n, 64) bytes are head (zero padded): the headerless reader setting when one is in
// force, else the header parsed from head.
int stream_header(kz_ctx* ctx, const uint8_t* head, size_t n, StreamHeader& sh) {
    if (ctx->headerless_reader.on) {
        sh = headerless_header(ctx);
        return 0;
    }
    return parse_stream_header(ctx, head, n, sh);
}

int count_transforms(uint64_t t48, uint64_t* ids) {
    int n = 0;
    for (int i = 0; i < 8; i++) {
        uint64_t t = (t48 >> (42 - 6 * i)) & 63;
        if (t != 0) ids[n++] = t;
    }
    if (n == 0) ids[n++] = 0;  // Factory.New :73-76 keeps one NONE
    return n;
}

// kanzi's skipBlocks option (encodingTask.encode, io/CompressedStream.go:778-800), device half: the order-0 histogram of every block
// d_base + off[b] (len[b] bytes, any alignment) and its entropy test (kz_skip.cu). The blocks of at most SMALL_BLOCK bytes, stored in any
// case, are not read. On return the work is queued, and *d_flags points at nb flag bytes of ctx->d_skip (1: the order-0 entropy reaches
// INCOMPRESSIBLE_THRESHOLD) for stored_blocks (kz_stream_plan.h).
int skip_test(kz_ctx* ctx, const uint8_t* d_base, const std::vector<uint64_t>& off, const std::vector<uint32_t>& len, const uint8_t** d_flags) {
    const uint32_t nb = (uint32_t)len.size();
    std::vector<SkipTile> tiles;
    for (uint32_t b = 0; b < nb; b++)
        if (len[b] > SMALL_BLOCK)
            for (uint32_t o = 0; o < len[b]; o += SKIP_TILE) tiles.push_back(SkipTile{off[b] + o, std::min(SKIP_TILE, len[b] - o), b});
    const size_t o_flags = (size_t)nb * 256 * 4;  // behind the histograms
    CK(ctx->d_skip.ensure(o_flags + nb));
    uint8_t* S = ctx->d_skip.as<uint8_t>();
    CK(cudaMemsetAsync(S, 0, o_flags, ctx->stream));
    Packer pk;
    const size_t o_tiles = pk.add(tiles.data(), tiles.size() * sizeof(SkipTile));
    const size_t o_len = pk.add(len.data(), (size_t)nb * 4);
    const size_t o_log2 = pk.add(host_log2_4096(), 257 * 4);
    int rc = upload(ctx, pk);
    if (rc) return rc;
    const uint8_t* T = ctx->d_tables.as<uint8_t>();
    if (!tiles.empty()) {
        LaunchScope ls(ctx, "skip_hist");
        skip_hist_kernel<<<(uint32_t)((tiles.size() + SKIP_HIST_WARPS - 1) / SKIP_HIST_WARPS), 32 * SKIP_HIST_WARPS, 0, ctx->stream>>>(
            d_base, (const SkipTile*)(T + o_tiles), (uint32_t)tiles.size(), (uint32_t*)S);
    }
    {
        LaunchScope ls(ctx, "skip_decide");
        skip_decide_kernel<<<(nb + 255) / 256, 256, 0, ctx->stream>>>((const uint32_t*)S, (const uint32_t*)(T + o_len), nb, (const uint32_t*)(T + o_log2),
                                                                     S + o_flags);
    }
    CK(cudaGetLastError());
    *d_flags = S + o_flags;
    return 0;
}

struct TransformPlan {
    int nt = 0;
    uint64_t ids[8];
    bool none() const { return nt == 1 && ids[0] == KZ_T_NONE; }
    // the transforms that exist as GPU stages; every plan but NONE is a sequence of them
    static bool seq_id(uint64_t t) {
        return t == KZ_T_BWT || t == KZ_T_BWTS || t == KZ_T_RANK || t == KZ_T_MTFT || t == KZ_T_ZRLT || t == KZ_T_ROLZ || t == KZ_T_PACK || t == KZ_T_DNA || t == KZ_T_LZ ||
               t == KZ_T_LZX || t == KZ_T_MM || t == KZ_T_TEXT || t == KZ_T_UTF || t == KZ_T_EXE;
    }
    // stages that read ctx["dataType"] in a way the block's magic number can change (LZ / LZX only look for DNA / small alphabets)
    bool uses_magic() const {
        for (int i = 0; i < nt; i++)
            if (ids[i] == KZ_T_ROLZ || ids[i] == KZ_T_PACK || ids[i] == KZ_T_DNA || ids[i] == KZ_T_MM || ids[i] == KZ_T_TEXT || ids[i] == KZ_T_UTF || ids[i] == KZ_T_EXE) return true;
        return false;
    }
};
const char* const NO_GPU_TRANSFORM = "transform not available on the GPU path (BWT, BWTS, LZ, LZX, ROLZ, RANK, MTFT, ZRLT, PACK, DNA, MM, TEXT, UTF, EXE are)";

// etype: the entropy codec of the stream. The reference picks the TEXT encoding from it (transform/Factory.go:99-119): encoding 2 for NONE /
// ANS0 / HUFFMAN / RANGE, encoding 1 otherwise; only encoding 2 (textCodec2) exists here, so TEXT with any other codec is refused
// rather than written in a form the reference could not read.
int plan_transforms(kz_ctx* ctx, uint64_t t48, uint32_t etype, TransformPlan& p, int err_code) {
    p.nt = count_transforms(t48, p.ids);
    for (int i = 0; i < p.nt; i++)
        if (p.ids[i] == KZ_T_TEXT && !(etype == KZ_E_NONE || etype == KZ_E_ANS0 || etype == KZ_E_HUFFMAN || etype == KZ_E_RANGE))
            return ctx->fail(err_code, "TEXT with this entropy codec selects the reference's text encoding 1, which the GPU path does not implement (NONE / ANS0 / HUFFMAN / RANGE select encoding 2)");
    for (int i = 0; i < p.nt; i++)
        if (p.ids[i] == KZ_T_TEXT && !text_available())
            return ctx->fail(err_code, "TEXT: the library was built without the static dictionary (kanzi-go_b200/gen_text_dict.py)");
    if (!p.none())
        for (int i = 0; i < p.nt; i++)
            if (!TransformPlan::seq_id(p.ids[i]))
                return ctx->fail(err_code, "transform sequence not available on the GPU path (sequences of BWT / BWTS / LZ / LZX / ROLZ / RANK / MTFT / ZRLT / PACK / DNA / MM / TEXT / UTF / EXE are)");
    return 0;
}


// ------------------------------------------------------------------------------------------------------------
// Transform sequences (ByteTransformSequence, transform/Sequence.go:64-186): every plan but NONE, one stage or several. Every stage
// processes all blocks of the batch; a stage that declines a block ("skip", Sequence.go:100-105) leaves its skip bit set and the block
// moves on unchanged.
// ------------------------------------------------------------------------------------------------------------
// The blocks of one stage call: block b is read at b * istride and written at b * ostride. A forward call passes `applied` (and `dts` when
// the caller keeps ctx["dataType"]); an inverse call passes neither.
struct StageIo {
    uint64_t istride, ostride;
    std::vector<uint32_t>& len;
    const std::vector<uint8_t>& active;
    std::vector<uint8_t>* applied;
    std::vector<int32_t>* dts;
};

// A stage with one descriptor and one StageResult per block (ROLZ, TEXT, UTF, EXE, MM, PACK / DNA; Block is RolzBlock for ROLZ, which
// carries a scratch offset, StageBlock otherwise). Every sub-batch of `sub` blocks (0: the whole batch) that holds an active block gets
// its descriptors (offsets, len, data_type; `desc` sets cap and the stage's own fields), ws(b0, nb, max_len) bytes of workspace for blocks
// b0 .. b0 + nb - 1, one upload of the descriptors with room for the results, one `launch` (the stage's kernels, given b0 as well) under a
// LaunchScope named `scope`, and the results
// copied back. Forward: status 0 = transformed, anything else = declined, ctx["dataType"] after the call is kept for every active block;
// a negative status fails with `bad` when one is given (EXE: a block the reference panics on). Inverse: any status but 0 fails with `bad`.
template <class Block, class Desc, class Ws, class Launch>
int run_desc_stage(kz_ctx* ctx, const StageIo& io, const char* scope, uint32_t sub, Desc desc, Ws ws, Launch launch, const char* bad = nullptr) {
    const uint32_t nblocks = (uint32_t)io.len.size();
    if (sub == 0) sub = nblocks;
    for (uint32_t b0 = 0; b0 < nblocks; b0 += sub) {
        const uint32_t nb = std::min(sub, nblocks - b0);
        uint32_t max_len = 0;
        for (uint32_t b = b0; b < b0 + nb; b++) max_len = std::max(max_len, io.active[b] ? io.len[b] : 0u);
        if (max_len == 0) continue;
        std::vector<Block> hb(nb);
        for (uint32_t k = 0; k < nb; k++) {
            const uint32_t b = b0 + k;
            hb[k] = Block{};
            hb[k].src_off = b * io.istride;
            hb[k].dst_off = b * io.ostride;
            hb[k].len = io.active[b] ? io.len[b] : 0;
            hb[k].data_type = io.dts ? (*io.dts)[b] : 0;
            desc(hb[k], b);
        }
        CK(ctx->d_ws.ensure(ws(b0, nb, max_len)));
        Packer pk;
        const size_t o_blk = pk.add(hb.data(), hb.size() * sizeof(Block));
        const size_t o_res = pk.reserve((size_t)nb * sizeof(StageResult));
        int rc = upload(ctx, pk);
        if (rc) return rc;
        uint8_t* T = ctx->d_tables.as<uint8_t>();
        {
            LaunchScope ls(ctx, scope);
            cudaError_t e = launch(b0, (const Block*)(T + o_blk), hb.data(), nb, max_len, (StageResult*)(T + o_res));
            if (e != cudaSuccess) return ctx->cuda_fail(e, scope);
        }
        std::vector<StageResult> hr(nb);
        CK(cudaMemcpyAsync(hr.data(), T + o_res, (size_t)nb * sizeof(StageResult), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (uint32_t k = 0; k < nb; k++) {
            const uint32_t b = b0 + k;
            if (!io.active[b] || io.len[b] == 0) continue;
            if (!io.applied) {
                if (hr[k].status) return ctx->fail(KZ_ERR_PROCESS_BLOCK, bad);
                io.len[b] = hr[k].out_len;
                continue;
            }
            if (hr[k].status < 0 && bad) return ctx->fail(KZ_ERR_PROCESS_BLOCK, bad);
            if (io.dts) (*io.dts)[b] = hr[k].data_type;
            if (hr[k].status == 0) {
                (*io.applied)[b] = 1;
                io.len[b] = hr[k].out_len;
            }
        }
    }
    return 0;
}

// One forward stage. Block b: d_in + b*istride (len[b] bytes) -> d_out + b*ostride. applied[b] = 1 and len[b] updated on success.
// bs[b]: ctx["blockSize"] of block b's stream, 0 when the caller has none (TEXT then takes the longest block of the call).
int apply_forward(kz_ctx* ctx, uint64_t t, const uint8_t* d_in, uint64_t istride, uint8_t* d_out, uint64_t ostride, std::vector<uint32_t>& len,
                  const std::vector<uint8_t>& active, std::vector<uint8_t>& applied, const std::vector<uint64_t>& bs, std::vector<int32_t>* dts = nullptr) {
    const uint32_t nblocks = (uint32_t)len.size();
    applied.assign(nblocks, 0);
    const StageIo io{istride, ostride, len, active, &applied, dts};
    if (t == KZ_T_BWT) {
        CK(ctx->d_lens.ensure((size_t)nblocks * 4 + 64));
        uint32_t* d_post = ctx->d_lens.as<uint32_t>();
        // all blocks of a sub-batch are suffix-sorted together (kz_bwt.cu: bwt_forward_batch)
        for (uint32_t b0 = 0; b0 < nblocks;) {
            std::vector<uint64_t> so, dof;
            std::vector<uint32_t> nn, num;
            uint64_t total = 0;
            uint32_t b = b0;
            for (; b < nblocks; b++) {
                if (!active[b] || len[b] < 2) continue;
                if (len[b] > bwt_forward_batch_max_total()) {  // a block the batch's key layout cannot hold (1 GiB): its own suffix sort
                    if (!nn.empty()) break;                    // flush what has been collected first
                    CK(ctx->d_ws.ensure(bwt_forward_workspace(len[b])));
                    LaunchScope ls(ctx, "bwt_forward");
                    cudaError_t e = bwt_forward_device(d_in + b * istride, len[b], d_out + b * ostride, d_post + b, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap,
                                                       ctx->stream, &ctx->launches);
                    if (e == cudaSuccess) applied[b] = 1;
                    else if (e != cudaErrorInvalidValue) return ctx->cuda_fail(e, "bwt_forward");
                    continue;
                }
                if (!nn.empty() && (total + len[b] > bwt_forward_batch_max_total() || nn.size() >= bwt_forward_batch_max_blocks())) break;
                so.push_back(b * istride), dof.push_back(b * ostride), nn.push_back(len[b]), num.push_back(b);
                total += len[b];
            }
            b0 = b;
            if (nn.empty()) continue;
            CK(ctx->d_ws.ensure(bwt_forward_batch_workspace(total, (uint32_t)nn.size())));
            LaunchScope ls(ctx, "bwt_forward");
            CtxLzHook round_hook(ctx);  // kz_bwt_profile bit 0: every round timed under its own name
            cudaError_t e = bwt_forward_batch(d_in, d_out, so.data(), dof.data(), nn.data(), num.data(), (uint32_t)nn.size(), d_post, ctx->d_ws.as<uint8_t>(),
                                              ctx->d_ws.cap, ctx->stream, &ctx->launches, (ctx->profile && (ctx->bwt_profile & 1)) ? &round_hook : nullptr,
                                              (ctx->bwt_profile & 2) != 0);
            if (e != cudaSuccess) return ctx->cuda_fail(e, "bwt_forward");
            for (uint32_t k : num) applied[k] = 1;
        }
        std::vector<uint32_t> post(nblocks);
        CK(cudaMemcpyAsync(post.data(), d_post, (size_t)nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (uint32_t b = 0; b < nblocks; b++)
            if (applied[b]) len[b] = post[b];
    } else if (t == KZ_T_BWTS) {  // BWTS.Forward: n bytes -> n bytes, never declines
        uint32_t max_len = 0;
        for (uint32_t b = 0; b < nblocks; b++) max_len = std::max(max_len, len[b]);
        CK(ctx->d_ws.ensure(bwts_forward_workspace(max_len)));
        for (uint32_t b = 0; b < nblocks; b++) {
            if (!active[b] || len[b] == 0) continue;
            LaunchScope ls(ctx, "bwts_forward");
            cudaError_t e = bwts_forward_device(d_in + b * istride, len[b], d_out + b * ostride, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, ctx->stream,
                                                &ctx->launches);
            if (e != cudaSuccess) return ctx->cuda_fail(e, "bwts_forward");
            applied[b] = 1;
        }
    } else if (t == KZ_T_ROLZ) {  // ROLZCodec.Forward: declines small blocks and blocks it cannot shrink
        uint32_t max_len = 0;
        for (uint32_t b = 0; b < nblocks; b++) max_len = std::max(max_len, len[b]);
        const size_t sstride = rolz_scratch_bytes(max_len);
        return run_desc_stage<RolzBlock>(
            ctx, io, "rolz_forward", 0,
            [&](RolzBlock& d, uint32_t b) {
                d.scratch_off = b * sstride;
                d.cap = (uint32_t)std::min<uint64_t>(ostride, 0xFFFFFFF0u);
            },
            [&](uint32_t, uint32_t nb, uint32_t) { return sstride * nb + 256; },
            [&](uint32_t, const RolzBlock* db, const RolzBlock*, uint32_t nb, uint32_t, StageResult* res) {
                rolz_forward_kernel<<<nb, 32, 0, ctx->stream>>>(d_in, db, (int)nb, ctx->d_ws.as<uint8_t>(), d_out, res);
                return cudaGetLastError();
            });
    } else if (t == KZ_T_LZ || t == KZ_T_LZX) {  // LZCodec as a stage of a sequence (e.g. "DNA+LZ" = kanzi -l 2)
        const bool extra = t == KZ_T_LZX;
        uint32_t max_len = 0;
        for (uint32_t b = 0; b < nblocks; b++) max_len = std::max(max_len, len[b]);
        if ((uint64_t)max_len + max_len / 64 + 128 > ostride) return ctx->fail(KZ_ERR_UNKNOWN, "internal: stage buffer too small for LZ");
        const uint64_t sstride = (lz_scratch_bytes(max_len) + 255) & ~size_t(255);
        std::vector<LzBlock> lb(nblocks);
        for (uint32_t b = 0; b < nblocks; b++) {
            lb[b].src_off = b * istride;
            lb[b].dst_off = b * ostride;
            lb[b].scratch_off = (uint64_t)b * sstride;
            lb[b].len = active[b] ? len[b] : 0;
            lb[b].cap = 0;
            lb[b].data_type = dts ? (*dts)[b] : 0;
            lb[b].pad = 0;
        }
        std::vector<LzResult> hres;
        {
            int rc = lz_forward_batch(ctx, d_in, d_out, lb, extra, hres);
            if (rc) return rc;
        }
        for (uint32_t b = 0; b < nblocks; b++)
            if (active[b] && len[b] && hres[b].status == 0) {
                applied[b] = 1;
                len[b] = hres[b].out_len;
            }
    } else if (t == KZ_T_TEXT) {  // TextCodec (encoding 2): declines unless the block looks like text
        if (!text_available()) return ctx->fail(KZ_ERR_CREATE_CODEC, "TEXT: the library was built without the static dictionary");
        std::vector<uint64_t> sbs(bs);
        const uint64_t longest = *std::max_element(len.begin(), len.end());
        for (uint64_t& v : sbs) v = v ? v : longest;
        uint64_t serial = 0;
        const int rc = run_desc_stage<StageBlock>(
            ctx, io, "text_forward", 64,                          // ~9 MB of dictionary per block
            [&](StageBlock& d, uint32_t b) { d.cap = len[b]; },  // MaxEncodedLen = srcLen (:1720-1724)
            [&](uint32_t b0, uint32_t nb, uint32_t max_len) { return text_workspace(&sbs[b0], nb, max_len); },
            [&](uint32_t b0, const StageBlock* db, const StageBlock* hb, uint32_t nb, uint32_t max_len, StageResult* res) {
                return text_forward_batch(d_in, d_out, db, hb, nb, max_len, &sbs[b0], ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, res, ctx->stream, &ctx->launches,
                                          &serial);
            });
        if (ctx->profile && serial) ctx->prof["text_forward_serial"].launches += serial;  // blocks the serial walk did (kz_kernel_time count)
        return rc;
    } else if (t == KZ_T_UTF) {  // UTFCodec.Forward: declines unless the block is UTF-8 with enough multi-byte sequences
        return run_desc_stage<StageBlock>(
            ctx, io, "utf_forward", 32,  // 16 MB of code point counters per block
            [&](StageBlock& d, uint32_t b) { d.cap = (uint32_t)std::min<uint64_t>((uint64_t)len[b] + 8192, 0xFFFFFFF0u); },  // MaxEncodedLen (:386-388)
            [](uint32_t, uint32_t nb, uint32_t) { return utf_workspace(nb); },
            [&](uint32_t, const StageBlock* db, const StageBlock*, uint32_t nb, uint32_t, StageResult* res) {
                return utf_forward_batch(d_in, d_out, db, nb, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, res, ctx->stream, &ctx->launches);
            });
    } else if (t == KZ_T_EXE) {  // EXECodec.Forward: declines unless the block is x86 / ARM64 code
        auto mel = [](uint32_t n) { return n <= 256 ? (uint64_t)n + 32 : (uint64_t)n + n / 8; };  // MaxEncodedLen (:701-708)
        for (uint32_t b = 0; b < nblocks; b++)
            if (active[b] && mel(len[b]) > ostride) return ctx->fail(KZ_ERR_UNKNOWN, "internal: stage buffer too small for EXE");
        return run_desc_stage<StageBlock>(
            ctx, io, "exe_forward", 0, [&](StageBlock& d, uint32_t b) { d.cap = (uint32_t)std::min<uint64_t>(mel(len[b]), 0xFFFFFFF0u); },
            [](uint32_t, uint32_t, uint32_t) { return (size_t)0; },
            [&](uint32_t, const StageBlock* db, const StageBlock*, uint32_t nb, uint32_t, StageResult* res) {
                exe_forward_kernel<<<nb, 32, 0, ctx->stream>>>(d_in, db, (int)nb, d_out, res);
                return cudaGetLastError();
            },
            "EXE codec: malformed executable header (the reference panics on this block)");
    } else if (t == KZ_T_MM) {  // FSDCodec.Forward: declines unless a fixed-step delta lowers the sampled entropy
        for (uint32_t b = 0; b < nblocks; b++)
            if (active[b] && fsd_max_encoded_len(len[b]) > ostride) return ctx->fail(KZ_ERR_UNKNOWN, "internal: stage buffer too small for MM");
        return run_desc_stage<StageBlock>(
            ctx, io, "fsd_forward", 1024,
            [&](StageBlock& d, uint32_t b) { d.cap = fsd_max_encoded_len(len[b]); },  // the sequence sizes dst with MaxEncodedLen (Sequence.go:81-93)
            [](uint32_t, uint32_t nb, uint32_t max_len) { return fsd_workspace(nb, max_len); },
            [&](uint32_t, const StageBlock* db, const StageBlock*, uint32_t nb, uint32_t max_len, StageResult* res) {
                return fsd_forward_batch(d_in, d_out, db, nb, max_len, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, res, ctx->stream, &ctx->launches);
            });
    } else if (t == KZ_T_PACK || t == KZ_T_DNA) {  // AliasCodec.Forward: bit packing of small alphabets / digram aliases; often declines
        return run_desc_stage<StageBlock>(
            ctx, io, "alias_forward", 256,  // blocks per launch sequence (bounds the workspace: ~390 KB per block)
            [&](StageBlock& d, uint32_t b) {
                d.cap = (uint32_t)std::min<uint64_t>((uint64_t)len[b] + 1024, 0xFFFFFFF0u);  // the sequence sizes dst with MaxEncodedLen (Sequence.go:81-93)
                d.flags = t == KZ_T_DNA ? 1u : 0u;
            },
            [](uint32_t, uint32_t nb, uint32_t max_len) { return alias_workspace(nb, max_len); },
            [&](uint32_t, const StageBlock* db, const StageBlock*, uint32_t nb, uint32_t max_len, StageResult* res) {
                return alias_forward_batch(d_in, d_out, db, nb, max_len, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, res, ctx->stream, &ctx->launches);
            });
    } else if (t == KZ_T_RANK || t == KZ_T_MTFT) {  // SBRT.Forward never declines (buffers are sized for MaxEncodedLen)
        std::vector<SbrtBlock> sb(nblocks);
        std::vector<uint32_t> seg_block;
        uint32_t max_segs = 0, max_len = 0;
        for (uint32_t b = 0; b < nblocks; b++) {
            sb[b].src_off = b * istride;
            sb[b].dst_off = b * ostride;
            sb[b].len = len[b];
            sb[b].seg_base = (uint32_t)seg_block.size();
            sb[b].active = active[b] && len[b] > 0;
            sb[b].pad = 0;
            const uint32_t nseg = sb[b].active ? (len[b] + SBRT_SEG_BYTES - 1) / SBRT_SEG_BYTES : 0;
            max_segs = std::max(max_segs, nseg);
            if (sb[b].active) max_len = std::max(max_len, len[b]);
            for (uint32_t s = 0; s < nseg; s++) seg_block.push_back(b);
            applied[b] = sb[b].active ? 1 : 0;
        }
        const uint32_t nsegs = (uint32_t)seg_block.size();
        if (nsegs) {
            Packer pk;
            const size_t o_sb = pk.add(sb.data(), sb.size() * sizeof(SbrtBlock));
            const size_t o_map = pk.add(seg_block.data(), seg_block.size() * 4);
            int rc = upload(ctx, pk);
            if (rc) return rc;
            CK(ctx->d_seg.ensure((size_t)nsegs * 512 * 4 + 64));
            uint8_t* T = ctx->d_tables.as<uint8_t>();
            const SbrtBlock* d_sb = (const SbrtBlock*)(T + o_sb);
            const int mode = t == KZ_T_MTFT ? 1 : 2;
            {
                LaunchScope ls(ctx, "sbrt_last2");
                sbrt_last2_kernel<<<dim3(max_segs, nblocks), 256, 0, ctx->stream>>>(d_in, d_sb, ctx->d_seg.as<int32_t>());
            }
            {
                LaunchScope ls(ctx, "sbrt_carry");
                sbrt_carry_kernel<<<nblocks, 256, 0, ctx->stream>>>(d_sb, ctx->d_seg.as<int32_t>());
            }
            {
                LaunchScope ls(ctx, "sbrt_rank");
                sbrt_rank_launch(d_in, d_sb, mode, (const uint32_t*)(T + o_map), nsegs, ctx->d_seg.as<int32_t>(), d_out, max_len, ctx->stream);
            }
            CK(cudaGetLastError());
            CK(cudaStreamSynchronize(ctx->stream));  // the tables live in d_tables, which the next stage reuses
        }
    } else if (t == KZ_T_ZRLT) {
        std::vector<ZrltBlock> zb(nblocks);
        for (uint32_t b = 0; b < nblocks; b++) {
            zb[b].src_off = b * istride;
            zb[b].dst_off = b * ostride;
            zb[b].len = len[b];
            zb[b].cap = len[b];
            zb[b].active = active[b] && len[b] > 0;
            zb[b].pad = 0;
        }
        Packer pk;
        const size_t o_zb = pk.add(zb.data(), zb.size() * sizeof(ZrltBlock));
        const size_t o_len = pk.reserve((size_t)nblocks * 4);
        const size_t o_st = pk.reserve((size_t)nblocks * 4);
        int rc = upload(ctx, pk);
        if (rc) return rc;
        uint8_t* T = ctx->d_tables.as<uint8_t>();
        {
            LaunchScope ls(ctx, "zrlt_forward");
            zrlt_forward_kernel<<<nblocks, 512, 0, ctx->stream>>>(d_in, (const ZrltBlock*)(T + o_zb), (int)nblocks, d_out, (uint32_t*)(T + o_len),
                                                                  (int32_t*)(T + o_st));
        }
        CK(cudaGetLastError());
        std::vector<uint32_t> hl(nblocks);
        std::vector<int32_t> hs(nblocks);
        CK(cudaMemcpyAsync(hl.data(), T + o_len, (size_t)nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(hs.data(), T + o_st, (size_t)nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (uint32_t b = 0; b < nblocks; b++) {
            if (zb[b].active && hs[b] == 0) {
                applied[b] = 1;
                len[b] = hl[b];
            }
        }
    } else {
        return ctx->fail(KZ_ERR_CREATE_CODEC, "transform not available on the GPU path");
    }
    return 0;
}

// kz_bwt_profile bits 8-19: the shape of the BWT inverse's walk (a profiling aid; 0 = the default of each field)
IbwtShape ibwt_shape(const kz_ctx* ctx) {
    IbwtShape sh;
    const uint32_t f = (uint32_t)ctx->bwt_profile;
    if (const uint32_t lg = (f >> 8) & 15) sh.stride = 1u << std::max(lg, 1u);
    if (const uint32_t st = (f >> 12) & 255) sh.stage = st * 16;
    return sh;
}
// One inverse stage, mirror of apply_forward. cap = capacity of a destination block; bs[b] = 0: TEXT takes cap as ctx["blockSize"].
int apply_inverse(kz_ctx* ctx, uint64_t t, const uint8_t* d_in, uint8_t* d_out, uint64_t stride, uint32_t cap, std::vector<uint32_t>& len,
                  const std::vector<uint8_t>& active, const std::vector<uint64_t>& bs) {
    const uint32_t nblocks = (uint32_t)len.size();
    const StageIo io{stride, stride, len, active, nullptr, nullptr};
    auto cap_all = [&](StageBlock& d, uint32_t) { d.cap = cap; };
    if (t == KZ_T_BWT) {
        std::vector<uint8_t> heads((size_t)nblocks * 64, 0);
        CK(cudaMemcpy2DAsync(heads.data(), 64, d_in, stride, 33, nblocks, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (uint32_t b0 = 0; b0 < nblocks;) {
            std::vector<uint64_t> so, dof;
            std::vector<uint32_t> ll, num;
            std::vector<uint8_t> hh;
            uint64_t total = 0;
            uint32_t max_len = 0;
            uint32_t b = b0;
            for (; b < nblocks; b++) {
                if (!active[b]) continue;
                if (!ll.empty() && (total + len[b] > bwt_inverse_batch_max_total() || ll.size() >= bwt_inverse_batch_max_blocks())) break;
                so.push_back(b * stride), dof.push_back(b * stride), ll.push_back(len[b]), num.push_back(b);
                hh.insert(hh.end(), heads.begin() + (size_t)b * 64, heads.begin() + (size_t)(b + 1) * 64);
                total += len[b];
                max_len = std::max(max_len, len[b]);
            }
            b0 = b;
            if (ll.empty()) continue;
            const IbwtShape shape = ibwt_shape(ctx);
            CK(ctx->d_ws.ensure(bwt_inverse_batch_workspace(total, (uint32_t)ll.size(), max_len, shape)));
            std::vector<uint32_t> produced(ll.size(), 0);
            LaunchScope ls(ctx, "bwt_inverse");
            CtxLzHook parts(ctx);  // kz_bwt_profile bit 0: the parts timed under their own names
            cudaError_t e = bwt_inverse_batch(d_in, d_out, so.data(), dof.data(), ll.data(), hh.data(), (uint32_t)ll.size(), cap, produced.data(),
                                              ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, ctx->stream, &ctx->launches, shape,
                                              (ctx->profile && (ctx->bwt_profile & 1)) ? &parts : nullptr);
            if (e == cudaErrorInvalidValue) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "BWT inverse transform failed: invalid header or data");
            if (e != cudaSuccess) return ctx->cuda_fail(e, "bwt_inverse");
            for (size_t k = 0; k < num.size(); k++) len[num[k]] = produced[k];
        }
    } else if (t == KZ_T_BWTS) {
        uint32_t max_len = 0;
        for (uint32_t b = 0; b < nblocks; b++) max_len = std::max(max_len, len[b]);
        CK(ctx->d_ws.ensure(bwts_inverse_workspace(max_len)));
        for (uint32_t b = 0; b < nblocks; b++) {
            if (!active[b] || len[b] == 0) continue;
            if (len[b] > cap) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "BWTS inverse transform failed: output buffer too small");
            LaunchScope ls(ctx, "bwts_inverse");
            cudaError_t e = bwts_inverse_device(d_in + b * stride, len[b], d_out + b * stride, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, ctx->stream, &ctx->launches);
            if (e != cudaSuccess) return ctx->cuda_fail(e, "bwts_inverse");
        }
    } else if (t == KZ_T_ROLZ) {
        const size_t sstride = rolz_scratch_bytes(cap);
        return run_desc_stage<RolzBlock>(
            ctx, io, "rolz_inverse", 0,
            [&](RolzBlock& d, uint32_t b) {
                d.scratch_off = b * sstride;
                d.cap = cap;
            },
            [&](uint32_t, uint32_t nb, uint32_t) { return sstride * nb + 256; },
            [&](uint32_t, const RolzBlock* db, const RolzBlock*, uint32_t nb, uint32_t, StageResult* res) {
                rolz_inverse_kernel<<<nb, 32, 0, ctx->stream>>>(d_in, db, (int)nb, ctx->d_ws.as<uint8_t>(), d_out, res);
                return cudaGetLastError();
            },
            "ROLZ codec inverse transform failed: invalid data");
    } else if (t == KZ_T_LZ || t == KZ_T_LZX) {
        std::vector<LzBlock> lb(nblocks);
        for (uint32_t b = 0; b < nblocks; b++) {
            lb[b].src_off = b * stride;
            lb[b].dst_off = b * stride;
            lb[b].scratch_off = 0;
            lb[b].len = active[b] ? len[b] : 0;
            lb[b].cap = cap;
            lb[b].data_type = 0;
            lb[b].pad = 0;
        }
        std::vector<uint32_t> hl(nblocks);
        std::vector<int32_t> hs(nblocks);
        {
            CtxLzWorkspace W(ctx);
            CtxLzHook H(ctx);
            cudaError_t e = lz_inverse_parallel(d_in, d_out, lb, W, ctx->stream, hl, hs, &H, &ctx->launches);
            if (e != cudaSuccess) return ctx->cuda_fail(e, "lz_inverse");
        }
        for (uint32_t b = 0; b < nblocks; b++) {
            if (!active[b] || len[b] == 0) continue;
            if (hs[b]) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "LZCodec inverse transform failed");
            len[b] = hl[b];
        }
    } else if (t == KZ_T_TEXT) {
        if (!text_available()) return ctx->fail(KZ_ERR_CREATE_CODEC, "TEXT: the library was built without the static dictionary");
        std::vector<uint64_t> sbs(bs);
        for (uint64_t& v : sbs) v = v ? v : cap;
        uint64_t serial = 0;
        const int rc = run_desc_stage<StageBlock>(
            ctx, io, "text_inverse", 64, cap_all, [&](uint32_t b0, uint32_t nb, uint32_t max_len) { return text_workspace_inverse(&sbs[b0], nb, max_len); },
            [&](uint32_t b0, const StageBlock* db, const StageBlock* hb, uint32_t nb, uint32_t, StageResult* res) {
                return text_inverse_batch(d_in, d_out, db, hb, nb, &sbs[b0], ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, res, ctx->stream, &ctx->launches,
                                          &serial);
            },
            "Text transform failed: invalid data");
        if (ctx->profile && serial) ctx->prof["text_inverse_serial"].launches += serial;
        return rc;
    } else if (t == KZ_T_UTF) {
        return run_desc_stage<StageBlock>(
            ctx, io, "utf_inverse", 32, cap_all, [](uint32_t, uint32_t nb, uint32_t) { return utf_workspace(nb); },
            [&](uint32_t, const StageBlock* db, const StageBlock*, uint32_t nb, uint32_t, StageResult* res) {
                return utf_inverse_batch(d_in, d_out, db, nb, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, res, ctx->stream, &ctx->launches);
            },
            "UTF inverse transform failed: invalid data");
    } else if (t == KZ_T_EXE) {
        return run_desc_stage<StageBlock>(
            ctx, io, "exe_inverse", 0, cap_all, [](uint32_t, uint32_t, uint32_t) { return (size_t)0; },
            [&](uint32_t, const StageBlock* db, const StageBlock*, uint32_t nb, uint32_t, StageResult* res) {
                exe_inverse_kernel<<<nb, 32, 0, ctx->stream>>>(d_in, db, (int)nb, d_out, res);
                return cudaGetLastError();
            },
            "ExeCodec inverse transform failed: invalid data");
    } else if (t == KZ_T_MM) {
        uint64_t total_len = 0;
        for (uint32_t b = 0; b < nblocks; b++) total_len += active[b] ? len[b] : 0;
        return run_desc_stage<StageBlock>(
            ctx, io, "fsd_inverse", 0, cap_all, [&](uint32_t, uint32_t nb, uint32_t) { return fsd_inverse_workspace(nb, total_len); },
            [&](uint32_t, const StageBlock*, const StageBlock* hb, uint32_t nb, uint32_t, StageResult* res) {
                return fsd_inverse_tiles(d_in, d_out, hb, nb, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, res, ctx->stream, &ctx->launches);
            },
            "FSD inverse transform failed: invalid data");
    } else if (t == KZ_T_PACK || t == KZ_T_DNA) {
        return run_desc_stage<StageBlock>(
            ctx, io, "alias_inverse", 256, cap_all, [&](uint32_t, uint32_t nb, uint32_t) { return alias_workspace(nb, cap); },
            [&](uint32_t, const StageBlock* db, const StageBlock*, uint32_t nb, uint32_t, StageResult* res) {
                return alias_inverse_batch(d_in, d_out, db, nb, cap, ctx->d_ws.as<uint8_t>(), ctx->d_ws.cap, res, ctx->stream, &ctx->launches);
            },
            "Alias codec inverse transform failed: invalid data");
    } else if (t == KZ_T_RANK || t == KZ_T_MTFT) {
        std::vector<SbrtBlock> sb(nblocks);
        for (uint32_t b = 0; b < nblocks; b++) {
            sb[b].src_off = b * stride;
            sb[b].dst_off = b * stride;
            sb[b].len = len[b];
            sb[b].seg_base = 0;
            sb[b].active = active[b] && len[b] > 0;
            sb[b].pad = 0;
            if (sb[b].active && len[b] > cap) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "SBRT inverse transform failed: output buffer too small");
        }
        Packer pk;
        const size_t o_sb = pk.add(sb.data(), sb.size() * sizeof(SbrtBlock));
        int rc = upload(ctx, pk);
        if (rc) return rc;
        {
            LaunchScope ls(ctx, "sbrt_inverse");
            uint32_t longest = 0;
            for (uint32_t b = 0; b < nblocks; b++) longest = std::max(longest, len[b]);
            sbrt_inverse_launch_len(d_in, (const SbrtBlock*)(ctx->d_tables.as<uint8_t>() + o_sb), (int)nblocks, t == KZ_T_MTFT ? 1 : 2, d_out, longest, ctx->stream);
        }
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(ctx->stream));
    } else if (t == KZ_T_ZRLT) {
        std::vector<ZrltBlock> zb(nblocks);
        for (uint32_t b = 0; b < nblocks; b++) {
            zb[b].src_off = b * stride;
            zb[b].dst_off = b * stride;
            zb[b].len = len[b];
            zb[b].cap = cap;
            zb[b].active = active[b] && len[b] > 0;
            zb[b].pad = 0;
        }
        Packer pk;
        const size_t o_zb = pk.add(zb.data(), zb.size() * sizeof(ZrltBlock));
        const size_t o_len = pk.reserve((size_t)nblocks * 4);
        const size_t o_st = pk.reserve((size_t)nblocks * 4);
        int rc = upload(ctx, pk);
        if (rc) return rc;
        uint8_t* T = ctx->d_tables.as<uint8_t>();
        CK(cudaMemsetAsync(d_out, 0, stride * nblocks, ctx->stream));  // runs of zeros are never written, only skipped
        {
            LaunchScope ls(ctx, "zrlt_inverse");
            zrlt_inverse_kernel<<<nblocks, 512, 0, ctx->stream>>>(d_in, (const ZrltBlock*)(T + o_zb), (int)nblocks, d_out, (uint32_t*)(T + o_len),
                                                                  (int32_t*)(T + o_st));
        }
        CK(cudaGetLastError());
        std::vector<uint32_t> hl(nblocks);
        std::vector<int32_t> hs(nblocks);
        CK(cudaMemcpyAsync(hl.data(), T + o_len, (size_t)nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(hs.data(), T + o_st, (size_t)nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (uint32_t b = 0; b < nblocks; b++) {
            if (!zb[b].active) continue;
            if (hs[b]) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "ZRLT inverse transform failed: output buffer is too small");
            len[b] = hl[b];
        }
    } else {
        return ctx->fail(KZ_ERR_INVALID_CODEC, "transform not available on the GPU path");
    }
    return 0;
}

// What encodingTask.encode (io/CompressedStream.go:753-816) finds out about the blocks of a batch before the transforms run. An empty
// vector stands for its default on every block.
struct BlockPrep {
    std::vector<int32_t> dt;         // the initial ctx["dataType"], from the block's magic number (default 0)
    std::vector<uint8_t> store;      // skipBlocks: 1 = the block is stored raw (default 0)
    std::vector<uint64_t> checksum;  // the hash of the original block (default: no checksums)
    // the entries of blocks idx[0 .. k - 1]
    BlockPrep pick(const uint32_t* idx, uint32_t k) const {
        BlockPrep p;
        auto take = [&](const auto& from, auto& to) {
            for (uint32_t j = 0; j < k && !from.empty(); j++) to.push_back(from[idx[j]]);
        };
        take(dt, p.dt);
        take(store, p.store);
        take(checksum, p.checksum);
        return p;
    }
};

// The BlockPrep of the blocks bl over d_base for a plan, the skipBlocks setting and a checksum width: their first four bytes (from
// host_heads, 4 zero-padded bytes per block, when the caller has them in host memory) decide the data types when the plan reads them
// (uses_magic) and, with skip, which blocks are stored; checksum_bits != 0 hashes the blocks.
int prepare_blocks(kz_ctx* ctx, const TransformPlan& plan, bool skip, uint32_t checksum_bits, const uint8_t* d_base, const BlockList& bl, BlockPrep& prep,
                   const std::vector<uint8_t>* host_heads = nullptr) {
    const uint32_t nb = bl.size();
    prep = BlockPrep();
    if (nb == 0) return 0;
    if (plan.uses_magic() || skip) {
        const uint8_t* d_flags = nullptr;
        if (skip) {
            int rc = skip_test(ctx, d_base, bl.off, bl.len, &d_flags);
            if (rc) return rc;
        }
        std::vector<uint8_t> heads = host_heads ? *host_heads : std::vector<uint8_t>(4 * (size_t)nb), flags(skip ? nb : 0);
        int rc = gather_heads(ctx, d_base, bl.off.data(), bl.len.data(), host_heads ? 0 : nb, 4, heads.data(), d_flags, flags.size(), flags.data());
        if (rc) return rc;
        if (plan.uses_magic()) {
            prep.dt.resize(nb);
            for (uint32_t b = 0; b < nb; b++) prep.dt[b] = magic_data_type(&heads[(size_t)b * 4], bl.len[b]);
        }
        if (skip) {
            const StoreCounts c = stored_blocks(heads.data(), flags.data(), bl.len.data(), nb, prep.store);
            if (ctx->profile) {  // bytes_in = blocks, bytes_out = bytes
                auto& m = ctx->prof["skip:magic"];
                m.bytes_in += c.magic_blocks, m.bytes_out += c.magic_bytes, m.launches++;
                auto& e = ctx->prof["skip:entropy"];
                e.bytes_in += c.entropy_blocks, e.bytes_out += c.entropy_bytes, e.launches++;
            }
        }
    }
    if (checksum_bits) return hash_blocks(ctx, d_base, bl.off, bl.len, checksum_bits, prep.checksum);
    return 0;
}

// Forward transform stage (ByteTransformSequence.Forward, transform/Sequence.go:64-125) of every block of a batch.
// Block b is d_src[b*stride : +len_b]. On return *d_data is the base of the post-transform data and jobs[] describes
// every block for the entropy stage. NONE leaves the data in place; the stages alternate between ctx->d_tmp and ctx->d_tmp2.
// A block that prep stores (skipBlocks) is a COPY block, like a block of at most SMALL_BLOCK bytes: no stage runs on it, and
// a batch of nothing but COPY blocks runs no stage at all. bs[b]: ctx["blockSize"] of block b's stream (apply_forward).
int forward_stage(kz_ctx* ctx, const TransformPlan& plan, const uint8_t* d_src, uint64_t stride, std::vector<uint32_t> len, const std::vector<uint64_t>& bs,
                  const BlockPrep& prep, const uint8_t** d_data, std::vector<EncJob>& jobs) {
    const uint32_t nblocks = (uint32_t)len.size();
    jobs.resize(nblocks);
    uint32_t max_len = 0;
    for (uint32_t b = 0; b < nblocks; b++) max_len = std::max(max_len, len[b]);
    *d_data = d_src;
    for (uint32_t b = 0; b < nblocks; b++) {
        EncJob& j = jobs[b];
        j.data_off = (uint64_t)b * stride;
        j.post_len = len[b];
        j.ntransforms = (uint32_t)plan.nt;
        j.skip_flags = 0x7F;  // NullTransform succeeds: bit 7 cleared (Sequence.go:65,107)
        j.copy = len[b] <= SMALL_BLOCK || (!prep.store.empty() && prep.store[b]);  // io/CompressedStream.go:773-799: transform and entropy forced to NONE
        j.checksum = prep.checksum.empty() ? 0 : prep.checksum[b];
    }
    if (plan.none() || nblocks == 0) return 0;
    // ctx["dataType"] of every block: the value from the block's magic number (encodingTask.encode :808-816), updated by the stages
    std::vector<int32_t> dts = prep.dt;
    dts.resize(nblocks, 0);
    std::vector<uint8_t> active(nblocks), applied;
    bool any = false;
    for (uint32_t b = 0; b < nblocks; b++) {
        active[b] = !jobs[b].copy && len[b] > 0;
        any = any || active[b];
    }
    if (!any) return 0;
    // room for the largest stage output: +33 bytes per BWT / SBRT stage, n/64 + 128 for LZ, n/16 for MM, headers of PACK
    const uint64_t gstride = ((uint64_t)max_len + max_len / 8 + 33ull * plan.nt + 8192 + 1024 + 256 + 15) & ~15ull;
    CK(ctx->d_tmp.ensure(gstride * nblocks + 64));
    if (plan.nt > 1) CK(ctx->d_tmp2.ensure(gstride * nblocks + 64));  // stage i writes to d_tmp (i even) or d_tmp2 (i odd)
    std::vector<uint8_t> flags(nblocks, 0xFF);
    const uint8_t* cur = d_src;
    uint64_t cur_stride = stride;
    for (int i = 0; i < plan.nt; i++) {
        uint8_t* outb = (i & 1) ? ctx->d_tmp2.as<uint8_t>() : ctx->d_tmp.as<uint8_t>();
        uint64_t bytes_in = 0, bytes_out = 0;
        for (uint32_t b = 0; b < nblocks; b++) bytes_in += active[b] ? len[b] : 0;
        int rc = apply_forward(ctx, plan.ids[i], cur, cur_stride, outb, gstride, len, active, applied, bs, &dts);
        if (rc) return rc;
        for (uint32_t b = 0; b < nblocks; b++) bytes_out += active[b] ? len[b] : 0;
        note_stage_bytes(ctx, "fwd", plan.ids[i], bytes_in, bytes_out);
        CopyList declined;
        for (uint32_t b = 0; b < nblocks; b++) {
            if (applied[b]) flags[b] &= (uint8_t)~(1u << (7 - i));
            else declined.add(cur + b * cur_stride, outb + b * gstride, len[b]);
        }
        rc = run_copies(ctx, declined);
        if (rc) return rc;
        cur = outb;
        cur_stride = gstride;
    }
    for (uint32_t b = 0; b < nblocks; b++) {
        EncJob& j = jobs[b];
        j.data_off = b * gstride;
        j.post_len = len[b];
        if (!j.copy) j.skip_flags = flags[b];
    }
    *d_data = cur;
    return 0;
}

// Transforms and entropy codes the blocks of a batch laid out in slots of one stride (block j: len[j] bytes at d_slots + j * stride). Block
// j's bit string goes to ctx->d_enc + j * *ostride (ostride: kz_max_block_output of the longest block, rounded to 16) and is bits[j] long.
// bs[j]: ctx["blockSize"] of block j's stream.
int encode_slots(kz_ctx* ctx, const TransformPlan& plan, uint32_t etype, uint32_t checksum_bits, const uint8_t* d_slots, uint64_t stride,
                 const std::vector<uint32_t>& len, const std::vector<uint64_t>& bs, const BlockPrep& prep, uint64_t* ostride, std::vector<uint64_t>& bits) {
    const uint32_t k = (uint32_t)len.size();
    const uint8_t* d_data = nullptr;
    std::vector<EncJob> jobs;
    int rc = forward_stage(ctx, plan, d_slots, stride, len, bs, prep, &d_data, jobs);
    if (rc) return rc;
    *ostride = round16(kz_max_block_output(*std::max_element(len.begin(), len.end())));
    CK(ctx->d_enc.ensure(*ostride * k + 64));
    std::vector<uint64_t> base(k);
    for (uint32_t j = 0; j < k; j++) base[j] = 8 * (uint64_t)j * *ostride;
    EncResult res;
    rc = encode_batch(ctx, LAYOUT_BLOCKS, etype, checksum_bits, d_data, jobs, {}, 0, false, false, ctx->d_enc.as<uint8_t>(), *ostride * k, base, res);
    if (rc) return rc;
    bits = res.blk_bits;
    return 0;
}

// Grows b to hold `need` bytes, keeping its first `used` bytes (DevBuf::ensure drops them).
int grow_keeping(kz_ctx* ctx, DevBuf& b, uint64_t used, uint64_t need) {
    if (need + 64 + 256 <= b.cap) return 0;
    DevBuf nb;
    CK(nb.ensure(std::max<size_t>(need + 64, 2 * b.cap)));
    if (used) CK(cudaMemcpyAsync(nb.p, b.p, used, cudaMemcpyDeviceToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    b.release();
    b = nb;
    return 0;
}

// The bit strings of blocks encoded pass by pass, kept for one assembly behind the last pass: record r is bits[r] bits at offset[r] of
// ctx->d_bits, each record at a 16-byte aligned offset; `used` bytes are taken.
struct RecordArena {
    std::vector<uint64_t> bits, offset;
    uint64_t used = 0;
    explicit RecordArena(size_t n) : bits(n), offset(n) {}
    const uint8_t* record(kz_ctx* ctx, size_t r) const { return ctx->d_bits.as<uint8_t>() + offset[r]; }

    // encode_slots over the k blocks of one pass, then block j's bit string packed behind the arena's records as record rec[j]
    int encode_pass(kz_ctx* ctx, const TransformPlan& plan, uint32_t etype, uint32_t checksum_bits, const uint8_t* d_slots, uint64_t stride,
                    const std::vector<uint32_t>& len, const std::vector<uint64_t>& bs, const BlockPrep& prep, const uint32_t* rec) {
        const uint32_t k = (uint32_t)len.size();
        uint64_t ostride = 0;
        std::vector<uint64_t> b;
        int rc = encode_slots(ctx, plan, etype, checksum_bits, d_slots, stride, len, bs, prep, &ostride, b);
        if (rc) return rc;
        uint64_t need = used;
        for (uint32_t j = 0; j < k; j++) need += round16((b[j] + 7) / 8);
        rc = grow_keeping(ctx, ctx->d_bits, used, need);  // the records of the earlier passes stay
        if (rc) return rc;
        CopyList pack;
        for (uint32_t j = 0; j < k; j++) {
            bits[rec[j]] = b[j];
            offset[rec[j]] = used;
            pack.add(ctx->d_enc.as<uint8_t>() + j * ostride, ctx->d_bits.as<uint8_t>() + used, (b[j] + 7) / 8);
            used += round16((b[j] + 7) / 8);
        }
        return run_copies(ctx, pack);
    }
};

// Inverse transform stage (ByteTransformSequence.Inverse, transform/Sequence.go:131-186) of every block of a batch. The entropy
// stage left block b's pre_len bytes at d_pre + b*pstride, a scratch buffer of this context with room for pstride - 64 bytes per
// block; the stages alternate between it and ctx->d_tmp2. out_len[b] = decoded length of block b. Once the lengths are known,
// place(b, len) is called for every block in order and gives its offset in d_dst, or NO_ROOM: the block is not copied. The placed
// blocks are then copied by one batch_copy_kernel launch.
const uint64_t NO_ROOM = ~0ull;
template <class Place>
int inverse_stage(kz_ctx* ctx, const TransformPlan& plan, std::vector<DecJob>& jobs, uint8_t* d_pre, uint64_t pstride, uint8_t* d_dst, Place&& place,
                  std::vector<uint32_t>& out_len) {
    const uint32_t nblocks = (uint32_t)jobs.size();
    out_len.assign(nblocks, 0);
    if (nblocks == 0) return 0;
    const uint32_t blk_cap = (uint32_t)std::min<uint64_t>(pstride - 64, 0xFFFFFFF0u);
    std::vector<uint32_t> len(nblocks);
    std::vector<uint64_t> bs(nblocks);
    for (uint32_t b = 0; b < nblocks; b++) len[b] = jobs[b].pre_len, bs[b] = jobs[b].block_size;
    CK(ctx->d_tmp2.ensure(pstride * nblocks + 64));
    uint8_t* cur = d_pre;
    uint8_t* other = ctx->d_tmp2.as<uint8_t>();
    if (other == cur) return ctx->fail(KZ_ERR_UNKNOWN, "internal: scratch buffers alias");
    std::vector<uint8_t> active(nblocks);
    for (int i = plan.nt - 1; i >= 0; i--) {
        bool any = false;
        for (uint32_t b = 0; b < nblocks; b++) {
            active[b] = !jobs[b].copy && !(jobs[b].skip_flags & (1u << (7 - i))) && len[b] > 0;
            any = any || active[b];
        }
        if (!any) continue;
        uint64_t bytes_in = 0, bytes_out = 0;
        for (uint32_t b = 0; b < nblocks; b++) bytes_in += active[b] ? len[b] : 0;
        int rc = apply_inverse(ctx, plan.ids[i], cur, other, pstride, blk_cap, len, active, bs);
        if (rc) return rc;
        for (uint32_t b = 0; b < nblocks; b++) bytes_out += active[b] ? len[b] : 0;
        note_stage_bytes(ctx, "inv", plan.ids[i], bytes_in, bytes_out);
        CopyList skipped;
        for (uint32_t b = 0; b < nblocks; b++)
            if (!active[b]) skipped.add(cur + b * pstride, other + b * pstride, len[b]);
        rc = run_copies(ctx, skipped);
        if (rc) return rc;
        std::swap(cur, other);
    }
    CopyList out;
    for (uint32_t b = 0; b < nblocks; b++) {
        const uint64_t at = place(b, len[b]);
        if (at != NO_ROOM) out.add(cur + b * pstride, d_dst + at, len[b]);
        out_len[b] = len[b];
    }
    int rc = run_copies(ctx, out);
    if (rc) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// Destinations of blocks decoded back to back into an output buffer of cap bytes: decode_walked's place() for one stream.
struct BackToBack {
    uint64_t cap, off = 0;
    uint64_t operator()(uint32_t, uint32_t len) {
        if (off + len > cap) return NO_ROOM;
        off += len;
        return off - len;
    }
};

// The block stages of walked records of one stream header: jobs (bit_off / bits set) are the blocks, in order; block b belongs to stream
// owner[b], and last[b] says it is (or may be) its stream's last record, which exempts it from NONE's rule that a block is a multiple of
// 16 long. place(b, len) gives block b's offset in d_dst, or NO_ROOM. fail[o] is the failure held for stream o: a block failure is noted
// there (DecodeFailure: earliest stage, then earliest block), and the blocks of o skip every stage whose failure could not beat it. In
// this order, as decompress_device_impl always checked them:
//   1. headers: per block, its header status, then for NONE its place and the multiple-of-16 rule;
//   2. entropy decode: NONE straight to the placed destination, other plans into ctx->d_tmp slots of decode_stride;
//   3. inverse transforms into their place (KZ_ERR_WRITE_FILE when there is no room);
//   4. checksums of the bytes where they landed.
// A failing decode_batch or inverse_stage cannot name the block: its failure goes to every stream of the batch at that stage. The return
// value is kept for call-level errors (CUDA, allocation, a bad hash launch).
template <class Place>
int decode_walked(kz_ctx* ctx, const StreamHeader& sh, const TransformPlan& plan, const uint32_t* d_words, uint64_t words_len, std::vector<DecJob>& jobs,
                  const std::vector<uint32_t>& owner, const std::vector<uint8_t>& last, Place&& place, uint8_t* d_dst, DecodeFailure* fail) {
    const uint32_t nb = (uint32_t)jobs.size();
    std::vector<uint32_t> idx;  // the blocks of the stage in progress
    std::vector<DecJob> run;
    auto stage = [&](int s) {   // the blocks whose stream can still fail at stage s
        idx.clear();
        run.clear();
        for (uint32_t b = 0; b < nb; b++)
            if (fail[owner[b]].runs(s)) idx.push_back(b), run.push_back(jobs[b]);
        return !run.empty();
    };
    auto done = [&]() {
        for (size_t i = 0; i < idx.size(); i++) jobs[idx[i]] = run[i];
    };
    auto note_all = [&](int s, int rc) {
        for (uint32_t b : idx) fail[owner[b]].note(s, rc, ctx->err);
    };
    if (!stage(STAGE_HEADER)) return 0;
    int rc = decode_parse_headers(ctx, d_words, run, sh.checksum_bits);
    if (rc) return rc;
    done();
    for (uint32_t b = 0; b < nb; b++) {
        DecodeFailure& f = fail[owner[b]];
        DecJob& j = jobs[b];
        if (!f.runs(STAGE_HEADER)) continue;
        if (j.status) {
            f.note(STAGE_HEADER, j.status, "Invalid compressed block header");
        } else if (plan.none()) {  // NONE: the decoded length is pre_len
            j.out_off = place(b, j.pre_len);
            if (j.out_off == NO_ROOM) f.note(STAGE_HEADER, -KZ_ERR_WRITE_FILE, "output buffer too small");
            else if (!last[b] && (j.pre_len & 15)) f.note(STAGE_HEADER, -KZ_ERR_PROCESS_BLOCK, "unexpected block length");
        }
    }
    if (!stage(STAGE_DECODE)) return 0;
    uint64_t stride = 0;
    if (!plan.none()) {
        for (const DecJob& j : run) stride = std::max(stride, decode_stride(j.block_size, j.pre_len));
        CK(ctx->d_tmp.ensure(stride * run.size() + 64));
        for (size_t i = 0; i < run.size(); i++) run[i].out_off = i * stride;
    }
    rc = decode_batch(ctx, sh.etype, d_words, words_len, run, plan.none() ? d_dst : ctx->d_tmp.as<uint8_t>());
    if (rc) note_all(STAGE_DECODE, rc);
    done();
    for (uint32_t b : idx)
        if (jobs[b].status) fail[owner[b]].note(STAGE_DECODE, jobs[b].status, "Invalid bitstream: block decoding failed");
    if (!stage(STAGE_INVERSE)) return 0;
    std::vector<uint64_t> at(nb, NO_ROOM);
    std::vector<uint32_t> len(nb, 0);
    if (plan.none()) {
        for (uint32_t b : idx) at[b] = jobs[b].out_off, len[b] = jobs[b].pre_len;
    } else {
        std::vector<uint32_t> olen;
        auto put = [&](uint32_t i, uint32_t n) {
            const uint32_t b = idx[i];
            DecodeFailure& f = fail[owner[b]];
            if (!f.runs(STAGE_INVERSE)) return NO_ROOM;  // an earlier block of the stream had no room
            at[b] = place(b, n);
            if (at[b] == NO_ROOM) f.note(STAGE_INVERSE, -KZ_ERR_WRITE_FILE, "output buffer too small");
            return at[b];
        };
        rc = inverse_stage(ctx, plan, run, ctx->d_tmp.as<uint8_t>(), stride, d_dst, put, olen);
        if (rc) note_all(STAGE_INVERSE, rc);
        for (size_t i = 0; i < olen.size(); i++) len[idx[i]] = olen[i];
    }
    if (!sh.checksum_bits || !stage(STAGE_CHECKSUM)) return 0;
    std::vector<uint64_t> hoff, hv;
    std::vector<uint32_t> hlen;
    for (uint32_t b : idx) hoff.push_back(at[b]), hlen.push_back(len[b]);
    rc = hash_blocks(ctx, d_dst, hoff, hlen, sh.checksum_bits, hv);
    if (rc) return rc;
    for (size_t i = 0; i < idx.size(); i++) {
        const uint64_t want = sh.checksum_bits == 32 ? (run[i].checksum & 0xFFFFFFFFull) : run[i].checksum;
        if (hv[i] != want) fail[owner[idx[i]]].note(STAGE_CHECKSUM, -KZ_ERR_CRC_CHECK, CHECKSUM_MISMATCH);
    }
    return 0;
}

// The block stages of block records of one header, each block on its own: decode_walked with one DecodeFailure per block, then every
// failed block of a batch of several is decoded again alone, so that fail[i] is what decoding block i alone gives. A failing stage call
// cannot name its block, and one block's failure may hide a later one's; only corrupt input pays. A block that place refused is not
// decoded again. jobs (bit_off / bits set), last and place are decode_walked's; len[i] is the decoded length place was last given for
// block i (0 when it never was).
template <class Place>
int decode_isolated(kz_ctx* ctx, const StreamHeader& sh, const TransformPlan& plan, const uint32_t* d_words, uint64_t words_len, const std::vector<DecJob>& jobs,
                    const std::vector<uint8_t>& last, Place&& place, uint8_t* d_dst, std::vector<DecodeFailure>& fail, std::vector<uint32_t>& len) {
    const uint32_t nb = (uint32_t)jobs.size();
    fail.assign(nb, DecodeFailure());
    len.assign(nb, 0);
    std::vector<uint8_t> refused(nb, 0);
    auto decode = [&](const std::vector<uint32_t>& ids) {
        std::vector<DecJob> run;
        std::vector<uint32_t> owner;
        std::vector<uint8_t> run_last;
        for (uint32_t b : ids) run.push_back(jobs[b]), owner.push_back((uint32_t)owner.size()), run_last.push_back(last[b]);
        std::vector<DecodeFailure> f(ids.size());
        auto put = [&](uint32_t i, uint32_t n) {
            const uint32_t b = ids[i];
            const uint64_t at = place(b, n);
            len[b] = n;
            refused[b] = at == NO_ROOM;
            return at;
        };
        int rc = decode_walked(ctx, sh, plan, d_words, words_len, run, owner, run_last, put, d_dst, f.data());
        for (size_t i = 0; i < ids.size(); i++) fail[ids[i]] = f[i];
        return rc;
    };
    std::vector<uint32_t> all(nb);
    std::iota(all.begin(), all.end(), 0u);
    int rc = decode(all);
    if (rc || nb == 1) return rc;
    for (uint32_t b = 0; b < nb && !rc; b++)
        if (fail[b].failed() && !refused[b]) rc = decode({b});
    return rc;
}


}  // namespace

// ------------------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------------------
extern "C" {

int kz_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int kz_init(int device, kz_ctx** out) {
    if (!out) return -KZ_ERR_INVALID_PARAM;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return -KZ_ERR_CREATE_COMPRESSOR;
    if (cudaSetDevice(device) != cudaSuccess) return -KZ_ERR_CREATE_COMPRESSOR;
    kz_ctx* ctx = new kz_ctx();
    ctx->device = device;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete ctx;
        return -KZ_ERR_CREATE_COMPRESSOR;
    }
    if (cudaEventCreateWithFlags(&ctx->caller_done, cudaEventDisableTiming) != cudaSuccess) {
        cudaStreamDestroy(ctx->stream);
        delete ctx;
        return -KZ_ERR_CREATE_COMPRESSOR;
    }
    cudaFuncSetAttribute(ans0_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ENC_SMEM);
    cudaFuncSetAttribute(ans0_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DEC_SMEM);
    cudaFuncSetAttribute(huf_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HUF_DEC_SMEM);
    *out = ctx;
    return 0;
}

void kz_destroy(kz_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->session) close_session(ctx->session);
    cudaStreamSynchronize(ctx->stream);
    for (kz_cache* c : ctx->caches) {  // caches not freed before: their handles stay valid for kz_cache_free
        cudaFree(c->d_pages);
        c->d_pages = nullptr;
        c->ctx = nullptr;
    }
    drain_profile(ctx);
    for (auto e : ctx->event_pool) cudaEventDestroy(e);
    ctx->each_dev_buf([](DevBuf& b) { b.release(); });
    ctx->h_stage.release();
    ctx->h_dl.release();
    ctx->h_io.release();
    cudaEventDestroy(ctx->caller_done);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* kz_last_error(kz_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

void* kz_alloc_pinned(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
    return p;
}
void kz_free_pinned(void* p) {
    if (p) cudaFreeHost(p);
}

void* kz_cuda_stream(kz_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

uint64_t kz_launch_count(kz_ctx* ctx, int reset) {
    uint64_t v = ctx->launches;
    if (reset) ctx->launches = 0;
    return v;
}

void kz_profile(kz_ctx* ctx, int enable) {
    drain_profile(ctx);
    ctx->profile = enable != 0;
}
uint32_t kz_kernel_time(kz_ctx* ctx, const char* name, double* total_ms) {
    drain_profile(ctx);
    auto it = ctx->prof.find(name);
    if (it == ctx->prof.end()) {
        if (total_ms) *total_ms = 0;
        return 0;
    }
    if (total_ms) *total_ms = it->second.ms;
    return it->second.launches;
}
void kz_bwt_profile(kz_ctx* ctx, int flags) {
    if (ctx) ctx->bwt_profile = flags;
}
void kz_profile_reset(kz_ctx* ctx) {
    drain_profile(ctx);
    ctx->prof.clear();
}
size_t kz_profile_names(kz_ctx* ctx, char* buf, size_t cap) {
    drain_profile(ctx);
    std::string all;
    for (auto& kv : ctx->prof) all += kv.first + "\n";
    if (buf && cap) {
        const size_t k = std::min(cap - 1, all.size());
        memcpy(buf, all.data(), k);
        buf[k] = 0;
    }
    return all.size() + 1;
}
uint32_t kz_stage_bytes(kz_ctx* ctx, const char* name, uint64_t* bytes_in, uint64_t* bytes_out) {
    auto it = ctx->prof.find(name);
    if (bytes_in) *bytes_in = it == ctx->prof.end() ? 0 : it->second.bytes_in;
    if (bytes_out) *bytes_out = it == ctx->prof.end() ? 0 : it->second.bytes_out;
    return it == ctx->prof.end() ? 0 : it->second.launches;
}

// worst cases: ANS0/Huffman ~440/550 header bytes per 16 KiB chunk; ANS1 256 context tables (<= 104 KiB) per 4 MiB chunk
size_t kz_max_block_output(size_t n) { return n + (n >> 3) + 1024 + 64 * (n / 16384 + 1) + 106496 * (n / (4u << 20) + 1); }
size_t kz_max_stream_output(size_t n, uint32_t block_size) {
    size_t nblocks = block_size ? (n + block_size - 1) / block_size : 1;
    return n + (n >> 3) + 64 * (n / 16384 + 1) + 32 * nblocks + 1024 + 106496 * (n / (4u << 20) + nblocks + 1);
}

int kz_set_block_range(kz_ctx* ctx, int64_t from_block, int64_t to_block) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    ctx->range_from = from_block < 0 ? -1 : from_block;
    ctx->range_to = to_block < 0 ? -1 : to_block;
    return 0;
}

int kz_set_skip_blocks(kz_ctx* ctx, int on) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    ctx->skip_blocks = on != 0;
    return 0;
}
int kz_set_headerless_writer(kz_ctx* ctx, int on) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    ctx->headerless_writer = on != 0;
    return 0;
}

// Reader.validateHeaderless (io/CompressedStream.go:1178-1280) over ids instead of names: entropy.GetType and transform.GetType accept the
// names of entropy ids 0..9 but PAQ (3) and of transform ids 0..19 but SNAPPY (4) (EntropyCodecFactory.go:170-206, Factory.go:330-395).
int kz_set_headerless_reader(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, int64_t output_size,
                             uint32_t bs_version) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    if (bs_version > BS_VERSION) return ctx->fail(KZ_ERR_INVALID_PARAM, "Invalid bitstream version, cannot read this version of the stream");
    if (bs_version < BS_VERSION) return ctx->fail(KZ_ERR_STREAM_VERSION, "Only bitstream version 6 is supported");
    if (etype > 9 || etype == 3) return ctx->fail(KZ_ERR_INVALID_PARAM, "Unsupported entropy codec type");
    if (t48 >> 48) return ctx->fail(KZ_ERR_INVALID_PARAM, "Unknown transform type");
    for (int i = 0; i < 8; i++) {
        const uint64_t t = (t48 >> (42 - 6 * i)) & 63;
        if (t > 19 || t == 4) return ctx->fail(KZ_ERR_INVALID_PARAM, "Unknown transform type");
    }
    if (block_size < 1024 || block_size > (1u << 30)) return ctx->fail(KZ_ERR_INVALID_PARAM, "Invalid block size");
    if (checksum_bits != 0 && checksum_bits != 32 && checksum_bits != 64)
        return ctx->fail(KZ_ERR_INVALID_PARAM, "The block checksum size must be 32 or 64 bits");
    if (!etype_supported(etype)) return ctx->fail(KZ_ERR_CREATE_CODEC, "entropy codec not available on the GPU path");
    TransformPlan plan;
    int rc = plan_transforms(ctx, t48, etype, plan, KZ_ERR_CREATE_CODEC);
    if (rc) return rc;
    kz_ctx::Headerless& h = ctx->headerless_reader;
    h.on = true;
    h.t48 = t48;
    h.etype = etype;
    h.block_size = block_size;
    h.checksum_bits = checksum_bits;
    h.output_size = output_size < 0 || output_size >= ((int64_t)1 << 48) ? 0 : output_size;  // :1264-1268
    return 0;
}

int kz_clear_headerless_reader(kz_ctx* ctx) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    ctx->headerless_reader = kz_ctx::Headerless();
    return 0;
}

void kz_set_stream_block_size(kz_ctx* ctx, uint64_t block_size) {
    if (ctx) ctx->user_stream_bs = block_size;
}

size_t kz_transform_max_encoded_len(uint64_t type, size_t n) {
    switch (type) {
        case KZ_T_NONE: return n;
        case KZ_T_BWT: return n + 33;  // transform/BWTBlockCodec.go:228
        case KZ_T_RANK:
        case KZ_T_MTFT: return n + 33;  // transform/SBRT.go:229-231
        case KZ_T_ZRLT: return n;       // transform/ZRLT.go:228-230
        case KZ_T_BWTS: return n;       // transform/BWTS.go:291-293
        case KZ_T_ROLZ: return n <= 512 ? n + 64 : n;  // transform/ROLZCodec.go:916-918
        case KZ_T_PACK: case KZ_T_DNA: return n + 1024;  // transform/AliasCodec.go:437-439
        case KZ_T_MM: return n + std::max<size_t>(n >> 4, 64);  // transform/FSDCodec.go:128-130
        case KZ_T_TEXT: return n;  // transform/TextCodec.go:1720-1724
        case KZ_T_UTF: return n + 8192;  // transform/UTFCodec.go:386-388
        case KZ_T_EXE: return n <= 256 ? n + 32 : n + n / 8;  // transform/EXECodec.go:701-708
        case KZ_T_LZ:
        case KZ_T_LZX: return n <= 1024 ? n + 16 : n + n / 64;  // transform/LZCodec.go:935-941
        default: return 0;
    }
}

// ---- whole stream, device resident ---------------------------------------------------------------------------
// What compress_device_impl runs on the n bytes at d_src, cut into blocks of block_size: prepare_blocks, the forward transforms and the
// LAYOUT_STREAM encode behind the leading segment `lead` (lead_bits bits: the stream header, or a writer session's carry), with the end
// marker unless `fragment`. A writer session runs every batch of its stream through it, its leading segment volatile.
static int encode_stream_blocks(kz_ctx* ctx, const TransformPlan& plan, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, bool skip,
                                const void* d_src, size_t n, const std::vector<uint8_t>& lead, uint32_t lead_bits, bool fragment, bool volatile_lead,
                                void* d_dst, size_t cap, EncResult& res) {
    const uint64_t off = 0, len = n;
    const BlockList bl = cut_blocks(&off, &len, 1, block_size);
    BlockPrep prep;
    int rc = prepare_blocks(ctx, plan, skip, checksum_bits, (const uint8_t*)d_src, bl, prep);
    if (rc) return rc;
    const uint8_t* d_data = nullptr;
    std::vector<EncJob> jobs;
    rc = forward_stage(ctx, plan, (const uint8_t*)d_src, block_size, bl.len, std::vector<uint64_t>(bl.size(), block_size), prep, &d_data, jobs);
    if (rc) return rc;
    return encode_batch(ctx, LAYOUT_STREAM, etype, checksum_bits, d_data, jobs, lead, lead_bits, fragment, volatile_lead, (uint8_t*)d_dst, cap, {}, res);
}

static int compress_device_impl(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, int64_t input_size, const void* d_src,
                                size_t n, void* d_dst, size_t cap, size_t* out_n, bool fragment, uint64_t* out_bits) {
    if (!ctx || !out_n) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    int rc = check_encode_args(ctx, block_size, checksum_bits);
    if (rc) return rc;
    if (((uintptr_t)d_src & 15) || ((uintptr_t)d_dst & 15)) return ctx->fail(KZ_ERR_INVALID_PARAM, "device buffers must be 16-byte aligned");
    TransformPlan plan;
    rc = plan_transforms(ctx, t48, etype, plan, KZ_ERR_CREATE_CODEC);
    if (rc) return rc;
    std::vector<uint8_t> hdr;
    uint32_t hdr_bits = build_stream_header(hdr, t48, etype, block_size, checksum_bits, input_size);
    if (fragment || ctx->headerless_writer) hdr_bits = 0;  // an empty leading segment (Writer.writeHeader :430)
    EncResult res;
    rc = encode_stream_blocks(ctx, plan, etype, block_size, checksum_bits, ctx->skip_blocks, d_src, n, hdr, hdr_bits, fragment, false, d_dst, cap, res);
    if (rc) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    *out_n = (size_t)((res.total_bits + 7) / 8);
    if (out_bits) *out_bits = res.total_bits;
    return 0;
}

// The device variants read and write buffers that the caller filled or allocated with work of its own, typically PyTorch's on the legacy
// default stream. The context's stream is non-blocking and would not wait for that work: each device variant first orders it after
// everything already queued on the legacy default stream (which itself follows every blocking stream), on the device, without a host wait.
static int after_caller_work(kz_ctx* ctx) {
    if (!ctx) return 0;  // the entry point's own argument check reports it
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventRecord(ctx->caller_done, cudaStreamLegacy));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->caller_done, 0));
    return 0;
}

int kz_compress_stream_device(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, int64_t input_size,
                              const void* d_src, size_t n, void* d_dst, size_t cap, size_t* out_n) {
    if (int rc = after_caller_work(ctx)) return rc;
    return compress_device_impl(ctx, t48, etype, block_size, checksum_bits, input_size, d_src, n, d_dst, cap, out_n, false, nullptr);
}
// The block records (5 b | lw b | payload each) of n bytes at d_src, without stream header and without end marker: what one rank of a sharded
// compression contributes (blocks are independent, io/CompressedStream.go:896-898). *out_bits = exact bit length.
int kz_compress_fragment_device(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, const void* d_src, size_t n, void* d_dst,
                                size_t cap, uint64_t* out_bits) {
    if (int rc = after_caller_work(ctx)) return rc;
    size_t bytes = 0;
    if (!out_bits) return -KZ_ERR_INVALID_PARAM;
    return compress_device_impl(ctx, t48, etype, block_size, checksum_bits, 0, d_src, n, d_dst, cap, &bytes, true, out_bits);
}

// Stream header bytes (Writer.writeHeader, io/CompressedStream.go:429-519) for the rank that commits a sharded stream. out: >= 32 bytes.
int kz_stream_header(uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, int64_t input_size, uint8_t* out, uint32_t* out_bits) {
    if (!out || !out_bits) return -KZ_ERR_INVALID_PARAM;
    std::vector<uint8_t> hdr;
    *out_bits = build_stream_header(hdr, t48, etype, block_size, checksum_bits, input_size);
    memset(out, 0, 32);
    memcpy(out, hdr.data(), std::min<size_t>(hdr.size(), 32));
    return 0;
}

// Bit-granular concatenation of nseg device bit strings (MSB first) into d_dst: the ordered commit of Writer.processBlock (:951-976) for
// fragments gathered from other ranks. Segments are cut into 64 KiB pieces, one CTA each. *total_bits = length of the result.
int kz_concat_bits_device(kz_ctx* ctx, uint32_t nseg, const void* const* d_seg, const uint64_t* seg_bits, void* d_dst, size_t cap, uint64_t* total_bits) {
    if (int rc = after_caller_work(ctx)) return rc;
    if (!ctx || !total_bits || (nseg && (!d_seg || !seg_bits)) || !d_dst) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    SegmentList sl;
    for (uint32_t i = 0; i < nseg; i++) {
        if (((uintptr_t)d_seg[i] & 3) != 0) return ctx->fail(KZ_ERR_INVALID_PARAM, "segments must be 4-byte aligned");
        sl.add_device((const uint8_t*)d_seg[i], 0, seg_bits[i]);
    }
    *total_bits = sl.next;
    if ((sl.next + 7) / 8 + 8 > cap) return ctx->fail(KZ_ERR_WRITE_FILE, "output buffer too small");
    return sl.write(ctx, (uint8_t*)d_dst);
}

// A stream's blocks decoded to d_dst (cap bytes). given: the header fields (as sharded decompression gets them from rank 0) and the first
// record at start_bit, stop_after records (0: up to the end marker); else the stream's header or the headerless reader setting.
static int decompress_device_impl(kz_ctx* ctx, const StreamHeader* given, uint64_t start_bit, uint32_t stop_after, int64_t from, int64_t to, const void* d_src,
                                  size_t n, void* d_dst, size_t cap, size_t* out_n) {
    if (!ctx || !out_n) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    if (((uintptr_t)d_src & 15) || ((uintptr_t)d_dst & 15)) return ctx->fail(KZ_ERR_INVALID_PARAM, "device buffers must be 16-byte aligned");
    StreamHeader sh;
    int rc = 0;
    if (given) {
        sh = *given;
        sh.bits = start_bit;
    } else {  // the stream's header, or the headerless reader setting (a headerless stream has no header to read)
        uint8_t head[64];
        const uint64_t off = 0, len = ctx->headerless_reader.on ? 0 : n;
        rc = gather_heads(ctx, (const uint8_t*)d_src, &off, &len, 1, 64, head);
        if (rc == 0) rc = stream_header(ctx, head, n, sh);
        if (rc) return rc;
    }
    TransformPlan plan;
    rc = plan_transforms(ctx, sh.t48, sh.etype, plan, KZ_ERR_INVALID_CODEC);
    if (rc) return rc;
    const uint32_t* d_words = (const uint32_t*)d_src;
    // at most cap / 1024 + 16 decoded blocks are stored (blocks are at least 1 KiB)
    std::vector<WalkJob> wj{WalkJob{sh.bits, 8ull * n, 0, (uint32_t)std::min<uint64_t>((uint64_t)cap / 1024 + 16, 1u << 22), stop_after}};
    std::vector<Walked> w;
    rc = walk_streams(ctx, d_words, wj, from, to, w);
    if (rc) return rc;
    if (w[0].status) return ctx->fail(-w[0].status, "Invalid bitstream: corrupted block length");
    if (w[0].overflow) return ctx->fail(KZ_ERR_BLOCK_SIZE, "Invalid bitstream: more blocks than the output buffer can hold");
    std::vector<DecJob> jobs;
    std::vector<uint32_t> owner;
    std::vector<uint8_t> last;
    w[0].append(0, sh.block_size, jobs, owner, last);
    BackToBack place{cap};
    DecodeFailure f;
    rc = decode_walked(ctx, sh, plan, d_words, (n + 3) / 4 + 16, jobs, owner, last, place, (uint8_t*)d_dst, &f);  // >= 64 readable bytes past n
    if (rc) return rc;
    if (f.failed()) return ctx->fail(-f.code, f.msg);
    *out_n = (size_t)place.off;
    return 0;
}

int kz_decompress_stream_device(kz_ctx* ctx, const void* d_src, size_t n, void* d_dst, size_t cap, size_t* out_n) {
    if (int rc = after_caller_work(ctx)) return rc;
    return decompress_device_impl(ctx, nullptr, 0, 0, ctx ? ctx->range_from : -1, ctx ? ctx->range_to : -1, d_src, n, d_dst, cap, out_n);
}
// Decodes `nblocks` block records that start at bit `start_bit` of the fragment at d_src (frag_bytes bytes, >= 64 readable bytes behind them):
// what one rank of a sharded decompression does with its part of the stream. The stream parameters come from the header rank 0 parsed.
int kz_decompress_fragment_device(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, const void* d_src, size_t frag_bytes,
                                  uint64_t start_bit, uint32_t nblocks, void* d_dst, size_t cap, size_t* out_n) {
    if (int rc = after_caller_work(ctx)) return rc;
    if (!ctx || !out_n) return -KZ_ERR_INVALID_PARAM;
    *out_n = 0;
    if (nblocks == 0) return 0;
    StreamHeader sh;
    sh.t48 = t48;
    sh.etype = etype;
    sh.block_size = block_size;
    sh.checksum_bits = checksum_bits;
    sh.input_size = 0;
    sh.bits = 0;
    return decompress_device_impl(ctx, &sh, start_bit, nblocks, -1, -1, d_src, frag_bytes, d_dst, cap, out_n);
}
// Parses the header of the stream at d_src and walks its block records: rec_bit[b] = first bit of record b (its 5-bit prefix), rec_bit[nblocks] =
// first bit behind the last record (the end marker). rec_bit must hold max_blocks + 1 entries. With a headerless reader setting the fields are
// the setting's and rec_bit[0] = 0.
int kz_stream_index_device(kz_ctx* ctx, const void* d_src, size_t n, uint32_t max_blocks, uint64_t* t48, uint32_t* etype, uint32_t* block_size,
                           uint32_t* checksum_bits, int64_t* input_size, uint64_t* rec_bit, uint32_t* nblocks) {
    if (int rc = after_caller_work(ctx)) return rc;
    if (!ctx || !d_src || !rec_bit || !nblocks) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    StreamHeader sh;
    uint8_t head[64];
    const uint64_t off = 0, len = n;
    int rc = gather_heads(ctx, (const uint8_t*)d_src, &off, &len, 1, 64, head);
    if (rc == 0) rc = stream_header(ctx, head, n, sh);
    if (rc) return rc;
    if (t48) *t48 = sh.t48;
    if (etype) *etype = sh.etype;
    if (block_size) *block_size = sh.block_size;
    if (checksum_bits) *checksum_bits = sh.checksum_bits;
    if (input_size) *input_size = sh.input_size;
    std::vector<WalkJob> wj{WalkJob{sh.bits, 8ull * n, 0, max_blocks, 0}};
    std::vector<Walked> w;
    rc = walk_streams(ctx, (const uint32_t*)d_src, wj, -1, -1, w);
    if (rc) return rc;
    if (w[0].status) return ctx->fail(-w[0].status, "Invalid bitstream: corrupted block length");
    rec_bit[0] = sh.bits;
    for (size_t b = 0; b < w[0].bit_off.size(); b++) rec_bit[b + 1] = w[0].bit_off[b] + w[0].bits[b];
    *nblocks = (uint32_t)w[0].n;
    return 0;
}
// ---- whole stream, host buffers ------------------------------------------------------------------------------
int kz_compress_stream(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, int64_t input_size,
                       const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n) {
    if (!ctx || !out_n || (!src && n) || !dst) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    const size_t dcap = kz_max_stream_output(n, block_size);
    CK(ctx->d_in.ensure(n + 64));
    CK(ctx->d_out.ensure(dcap + 64));
    if (n) CK(cudaMemcpyAsync(ctx->d_in.p, src, n, cudaMemcpyHostToDevice, ctx->stream));
    size_t produced = 0;
    int rc = kz_compress_stream_device(ctx, t48, etype, block_size, checksum_bits, input_size, ctx->d_in.p, n, ctx->d_out.p, dcap, &produced);
    if (rc) return rc;
    if (produced > cap) return ctx->fail(KZ_ERR_WRITE_FILE, "output buffer too small");
    CK(cudaMemcpyAsync(dst, ctx->d_out.p, produced, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *out_n = produced;
    return 0;
}

int kz_decompress_stream(kz_ctx* ctx, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n) {
    if (!ctx || !out_n || !src || (!dst && cap)) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    CK(ctx->d_in.ensure(n + 128));
    CK(ctx->d_out.ensure(cap + 64));
    CK(cudaMemsetAsync((uint8_t*)ctx->d_in.p + (n & ~size_t(3)), 0, 128, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_in.p, src, n, cudaMemcpyHostToDevice, ctx->stream));
    size_t produced = 0;
    int rc = kz_decompress_stream_device(ctx, ctx->d_in.p, n, ctx->d_out.p, cap, &produced);
    if (rc) return rc;
    if (produced) CK(cudaMemcpyAsync(dst, ctx->d_out.p, produced, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *out_n = produced;
    return 0;
}

// ---- many independent streams in one call (kz_compress_streams / kz_decompress_streams and their _device variants) ------------
// Every input file of BlockCompressor is a stream of its own (app/BlockCompressor.go:543-613); blocks are independent
// (io/CompressedStream.go:896-898), so the blocks of all streams run through the stages together, pass by pass (kz_stream_plan.h).

static int check_stream_args(kz_ctx* ctx, uint32_t nstreams, const void* src, const uint64_t* src_off, const uint64_t* src_len, const void* dst,
                             const uint64_t* dst_off, const uint64_t* dst_cap, const uint64_t* out_len, const int32_t* status, bool device) {
    if (nstreams && (!src_off || !src_len || !dst_off || !dst_cap || !out_len || !status)) return ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument array");
    int rc = check_spans(ctx, src, src_off, src_len, nstreams, device);
    return rc ? rc : check_spans(ctx, dst, dst_off, dst_cap, nstreams, device);
}

// The return value and statuses of a many-stream call: a call-level failure rc sets every status; otherwise the first failing stream's code.
static int finish_streams(uint32_t nstreams, int32_t* status, uint64_t* out_len, int rc) {
    if (rc) {
        for (uint32_t s = 0; s < nstreams; s++) {
            if (status) status[s] = rc;
            if (out_len) out_len[s] = 0;
        }
        return rc;
    }
    for (uint32_t s = 0; s < nstreams; s++)
        if (status[s]) return status[s];
    return 0;
}

// Compresses stream s = d_src[src_off[s] : + src_len[s]] with blocks of block_size[s] bytes. Stream s is assembled in ctx->d_asm at
// 8 * stage_off[s] (16-byte aligned); its length is out_len[s], status[s] = -KZ_ERR_WRITE_FILE when it exceeds dst_cap[s]. A stream whose
// block size kz_compress_stream refuses gets -KZ_ERR_INVALID_PARAM and no blocks; the other streams' blocks share every pass, whatever
// their block sizes.
static int compress_streams_impl(kz_ctx* ctx, uint64_t t48, uint32_t etype, const uint32_t* block_size, uint32_t checksum_bits, uint32_t nstreams,
                                 const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size,
                                 const uint64_t* dst_cap, uint64_t* out_len, int32_t* status, std::vector<uint64_t>& stage_off, uint64_t* stage_total) {
    int rc = check_checksum_bits(ctx, checksum_bits);
    if (rc) return rc;
    if (!etype_supported(etype)) return ctx->fail(KZ_ERR_CREATE_CODEC, "entropy codec not available on the GPU path");
    TransformPlan plan;
    rc = plan_transforms(ctx, t48, etype, plan, KZ_ERR_CREATE_CODEC);
    if (rc) return rc;
    // the blocks of every stream, stream after stream, prepared together before the passes; a refused stream has none
    std::vector<uint64_t> cut_len(src_len, src_len + nstreams);
    for (uint32_t s = 0; s < nstreams; s++)
        if (!block_size_ok(block_size[s])) cut_len[s] = 0;
    const BlockList bl = cut_blocks(src_off, cut_len.data(), nstreams, block_size);
    const uint32_t nb = bl.size();
    std::vector<uint64_t> bbs(nb);  // ctx["blockSize"] of every block
    for (uint32_t s = 0; s < nstreams; s++)
        for (uint32_t b = bl.first[s]; b < bl.first[s + 1]; b++) bbs[b] = block_size[s];
    BlockPrep prep;
    rc = prepare_blocks(ctx, plan, ctx->skip_blocks, checksum_bits, d_src, bl, prep);
    if (rc) return rc;
    // passes: transforms and entropy coding of the blocks of a pass, then their bit strings packed into the arena as records b
    const EntropyScratch es = entropy_scratch(etype);
    const PassPlan P = plan_compress_passes(bl.len, [&](uint64_t s) { return compress_block_cost(s, es); });
    RecordArena arena(nb);
    for (uint32_t p = 0; p < P.npasses(); p++) {
        const uint32_t i0 = P.first[p], k = P.first[p + 1] - i0;
        const uint64_t s = P.stride[p];
        CK(ctx->d_slots.ensure(s * k + 64));
        uint8_t* slots = ctx->d_slots.as<uint8_t>();
        std::vector<uint32_t> lens(k);
        std::vector<uint64_t> pbs(k);
        CopyList place;
        for (uint32_t j = 0; j < k; j++) {
            const uint32_t b = P.order[i0 + j];
            lens[j] = bl.len[b];
            pbs[j] = bbs[b];
            place.add(d_src + bl.off[b], slots + j * s, bl.len[b]);
        }
        rc = run_copies(ctx, place);
        if (rc) return rc;
        rc = arena.encode_pass(ctx, plan, etype, checksum_bits, slots, s, lens, pbs, prep.pick(&P.order[i0], k), &P.order[i0]);
        if (rc) return rc;
    }
    // assembly (Writer.processBlock :951-976, Close :593-594): stream header, then 5 b | lw b prefix and bit string of every block, then the
    // end marker. Lengths are known here, so the host lays out every segment; one concat writes all streams.
    stage_off.assign(nstreams, 0);
    uint64_t stage = 0;
    SegmentList sl;
    for (uint32_t s = 0; s < nstreams; s++) {
        if (!block_size_ok(block_size[s])) {
            out_len[s] = 0;
            status[s] = -KZ_ERR_INVALID_PARAM;
            continue;
        }
        std::vector<uint8_t> hdr, pre(8 * (size_t)(bl.first[s + 1] - bl.first[s]), 0);
        const uint32_t hdr_bits =
            ctx->headerless_writer ? 0 : build_stream_header(hdr, t48, etype, block_size[s], checksum_bits, input_size ? input_size[s] : 0);  // Writer.writeHeader :430
        std::vector<uint32_t> pre_bits;
        uint64_t bits = hdr_bits + END_MARKER_BITS;
        for (uint32_t b = bl.first[s]; b < bl.first[s + 1]; b++) {
            pre_bits.push_back(write_block_prefix(&pre[8 * pre_bits.size()], arena.bits[b]));
            bits += pre_bits.back() + arena.bits[b];
        }
        out_len[s] = (bits + 7) / 8;
        status[s] = out_len[s] > dst_cap[s] ? -KZ_ERR_WRITE_FILE : 0;
        if (status[s]) continue;
        stage_off[s] = stage;
        sl.at(8 * stage);
        sl.add_host(hdr.data(), hdr_bits);
        for (uint32_t b = bl.first[s], j = 0; b < bl.first[s + 1]; b++, j++) {
            sl.add_host(&pre[8 * j], pre_bits[j]);
            sl.add_device(arena.record(ctx, b), 0, arena.bits[b]);
        }
        sl.add_end_marker();
        stage += round16(out_len[s]);
    }
    *stage_total = stage;
    CK(ctx->d_asm.ensure(stage + 64));
    return sl.write(ctx, ctx->d_asm.as<uint8_t>());
}

// One group of streams whose headers differ at most in block size (sh: the first one's; shs[s]: stream s's, which gives its first record's
// bit and its block size): walk, then decode_walked pass by pass (plan_decompress_passes by block size), each block written behind the
// previous one of its stream at d_dst + dst_off[s]. A stream on which anything goes wrong (a bad record, block header, entropy payload or checksum, too
// little room, or a failing stage call of a pass it has blocks in) is put on `alone`; the caller decodes it again on its own with the
// single-stream path, so that its status is the code kz_decompress_stream_device gives for the same bytes.
static int decode_stream_group(kz_ctx* ctx, const StreamHeader& sh, const TransformPlan& plan, const std::vector<uint32_t>& grp,
                               const std::vector<StreamHeader>& shs, const uint8_t* d_src, uint64_t src_bytes, const uint64_t* src_off,
                               const uint64_t* src_len, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len,
                               int32_t* status, std::vector<uint32_t>& alone) {
    const uint32_t ng = (uint32_t)grp.size();
    const uint32_t* d_words = (const uint32_t*)d_src;
    // as many records per stream as the single-stream path allows, and no more than its bytes can hold
    std::vector<WalkJob> wj(ng);
    for (uint32_t g = 0; g < ng; g++) {
        const uint32_t s = grp[g];
        const uint64_t by_cap = std::min<uint64_t>(dst_cap[s] / 1024 + 16, 1u << 22);
        wj[g] = WalkJob{8 * src_off[s] + shs[s].bits, 8 * (src_off[s] + src_len[s]), 0, (uint32_t)std::min<uint64_t>(by_cap, 8 * src_len[s] / 9 + 1), 0};
    }
    std::vector<Walked> w;
    int rc = walk_streams(ctx, d_words, wj, ctx->range_from, ctx->range_to, w);
    if (rc) return rc;
    std::vector<DecodeFailure> fail(ng);
    std::vector<DecJob> all;
    std::vector<uint32_t> own;
    std::vector<uint8_t> last;
    for (uint32_t g = 0; g < ng; g++) {
        if (w[g].status || w[g].overflow) fail[g].note(STAGE_WALK, w[g].status ? w[g].status : -KZ_ERR_BLOCK_SIZE, "");
        else w[g].append(g, shs[grp[g]].block_size, all, own, last);
    }
    std::vector<uint64_t> written(ng, 0);
    auto place = [&](uint32_t g, uint32_t len) {  // behind the stream's earlier blocks, within its dst_cap
        const uint32_t s = grp[g];
        if (written[g] + len > dst_cap[s]) return NO_ROOM;
        written[g] += len;
        return dst_off[s] + written[g] - len;
    };
    std::vector<uint32_t> bs(all.size());
    for (size_t b = 0; b < all.size(); b++) bs[b] = all[b].block_size;
    // the blocks of a stream have one block size, so they stay in order within and across passes, and place() sees them in order
    const PassPlan P = plan_decompress_passes(bs);
    for (uint32_t p = 0; p < P.npasses(); p++) {
        std::vector<DecJob> jobs;
        std::vector<uint32_t> owner;
        std::vector<uint8_t> run_last;
        for (uint32_t i = P.first[p]; i < P.first[p + 1]; i++) {
            const uint32_t b = P.order[i];
            jobs.push_back(all[b]), owner.push_back(own[b]), run_last.push_back(last[b]);
        }
        rc = decode_walked(ctx, sh, plan, d_words, (src_bytes + 3) / 4 + 16, jobs, owner, run_last,
                           [&](uint32_t b, uint32_t len) { return place(owner[b], len); }, d_dst, fail.data());
        if (rc) return rc;
    }
    for (uint32_t g = 0; g < ng; g++) {
        const uint32_t s = grp[g];
        if (fail[g].failed()) {
            alone.push_back(s);
        } else {
            status[s] = 0;
            out_len[s] = written[g];
        }
    }
    return 0;
}

// Decodes stream s = d_src[src_off[s] : + src_len[s]] (>= 64 readable bytes behind it) to d_dst + dst_off[s]. src_bytes: readable bytes at d_src.
static int decompress_streams_impl(kz_ctx* ctx, uint32_t nstreams, const uint8_t* d_src, uint64_t src_bytes, const uint64_t* src_off, const uint64_t* src_len,
                                   uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status) {
    for (uint32_t s = 0; s < nstreams; s++) status[s] = 0, out_len[s] = 0;
    if (nstreams == 0) return 0;
    // headers: the first 64 bytes of every stream in one gather (a headerless stream has none to read), then each stream's header or the
    // headerless reader setting; the streams whose header fields differ at most in block size form a group and share its passes
    std::vector<uint8_t> head(64 * (size_t)nstreams);
    std::vector<uint64_t> head_len(nstreams, 0);
    if (!ctx->headerless_reader.on) head_len.assign(src_len, src_len + nstreams);
    int rc = gather_heads(ctx, d_src, src_off, head_len.data(), nstreams, 64, head.data());
    if (rc) return rc;
    std::vector<StreamHeader> sh(nstreams);
    std::vector<TransformPlan> plan(nstreams);
    std::map<std::tuple<uint64_t, uint32_t, uint32_t>, std::vector<uint32_t>> groups;
    for (uint32_t s = 0; s < nstreams; s++) {
        status[s] = stream_header(ctx, &head[64 * (size_t)s], src_len[s], sh[s]);
        if (status[s]) continue;
        rc = plan_transforms(ctx, sh[s].t48, sh[s].etype, plan[s], KZ_ERR_INVALID_CODEC);
        if (rc) return rc;
        if (!etype_supported(sh[s].etype)) return ctx->fail(KZ_ERR_INVALID_CODEC, "entropy codec not available on the GPU path");
        groups[std::make_tuple(sh[s].t48, sh[s].etype, sh[s].checksum_bits)].push_back(s);
    }
    std::vector<uint32_t> alone;
    for (auto& kv : groups) {
        const uint32_t s0 = kv.second[0];
        rc = decode_stream_group(ctx, sh[s0], plan[s0], kv.second, sh, d_src, src_bytes, src_off, src_len, d_dst, dst_off, dst_cap, out_len, status, alone);
        if (rc) return rc;
    }
    for (uint32_t s : alone) {  // only corrupt input, too little room or a failing stage call gets here
        size_t n = 0;
        status[s] = decompress_device_impl(ctx, nullptr, 0, 0, ctx->range_from, ctx->range_to, d_src + src_off[s], src_len[s], d_dst + dst_off[s], dst_cap[s], &n);
        out_len[s] = status[s] ? 0 : n;
    }
    return 0;
}

// kz_compress_streams[_bs][_device]: block_size has nstreams entries. one_size != nullptr: the call has one block size, *one_size, which is
// checked at call level as kz_compress_stream checks it.
static int compress_streams_device(kz_ctx* ctx, uint64_t t48, uint32_t etype, const uint32_t* block_size, const uint32_t* one_size, uint32_t checksum_bits,
                                   uint32_t nstreams, const void* d_src, const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, void* d_dst,
                                   const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    int rc = check_stream_args(ctx, nstreams, d_src, src_off, src_len, d_dst, dst_off, dst_cap, out_len, status, true);
    if (!rc && !block_size) rc = ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument array");
    if (rc) return finish_streams(nstreams, status, out_len, rc);
    if (cudaSetDevice(ctx->device) != cudaSuccess) return finish_streams(nstreams, status, out_len, -KZ_ERR_PROCESS_BLOCK);
    if (one_size && (rc = check_encode_args(ctx, *one_size, checksum_bits)) != 0) return finish_streams(nstreams, status, out_len, rc);
    std::vector<uint64_t> stage_off;
    uint64_t stage_total = 0;
    rc = compress_streams_impl(ctx, t48, etype, block_size, checksum_bits, nstreams, (const uint8_t*)d_src, src_off, src_len, input_size, dst_cap, out_len,
                               status, stage_off, &stage_total);
    if (!rc) {
        CopyList out;
        for (uint32_t s = 0; s < nstreams; s++)
            if (!status[s]) out.add(ctx->d_asm.as<uint8_t>() + stage_off[s], (uint8_t*)d_dst + dst_off[s], out_len[s]);
        rc = run_copies(ctx, out);
        if (!rc && cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = ctx->cuda_fail(cudaGetLastError(), "compress_streams");
    }
    return finish_streams(nstreams, status, out_len, rc);
}

static int compress_streams_host(kz_ctx* ctx, uint64_t t48, uint32_t etype, const uint32_t* block_size, const uint32_t* one_size, uint32_t checksum_bits,
                                 uint32_t nstreams, const uint8_t* src, const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, uint8_t* dst,
                                 const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    int rc = check_stream_args(ctx, nstreams, src, src_off, src_len, dst, dst_off, dst_cap, out_len, status, false);
    if (!rc && !block_size) rc = ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument array");
    if (rc) return finish_streams(nstreams, status, out_len, rc);
    rc = [&]() -> int {
        CK(cudaSetDevice(ctx->device));
        if (one_size) {
            int r = check_encode_args(ctx, *one_size, checksum_bits);
            if (r) return r;
        }
        // the inputs packed at 16-byte aligned offsets and moved in one transfer
        std::vector<UploadPiece> in(nstreams);
        for (uint32_t s = 0; s < nstreams; s++) in[s] = UploadPiece{src + src_off[s], src_len[s], src_len[s]};
        std::vector<uint64_t> in_off, stage_off;
        uint64_t total = 0, stage_total = 0;
        int r = upload_pieces(ctx, in, in_off, &total);
        if (r) return r;
        r = compress_streams_impl(ctx, t48, etype, block_size, checksum_bits, nstreams, ctx->d_in.as<uint8_t>(), in_off.data(), src_len, input_size, dst_cap,
                                  out_len, status, stage_off, &stage_total);
        if (r) return r;
        std::vector<DownloadPiece> out;
        for (uint32_t s = 0; s < nstreams; s++)
            if (!status[s]) out.push_back(DownloadPiece{dst + dst_off[s], stage_off[s], out_len[s]});
        return download_pieces(ctx, ctx->d_asm.as<uint8_t>(), stage_total, out);
    }();
    return finish_streams(nstreams, status, out_len, rc);
}

int kz_compress_streams_device(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, uint32_t nstreams, const void* d_src,
                               const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, void* d_dst, const uint64_t* dst_off,
                               const uint64_t* dst_cap, uint64_t* out_len, int32_t* status) {
    if (int rc = after_caller_work(ctx)) return finish_streams(nstreams, status, out_len, rc);
    const std::vector<uint32_t> bs(std::max(nstreams, 1u), block_size);
    return compress_streams_device(ctx, t48, etype, bs.data(), &block_size, checksum_bits, nstreams, d_src, src_off, src_len, input_size, d_dst, dst_off, dst_cap,
                                   out_len, status);
}

int kz_compress_streams(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, uint32_t nstreams, const uint8_t* src,
                        const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, uint8_t* dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                        uint64_t* out_len, int32_t* status) {
    const std::vector<uint32_t> bs(std::max(nstreams, 1u), block_size);
    return compress_streams_host(ctx, t48, etype, bs.data(), &block_size, checksum_bits, nstreams, src, src_off, src_len, input_size, dst, dst_off, dst_cap,
                                 out_len, status);
}

int kz_compress_streams_bs_device(kz_ctx* ctx, uint64_t t48, uint32_t etype, const uint32_t* block_size, uint32_t checksum_bits, uint32_t nstreams,
                                  const void* d_src, const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, void* d_dst,
                                  const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status) {
    if (int rc = after_caller_work(ctx)) return finish_streams(nstreams, status, out_len, rc);
    return compress_streams_device(ctx, t48, etype, block_size, nullptr, checksum_bits, nstreams, d_src, src_off, src_len, input_size, d_dst, dst_off, dst_cap,
                                   out_len, status);
}

int kz_compress_streams_bs(kz_ctx* ctx, uint64_t t48, uint32_t etype, const uint32_t* block_size, uint32_t checksum_bits, uint32_t nstreams, const uint8_t* src,
                           const uint64_t* src_off, const uint64_t* src_len, const int64_t* input_size, uint8_t* dst, const uint64_t* dst_off,
                           const uint64_t* dst_cap, uint64_t* out_len, int32_t* status) {
    return compress_streams_host(ctx, t48, etype, block_size, nullptr, checksum_bits, nstreams, src, src_off, src_len, input_size, dst, dst_off, dst_cap,
                                 out_len, status);
}

int kz_decompress_streams_device(kz_ctx* ctx, uint32_t nstreams, const void* d_src, const uint64_t* src_off, const uint64_t* src_len, void* d_dst,
                                 const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status) {
    if (int rc = after_caller_work(ctx)) return finish_streams(nstreams, status, out_len, rc);
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    int rc = check_stream_args(ctx, nstreams, d_src, src_off, src_len, d_dst, dst_off, dst_cap, out_len, status, true);
    if (rc) return finish_streams(nstreams, status, out_len, rc);
    uint64_t src_bytes = 0;
    for (uint32_t s = 0; s < nstreams; s++) src_bytes = std::max(src_bytes, src_off[s] + src_len[s]);
    rc = [&]() -> int {
        CK(cudaSetDevice(ctx->device));
        return decompress_streams_impl(ctx, nstreams, (const uint8_t*)d_src, src_bytes, src_off, src_len, (uint8_t*)d_dst, dst_off, dst_cap, out_len, status);
    }();
    return finish_streams(nstreams, status, out_len, rc);
}

int kz_decompress_streams(kz_ctx* ctx, uint32_t nstreams, const uint8_t* src, const uint64_t* src_off, const uint64_t* src_len, uint8_t* dst,
                          const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* out_len, int32_t* status) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    int rc = check_stream_args(ctx, nstreams, src, src_off, src_len, dst, dst_off, dst_cap, out_len, status, false);
    if (rc) return finish_streams(nstreams, status, out_len, rc);
    rc = [&]() -> int {
        CK(cudaSetDevice(ctx->device));
        // inputs packed at 16-byte aligned offsets with 64 zero bytes behind each (what kz_decompress_stream gives a single stream);
        // outputs staged at 16-byte aligned offsets of dst_cap[s] bytes each, packed by length and moved back in one transfer
        std::vector<UploadPiece> in(nstreams);
        std::vector<uint64_t> in_off, st_off(nstreams), pk_off(nstreams);
        uint64_t total = 0, st_total = 0;
        for (uint32_t s = 0; s < nstreams; s++) {
            in[s] = UploadPiece{src + src_off[s], src_len[s], src_len[s] + 64};
            st_off[s] = st_total, st_total += round16(dst_cap[s]);
        }
        int r = upload_pieces(ctx, in, in_off, &total);
        if (r) return r;
        CK(ctx->d_out.ensure(st_total + 64));
        r = decompress_streams_impl(ctx, nstreams, ctx->d_in.as<uint8_t>(), total, in_off.data(), src_len, ctx->d_out.as<uint8_t>(), st_off.data(), dst_cap,
                                        out_len, status);
        if (r) return r;
        uint64_t pk_total = 0;
        for (uint32_t s = 0; s < nstreams; s++) {
            pk_off[s] = pk_total;
            if (!status[s]) pk_total += round16(out_len[s]);
        }
        CK(ctx->d_asm.ensure(pk_total + 64));
        CopyList pack;
        for (uint32_t s = 0; s < nstreams; s++)
            if (!status[s]) pack.add(ctx->d_out.as<uint8_t>() + st_off[s], ctx->d_asm.as<uint8_t>() + pk_off[s], out_len[s]);
        r = run_copies(ctx, pack);
        if (r) return r;
        std::vector<DownloadPiece> out;
        for (uint32_t s = 0; s < nstreams; s++)
            if (!status[s]) out.push_back(DownloadPiece{dst + dst_off[s], pk_off[s], out_len[s]});
        return download_pieces(ctx, ctx->d_asm.as<uint8_t>(), pk_total, out);
    }();
    return finish_streams(nstreams, status, out_len, rc);
}

// ---- stream index and batched range reads (kz_index_*, kz_read_ranges[_device]; plan and blob in kz_read_plan.h) -------------
}  // extern "C"

struct kz_index : kz::StreamIndex {};

namespace {

StreamHeader index_header(const kz_index& ix) {
    StreamHeader sh;
    sh.t48 = ix.t48;
    sh.etype = ix.etype;
    sh.block_size = ix.block_size;
    sh.checksum_bits = ix.checksum_bits;
    sh.input_size = ix.input_size;
    sh.bits = ix.header_bits;
    return sh;
}

// One stream of a read: its index, where its bytes start (src + at in the host variant, d_src + at, a multiple of 16, in the device
// variant) and how many there are.
struct ReadSource {
    kz_index* ix;
    uint64_t at, n;
};

// The stream bytes of one read pass as decode_walked sees them: the device streams themselves, or the packed windows of the host variant.
struct PassInput {
    const uint32_t* d_words = nullptr;
    uint64_t words_len = 0;
};

// Host variant: uploads only the byte windows that hold the records of pairs ks (plan order: stream after stream, blocks ascending): each
// starts at a multiple of 16 and carries the 64 bytes the decoders may read behind a record (zeros where its stream ends); windows of one
// stream that meet are merged. One transfer per pass. bit_off[k]: the first payload bit of pair k's record in the packed buffer.
int upload_windows(kz_ctx* ctx, const std::vector<ReadSource>& S, const ReadPlan& P, const uint8_t* src, const std::vector<uint32_t>& ks,
                   std::vector<uint64_t>& bit_off, PassInput& in) {
    struct Window {
        uint32_t s;
        uint64_t lo, hi;  // bytes [lo, hi) of stream s
    };
    std::vector<Window> win;
    std::vector<uint32_t> win_of(ks.size());
    for (size_t i = 0; i < ks.size(); i++) {
        const uint32_t s = P.stream[ks[i]];
        const kz_index& ix = *S[s].ix;
        const uint64_t b = P.blocks[ks[i]];
        const uint64_t lo = (ix.start[b] / 8) & ~15ull, hi = (ix.start[b] + ix.bits[b] + 7) / 8 + 64;
        if (win.empty() || win.back().s != s || lo > win.back().hi) win.push_back(Window{s, lo, hi});
        else win.back().hi = std::max(win.back().hi, hi);
        win_of[i] = (uint32_t)win.size() - 1;
    }
    std::vector<UploadPiece> pieces;
    for (const Window& w : win) pieces.push_back(UploadPiece{src + S[w.s].at + w.lo, std::min<uint64_t>(w.hi, S[w.s].n) - w.lo, w.hi - w.lo});
    std::vector<uint64_t> at;
    uint64_t total = 0;
    int rc = upload_pieces(ctx, pieces, at, &total);
    if (rc) return rc;
    in.d_words = ctx->d_in.as<uint32_t>();
    in.words_len = (total + 3) / 4 + 16;
    for (size_t i = 0; i < ks.size(); i++) {
        const Window& w = win[win_of[i]];
        bit_off[ks[i]] = S[w.s].ix->start[P.blocks[ks[i]]] - 8 * w.lo + 8 * at[win_of[i]];
    }
    if (ctx->profile) {
        auto& e = ctx->prof["read:h2d"];
        e.bytes_in += win.size(), e.bytes_out += total, e.launches++;
    }
    return 0;
}

// The keys of the cached read's pairs: the record hash of every record (kz_xxh64_core.cuh) and the header fields a record's decode
// depends on. Host variant: hashed on the CPU from the caller's streams. Device variant: one record_hash launch over every tile of the
// records of every stream, one thread per record for the roots, one copy of the keys back.
int cache_keys(kz_ctx* ctx, const std::vector<ReadSource>& S, const ReadPlan& P, const uint8_t* src, const uint8_t* d_src, std::vector<CacheKey>& key) {
    const uint32_t nk = (uint32_t)P.blocks.size();
    key.assign(nk, CacheKey());
    for (uint32_t k = 0; k < nk; k++) {
        const kz_index& ix = *S[P.stream[k]].ix;
        key[k].bits = ix.bits[P.blocks[k]];
        key[k].t48 = ix.t48;
        key[k].etype = ix.etype;
        key[k].checksum_bits = ix.checksum_bits;
        key[k].block_size = ix.block_size;
        key[k].last = P.blocks[k] + 1 == ix.nblocks();
    }
    if (nk == 0) return 0;
    if (src) {
        HostScope hs(ctx, "record_hash");
        for (uint32_t k = 0; k < nk; k++) {
            const ReadSource& r = S[P.stream[k]];
            key[k].hash = record_hash_host(src + r.at, r.ix->start[P.blocks[k]], r.ix->bits[P.blocks[k]]);
        }
        return 0;
    }
    std::vector<RecordHashJob> jobs(nk);
    uint64_t ntiles = 0;
    for (uint32_t k = 0; k < nk; k++) {
        const ReadSource& r = S[P.stream[k]];
        jobs[k] = RecordHashJob{8 * r.at + r.ix->start[P.blocks[k]], r.ix->bits[P.blocks[k]], ntiles};
        ntiles += record_tiles(r.ix->bits[P.blocks[k]]);
    }
    Packer pk;
    const size_t o_j = pk.add(jobs.data(), jobs.size() * sizeof(RecordHashJob));
    int rc = upload(ctx, pk);
    if (rc) return rc;
    CK(ctx->d_ws.ensure((ntiles + nk) * 8));
    const RecordHashJob* d_jobs = (const RecordHashJob*)(ctx->d_tables.as<uint8_t>() + o_j);
    uint64_t* d_dig = ctx->d_ws.as<uint64_t>();
    uint64_t* d_key = d_dig + ntiles;
    {
        LaunchScope ls(ctx, "record_hash");
        record_hash_tiles_kernel<<<(unsigned)((ntiles + RECORD_HASH_WARPS - 1) / RECORD_HASH_WARPS), 32 * RECORD_HASH_WARPS, 0, ctx->stream>>>(
            (const uint32_t*)d_src, d_jobs, (int)nk, ntiles, d_dig);
    }
    {
        LaunchScope ls(ctx, "record_hash");
        record_hash_root_kernel<<<(nk + 127) / 128, 128, 0, ctx->stream>>>(d_jobs, (int)nk, d_dig, d_key);
    }
    CK(cudaGetLastError());
    std::vector<uint64_t> h(nk);
    CK(cudaMemcpyAsync(h.data(), d_key, (size_t)nk * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (uint32_t k = 0; k < nk; k++) key[k].hash = h[k];
    return 0;
}

// One batched read over the streams S, every one already checked against its index (read_stream_check). src is the host buffer the
// streams lie in (host variant: dst is host memory too) or null (d_src holds them, dst is device memory). Request i reads stream
// req_src[i] (null: every request reads S[0]).
// cache: null, or the block cache of a cached read. With a cache the blocks found in it form a pass of their own, served first by one
// copy launch out of its pages; the others (the misses) run through the decode passes as every block does without a cache, and each
// that decodes is inserted behind its pass.
// Every rule that makes a one-stream read's results holds per stream: a pair's pass is cut from its decode group only, the unseekable rule
// is kept per stream, and a failed block of a pass of several is decoded again alone. So what a request gets does not depend on which
// other streams share the call.
int read_ranges_impl(kz_ctx* ctx, kz_cache* cache, const uint8_t* src, const uint8_t* d_src, const std::vector<ReadSource>& S, uint32_t nreq,
                     const uint32_t* req_src, const uint64_t* off, const uint64_t* len, uint8_t* dst, const uint64_t* dst_off, uint64_t* out_len,
                     int32_t* status) {
    const bool host = src != nullptr;
    const uint32_t ns = (uint32_t)S.size();
    // decode groups, numbered in the order they first appear: the header and transform plan of each
    std::map<std::tuple<uint64_t, uint32_t, uint32_t, uint32_t>, uint32_t> group_of;
    std::vector<StreamHeader> gsh;
    std::vector<TransformPlan> gplan;
    std::vector<ReadStream> RS(ns);
    uint64_t src_end = 0;
    int rc = 0;
    for (uint32_t s = 0; s < ns; s++) {
        const kz_index& ix = *S[s].ix;
        auto it = group_of.find(std::make_tuple(ix.t48, ix.etype, ix.block_size, ix.checksum_bits));
        if (it == group_of.end()) {
            it = group_of.emplace(std::make_tuple(ix.t48, ix.etype, ix.block_size, ix.checksum_bits), (uint32_t)gsh.size()).first;
            gsh.push_back(index_header(ix));
            gplan.emplace_back();
            rc = plan_transforms(ctx, ix.t48, ix.etype, gplan.back(), KZ_ERR_CREATE_CODEC);
            if (rc) return rc;
        }
        RS[s] = ReadStream{ix.nblocks(), ix.block_size, ix.size, it->second};
        src_end = std::max(src_end, S[s].at + S[s].n);
    }
    const ReadPlan P = plan_reads_streams(RS, nreq, req_src, off, len);
    const uint32_t nk = (uint32_t)P.blocks.size();
    auto IX = [&](uint32_t k) -> kz_index& { return *S[P.stream[k]].ix; };
    auto is_last = [&](uint32_t k) { return P.blocks[k] + 1 == IX(k).nblocks(); };
    // The pairs to decode, pass after pass: order[first[p] .. first[p + 1]) (in plan order). Without a cache every touched pair; with
    // one the pairs it lacks (hit[k] names the entry of the others).
    std::vector<CacheKey> key;
    std::vector<const CacheEntry*> hit(cache ? nk : 0, nullptr);
    std::vector<uint32_t> order, first;
    if (cache) {
        rc = cache_keys(ctx, S, P, src, d_src, key);
        if (rc) return rc;
        for (uint32_t k = 0; k < nk; k++)
            if (!(hit[k] = cache->pc.lookup(key[k]))) order.push_back(k);
        first = plan_read_passes(RS, P.stream, order);
    } else {
        order.resize(nk);
        std::iota(order.begin(), order.end(), 0u);
        first = P.first;
    }
    const uint32_t npasses = (uint32_t)first.size() - 1;
    const uint32_t hp = cache ? 1 : 0;  // the pass number of the first decode pass (the cache's blocks are pass 0)
    // A request is staged (its slices gathered in ctx->d_asm, delivered when every block it touches has decoded) when it goes to host
    // memory or its blocks lie in more than one pass: nothing is written for a request that fails. A request on cached blocks only is
    // staged too when one of them lies behind a block of its stream still to decode, whose length may make it unseekable.
    std::vector<uint32_t> pass_of(nk, 0), slot_of(nk, 0), first_miss(ns, nk);
    for (uint32_t p = 0; p < npasses; p++)
        for (uint32_t i = first[p]; i < first[p + 1]; i++) pass_of[order[i]] = hp + p, slot_of[order[i]] = i - first[p];
    for (uint32_t k : order) first_miss[P.stream[k]] = std::min(first_miss[P.stream[k]], k);
    std::vector<uint32_t> first_pass(nreq, 0);
    std::vector<uint8_t> staged(nreq, host);
    for (uint32_t k = 0; k < nk; k++)
        for (uint64_t s = P.slice_of[k]; s < P.slice_of[k + 1]; s++) {
            const ReadSlice& sl = P.slices[s];
            if (sl.at == 0) first_pass[sl.req] = pass_of[k];
        }
    for (const ReadSlice& sl : P.slices)
        if (pass_of[sl.block] != first_pass[sl.req] || (cache && hit[sl.block] && sl.block > first_miss[P.stream[sl.block]])) staged[sl.req] = 1;
    std::vector<uint64_t> stage_at(nreq, 0);
    uint64_t stage_total = 0;
    for (uint32_t i = 0; i < nreq; i++)
        if (staged[i]) stage_at[i] = stage_total, stage_total += P.want[i];
    if (stage_total) CK(ctx->d_asm.ensure(stage_total + 64));

    std::vector<int32_t> blk_status(nk, 0);
    std::vector<uint32_t> blk_len(nk, 0);
    std::vector<uint64_t> bit_off(nk, 0);
    for (uint32_t i = 0; i < nreq; i++) status[i] = 0, out_len[i] = 0;
    std::vector<uint32_t> uns(ns, nk);  // per stream: its first touched pair whose length breaks the block arithmetic
    auto broken = [&](uint32_t k) { return k >= uns[P.stream[k]]; };
    uint64_t dec_blocks = 0, dec_bytes = 0, out_slices = 0, out_bytes = 0;
    uint8_t* pages = cache ? (uint8_t*)cache->d_pages : nullptr;
    bool hit_copies = false;  // the copies out of the cache were queued; the call returns only after they ran
    if (cache) {
        // the cached blocks: their lengths are known, so is the unseekable rule among them; a request on them alone that is not staged
        // gets its status now, before its bytes are written
        uint64_t hits = 0, hit_bytes = 0, served = 0;
        for (uint32_t k = 0; k < nk; k++)
            if (hit[k]) {
                blk_len[k] = hit[k]->len;
                if (is_last(k) ? blk_len[k] == 0 : blk_len[k] != IX(k).block_size) uns[P.stream[k]] = std::min(uns[P.stream[k]], k);
                hits++, hit_bytes += blk_len[k];
            }
        for (uint32_t k = 0; k < nk; k++)
            if (hit[k] && broken(k))
                for (uint64_t s = P.slice_of[k]; s < P.slice_of[k + 1]; s++)
                    if (!staged[P.slices[s].req]) status[P.slices[s].req] = -KZ_ERR_INVALID_FILE;
        CopyList out;
        for (uint32_t k = 0; k < nk; k++) {
            if (!hit[k] || broken(k)) continue;
            for (uint64_t s = P.slice_of[k]; s < P.slice_of[k + 1]; s++) {
                const ReadSlice& sl = P.slices[s];
                if (status[sl.req] || sl.in_block >= blk_len[k]) continue;
                const uint64_t m = std::min<uint64_t>(sl.len, blk_len[k] - sl.in_block);
                uint8_t* to = staged[sl.req] ? ctx->d_asm.as<uint8_t>() + stage_at[sl.req] + sl.at : dst + dst_off[sl.req] + sl.at;
                cache_slice_copies(*hit[k], sl.in_block, m, [&](uint32_t page, uint64_t in_page, uint64_t at, uint64_t c) {
                    out.add(pages + page * CACHE_PAGE + in_page, to + at, c);
                });
                out_len[sl.req] += m;
                out_slices++, out_bytes += m, served += m;
            }
        }
        rc = run_copies(ctx, out);
        if (rc) return rc;
        hit_copies = !out.jobs.empty();
        cache->pc.note_served(served);
        if (ctx->profile) {
            auto& h = ctx->prof["read:cache_hit"];
            h.bytes_in += hits, h.bytes_out += hit_bytes, h.launches++;
        }
    }
    const CacheStats before = cache ? cache->pc.stats() : CacheStats();
    uint64_t miss_blocks = 0, miss_bytes = 0, ins_bytes = 0;
    for (uint32_t p = 0; p < npasses; p++) {
        const uint32_t a = first[p], e = first[p + 1];
        // a stream's blocks of the pass are decoded when its first one there lies before its unseekable block, as a one-stream read
        // decodes a pass whose first block does
        std::vector<uint32_t> ks;
        bool take = false;
        for (uint32_t i = a; i < e; i++) {
            const uint32_t k = order[i];
            if (i == a || P.stream[k] != P.stream[order[i - 1]]) take = !broken(k);
            if (take) ks.push_back(k);
        }
        if (ks.empty()) continue;
        const StreamHeader& sh = gsh[RS[P.stream[ks[0]]].group];
        const TransformPlan& plan = gplan[RS[P.stream[ks[0]]].group];
        const uint32_t bs = sh.block_size;
        const uint64_t astride = decompress_slot(bs);
        PassInput in;
        if (host) {
            rc = upload_windows(ctx, S, P, src, ks, bit_off, in);
            if (rc) return rc;
        } else {
            in.d_words = (const uint32_t*)d_src;
            in.words_len = (src_end + 3) / 4 + 16;
            for (uint32_t k : ks) bit_off[k] = 8 * S[P.stream[k]].at + IX(k).start[P.blocks[k]];
        }
        CK(ctx->d_slots.ensure(astride * (e - a) + 64));
        uint8_t* arena = ctx->d_slots.as<uint8_t>();
        // the pairs ks of the pass into their arena slots; a block longer than block_size has no slot and fails
        std::vector<DecJob> jobs(ks.size(), DecJob());
        std::vector<uint8_t> last(ks.size());
        for (size_t i = 0; i < ks.size(); i++) {
            jobs[i].bit_off = bit_off[ks[i]];
            jobs[i].bits = IX(ks[i]).bits[P.blocks[ks[i]]];
            jobs[i].block_size = sh.block_size;
            last[i] = is_last(ks[i]);
        }
        std::vector<DecodeFailure> fail;
        std::vector<uint32_t> olen;
        rc = decode_isolated(ctx, sh, plan, in.d_words, in.words_len, jobs, last,
                             [&](uint32_t i, uint32_t n) { return n > bs ? NO_ROOM : (uint64_t)slot_of[ks[i]] * astride; }, arena, fail, olen);
        if (rc) return rc;
        for (size_t i = 0; i < ks.size(); i++) blk_status[ks[i]] = fail[i].code, blk_len[ks[i]] = olen[i];
        for (uint32_t k : ks) {
            const uint32_t s = P.stream[k];
            if (blk_len[k] > bs || (!blk_status[k] && (is_last(k) ? blk_len[k] == 0 : blk_len[k] != bs))) uns[s] = std::min(uns[s], k);
            if (!blk_status[k]) dec_blocks++, dec_bytes += blk_len[k];
            if (is_last(k) && !blk_status[k] && uns[s] == nk) IX(k).size = (int64_t)((IX(k).nblocks() - 1) * bs + blk_len[k]);
        }
        // every block of the pass that decoded goes into the cache; an entry this pass made and evicted again gets no copy
        std::vector<std::pair<uint32_t, uint64_t>> fresh;  // (pair, serial)
        if (cache)
            for (uint32_t k : ks) {
                miss_blocks++, miss_bytes += blk_status[k] ? 0 : blk_len[k];
                if (blk_status[k]) continue;
                bool made = false;
                const CacheEntry* en = cache->pc.insert(key[k], blk_len[k], &made);
                if (made) fresh.push_back({k, en->serial}), ins_bytes += blk_len[k];
            }
        for (uint32_t k : ks) {
            if (broken(k)) blk_status[k] = -KZ_ERR_INVALID_FILE;
            if (blk_status[k])
                for (uint64_t s = P.slice_of[k]; s < P.slice_of[k + 1]; s++)
                    if (!status[P.slices[s].req]) status[P.slices[s].req] = blk_status[k];
        }
        CopyList out;
        for (uint32_t k : ks)
            for (uint64_t s = P.slice_of[k]; s < P.slice_of[k + 1]; s++) {
                const ReadSlice& sl = P.slices[s];
                if (status[sl.req] || sl.in_block >= blk_len[k]) continue;
                const uint64_t m = std::min<uint64_t>(sl.len, blk_len[k] - sl.in_block);
                uint8_t* to = staged[sl.req] ? ctx->d_asm.as<uint8_t>() + stage_at[sl.req] + sl.at : dst + dst_off[sl.req] + sl.at;
                out.add(arena + (uint64_t)slot_of[k] * astride + sl.in_block, to, m);
                out_len[sl.req] += m;
                out_slices++, out_bytes += m;
            }
        for (const auto& f : fresh)
            if (const CacheEntry* en = cache->pc.peek(key[f.first], f.second))
                cache_slice_copies(*en, 0, en->len, [&](uint32_t page, uint64_t in_page, uint64_t at, uint64_t c) {
                    out.add(arena + (uint64_t)slot_of[f.first] * astride + at, pages + page * CACHE_PAGE + in_page, c);
                });
        rc = run_copies(ctx, out);
        if (rc) return rc;
        CK(cudaStreamSynchronize(ctx->stream));  // the arena and the windows are reused by the next pass
    }
    if (cache) {
        // a cached last block sets the size as a decoded one does
        for (uint32_t k = 0; k < nk; k++)
            if (hit[k] && is_last(k) && uns[P.stream[k]] == nk) IX(k).size = (int64_t)((IX(k).nblocks() - 1) * IX(k).block_size + blk_len[k]);
        if (ctx->profile) {
            const CacheStats& after = cache->pc.stats();
            auto& m = ctx->prof["read:cache_miss"];
            m.bytes_in += miss_blocks, m.bytes_out += miss_bytes, m.launches++;
            auto& i = ctx->prof["read:cache_insert"];
            i.bytes_in += after.inserts - before.inserts, i.bytes_out += ins_bytes, i.launches++;
            auto& v = ctx->prof["read:cache_evict"];
            v.bytes_in += after.evictions - before.evictions, v.bytes_out += before.resident + ins_bytes - after.resident, v.launches++;
        }
    }
    if (std::any_of(uns.begin(), uns.end(), [&](uint32_t u) { return u != nk; })) {
        ctx->err = "Invalid bitstream: a block before the last is not block_size bytes long";
        for (uint32_t k = 0; k < nk; k++)
            if (broken(k))
                for (uint64_t s = P.slice_of[k]; s < P.slice_of[k + 1]; s++)
                    if (!status[P.slices[s].req]) status[P.slices[s].req] = -KZ_ERR_INVALID_FILE;
    }
    for (uint32_t i = 0; i < nreq; i++)
        if (status[i]) out_len[i] = 0;
    // delivery of the staged requests: one transfer to the host, or one copy launch on the device
    if (host && stage_total) {
        std::vector<DownloadPiece> out;
        for (uint32_t i = 0; i < nreq; i++)
            if (!status[i] && out_len[i]) out.push_back(DownloadPiece{dst + dst_off[i], stage_at[i], out_len[i]});
        rc = download_pieces(ctx, ctx->d_asm.as<uint8_t>(), stage_total, out);
        if (rc) return rc;
    } else if (stage_total) {
        CopyList deliver;
        for (uint32_t i = 0; i < nreq; i++)
            if (staged[i] && !status[i]) deliver.add(ctx->d_asm.as<uint8_t>() + stage_at[i], dst + dst_off[i], out_len[i]);
        rc = run_copies(ctx, deliver);
        if (rc) return rc;
        CK(cudaStreamSynchronize(ctx->stream));
    }
    // A call whose blocks were all cached (or whose misses lie behind an unseekable block) has no decode pass and may have no staged
    // delivery: nothing above waited for the copies out of the cache. The bytes are complete, and a failed copy is reported, on return.
    if (hit_copies) CK(cudaStreamSynchronize(ctx->stream));
    if (ctx->profile) {
        auto& b = ctx->prof["read:blocks"];
        b.bytes_in += dec_blocks, b.bytes_out += dec_bytes, b.launches++;
        auto& o = ctx->prof["read:out"];
        o.bytes_in += out_slices, o.bytes_out += out_bytes, o.launches++;
    }
    return 0;
}

// The call-level checks of every read: no open session, the cache (if any) of this context, destinations that do not overflow.
int read_call_checks(kz_ctx* ctx, kz_cache* cache, uint32_t nreq, const uint64_t* len, const void* dst, const uint64_t* dst_off) {
    if (ctx->session) return ctx->fail(KZ_ERR_INVALID_PARAM, "a session is open on this context");
    if (cache && cache->ctx != ctx) return ctx->fail(KZ_ERR_INVALID_PARAM, "the block cache belongs to another context");
    for (uint32_t i = 0; i < nreq; i++) {
        if (dst_off[i] + len[i] < dst_off[i]) return ctx->fail(KZ_ERR_INVALID_PARAM, "offset + length overflows");
        if (len[i] && !dst) return ctx->fail(KZ_ERR_INVALID_PARAM, "null buffer");
    }
    return 0;
}

// Whether a stream of n bytes whose first min(n, 32) bytes are head (zero padded) is the one ix was built from, and whether the GPU path
// has its chain and codec: 0, or the code kz_read_ranges fails a read of it with.
int read_stream_check(kz_ctx* ctx, const kz_index* ix, uint64_t n, const uint8_t* head) {
    if (n != ix->stream_bytes) return ctx->fail(KZ_ERR_INVALID_PARAM, "the index was built from a stream of another length");
    if (memcmp(head, ix->head, INDEX_HEAD)) return ctx->fail(KZ_ERR_INVALID_PARAM, "the index was built from another stream");
    TransformPlan plan;
    int rc = plan_transforms(ctx, ix->t48, ix->etype, plan, KZ_ERR_CREATE_CODEC);
    if (rc) return rc;
    if (!etype_supported(ix->etype)) return ctx->fail(KZ_ERR_CREATE_CODEC, "entropy codec not available on the GPU path");
    return 0;
}

int read_ranges(kz_ctx* ctx, kz_index* ix, kz_cache* cache, const uint8_t* src, const void* d_src, size_t n, uint32_t nreq, const uint64_t* off,
                const uint64_t* len, void* dst, const uint64_t* dst_off, uint64_t* out_len, int32_t* status) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    const int rc = [&]() -> int {
        if (!ix || (!src && !d_src) || (nreq && (!off || !len || !dst_off || !out_len || !status))) return ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument");
        if (cudaSetDevice(ctx->device) != cudaSuccess) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "cudaSetDevice failed");
        int r = read_call_checks(ctx, cache, nreq, len, dst, dst_off);
        if (r) return r;
        if (!src && ((uintptr_t)d_src & 15)) return ctx->fail(KZ_ERR_INVALID_PARAM, "device buffers must be 16-byte aligned");
        // the stream the index was built from: its length and its leading bytes
        uint8_t head[INDEX_HEAD];
        const uint64_t at = 0, nh = n == ix->stream_bytes ? n : 0;
        if ((r = read_heads(ctx, src ? src : (const uint8_t*)d_src, !src, &at, &nh, 1, head))) return r;
        r = read_stream_check(ctx, ix, n, head);
        if (r) return r;
        return read_ranges_impl(ctx, cache, src, (const uint8_t*)d_src, {ReadSource{ix, 0, n}}, nreq, nullptr, off, len, (uint8_t*)dst, dst_off, out_len,
                                status);
    }();
    return finish_streams(nreq, status, out_len, rc);
}

// kz_read_ranges_streams[_device]: the streams the requests name are checked one by one (a failure fails that stream's requests only),
// then the requests on the streams that pass are served by one read_ranges_impl call.
int read_ranges_streams(kz_ctx* ctx, kz_cache* cache, uint32_t nstreams, kz_index* const* ix, const uint8_t* base, bool device, const uint64_t* src_off,
                        const uint64_t* src_len, uint32_t nreq, const uint32_t* req_stream, const uint64_t* off, const uint64_t* len, void* dst,
                        const uint64_t* dst_off, uint64_t* out_len, int32_t* status) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    const int rc = [&]() -> int {
        if (nreq && (!ix || !src_off || !src_len || !req_stream || !off || !len || !dst_off || !out_len || !status))
            return ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument");
        if (cudaSetDevice(ctx->device) != cudaSuccess) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "cudaSetDevice failed");
        int r = read_call_checks(ctx, cache, nreq, len, dst, dst_off);
        if (r) return r;
        std::vector<uint8_t> named(nstreams, 0);
        for (uint32_t i = 0; i < nreq; i++) {
            if (req_stream[i] >= nstreams) return ctx->fail(KZ_ERR_INVALID_PARAM, "a request names a stream past nstreams");
            named[req_stream[i]] = 1;
        }
        // the spans of the named streams, and their first 32 bytes (one device stream: copied straight back, as kz_read_ranges_device does)
        std::vector<uint32_t> names;
        std::vector<uint64_t> hoff, hlen;
        for (uint32_t s = 0; s < nstreams; s++)
            if (named[s]) names.push_back(s), hoff.push_back(src_off[s]), hlen.push_back(src_len[s]);
        const size_t nn = names.size();
        if ((r = check_spans(ctx, base, hoff.data(), hlen.data(), nn, device))) return r;
        std::vector<uint8_t> head(INDEX_HEAD * nn);
        if ((r = read_heads(ctx, base, device, hoff.data(), hlen.data(), nn, head.data()))) return r;
        // per stream: a missing or stale index or a chain without a GPU path fails the stream's requests with kz_read_ranges's code
        std::vector<int32_t> code(nstreams, 0);
        std::vector<uint32_t> slot(nstreams, 0);
        std::vector<ReadSource> S;
        for (size_t j = 0; j < nn; j++) {
            const uint32_t s = names[j];
            code[s] = ix[s] ? read_stream_check(ctx, ix[s], src_len[s], &head[INDEX_HEAD * j]) : ctx->fail(KZ_ERR_INVALID_PARAM, "missing index");
            if (!code[s]) slot[s] = (uint32_t)S.size(), S.push_back(ReadSource{ix[s], src_off[s], src_len[s]});
        }
        std::vector<uint32_t> keep, rs;
        std::vector<uint64_t> o, l, d;
        for (uint32_t i = 0; i < nreq; i++) {
            status[i] = code[req_stream[i]], out_len[i] = 0;
            if (status[i]) continue;
            keep.push_back(i), rs.push_back(slot[req_stream[i]]), o.push_back(off[i]), l.push_back(len[i]), d.push_back(dst_off[i]);
        }
        std::vector<uint64_t> kl(keep.size());
        std::vector<int32_t> ks(keep.size());
        r = read_ranges_impl(ctx, cache, device ? nullptr : base, device ? base : nullptr, S, (uint32_t)keep.size(), rs.data(), o.data(), l.data(),
                             (uint8_t*)dst, d.data(), kl.data(), ks.data());
        if (r) return r;
        for (size_t j = 0; j < keep.size(); j++) status[keep[j]] = ks[j], out_len[keep[j]] = kl[j];
        return 0;
    }();
    return finish_streams(nreq, status, out_len, rc);
}

// The indexes of the streams d_src + src_off[s] (src_len[s] bytes each, >= 64 readable bytes behind each), kz_index_build_device being
// the one-stream case: every header in one gather_heads, every stream's records in the two walk_streams launches of one build.
int index_build_streams(kz_ctx* ctx, uint32_t ns, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, kz_index** out, int32_t* status) {
    if (ctx->session) return ctx->fail(KZ_ERR_INVALID_PARAM, "a session is open on this context");
    std::vector<uint8_t> head(64 * (size_t)ns);
    int rc = gather_heads(ctx, d_src, src_off, src_len, ns, 64, head.data());
    if (rc) return rc;
    std::vector<StreamHeader> sh(ns);
    std::vector<WalkJob> wj;
    std::vector<uint32_t> who;
    for (uint32_t s = 0; s < ns; s++) {
        if ((status[s] = stream_header(ctx, &head[64 * (size_t)s], src_len[s], sh[s]))) continue;
        TransformPlan plan;
        if ((status[s] = plan_transforms(ctx, sh[s].t48, sh[s].etype, plan, KZ_ERR_CREATE_CODEC))) continue;
        if (!etype_supported(sh[s].etype)) {
            status[s] = ctx->fail(KZ_ERR_CREATE_CODEC, "entropy codec not available on the GPU path");
            continue;
        }
        who.push_back(s);
        wj.push_back(WalkJob{8 * src_off[s] + sh[s].bits, 8 * (src_off[s] + src_len[s]), 0, 0, 0});
    }
    // every record is kept, so the walk runs twice: once storing nothing (an empty block range) for the count, once to store them
    std::vector<Walked> w;
    if (!wj.empty()) {
        rc = walk_streams(ctx, (const uint32_t*)d_src, wj, 0, 1, w);
        if (rc) return rc;
    }
    std::vector<WalkJob> wj2;
    std::vector<uint32_t> who2;
    std::vector<Walked> w2;
    for (size_t j = 0; j < who.size(); j++) {
        const uint32_t s = who[j];
        if (w[j].status) status[s] = ctx->fail(-w[j].status, "Invalid bitstream: corrupted block length");
        else if (w[j].n) wj2.push_back(WalkJob{8 * src_off[s] + sh[s].bits, 8 * (src_off[s] + src_len[s]), 0, (uint32_t)w[j].n, 0}), who2.push_back(s);
    }
    if (!wj2.empty()) {
        rc = walk_streams(ctx, (const uint32_t*)d_src, wj2, -1, -1, w2);
        if (rc) return rc;
    }
    std::vector<std::unique_ptr<kz_index>> built(ns);
    size_t j2 = 0;
    for (size_t j = 0; j < who.size(); j++) {
        const uint32_t s = who[j];
        if (status[s]) continue;
        const Walked* ws = nullptr;
        if (w[j].n) {
            ws = &w2[j2++];
            if (ws->status) {
                status[s] = ctx->fail(-ws->status, "Invalid bitstream: corrupted block length");
                continue;
            }
        }
        std::unique_ptr<kz_index> ix(new kz_index());
        ix->t48 = sh[s].t48;
        ix->etype = sh[s].etype;
        ix->block_size = sh[s].block_size;
        ix->checksum_bits = sh[s].checksum_bits;
        ix->header_bits = (uint32_t)sh[s].bits;
        ix->input_size = sh[s].input_size;
        ix->stream_bytes = src_len[s];
        memcpy(ix->head, &head[64 * (size_t)s], INDEX_HEAD);
        if (ws) {
            ix->start = ws->bit_off;
            ix->bits = ws->bits;
            for (uint64_t& b : ix->start) b -= 8 * src_off[s];
        }
        ix->size = ix->start.empty() ? 0 : -1;
        if (!index_consistent(*ix)) status[s] = ctx->fail(KZ_ERR_INVALID_FILE, "Invalid bitstream: the records do not form an index");
        else built[s] = std::move(ix);
    }
    for (uint32_t s = 0; s < ns; s++) out[s] = built[s].release();
    return 0;
}

int check_index_streams_args(kz_ctx* ctx, uint32_t ns, const void* src, const uint64_t* src_off, const uint64_t* src_len, kz_index** out, int32_t* status,
                             bool device) {
    for (uint32_t s = 0; out && s < ns; s++) out[s] = nullptr;
    if (ns && (!src_off || !src_len || !out || !status)) return ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument array");
    return check_spans(ctx, src, src_off, src_len, ns, device);
}

// ---- writes into compressed streams (kz_write_ranges[_device], kz_write_ranges_streams[_device]; plan in kz_write_plan.h) ----------
// The blocks plan_writes_streams re-encodes go through the stages in passes of one group: the ones whose old bytes survive are decoded into
// their slots, the write slices and the zero gaps (copied from a zeroed area behind the slots) are copied over them by one launch, and the
// slots are encoded; every pass's records are packed into ctx->d_bits. One concat then lays out the tail of every new stream: the carry,
// the new records behind their prefixes, the old records behind them moved to their new bit (read where they lie, at any bit), and the
// end marker. An index is updated only when its slot succeeded.
// Host variant (src set): each slot's old stream from the first byte a record the call may read or move lies in, and the write bytes,
// go up in one transfer, and the tails come back in one. Device variant: d_src, d_data and dst are device memory.

// One slot of a write call: the stream ix was built from (n bytes at byte `at` of the source) and its output window.
struct WriteSlot {
    kz_index* ix;
    uint64_t at, n, dst_off, cap;
};

// The writes i (write i to slot w_slot[i], null: every write to S[0]) on slots that passed their checks. keep, out_n and status are per
// slot; each slot gets what a call on it alone gives. The return value is a call-level failure (CUDA, allocation, an encode failure).
int write_ranges_impl(kz_ctx* ctx, const uint8_t* src, const uint8_t* d_src, const std::vector<WriteSlot>& S, uint32_t nw, const uint32_t* w_slot,
                      const uint64_t* off, const uint64_t* len, const uint8_t* data, const uint64_t* data_off, uint8_t* dst, uint64_t* keep,
                      uint64_t* out_n, int32_t* status) {
    const bool host = src != nullptr;
    const uint32_t ns = (uint32_t)S.size();
    auto slot_of = [&](uint32_t i) { return w_slot ? w_slot[i] : 0u; };
    for (uint32_t s = 0; s < ns; s++) keep[s] = S[s].n, out_n[s] = 0, status[s] = 0;
    // groups, numbered in the order they first appear: the header, transform plan and encode cost of each
    std::map<std::tuple<uint64_t, uint32_t, uint32_t, uint32_t>, uint32_t> group_of;
    std::vector<StreamHeader> gsh;
    std::vector<TransformPlan> gplan;
    std::vector<uint64_t> gcost;
    std::vector<StreamIndex> X(ns);  // what the plan knows; the indexes change only on success
    std::vector<WriteStream> WS(ns);
    for (uint32_t s = 0; s < ns; s++) {
        const kz_index& ix = *S[s].ix;
        const auto key = std::make_tuple(ix.t48, ix.etype, ix.block_size, ix.checksum_bits);
        auto it = group_of.find(key);
        if (it == group_of.end()) {
            it = group_of.emplace(key, (uint32_t)gsh.size()).first;
            gsh.push_back(index_header(ix));
            gplan.emplace_back();
            int rc = plan_transforms(ctx, ix.t48, ix.etype, gplan.back(), KZ_ERR_CREATE_CODEC);
            if (rc) return rc;
            gcost.push_back(compress_block_cost(round16(ix.block_size), entropy_scratch(ix.etype)));
        }
        X[s] = ix;
        WS[s] = WriteStream{&X[s], it->second, gcost[it->second]};
    }
    // live[s]: the slot still makes a new tail; a failed slot, or one whose writes change nothing, takes no further part
    std::vector<uint8_t> live(ns, 0), need(ns, 0);
    auto fail = [&](uint32_t s, int code) {
        status[s] = code;
        live[s] = 0;
        WS[s].x = nullptr;
    };
    WriteStreamsPlan W = plan_writes_streams(WS, nw, w_slot, off, len);
    std::vector<uint64_t> low(ns, 0);  // with the size to learn: the first block a write names, or the last block
    for (uint32_t s = 0; s < ns; s++) {
        const WritePlan& P = W.plans[s];
        low[s] = X[s].nblocks() ? X[s].nblocks() - 1 : 0;
        if (P.status == WRITE_TOO_LARGE) fail(s, ctx->fail(KZ_ERR_INVALID_PARAM, "the data would grow past what an index holds"));
        else if (P.status == WRITE_NEED_SIZE) live[s] = need[s] = 1;
        else if (P.nothing()) WS[s].x = nullptr;
        else live[s] = 1;
    }
    if (!std::count(live.begin(), live.end(), 1)) return 0;
    for (uint32_t i = 0; i < nw; i++) {
        const uint32_t s = slot_of(i);
        if (need[s] && len[i] && off[i] != WRITE_APPEND) low[s] = std::min<uint64_t>(low[s], off[i] / X[s].block_size);
    }
    // the old streams and the write bytes on the device: slot s's stream bit b lies at bit b + org[s] of d_words, write i at d_wdata + w_at[i]
    std::vector<uint64_t> org(ns, 0), w_at(nw, 0);
    const uint8_t* d_words = d_src;
    const uint8_t* d_wdata = data;
    uint64_t words_bytes = 0;
    if (host) {
        std::vector<UploadPiece> up;
        std::vector<uint32_t> up_slot;
        uint64_t pieces = 0, bytes = 0;
        for (uint32_t s = 0; s < ns; s++) {
            if (!live[s]) continue;
            const uint64_t ubase = ((need[s] ? record_prefix_bit(X[s], low[s]) : W.plans[s].cut) / 8) & ~15ull, tail = S[s].n - ubase;
            org[s] = 0 - 8 * ubase;  // + 8 * (its offset in d_in), below
            up.push_back(UploadPiece{src + S[s].at + ubase, tail, tail + 128}), up_slot.push_back(s);
            pieces += tail ? 1 : 0, bytes += tail;
        }
        const size_t nslots = up.size();
        uint64_t wtotal = 0;
        for (uint32_t i = 0; i < nw; i++)
            if (len[i] && live[slot_of(i)]) up.push_back(UploadPiece{data + data_off[i], len[i], len[i]}), wtotal += len[i];
        std::vector<uint64_t> at;
        int rc = upload_pieces(ctx, up, at, &words_bytes);
        if (rc) return rc;
        for (size_t k = 0; k < nslots; k++) org[up_slot[k]] += 8 * at[k];
        for (uint32_t i = 0, k = (uint32_t)nslots; i < nw; i++)
            if (len[i] && live[slot_of(i)]) w_at[i] = at[k++];
        d_words = d_wdata = ctx->d_in.as<uint8_t>();
        if (ctx->profile) {
            auto& e = ctx->prof["write:h2d"];
            e.bytes_in += pieces + (wtotal ? 1 : 0), e.bytes_out += bytes + wtotal, e.launches++;
        }
    } else {
        for (uint32_t s = 0; s < ns; s++) org[s] = 8 * S[s].at, words_bytes = std::max(words_bytes, S[s].at + S[s].n);
        for (uint32_t i = 0; i < nw; i++) w_at[i] = len[i] ? data_off[i] : 0;
    }
    const uint32_t* d_w32 = (const uint32_t*)d_words;
    const uint64_t words_len = (words_bytes + 3) / 4 + 16;
    auto job_of = [&](uint32_t s, uint64_t b) {
        DecJob j = DecJob();
        j.bit_off = X[s].start[b] + org[s];
        j.bits = X[s].bits[b];
        j.block_size = X[s].block_size;
        return j;
    };
    // the failure of decoded block b of slot s: its own code, or a length that breaks the block arithmetic
    auto check_decoded = [&](uint32_t s, uint64_t b, const DecodeFailure& f, uint32_t m) {
        const uint64_t nb = X[s].nblocks(), bs = X[s].block_size;
        if (m > bs || (!f.failed() && (b + 1 == nb ? m == 0 || (X[s].size >= 0 && m != (uint64_t)X[s].size - (nb - 1) * bs) : m != bs)))
            return ctx->fail(KZ_ERR_INVALID_FILE, "Invalid bitstream: a block before the last is not block_size bytes long");
        if (f.failed()) return ctx->fail(-f.code, f.msg);
        return 0;
    };
    std::vector<uint64_t> dec_blocks(ns, 0), dec_bytes(ns, 0);
    // slots whose size the result depends on: their old last blocks decoded, group by group in passes, packed into ctx->d_out at
    // learned[s], where the encode passes copy them from
    std::vector<uint64_t> learned(ns, NO_ROOM);
    if (std::count(need.begin(), need.end(), 1)) {
        uint64_t used = 0;
        for (uint32_t g = 0; g < (uint32_t)gsh.size(); g++) {
            std::vector<uint32_t> ss;
            for (uint32_t s = 0; s < ns; s++)
                if (need[s] && live[s] && WS[s].group == g) ss.push_back(s);
            if (ss.empty()) continue;
            const uint32_t bs = gsh[g].block_size;
            const PassPlan pp = plan_decompress_passes((uint32_t)ss.size(), decompress_slot(bs), read_block_cost(bs));
            for (uint32_t p = 0; p < pp.npasses(); p++) {
                const uint32_t a = pp.first[p], k = pp.first[p + 1] - a;
                int rc = grow_keeping(ctx, ctx->d_out, used, used + k * decompress_slot(bs));
                if (rc) return rc;
                std::vector<DecJob> jobs;
                for (uint32_t i = a; i < a + k; i++) jobs.push_back(job_of(ss[i], X[ss[i]].nblocks() - 1));
                std::vector<uint64_t> at(k, NO_ROOM);  // a block decoded again alone keeps the place it was first given
                std::vector<DecodeFailure> fl;
                std::vector<uint32_t> olen;
                rc = decode_isolated(ctx, gsh[g], gplan[g], d_w32, words_len, jobs, std::vector<uint8_t>(k, 1),
                                     [&](uint32_t i, uint32_t m) {
                                         if (m > bs) return NO_ROOM;
                                         if (at[i] == NO_ROOM) at[i] = used, used += round16(m);
                                         return at[i];
                                     },
                                     ctx->d_out.as<uint8_t>(), fl, olen);
                if (rc) return rc;
                for (uint32_t i = 0; i < k; i++) {
                    const uint32_t s = ss[a + i];
                    const uint64_t nb = X[s].nblocks();
                    if ((rc = check_decoded(s, nb - 1, fl[i], olen[i]))) {
                        fail(s, rc);
                        continue;
                    }
                    X[s].size = (int64_t)((nb - 1) * bs + olen[i]);
                    learned[s] = at[i];
                    dec_blocks[s]++, dec_bytes[s] += olen[i];
                }
            }
        }
        W = plan_writes_streams(WS, nw, w_slot, off, len);
        for (uint32_t s = 0; s < ns; s++) {
            if (!need[s] || !live[s]) continue;
            if (W.plans[s].status != WRITE_OK) fail(s, ctx->fail(KZ_ERR_INVALID_PARAM, "the data would grow past what an index holds"));
            else if (W.plans[s].nothing()) live[s] = 0;
        }
    }
    // passes: decode, apply the writes, encode; each pass's records packed into ctx->d_bits as records of their pairs
    const uint32_t npairs = (uint32_t)W.stream.size();
    RecordArena arena(npairs);
    std::vector<uint64_t> enc_bytes(ns, 0);
    for (uint32_t p = 0; p < W.npasses(); p++) {
        const uint32_t a = W.first[p], k = W.first[p + 1] - a;
        const uint32_t g = WS[W.stream[a]].group, bs = gsh[g].block_size;
        const uint64_t astride = decompress_slot(bs);
        uint32_t zmax = 0;  // the longest zero gap of the pass: the zeroed area behind the slots
        bool any = false;
        for (uint32_t i = a; i < a + k; i++) {
            const uint32_t s = W.stream[i];
            if (!live[s]) continue;
            any = true;
            const WritePlan& P = W.plans[s];
            for (uint64_t q = P.piece_of[W.enc[i]]; q < P.piece_of[W.enc[i] + 1]; q++)
                if (P.pieces[q].kind == PIECE_ZERO) zmax = std::max(zmax, P.pieces[q].len);
        }
        if (!any) continue;
        CK(ctx->d_slots.ensure(astride * k + zmax + 64));
        uint8_t* slots = ctx->d_slots.as<uint8_t>();
        uint8_t* zero = slots + astride * k;
        if (zmax) CK(cudaMemsetAsync(zero, 0, zmax, ctx->stream));
        std::vector<uint32_t> who;
        std::vector<DecJob> jobs;
        std::vector<uint8_t> last;
        CopyList fill;
        for (uint32_t i = a; i < a + k; i++) {
            const uint32_t s = W.stream[i], j = W.enc[i];
            const WritePlan& P = W.plans[s];
            if (!live[s] || !P.decode[j]) continue;
            const uint64_t b = P.enc[j], nb = X[s].nblocks();
            if (learned[s] != NO_ROOM && b + 1 == nb) {
                // only the old bytes that survive: the write and zero copies of the same launch cover the rest, and copies of one launch
                // run in no particular order
                for (uint64_t q = P.piece_of[j]; q < P.piece_of[j + 1]; q++)
                    if (P.pieces[q].kind == PIECE_OLD)
                        fill.add(ctx->d_out.as<uint8_t>() + learned[s] + P.pieces[q].at, slots + (uint64_t)(i - a) * astride + P.pieces[q].at,
                                 P.pieces[q].len);
                continue;
            }
            who.push_back(i), jobs.push_back(job_of(s, b)), last.push_back(b + 1 == nb);
        }
        if (!jobs.empty()) {
            std::vector<DecodeFailure> fl;
            std::vector<uint32_t> olen;
            int rc = decode_isolated(ctx, gsh[g], gplan[g], d_w32, words_len, jobs, last,
                                     [&](uint32_t q, uint32_t m) { return m > bs ? NO_ROOM : (uint64_t)(who[q] - a) * astride; }, slots, fl, olen);
            if (rc) return rc;
            // a slot's first failing block in block order decides its code, as in a call on it alone
            for (size_t q = 0; q < who.size(); q++) {
                const uint32_t s = W.stream[who[q]];
                if (!live[s]) continue;
                if ((rc = check_decoded(s, W.plans[s].enc[W.enc[who[q]]], fl[q], olen[q]))) fail(s, rc);
                else dec_blocks[s]++, dec_bytes[s] += olen[q];
            }
        }
        any = false;
        for (uint32_t i = a; i < a + k; i++) {
            const uint32_t s = W.stream[i];
            if (!live[s]) continue;
            any = true;
            const WritePlan& P = W.plans[s];
            for (uint64_t q = P.piece_of[W.enc[i]]; q < P.piece_of[W.enc[i] + 1]; q++) {
                const WritePiece& pc = P.pieces[q];
                uint8_t* to = slots + (uint64_t)(i - a) * astride + pc.at;
                if (pc.kind == PIECE_WRITE) fill.add(d_wdata + w_at[pc.write] + pc.from, to, pc.len);
                else if (pc.kind == PIECE_ZERO) fill.add(zero, to, pc.len);
            }
        }
        if (!any) {  // every slot of the pass failed: nothing to encode
            CK(cudaStreamSynchronize(ctx->stream));
            continue;
        }
        int rc = run_copies(ctx, fill);
        if (rc) return rc;
        BlockList bl;
        std::vector<uint32_t> lens(k), rec(k);
        for (uint32_t i = 0; i < k; i++) {
            const uint32_t s = W.stream[a + i];
            lens[i] = W.plans[s].enc_len[W.enc[a + i]];
            bl.off.push_back((uint64_t)i * astride), bl.len.push_back(lens[i]);
            rec[i] = a + i;
            enc_bytes[s] += lens[i];
        }
        bl.first = {0, k};
        BlockPrep prep;
        if ((rc = prepare_blocks(ctx, gplan[g], ctx->skip_blocks, gsh[g].checksum_bits, slots, bl, prep))) return rc;
        rc = arena.encode_pass(ctx, gplan[g], gsh[g].etype, gsh[g].checksum_bits, slots, astride, lens, std::vector<uint64_t>(k, bs), prep, rec.data());
        if (rc) return rc;
        CK(cudaStreamSynchronize(ctx->stream));  // the slots and the copy lists are reused by the next pass
    }
    // the new record tables, then every tail: one concat of the segments behind byte floor(cut / 8) of each slot, the tail of slot s at
    // dst + dst_off[s] (host variant: at stage_at[s] of ctx->d_out)
    std::vector<uint8_t> pre(8 * (size_t)npairs, 0);
    std::vector<uint32_t> pre_bits(npairs, 0);
    std::vector<StreamIndex> Y(ns);
    std::vector<uint64_t> kp(ns, 0), tail_bytes(ns, 0), stage_at(ns, 0), moved_runs(ns, 0), moved_bits(ns, 0);
    uint64_t stage_total = 0;
    SegmentList sl;
    for (uint32_t s = 0; s < ns; s++) {
        if (!live[s]) continue;
        const WritePlan& P = W.plans[s];
        const uint64_t base = W.pair_of[s], ne = P.enc.size();
        std::vector<uint64_t> bits(ne);
        std::vector<uint32_t> pb(ne);
        for (uint64_t j = 0; j < ne; j++) bits[j] = arena.bits[base + j], pb[j] = pre_bits[base + j] = write_block_prefix(&pre[8 * (base + j)], bits[j]);
        const uint64_t total_bits = splice_records(X[s], P, bits, pb, END_MARKER_BITS, Y[s]);
        kp[s] = P.cut / 8;
        const uint64_t tail_bits = total_bits - 8 * kp[s];
        tail_bytes[s] = (tail_bits + 7) / 8;
        const uint64_t need_cap = (tail_bits + 31) / 32 * 4;  // the concat writes whole 32-bit words
        if (need_cap > S[s].cap) {
            out_n[s] = need_cap;
            fail(s, ctx->fail(KZ_ERR_WRITE_FILE, "output buffer too small"));
            continue;
        }
        if (!dst) {
            fail(s, ctx->fail(KZ_ERR_INVALID_PARAM, "null buffer"));
            continue;
        }
        stage_at[s] = stage_total, stage_total += round16(need_cap);
        sl.at(8 * (host ? stage_at[s] : S[s].dst_off));
        for (const WriteSeg& sg : P.segs) {
            if (sg.kind == SEG_CARRY) {
                sl.add_device(d_words, sg.bit + org[s], sg.bits);
            } else if (sg.kind == SEG_NEW) {
                for (uint64_t j = base + sg.first; j < base + sg.first + sg.count; j++) {
                    sl.add_host(&pre[8 * j], pre_bits[j]);
                    sl.add_device(arena.record(ctx, j), 0, arena.bits[j]);
                }
            } else if (sg.kind == SEG_OLD) {
                sl.add_device(d_words, sg.bit + org[s], sg.bits);
                moved_runs[s]++, moved_bits[s] += sg.bits;
            } else {
                sl.add_end_marker();
            }
        }
    }
    if (!std::count(live.begin(), live.end(), 1)) return 0;
    uint8_t* d_out = dst;
    if (host) {
        CK(ctx->d_out.ensure(stage_total + 64));
        d_out = ctx->d_out.as<uint8_t>();
    }
    int rc = sl.write(ctx, d_out);
    if (rc) return rc;
    // each new stream's first 32 bytes: the old ones before floor(cut / 8), the tail's behind it
    auto nlead = [&](uint32_t s) { return kp[s] < INDEX_HEAD ? std::min<uint64_t>(INDEX_HEAD - kp[s], tail_bytes[s]) : 0; };
    std::vector<uint8_t> lead(INDEX_HEAD * (size_t)ns, 0);
    if (host) {
        std::vector<DownloadPiece> down;
        for (uint32_t s = 0; s < ns; s++)
            if (live[s]) down.push_back(DownloadPiece{dst + S[s].dst_off, stage_at[s], tail_bytes[s]});
        if ((rc = download_pieces(ctx, d_out, stage_total, down))) return rc;
        for (uint32_t s = 0; s < ns; s++)
            if (live[s]) memcpy(&lead[INDEX_HEAD * (size_t)s], dst + S[s].dst_off, nlead(s));
    } else {
        std::vector<uint32_t> ls;
        std::vector<uint64_t> loff, llen;
        for (uint32_t s = 0; s < ns; s++)
            if (live[s] && nlead(s)) ls.push_back(s), loff.push_back(S[s].dst_off), llen.push_back(nlead(s));
        std::vector<uint8_t> got(INDEX_HEAD * ls.size());
        if ((rc = gather_heads(ctx, d_out, loff.data(), llen.data(), ls.size(), (uint32_t)INDEX_HEAD, got.data()))) return rc;
        for (size_t q = 0; q < ls.size(); q++) memcpy(&lead[INDEX_HEAD * (size_t)ls[q]], &got[INDEX_HEAD * q], INDEX_HEAD);
    }
    uint64_t dec_b = 0, dec_n = 0, enc_b = 0, enc_n = 0, mv_r = 0, mv_b = 0;
    for (uint32_t s = 0; s < ns; s++) {
        if (!live[s]) continue;
        StreamIndex& y = Y[s];
        const uint64_t h = std::min<uint64_t>(kp[s], INDEX_HEAD);
        memset(y.head + h, 0, INDEX_HEAD - h);
        memcpy(y.head + h, &lead[INDEX_HEAD * (size_t)s], nlead(s));
        static_cast<StreamIndex&>(*S[s].ix) = y;
        keep[s] = kp[s];
        out_n[s] = tail_bytes[s];
        dec_b += dec_blocks[s], dec_n += dec_bytes[s], enc_b += W.plans[s].enc.size(), enc_n += enc_bytes[s], mv_r += moved_runs[s], mv_b += moved_bits[s];
    }
    if (ctx->profile) {
        auto note = [&](const char* name, uint64_t a, uint64_t b) {
            auto& e = ctx->prof[name];
            e.bytes_in += a, e.bytes_out += b, e.launches++;
        };
        note("write:decoded", dec_b, dec_n);
        note("write:encoded", enc_b, enc_n);
        note("write:moved", mv_r, mv_b);
    }
    return 0;
}

// kz_write_ranges[_device]: the one-slot case of write_ranges_impl, behind its own checks.
int write_ranges(kz_ctx* ctx, kz_index* ix, const uint8_t* src, const uint8_t* d_src, size_t n, uint32_t nw, const uint64_t* off, const uint64_t* len,
                 const uint8_t* data, const uint64_t* data_off, uint8_t* dst, size_t cap, uint64_t* keep, size_t* out_n) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    if (!ix || !keep || !out_n || (!src && !d_src) || (nw && (!off || !len))) return ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument");
    *keep = n;
    *out_n = 0;
    const bool host = src != nullptr;
    CK(cudaSetDevice(ctx->device));
    if (ctx->session) return ctx->fail(KZ_ERR_INVALID_PARAM, "a session is open on this context");
    for (uint32_t i = 0; i < nw; i++) {
        if (!len[i]) continue;
        if (!data || !data_off) return ctx->fail(KZ_ERR_INVALID_PARAM, "null buffer");
        if (data_off[i] + len[i] < data_off[i]) return ctx->fail(KZ_ERR_INVALID_PARAM, "offset + length overflows");
    }
    if (!host && (((uintptr_t)d_src & 15) || ((uintptr_t)dst & 15))) return ctx->fail(KZ_ERR_INVALID_PARAM, "device buffers must be 16-byte aligned");
    if (!host && dst && dst < d_src + n && d_src < dst + cap) return ctx->fail(KZ_ERR_INVALID_PARAM, "the output overlaps the stream");
    uint8_t head[INDEX_HEAD];
    const uint64_t at0 = 0, nh = n == ix->stream_bytes ? n : 0;
    int rc = read_heads(ctx, host ? src : d_src, !host, &at0, &nh, 1, head);
    if (rc || (rc = read_stream_check(ctx, ix, n, head))) return rc;
    uint64_t k = n, o = 0;
    int32_t st = 0;
    rc = write_ranges_impl(ctx, src, d_src, {WriteSlot{ix, 0, n, 0, cap}}, nw, nullptr, off, len, data, data_off, dst, &k, &o, &st);
    if (rc) return rc;
    *keep = k;
    *out_n = (size_t)o;
    return st;
}

// kz_write_ranges_streams[_device]: the call-level checks, then each slot a write names checked against its own bytes (a failure fails
// that slot only), then the writes on the slots that pass served by one write_ranges_impl call.
int write_ranges_streams(kz_ctx* ctx, uint32_t nstreams, kz_index* const* ix, const uint8_t* base, bool device, const uint64_t* src_off,
                         const uint64_t* src_len, uint32_t nw, const uint32_t* w_stream, const uint64_t* off, const uint64_t* len, const uint8_t* data,
                         const uint64_t* data_off, uint8_t* dst, const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* keep, uint64_t* out_n,
                         int32_t* status) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    const int rc = [&]() -> int {
        if (nstreams && (!keep || !out_n || !status)) return ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument");
        for (uint32_t s = 0; s < nstreams; s++) keep[s] = src_len ? src_len[s] : 0, out_n[s] = 0, status[s] = 0;
        if (nw && (!ix || !src_off || !src_len || !w_stream || !off || !len || !dst_off || !dst_cap))
            return ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument");
        if (cudaSetDevice(ctx->device) != cudaSuccess) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "cudaSetDevice failed");
        if (ctx->session) return ctx->fail(KZ_ERR_INVALID_PARAM, "a session is open on this context");
        std::vector<uint8_t> named(nstreams, 0);
        for (uint32_t i = 0; i < nw; i++) {
            if (w_stream[i] >= nstreams) return ctx->fail(KZ_ERR_INVALID_PARAM, "a write names a stream past nstreams");
            if (!len[i]) continue;
            if (!data || !data_off) return ctx->fail(KZ_ERR_INVALID_PARAM, "null buffer");
            if (data_off[i] + len[i] < data_off[i]) return ctx->fail(KZ_ERR_INVALID_PARAM, "offset + length overflows");
            named[w_stream[i]] = 1;
        }
        std::vector<uint32_t> names;
        std::vector<uint64_t> hoff, hlen;
        std::set<const kz_index*> seen;
        for (uint32_t s = 0; s < nstreams; s++) {
            if (!named[s]) continue;
            if (ix[s] && !seen.insert(ix[s]).second) return ctx->fail(KZ_ERR_INVALID_PARAM, "one index in two slots that writes name");
            if (dst_off[s] + dst_cap[s] < dst_off[s]) return ctx->fail(KZ_ERR_INVALID_PARAM, "offset + length overflows");
            if (dst_cap[s] && !dst) return ctx->fail(KZ_ERR_INVALID_PARAM, "null buffer");
            if (device && (dst_off[s] & 15)) return ctx->fail(KZ_ERR_INVALID_PARAM, "device offsets must be multiples of 16");
            names.push_back(s), hoff.push_back(src_off[s]), hlen.push_back(src_len[s]);
        }
        const size_t nn = names.size();
        if (!nn) return 0;  // no slot is named: no buffer is read or written, so none is checked
        int r = check_spans(ctx, base, hoff.data(), hlen.data(), nn, device);
        if (r) return r;
        if (device) {
            if ((uintptr_t)dst & 15) return ctx->fail(KZ_ERR_INVALID_PARAM, "device buffers must be 16-byte aligned");
            // the output windows may overlap neither each other nor a named stream: a sweep over both, ordered by first address
            struct Span {
                uintptr_t a, e;
                bool window;
            };
            std::vector<Span> sp;
            for (uint32_t s : names) {
                if (dst_cap[s]) sp.push_back(Span{(uintptr_t)dst + dst_off[s], (uintptr_t)dst + dst_off[s] + dst_cap[s], true});
                if (src_len[s]) sp.push_back(Span{(uintptr_t)base + src_off[s], (uintptr_t)base + src_off[s] + src_len[s], false});
            }
            std::sort(sp.begin(), sp.end(), [](const Span& x, const Span& y) { return x.a < y.a; });
            uintptr_t wend = 0, send = 0;
            for (const Span& x : sp) {
                if (x.a < wend || (x.window && x.a < send)) return ctx->fail(KZ_ERR_INVALID_PARAM, "an output window overlaps another or a stream");
                if (x.window) wend = std::max(wend, x.e);
                else send = std::max(send, x.e);
            }
        }
        std::vector<uint8_t> head(INDEX_HEAD * nn);
        if ((r = read_heads(ctx, base, device, hoff.data(), hlen.data(), nn, head.data()))) return r;
        // per slot: a missing or stale index or a chain without a GPU path fails the slot with kz_write_ranges's code
        std::vector<uint32_t> slot(nstreams, 0);
        std::vector<WriteSlot> S;
        std::vector<uint32_t> who;
        for (size_t j = 0; j < nn; j++) {
            const uint32_t s = names[j];
            status[s] = ix[s] ? read_stream_check(ctx, ix[s], src_len[s], &head[INDEX_HEAD * j]) : ctx->fail(KZ_ERR_INVALID_PARAM, "missing index");
            if (!status[s]) slot[s] = (uint32_t)S.size(), S.push_back(WriteSlot{ix[s], src_off[s], src_len[s], dst_off[s], dst_cap[s]}), who.push_back(s);
        }
        std::vector<uint32_t> ws;
        std::vector<uint64_t> o, l, d;
        for (uint32_t i = 0; i < nw; i++)
            if (len[i] && !status[w_stream[i]]) ws.push_back(slot[w_stream[i]]), o.push_back(off[i]), l.push_back(len[i]), d.push_back(data_off[i]);
        std::vector<uint64_t> k(S.size()), on(S.size());
        std::vector<int32_t> st(S.size());
        r = write_ranges_impl(ctx, device ? nullptr : base, device ? base : nullptr, S, (uint32_t)ws.size(), ws.data(), o.data(), l.data(), data,
                              d.data(), dst, k.data(), on.data(), st.data());
        if (r) return r;
        for (size_t j = 0; j < S.size(); j++) keep[who[j]] = k[j], out_n[who[j]] = on[j], status[who[j]] = st[j];
        return 0;
    }();
    return finish_streams(nstreams, status, out_n, rc);
}

}  // namespace

extern "C" {

int kz_index_build_device(kz_ctx* ctx, const void* d_src, size_t n, kz_index** out) {
    if (int rc = after_caller_work(ctx)) return rc;
    if (!ctx || !out || (!d_src && n)) return -KZ_ERR_INVALID_PARAM;
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    if (ctx->session) return ctx->fail(KZ_ERR_INVALID_PARAM, "a session is open on this context");
    if ((uintptr_t)d_src & 15) return ctx->fail(KZ_ERR_INVALID_PARAM, "device buffers must be 16-byte aligned");
    const uint64_t off = 0, len = n;
    int32_t status = 0;
    const int rc = index_build_streams(ctx, 1, (const uint8_t*)d_src, &off, &len, out, &status);
    return rc ? rc : status;
}

int kz_index_build(kz_ctx* ctx, const uint8_t* src, size_t n, kz_index** out) {
    if (!ctx || !out || !src) return -KZ_ERR_INVALID_PARAM;
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    CK(ctx->d_in.ensure(n + 128));
    CK(cudaMemsetAsync((uint8_t*)ctx->d_in.p + (n & ~size_t(3)), 0, 128, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_in.p, src, n, cudaMemcpyHostToDevice, ctx->stream));
    return kz_index_build_device(ctx, ctx->d_in.p, n, out);
}

int kz_index_info(const kz_index* ix, uint64_t* t48, uint32_t* etype, uint32_t* block_size, uint32_t* checksum_bits, int64_t* input_size,
                  uint64_t* nblocks, uint64_t* stream_bytes, int64_t* size) {
    if (!ix) return -KZ_ERR_INVALID_PARAM;
    if (t48) *t48 = ix->t48;
    if (etype) *etype = ix->etype;
    if (block_size) *block_size = ix->block_size;
    if (checksum_bits) *checksum_bits = ix->checksum_bits;
    if (input_size) *input_size = ix->input_size;
    if (nblocks) *nblocks = ix->nblocks();
    if (stream_bytes) *stream_bytes = ix->stream_bytes;
    if (size) *size = ix->size;
    return 0;
}

size_t kz_index_save(const kz_index* ix, uint8_t* dst, size_t cap) {
    if (!ix) return 0;
    const size_t need = index_blob_bytes(ix->nblocks());
    if (dst && cap >= need) index_save(*ix, dst);
    return need;
}

int kz_index_load(const uint8_t* blob, size_t n, kz_index** out) {
    if (!out) return -KZ_ERR_INVALID_PARAM;
    *out = nullptr;
    std::unique_ptr<kz_index> ix(new kz_index());
    if (!index_load(blob, n, *ix)) return -KZ_ERR_INVALID_FILE;
    *out = ix.release();
    return 0;
}

void kz_index_free(kz_index* ix) { delete ix; }

int kz_read_ranges(kz_ctx* ctx, kz_index* ix, const uint8_t* src, size_t n, uint32_t nreq, const uint64_t* off, const uint64_t* len, uint8_t* dst,
                   const uint64_t* dst_off, uint64_t* out_len, int32_t* status) {
    return read_ranges(ctx, ix, nullptr, src, nullptr, n, nreq, off, len, dst, dst_off, out_len, status);
}

int kz_read_ranges_device(kz_ctx* ctx, kz_index* ix, const void* d_src, size_t n, uint32_t nreq, const uint64_t* off, const uint64_t* len, void* d_dst,
                          const uint64_t* dst_off, uint64_t* out_len, int32_t* status) {
    if (int rc = after_caller_work(ctx)) return finish_streams(nreq, status, out_len, rc);
    return read_ranges(ctx, ix, nullptr, nullptr, d_src, n, nreq, off, len, d_dst, dst_off, out_len, status);
}

int kz_write_ranges(kz_ctx* ctx, kz_index* ix, const uint8_t* src, size_t n, uint32_t nw, const uint64_t* off, const uint64_t* len, const uint8_t* data,
                    const uint64_t* data_off, uint8_t* dst, size_t cap, uint64_t* keep, size_t* out_n) {
    if (!src) return ctx ? ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument") : -KZ_ERR_INVALID_PARAM;
    return write_ranges(ctx, ix, src, nullptr, n, nw, off, len, data, data_off, dst, cap, keep, out_n);
}

int kz_write_ranges_device(kz_ctx* ctx, kz_index* ix, const void* d_src, size_t n, uint32_t nw, const uint64_t* off, const uint64_t* len,
                           const void* d_data, const uint64_t* data_off, void* d_dst, size_t cap, uint64_t* keep, size_t* out_n) {
    if (int rc = after_caller_work(ctx)) return rc;
    if (!d_src) return ctx ? ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument") : -KZ_ERR_INVALID_PARAM;
    return write_ranges(ctx, ix, nullptr, (const uint8_t*)d_src, n, nw, off, len, (const uint8_t*)d_data, data_off, (uint8_t*)d_dst, cap, keep, out_n);
}

int kz_write_ranges_streams(kz_ctx* ctx, uint32_t nstreams, kz_index* const* ix, const uint8_t* src, const uint64_t* src_off, const uint64_t* src_len,
                            uint32_t nw, const uint32_t* w_stream, const uint64_t* off, const uint64_t* len, const uint8_t* data, const uint64_t* data_off,
                            uint8_t* dst, const uint64_t* dst_off, const uint64_t* dst_cap, uint64_t* keep, uint64_t* out_n, int32_t* status) {
    return write_ranges_streams(ctx, nstreams, ix, src, false, src_off, src_len, nw, w_stream, off, len, data, data_off, dst, dst_off, dst_cap, keep, out_n,
                                status);
}

int kz_write_ranges_streams_device(kz_ctx* ctx, uint32_t nstreams, kz_index* const* ix, const void* d_src, const uint64_t* src_off,
                                   const uint64_t* src_len, uint32_t nw, const uint32_t* w_stream, const uint64_t* off, const uint64_t* len,
                                   const void* d_data, const uint64_t* data_off, void* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                                   uint64_t* keep, uint64_t* out_n, int32_t* status) {
    if (int rc = after_caller_work(ctx)) return finish_streams(nstreams, status, out_n, rc);
    return write_ranges_streams(ctx, nstreams, ix, (const uint8_t*)d_src, true, src_off, src_len, nw, w_stream, off, len, (const uint8_t*)d_data, data_off,
                                (uint8_t*)d_dst, dst_off, dst_cap, keep, out_n, status);
}

// ---- many streams per call (kz_index_build_streams[_device], kz_read_ranges_streams[_device]) ----------------------------------------
int kz_index_build_streams_device(kz_ctx* ctx, uint32_t nstreams, const void* d_src, const uint64_t* src_off, const uint64_t* src_len, kz_index** out,
                                  int32_t* status) {
    if (int rc = after_caller_work(ctx)) return finish_streams(nstreams, status, nullptr, rc);
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    int rc = check_index_streams_args(ctx, nstreams, d_src, src_off, src_len, out, status, true);
    if (!rc && cudaSetDevice(ctx->device) != cudaSuccess) rc = ctx->fail(KZ_ERR_PROCESS_BLOCK, "cudaSetDevice failed");
    if (!rc) rc = index_build_streams(ctx, nstreams, (const uint8_t*)d_src, src_off, src_len, out, status);
    return finish_streams(nstreams, status, nullptr, rc);
}

int kz_index_build_streams(kz_ctx* ctx, uint32_t nstreams, const uint8_t* src, const uint64_t* src_off, const uint64_t* src_len, kz_index** out,
                           int32_t* status) {
    if (!ctx) return -KZ_ERR_INVALID_PARAM;
    int rc = check_index_streams_args(ctx, nstreams, src, src_off, src_len, out, status, false);
    if (!rc) rc = [&]() -> int {
        CK(cudaSetDevice(ctx->device));
        // the streams packed at 16-byte aligned offsets with 64 zero bytes behind each, moved in one transfer
        std::vector<UploadPiece> in(nstreams);
        for (uint32_t s = 0; s < nstreams; s++) in[s] = UploadPiece{src + src_off[s], src_len[s], src_len[s] + 64};
        std::vector<uint64_t> in_off;
        uint64_t total = 0;
        int r = upload_pieces(ctx, in, in_off, &total);
        if (r) return r;
        return index_build_streams(ctx, nstreams, ctx->d_in.as<uint8_t>(), in_off.data(), src_len, out, status);
    }();
    return finish_streams(nstreams, status, nullptr, rc);
}

int kz_read_ranges_streams(kz_ctx* ctx, kz_cache* cache, uint32_t nstreams, kz_index* const* ix, const uint8_t* src, const uint64_t* src_off,
                           const uint64_t* src_len, uint32_t nreq, const uint32_t* req_stream, const uint64_t* off, const uint64_t* len, uint8_t* dst,
                           const uint64_t* dst_off, uint64_t* out_len, int32_t* status) {
    return read_ranges_streams(ctx, cache, nstreams, ix, src, false, src_off, src_len, nreq, req_stream, off, len, dst, dst_off, out_len, status);
}

int kz_read_ranges_streams_device(kz_ctx* ctx, kz_cache* cache, uint32_t nstreams, kz_index* const* ix, const void* d_src, const uint64_t* src_off,
                                  const uint64_t* src_len, uint32_t nreq, const uint32_t* req_stream, const uint64_t* off, const uint64_t* len, void* d_dst,
                                  const uint64_t* dst_off, uint64_t* out_len, int32_t* status) {
    if (int rc = after_caller_work(ctx)) return finish_streams(nreq, status, out_len, rc);
    return read_ranges_streams(ctx, cache, nstreams, ix, (const uint8_t*)d_src, true, src_off, src_len, nreq, req_stream, off, len, d_dst, dst_off, out_len,
                               status);
}

// ---- block cache (kz_cache_*, kz_read_ranges_cached[_device]; bookkeeping in kz_block_cache.h) ---------------------------------------
int kz_cache_create(kz_ctx* ctx, uint64_t budget_bytes, kz_cache** out) {
    if (!ctx || !out) return -KZ_ERR_INVALID_PARAM;
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    if (ctx->session) return ctx->fail(KZ_ERR_INVALID_PARAM, "a session is open on this context");
    std::unique_ptr<kz_cache> c(new kz_cache(ctx, budget_bytes));
    if (c->pc.npages()) CK(cudaMalloc(&c->d_pages, (size_t)c->pc.npages() * CACHE_PAGE));
    ctx->caches.push_back(c.get());
    *out = c.release();
    return 0;
}

void kz_cache_free(kz_cache* c) {
    if (!c) return;
    if (kz_ctx* ctx = c->ctx) {
        cudaSetDevice(ctx->device);
        cudaStreamSynchronize(ctx->stream);
        cudaFree(c->d_pages);
        ctx->caches.erase(std::find(ctx->caches.begin(), ctx->caches.end(), c));
    }
    delete c;
}

int kz_cache_clear(kz_cache* c) {
    if (!c || !c->ctx) return -KZ_ERR_INVALID_PARAM;
    c->pc.clear();
    return 0;
}

int kz_cache_stats(const kz_cache* c, uint64_t* entries, uint64_t* resident_bytes, uint64_t* budget_bytes, uint64_t* hits, uint64_t* misses, uint64_t* inserts,
                   uint64_t* evictions, uint64_t* served_bytes) {
    if (!c) return -KZ_ERR_INVALID_PARAM;
    const CacheStats& st = c->pc.stats();
    const std::pair<uint64_t*, uint64_t> f[] = {{entries, st.entries}, {resident_bytes, st.resident}, {budget_bytes, st.budget}, {hits, st.hits},
                                                {misses, st.misses},   {inserts, st.inserts},         {evictions, st.evictions}, {served_bytes, st.served}};
    for (const auto& x : f)
        if (x.first) *x.first = x.second;
    return 0;
}

int kz_read_ranges_cached(kz_ctx* ctx, kz_cache* cache, kz_index* ix, const uint8_t* src, size_t n, uint32_t nreq, const uint64_t* off, const uint64_t* len,
                          uint8_t* dst, const uint64_t* dst_off, uint64_t* out_len, int32_t* status) {
    if (ctx && !cache) return finish_streams(nreq, status, out_len, ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument"));
    return read_ranges(ctx, ix, cache, src, nullptr, n, nreq, off, len, dst, dst_off, out_len, status);
}

int kz_read_ranges_cached_device(kz_ctx* ctx, kz_cache* cache, kz_index* ix, const void* d_src, size_t n, uint32_t nreq, const uint64_t* off,
                                 const uint64_t* len, void* d_dst, const uint64_t* dst_off, uint64_t* out_len, int32_t* status) {
    if (int rc = after_caller_work(ctx)) return finish_streams(nreq, status, out_len, rc);
    if (ctx && !cache) return finish_streams(nreq, status, out_len, ctx->fail(KZ_ERR_INVALID_PARAM, "missing argument"));
    return read_ranges(ctx, ix, cache, nullptr, d_src, n, nreq, off, len, d_dst, dst_off, out_len, status);
}

// ---- block batch, host buffers (Writer.processBlock / Reader.processBlock replacement) -----------------------
int kz_encode_blocks(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t checksum_bits, const uint8_t* slab, uint64_t block_stride,
                     const uint32_t* block_len, uint32_t nblocks, uint8_t* out, uint64_t out_stride, uint64_t* out_bits, int32_t* status) {
    if (!ctx || !slab || !block_len || !out || !out_bits) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    if (checksum_bits != 0 && checksum_bits != 32 && checksum_bits != 64) return ctx->fail(KZ_ERR_INVALID_PARAM, "checksum must be 0, 32 or 64 bits");
    if (nblocks == 0) return 0;
    // device layout: block b at b * dstride (16-byte aligned)
    uint32_t max_len = 0;
    for (uint32_t b = 0; b < nblocks; b++) max_len = std::max(max_len, block_len[b]);
    const uint64_t dstride = ((uint64_t)max_len + 15) & ~15ull;
    uint64_t ostride = round16(kz_max_block_output(max_len));  // encode_slots' stride
    if (out_stride < ostride) return ctx->fail(KZ_ERR_INVALID_PARAM, "out_stride must be >= kz_max_block_output(max block length)");
    CK(ctx->d_in.ensure(dstride * nblocks + 64));
    for (uint32_t b = 0; b < nblocks; b++)
        if (block_len[b])
            CK(cudaMemcpyAsync((uint8_t*)ctx->d_in.p + b * dstride, slab + b * block_stride, block_len[b], cudaMemcpyHostToDevice, ctx->stream));
    TransformPlan plan;
    int rc = plan_transforms(ctx, t48, etype, plan, KZ_ERR_CREATE_CODEC);
    if (rc) return rc;
    // the blocks' heads are in host memory: preparing them costs no round trip
    BlockList bl;
    bl.len.assign(block_len, block_len + nblocks);
    bl.first = {0, nblocks};
    std::vector<uint8_t> heads(4 * (size_t)nblocks, 0);
    for (uint32_t b = 0; b < nblocks; b++) {
        bl.off.push_back(b * dstride);
        memcpy(&heads[(size_t)b * 4], slab + b * block_stride, std::min<uint32_t>(4, block_len[b]));
    }
    BlockPrep prep;
    rc = prepare_blocks(ctx, plan, ctx->skip_blocks, checksum_bits, ctx->d_in.as<uint8_t>(), bl, prep, &heads);
    if (rc) return rc;
    std::vector<uint64_t> bits;
    rc = encode_slots(ctx, plan, etype, checksum_bits, ctx->d_in.as<uint8_t>(), dstride, bl.len, std::vector<uint64_t>(nblocks, ctx->user_stream_bs), prep,
                      &ostride, bits);
    if (rc) return rc;
    for (uint32_t b = 0; b < nblocks; b++) {
        out_bits[b] = bits[b];
        if (status) status[b] = 0;
        size_t nbytes = (size_t)((bits[b] + 7) / 8);
        CK(cudaMemcpyAsync(out + b * out_stride, ctx->d_enc.as<uint8_t>() + b * ostride, nbytes, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int kz_decode_blocks(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t checksum_bits, const uint8_t* in, const uint64_t* in_off,
                     const uint64_t* in_bits, uint32_t nblocks, uint32_t block_size, uint8_t* out, uint64_t out_stride, uint32_t* out_len,
                     int32_t* status) {
    if (!ctx || !in || !in_off || !in_bits || !out || !out_len) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    if (checksum_bits != 0 && checksum_bits != 32 && checksum_bits != 64) return ctx->fail(KZ_ERR_INVALID_PARAM, "checksum must be 0, 32 or 64 bits");
    TransformPlan plan;
    {
        int prc = plan_transforms(ctx, t48, etype, plan, KZ_ERR_INVALID_CODEC);
        if (prc) return prc;
    }
    if (nblocks == 0) return 0;
    // pack the block bit strings at 16-byte aligned device offsets
    std::vector<DecJob> jobs(nblocks);
    uint64_t doff = 0;
    for (uint32_t b = 0; b < nblocks; b++) {
        jobs[b] = DecJob();
        jobs[b].bit_off = 8 * doff;
        jobs[b].bits = in_bits[b];
        jobs[b].block_size = block_size;
        doff += (((in_bits[b] + 7) / 8) + 8 + 15) & ~15ull;
    }
    const uint64_t dsz = doff;
    CK(ctx->d_in.ensure(dsz + 128));
    CK(cudaMemsetAsync(ctx->d_in.p, 0, dsz + 128, ctx->stream));
    for (uint32_t b = 0; b < nblocks; b++)
        CK(cudaMemcpyAsync((uint8_t*)ctx->d_in.p + jobs[b].bit_off / 8, in + in_off[b], (size_t)((in_bits[b] + 7) / 8), cudaMemcpyHostToDevice, ctx->stream));
    const StreamHeader sh = {t48, etype, block_size, checksum_bits, 0, 0};
    // block b is staged at b * slot: a block header claims at most max(2048, 1.5 x block_size) bytes (parse_block_header), and no stage
    // writes more than decode_walked's stride for that claim allows
    const uint32_t claim = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(2048, (uint64_t)block_size + block_size / 2), 1u << 30);
    const uint64_t slot = decode_stride(block_size, claim);
    CK(ctx->d_out.ensure(slot * nblocks + 64));
    std::vector<DecodeFailure> fail;
    std::vector<uint32_t> len;
    // every block may be its stream's last: NONE's multiple-of-16 rule does not apply to a batch of blocks
    int rc = decode_isolated(ctx, sh, plan, ctx->d_in.as<uint32_t>(), dsz / 4 + 16, jobs, std::vector<uint8_t>(nblocks, 1),
                             [&](uint32_t b, uint32_t n) { return n <= out_stride ? b * slot : NO_ROOM; }, ctx->d_out.as<uint8_t>(), fail, len);
    if (rc) return rc;
    for (uint32_t b = 0; b < nblocks; b++) {
        if (status) status[b] = fail[b].code;
        out_len[b] = fail[b].failed() ? 0 : len[b];
        if (out_len[b]) CK(cudaMemcpyAsync(out + b * out_stride, ctx->d_out.as<uint8_t>() + b * slot, out_len[b], cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream));
    for (uint32_t b = 0; b < nblocks; b++)
        if (fail[b].failed()) return ctx->fail(-fail[b].code, fail[b].msg);
    return 0;
}

// ---- single block entropy codec (EntropyEncoder.Write / EntropyDecoder.Read) ----------------------------------
int kz_entropy_encode(kz_ctx* ctx, uint32_t type, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, uint64_t* out_bits) {
    if (!ctx || (!src && n) || !dst || !out_bits) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    if (n > (1u << 30)) return ctx->fail(KZ_ERR_BLOCK_SIZE, "block too large");
    *out_bits = 0;
    if (n == 0) return 0;
    const size_t dcap = kz_max_block_output(n);
    CK(ctx->d_in.ensure(n + 64));
    CK(ctx->d_out.ensure(dcap + 64));
    CK(cudaMemcpyAsync(ctx->d_in.p, src, n, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<EncJob> jobs(1);
    jobs[0].data_off = 0;
    jobs[0].post_len = (uint32_t)n;
    jobs[0].ntransforms = 1;
    jobs[0].skip_flags = 0;
    jobs[0].copy = false;
    jobs[0].checksum = 0;
    EncResult res;
    int rc = encode_batch(ctx, LAYOUT_RAW, type, 0, ctx->d_in.as<uint8_t>(), jobs, {}, 0, false, false, ctx->d_out.as<uint8_t>(), dcap, {0}, res);
    if (rc) return rc;
    const size_t nbytes = (size_t)((res.blk_bits[0] + 7) / 8);
    if (nbytes > cap) return ctx->fail(KZ_ERR_WRITE_FILE, "output buffer too small");
    CK(cudaMemcpyAsync(dst, ctx->d_out.p, nbytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *out_bits = res.blk_bits[0];
    return 0;
}

int kz_entropy_decode(kz_ctx* ctx, uint32_t type, const uint8_t* src, size_t src_bytes, uint8_t* dst, size_t n, uint64_t* consumed_bits) {
    if (!ctx || !src || (!dst && n)) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    if (consumed_bits) *consumed_bits = 0;
    if (n == 0) return 0;
    if (n > (1u << 30)) return ctx->fail(KZ_ERR_BLOCK_SIZE, "block too large");
    CK(ctx->d_in.ensure(src_bytes + 128));
    CK(ctx->d_out.ensure(n + 64));
    CK(cudaMemsetAsync((uint8_t*)ctx->d_in.p + (src_bytes & ~size_t(3)), 0, 128, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_in.p, src, src_bytes, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<DecJob> jobs(1);
    jobs[0] = DecJob();
    jobs[0].bit_off = 0;
    jobs[0].bits = 8ull * src_bytes;
    jobs[0].out_off = 0;
    jobs[0].pre_len = (uint32_t)n;
    jobs[0].data_bit = 0;
    jobs[0].copy = false;
    jobs[0].status = 0;
    int rc = decode_batch(ctx, type, ctx->d_in.as<uint32_t>(), src_bytes / 4 + 16, jobs, ctx->d_out.as<uint8_t>());
    if (rc) return rc;
    if (jobs[0].status) return ctx->fail(-jobs[0].status, "Invalid bitstream: entropy decoding failed");
    CK(cudaMemcpyAsync(dst, ctx->d_out.p, n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (consumed_bits) *consumed_bits = jobs[0].end_pos;
    return 0;
}

// One transform on one block: the argument checks of each reference codec, then the stage a sequence of that one transform runs
int kz_transform_forward(kz_ctx* ctx, uint64_t type, int* data_type, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n) {
    if (!ctx || (!src && n) || !dst || !out_n) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    *out_n = 0;
    if (!TransformPlan::seq_id(type)) return ctx->fail(KZ_ERR_CREATE_CODEC, NO_GPU_TRANSFORM);
    if (n == 0) return 0;
    if (n > (1u << 30)) return ctx->fail(KZ_ERR_BLOCK_SIZE, type == KZ_T_BWT ? "The max BWT block size is 1 GiB" : "block too large");
    if (cap < kz_transform_max_encoded_len(type, n)) {
        // BWTBlockCodec and LZXCodec refuse the call; every other Forward returns an error, and the sequence skips the transform
        if (type == KZ_T_BWT || type == KZ_T_LZ || type == KZ_T_LZX) return ctx->fail(KZ_ERR_INVALID_PARAM, "Output buffer is too small");
        return 1;
    }
    if (type == KZ_T_BWT && n < 2) return 1;  // BWTBlockCodec.Forward: invalid index size -> the sequence skips the transform
    const uint64_t stride = ((uint64_t)n + n / 8 + 8192 + 1024 + 64 + 64 + 15) & ~15ull;
    CK(ctx->d_in.ensure(stride));
    CK(ctx->d_out.ensure(stride));
    CK(cudaMemcpyAsync(ctx->d_in.p, src, n, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<uint32_t> len(1, (uint32_t)n);
    std::vector<uint8_t> active(1, 1), applied;
    std::vector<int32_t> dt1(1, data_type ? *data_type : 0);  // ctx["dataType"]; BWT / BWTS / LZ / LZX / RANK / MTFT / ZRLT leave it as it is
    int rc = apply_forward(ctx, type, ctx->d_in.as<uint8_t>(), stride, ctx->d_out.as<uint8_t>(), stride, len, active, applied,
                           std::vector<uint64_t>(1, ctx->user_stream_bs), &dt1);
    if (rc) return rc;
    if (data_type) *data_type = dt1[0];
    if (!applied[0]) return 1;
    CK(cudaMemcpyAsync(dst, ctx->d_out.p, len[0], cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *out_n = len[0];
    return 0;
}

// cap = len(dst) of the reference call
int kz_transform_inverse(kz_ctx* ctx, uint64_t type, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n) {
    if (!ctx || (!src && n) || !dst || !out_n) return -KZ_ERR_INVALID_PARAM;
    CK(cudaSetDevice(ctx->device));
    *out_n = 0;
    if (!TransformPlan::seq_id(type)) return ctx->fail(KZ_ERR_CREATE_CODEC, NO_GPU_TRANSFORM);
    if (n == 0) return 0;
    if (type == KZ_T_BWT) {
        if (n == 1) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "BWT inverse transform failed: invalid size");
        if (n > (1u << 30) + 33) return ctx->fail(KZ_ERR_BLOCK_SIZE, "The max BWT block size is 1 GiB");
        cap = std::min(cap, n);  // the block is shorter than its header + BWT bytes: more room changes nothing
    } else if (type == KZ_T_LZ || type == KZ_T_LZX) {  // LZXCodec.inverseV6
        if (cap == 0) return 0;  // LZCodec.go:622-624
        if (n > (1u << 30) || cap > (1u << 30) + 64) return ctx->fail(KZ_ERR_BLOCK_SIZE, "block too large");
    } else {
        if (cap == 0) return 0;
        if (n > (1u << 30) || cap > (1u << 30) + 4096) return ctx->fail(KZ_ERR_BLOCK_SIZE, "block too large");
    }
    const uint64_t stride = ((uint64_t)std::max(n, cap) + 64 + 15) & ~15ull;
    CK(ctx->d_in.ensure(stride));
    CK(ctx->d_out.ensure(stride));
    CK(cudaMemcpyAsync(ctx->d_in.p, src, n, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<uint32_t> len(1, (uint32_t)n);
    std::vector<uint8_t> active(1, 1);
    int rc = apply_inverse(ctx, type, ctx->d_in.as<uint8_t>(), ctx->d_out.as<uint8_t>(), stride, (uint32_t)cap, len, active,
                           std::vector<uint64_t>(1, ctx->user_stream_bs));
    if (rc) return rc;
    if (len[0]) CK(cudaMemcpyAsync(dst, ctx->d_out.p, len[0], cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *out_n = len[0];
    return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------
// Streaming sessions (kz_writer_* / kz_reader_*): one stream of any length in bounded device and pinned memory, the role of
// CompressedOutputStream / CompressedInputStream (io/CompressedStream.go:524-710, :1556-1744), which cut `jobs` blocks per batch.
// ------------------------------------------------------------------------------------------------------------
namespace kz {

const int SESSION_STOPPED = 1;                 // a worker step that saw the session being freed
const uint64_t READER_BATCH_BYTES = 256ull << 20;  // kz_reader_open with batch_blocks 0: about this many decoded bytes per batch

// The pump both sessions share. The caller's thread fills pinned input slot (given % 2), issues its host-to-device copy on `copy` and
// hands it to the worker; the worker is the only thread that drives ctx while the session is open: it waits on the slot's event on
// ctx->stream, computes, copies the finished bytes into pinned output slot (made % 2) and publishes them; the caller's thread hands them
// out. So the caller's I/O and the copies of batch k + 1 overlap the kernels of batch k. All counters are guarded by m.
struct Session {
    kz_ctx* ctx;
    uint32_t batch_blocks;
    std::thread worker;
    std::mutex m;
    std::condition_variable cv;
    cudaStream_t copy = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    PinnedBuf h_in[2], h_out[2];
    DevBuf d_in[2];
    size_t in_cap = 0;                        // bytes per input slot
    size_t in_len[2] = {0, 0};                // filled bytes of each input slot
    bool in_last[2] = {false, false};
    size_t out_len[2] = {0, 0}, out_pos = 0;  // published bytes of each output slot, bytes of slot (taken % 2) handed out
    uint64_t given = 0, done = 0;             // input slots handed to the worker / finished by it
    uint64_t made = 0, taken = 0;             // output slots published / handed out completely
    bool last_given = false, finished = false, stop = false;
    int err = 0;                              // sticky: 0 or -(error code)
    size_t scratch = 0;                       // ctx->scratch_bytes() after the worker's last step

    explicit Session(kz_ctx* c, uint32_t bb) : ctx(c), batch_blocks(bb) {}
    virtual ~Session() {}
    virtual int run(int k, bool last) = 0;  // worker: input slot k
    virtual size_t own_device_bytes() = 0;
    virtual void release_own() = 0;

    int open_common() {
        if (cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking) != cudaSuccess) return ctx->fail(KZ_ERR_CREATE_COMPRESSOR, "cannot create the copy stream");
        for (auto& e : ev)
            if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return ctx->fail(KZ_ERR_CREATE_COMPRESSOR, "cannot create events");
        scratch = ctx->scratch_bytes();
        ctx->session = this;
        worker = std::thread([this] { main(); });
        return 0;
    }
    int alloc_inputs(size_t cap) {
        in_cap = cap;
        for (int k = 0; k < 2; k++) {
            CK(h_in[k].ensure(cap));
            CK(d_in[k].ensure(cap));
        }
        return 0;
    }

    void main() {
        cudaSetDevice(ctx->device);
        for (;;) {
            int k;
            bool last;
            {
                std::unique_lock<std::mutex> l(m);
                cv.wait(l, [&] { return stop || done < given; });
                if (stop) return;
                k = (int)(done % 2);
                last = in_last[k];
            }
            int rc = run(k, last);
            std::lock_guard<std::mutex> l(m);
            scratch = ctx->scratch_bytes();
            in_len[k] = 0;
            done++;
            if (rc < 0 && !err) err = rc;
            if (rc == 0 && last) finished = true;
            cv.notify_all();
            if (rc || last) return;
        }
    }

    // worker: copies copy_n finished bytes at d_src into the next free output slot and publishes the first give_n of them; *tail = the
    // byte behind them (the writer's carry)
    int publish(const void* d_src, size_t copy_n, size_t give_n, uint8_t* tail = nullptr) {
        if (copy_n == 0) return 0;
        int j;
        {
            std::unique_lock<std::mutex> l(m);
            cv.wait(l, [&] { return stop || made - taken < 2; });
            if (stop) return SESSION_STOPPED;
            j = (int)(made % 2);
        }
        CK(cudaMemcpyAsync(h_out[j].p, d_src, copy_n, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (tail) *tail = give_n < copy_n ? ((const uint8_t*)h_out[j].p)[give_n] : 0;
        std::lock_guard<std::mutex> l(m);
        out_len[j] = give_n;
        made++;
        cv.notify_all();
        return 0;
    }

    // caller: a failure found on the caller's side; the worker is joined before ctx is touched
    int fail(int code, const std::string& msg) {
        bool mine = false;
        {
            std::lock_guard<std::mutex> l(m);
            if (!err) {
                err = -code;
                mine = true;
            }
            stop = true;
            cv.notify_all();
        }
        if (worker.joinable()) worker.join();
        if (mine) ctx->err = msg;
        return err;
    }
    int cuda_fail(cudaError_t e, const char* what) { return fail(KZ_ERR_PROCESS_BLOCK, std::string(what) + ": " + cudaGetErrorString(e)); }

    // caller: hands out published bytes; returns the count
    size_t take(uint8_t* dst, size_t cap) {
        size_t got = 0;
        for (;;) {
            int j;
            size_t avail;
            {
                std::lock_guard<std::mutex> l(m);
                if (taken == made) return got;
                j = (int)(taken % 2);
                avail = out_len[j] - out_pos;
                if (avail == 0 || got == cap) {
                    if (avail == 0) {
                        out_pos = 0;
                        taken++;
                        cv.notify_all();
                        continue;
                    }
                    return got;
                }
            }
            const size_t c = std::min(avail, cap - got);
            memcpy(dst + got, (const uint8_t*)h_out[j].p + out_pos, c);
            got += c;
            out_pos += c;
        }
    }
    bool slot_free() {
        std::lock_guard<std::mutex> l(m);
        return given - done < 2;
    }
    // caller: hands input slot k (filled) to the worker
    int give(int k, bool last) {
        if (in_len[k]) {
            cudaError_t e = cudaMemcpyAsync(d_in[k].p, h_in[k].p, in_len[k], cudaMemcpyHostToDevice, copy);
            if (e != cudaSuccess) return cuda_fail(e, "session input copy");
        }
        cudaError_t e = cudaEventRecord(ev[k], copy);
        if (e != cudaSuccess) return cuda_fail(e, "session input event");
        std::lock_guard<std::mutex> l(m);
        in_last[k] = last;
        given++;
        if (last) last_given = true;
        cv.notify_all();
        return 0;
    }
    // caller: copies up to n bytes into the input slots, handing over every full one; returns the count or a negative error
    int64_t feed(const uint8_t* src, size_t n) {
        size_t c = 0;
        while (c < n && slot_free()) {
            const int k = (int)(given % 2);
            const size_t t = std::min(n - c, in_cap - in_len[k]);
            memcpy((uint8_t*)h_in[k].p + in_len[k], src + c, t);
            in_len[k] += t;
            c += t;
            if (in_len[k] == in_cap) {
                int rc = give(k, false);
                if (rc) return rc;
            }
        }
        return (int64_t)c;
    }
    // caller: nothing could be done without waiting. 1 = return to the caller empty-handed (nothing in flight that could change it)
    int wait_for_worker(bool have_input, bool have_room) {
        std::unique_lock<std::mutex> l(m);
        if (err) return err;
        if (!have_room && taken < made) return 1;  // finished bytes wait for room
        if (!have_input && done == given) return 1;
        const uint64_t d0 = done, m0 = made;
        cv.wait(l, [&] { return err || done != d0 || made != m0; });
        return err;
    }

    // the zlib-style pump of write / read: consume or produce at least one byte unless nothing can happen
    int pump(const uint8_t* src, size_t n, size_t* consumed, uint8_t* dst, size_t cap, size_t* produced) {
        for (;;) {
            bool lg;
            {
                std::lock_guard<std::mutex> l(m);
                if (err) return err;
                lg = last_given;
            }
            if (lg) return fail(KZ_ERR_INVALID_PARAM, "session: write or read after finish");
            *produced += take(dst + *produced, cap - *produced);
            int64_t c = accept(src + *consumed, n - *consumed);
            if (c < 0) return (int)c;
            *consumed += (size_t)c;
            if (*consumed || *produced || (n == 0 && cap == 0)) return 0;
            int rc = wait_for_worker(n > 0, cap > 0);
            if (rc < 0) return rc;
            if (rc == 1) return 0;
        }
    }
    // end of input: 0 = every byte handed out, 1 = call again with room
    int finish(uint8_t* dst, size_t cap, size_t* produced) {
        for (;;) {
            {
                std::lock_guard<std::mutex> l(m);
                if (err) return err;
            }
            *produced += take(dst + *produced, cap - *produced);
            bool lg;
            {
                std::lock_guard<std::mutex> l(m);
                lg = last_given;
            }
            if (!lg && slot_free()) {
                int rc = hand_last();
                if (rc) return rc;
            }
            std::unique_lock<std::mutex> l(m);
            if (err) return err;
            if (finished && taken == made) return 0;
            if (*produced == cap) return 1;
            if (taken < made) continue;
            const uint64_t d0 = done, m0 = made;
            cv.wait(l, [&] { return err || done != d0 || made != m0; });
        }
    }
    virtual int64_t accept(const uint8_t* src, size_t n) { return feed(src, n); }
    virtual int hand_last() { return give((int)(given % 2), true); }

    // kz_*_free: joins the worker (after the step in flight), waits for the copies in flight and leaves ctx usable
    void close() {
        {
            std::lock_guard<std::mutex> l(m);
            stop = true;
            cv.notify_all();
        }
        if (worker.joinable()) worker.join();
        cudaSetDevice(ctx->device);
        if (copy) cudaStreamSynchronize(copy);
        cudaStreamSynchronize(ctx->stream);
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        if (copy) cudaStreamDestroy(copy);
        for (int k = 0; k < 2; k++) {
            h_in[k].release();
            h_out[k].release();
            d_in[k].release();
        }
        release_own();
        if (ctx->session == this) ctx->session = nullptr;
        ctx = nullptr;  // closed: only kz_*_free may follow
    }
    size_t device_bytes() {
        std::lock_guard<std::mutex> l(m);
        return scratch + d_in[0].cap + d_in[1].cap + own_device_bytes();
    }
};

// kz_destroy with a session open: the session is closed first; its handle is then only good for kz_*_free
void close_session(Session* s) { s->close(); }

}  // namespace kz

struct kz_writer : kz::Session {
    TransformPlan plan;
    uint64_t t48 = 0;
    uint32_t etype = 0, block_size = 0, checksum_bits = 0;
    int64_t input_size = 0;
    bool headerless = false;  // the context's headerless writer setting when the session opened (kz_set_headerless_writer)
    bool skip = false;        // and its skipBlocks setting (kz_set_skip_blocks)
    DevBuf d_out;            // the finished bytes of one batch
    size_t out_cap = 0;
    uint64_t batches = 0;    // batches encoded (worker)
    uint8_t carry = 0;       // the last total_bits mod 8 bits of the previous batch, MSB first (worker)
    uint32_t carry_bits = 0;

    using Session::Session;
    size_t own_device_bytes() override { return d_out.cap; }
    void release_own() override { d_out.release(); }

    // worker: one batch = the blocks of input slot k behind the stream header (first batch; nothing when headerless) or the carry; the end
    // marker only in the last
    int run(int k, bool last) override {
        CK(cudaStreamWaitEvent(ctx->stream, ev[k], 0));
        std::vector<uint8_t> lead(64, 0);
        uint32_t lead_bits = carry_bits;
        if (batches == 0) lead_bits = headerless ? 0 : build_stream_header(lead, t48, etype, block_size, checksum_bits, input_size);
        else lead[0] = carry;
        EncResult res;
        int rc = encode_stream_blocks(ctx, plan, etype, block_size, checksum_bits, skip, d_in[k].p, in_len[k], lead, lead_bits, !last, true, d_out.p, out_cap,
                                      res);
        if (rc) return rc;
        CK(cudaStreamSynchronize(ctx->stream));
        batches++;
        const uint64_t give_n = batch_bytes_out(res.total_bits, last, &carry_bits);
        return publish(d_out.p, (size_t)((res.total_bits + 7) / 8), (size_t)give_n, &carry);
    }
};

struct kz_reader : kz::Session {
    StreamHeader sh;
    TransformPlan plan;
    uint8_t head[64];
    size_t head_len = 0;
    bool have_header = false;
    DevBuf win[2], d_dec, d_walk;  // window buffers (the unconsumed bits move between them), decoded bytes of one batch, walk results
    size_t win_cap = 0, dec_cap = 0;
    uint64_t max_rec_bits = 0;
    // worker state
    int cur = 0;
    uint64_t fill = 0, start_bit = 0;  // valid bytes of win[cur], first bit not yet walked
    bool ended = false;                // the end marker was read (guarded by m: the caller drops input after it)
    bool odd_tail = false;             // NONE: the last block handed out has a length that is not a multiple of 16
    int64_t range_from = -1, range_to = -1;  // the context's block range when the session opened (kz_set_block_range)
    uint64_t walked = 0;                     // records walked so far

    using Session::Session;
    size_t own_device_bytes() override { return win[0].cap + win[1].cap + d_dec.cap + d_walk.cap; }
    void release_own() override {
        win[0].release();
        win[1].release();
        d_dec.release();
        d_walk.release();
    }

    // caller: the stream header is parsed from the first 64 bytes (or fewer at finish, as kz_decompress_stream does); the buffers are
    // sized from it. A headerless session has sh from the setting and starts at open.
    int start(bool headerless) {
        int rc = headerless ? 0 : parse_stream_header(ctx, head, head_len, sh);
        if (rc == 0) rc = plan_transforms(ctx, sh.t48, sh.etype, plan, KZ_ERR_INVALID_CODEC);
        if (rc) return fail(-rc, ctx->err);
        const uint64_t bs = sh.block_size;
        if (batch_blocks == 0) batch_blocks = (uint32_t)std::min<uint64_t>(1024, std::max<uint64_t>(1, READER_BATCH_BYTES / bs));
        // one decode slot per block, at the longest a block header can claim (parse_block_header's bound on the pre-transform length)
        const uint64_t max_len = std::min<uint64_t>(std::max<uint64_t>(2048, bs + bs / 2), 1ull << 30);
        max_rec_bits = 8ull * kz_max_block_output(bs);
        dec_cap = (size_t)(batch_blocks * decode_stride(sh.block_size, (uint32_t)max_len));
        const size_t in_bytes = (size_t)batch_blocks * bs;
        win_cap = (size_t)(max_rec_bits / 8 + 64 + in_bytes);
        cudaError_t e = cudaSuccess;
        for (int k = 0; k < 2 && e == cudaSuccess; k++) {
            e = h_in[k].ensure(in_bytes);
            if (e == cudaSuccess) e = d_in[k].ensure(in_bytes);
            if (e == cudaSuccess) e = h_out[k].ensure(dec_cap);
            if (e == cudaSuccess) e = win[k].ensure(win_cap);
        }
        if (e == cudaSuccess) e = d_dec.ensure(dec_cap);
        if (e == cudaSuccess) e = d_walk.ensure((size_t)batch_blocks * 16 + sizeof(WalkResult) + 64);
        if (e != cudaSuccess) return cuda_fail(e, "session buffers");
        in_cap = in_bytes;
        start_bit = sh.bits;
        have_header = true;
        memcpy(h_in[0].p, head, head_len);  // slot 0 is the first one filled (in_cap >= 1024 > head_len)
        in_len[0] = head_len;
        return 0;
    }
    int64_t accept(const uint8_t* src, size_t n) override {
        size_t c = 0;
        if (!have_header) {
            c = std::min(n, sizeof(head) - head_len);
            memcpy(head + head_len, src, c);
            head_len += c;
            if (head_len < sizeof(head)) return (int64_t)c;
            int rc = start(false);
            if (rc) return rc;
        }
        {
            std::lock_guard<std::mutex> l(m);
            if (ended) return (int64_t)n;  // bytes behind the end marker are ignored
        }
        int64_t f = feed(src + c, n - c);
        return f < 0 ? f : (int64_t)c + f;
    }
    int hand_last() override {
        if (!have_header) {
            int rc = start(false);
            if (rc) return rc;
        }
        return give((int)(given % 2), true);
    }

    // worker: appends input slot k to the window, then walks and decodes every complete record, batch_blocks at a time
    int run(int k, bool last) override {
        bool end_seen;
        {
            std::lock_guard<std::mutex> l(m);
            end_seen = ended;
        }
        if (!end_seen) {
            CK(cudaStreamWaitEvent(ctx->stream, ev[k], 0));
            if (fill + in_len[k] + 64 > win[cur].cap) return ctx->fail(KZ_ERR_UNKNOWN, "internal: reader window overflow");
            CopyList cl;
            cl.add(d_in[k].p, win[cur].as<uint8_t>() + fill, in_len[k]);
            int rc = run_copies(ctx, cl);
            if (rc) return rc;
            fill += in_len[k];
            rc = walk_and_decode();
            if (rc) return rc;
            {
                std::lock_guard<std::mutex> l(m);
                end_seen = ended;
            }
            if (!end_seen) {  // the unconsumed bits move to the start of the other window buffer (from a 16-byte boundary)
                const uint64_t from = (start_bit / 8) & ~15ull;
                CopyList tail;
                tail.add(win[cur].as<uint8_t>() + from, win[cur ^ 1].as<uint8_t>(), fill - from);
                rc = run_copies(ctx, tail);
                if (rc) return rc;
                CK(cudaStreamSynchronize(ctx->stream));
                cur ^= 1;
                fill -= from;
                start_bit -= 8 * from;
            }
        }
        CK(cudaStreamSynchronize(ctx->stream));  // input slot k is free again
        if (last && !end_seen) return ctx->fail(KZ_ERR_PROCESS_BLOCK, "Invalid bitstream: truncated stream");
        return 0;
    }

    int walk_and_decode() {
        const uint32_t* W = win[cur].as<uint32_t>();
        uint64_t* d_boff = d_walk.as<uint64_t>();
        uint64_t* d_bbits = d_boff + batch_blocks;
        WalkResult* d_res = (WalkResult*)(d_bbits + batch_blocks);
        std::vector<uint64_t> boff(batch_blocks), bbits(batch_blocks);
        for (;;) {
            {
                LaunchScope ls(ctx, "record_walk");
                record_walk_kernel<<<1, 1, 0, ctx->stream>>>(W, start_bit, 8 * fill, batch_blocks, max_rec_bits, d_boff, d_bbits, d_res);
            }
            CK(cudaGetLastError());
            WalkResult r;
            CK(cudaMemcpyAsync(&r, d_res, sizeof(r), cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaMemcpyAsync(boff.data(), d_boff, (size_t)batch_blocks * 8, cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaMemcpyAsync(bbits.data(), d_bbits, (size_t)batch_blocks * 8, cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            if (r.status) return ctx->fail(-r.status, "Invalid bitstream: corrupted block length");
            if (r.count) {
                // only the records in the block range are decoded; the others were walked and their bits are dropped with the window
                uint32_t lo, hi;
                block_range_slice(range_from, range_to, walked, r.count, &lo, &hi);
                walked += r.count;
                // NONE: a decoded block that was not the stream's last record must be a multiple of 16 long
                if (plan.none() && odd_tail) pend.note(STAGE_HEADER, -KZ_ERR_PROCESS_BLOCK, "unexpected block length");
                odd_tail = false;
                if (hi > lo) {
                    int rc = decode(hi - lo, &boff[lo], &bbits[lo], hi == r.count);
                    if (rc) return rc;
                }
            }
            start_bit = r.next_bit;
            if (r.ended) {
                {
                    std::lock_guard<std::mutex> l(m);
                    ended = true;
                }
                return pend.failed() ? ctx->fail(-pend.code, pend.msg) : 0;
            }
            if (r.count < batch_blocks) return 0;
        }
    }

    // A block-level failure (block header, entropy decode, inverse transform, checksum) is not reported when it is found:
    // decompress_device_impl walks every record of the stream before it decodes any, so a walk error (a length over the limits, a
    // truncated stream) found later takes precedence, and after the walk the failure of the earliest stage wins, the earliest block
    // within a stage. The reader keeps the failure that wins so far, hands out nothing more, runs each later batch only through the
    // stages whose failures could still win (decode_walked skips the others), and reports at the end marker or at the walk error.
    DecodeFailure pend;

    // nb records of one batch, as decompress_device_impl decodes a whole stream; the decoded bytes are published back to back.
    // ends_batch: the last of them is the last record walked so far.
    int decode(uint32_t nb, const uint64_t* boff, const uint64_t* bbits, bool ends_batch) {
        std::vector<DecJob> jobs(nb);
        for (uint32_t b = 0; b < nb; b++) {
            jobs[b] = DecJob();
            jobs[b].bit_off = boff[b];
            jobs[b].bits = bbits[b];
            jobs[b].block_size = sh.block_size;
        }
        std::vector<uint8_t> last(nb, 0);
        last[nb - 1] = ends_batch;
        BackToBack place{dec_cap};
        int rc = decode_walked(ctx, sh, plan, win[cur].as<uint32_t>(), (fill + 3) / 4 + 16, jobs, std::vector<uint32_t>(nb, 0), last, place,
                               d_dec.as<uint8_t>(), &pend);
        if (rc) return rc;
        if (plan.none()) odd_tail = (jobs[nb - 1].pre_len & 15) != 0;
        return pend.failed() ? 0 : publish(d_dec.p, (size_t)place.off, (size_t)place.off);
    }
};

extern "C" {

int kz_writer_open(kz_ctx* ctx, uint64_t t48, uint32_t etype, uint32_t block_size, uint32_t checksum_bits, uint32_t batch_blocks, int64_t input_size_hint,
                   kz_writer** out) {
    if (!ctx || !out) return -KZ_ERR_INVALID_PARAM;
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    if (ctx->session) return ctx->fail(KZ_ERR_INVALID_PARAM, "a session is already open on this context");
    int rc = check_encode_args(ctx, block_size, checksum_bits);
    if (rc) return rc;
    if (batch_blocks < 1 || batch_blocks > 1024) return ctx->fail(KZ_ERR_INVALID_PARAM, "batch_blocks must be in [1..1024]");
    if (!etype_supported(etype)) return ctx->fail(KZ_ERR_CREATE_CODEC, "entropy codec not available on the GPU path");
    TransformPlan plan;
    rc = plan_transforms(ctx, t48, etype, plan, KZ_ERR_CREATE_CODEC);
    if (rc) return rc;
    kz_writer* w = new kz_writer(ctx, batch_blocks);
    w->plan = plan;
    w->t48 = t48;
    w->etype = etype;
    w->block_size = block_size;
    w->checksum_bits = checksum_bits;
    w->input_size = input_size_hint;
    w->headerless = ctx->headerless_writer;
    w->skip = ctx->skip_blocks;
    const size_t in_bytes = (size_t)batch_blocks * block_size;
    w->out_cap = kz_max_stream_output(in_bytes, block_size) + 64;
    rc = w->alloc_inputs(in_bytes);
    for (int k = 0; k < 2 && rc == 0; k++)
        if (w->h_out[k].ensure(w->out_cap) != cudaSuccess) rc = ctx->fail(KZ_ERR_CREATE_COMPRESSOR, "cannot allocate pinned output slots");
    if (rc == 0 && w->d_out.ensure(w->out_cap) != cudaSuccess) rc = ctx->fail(KZ_ERR_CREATE_COMPRESSOR, "cannot allocate the device output buffer");
    if (rc == 0) rc = w->open_common();
    if (rc) {
        w->close();
        delete w;
        return rc;
    }
    *out = w;
    return 0;
}

int kz_writer_write(kz_writer* w, const uint8_t* src, size_t n, size_t* consumed, uint8_t* dst, size_t cap, size_t* produced) {
    if (!w || !consumed || !produced || (!src && n) || (!dst && cap)) return -KZ_ERR_INVALID_PARAM;
    *consumed = *produced = 0;
    if (!w->ctx) return -KZ_ERR_INVALID_PARAM;  // its context was destroyed
    if (cudaSetDevice(w->ctx->device) != cudaSuccess) return w->fail(KZ_ERR_PROCESS_BLOCK, "cudaSetDevice failed");
    return w->pump(src, n, consumed, dst, cap, produced);
}

int kz_writer_finish(kz_writer* w, uint8_t* dst, size_t cap, size_t* produced) {
    if (!w || !produced || (!dst && cap)) return -KZ_ERR_INVALID_PARAM;
    *produced = 0;
    if (!w->ctx) return -KZ_ERR_INVALID_PARAM;  // its context was destroyed
    if (cudaSetDevice(w->ctx->device) != cudaSuccess) return w->fail(KZ_ERR_PROCESS_BLOCK, "cudaSetDevice failed");
    return w->finish(dst, cap, produced);
}

void kz_writer_free(kz_writer* w) {
    if (!w) return;
    if (w->ctx) w->close();
    delete w;
}

int kz_reader_open(kz_ctx* ctx, uint32_t batch_blocks, kz_reader** out) {
    if (!ctx || !out) return -KZ_ERR_INVALID_PARAM;
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    if (ctx->session) return ctx->fail(KZ_ERR_INVALID_PARAM, "a session is already open on this context");
    if (batch_blocks > 1024) return ctx->fail(KZ_ERR_INVALID_PARAM, "batch_blocks must be in [0..1024]");
    kz_reader* r = new kz_reader(ctx, batch_blocks);
    r->range_from = ctx->range_from;
    r->range_to = ctx->range_to;
    int rc = r->open_common();
    if (rc == 0 && ctx->headerless_reader.on) {
        r->sh = headerless_header(ctx);
        rc = r->start(true);
    }
    if (rc) {
        r->close();
        delete r;
        return rc;
    }
    *out = r;
    return 0;
}

int kz_reader_read(kz_reader* r, const uint8_t* src, size_t n, size_t* consumed, uint8_t* dst, size_t cap, size_t* produced) {
    if (!r || !consumed || !produced || (!src && n) || (!dst && cap)) return -KZ_ERR_INVALID_PARAM;
    *consumed = *produced = 0;
    if (!r->ctx) return -KZ_ERR_INVALID_PARAM;  // its context was destroyed
    if (cudaSetDevice(r->ctx->device) != cudaSuccess) return r->fail(KZ_ERR_PROCESS_BLOCK, "cudaSetDevice failed");
    return r->pump(src, n, consumed, dst, cap, produced);
}

int kz_reader_finish(kz_reader* r, uint8_t* dst, size_t cap, size_t* produced) {
    if (!r || !produced || (!dst && cap)) return -KZ_ERR_INVALID_PARAM;
    *produced = 0;
    if (!r->ctx) return -KZ_ERR_INVALID_PARAM;  // its context was destroyed
    if (cudaSetDevice(r->ctx->device) != cudaSuccess) return r->fail(KZ_ERR_PROCESS_BLOCK, "cudaSetDevice failed");
    return r->finish(dst, cap, produced);
}

void kz_reader_free(kz_reader* r) {
    if (!r) return;
    if (r->ctx) r->close();
    delete r;
}

size_t kz_device_bytes(kz_ctx* ctx) {
    if (!ctx) return 0;
    size_t caches = 0;
    for (const kz_cache* c : ctx->caches) caches += c->device_bytes();
    return (ctx->session ? ctx->session->device_bytes() : ctx->scratch_bytes()) + caches;
}

}  // extern "C"
