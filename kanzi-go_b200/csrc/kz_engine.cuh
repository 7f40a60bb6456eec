// Host-side engine state behind the C ABI (include/kanzi_b200.h): one context per GPU, owning a stream and
// reusable HBM scratch. The entry points in kz_api.cu are thin wrappers over the methods declared here.
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <string>
#include <vector>

#include "kz_ans.cuh"

namespace kz {

struct Session;
void close_session(Session* s);

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    // grows geometrically; contents are NOT preserved. Always leaves >= 256 bytes of readable slack past n.
    cudaError_t ensure(size_t n) {
        n += 256;
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = n + (n >> 3);
        want = (want + 4095) & ~size_t(4095);
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <class T>
    T* as() const { return reinterpret_cast<T*>(p); }
};

struct PinnedBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        size_t want = n + (n >> 2) + 4096;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() {
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
    }
};

// collects small host tables, uploads them with one async copy, hands back device addresses
struct Packer {
    std::vector<uint8_t> bytes;
    size_t add(const void* src, size_t n) {
        size_t off = (bytes.size() + 255) & ~size_t(255);
        bytes.resize(off + n);
        if (n) memcpy(bytes.data() + off, src, n);
        return off;
    }
    size_t reserve(size_t n) {  // zero-filled region
        size_t off = (bytes.size() + 255) & ~size_t(255);
        bytes.resize(off + n, 0);
        return off;
    }
};

// packed host tables of one encode batch (see encode_batch), kept for the next batch with an identical description
struct EncPlan {
    bool valid = false;
    std::vector<uint8_t> key;
    Packer pk;
    size_t o_small = 0, o_src = 0, o_bits = 0, o_first = 0, o_chunks = 0, o_cseg = 0, o_base = 0, o_off = 0, o_dst = 0, o_blkbits = 0, o_total = 0,
           o_hbits = 0, o_asz = 0, o_estatus = 0;
    int nsegs = 0, nchunks = 0;
    uint32_t max_chunk = 0;
    template <class F>
    void build(const std::vector<uint8_t>& k, F&& fill) {
        fill(*this);
        key = k;
        valid = true;
    }
};

struct ProfEntry {
    double ms = 0;
    uint32_t launches = 0;
    uint64_t bytes_in = 0, bytes_out = 0;  // "stage:*" entries only
};

struct EncJob {          // one block handed to the entropy stage
    uint64_t data_off;   // byte offset of the post-transform data inside the device data buffer (16-byte aligned)
    uint32_t post_len;   // post-transform length (what the entropy coder sees)
    uint32_t ntransforms;
    uint8_t skip_flags;
    bool copy;           // COPY block (io/CompressedStream.go:773-801)
    uint64_t checksum;
};

enum EncLayout { LAYOUT_STREAM = 0, LAYOUT_BLOCKS = 1, LAYOUT_RAW = 2 };

struct DecJob {          // one block handed to the entropy decode stage
    uint64_t bit_off;    // absolute bit offset of the block's bit string in the device stream buffer
    uint64_t bits;
    uint64_t out_off;    // byte offset in the device output buffer (16-byte aligned) for the entropy output
    uint32_t pre_len;    // filled by parse_headers
    uint8_t mode, skip_flags;
    bool copy;
    uint64_t checksum;
    uint64_t data_bit;
    uint64_t end_pos;    // bit position after the entropy data (filled for ANS/Huffman by the walk kernels)
    int32_t status;
    uint32_t block_size; // blockSize of the block's stream: bounds its header's length claim and its decode slot; TEXT sizes its hash map by it
};

}  // namespace kz

struct kz_cache;

struct kz_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t caller_done = nullptr;  // after_caller_work: recorded on the legacy default stream, waited on by `stream`
    std::string err;
    uint64_t launches = 0;
    bool profile = false;
    int bwt_profile = 0;  // kz_bwt_profile: bit 0 times the BWT forward rounds (with profile), bit 1 forces the 56-bit rounds
    kz::EncPlan enc_plan;
    uint64_t user_stream_bs = 0;  // kz_set_stream_block_size: ctx["blockSize"] for the block / single-transform entry points
    int64_t range_from = -1, range_to = -1;  // kz_set_block_range: ctx["from"] / ctx["to"] of the stream-level decodes (-1 = not given)
    bool headerless_writer = false;          // kz_set_headerless_writer: the stream-level encodes write no stream header
    bool skip_blocks = false;                // kz_set_skip_blocks: the encodes store incompressible blocks raw (ctx["skipBlocks"])
    struct Headerless {                      // kz_set_headerless_reader: the stream-level decodes take these instead of a header
        bool on = false;
        uint64_t t48 = 0;
        uint32_t etype = 0, block_size = 0, checksum_bits = 0;
        int64_t output_size = 0;             // 0 = not given
    } headerless_reader;
    std::map<std::string, kz::ProfEntry> prof;
    struct Pending {
        std::string name;
        cudaEvent_t a, b;
    };
    std::vector<Pending> pending;
    std::vector<cudaEvent_t> event_pool;

    // scratch
    kz::DevBuf d_in, d_out, d_tmp, d_tmp2, d_seg, d_chunks, d_tables, d_enc_tab, d_hdr, d_pay, d_small, d_dl, d_rcp, d_ws, d_lens, d_hist;
    // many-stream entry points: copy lists, pass slots, pass entropy output, compact block bit strings, stream assembly / staging
    kz::DevBuf d_copy, d_slots, d_enc, d_bits, d_asm;
    kz::DevBuf d_skip;  // skipBlocks test: block histograms, heads and entropy flags
    kz::PinnedBuf h_stage, h_dl, h_io;  // h_io: packed inputs / outputs of the host-buffer many-stream entry points
    // the open writer / reader session (the end of kz_api.cu), if any; kz_destroy closes it. kz_device_bytes asks it, because its
    // worker thread grows the scratch
    kz::Session* session = nullptr;
    // the block caches made on this context (kz_cache_create) and not freed yet: kz_device_bytes counts their pages, kz_destroy frees them
    std::vector<kz_cache*> caches;

    template <class F>
    void each_dev_buf(F&& f) {
        kz::DevBuf* bufs[] = {&d_in, &d_out, &d_tmp, &d_tmp2, &d_seg, &d_chunks, &d_tables, &d_enc_tab, &d_hdr, &d_pay, &d_small, &d_dl, &d_rcp, &d_ws, &d_lens,
                              &d_hist, &d_copy, &d_slots, &d_enc, &d_bits, &d_asm, &d_skip};
        for (auto b : bufs) f(*b);
    }
    size_t scratch_bytes() {
        size_t s = 0;
        each_dev_buf([&](kz::DevBuf& b) { s += b.cap; });
        return s;
    }

    int fail(int code, const std::string& msg) {
        err = msg;
        return -code;
    }
    int cuda_fail(cudaError_t e, const char* what) {
        err = std::string(what) + ": " + cudaGetErrorString(e);
        return -KZ_E_PROCESS_BLOCK;
    }
};
