// Pass planner of the many-stream entry points (kz_compress_streams / kz_decompress_streams, kz_api.cu), the block cutting and
// per-block decisions of every encode path, and the slot and error-order rules of every stream-level decode. Pure host code: no CUDA
// types, so that tests/host/stream_plan_host.cpp compiles it with g++ and checks it on the CPU.
//
// A pass is a set of blocks that run through the transform and entropy stages together. Every block of a pass gets a slot of the
// pass's stride in the device scratch buffers, so the scratch of a pass is (number of blocks) x cost(stride). The planner keeps that
// product under a fixed budget, and keeps the stride close to every member's length, so that a batch of many small files and one
// large one does not give every small file a slot as long as the large one.
#pragma once
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <string>
#include <vector>

namespace kz {

// Device scratch bytes one pass may take (the block costs below). A block whose own cost is larger runs alone in a pass of its own.
const uint64_t STREAM_PASS_BUDGET = 1ull << 30;

struct PassPlan {
    std::vector<uint32_t> first;       // pass p holds the blocks order[first[p] .. first[p + 1])
    std::vector<uint32_t> order;       // block indexes, pass after pass
    std::vector<uint64_t> stride;      // slot stride of each pass (a multiple of 16)
    std::vector<uint32_t> pass, slot;  // per block: its pass, and its slot inside that pass
    uint64_t scratch = 0;              // largest (blocks of a pass) x cost(stride) over the passes
    uint32_t npasses() const { return (uint32_t)stride.size(); }
};

inline uint64_t round16(uint64_t n) { return (n + 15) & ~15ull; }

const size_t SMALL_BLOCK = 15;  // io/CompressedStream.go:51: blocks of at most this many bytes are stored, whatever the options

// Blocks over a base address: block b is len[b] bytes at off[b]. Cut from streams (cut_blocks), stream s holds blocks
// first[s] .. first[s + 1] - 1; a list that was not cut from streams has first = {0, size()}.
struct BlockList {
    std::vector<uint64_t> off;
    std::vector<uint32_t> len;
    std::vector<uint32_t> first;
    uint32_t size() const { return (uint32_t)len.size(); }
};

// Writer.Write cuts its input into blockSize pieces: stream s (src_len[s] bytes at src_off[s]) becomes blocks of block_size bytes and a
// shorter last one; an empty stream has no blocks.
inline BlockList cut_blocks(const uint64_t* src_off, const uint64_t* src_len, uint32_t nstreams, uint32_t block_size) {
    BlockList L;
    L.first.resize(nstreams + 1);
    for (uint32_t s = 0; s < nstreams; s++) {
        L.first[s] = L.size();
        for (uint64_t o = 0; o < src_len[s]; o += block_size) {
            L.off.push_back(src_off[s] + o);
            L.len.push_back((uint32_t)std::min<uint64_t>(block_size, src_len[s] - o));
        }
    }
    L.first[nstreams] = L.size();
    return L;
}

// The data type encodingTask.encode derives from the first four bytes of a block before the transforms run
// (io/CompressedStream.go:806-816 over internal/Magic.go:73-112 GetMagicType and :116-206 IsDataCompressed / IsDataMultimedia /
// IsDataExecutable): 7 = DT_BIN for compressed containers, 2 = DT_MULTIMEDIA, 3 = DT_EXE, 0 = DT_UNDEFINED otherwise.
inline int32_t magic_data_type(const uint8_t* p, size_t n) {
    if (n < 4) return 0;
    const uint32_t key = ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
    const uint32_t k24 = key >> 8, k16 = key >> 16;
    // compressed: JPEG (APP0 marker only: the other FFD8FFEx keys match no class), GIF, PNG, 7z, zstd, brotli, CAB, ZIP, FLAC, xz, KANZ, RAR,
    // bzip2 / ID3 (24 bits), gzip (16 bits)
    switch (key) {
        case 0xFFD8FFE0u: case 0x47494638u: case 0x89504E47u: case 0x377ABCAFu: case 0x28B52FFDu: case 0x81CFB2CEu: case 0x4D534346u:
        case 0x504B0304u: case 0x664C6143u: case 0xFD377A58u: case 0x4B414E5Au: case 0x52617221u:
            return 7;
        default: break;
    }
    if ((key & ~0x0Fu) == 0xFFD8FFE0u) return 0;  // GetMagicType returns the key itself: no class matches
    if (k24 == 0x425A68u || k24 == 0x494433u) return 7;
    if (key == 0x25504446u) return 0;  // PDF: recognised, in no class
    if (key == 0x52494646u) return 2;  // RIFF
    if (key == 0x7F454C46u || key == 0xFEEDFACEu || key == 0xCEFAEDFEu || key == 0xFEEDFACFu || key == 0xCFFAEDFEu) return 3;  // ELF, Mach-O
    if (k16 == 0x1F8Bu) return 7;  // gzip
    if (k16 == 0x424Du) return 2;  // BMP
    if (k16 == 0x4D5Au) return 3;  // MZ
    if (k16 == 0x5034u || k16 == 0x5035u || k16 == 0x5036u) {  // binary PBM / PGM / PPM: "P4".."P6" followed by white space
        const uint32_t sub = (key >> 8) & 0xFF;
        if (sub == 0x07 || sub == 0x0A || sub == 0x0D || sub == 0x20) return 2;
    }
    return 0;
}

// The blocks and bytes stored_blocks stores for each reason
struct StoreCounts {
    uint64_t magic_blocks = 0, magic_bytes = 0, entropy_blocks = 0, entropy_bytes = 0;
};

// kanzi's skipBlocks option (encodingTask.encode, io/CompressedStream.go:778-800), host half: block b (len[b] bytes, heads[4b ..] its
// first four bytes, zero padded) is stored when it has more than SMALL_BLOCK bytes and its head is the magic number of a compressed
// format (magic_data_type 7: IsDataCompressed(GetMagicType)) or its entropy flag (flags[b], the device half's test) is set. Blocks of at
// most SMALL_BLOCK bytes are stored in any case, by the COPY rule of the forward stage: store[b] stays 0 for them.
inline StoreCounts stored_blocks(const uint8_t* heads, const uint8_t* flags, const uint32_t* len, uint32_t nb, std::vector<uint8_t>& store) {
    StoreCounts c;
    store.assign(nb, 0);
    for (uint32_t b = 0; b < nb; b++) {
        if (len[b] <= SMALL_BLOCK) continue;
        if (magic_data_type(&heads[(size_t)b * 4], len[b]) == 7) {
            store[b] = 1, c.magic_blocks++, c.magic_bytes += len[b];
        } else if (flags[b]) {
            store[b] = 1, c.entropy_blocks++, c.entropy_bytes += len[b];
        }
    }
    return c;
}

// Scratch the entropy stage (encode_batch) takes per chunk of a codec: its chunk size, and fixed + per_byte x (chunk bytes) bytes of
// tables, headers, payload and histograms per chunk. NONE has no chunks (chunk = 0).
struct EntropyScratch {
    uint64_t chunk = 0, fixed = 0, per_byte = 0;
};

// Device bytes one block of a compression pass of stride s takes: its input slot, the two stage buffers of forward_stage (at most
// s + s/8 + 33 bytes per transform + 9,472 bytes each), its entropy output slot (kz_max_block_output(s)) and the entropy stage's
// per-chunk scratch. The transforms' own workspaces are not counted: they are sized per sub-batch of a fixed number of blocks
// (run_desc_stage in kz_api.cu) or per block (BWT, BWTS, LZ), not per pass.
inline uint64_t compress_block_cost(uint64_t s, const EntropyScratch& e) {
    const uint64_t stage = round16(s + s / 8 + 33 * 8 + 8192 + 1024 + 256);
    const uint64_t enc = round16(s + (s >> 3) + 1024 + 64 * (s / 16384 + 1) + 106496 * (s / (4u << 20) + 1));
    const uint64_t chunks = e.chunk ? (s + e.chunk - 1) / e.chunk : 0;
    return s + 2 * stage + enc + chunks * (e.fixed + e.per_byte * std::min(s, e.chunk));
}

// Reader.processBlock (io/CompressedStream.go:1649-1653) sizes each task buffer blockSize + max(512, blockSize >> 4); a decode slot
// holds that plus 64 bytes of slack, and a block takes one slot in each of the two buffers the inverse stages alternate between.
inline uint64_t decompress_slot(uint32_t block_size) { return round16((uint64_t)block_size + std::max<uint64_t>(512, block_size >> 4) + 64); }
inline uint64_t decompress_block_cost(uint32_t block_size) { return 2 * decompress_slot(block_size); }
// The slot stride of a batch of blocks whose longest entropy output is max_pre bytes: decompress_slot, or longer when a block header
// claims more (parse_block_header bounds the claim by max(2048, 1.5 x block_size)).
inline uint64_t decode_stride(uint32_t block_size, uint32_t max_pre) { return std::max(decompress_slot(block_size), round16((uint64_t)max_pre + 64)); }

// The stages of a stream-level block decode (decode_walked in kz_api.cu), in the order they run. STAGE_WALK is the record walk before
// them; STAGE_DONE is past the last stage.
enum DecodeStage { STAGE_WALK = 0, STAGE_HEADER, STAGE_DECODE, STAGE_INVERSE, STAGE_CHECKSUM, STAGE_DONE };

// The failure that decides one stream's status (DESIGN §5.2, "Error order"): the earliest stage wins, and within a stage the earliest
// block. Blocks are noted in block order, so within a stage the failure noted first stays.
struct DecodeFailure {
    int stage = STAGE_DONE;
    int code = 0;     // -(error code)
    std::string msg;  // the message of ctx->err that goes with it
    bool failed() const { return stage != STAGE_DONE; }
    // whether a failure at stage s could still win: the stream's blocks skip every stage that could not
    bool runs(int s) const { return s < stage; }
    void note(int s, int c, const std::string& m) {
        if (!runs(s)) return;
        stage = s;
        code = c;
        msg = m;
    }
};

// Compression: blocks of lengths len[], longest first. A pass opens with the longest block left, whose rounded length is the pass's
// stride s; it admits shorter blocks while s <= 2 x len + 16 and while (blocks + 1) x cost(s) <= budget.
template <class Cost>
PassPlan plan_compress_passes(const std::vector<uint32_t>& len, Cost cost, uint64_t budget = STREAM_PASS_BUDGET) {
    PassPlan P;
    const uint32_t n = (uint32_t)len.size();
    P.order.resize(n);
    std::iota(P.order.begin(), P.order.end(), 0u);
    std::stable_sort(P.order.begin(), P.order.end(), [&](uint32_t a, uint32_t b) { return len[a] > len[b]; });
    P.pass.assign(n, 0);
    P.slot.assign(n, 0);
    auto rlen = [&](uint32_t b) { return round16(std::max<uint64_t>(len[b], 1)); };
    for (uint32_t i = 0; i < n;) {
        const uint32_t p = P.npasses();
        const uint64_t s = rlen(P.order[i]), c = cost(s);
        P.first.push_back(i);
        P.stride.push_back(s);
        uint32_t k = 0;
        while (i < n && s <= 2 * std::max<uint64_t>(len[P.order[i]], 1) + 16 && (k == 0 || (uint64_t)(k + 1) * c <= budget)) {
            P.pass[P.order[i]] = p;
            P.slot[P.order[i]] = k++;
            i++;
        }
        P.scratch = std::max(P.scratch, (uint64_t)k * c);
    }
    P.first.push_back(n);
    return P;
}

// Decompression: a block's decoded length is only bounded by its stream's block size, so every block of a group gets the same stride
// and cost; the budget caps the number of blocks of a pass. Blocks keep their order (stream after stream).
inline PassPlan plan_decompress_passes(uint32_t n, uint64_t stride, uint64_t cost, uint64_t budget = STREAM_PASS_BUDGET) {
    PassPlan P;
    const uint32_t per = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(budget / std::max<uint64_t>(cost, 1), 0xFFFFFFFFu));
    P.order.resize(n);
    std::iota(P.order.begin(), P.order.end(), 0u);
    P.pass.resize(n);
    P.slot.resize(n);
    for (uint32_t i = 0; i < n; i += per) {
        const uint32_t p = P.npasses(), k = std::min(per, n - i);
        P.first.push_back(i);
        P.stride.push_back(stride);
        for (uint32_t j = 0; j < k; j++) {
            P.pass[i + j] = p;
            P.slot[i + j] = j;
        }
        P.scratch = std::max(P.scratch, (uint64_t)k * cost);
    }
    P.first.push_back(n);
    return P;
}

}  // namespace kz
