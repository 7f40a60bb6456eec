// ORACLE — TEST INFRASTRUCTURE ONLY (see kzo.hpp). Pre-transforms of the `-l 2..4` chains, restated from
//   PACK / DNA : v2/transform/AliasCodec.go   (AliasCodec.Forward :74-273, Inverse :278-434, MaxEncodedLen :437-439)
//   MM         : v2/transform/FSDCodec.go     (FSDCodec.Forward :135-312, Inverse :317-404, MaxEncodedLen :128-130)
//   UTF        : v2/transform/UTFCodec.go     (UTFCodec.Forward :87-262, Inverse :267-383, validateUTF :393-515, packUTF :517-545,
//                                              unpackUTF1 :577-610)
// "return false" = the reference returns an error (forward: skip this transform; inverse: fatal for the block).
// PARITY PINNING: like the rest of the oracle (no Go toolchain, no byte-level vectors in the reference's tests) — round trips plus
// the structural checks of tests/test_oracle_pre.py.
#include <algorithm>
#include <cstring>
#include <vector>

#include "kzo.hpp"
#include "kzo_transforms.hpp"

namespace kzo {

// ------------------------------------------------------------------------------------------------------------------
// PACK / DNA (AliasCodec)
// ------------------------------------------------------------------------------------------------------------------
size_t alias_max_encoded_len(size_t n) { return n + 1024; }  // :437-439

bool alias_forward(Ctx& ctx, bool only_dna, const uint8_t* src, size_t count, uint8_t* dst, size_t cap, size_t* out_n) {
    *out_n = 0;
    if (count == 0) return true;
    if (cap < alias_max_encoded_len(count)) return false;  // :83-85
    if (count < 1024) return false;                        // _ALIAS_MIN_BLOCKSIZE :87-89
    int dt = ctx.data_type;                                // :91-110
    if (dt == DT_MULTIMEDIA || dt == DT_UTF8) return false;
    if (dt == DT_EXE || dt == DT_BIN) return false;
    if (only_dna && dt != DT_UNDEFINED && dt != DT_DNA) return false;
    // :112-127 missing 1-byte symbols
    std::vector<int> freqs0(256, 0);
    histogram_order0(src, count, freqs0.data());
    int n0 = 0;
    int absent[256];
    for (int i = 0; i < 256; i++)
        if (freqs0[i] == 0) absent[n0++] = i;
    if (n0 < 16) return false;
    if (dt == DT_UNDEFINED) {  // :129-139
        dt = detect_simple_type(count, freqs0.data());
        if (dt != DT_UNDEFINED) ctx.data_type = dt;
        if (dt != DT_DNA && only_dna) return false;
    }
    size_t src_idx = 0, dst_idx = 0;
    if (n0 >= 240) {  // :145-207 small alphabet: pack 4 or 2 symbols per byte
        dst[0] = uint8_t(n0);
        if (n0 == 255) {  // one symbol
            dst[1] = src[0];
            const uint32_t c = uint32_t(count);
            dst[2] = uint8_t(c);
            dst[3] = uint8_t(c >> 8);
            dst[4] = uint8_t(c >> 16);
            dst[5] = uint8_t(c >> 24);
            src_idx = count;
            dst_idx = 6;
        } else {
            uint8_t map8[256] = {0};
            dst_idx = 1;
            int j = 0;
            for (int i = 0; i < 256; i++)
                if (freqs0[i] != 0) {
                    dst[dst_idx++] = uint8_t(i);
                    map8[i] = uint8_t(j++);
                }
            if (n0 >= 252) {  // 4 symbols or less
                const size_t c3 = count & 3;
                dst[dst_idx++] = uint8_t(c3);
                std::memcpy(dst + dst_idx, src, c3);
                src_idx += c3;
                dst_idx += c3;
                while (src_idx < count) {
                    dst[dst_idx++] = uint8_t((map8[src[src_idx]] << 6) | (map8[src[src_idx + 1]] << 4) | (map8[src[src_idx + 2]] << 2) | map8[src[src_idx + 3]]);
                    src_idx += 4;
                }
            } else {  // 16 symbols or less
                dst[dst_idx++] = uint8_t(count & 1);
                if (count & 1) dst[dst_idx++] = src[src_idx++];
                while (src_idx < count) {
                    dst[dst_idx++] = uint8_t((map8[src[src_idx]] << 4) | map8[src[src_idx + 1]]);
                    src_idx += 2;
                }
            }
        }
    } else {  // :208-287 digram aliasing
        // ComputeHistogram(order 1, no totals) = counts of (prev << 8 | cur) with prev = 0 for the first byte (Global.go:305-341)
        std::vector<int> freqs1(65536, 0);
        {
            unsigned prv = 0;
            for (size_t i = 0; i < count; i++) {
                freqs1[(prv << 8) | src[i]]++;
                prv = src[i];
            }
        }
        struct Sd {
            int val, freq;
        };
        std::vector<Sd> symb;
        symb.reserve(65536);
        for (int i = 0; i < 65536; i++)
            if (freqs1[i] != 0) symb.push_back({i, freqs1[i]});
        const int n1 = int(symb.size());
        if (n0 > n1) {
            n0 = n1;
            if (n0 < 16) return false;
        }
        // decreasing frequency, then decreasing value (total order: stability is irrelevant)
        std::stable_sort(symb.begin(), symb.end(), [](const Sd& a, const Sd& b) { return a.freq != b.freq ? a.freq > b.freq : a.val > b.val; });
        std::vector<int16_t> map16(65536);
        for (int i = 0; i < 65536; i++) map16[i] = int16_t(0x100 | (i >> 8));
        int savings = 0;
        dst[0] = uint8_t(n0);
        dst[1] = 0;
        dst_idx = 2;
        for (int i = 0; i < n0; i++) {
            savings += symb[i].freq;
            const int idx = symb[i].val;
            map16[idx] = int16_t(0x200 | absent[i]);
            dst[dst_idx] = uint8_t(idx >> 8);
            dst[dst_idx + 1] = uint8_t(idx);
            dst[dst_idx + 2] = uint8_t(absent[i]);
            dst_idx += 3;
        }
        if (savings < int(count / 20)) return false;
        const size_t src_end = count - 1;
        while (src_idx < src_end) {
            const int alias = map16[(int(src[src_idx]) << 8) | src[src_idx + 1]];
            dst[dst_idx++] = uint8_t(alias);
            src_idx += size_t(alias >> 8);
        }
        if (src_idx != count) {
            dst[1] = 1;
            dst[dst_idx++] = src[src_idx++];
        }
    }
    if (dst_idx >= count) return false;  // :289-291
    *out_n = dst_idx;
    return true;
}

bool alias_inverse(const uint8_t* src, size_t len, uint8_t* dst, size_t cap, size_t* out_n) {
    *out_n = 0;
    if (len == 0 || cap == 0) return true;  // :298-300
    if (len < 2) return false;
    int n = src[0];
    if (n < 16) return false;
    size_t src_idx = 0, dst_idx = 0;
    if (n >= 240) {
        const size_t src_end = len;
        n = 256 - n;
        src_idx = 1;
        if (n == 1) {
            if (len < 6) return false;  // the reference would panic on the 4-byte read -> block error
            const uint8_t val = src[1];
            const size_t osize = size_t(src[2]) | (size_t(src[3]) << 8) | (size_t(src[4]) << 16) | (size_t(src[5]) << 24);
            if (osize > cap) return false;
            std::memset(dst, val, osize);
            src_idx = src_end;
            dst_idx = osize;
        } else {
            uint8_t idx2symb[16] = {0};
            if (src_idx + size_t(n) + 1 > len) return false;  // out-of-range read in the reference = panic = block error
            for (int i = 0; i < n; i++) idx2symb[i] = src[src_idx++];
            const int adjust = src[src_idx++];
            if (adjust < 0 || adjust > 3) return false;
            if (n <= 4) {
                if (src_idx + size_t(adjust) > len) return false;
                if (dst_idx + size_t(adjust) + 4 * (src_end - src_idx - size_t(adjust)) > cap) return false;
                std::memcpy(dst + dst_idx, src + src_idx, size_t(adjust));
                src_idx += size_t(adjust);
                dst_idx += size_t(adjust);
                while (src_idx < src_end) {
                    const int v = src[src_idx++];
                    dst[dst_idx] = idx2symb[(v >> 6) & 3];
                    dst[dst_idx + 1] = idx2symb[(v >> 4) & 3];
                    dst[dst_idx + 2] = idx2symb[(v >> 2) & 3];
                    dst[dst_idx + 3] = idx2symb[v & 3];
                    dst_idx += 4;
                }
            } else {
                if (adjust != 0) {
                    if (src_idx >= len || dst_idx >= cap) return false;
                    dst[dst_idx++] = src[src_idx++];
                }
                if (dst_idx + 2 * (src_end - src_idx) > cap) return false;
                while (src_idx < src_end) {
                    const int v = src[src_idx++];
                    dst[dst_idx] = idx2symb[v >> 4];
                    dst[dst_idx + 1] = idx2symb[v & 0x0F];
                    dst_idx += 2;
                }
            }
        }
    } else {
        int map16[256];
        if (2 + 3 * size_t(n) > len) return false;  // the map is read whole (:415-418); src[1] may reach into it or past the start (:408)
        const size_t src_end = size_t(src[1]) < len ? len - src[1] : 0;
        src_idx = 2;
        for (int i = 0; i < 256; i++) map16[i] = 0x10000 | i;
        for (int i = 0; i < n; i++) {
            map16[src[src_idx + 2]] = 0x20000 | int(src[src_idx]) | (int(src[src_idx + 1]) << 8);
            src_idx += 3;
        }
        while (src_idx < src_end) {
            const int val = map16[src[src_idx++]];
            if (dst_idx + 2 > cap) return false;
            dst[dst_idx] = uint8_t(val);
            dst[dst_idx + 1] = uint8_t(val >> 8);
            dst_idx += size_t(val >> 16);
        }
        if (src[1] != 0) {
            if (src_idx >= len || dst_idx >= cap) return false;
            dst[dst_idx++] = src[src_idx++];
        }
    }
    *out_n = dst_idx;
    return true;
}

// ------------------------------------------------------------------------------------------------------------------
// MM (FSDCodec: fixed step delta)
// ------------------------------------------------------------------------------------------------------------------
size_t fsd_max_encoded_len(size_t n) { return n + std::max<size_t>(n >> 4, 64); }  // :128-130

namespace {
// _FSD_ZIGZAG1 (:30-63): index 127 + delta, delta in [-127, 127] -> zigzag(delta); index 255 unused (= 255)
inline uint8_t zigzag1(int d) { return d < 127 ? uint8_t(253 - 2 * d) : (d == 255 ? 255 : uint8_t(2 * (d - 127))); }
// _FSD_ZIGZAG2 (:65-98): inverse, 255 -> -128
inline int zigzag2(int z) { return (z & 1) ? -((z + 1) >> 1) : (z >> 1); }
}  // namespace

bool fsd_forward(Ctx& ctx, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n) {
    *out_n = 0;
    if (n == 0) return true;
    const int count = int(n);
    const int dst_end = int(fsd_max_encoded_len(n));
    if (cap < size_t(dst_end)) return false;
    if (count < 1024) return false;  // _FSD_MIN_BLOCK_LENGTH
    if (ctx.data_type != DT_UNDEFINED && ctx.data_type != DT_MULTIMEDIA && ctx.data_type != DT_BIN) return false;  // :160-168
    const uint32_t magic = get_magic_type(src, n);
    switch (magic) {  // :170-187 BMP, RIFF, PBM, PGM, PPM, none
        case 0x424Du: case 0x52494646u: case 0x5034u: case 0x5035u: case 0x5036u: case 0u: break;
        default: return false;
    }
    const int count10 = count / 10;
    const int count5 = 2 * count10;
    const uint8_t* in0 = src;
    const uint8_t* in1 = src + 2 * count5;
    const uint8_t* in2 = src + 4 * count5;
    static const int distances[7] = {0, 1, 2, 3, 4, 8, 16};
    std::vector<int> histo(7 * 256, 0);
    for (int i = count10; i < count5; i++) {  // :197-222
        const uint8_t* ins[3] = {in0, in1, in2};
        for (const uint8_t* in : ins) {
            const uint8_t b = in[i];
            histo[b]++;
            for (int k = 1; k < 7; k++) histo[k * 256 + (b ^ in[i - distances[k]])]++;
        }
    }
    int ent[7];
    int min_idx = 0;
    for (int i = 0; i < 7; i++) {
        ent[i] = first_order_entropy_1024(size_t(3 * count10), &histo[i * 256]);
        if (ent[i] < ent[min_idx]) min_idx = i;
    }
    if (ent[min_idx] >= ent[0]) {  // :236-243
        ctx.data_type = detect_simple_type(size_t(3 * count10), &histo[0]);
        return false;
    }
    ctx.data_type = DT_MULTIMEDIA;
    const int dist = distances[min_idx];
    int large_deltas = 0;
    for (int i = 2 * count5; i < 3 * count5; i++) {  // :253-260
        const int delta = int(src[i]) - int(src[i - dist]);
        if (delta < -127 || delta > 127) large_deltas++;
    }
    const uint8_t mode = large_deltas > (count5 >> 5) ? 1 : 0;  // xor coding : delta coding
    dst[0] = mode;
    dst[1] = uint8_t(dist);
    int src_idx = 0, dst_idx = 2;
    for (int i = 0; i < dist; i++) dst[dst_idx++] = src[src_idx++];
    if (mode == 0) {
        while (src_idx < count && dst_idx < dst_end - 1) {
            const int delta = 127 + int(src[src_idx]) - int(src[src_idx - dist]);
            if (delta >= 0 && delta < 255) {
                dst[dst_idx++] = zigzag1(delta);
                src_idx++;
                continue;
            }
            dst[dst_idx] = 0xFF;  // escape
            dst[dst_idx + 1] = src[src_idx] ^ src[src_idx - dist];
            src_idx++;
            dst_idx += 2;
        }
    } else {
        while (src_idx < count) {
            dst[dst_idx++] = src[src_idx] ^ src[src_idx - dist];
            src_idx++;
        }
    }
    if (src_idx != count) return false;
    // :296-310 extra check on two sub-blocks of the output
    std::vector<int> h0(256, 0);
    const uint8_t* out1 = dst + 1 * count5;
    const uint8_t* out2 = dst + 3 * count5;
    for (int i = 0; i < count10; i++) {
        h0[out1[i]]++;
        h0[out2[i]]++;
    }
    *out_n = size_t(dst_idx);
    if (first_order_entropy_1024(size_t(count5), h0.data()) >= ent[0]) return false;
    return true;
}

bool fsd_inverse(const uint8_t* src, size_t len, uint8_t* dst, size_t cap, size_t* out_n) {
    *out_n = 0;
    if (len == 0 || cap == 0) return true;  // :327-329
    if (len < 2) return false;
    const uint8_t mode = src[0];
    const int dist = src[1];
    if (dist < 1 || (dist > 4 && dist != 8 && dist != 16)) return false;
    const size_t src_end = len, dst_end = cap;
    size_t src_idx = 2, dst_idx = 0;
    if (src_end - src_idx < size_t(dist)) return false;
    if (dst_end < size_t(dist)) return false;
    for (int i = 0; i < dist; i++) dst[dst_idx++] = src[src_idx++];
    bool ok = true;
    if (mode == 0) {
        while (src_idx < src_end && dst_idx < dst_end) {
            if (src[src_idx] != 0xFF) {
                dst[dst_idx] = uint8_t(int(dst[dst_idx - dist]) + zigzag2(src[src_idx]));
                src_idx++;
                dst_idx++;
                continue;
            }
            src_idx++;
            if (src_idx >= src_end) {
                ok = false;
                break;
            }
            dst[dst_idx] = src[src_idx] ^ dst[dst_idx - dist];
            src_idx++;
            dst_idx++;
        }
    } else if (mode == 1) {
        while (src_idx < src_end && dst_idx < dst_end) {
            dst[dst_idx] = src[src_idx] ^ dst[dst_idx - dist];
            dst_idx++;
            src_idx++;
        }
    } else {
        return false;
    }
    if (src_idx != src_end) ok = false;
    *out_n = dst_idx;
    return ok;
}

// ------------------------------------------------------------------------------------------------------------------
// UTF (UTFCodec)
// ------------------------------------------------------------------------------------------------------------------
size_t utf_max_encoded_len(size_t n) { return n + 8192; }  // :386-388

namespace {
// _UTF_SIZES (:31-48): length of the sequence introduced by a leading byte, 0 = not a valid leading byte
inline int utf_size(uint8_t b) {
    if (b < 0x80) return 1;
    if (b < 0xC2) return 0;
    if (b < 0xE0) return 2;
    if (b < 0xF0) return 3;
    if (b < 0xF5) return 4;
    return 0;
}
// packUTF :517-545
inline int pack_utf(const uint8_t* in, uint32_t* out) {
    const int s = utf_size(in[0]);
    switch (s) {
        case 1: *out = in[0]; break;
        case 2: *out = (1u << 19) | (uint32_t(in[0]) << 8) | in[1]; break;
        case 3: *out = (2u << 19) | ((uint32_t(in[0]) & 0x0F) << 12) | ((uint32_t(in[1]) & 0x3F) << 6) | (uint32_t(in[2]) & 0x3F); break;
        case 4:
            *out = (4u << 19) | ((uint32_t(in[0]) & 0x07) << 18) | ((uint32_t(in[1]) & 0x3F) << 12) | ((uint32_t(in[2]) & 0x3F) << 6) | (uint32_t(in[3]) & 0x3F);
            break;
        default: *out = 0; break;
    }
    return s;
}
// unpackUTF1 :577-610 (bitstream >= 4)
inline int unpack_utf1(uint32_t in, uint8_t* out) {
    const uint32_t sz = in >> 19;
    if (sz == 0) {
        out[0] = uint8_t(in);
        return 1;
    }
    if (sz == 1) {
        out[0] = uint8_t(in >> 8);
        out[1] = uint8_t(in);
        return 2;
    }
    if (sz == 2) {
        out[0] = uint8_t(((in >> 12) & 0x0F) | 0xE0);
        out[1] = uint8_t(((in >> 6) & 0x3F) | 0x80);
        out[2] = uint8_t((in & 0x3F) | 0x80);
        return 3;
    }
    if (sz >= 4 && sz <= 7) {
        out[0] = uint8_t(((in >> 18) & 0x07) | 0xF0);
        out[1] = uint8_t(((in >> 12) & 0x3F) | 0x80);
        out[2] = uint8_t(((in >> 6) & 0x3F) | 0x80);
        out[3] = uint8_t((in & 0x3F) | 0x80);
        return 4;
    }
    return 0;
}
// validateUTF :393-515. The early exits of the reference (:418-429, every 4096 bytes) test the same condition as the final one
// on a prefix of the counts, so "any forbidden leading byte anywhere" decides; the digram rules follow.
bool validate_utf(const uint8_t* block, size_t count) {
    std::vector<int> freqs0(256, 0);
    std::vector<int> freqs1(65536, 0);
    uint8_t prv = 0;
    for (size_t i = 0; i < count; i++) {
        const uint8_t cur = block[i];
        freqs0[cur]++;
        freqs1[(size_t(prv) << 8) | cur]++;
        prv = cur;
    }
    {
        // 1-byte rules. In the reference the check after the loop only runs when count is not a multiple of 4, and the in-loop
        // check (i & 0xFFF == 0) sees the counts up to and including the 4 bytes at i: a forbidden byte in the last partial window
        // of a multiple-of-4 block is not caught here — it is caught later by packUTF returning 0 (Forward :158-176).
        const size_t end4 = count & ~size_t(3);
        size_t checked = 0;  // number of leading bytes covered by the last executed check
        if (end4 != count) checked = count;
        else if (end4 > 0) checked = ((end4 - 4) & ~size_t(0xFFF)) + 4;
        std::vector<int> f(256, 0);
        for (size_t i = 0; i < checked; i++) f[block[i]]++;
        int sum = f[0xC0] + f[0xC1];
        for (int i = 0xF5; i < 256; i++) sum += f[i];
        if (sum != 0) return false;
    }
    int sum = 0, sum2 = 0;
    auto f1 = [&](int a, int b) { return freqs1[(a << 8) | b]; };
    for (int i = 0; i < 256; i++) {
        if (i < 0xA0 || i > 0xBF) sum += f1(0xE0, i);
        if (i < 0x80 || i > 0x9F) sum += f1(0xED, i);
        if (i < 0x90 || i > 0xBF) sum += f1(0xF0, i);
        if (i < 0x80 || i > 0x8F) sum += f1(0xF4, i);
        if (i < 0x80 || i > 0xBF) {
            for (int j = 0xC2; j <= 0xDF; j++) sum += f1(j, i);
            for (int j = 0xE1; j <= 0xEC; j++) sum += f1(j, i);
            sum += f1(0xF1, i) + f1(0xF2, i) + f1(0xF3, i);
            sum += f1(0xEE, i);
            sum += f1(0xEF, i);
        } else {
            sum2 += freqs0[i];
        }
        if (sum != 0) return false;
    }
    return sum2 >= int(count / 8);
}
}  // namespace

bool utf_forward(Ctx& ctx, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n) {
    *out_n = 0;
    if (n == 0) return true;
    if (n < 1024) return false;  // _UTF_MIN_BLOCKSIZE
    if (cap < utf_max_encoded_len(n)) return false;
    const int count = int(n);
    bool must_validate = true;
    if (ctx.data_type != DT_UNDEFINED && ctx.data_type != DT_UTF8) return false;  // :105-114
    must_validate = ctx.data_type != DT_UTF8;
    int start = 0;
    if (src[1] == 0xEF && src[2] == 0xBB && src[3] == 0xBF) {  // BigEndian.Uint32(src) & 0x00FFFFFF == 0xEFBBBF (:119)
        start = 3;
    } else {
        while (start < 4 && utf_size(src[start]) == 0) start++;
    }
    if (must_validate && !validate_utf(src + start, size_t(count - 4 - start))) return false;
    ctx.data_type = DT_UTF8;
    std::vector<int32_t> alias_map(size_t(1) << 22, 0);
    struct Sd {
        int32_t sym, freq;
    };
    std::vector<Sd> symb;
    int nsym = 0;
    for (int i = start; i < count - 4;) {  // :146-170
        uint32_t val;
        const int s = pack_utf(src + i, &val);
        bool res = s != 0;
        res = res && (s != 3 || (src[i + 2] & 0xC0) == 0x80);
        res = res && (s != 4 || ((((uint32_t(src[i + 2]) << 8) | src[i + 3]) & 0xC0C0u) == 0x8080u));
        if (alias_map[val] == 0) {
            symb.push_back({int32_t(val), 0});
            nsym++;
            res = res && nsym < 32768;
        }
        if (!res) return false;
        alias_map[val]++;
        i += s;
    }
    if (nsym == 0) return false;
    const int max_target = count - count / 10;
    if (3 * nsym + 6 >= max_target) return false;
    for (int i = 0; i < nsym; i++) symb[i].freq = alias_map[symb[i].sym];
    // increasing frequency, then increasing symbol (total order)
    std::stable_sort(symb.begin(), symb.end(), [](const Sd& a, const Sd& b) { return a.freq != b.freq ? a.freq < b.freq : a.sym < b.sym; });
    int dst_idx = 2;
    dst[dst_idx++] = uint8_t(nsym >> 8);
    dst[dst_idx++] = uint8_t(nsym);
    int estimate = dst_idx + 6;
    for (int i = 0; i < nsym; i++) {
        const int r = nsym - 1 - i;
        const int32_t s = symb[r].sym;
        dst[dst_idx] = uint8_t(s >> 16);
        dst[dst_idx + 1] = uint8_t(s >> 8);
        dst[dst_idx + 2] = uint8_t(s);
        dst_idx += 3;
        if (i < 128) {
            estimate += symb[r].freq;
            alias_map[s] = i;
        } else {
            estimate += 2 * symb[r].freq;
            alias_map[s] = 0x10080 | ((i << 1) & 0xFF00) | (i & 0x7F);
        }
    }
    if (estimate >= max_target) return false;
    for (int i = 0; i < start; i++) dst[dst_idx++] = src[i];
    int src_idx = start;
    while (src_idx < count - 4) {
        uint32_t val;
        src_idx += pack_utf(src + src_idx, &val);
        const int32_t alias = alias_map[val];
        dst[dst_idx++] = uint8_t(alias);
        dst[dst_idx] = uint8_t(alias >> 8);
        dst_idx += alias >> 16;
    }
    dst[0] = uint8_t(start);
    dst[1] = uint8_t(src_idx - (count - 4));
    while (src_idx < count) dst[dst_idx++] = src[src_idx++];
    *out_n = size_t(dst_idx);
    if (dst_idx >= max_target) return false;
    return true;
}

bool utf_inverse(const uint8_t* src, size_t len, uint8_t* dst, size_t cap, size_t* out_n) {
    *out_n = 0;
    if (len == 0) return true;
    if (len < 4) return false;
    const int count = int(len);
    const int start = src[0] & 3;
    const int adjust = src[1] & 3;
    const int n = (int(src[2]) << 8) + src[3];
    if (n == 0 || n >= 32768 || 4 + 3 * n > count) return false;
    struct Sym {
        uint8_t value[4];
        uint8_t length;
    };
    std::vector<Sym> m(size_t(n), Sym{{0, 0, 0, 0}, 0});
    int src_idx = 4;
    for (int i = 0; i < n; i++) {
        const uint32_t s = (uint32_t(src[src_idx]) << 16) | (uint32_t(src[src_idx + 1]) << 8) | src[src_idx + 2];
        const int sl = unpack_utf1(s, m[i].value);
        if (sl == 0) return false;
        m[i].length = uint8_t(sl);
        src_idx += 3;
    }
    const int src_end = count - 4 + adjust;
    int dst_idx = 0;
    const int dst_end = int(cap) - 4;
    if (dst_end < 0) return false;
    if (src_end < src_idx || src_end > count || src_idx + start > count) return false;
    for (int i = 0; i < start; i++) dst[dst_idx++] = src[src_idx++];
    while (src_idx < src_end && dst_idx < dst_end) {
        int alias = src[src_idx++];
        if (alias >= 128) {
            if (src_idx >= src_end) return false;
            alias = (int(src[src_idx]) << 7) + (alias & 0x7F);
            src_idx++;
        }
        if (alias >= n) return false;  // entries past n are zero-length symbols in the reference: the block cannot round-trip
        const Sym& s = m[size_t(alias)];
        std::memcpy(dst + dst_idx, s.value, 4);
        dst_idx += s.length;
    }
    if (src_idx < src_end || dst_idx > int(cap) - count + src_end) return false;
    for (int i = src_end; i < count; i++) dst[dst_idx++] = src[src_idx++];
    *out_n = size_t(dst_idx);
    return true;
}

}  // namespace kzo
