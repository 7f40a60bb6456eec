// ORACLE — TEST INFRASTRUCTURE ONLY (see kzo.hpp). LZ / LZX codec: greedy hash-table LZ77 with two repeat distances.
// Follows v2/transform/LZCodec.go: LZXCodec.Forward :249-591, findMatchLZX :593-608, emitLengthLZ/readLengthLZ :193-232,
// hash :238-244, inverseV6 :621-778, MaxEncodedLen :935-941. `extra` = LZX (19-bit hash, check at position+2).
#include <algorithm>
#include <cstring>

#include "kzo.hpp"
#include "kzo_transforms.hpp"

namespace kzo {
namespace {
const uint64_t HASH_SEED = 0x1E35A7BD;                     // :29
const int MAX_DISTANCE1 = (1 << 16) - 2;                   // :36
const int MAX_DISTANCE2 = (1 << 24) - 2;                   // :37
const int MIN_MATCH4 = 4, MIN_MATCH6 = 6;                  // :38-39
const int MAX_MATCH = 65535 + 254 + MIN_MATCH4;            // :41
const int MIN_BLOCK_LENGTH = 24;                           // :42

inline uint64_t le64(const uint8_t* p) { uint64_t v; std::memcpy(&v, p, 8); return v; }
inline uint32_t le32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }

inline uint32_t lz_hash(uint64_t v, bool extra) {  // :238-244 (5 low bytes of v)
    return extra ? uint32_t(((v << 24) * HASH_SEED) >> (64 - 19)) : uint32_t(((v << 24) * HASH_SEED) >> (64 - 16));
}

int emit_length(uint8_t* block, int length) {  // :193-213
    if (length < 254) {
        block[0] = uint8_t(length);
        return 1;
    }
    if (length < 65536 + 254) {
        length -= 254;
        block[0] = 254;
        block[1] = uint8_t(length >> 8);
        block[2] = uint8_t(length);
        return 3;
    }
    length -= 255;
    block[0] = 255;
    block[1] = uint8_t(length >> 16);
    block[2] = uint8_t(length >> 8);
    block[3] = uint8_t(length);
    return 4;
}

int find_match(const uint8_t* src, int src_idx, int ref, int max_match) {  // :593-608
    int best = 0;
    while (best + 8 <= max_match) {
        uint64_t diff = le64(src + src_idx + best) ^ le64(src + ref + best);
        if (diff != 0) {
            best += __builtin_ctzll(diff) >> 3;
            break;
        }
        best += 8;
    }
    return best;
}
}  // namespace

size_t lz_max_encoded_len(size_t n) { return n <= 1024 ? n + 16 : n + n / 64; }

bool lz_forward(Ctx& ctx, bool extra, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n) {
    if (n == 0) {
        *out_n = 0;
        return true;
    }
    const int count = int(n);
    if (cap < lz_max_encoded_len(n)) return false;
    if (count < MIN_BLOCK_LENGTH) return false;
    std::vector<int32_t> hashes(size_t(1) << (extra ? 19 : 16), 0);
    const size_t min_buf = std::max<size_t>(n / 5, 256);
    std::vector<uint8_t> m_len_buf(min_buf), m_buf(min_buf), tk_buf(min_buf);
    const int src_end = count - 16 - 2;
    int max_dist = MAX_DISTANCE2;
    dst[12] = 1;
    if (src_end < 4 * MAX_DISTANCE1) {
        max_dist = MAX_DISTANCE1;
        dst[12] = 0;
    }
    int min_match = MIN_MATCH4;
    if (ctx.data_type == DT_DNA) min_match = MIN_MATCH6;
    else if (ctx.data_type == DT_SMALL_ALPHABET) return false;
    dst[12] |= uint8_t(((min_match - 2) & 7) << 1);
    int src_idx = 0, dst_idx = 13, anchor = 0, m_len_idx = 0, m_idx = 0, tk_idx = 0;
    int repd[2] = {count, count};
    int repd_idx = 0, src_inc = 0;
    auto grow = [](std::vector<uint8_t>& v, int used) {
        if (used >= int(v.size()) - 8) v.resize(v.size() + v.size() / 2 + 16);
    };
    while (src_idx < src_end) {
        int best_len = 0;
        const uint32_t h0 = lz_hash(le64(src + src_idx), extra);
        const int ref0 = hashes[h0];
        hashes[h0] = src_idx;
        const uint64_t p = le64(src + src_idx);
        const int src_idx1 = src_idx + 1;
        const int max_match = std::min(src_end - src_idx1, MAX_MATCH);
        int ref = src_idx1 - repd[repd_idx];
        const int min_ref = std::max(src_idx - max_dist, 0);
        if (ref > min_ref && uint32_t(p >> 8) == le32(src + ref)) {  // repeat distances first (:331-345)
            best_len = find_match(src, src_idx1, ref, max_match);
        } else {
            ref = src_idx1 - repd[repd_idx ^ 1];
            if (ref > min_ref && uint32_t(p >> 8) == le32(src + ref)) best_len = find_match(src, src_idx1, ref, max_match);
        }
        if (best_len < min_match) {
            ref = ref0;
            bool found = false;
            if (ref > min_ref && uint32_t(p) == le32(src + ref)) {
                best_len = find_match(src, src_idx, ref, std::min(src_end - src_idx, MAX_MATCH));
                found = best_len >= min_match;
            }
            if (!found) {  // :355-359
                src_idx = src_idx1 + (src_inc >> 6);
                src_inc++;
                repd_idx = 0;
                continue;
            }
            if (ref != src_idx - repd[0] && ref != src_idx - repd[1]) {  // :361-399 lazy checks
                const uint32_t h1 = lz_hash(le64(src + src_idx1), extra);
                const int ref1 = hashes[h1];
                hashes[h1] = src_idx1;
                if (ref1 > min_ref + 1 && le32(src + src_idx1 + best_len - 3) == le32(src + ref1 + best_len - 3)) {
                    const int best_len1 = find_match(src, src_idx1, ref1, max_match);
                    if (best_len1 >= best_len) {
                        ref = ref1;
                        best_len = best_len1;
                        src_idx = src_idx1;
                    }
                }
                if (extra) {
                    const int src_idx2 = src_idx1 + 1;
                    const uint32_t h2 = lz_hash(le64(src + src_idx2), extra);
                    const int ref2 = hashes[h2];
                    hashes[h2] = src_idx2;
                    if (ref2 > min_ref + 2 && le32(src + src_idx2 + best_len - 3) == le32(src + ref2 + best_len - 3)) {
                        const int best_len2 = find_match(src, src_idx2, ref2, std::min(src_end - src_idx2, MAX_MATCH));
                        if (best_len2 >= best_len) {
                            ref = ref2;
                            best_len = best_len2;
                            src_idx = src_idx2;
                        }
                    }
                }
            }
            while (src_idx > anchor && ref > min_ref && src[src_idx - 1] == src[ref - 1]) {  // :402-406 extend backwards
                best_len++;
                ref--;
                src_idx--;
            }
            if (best_len > MAX_MATCH) {
                src_idx += best_len - MAX_MATCH;
                ref += best_len - MAX_MATCH;
                best_len = MAX_MATCH;
            }
        } else {  // :413-422 repeat match found at src_idx+1
            if (src[src_idx] == src[ref - 1] && best_len < MAX_MATCH) {
                best_len++;
                ref--;
            } else {
                src_idx++;
                hashes[lz_hash(le64(src + src_idx), extra)] = src_idx;
            }
        }
        src_inc = 0;
        const int dist = src_idx - ref;
        const int m_len = best_len - min_match;
        int token, m_len_th;
        if (dist == repd[0]) {
            token = 0x00;
            m_len_th = 3;
        } else if (dist == repd[1]) {
            token = 0x04;
            m_len_th = 3;
        } else {
            m_len_th = 7;
            if (dist >= 256) {
                if (dist >= 65536) {
                    m_buf[m_idx] = uint8_t(dist >> 16);
                    m_buf[m_idx + 1] = uint8_t(dist >> 8);
                    m_idx += 2;
                    token = 0x18;
                } else {
                    m_buf[m_idx] = uint8_t(dist >> 8);
                    m_idx++;
                    token = 0x10;
                }
            } else {
                token = 0x08;
            }
            m_buf[m_idx++] = uint8_t(dist);
        }
        if (m_len >= m_len_th) {
            token += m_len_th;
            m_len_idx += emit_length(&m_len_buf[m_len_idx], m_len - m_len_th);
        } else {
            token += m_len;
        }
        repd[1] = repd[0];
        repd[0] = dist;
        repd_idx = 1;
        const int lit_len = src_idx - anchor;
        if (lit_len == 0) {
            tk_buf[tk_idx++] = uint8_t(token);
        } else {
            if (lit_len >= 7) {
                if (lit_len >= (1 << 24)) return false;
                tk_buf[tk_idx++] = uint8_t((7 << 5) | token);
                dst_idx += emit_length(dst + dst_idx, lit_len - 7);
            } else {
                tk_buf[tk_idx++] = uint8_t((lit_len << 5) | token);
            }
            std::memcpy(dst + dst_idx, src + anchor, size_t(lit_len));
            dst_idx += lit_len;
        }
        grow(m_buf, m_idx);
        grow(m_len_buf, m_len_idx);
        grow(tk_buf, tk_idx);
        anchor = src_idx + best_len;  // :505-541: every position inside the match is inserted, in increasing order
        src_idx++;
        while (src_idx < anchor) {
            hashes[lz_hash(le64(src + src_idx), extra)] = src_idx;
            src_idx++;
        }
    }
    const int lit_len = count - anchor;  // :544-577
    if (dst_idx + lit_len + tk_idx + m_idx >= count) return false;
    if (lit_len >= 7) {
        tk_buf[tk_idx++] = uint8_t(7 << 5);
        dst_idx += emit_length(dst + dst_idx, lit_len - 7);
    } else {
        tk_buf[tk_idx++] = uint8_t(lit_len << 5);
    }
    std::memcpy(dst + dst_idx, src + anchor, size_t(lit_len));
    dst_idx += lit_len;
    const uint32_t a = uint32_t(dst_idx), b = uint32_t(tk_idx), c = uint32_t(m_idx);
    std::memcpy(dst, &a, 4);
    std::memcpy(dst + 4, &b, 4);
    std::memcpy(dst + 8, &c, 4);
    std::memcpy(dst + dst_idx, tk_buf.data(), size_t(tk_idx));
    dst_idx += tk_idx;
    std::memcpy(dst + dst_idx, m_buf.data(), size_t(m_idx));
    dst_idx += m_idx;
    std::memcpy(dst + dst_idx, m_len_buf.data(), size_t(m_len_idx));
    dst_idx += m_len_idx;
    if (dst_idx > count - count / 100) return false;  // :586-588
    *out_n = size_t(dst_idx);
    return true;
}

bool lz_inverse(Ctx&, bool, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_n) {
    if (n == 0 || cap == 0) {  // :622-624
        *out_n = 0;
        return true;
    }
    const int64_t count = int64_t(n);
    if (count < 13) return false;
    int64_t tk_idx = le32(src), m_idx = le32(src + 4), m_len_idx = le32(src + 8);
    m_idx += tk_idx;
    m_len_idx += m_idx;
    if (tk_idx > count || m_idx > count || m_len_idx > count) return false;
    const int64_t src_end = tk_idx - 13;
    const int64_t dst_end = int64_t(cap) - 16;
    const int64_t max_dist = (src[12] & 1) ? MAX_DISTANCE2 : MAX_DISTANCE1;
    const int64_t min_match = ((src[12] >> 1) & 7) + 2;
    int64_t src_idx = 13, dst_idx = 0;
    int64_t repd0 = count, repd1 = count;
    auto read_length = [&](int64_t& idx, int64_t limit, bool& ok) -> int64_t {  // :215-232
        if (idx >= limit) { ok = false; return 0; }
        int64_t res = src[idx];
        if (res < 254) { idx += 1; return res; }
        if (res == 254) {
            if (idx + 3 > limit) { ok = false; return 0; }
            res += (int64_t(src[idx + 1]) << 8) + src[idx + 2];
            idx += 3;
            return res;
        }
        if (idx + 4 > limit) { ok = false; return 0; }
        res += (int64_t(src[idx + 1]) << 16) + (int64_t(src[idx + 2]) << 8) + src[idx + 3];
        idx += 4;
        return res;
    };
    bool ok = true;
    for (;;) {
        if (tk_idx >= count) return false;
        const int token = src[tk_idx++];
        if (token >= 32) {
            int64_t lit_len;
            if (token >= 0xE0) {
                lit_len = 7 + read_length(src_idx, count, ok);
                if (!ok) return false;
            } else {
                lit_len = token >> 5;
            }
            if (src_idx + lit_len > count || dst_idx + lit_len > int64_t(cap)) return false;
            std::memcpy(dst + dst_idx, src + src_idx, size_t(lit_len));
            src_idx += lit_len;
            dst_idx += lit_len;
            if (src_idx >= src_end) break;
        }
        int64_t m_len, dist;
        const int f = token & 0x18;
        if (f == 0) {
            m_len = token & 3;
            if (m_len == 3) {
                m_len += min_match + read_length(m_len_idx, count, ok);
                if (!ok) return false;
            } else {
                m_len += min_match;
            }
            dist = (token & 4) == 0 ? repd0 : repd1;
        } else {
            m_len = token & 7;
            if (m_len == 7) {
                m_len += min_match + read_length(m_len_idx, count, ok);
                if (!ok) return false;
            } else {
                m_len += min_match;
            }
            const int nb = f == 0x18 ? 3 : (f == 0x10 ? 2 : 1);
            if (m_idx + nb > count) return false;
            dist = src[m_idx++];
            if (f >= 0x10) {
                dist = (dist << 8) | src[m_idx++];
                if (f == 0x18) dist = (dist << 8) | src[m_idx++];
            }
        }
        repd1 = repd0;
        repd0 = dist;
        const int64_t m_end = dst_idx + m_len;
        const int64_t ref = dst_idx - dist;
        if (ref < 0 || dist > max_dist || m_end > dst_end) return false;
        for (int64_t i = 0; i < m_len; i++) dst[dst_idx + i] = dst[ref + i];  // byte-wise copy == the 16-byte block copy for dist >= 16
        dst_idx = m_end;
    }
    if (src_idx != src_end + 13) return false;
    *out_n = size_t(dst_idx);
    return true;
}

}  // namespace kzo
