// Reduced offset LZ (kanzi ROLZ, rolzCodec1: literals / tokens / lengths / match indexes coded with static rANS) on sm_90a.
//
// Reference semantics reproduced bit-exactly (paths relative to the reference's v2/ directory):
//   transform/ROLZCodec.go:57-86 keys, hash, emitCopy; :246-296 findMatch; :301-596 Forward; :601-913 Inverse;
//   :916-971 MaxEncodedLen, emitLengthROLZ, readLengthROLZ; internal/Global.go:346-419 DetectSimpleType;
//   entropy/ANSRangeCodec.go (order 0 with 32 KiB chunks for tokens / lengths / indexes, order 0 or 1 for literals) and
//   entropy/EntropyUtils.go:123-260 NormalizeFrequencies, restated here for ONE thread.
//
// What the format allows: the match table (16 positions per 2-byte context, replaced round robin) is state that the
// decoder rebuilds while it decodes, and the encoder's choices depend on it position by position: one serial chain per
// block in both directions, and the four byte streams of a chunk are entropy coded inside the transform. First correct
// path: one warp per block, lane 0 walks the chain (parse / replay and the nested rANS coding), the other lanes only
// help with clearing tables and copying. Blocks of a batch run concurrently. This is far from the CPU's speed per block
// (same verdict as the survey: adaptive / serial stages do not map to a GPU); it exists for format coverage and parity.
#include "kz_rolz.cuh"

namespace kz {

namespace {

const uint32_t RZ_HASH_SIZE = 1 << 16;
const int RZ_MIN3 = 3, RZ_MIN4 = 4, RZ_MIN7 = 7;
const int RZ_MAX_MATCH1 = RZ_MIN3 + 65535;
const int RZ_LOG_POS = 4;
const int RZ_CHUNK = 16 * 1024 * 1024;
const uint32_t RZ_HASH_MASK = ~(uint32_t)(RZ_CHUNK - 1);
const uint64_t RZ_SEED = 200002979ull;
const int RZ_ANS_TOP = 1 << 15;

KZ_D uint32_t rz_le16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
KZ_D uint32_t rz_le32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
KZ_D uint64_t rz_le64(const uint8_t* p) { return (uint64_t)rz_le32(p) | ((uint64_t)rz_le32(p + 4) << 32); }
KZ_D uint32_t rz_key1(const uint8_t* p) { return rz_le16(p); }
KZ_D uint32_t rz_key2(const uint8_t* p) { return (uint32_t)((rz_le64(p) * RZ_SEED) >> 40) & 0xFFFFu; }
KZ_D uint32_t rz_hash(const uint8_t* p) { return ((rz_le32(p) << 8) * (uint32_t)RZ_SEED) & RZ_HASH_MASK; }

KZ_D int rz_emit_length(uint8_t* block, int lit_len) {  // :921-943
    int idx = 0;
    if (lit_len >= 1 << 7) {
        if (lit_len >= 1 << 14) {
            if (lit_len >= 1 << 21) block[idx++] = (uint8_t)(0x80 | (lit_len >> 21));
            block[idx++] = (uint8_t)(0x80 | (lit_len >> 14));
        }
        block[idx++] = (uint8_t)(0x80 | (lit_len >> 7));
    }
    block[idx] = (uint8_t)(lit_len & 0x7F);
    return idx + 1;
}
KZ_D int rz_read_length(const uint8_t* buf, int* idx_out) {  // :946-971
    uint32_t next = buf[0];
    int idx = 1;
    int lit_len = (int)(next & 0x7F);
    if (next >= 128) {
        next = buf[idx++];
        lit_len = (lit_len << 7) | (int)(next & 0x7F);
        if (next >= 128) {
            next = buf[idx++];
            lit_len = (lit_len << 7) | (int)(next & 0x7F);
            if (next >= 128) {
                next = buf[idx++];
                lit_len = (lit_len << 7) | (int)(next & 0x7F);
            }
        }
    }
    *idx_out = idx;
    return lit_len;
}

// ---- serial MSB-first bit I/O over global memory (private stream of a ROLZ chunk: starts byte aligned)
struct RzWriter {
    uint8_t* p;        // next byte to write
    const uint8_t* lim;
    uint64_t acc;      // pending bits, right aligned
    uint32_t n;        // pending bit count (< 8 after every call)
    bool over;
    KZ_D void init(uint8_t* dst, const uint8_t* limit) {
        p = dst;
        lim = limit;
        acc = 0;
        n = 0;
        over = false;
    }
    KZ_D void put(uint64_t v, uint32_t bits) {  // bits <= 32
        acc = (acc << bits) | (v & ((1ull << bits) - 1ull));
        n += bits;
        while (n >= 8) {
            n -= 8;
            if (p < lim) *p = (uint8_t)(acc >> n);
            else over = true;
            p++;
        }
    }
    KZ_D void put_bytes(const uint8_t* b, uint32_t cnt) {
        for (uint32_t i = 0; i < cnt; i++) put(b[i], 8);
    }
    KZ_D void close() {  // zero padding to a byte (DefaultOutputBitStream.Close)
        if (n) put(0, 8 - n);
    }
};
struct RzReader {
    const uint8_t* base;
    uint64_t pos, end;  // bits
    bool over;
    KZ_D void init(const uint8_t* b, uint64_t nbytes) {
        base = b;
        pos = 0;
        end = 8 * nbytes;
        over = false;
    }
    KZ_D uint32_t get(uint32_t bits) {  // bits <= 32
        if (pos + bits > end) {
            over = true;
            pos += bits;
            return 0;
        }
        uint64_t v = 0;
        const uint64_t b0 = pos >> 3;
        const uint32_t o = (uint32_t)pos & 7;
        const uint32_t nb = (o + bits + 7) >> 3;  // <= 5
        for (uint32_t i = 0; i < nb; i++) v = (v << 8) | base[b0 + i];
        pos += bits;
        return (uint32_t)((v >> (8 * nb - o - bits)) & ((1ull << bits) - 1ull));
    }
    KZ_D uint32_t varint() {  // EntropyUtils.go:278-296
        uint32_t res = 0, shift = 0;
        for (int i = 0; i < 4; i++) {
            const uint32_t v = get(8);
            res |= (v & 0x7F) << shift;
            if (v < 128) return res;
            shift += 7;
        }
        return res | ((get(8) & 0x0F) << 28);
    }
};

// ---- NormalizeFrequencies (EntropyUtils.go:123-260), one thread. freqs[256] in/out, alphabet[256] out; returns alphabet size
KZ_D int rz_normalize(int* freqs, int* alphabet, int total, int scale) {
    if (total == 0) return 0;
    int asz = 0;
    if (total == scale) {
        for (int i = 0; i < 256; i++)
            if (freqs[i] != 0) alphabet[asz++] = i;
        return asz;
    }
    int sum_scaled = 0, sum = 0, idx_max = 0;
    for (int i = 0; i < 256; i++) {
        alphabet[i] = 0;
        const int f = freqs[i];
        if (f == 0) continue;
        const int64_t sf = (int64_t)f * (int64_t)scale;
        const int scaled = (sf <= (int64_t)total) ? 1 : (int)((sf + ((int64_t)total >> 1)) / (int64_t)total);
        alphabet[asz++] = i;
        sum_scaled += scaled;
        freqs[i] = scaled;
        sum += f;
        if (scaled > freqs[idx_max]) idx_max = i;
        if (sum >= total) break;
    }
    if (asz == 0) return 0;
    if (asz == 1) {
        freqs[alphabet[0]] = scale;
        return 1;
    }
    if (sum_scaled == scale) return asz;
    int delta = sum_scaled - scale;
    const int err_thr = freqs[idx_max] >> 4;
    const int abs_delta = delta < 0 ? -delta : delta;
    if (abs_delta <= err_thr) {
        freqs[idx_max] -= delta;
        return asz;
    }
    int inc;
    if (delta < 0) {
        delta += err_thr;
        freqs[idx_max] += err_thr;
        inc = 1;
        delta = -delta;
    } else {
        delta -= err_thr;
        freqs[idx_max] -= err_thr;
        inc = -1;
    }
    int round = 1;
    while (round < 6 && delta > 0) {
        int adjustments = 0;
        round++;
        for (int k = 0; k < asz; k++) {
            const int idx = alphabet[k];
            if (freqs[idx] <= 2) continue;
            freqs[idx] += inc;
            adjustments++;
            delta--;
            if (delta == 0) break;
        }
        if (adjustments == 0) break;
    }
    const int fm = freqs[idx_max] - delta;
    freqs[idx_max] = fm > 1 ? fm : 1;
    return asz;
}

// EncodeAlphabet (EntropyUtils.go:38-67)
KZ_D void rz_encode_alphabet(RzWriter& bw, const int* alphabet, int count) {
    if (count == 0) {
        bw.put(1, 2);  // '0','1'
    } else if (count == 256) {
        bw.put(0, 2);
    } else {
        bw.put(1, 1);
        uint8_t masks[32];
        for (int i = 0; i < 32; i++) masks[i] = 0;
        for (int i = 0; i < count; i++) masks[alphabet[i] >> 3] |= (uint8_t)(1u << (alphabet[i] & 7));
        const int last = alphabet[count - 1] >> 3;
        bw.put((uint32_t)last, 5);
        for (int i = 0; i <= last; i++) bw.put(masks[i], 8);
    }
}
KZ_D int rz_decode_alphabet(RzReader& br, int* alphabet) {  // :71-118
    if (br.get(1) == 0) {
        if (br.get(1) == 1) return 0;
        for (int i = 0; i < 256; i++) alphabet[i] = i;
        return 256;
    }
    const int last = (int)br.get(5);
    int count = 0;
    for (int i = 0; i <= last; i++) {
        const uint32_t m = br.get(8);
        for (int j = 0; j < 8; j++)
            if ((m >> j) & 1) alphabet[count++] = 8 * i + j;
    }
    return count;
}

// per symbol encoder entry (encSymbol.reset, ANSRangeCodec.go:446-468)
struct RzEncSym {
    uint32_t x_max;      // ((ANS_TOP >> lr) << 16) * freq  (fits: freq < 2^lr)
    uint32_t bias;
    uint32_t inv_freq;
    uint16_t cmpl_freq;
    uint16_t inv_shift;
};
KZ_D void rz_enc_reset(RzEncSym& s, int cum, int freq, uint32_t lr) {
    if (freq > (1 << lr) - 1) freq = (1 << lr) - 1;
    s.x_max = (uint32_t)((RZ_ANS_TOP >> lr) << 16) * (uint32_t)freq;
    s.cmpl_freq = (uint16_t)((1 << lr) - freq);
    if (freq < 2) {
        s.inv_freq = 0xFFFFFFFFu;
        s.inv_shift = 32;
        s.bias = (uint32_t)(cum + (1 << lr) - 1);
    } else {
        uint32_t shift = 0;
        while (freq > (1 << shift)) shift++;
        s.inv_freq = (uint32_t)((((uint64_t)1 << (shift + 31)) + (uint64_t)(freq - 1)) / (uint64_t)freq);
        s.inv_shift = (uint16_t)(32 + shift - 1);
        s.bias = (uint32_t)cum;
    }
}

// scratch of the nested rANS codec (global memory, per block)
struct RzAns {
    int* freqs;        // 256 * 257 ints (order 1) / 257 (order 0)
    RzEncSym* esym;    // 65536 entries (encode)
    uint32_t* dsym;    // 65536 entries cum | freq << 16 (decode)
    uint8_t* f2s;      // 256 << 11 bytes (order 1, lr 11) or 1 << 12 (order 0)
    uint8_t* buf;      // rANS byte buffer
    uint32_t buf_size;
};

// ANSRangeEncoder.Write (:274-311) with rebuildStatistics / updateFrequencies / encodeHeader / encodeChunk, order 0 or 1
KZ_D void rz_ans_encode(RzWriter& bw, const RzAns& A, const uint8_t* block, uint32_t len, int order, uint32_t chunk_size, bool* fail) {
    if (len <= 32) {
        bw.put_bytes(block, len);
        return;
    }
    uint32_t chunk = chunk_size ? chunk_size : 16384u;
    if (order == 1) chunk = chunk << 8;  // <= 1 << 27 for the sizes used here
    const uint32_t lr = order ? 11u : 12u;  // max(logRange - order, 8)
    const int dim = 255 * order + 1;
    uint32_t start = 0;
    int alphabet[256];
    while (start < len) {
        const uint32_t end = start + chunk < len ? start + chunk : len;
        const uint8_t* blk = block + start;
        const uint32_t n = end - start;
        // ---- rebuildStatistics (:408-427)
        for (int i = 0; i < dim * 257; i++) A.freqs[i] = 0;
        if (order == 0) {
            for (uint32_t i = 0; i < n; i++) A.freqs[blk[i]]++;
            A.freqs[256] = (int)n;
        } else {
            const uint32_t q = n >> 2;
            const uint32_t parts = q == 0 ? 1 : 4;
            for (uint32_t k = 0; k < parts; k++) {  // internal/Global.go:252-303: the context of the first byte of a slice is 0
                const uint8_t* p = q == 0 ? blk : blk + k * q;
                const uint32_t m = q == 0 ? n : q;
                uint32_t prv = 0;
                for (uint32_t i = 0; i < m; i++) {
                    A.freqs[257 * prv + p[i]]++;
                    A.freqs[257 * prv + 256]++;
                    prv = p[i];
                }
            }
        }
        // ---- updateFrequencies (:171-213) + encodeHeader (:216-270)
        int total_asz = 0;
        bw.put(lr - 8, 3);
        for (int i = 0; i < 256; i++) alphabet[i] = 0;
        for (int k = 0; k < dim; k++) {
            int* f = A.freqs + 257 * k;
            RzEncSym* symb = A.esym + ((size_t)k << 8);
            const int asz = rz_normalize(f, alphabet, f[256], 1 << lr);
            if (asz > 0) {
                int sum = 0;
                for (int i = 0, count = 0; i < 256; i++) {
                    if (f[i] == 0) continue;
                    rz_enc_reset(symb[i], sum, f[i], lr);
                    sum += f[i];
                    if (++count >= asz) break;
                }
            }
            rz_encode_alphabet(bw, alphabet, asz);
            if (asz > 1) {
                const int chk = asz < 64 ? 6 : 8;
                uint32_t llr = 3;
                while ((1u << llr) <= lr) llr++;
                for (int i = 1; i < asz; i += chk) {
                    int mx = f[alphabet[i]] - 1;
                    uint32_t log_max = 0;
                    const int endj = i + chk < asz ? i + chk : asz;
                    for (int j = i + 1; j < endj; j++) mx = max(mx, f[alphabet[j]] - 1);
                    while ((1 << log_max) <= mx) log_max++;
                    bw.put(log_max, llr);
                    if (log_max == 0) continue;
                    for (int j = i; j < endj; j++) bw.put((uint32_t)(f[alphabet[j]] - 1), log_max);
                }
            }
            total_asz += asz;
        }
        // ---- encodeChunk (:331-405)
        if (order == 1 || total_asz > 1) {
            uint32_t st0 = RZ_ANS_TOP, st1 = RZ_ANS_TOP, st2 = RZ_ANS_TOP, st3 = RZ_ANS_TOP;
            int64_t np = (int64_t)A.buf_size - 1;
            uint8_t* buffer = A.buf;
            const int64_t end4 = (int64_t)(n & ~3u);
            for (int64_t i = (int64_t)n - 1; i >= end4; i--) buffer[np--] = blk[i];
            auto enc = [&](uint32_t& st, const RzEncSym& s) {  // encodeSymbol :313-329
                const int x = st >= s.x_max ? 1 : 0;
                buffer[np] = (uint8_t)st;
                np -= x;
                buffer[np] = (uint8_t)(st >> 8);
                np -= x;
                if (x) st >>= 16;
                st = st + s.bias + (uint32_t)(((uint64_t)st * s.inv_freq) >> s.inv_shift) * (uint32_t)s.cmpl_freq;
            };
            if (order == 0) {
                const RzEncSym* symb = A.esym;
                for (int64_t i = end4 - 1; i > 0; i -= 4) {
                    enc(st0, symb[blk[i]]);
                    enc(st1, symb[blk[i - 1]]);
                    enc(st2, symb[blk[i - 2]]);
                    enc(st3, symb[blk[i - 3]]);
                }
            } else if (n > 1) {
                const int64_t quarter = end4 >> 2;
                if (quarter == 0) {  // the reference indexes block[-1] here and panics (SURVEY App. C.6)
                    *fail = true;
                    return;
                }
                int64_t i0 = quarter - 2, i1 = 2 * quarter - 2, i2 = 3 * quarter - 2, i3 = end4 - 2;
                uint32_t prv0 = blk[i0 + 1], prv1 = blk[i1 + 1], prv2 = blk[i2 + 1], prv3 = blk[i3 + 1];
                while (i0 >= 0) {
                    const uint32_t c0 = blk[i0], c1 = blk[i1], c2 = blk[i2], c3 = blk[i3];
                    enc(st0, A.esym[(c0 << 8) | prv0]);
                    enc(st1, A.esym[(c1 << 8) | prv1]);
                    enc(st2, A.esym[(c2 << 8) | prv2]);
                    enc(st3, A.esym[(c3 << 8) | prv3]);
                    prv0 = c0, prv1 = c1, prv2 = c2, prv3 = c3;
                    i0--, i1--, i2--, i3--;
                }
                enc(st0, A.esym[prv0]);
                enc(st1, A.esym[prv1]);
                enc(st2, A.esym[prv2]);
                enc(st3, A.esym[prv3]);
            }
            np++;
            const uint32_t sz = (uint32_t)((int64_t)A.buf_size - np);
            uint32_t v = sz;  // WriteVarInt :264-275
            while (v >= 128) {
                bw.put(0x80 | (v & 0x7F), 8);
                v >>= 7;
            }
            bw.put(v, 8);
            bw.put(st0, 32);
            bw.put(st1, 32);
            bw.put(st2, 32);
            bw.put(st3, 32);
            if (sz) bw.put_bytes(buffer + np, sz);
        }
        start = end;
    }
}

// ANSRangeDecoder.Read (:714-757) with decodeHeader (:605-710) and decodeChunkV2 (:860-957), order 0 or 1. Returns false on error.
KZ_D bool rz_ans_decode(RzReader& br, const RzAns& A, uint8_t* block, uint32_t len, int order, uint32_t chunk_size) {
    if (len <= 32) {
        for (uint32_t i = 0; i < len; i++) block[i] = (uint8_t)br.get(8);
        return !br.over;
    }
    uint32_t chunk = chunk_size ? chunk_size : 16384u;
    if (order == 1) chunk = chunk << 8;
    const int dim = 255 * order + 1;
    uint32_t start = 0;
    int alphabet[256];
    while (start < len) {
        const uint32_t end = start + chunk < len ? start + chunk : len;
        uint8_t* blk = block + start;
        const uint32_t n = end - start;
        // ---- decodeHeader
        const uint32_t lr = 8 + br.get(3);
        if (lr > (order ? 11u : 12u)) return false;  // tables are sized for the encoder's ranges
        const int scale = 1 << lr;
        uint32_t llr = 3;
        while ((1u << llr) <= lr) llr++;
        int res = 0, alpha0 = 0;
        for (int k = 0; k < dim; k++) {
            const int asz = rz_decode_alphabet(br, alphabet);
            if (asz == 0) continue;
            int* f = A.freqs + ((size_t)k << 8);
            if (asz != 256)
                for (int i = 0; i < 256; i++) f[i] = 0;
            const int chk = asz < 64 ? 6 : 8;
            int sum = 0;
            for (int i = 1; i < asz; i += chk) {
                const uint32_t log_max = br.get(llr);
                if ((1 << log_max) > scale) return false;
                const int endj = i + chk < asz ? i + chk : asz;
                for (int j = i; j < endj; j++) {
                    int freq = 1;
                    if (log_max > 0) {
                        freq = (int)(1 + br.get(log_max));
                        if (freq <= 0 || freq >= scale) return false;
                    }
                    f[alphabet[j]] = freq;
                    sum += freq;
                }
            }
            if (scale <= sum) return false;
            f[alphabet[0]] = scale - sum;
            sum = 0;
            uint32_t* symb = A.dsym + ((size_t)k << 8);
            uint8_t* freq2sym = A.f2s + ((size_t)k << lr);
            for (int i = 0; i < 256; i++) {
                if (f[i] == 0) continue;
                if (sum + f[i] > scale) return false;
                for (int j = 0; j < f[i]; j++) freq2sym[sum + j] = (uint8_t)i;
                const int fr = f[i] < scale - 1 ? f[i] : scale - 1;
                symb[i] = (uint32_t)sum | ((uint32_t)fr << 16);
                sum += f[i];
            }
            res += asz;
            alpha0 = alphabet[0];
        }
        if (br.over || res == 0) return false;
        if (order == 0 && res == 1) {
            for (uint32_t i = 0; i < n; i++) blk[i] = (uint8_t)alpha0;
            start = end;
            continue;
        }
        // ---- decodeChunkV2
        const uint32_t sz = br.varint();
        if (sz >= (1u << 27)) return false;
        uint32_t st0 = br.get(32), st1 = br.get(32), st2 = br.get(32), st3 = br.get(32);
        if (br.over || br.pos + 8ull * sz > br.end) return false;
        // the payload is read straight from the stream: byte i of the rANS buffer = 8 bits at pos + 8 i (zero past the end)
        const uint64_t p0 = br.pos;
        uint32_t np = 0;
        auto fetch16 = [&](uint32_t at) -> uint32_t {  // buffer[at] << 8 | buffer[at + 1], zeros beyond sz (:888-893 guard)
            uint32_t v = 0;
            for (uint32_t q = 0; q < 2; q++) {
                v <<= 8;
                if (at + q < sz) {
                    const uint64_t bp = p0 + 8ull * (at + q);
                    const uint32_t o = (uint32_t)bp & 7;
                    const uint32_t two = ((uint32_t)br.base[bp >> 3] << 8) | br.base[(bp >> 3) + 1];
                    v |= (two >> (8 - o)) & 0xFF;
                }
            }
            return v;
        };
        const uint32_t mask = (1u << lr) - 1;
        auto dec = [&](uint32_t& st, uint32_t s) {  // decodeSymbol :846-858
            st = (s >> 16) * (st >> lr) + (st & mask) - (s & 0xFFFF);
            if (st < (uint32_t)RZ_ANS_TOP) {
                st = (st << 16) | fetch16(np);
                np += 2;
            }
        };
        const uint32_t end4 = n & ~3u;
        if (order == 0) {
            for (uint32_t i = 0; i < end4; i += 4) {
                const uint32_t c3 = A.f2s[st3 & mask];
                blk[i] = (uint8_t)c3;
                dec(st3, A.dsym[c3]);
                const uint32_t c2 = A.f2s[st2 & mask];
                blk[i + 1] = (uint8_t)c2;
                dec(st2, A.dsym[c2]);
                const uint32_t c1 = A.f2s[st1 & mask];
                blk[i + 2] = (uint8_t)c1;
                dec(st1, A.dsym[c1]);
                const uint32_t c0 = A.f2s[st0 & mask];
                blk[i + 3] = (uint8_t)c0;
                dec(st0, A.dsym[c0]);
            }
        } else {
            const uint32_t quarter = end4 >> 2;
            uint32_t i0 = 0, i1 = quarter, i2 = 2 * quarter, i3 = 3 * quarter;
            uint32_t p0c = 0, p1c = 0, p2c = 0, p3c = 0;
            while (i0 < quarter) {
                const uint32_t c3 = A.f2s[((size_t)p3c << lr) + (st3 & mask)];
                blk[i3] = (uint8_t)c3;
                dec(st3, A.dsym[(p3c << 8) + c3]);
                const uint32_t c2 = A.f2s[((size_t)p2c << lr) + (st2 & mask)];
                blk[i2] = (uint8_t)c2;
                dec(st2, A.dsym[(p2c << 8) + c2]);
                const uint32_t c1 = A.f2s[((size_t)p1c << lr) + (st1 & mask)];
                blk[i1] = (uint8_t)c1;
                dec(st1, A.dsym[(p1c << 8) + c1]);
                const uint32_t c0 = A.f2s[((size_t)p0c << lr) + (st0 & mask)];
                blk[i0] = (uint8_t)c0;
                dec(st0, A.dsym[(p0c << 8) + c0]);
                p3c = c3, p2c = c2, p1c = c1, p0c = c0;
                i0++, i1++, i2++, i3++;
            }
        }
        for (uint32_t i = end4; i < n; i++) {
            blk[i] = (uint8_t)(fetch16(np) >> 8);
            np++;
        }
        br.pos = p0 + 8ull * sz;
        start = end;
    }
    return !br.over;
}

// findMatch (:246-296)
KZ_D void rz_find_match(const uint8_t* buf, int buf_len, int pos, uint32_t hash32, int32_t counter, const uint32_t* m, int min_match, int* idx, int* len) {
    int max_match = min(RZ_MAX_MATCH1, buf_len - pos);
    *idx = -1;
    *len = -1;
    if (max_match < min_match) return;
    max_match -= 8;
    int best_len = 0, best_idx = -1;
    const uint8_t* cur = buf + pos;
    const int32_t pos_checks = 1 << RZ_LOG_POS, mask_checks = pos_checks - 1;
    for (int32_t i = counter; i > counter - pos_checks; i--) {
        uint32_t ref = m[i & mask_checks];
        if ((ref & RZ_HASH_MASK) != hash32) continue;
        ref &= ~RZ_HASH_MASK;
        const uint8_t* rb = buf + ref;
        if (rb[best_len] != cur[best_len]) continue;
        int n = 0;
        while (n < max_match) {
            const uint64_t diff = rz_le64(rb + n) ^ rz_le64(cur + n);
            if (diff != 0) {
                n += (__ffsll((long long)diff) - 1) >> 3;
                break;
            }
            n += 8;
        }
        if (n > best_len) {
            best_idx = (int)i;
            best_len = n;
        }
    }
    if (best_len < min_match) return;
    *idx = (int)counter - best_idx;
    *len = best_len - min_match;
}

KZ_D int rz_detect_simple_type(uint32_t count, const int* f) {  // internal/Global.go:346-419
    if (count == 0) return 0;
    const char* DNA = "acgntuACGNTU\"";
    const char* NUM = "0123456789+-*/=,.:; ";
    const char* B64 = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    int64_t sum = 0;
    for (int i = 0; i < 12; i++) sum += f[(uint8_t)DNA[i]];
    if (sum > (int64_t)count - (int64_t)count / 12) return 6;  // DT_DNA
    sum = 0;
    for (int i = 0; i < 20; i++) sum += f[(uint8_t)NUM[i]];
    if (sum == (int64_t)count) return 4;  // DT_NUMERIC
    sum = 0;
    for (int i = 0; i < 64; i++) sum += f[(uint8_t)B64[i]];
    if (sum + f[0x3D] == (int64_t)count) return 5;  // DT_BASE64
    sum = 0;
    for (int i = 0; i < 256; i++)
        if (f[i] > 0) sum++;
    if (sum == 256) return 7;  // DT_BIN
    if (sum <= 4) return 9;    // DT_SMALL_ALPHABET
    return 0;
}

KZ_D RzAns rz_ans_scratch(uint8_t* s, uint32_t buf_size) {
    RzAns A;
    A.freqs = reinterpret_cast<int*>(s);
    s += (size_t)256 * 257 * 4 + 64;
    A.esym = reinterpret_cast<RzEncSym*>(s);
    A.dsym = reinterpret_cast<uint32_t*>(s);
    s += (size_t)65536 * sizeof(RzEncSym);
    A.f2s = s;
    s += (size_t)256 << 11;
    A.buf = s;
    A.buf_size = buf_size;
    return A;
}

}  // namespace

size_t rolz_scratch_bytes(size_t n) {
    const size_t chunk = n < (size_t)RZ_CHUNK ? n : (size_t)RZ_CHUNK;
    size_t s = ((size_t)RZ_HASH_SIZE << RZ_LOG_POS) * 4 + (size_t)RZ_HASH_SIZE * 4;  // matches, counters
    s += (chunk + 64 + 64) + (chunk / 5 + 64) + 2 * (chunk / 4 + 64);              // lit, len, midx, tk
    s += (size_t)256 * 257 * 4 + 64 + (size_t)65536 * sizeof(RzEncSym) + ((size_t)256 << 11);
    s += rolz_ans_buffer(chunk) + 256;
    return (s + 255) & ~(size_t)255;
}

// ---- forward: ROLZCodec.Forward :150-168 + rolzCodec1.Forward :301-596. res[b]: status 0 = ok, 1 = skip
__global__ void __launch_bounds__(32) rolz_forward_kernel(const uint8_t* __restrict__ in, const RolzBlock* __restrict__ blocks, int nblocks,
                                                          uint8_t* __restrict__ scratch_all, uint8_t* __restrict__ out, StageResult* __restrict__ res) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const RolzBlock blk = blocks[b];
    StageResult r;
    r.status = 1;
    r.out_len = 0;
    r.data_type = blk.data_type;
    const uint32_t n = blk.len;
    if (n < 64 || n > (1u << 30) || blk.cap < (n <= 512 ? n + 64 : n)) {
        if (lane == 0) res[b] = r;
        return;
    }
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    uint8_t* S = scratch_all + blk.scratch_off;
    uint32_t* matches = reinterpret_cast<uint32_t*>(S);
    int32_t* counters = reinterpret_cast<int32_t*>(S + ((size_t)RZ_HASH_SIZE << RZ_LOG_POS) * 4);
    uint8_t* p = S + ((size_t)RZ_HASH_SIZE << RZ_LOG_POS) * 4 + (size_t)RZ_HASH_SIZE * 4;
    const uint32_t size_chunk0 = n < (uint32_t)RZ_CHUNK ? n : (uint32_t)RZ_CHUNK;
    uint8_t* lit_buf = p;
    p += size_chunk0 + 128;
    uint8_t* len_buf = p;
    p += size_chunk0 / 5 + 64;
    uint8_t* midx_buf = p;
    p += size_chunk0 / 4 + 64;
    uint8_t* tk_buf = p;
    p += size_chunk0 / 4 + 64;
    p = reinterpret_cast<uint8_t*>(((uintptr_t)p + 15) & ~(uintptr_t)15);
    const RzAns A = rz_ans_scratch(p, (uint32_t)rolz_ans_buffer(size_chunk0));
    for (uint32_t i = lane; i < RZ_HASH_SIZE; i += 32) counters[i] = 0;
    __syncwarp();
    const int len_src = (int)n, src_end = len_src - 4;
    const int lit_order = len_src < (1 << 17) ? 0 : 1;
    uint8_t flags = (uint8_t)lit_order;
    int min_match = RZ_MIN3, delta = 2;
    int dt = blk.data_type;
    if (dt == 0) {  // DT_UNDEFINED: DetectSimpleType on the order 0 histogram of the block (:334-345)
        for (int i = lane; i < 256; i += 32) A.freqs[i] = 0;
        __syncwarp();
        for (uint32_t i = lane; i < n; i += 32) atomicAdd(&A.freqs[src[i]], 1);
        __syncwarp();
        dt = rz_detect_simple_type(n, A.freqs);
        if (dt != 0) r.data_type = dt;
    }
    if (dt == 3 /*DT_EXE*/) {
        delta = 3;
        flags |= 8;
    } else if (dt == 6 /*DT_DNA*/) {
        delta = 8;
        min_match = RZ_MIN7;
        flags |= 4;
    } else if (dt == 2 /*DT_MULTIMEDIA*/) {
        delta = 8;
        min_match = RZ_MIN4;
        flags |= 2;
    }
    flags |= (uint8_t)(RZ_LOG_POS << 4);
    const int32_t mask_checks = (1 << RZ_LOG_POS) - 1;
    int src_idx = 0;
    uint32_t dst_idx = 5;
    int size_chunk = (int)size_chunk0, start_chunk = 0;
    bool ok = true;
    while (start_chunk < src_end && ok) {
        for (uint32_t i = lane; i < (RZ_HASH_SIZE << RZ_LOG_POS); i += 32) matches[i] = 0;
        __syncwarp();
        int end_chunk = start_chunk + size_chunk;
        if (end_chunk >= src_end) {
            end_chunk = src_end;
            size_chunk = end_chunk - start_chunk;
        }
        if (lane == 0) {
            int lit_idx = 0, len_idx = 0, m_idx = 0, tk_idx = 0;
            const uint8_t* buf = src + start_chunk;
            src_idx = 0;
            const int nfirst = min(src_end - start_chunk, 8);
            for (int j = 0; j < nfirst; j++) lit_buf[lit_idx++] = buf[src_idx++];
            int first_lit_idx = src_idx, src_inc = 0;
            while (src_idx < size_chunk) {
                uint32_t key = min_match == RZ_MIN3 ? rz_key1(buf + src_idx - delta) : rz_key2(buf + src_idx - delta);
                uint32_t* m = matches + ((size_t)key << RZ_LOG_POS);
                uint32_t hash32 = rz_hash(buf + src_idx);
                int match_idx, match_len;
                rz_find_match(buf, size_chunk, src_idx, hash32, counters[key], m, min_match, &match_idx, &match_len);
                counters[key] = (counters[key] + 1) & mask_checks;
                m[counters[key]] = hash32 | (uint32_t)src_idx;
                if (match_idx < 0) {
                    src_idx++;
                    src_idx += src_inc >> 6;
                    src_inc++;
                    continue;
                }
                const int src_idx1 = src_idx + 1;
                key = min_match == RZ_MIN3 ? rz_key1(buf + src_idx1 - delta) : rz_key2(buf + src_idx1 - delta);
                m = matches + ((size_t)key << RZ_LOG_POS);
                hash32 = rz_hash(buf + src_idx1);
                int match_idx1, match_len1;
                rz_find_match(buf, size_chunk, src_idx1, hash32, counters[key], m, min_match, &match_idx1, &match_len1);
                if (match_idx1 >= 0 && match_len1 > match_len) {
                    match_idx = match_idx1;
                    match_len = match_len1;
                    src_idx = src_idx1;
                    counters[key] = (counters[key] + 1) & mask_checks;
                    m[counters[key]] = hash32 | (uint32_t)src_idx;
                }
                const int lit_len = src_idx - first_lit_idx;
                uint8_t token;
                if (match_len >= 7) {
                    token = 7;
                    len_idx += rz_emit_length(len_buf + len_idx, match_len - 7);
                } else {
                    token = (uint8_t)match_len;
                }
                if (lit_len > 0) {
                    if (lit_len >= 31) {
                        token |= 0xF8;
                        len_idx += rz_emit_length(len_buf + len_idx, lit_len - 31);
                    } else {
                        token |= (uint8_t)(lit_len << 3);
                    }
                    for (int j = 0; j < lit_len; j++) lit_buf[lit_idx + j] = buf[first_lit_idx + j];
                    lit_idx += lit_len;
                }
                tk_buf[tk_idx++] = token;
                midx_buf[m_idx++] = (uint8_t)match_idx;
                src_idx += match_len + min_match;
                first_lit_idx = src_idx;
                src_inc = 0;
            }
            src_idx = size_chunk;
            const int lit_len = src_idx - first_lit_idx;
            if (tk_idx != 0) tk_buf[tk_idx++] = lit_len >= 31 ? (uint8_t)0xF8 : (uint8_t)(lit_len << 3);
            if (lit_len > 0) {
                if (lit_len >= 31) len_idx += rz_emit_length(len_buf + len_idx, lit_len - 31);
                for (int j = 0; j < lit_len; j++) lit_buf[lit_idx + j] = buf[first_lit_idx + j];
                lit_idx += lit_len;
            }
            // private bitstream of the chunk (:509-555), written straight into the output
            RzWriter bw;
            bw.init(dst + dst_idx, dst + blk.cap);
            bw.put((uint32_t)lit_idx, 32);
            bw.put((uint32_t)tk_idx, 32);
            bw.put((uint32_t)len_idx, 32);
            bw.put((uint32_t)m_idx, 32);
            bool fail = false;
            rz_ans_encode(bw, A, lit_buf, (uint32_t)lit_idx, lit_order, 0, &fail);
            rz_ans_encode(bw, A, tk_buf, (uint32_t)tk_idx, 0, 32768, &fail);
            rz_ans_encode(bw, A, len_buf, (uint32_t)len_idx, 0, 32768, &fail);
            rz_ans_encode(bw, A, midx_buf, (uint32_t)m_idx, 0, 32768, &fail);
            bw.close();
            if (fail || bw.over) ok = false;
            dst_idx = (uint32_t)(bw.p - dst);
        }
        ok = __shfl_sync(0xFFFFFFFFu, (int)ok, 0) != 0;
        dst_idx = __shfl_sync(0xFFFFFFFFu, dst_idx, 0);
        start_chunk = end_chunk;
        __syncwarp();
    }
    if (lane == 0) {
        if (ok && dst_idx + 4 <= blk.cap) {
            const int last = src_end;  // srcIdx += startChunk - sizeChunk after the loop
            dst[0] = (uint8_t)(n >> 24), dst[1] = (uint8_t)(n >> 16), dst[2] = (uint8_t)(n >> 8), dst[3] = (uint8_t)n;
            dst[4] = flags;
            dst[dst_idx] = src[last], dst[dst_idx + 1] = src[last + 1], dst[dst_idx + 2] = src[last + 2], dst[dst_idx + 3] = src[last + 3];
            dst_idx += 4;
            if (dst_idx < n) {  // else "no compression": skip
                r.status = 0;
                r.out_len = dst_idx;
            }
        }
        res[b] = r;
    }
}

// ---- inverse: ROLZCodec.Inverse :173-191 + rolzCodec1.Inverse :601-913 (bitstream version 6). status: 0 ok, -13 error
__global__ void __launch_bounds__(32) rolz_inverse_kernel(const uint8_t* __restrict__ in, const RolzBlock* __restrict__ blocks, int nblocks,
                                                          uint8_t* __restrict__ scratch_all, uint8_t* __restrict__ out, StageResult* __restrict__ res) {
    const int b = blockIdx.x, lane = threadIdx.x;
    if (b >= nblocks) return;
    const RolzBlock blk = blocks[b];
    StageResult r;
    r.status = -KZ_E_PROCESS_BLOCK;
    r.out_len = 0;
    r.data_type = 0;
    const uint8_t* src = in + blk.src_off;
    uint8_t* dst = out + blk.dst_off;
    const int len_src = (int)blk.len;
    const int64_t len_dst = blk.cap;
    if (len_src < 5) {
        if (lane == 0) res[b] = r;
        return;
    }
    const int dst_end = (int)(((uint32_t)src[0] << 24) | ((uint32_t)src[1] << 16) | ((uint32_t)src[2] << 8) | src[3]) - 4;
    if (dst_end <= 0 || (int64_t)dst_end > len_dst) {
        if (lane == 0) res[b] = r;
        return;
    }
    uint8_t* S = scratch_all + blk.scratch_off;
    uint32_t* matches = reinterpret_cast<uint32_t*>(S);
    int32_t* counters = reinterpret_cast<int32_t*>(S + ((size_t)RZ_HASH_SIZE << RZ_LOG_POS) * 4);
    uint8_t* p = S + ((size_t)RZ_HASH_SIZE << RZ_LOG_POS) * 4 + (size_t)RZ_HASH_SIZE * 4;
    int size_chunk = (int)(len_dst < (int64_t)RZ_CHUNK ? len_dst : (int64_t)RZ_CHUNK);
    const uint32_t sc0 = (uint32_t)size_chunk;
    uint8_t* lit_buf = p;
    p += sc0 + 128;
    uint8_t* mlen_buf = p;
    p += sc0 / 5 + 64;
    uint8_t* midx_buf = p;
    p += sc0 / 4 + 64;
    uint8_t* tk_buf = p;
    p += sc0 / 4 + 64;
    p = reinterpret_cast<uint8_t*>(((uintptr_t)p + 15) & ~(uintptr_t)15);
    const RzAns A = rz_ans_scratch(p, 0);
    const int lit_cap = size_chunk, mlen_cap = size_chunk / 5, midx_cap = size_chunk / 4, tk_cap = size_chunk / 4;
    for (uint32_t i = lane; i < RZ_HASH_SIZE; i += 32) counters[i] = 0;
    const uint8_t flags = src[4];
    const int lit_order = flags & 1;
    int delta = 2, min_match = RZ_MIN3;
    if ((flags & 0x0E) == 2) {
        min_match = RZ_MIN4;
        delta = 8;
    } else if ((flags & 0x0E) == 4) {
        min_match = RZ_MIN7;
        delta = 8;
    } else if ((flags & 0x0E) == 8) {
        delta = 3;
    }
    const uint32_t log_pos = flags >> 4;
    if (log_pos != (uint32_t)RZ_LOG_POS) {  // the encoder always writes 4; other table shapes are not sized here
        if (lane == 0) res[b] = r;
        return;
    }
    const int32_t mask_checks = (1 << RZ_LOG_POS) - 1;
    int start_chunk = 0, src_idx = 5, dst_idx = 0;
    bool ok = true;
    while (start_chunk < dst_end && ok) {
        for (uint32_t i = lane; i < (RZ_HASH_SIZE << RZ_LOG_POS); i += 32) matches[i] = 0;
        __syncwarp();
        int end_chunk = start_chunk + size_chunk;
        if (end_chunk > dst_end) end_chunk = dst_end;
        size_chunk = end_chunk - start_chunk;
        if (lane == 0) {
            uint8_t* buf = dst + start_chunk;
            int m_idx = 0, len_idx = 0, lit_idx = 0, tk_idx = 0;
            RzReader ibs;
            ibs.init(src + src_idx, (uint64_t)(len_src - src_idx));
            const int lit_len0 = (int)ibs.get(32), tk_len = (int)ibs.get(32), mlen_len = (int)ibs.get(32), midx_len = (int)ibs.get(32);
            const int first_lit_len = min(size_chunk, 8);
            if (ibs.over || lit_len0 < 0 || lit_len0 > lit_cap || tk_len < 0 || tk_len > tk_cap || mlen_len < 0 || mlen_len > mlen_cap || midx_len < 0 ||
                midx_len > midx_cap || lit_len0 < first_lit_len || lit_len0 > size_chunk || (tk_len == 0 && midx_len != 0) ||
                (tk_len > 0 && midx_len + 1 != tk_len)) {
                ok = false;
            }
            if (ok) ok = rz_ans_decode(ibs, A, lit_buf, (uint32_t)lit_len0, lit_order, 0);
            if (ok) ok = rz_ans_decode(ibs, A, tk_buf, (uint32_t)tk_len, 0, 32768);
            if (ok) ok = rz_ans_decode(ibs, A, mlen_buf, (uint32_t)mlen_len, 0, 32768);
            if (ok) ok = rz_ans_decode(ibs, A, midx_buf, (uint32_t)midx_len, 0, 32768);
            if (ok) {
                src_idx += (int)((ibs.pos + 7) >> 3);
                if (tk_len == 0) {  // only literals
                    if (lit_len0 != size_chunk) {
                        ok = false;
                    } else {
                        for (int i = 0; i < size_chunk; i++) buf[i] = lit_buf[i];
                        dst_idx = size_chunk;
                    }
                } else {
                    dst_idx = 0;
                    int mm = 8;
                    if (start_chunk >= dst_end) mm = dst_end - start_chunk;
                    for (int j = 0; j < mm; j++) buf[dst_idx++] = lit_buf[lit_idx++];
                    while (dst_idx < size_chunk && ok) {
                        const uint8_t token = tk_buf[tk_idx++];
                        int match_len = token & 0x07;
                        if (match_len == 7) {
                            int d;
                            match_len = rz_read_length(mlen_buf + len_idx, &d) + 7;
                            len_idx += d;
                        }
                        int lit_len;
                        if (token < 0xF8) {
                            lit_len = token >> 3;
                        } else {
                            int d;
                            lit_len = rz_read_length(mlen_buf + len_idx, &d) + 31;
                            len_idx += d;
                        }
                        if (lit_len > 0) {
                            if (dst_idx + lit_len > lit_cap) {
                                ok = false;
                                break;
                            }
                            int src_inc = 0;
                            uint8_t* d = buf + dst_idx - delta;
                            for (int j = 0; j < lit_len; j++) d[delta + j] = lit_buf[lit_idx + j];
                            for (int k = 0; k < lit_len; k++) {
                                const uint32_t key = min_match == RZ_MIN3 ? rz_key1(d + k) : rz_key2(d + k);
                                const int32_t cc = (counters[key] + 1) & mask_checks;
                                matches[((size_t)key << RZ_LOG_POS) + (size_t)cc] = (uint32_t)(dst_idx + k);
                                counters[key] = cc;
                                k += src_inc >> 6;
                                src_inc++;
                            }
                            lit_idx += lit_len;
                            dst_idx += lit_len;
                            if (dst_idx >= size_chunk) {
                                if (dst_idx == size_chunk) break;
                                ok = false;
                                break;
                            }
                        }
                        if (dst_idx + match_len + min_match > dst_end) {
                            ok = false;
                            break;
                        }
                        const int32_t match_idx = (int32_t)midx_buf[m_idx++];
                        const uint32_t key = min_match == RZ_MIN3 ? rz_key1(buf + dst_idx - delta) : rz_key2(buf + dst_idx - delta);
                        uint32_t* m = matches + ((size_t)key << RZ_LOG_POS);
                        int ref = (int)m[(counters[key] - match_idx) & mask_checks];
                        counters[key] = (counters[key] + 1) & mask_checks;
                        m[counters[key]] = (uint32_t)dst_idx;
                        int ml = match_len + min_match;
                        while (ml != 0) {  // emitCopy :69-84 (byte order is what matters)
                            buf[dst_idx++] = buf[ref++];
                            ml--;
                        }
                    }
                }
            }
        }
        ok = __shfl_sync(0xFFFFFFFFu, (int)ok, 0) != 0;
        src_idx = __shfl_sync(0xFFFFFFFFu, src_idx, 0);
        dst_idx = __shfl_sync(0xFFFFFFFFu, dst_idx, 0);
        start_chunk = end_chunk;
        __syncwarp();
    }
    if (lane == 0) {
        if (ok) {
            dst_idx += start_chunk - size_chunk;
            if ((int64_t)dst_idx + 4 <= len_dst && len_src - src_idx == 4) {
                dst[dst_idx] = src[src_idx], dst[dst_idx + 1] = src[src_idx + 1], dst[dst_idx + 2] = src[src_idx + 2], dst[dst_idx + 3] = src[src_idx + 3];
                r.status = 0;
                r.out_len = (uint32_t)(dst_idx + 4);
            }
        }
        res[b] = r;
    }
}

}  // namespace kz
