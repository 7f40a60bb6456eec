// The plan of a write into a compressed stream (kz_write_ranges, kz_api.cu). Pure host code: no CUDA types, so that
// tests/host/write_plan_host.cpp compiles it with g++ and checks it on the CPU under the sanitizers.
//
// Blocks are independent, every block but the last decodes to exactly block_size bytes, and nothing in a record depends on where it lies.
// So a write that touches blocks k .. m re-encodes only those: the new stream is the old one up to the prefix of record k, the new records,
// and the old records that follow them, moved by the change in bit length, then the end marker. The plan says which blocks are re-encoded,
// which of them are decoded first (the ones the writes do not cover completely), the pieces each re-encoded block is built from, the bit
// the new stream first differs at (the cut), and the segments of the new stream behind the cut.
#pragma once
#include <algorithm>
#include <cstdint>
#include <set>
#include <vector>

#include "kz_read_plan.h"

namespace kz {

const uint64_t WRITE_APPEND = ~0ull;  // KZ_WRITE_APPEND: the end of the data as it stands after the call's earlier writes

// Bytes [at, at + len) of a re-encoded block come from the decoded old block (same place), from write `write` (its data bytes from ..),
// or are zeros (the gap a write past the end leaves).
enum WritePieceKind : uint32_t { PIECE_OLD = 0, PIECE_WRITE = 1, PIECE_ZERO = 2 };
struct WritePiece {
    uint32_t kind, at, len, write;
    uint64_t from;
};

// Segments of the new stream behind byte floor(cut / 8), in stream order: the carry (the old bits of that byte before the cut), a run of
// re-encoded blocks enc[first .. first + count), a run of old records first .. first + count - 1 (source bits [bit, bit + bits) of the old
// stream, prefixes included), and the end marker.
enum WriteSegKind : uint32_t { SEG_CARRY = 0, SEG_NEW = 1, SEG_OLD = 2, SEG_END = 3 };
struct WriteSeg {
    uint32_t kind;
    uint64_t first, count, bit, bits;
};

enum WritePlanStatus { WRITE_OK = 0, WRITE_NEED_SIZE = 1, WRITE_TOO_LARGE = 2 };

struct WritePlan {
    int status = WRITE_OK;          // WRITE_NEED_SIZE: the old size is unknown and the result depends on it; WRITE_TOO_LARGE: see plan_writes
    uint64_t new_size = 0;          // decoded bytes after the writes (meaningful when size_known)
    bool size_known = false;
    uint64_t nblocks = 0;           // blocks after the writes (old blocks + new ones)
    std::vector<uint64_t> enc;      // the re-encoded blocks, ascending; those >= the old block count are new
    std::vector<uint32_t> enc_len;  // the length of each after the writes
    std::vector<uint8_t> decode;    // per re-encoded block: its old block is decoded first (some of its bytes survive)
    std::vector<WritePiece> pieces; // the pieces of enc[j] are pieces[piece_of[j] .. piece_of[j + 1]), ascending and tiling [0, enc_len[j])
    std::vector<uint64_t> piece_of;
    std::vector<uint32_t> first;    // pass p re-encodes enc[first[p] .. first[p + 1])
    uint64_t cut = 0;               // the first bit of the new stream that may differ from the old one
    std::vector<WriteSeg> segs;
    bool nothing() const { return enc.empty(); }
    uint32_t npasses() const { return first.empty() ? 0 : (uint32_t)first.size() - 1; }
};

// The first bit behind record b - 1 of x: the prefix of record b, or the end marker when b == nblocks.
inline uint64_t record_prefix_bit(const StreamIndex& x, uint64_t b) { return b == 0 ? x.header_bits : x.start[b - 1] + x.bits[b - 1]; }

// Device bytes one block of a write pass takes: a read's (its slot and the decode's two stage buffers) plus the encode's (enc_cost, the
// compress_block_cost of the stream's block size and codec).
inline uint64_t write_block_cost(uint32_t block_size, uint64_t enc_cost) { return read_block_cost(block_size) + enc_cost; }

// Everything of the plan but its passes: plan_writes_streams cuts those.
inline WritePlan plan_write_blocks(const StreamIndex& x, uint32_t nw, const uint64_t* off, const uint64_t* len) {
    WritePlan P;
    const uint64_t bs = x.block_size, nb = x.nblocks();
    const bool known = x.size >= 0;
    // an unknown size lies in (lo, hi]; where the result does not depend on it, hi stands in for it
    const uint64_t lo = nb ? (nb - 1) * bs : 0, hi = nb * bs;
    const uint64_t old_size = known ? (uint64_t)x.size : hi;
    struct W {
        uint64_t o, n;
        uint32_t i;
    };
    std::vector<W> ws;
    uint64_t end = old_size, reach = 0;  // reach: the end of the writes so far
    for (uint32_t i = 0; i < nw; i++) {
        if (!len[i]) continue;
        if (off[i] == WRITE_APPEND && !known && reach < hi) {
            P.status = WRITE_NEED_SIZE;
            return P;
        }
        const uint64_t o = off[i] == WRITE_APPEND ? end : off[i];
        if (o + len[i] < o || o + len[i] > (1ull << 62)) {
            P.status = WRITE_TOO_LARGE;
            return P;
        }
        ws.push_back(W{o, len[i], i});
        end = std::max(end, o + len[i]);
        reach = std::max(reach, o + len[i]);
    }
    if (!known && reach > lo) {  // the writes must cover [lo, hi)
        std::vector<std::pair<uint64_t, uint64_t>> iv;
        for (const W& w : ws)
            if (w.o < hi && w.o + w.n > lo) iv.push_back({std::max(w.o, lo), std::min(w.o + w.n, hi)});
        std::sort(iv.begin(), iv.end());
        uint64_t at = lo;
        for (const auto& v : iv)
            if (v.first <= at) at = std::max(at, v.second);
        if (at < hi) {
            P.status = WRITE_NEED_SIZE;
            return P;
        }
    }
    P.size_known = known || reach > lo;
    P.new_size = end;
    P.nblocks = P.size_known ? (end + bs - 1) / bs : nb;
    if (P.nblocks > (1ull << 62) / bs) {
        P.status = WRITE_TOO_LARGE;
        return P;
    }
    // the re-encoded blocks: those a write overlaps, and every block from the one holding the old end on when the data grows
    std::vector<std::pair<uint64_t, uint64_t>> rr;  // block ranges [a, b]
    for (const W& w : ws) rr.push_back({w.o / bs, (w.o + w.n - 1) / bs});
    if (P.size_known && end > old_size) rr.push_back({old_size / bs, (end - 1) / bs});
    std::sort(rr.begin(), rr.end());
    std::vector<std::pair<uint64_t, uint64_t>> runs;
    for (const auto& r : rr) {
        if (!runs.empty() && r.first <= runs.back().second + 1) runs.back().second = std::max(runs.back().second, r.second);
        else runs.push_back(r);
    }
    uint64_t count = 0;
    for (const auto& r : runs) count += r.second - r.first + 1;
    if (count > 0xFFFFFFFEull) {
        P.status = WRITE_TOO_LARGE;
        return P;
    }
    if (!count) return P;
    P.enc.reserve(count);
    for (const auto& r : runs)
        for (uint64_t b = r.first; b <= r.second; b++) P.enc.push_back(b);
    const uint64_t data_end = P.size_known ? end : hi;  // with the size unknown only blocks before the last are re-encoded
    P.enc_len.resize(count);
    for (uint64_t j = 0; j < count; j++) P.enc_len[j] = (uint32_t)std::min<uint64_t>(bs, data_end - P.enc[j] * bs);
    // pieces: a sweep over the write boundaries; inside each elementary interval the latest write wins, else the old data below
    // old_size, else zeros. Each interval is cut at the block boundaries of the re-encoded blocks it meets.
    std::vector<uint64_t> cuts{0, old_size, data_end};
    for (const W& w : ws) cuts.push_back(w.o), cuts.push_back(w.o + w.n);
    std::sort(cuts.begin(), cuts.end());
    cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
    std::vector<std::vector<uint32_t>> starts(cuts.size()), ends(cuts.size());
    auto at_cut = [&](uint64_t p) { return (size_t)(std::lower_bound(cuts.begin(), cuts.end(), p) - cuts.begin()); };
    for (uint32_t k = 0; k < (uint32_t)ws.size(); k++) starts[at_cut(ws[k].o)].push_back(k), ends[at_cut(ws[k].o + ws[k].n)].push_back(k);
    P.decode.assign(count, 0);
    P.piece_of.assign(count + 1, 0);
    std::set<uint32_t> active;
    std::vector<std::vector<WritePiece>> per(count);
    for (size_t c = 0; c + 1 < cuts.size(); c++) {
        for (uint32_t k : ends[c]) active.erase(k);
        for (uint32_t k : starts[c]) active.insert(k);
        const uint64_t p = cuts[c], q = std::min(cuts[c + 1], data_end);
        if (p >= q) continue;
        const bool wr = !active.empty();
        const uint32_t k = wr ? *active.rbegin() : 0;
        const uint32_t kind = wr ? PIECE_WRITE : p < old_size ? PIECE_OLD : PIECE_ZERO;
        for (size_t j = std::lower_bound(P.enc.begin(), P.enc.end(), p / bs) - P.enc.begin(); j < count && P.enc[j] * bs < q; j++) {
            const uint64_t a = std::max(p, P.enc[j] * bs), e = std::min(q, P.enc[j] * bs + bs);
            WritePiece pc{kind, (uint32_t)(a - P.enc[j] * bs), (uint32_t)(e - a), wr ? ws[k].i : 0u, wr ? a - ws[k].o : 0};
            std::vector<WritePiece>& v = per[j];
            if (!v.empty() && v.back().kind == pc.kind && v.back().write == pc.write && v.back().at + v.back().len == pc.at &&
                (pc.kind != PIECE_WRITE || v.back().from + v.back().len == pc.from))
                v.back().len += pc.len;
            else v.push_back(pc);
            if (kind == PIECE_OLD) P.decode[j] = 1;
        }
    }
    for (uint64_t j = 0; j < count; j++) {
        P.piece_of[j + 1] = P.piece_of[j] + per[j].size();
        P.pieces.insert(P.pieces.end(), per[j].begin(), per[j].end());
    }
    // the cut and the segments behind it
    const uint64_t k0 = P.enc[0];
    P.cut = record_prefix_bit(x, std::min(k0, nb));
    if (P.cut % 8) P.segs.push_back(WriteSeg{SEG_CARRY, 0, 0, P.cut & ~7ull, P.cut % 8});
    uint64_t j = 0;
    for (uint64_t b = k0; b < P.nblocks;) {
        if (j < count && P.enc[j] == b) {
            uint64_t e = j;
            while (e + 1 < count && P.enc[e + 1] == P.enc[e] + 1) e++;
            P.segs.push_back(WriteSeg{SEG_NEW, j, e - j + 1, 0, 0});
            b = P.enc[e] + 1, j = e + 1;
        } else {
            const uint64_t e = j < count ? std::min(P.enc[j], nb) : nb;  // old records b .. e - 1
            const uint64_t a = record_prefix_bit(x, b);
            P.segs.push_back(WriteSeg{SEG_OLD, b, e - b, a, record_prefix_bit(x, e) - a});
            b = e;
        }
    }
    P.segs.push_back(WriteSeg{SEG_END, 0, 0, 0, 0});
    return P;
}

// ---- the plan of writes into many streams (kz_write_ranges_streams) ----------------------------------------------------------------
// Each stream has a group, as in plan_reads_streams: streams of one group share transform48, entropy, block_size and checksum_bits, so
// their re-encoded blocks may share a pass (one decode, one copy launch, one encode); blocks of different groups never do.
struct WriteStream {
    const StreamIndex* x;  // null: the stream takes no part (no write names it, or it failed a check): its plan is empty
    uint32_t group;        // equal groups have equal block sizes and encode costs
    uint64_t enc_cost;     // compress_block_cost of the stream's block size and codec
};

struct WriteStreamsPlan {
    std::vector<WritePlan> plans;   // per stream: what plan_writes gives for its writes alone (passes included), its pieces naming
                                    // writes by their index in the call's arrays
    std::vector<uint32_t> stream;   // per re-encoded pair: its stream ...
    std::vector<uint32_t> enc;      // ... and its index into plans[stream].enc; pairs in plan order (group, then stream, then block)
    std::vector<uint64_t> pair_of;  // per stream: its first pair (a stream's pairs are contiguous)
    std::vector<uint32_t> first;    // pass p re-encodes pairs first[p] .. first[p + 1] - 1, all of one group
    uint32_t npasses() const { return first.empty() ? 0 : (uint32_t)first.size() - 1; }
};

// Write i goes to stream w_stream[i] (null: every write to stream 0); a stream's writes keep their array order. Groups are ordered by
// their first appearance among the streams, each group's run of pairs is cut into passes by plan_decompress_passes under
// write_block_cost. Only streams whose plan is WRITE_OK have pairs.
inline WriteStreamsPlan plan_writes_streams(const std::vector<WriteStream>& S, uint32_t nw, const uint32_t* w_stream, const uint64_t* off,
                                            const uint64_t* len, uint64_t budget = STREAM_PASS_BUDGET) {
    WriteStreamsPlan W;
    const uint32_t ns = (uint32_t)S.size();
    std::vector<std::vector<uint64_t>> o(ns), l(ns);
    std::vector<std::vector<uint32_t>> idx(ns);  // the writes of each stream, by their index in the call's arrays
    for (uint32_t i = 0; i < nw; i++) {
        const uint32_t s = w_stream ? w_stream[i] : 0u;
        if (len[i] && s < ns && S[s].x) o[s].push_back(off[i]), l[s].push_back(len[i]), idx[s].push_back(i);
    }
    W.plans.resize(ns);
    W.pair_of.assign(ns, 0);
    std::vector<uint32_t> groups;  // in order of first appearance
    for (uint32_t s = 0; s < ns; s++) {
        if (!S[s].x) continue;
        const StreamIndex& x = *S[s].x;
        WritePlan& P = W.plans[s];
        P = plan_write_blocks(x, (uint32_t)o[s].size(), o[s].data(), l[s].data());
        for (WritePiece& pc : P.pieces)
            if (pc.kind == PIECE_WRITE) pc.write = idx[s][pc.write];
        if (P.status == WRITE_OK && !P.nothing())
            P.first = plan_decompress_passes((uint32_t)P.enc.size(), decompress_slot(x.block_size), write_block_cost(x.block_size, S[s].enc_cost), budget).first;
        if (std::find(groups.begin(), groups.end(), S[s].group) == groups.end()) groups.push_back(S[s].group);
    }
    for (uint32_t g : groups) {
        const size_t a = W.stream.size();
        uint32_t bs = 0;
        uint64_t cost = 0;
        for (uint32_t s = 0; s < ns; s++) {
            if (!S[s].x || S[s].group != g) continue;
            W.pair_of[s] = W.stream.size();
            const WritePlan& P = W.plans[s];
            if (P.status != WRITE_OK) continue;
            for (uint32_t j = 0; j < (uint32_t)P.enc.size(); j++) W.stream.push_back(s), W.enc.push_back(j);
            bs = S[s].x->block_size, cost = S[s].enc_cost;
        }
        const uint32_t n = (uint32_t)(W.stream.size() - a);
        if (!n) continue;
        const PassPlan pp = plan_decompress_passes(n, decompress_slot(bs), write_block_cost(bs, cost), budget);
        for (uint32_t p = 0; p < pp.npasses(); p++) W.first.push_back((uint32_t)a + pp.first[p]);
    }
    W.first.push_back((uint32_t)W.stream.size());
    return W;
}

// The one-stream plan: writes i = 0 .. nw - 1 (len[i] bytes to decoded offset off[i], or to the current end when off[i] == WRITE_APPEND)
// on the stream x, whose decoded size is x.size (-1: unknown). With the size unknown the old last block's length decides the result when
// a KZ_WRITE_APPEND comes before the writes reach past the last block's range, or a write reaches into that range or beyond without the
// writes covering all of it: then status is WRITE_NEED_SIZE and the caller plans again with the size. WRITE_TOO_LARGE: an offset plus its
// length overflows, the blocks after the writes times the block size pass 2^62, or more than 2^32 - 2 blocks would be re-encoded.
inline WritePlan plan_writes(const StreamIndex& x, uint32_t nw, const uint64_t* off, const uint64_t* len, uint64_t enc_cost,
                             uint64_t budget = STREAM_PASS_BUDGET) {
    return plan_writes_streams({WriteStream{&x, 0, enc_cost}}, nw, nullptr, off, len, budget).plans[0];
}

// The index of the new stream: x with the records from the cut on laid out again. new_bits[j] / prefix_bits[j]: the payload and prefix
// bit lengths of re-encoded block j; end_marker_bits: the length of the end marker. size: the new size when the plan knows it, else x's.
// Returns the bit length of the new stream.
inline uint64_t splice_records(const StreamIndex& x, const WritePlan& P, const std::vector<uint64_t>& new_bits, const std::vector<uint32_t>& prefix_bits,
                               uint32_t end_marker_bits, StreamIndex& out) {
    out = x;
    if (P.nothing()) return 8 * x.stream_bytes;
    out.start.resize(P.nblocks);
    out.bits.resize(P.nblocks);
    uint64_t pos = P.cut;
    for (const WriteSeg& s : P.segs) {
        if (s.kind == SEG_NEW) {
            for (uint64_t j = s.first; j < s.first + s.count; j++) {
                out.start[P.enc[j]] = pos + prefix_bits[j];
                out.bits[P.enc[j]] = new_bits[j];
                pos += prefix_bits[j] + new_bits[j];
            }
        } else if (s.kind == SEG_OLD) {
            for (uint64_t b = s.first; b < s.first + s.count; b++) out.start[b] = x.start[b] - s.bit + pos, out.bits[b] = x.bits[b];
            pos += s.bits;
        } else if (s.kind == SEG_END) {
            pos += end_marker_bits;
        }
    }
    out.stream_bytes = (pos + 7) / 8;
    if (P.size_known) out.size = (int64_t)P.new_size;
    return pos;
}

}  // namespace kz
