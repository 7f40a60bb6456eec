// CPU harness of the write plan (kanzi-go_b200/csrc/kz_write_plan.h), for tests/test_write_plan_host.py. Built as a program under
// ASan / UBSan. It reads cases from stdin and prints each plan as one line of integers:
//   in:  nb block_size size header_bits nw enc_cost budget, then nb record starts, nb record lengths, nw offsets, nw lengths
//   out: status new_size size_known nblocks count cut npasses nsegs npieces | enc | enc_len | decode | piece_of | pieces (5 each) |
//        first | segs (5 each) | the spliced index: total_bits stream_bytes size, then nblocks starts and nblocks lengths
// The splice takes re-encoded block j to be 64 + 13 j bits long behind a prefix of 9 + (j % 4) bits, and an end marker of 8 bits.
#include <cinttypes>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_write_plan.h"

static bool read_u64(uint64_t& v) { return scanf("%" SCNu64, &v) == 1; }

int main() {
    uint64_t nb, bs, nw, hb, enc_cost, budget;
    int64_t size;
    while (read_u64(nb) && read_u64(bs) && scanf("%" SCNd64, &size) == 1 && read_u64(hb) && read_u64(nw) && read_u64(enc_cost) && read_u64(budget)) {
        kz::StreamIndex x;
        x.block_size = (uint32_t)bs;
        x.header_bits = (uint32_t)hb;
        x.size = size;
        x.start.resize(nb);
        x.bits.resize(nb);
        for (auto& v : x.start) read_u64(v);
        for (auto& v : x.bits) read_u64(v);
        x.stream_bytes = (kz::record_prefix_bit(x, nb) + 8 + 7) / 8;
        std::vector<uint64_t> off(nw), len(nw);
        for (auto& v : off) read_u64(v);
        for (auto& v : len) read_u64(v);
        const kz::WritePlan P = kz::plan_writes(x, (uint32_t)nw, off.data(), len.data(), enc_cost, budget);
        const size_t n = P.enc.size();
        printf("%d %" PRIu64 " %d %" PRIu64 " %zu %" PRIu64 " %u %zu %zu", P.status, P.new_size, (int)P.size_known, P.nblocks, n, P.cut, P.npasses(),
               P.segs.size(), P.pieces.size());
        for (size_t j = 0; j < n; j++) printf(" %" PRIu64, P.enc[j]);
        for (size_t j = 0; j < n; j++) printf(" %u", P.enc_len[j]);
        for (size_t j = 0; j < n; j++) printf(" %d", (int)P.decode[j]);
        for (size_t j = 0; j < P.piece_of.size() && n; j++) printf(" %" PRIu64, P.piece_of[j]);
        for (const kz::WritePiece& p : P.pieces) printf(" %u %u %u %u %" PRIu64, p.kind, p.at, p.len, p.write, p.from);
        for (size_t p = 0; p < P.first.size() && n; p++) printf(" %u", P.first[p]);
        for (const kz::WriteSeg& s : P.segs) printf(" %u %" PRIu64 " %" PRIu64 " %" PRIu64 " %" PRIu64, s.kind, s.first, s.count, s.bit, s.bits);
        if (P.status == kz::WRITE_OK) {
            std::vector<uint64_t> nbits(n);
            std::vector<uint32_t> pbits(n);
            for (size_t j = 0; j < n; j++) nbits[j] = 64 + 13 * j, pbits[j] = 9 + (uint32_t)(j % 4);
            kz::StreamIndex y;
            const uint64_t total = kz::splice_records(x, P, nbits, pbits, 8, y);
            printf(" %" PRIu64 " %" PRIu64 " %" PRId64, total, y.stream_bytes, y.size);
            for (uint64_t b = 0; b < y.nblocks(); b++) printf(" %" PRIu64, y.start[b]);
            for (uint64_t b = 0; b < y.nblocks(); b++) printf(" %" PRIu64, y.bits[b]);
        }
        printf("\n");
        fflush(stdout);
    }
    return 0;
}
