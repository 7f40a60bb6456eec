// CPU check of the many-stream read plan (plan_reads_streams in kanzi-go_b200/csrc/kz_read_plan.h) against a brute-force plan, for
// tests/test_read_plan_streams_host.py. Built under ASan / UBSan and run as `read_plan_streams_host <rounds> <seed>`.
//
// Random stream sets mix block sizes and decode groups, hold streams of zero blocks and decoded sizes known or -1; requests include zero
// lengths, offsets past the end and 1 << 62. Checked: every touched (stream, block) pair appears exactly once and in plan order (group,
// stream, block); no pass mixes groups or exceeds the budget, and each group is cut as plan_decompress_passes cuts it; the slices cover
// exactly the deliverable bytes of every request; a one-stream plan equals plan_reads.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <set>
#include <tuple>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_read_plan.h"

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd() {
    rng_state ^= rng_state << 13;
    rng_state ^= rng_state >> 7;
    rng_state ^= rng_state << 17;
    return rng_state;
}

static int fails = 0;
#define CHECK(c, ...)                                  \
    do {                                               \
        if (!(c)) {                                    \
            if (fails++ < 20) {                        \
                printf("line %d: %s: ", __LINE__, #c); \
                printf(__VA_ARGS__);                   \
                printf("\n");                          \
            }                                          \
        }                                              \
    } while (0)

static uint64_t total_of(const kz::ReadStream& s) { return s.size >= 0 ? (uint64_t)s.size : s.nblocks * s.block_size; }

static void check_plan(const std::vector<kz::ReadStream>& S, const std::vector<uint32_t>& rs, const std::vector<uint64_t>& off,
                       const std::vector<uint64_t>& len, uint64_t budget, int round) {
    const uint32_t nreq = (uint32_t)off.size();
    const kz::ReadPlan P = kz::plan_reads_streams(S, nreq, rs.data(), off.data(), len.data(), budget);
    // brute force: the clipped lengths and the set of touched pairs in (group, stream, block) order
    std::vector<uint64_t> want(nreq);
    std::set<std::tuple<uint32_t, uint32_t, uint64_t>> touched;
    for (uint32_t i = 0; i < nreq; i++) {
        const kz::ReadStream& s = S[rs[i]];
        const uint64_t total = total_of(s);
        want[i] = off[i] < total ? std::min(len[i], total - off[i]) : 0;
        for (uint64_t p = off[i]; p < off[i] + want[i]; p = (p / s.block_size + 1) * s.block_size) touched.insert({s.group, rs[i], p / s.block_size});
    }
    CHECK(P.want == want, "round %d: clipped lengths", round);
    CHECK(P.blocks.size() == touched.size() && P.stream.size() == touched.size(), "round %d: %zu pairs, expected %zu", round, P.blocks.size(),
          touched.size());
    if (P.blocks.size() != touched.size()) return;
    size_t k = 0;
    for (const auto& t : touched) {
        CHECK(P.stream[k] == std::get<1>(t) && P.blocks[k] == std::get<2>(t), "round %d: pair %zu out of order", round, k);
        k++;
    }
    const uint32_t nk = (uint32_t)P.blocks.size();
    // passes: one group each, within the budget (or one block), each group's run cut into chunks of budget / cost
    CHECK(!P.first.empty() && P.first.front() == 0 && P.first.back() == nk, "round %d: passes do not span the pairs", round);
    std::vector<uint32_t> expect{0};
    for (uint32_t a = 0, e; a < nk; a = e) {
        const kz::ReadStream& g = S[P.stream[a]];
        for (e = a; e < nk && S[P.stream[e]].group == g.group;) e++;
        const uint64_t per = std::max<uint64_t>(1, budget / kz::read_block_cost(g.block_size));
        for (uint64_t b = a + per; b < e; b += per) expect.push_back((uint32_t)b);
        expect.push_back(e);
    }
    CHECK(P.first == expect, "round %d: pass cuts", round);
    for (uint32_t p = 0; p + 1 < P.first.size(); p++) {
        const uint32_t a = P.first[p], e = P.first[p + 1];
        CHECK(e > a, "round %d: empty pass %u", round, p);
        for (uint32_t j = a; j < e; j++) CHECK(S[P.stream[j]].group == S[P.stream[a]].group, "round %d: pass %u mixes groups", round, p);
        CHECK(e - a == 1 || (e - a) * kz::read_block_cost(S[P.stream[a]].block_size) <= budget, "round %d: pass %u over the budget", round, p);
    }
    // slices: grouped by pair, inside their block, at the bytes the request names, tiling every request exactly once
    CHECK(P.slice_of.size() == nk + 1 && P.slice_of[0] == 0 && P.slice_of[nk] == P.slices.size(), "round %d: slice_of", round);
    std::vector<std::vector<std::pair<uint64_t, uint64_t>>> cover(nreq);
    for (uint32_t j = 0; j < nk; j++)
        for (uint64_t q = P.slice_of[j]; q < P.slice_of[j + 1]; q++) {
            const kz::ReadSlice& sl = P.slices[q];
            CHECK(sl.block == j, "round %d: slice %llu filed under the wrong pair", round, (unsigned long long)q);
            CHECK(sl.req < nreq && rs[sl.req] == P.stream[j], "round %d: slice on another stream", round);
            const uint32_t bs = S[P.stream[j]].block_size;
            CHECK(sl.len >= 1 && (uint64_t)sl.in_block + sl.len <= bs, "round %d: slice outside its block", round);
            CHECK(P.blocks[j] * bs + sl.in_block == off[sl.req] + sl.at, "round %d: slice at the wrong bytes", round);
            cover[sl.req].push_back({sl.at, sl.len});
        }
    for (uint32_t i = 0; i < nreq; i++) {
        std::sort(cover[i].begin(), cover[i].end());
        uint64_t at = 0;
        for (const auto& c : cover[i]) {
            CHECK(c.first == at, "round %d: request %u has a gap or an overlap at %llu", round, i, (unsigned long long)at);
            at = c.first + c.second;
        }
        CHECK(at == want[i], "round %d: request %u covers %llu of %llu bytes", round, i, (unsigned long long)at, (unsigned long long)want[i]);
    }
}

static void check_one_stream(const kz::ReadStream& s, const std::vector<uint64_t>& off, const std::vector<uint64_t>& len, uint64_t budget, int round) {
    const uint32_t nreq = (uint32_t)off.size();
    const std::vector<uint32_t> zero(nreq, 0);
    const kz::ReadPlan A = kz::plan_reads(s.nblocks, s.block_size, s.size, nreq, off.data(), len.data(), budget);
    const kz::ReadPlan B = kz::plan_reads_streams({kz::ReadStream{s.nblocks, s.block_size, s.size, 7}}, nreq, zero.data(), off.data(), len.data(), budget);
    bool same = A.stream == B.stream && A.blocks == B.blocks && A.first == B.first && A.slice_of == B.slice_of && A.want == B.want &&
                A.slices.size() == B.slices.size();
    for (size_t q = 0; same && q < A.slices.size(); q++) {
        const kz::ReadSlice &x = A.slices[q], &y = B.slices[q];
        same = x.req == y.req && x.block == y.block && x.in_block == y.in_block && x.len == y.len && x.at == y.at;
    }
    CHECK(same, "round %d: the one-stream plan differs from plan_reads", round);
}

int main(int argc, char** argv) {
    const int rounds = argc > 1 ? atoi(argv[1]) : 300;
    if (argc > 2) rng_state ^= strtoull(argv[2], nullptr, 10) * 0x2545F4914F6CDD1Dull;
    static const uint32_t SIZES[] = {1024, 4096, 65536, 1u << 20, 4u << 20, 1u << 30};
    uint64_t pairs = 0, passes = 0;
    for (int r = 0; r < rounds; r++) {
        // decode groups with their block sizes (two groups may share a block size), then streams in them
        const uint32_t ngroups = 1 + (uint32_t)(rnd() % 4);
        std::vector<uint32_t> gbs(ngroups);
        for (uint32_t& b : gbs) b = SIZES[rnd() % 6];
        const uint32_t ns = (uint32_t)(rnd() % 24);
        std::vector<kz::ReadStream> S(ns);
        for (kz::ReadStream& s : S) {
            s.group = (uint32_t)(rnd() % ngroups);
            s.block_size = gbs[s.group];
            const uint64_t cap = s.block_size >= (1u << 30) ? 4 : 60;
            s.nblocks = rnd() % 5 == 0 ? 0 : 1 + rnd() % cap;
            s.size = s.nblocks == 0 ? 0 : (rnd() % 2 ? -1 : (int64_t)((s.nblocks - 1) * s.block_size + 1 + rnd() % s.block_size));
        }
        std::vector<uint32_t> rs;
        std::vector<uint64_t> off, len;
        const uint32_t nreq = ns ? (uint32_t)(rnd() % 300) : 0;
        for (uint32_t i = 0; i < nreq; i++) {
            const uint32_t s = (uint32_t)(rnd() % ns);
            const uint64_t total = total_of(S[s]), bs = S[s].block_size;
            uint64_t o = rnd() % (total + 2 * bs), n = rnd() % (3 * bs);
            switch (rnd() % 10) {
                case 0: n = 0; break;                            // zero length
                case 1: o = total + rnd() % 100; break;          // at or past the end
                case 2: o = 1ull << 62; break;                   // far past the end
                case 3: o = 0, n = total + rnd() % 10; break;    // every block of the stream
                case 4: n = 1ull << 62; break;                   // runs to the end
                default: break;
            }
            rs.push_back(s), off.push_back(o), len.push_back(n);
        }
        const uint64_t budget = rnd() % 3 == 0 ? kz::STREAM_PASS_BUDGET : (rnd() % 2 ? (1ull << 20) : 1 + rnd() % (64ull << 20));
        check_plan(S, rs, off, len, budget, r);
        for (const kz::ReadStream& s : S) {
            std::vector<uint64_t> o1, l1;
            for (uint32_t i = 0; i < nreq; i++)
                if (&S[rs[i]] == &s) o1.push_back(off[i]), l1.push_back(len[i]);
            check_one_stream(s, o1, l1, budget, r);
        }
        const kz::ReadPlan P = kz::plan_reads_streams(S, nreq, rs.data(), off.data(), len.data(), budget);
        pairs += P.blocks.size(), passes += P.npasses();
    }
    if (fails) {
        printf("%d failures\n", fails);
        return 1;
    }
    printf("plan check done: %d rounds, %llu pairs, %llu passes\n", rounds, (unsigned long long)pairs, (unsigned long long)passes);
    return 0;
}
