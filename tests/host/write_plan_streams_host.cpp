// CPU check of the many-stream write plan (plan_writes_streams in kanzi-go_b200/csrc/kz_write_plan.h), for
// tests/test_write_plan_streams_host.py. Built under ASan / UBSan and run as `write_plan_streams_host <rounds> <seed>`.
//
// Random stream sets mix block sizes and groups, hold empty streams, sizes known or -1 and streams that take no part; writes interleave
// streams and include zero lengths, KZ_WRITE_APPEND, overlaps and offsets near 2^62. Checked: each stream's plan equals plan_writes over
// its own writes (pieces renamed to the call's write indexes); the re-encoded (stream, block) pairs appear exactly once, in plan order
// (group by first appearance, then stream, then block), and only for WRITE_OK plans; every pass holds one group, stays within the budget
// (or holds one pair), and each group's run is cut as plan_decompress_passes cuts it; the plan is the same when computed twice; a
// one-stream plan equals the single plan.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_write_plan.h"

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

static bool same_plan(const kz::WritePlan& A, const kz::WritePlan& B) {
    if (A.status != B.status || A.new_size != B.new_size || A.size_known != B.size_known || A.nblocks != B.nblocks || A.enc != B.enc ||
        A.enc_len != B.enc_len || A.decode != B.decode || A.piece_of != B.piece_of || A.first != B.first || A.cut != B.cut ||
        A.pieces.size() != B.pieces.size() || A.segs.size() != B.segs.size())
        return false;
    for (size_t q = 0; q < A.pieces.size(); q++) {
        const kz::WritePiece &x = A.pieces[q], &y = B.pieces[q];
        if (x.kind != y.kind || x.at != y.at || x.len != y.len || x.write != y.write || x.from != y.from) return false;
    }
    for (size_t q = 0; q < A.segs.size(); q++) {
        const kz::WriteSeg &x = A.segs[q], &y = B.segs[q];
        if (x.kind != y.kind || x.first != y.first || x.count != y.count || x.bit != y.bit || x.bits != y.bits) return false;
    }
    return true;
}

static bool same_streams_plan(const kz::WriteStreamsPlan& A, const kz::WriteStreamsPlan& B) {
    if (A.stream != B.stream || A.enc != B.enc || A.pair_of != B.pair_of || A.first != B.first || A.plans.size() != B.plans.size()) return false;
    for (size_t s = 0; s < A.plans.size(); s++)
        if (!same_plan(A.plans[s], B.plans[s])) return false;
    return true;
}

// a synthetic index of nb records behind a header of hb bits
static kz::StreamIndex make_index(uint64_t nb, uint32_t bs, int64_t size, uint32_t hb) {
    kz::StreamIndex x;
    x.block_size = bs;
    x.header_bits = hb;
    x.size = size;
    uint64_t pos = hb;
    for (uint64_t b = 0; b < nb; b++) {
        x.start.push_back(pos + 8 + rnd() % 32);
        x.bits.push_back(1 + rnd() % 300);
        pos = x.start.back() + x.bits.back();
    }
    x.stream_bytes = (pos + 8 + 7) / 8;
    return x;
}

static void check_plan(const std::vector<kz::WriteStream>& S, const std::vector<uint32_t>& ws, const std::vector<uint64_t>& off,
                       const std::vector<uint64_t>& len, uint64_t budget, int round) {
    const uint32_t ns = (uint32_t)S.size(), nw = (uint32_t)off.size();
    const kz::WriteStreamsPlan W = kz::plan_writes_streams(S, nw, ws.data(), off.data(), len.data(), budget);
    CHECK(same_streams_plan(W, kz::plan_writes_streams(S, nw, ws.data(), off.data(), len.data(), budget)), "round %d: not deterministic", round);
    CHECK(W.plans.size() == ns && W.pair_of.size() == ns, "round %d: per-stream tables", round);
    if (W.plans.size() != ns || W.pair_of.size() != ns) return;
    // each stream's plan is plan_writes over its own writes, the pieces naming the call's write indexes
    for (uint32_t s = 0; s < ns; s++) {
        if (!S[s].x) {
            CHECK(W.plans[s].nothing() && W.plans[s].status == kz::WRITE_OK, "round %d: stream %u takes no part but has a plan", round, s);
            continue;
        }
        std::vector<uint64_t> o, l;
        std::vector<uint32_t> idx;
        for (uint32_t i = 0; i < nw; i++)
            if (ws[i] == s) o.push_back(off[i]), l.push_back(len[i]), idx.push_back(i);
        kz::WritePlan P = kz::plan_writes(*S[s].x, (uint32_t)o.size(), o.data(), l.data(), S[s].enc_cost, budget);
        for (kz::WritePiece& pc : P.pieces)
            if (pc.kind == kz::PIECE_WRITE) pc.write = idx[pc.write];
        CHECK(same_plan(W.plans[s], P), "round %d: stream %u's plan differs from plan_writes", round, s);
    }
    // the pairs: exactly the re-encoded blocks of the WRITE_OK plans, in (group by first appearance, stream, block) order
    std::vector<uint32_t> gorder;
    for (uint32_t s = 0; s < ns; s++)
        if (S[s].x && std::find(gorder.begin(), gorder.end(), S[s].group) == gorder.end()) gorder.push_back(S[s].group);
    std::vector<uint32_t> es, ej;
    for (uint32_t g : gorder)
        for (uint32_t s = 0; s < ns; s++)
            if (S[s].x && S[s].group == g && W.plans[s].status == kz::WRITE_OK)
                for (uint32_t j = 0; j < (uint32_t)W.plans[s].enc.size(); j++) es.push_back(s), ej.push_back(j);
    CHECK(W.stream == es && W.enc == ej, "round %d: %zu pairs, expected %zu, or out of order", round, W.stream.size(), es.size());
    for (uint32_t s = 0; s < ns; s++)
        if (S[s].x && W.plans[s].status == kz::WRITE_OK && !W.plans[s].nothing())
            CHECK(W.pair_of[s] < W.stream.size() && W.stream[W.pair_of[s]] == s && W.enc[W.pair_of[s]] == 0, "round %d: pair_of[%u]", round, s);
    // passes: one group each, within the budget, each group's run cut as plan_decompress_passes cuts it
    const uint32_t n = (uint32_t)W.stream.size();
    CHECK(!W.first.empty() && W.first.front() == 0 && W.first.back() == n, "round %d: passes do not span the pairs", round);
    std::vector<uint32_t> expect;
    for (uint32_t a = 0, e; a < n; a = e) {
        const kz::WriteStream& g = S[W.stream[a]];
        for (e = a; e < n && S[W.stream[e]].group == g.group;) e++;
        const uint64_t per = std::max<uint64_t>(1, budget / kz::write_block_cost(g.x->block_size, g.enc_cost));
        for (uint64_t b = a; b < e; b += per) expect.push_back((uint32_t)b);
    }
    expect.push_back(n);
    CHECK(W.first == expect, "round %d: pass cuts", round);
    for (uint32_t p = 0; p + 1 < W.first.size(); p++) {
        const uint32_t a = W.first[p], e = W.first[p + 1];
        CHECK(e > a, "round %d: empty pass %u", round, p);
        if (e <= a) continue;
        const kz::WriteStream& g = S[W.stream[a]];
        for (uint32_t j = a; j < e; j++) CHECK(S[W.stream[j]].group == g.group, "round %d: pass %u mixes groups", round, p);
        CHECK(e - a == 1 || (e - a) * kz::write_block_cost(g.x->block_size, g.enc_cost) <= budget, "round %d: pass %u over the budget", round, p);
    }
}

static void check_one_stream(const kz::StreamIndex& x, uint64_t enc_cost, const std::vector<uint64_t>& off, const std::vector<uint64_t>& len,
                             uint64_t budget, int round) {
    const uint32_t nw = (uint32_t)off.size();
    const std::vector<uint32_t> zero(nw, 0);
    const kz::WritePlan A = kz::plan_writes(x, nw, off.data(), len.data(), enc_cost, budget);
    const kz::WriteStreamsPlan W = kz::plan_writes_streams({kz::WriteStream{&x, 5, enc_cost}}, nw, zero.data(), off.data(), len.data(), budget);
    CHECK(same_plan(A, W.plans[0]), "round %d: the one-stream plan differs from plan_writes", round);
    if (A.status == kz::WRITE_OK && !A.nothing()) {
        CHECK(W.first == A.first, "round %d: the one-stream passes differ from plan_writes's", round);
        std::vector<uint32_t> j(A.enc.size());
        for (uint32_t k = 0; k < (uint32_t)j.size(); k++) j[k] = k;
        CHECK(W.enc == j && W.stream == std::vector<uint32_t>(j.size(), 0u), "round %d: one-stream pairs", round);
    } else {
        CHECK(W.stream.empty() && W.first == std::vector<uint32_t>{0}, "round %d: a one-stream plan without blocks has pairs", round);
    }
}

int main(int argc, char** argv) {
    const int rounds = argc > 1 ? atoi(argv[1]) : 300;
    if (argc > 2) rng_state ^= strtoull(argv[2], nullptr, 10) * 0x2545F4914F6CDD1Dull;
    static const uint32_t SIZES[] = {1024, 4096, 65536, 1u << 20, 4u << 20};
    static const uint32_t HB[] = {0, 160, 176, 192, 208};
    uint64_t pairs = 0, passes = 0, need = 0;
    for (int r = 0; r < rounds; r++) {
        const uint32_t ngroups = 1 + (uint32_t)(rnd() % 4);
        std::vector<uint32_t> gbs(ngroups);
        std::vector<uint64_t> gcost(ngroups);
        for (uint32_t g = 0; g < ngroups; g++) gbs[g] = SIZES[rnd() % 5], gcost[g] = gbs[g] * (2 + rnd() % 4);
        const uint32_t ns = (uint32_t)(rnd() % 20);
        std::vector<kz::StreamIndex> X(ns);
        std::vector<kz::WriteStream> S(ns);
        for (uint32_t s = 0; s < ns; s++) {
            const uint32_t g = (uint32_t)(rnd() % ngroups), bs = gbs[g];
            const uint64_t nb = rnd() % 5 == 0 ? 0 : 1 + rnd() % 12;
            const int64_t size = nb == 0 ? 0 : rnd() % 3 == 0 ? -1 : (int64_t)((nb - 1) * bs + 1 + (rnd() % 3 == 0 ? bs - 1 : rnd() % bs));
            X[s] = make_index(nb, bs, size, HB[rnd() % 5]);
            S[s] = kz::WriteStream{rnd() % 8 == 0 ? nullptr : &X[s], g, gcost[g]};
        }
        std::vector<uint32_t> ws;
        std::vector<uint64_t> off, len;
        const uint32_t nw = ns ? (uint32_t)(rnd() % 60) : 0;
        for (uint32_t i = 0; i < nw; i++) {
            const uint32_t s = (uint32_t)(rnd() % ns);
            const uint64_t bs = X[s].block_size, total = X[s].nblocks() * bs;
            uint64_t o = rnd() % (total + 2 * bs + 1), n = 1 + rnd() % (2 * bs);
            switch (rnd() % 10) {
                case 0: n = 0; break;                                  // zero length
                case 1: o = kz::WRITE_APPEND; break;                   // append
                case 2: o = 0, n = total + rnd() % 10; break;          // the whole stream
                case 3: o = (1ull << 62) - rnd() % 4; break;           // near the limit
                case 4: o = total + rnd() % (3 * bs); break;           // past the end: a zero gap
                default: break;
            }
            ws.push_back(s), off.push_back(o), len.push_back(n);
        }
        const uint64_t budget = rnd() % 3 == 0 ? kz::STREAM_PASS_BUDGET : (rnd() % 2 ? (64ull << 20) : 1 + rnd() % (256ull << 20));
        check_plan(S, ws, off, len, budget, r);
        for (uint32_t s = 0; s < ns; s++) {
            std::vector<uint64_t> o1, l1;
            for (uint32_t i = 0; i < nw; i++)
                if (ws[i] == s) o1.push_back(off[i]), l1.push_back(len[i]);
            check_one_stream(X[s], S[s].enc_cost, o1, l1, budget, r);
        }
        const kz::WriteStreamsPlan W = kz::plan_writes_streams(S, nw, ws.data(), off.data(), len.data(), budget);
        pairs += W.stream.size(), passes += W.npasses();
        for (const kz::WritePlan& P : W.plans) need += P.status == kz::WRITE_NEED_SIZE;
    }
    if (fails) {
        printf("%d failures\n", fails);
        return 1;
    }
    printf("plan check done: %d rounds, %llu pairs, %llu passes, %llu plans that need the size\n", rounds, (unsigned long long)pairs,
           (unsigned long long)passes, (unsigned long long)need);
    return 0;
}
