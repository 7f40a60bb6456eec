// CPU model of sbrt_inverse_multi_kernel (kanzi-go_b200/csrc/kz_sbrt.cu), the RANK / MTFT inverse for blocks of at most 16 MiB, written
// thread by thread the way the kernel moves data (tests/test_sbrt_inv_multi_staged_host.py). tests/host/sbrt_inv_multi_host.cpp is the
// schedule before this one (ranks by shuffles, no sentinel slots); both give the same output and count the same events.
//   - 128 threads x 2 entries (q, x = p << 8 | symbol) in registers, thread t holding ranks 2 t and 2 t + 1;
//   - two mirror copies of the list, step j writing the copy of parity j & 1 and reading the other one; position k is slot k + 2 of a
//     copy, and slot 1 holds a sentinel with a q above any qc;
//   - the candidates for step j + 1 (entries r2 and r2 - 1, the sentinel for r2 == 0) loaded after step j;
//   - the decision of the entry at rank r2 after step j from the two candidates and qc;
//   - the entry above a thread's first one: a shuffle-up inside a warp, the copy of the previous step on lane 0 (the sentinel for thread 0);
//   - the ranks of round k staged in s_rk[k & 1] (warp 0 stores round k + 2 at step 30 of round k), every thread holding a round as 8 words
//     (mine) plus the first word of the next round, r3 taken from them and r / r2 carried from the steps before; then the tail, whose
//     ranks come from the staged bytes.
// The model also counts the events that reach each of these, so that the test can assert that its corpus keeps reaching them.
#include <cstdint>

namespace {

constexpr int THREADS = 128, S = 2;

enum Event {
    EV_FRESH_AT_R2,         // the entry at rank r2 after the step is the fresh one (decided by cb)
    EV_DOWN_TO_R2,          // the entry r2 - 1 moves down to r2
    EV_CAND_STAYS,          // r2 <= r and ca.q > qc: the candidate keeps its place
    EV_SENTINEL_MOVE,       // r2 == 0 and a move: the sentinel above position 0 decides
    EV_CA_TIE,              // r2 <= r and ca.q == qc
    EV_CB_TIE,              // a move at r2 > 0 with cb.q == qc
    EV_INSERT_64,           // the fresh entry lands exactly at rank 64: lane 0 of warp 1, through the mirror's up-entry
    EV_INSERT_128,
    EV_INSERT_192,
    EV_INSERT_WARP_TIE,     // the same at any of the three with q[nr] == qc before the step
    EV_CROSS_64,            // an entry crosses the boundary between warps 0 and 1 (nr < 64 <= r)
    EV_CROSS_128,
    EV_CROSS_192,
    EV_TAIL0,               // n mod 32 == 0 .. 31: EV_TAIL0 + (n mod 32)
    EV_COUNT = EV_TAIL0 + 32
};

const char* const kNames =
    "fresh_at_r2,down_to_r2,cand_stays,sentinel_move,ca_tie,cb_tie,insert_64,insert_128,insert_192,insert_warp_tie,cross_64,cross_128,cross_192,"
    "tail0,tail1,tail2,tail3,tail4,tail5,tail6,tail7,tail8,tail9,tail10,tail11,tail12,tail13,tail14,tail15,tail16,tail17,tail18,tail19,tail20,"
    "tail21,tail22,tail23,tail24,tail25,tail26,tail27,tail28,tail29,tail30,tail31";

struct E {
    uint32_t q, x;
};

struct Model {
    bool rank_mode;
    uint64_t* ev;
    uint32_t Q[THREADS][S], X[THREADS][S];
    E s_e[2][258];
    E ca, cb;  // the candidates: every thread loads the same two entries

    explicit Model(bool rm, uint64_t* events) : rank_mode(rm), ev(events) {
        for (int t = 0; t < THREADS; t++)
            for (int k = 0; k < S; k++) {
                Q[t][k] = 0;
                X[t][k] = uint32_t(S * t + k);
                s_e[0][2 + S * t + k] = s_e[1][2 + S * t + k] = E{0u, uint32_t(S * t + k)};
            }
        s_e[0][1] = s_e[1][1] = E{0xFFFFFFFFu, 0u};  // above position 0: a q larger than any qc
        s_e[0][0] = s_e[1][0] = E{0u, 0u};
    }

    void load_candidates(uint32_t r2, int par) {
        ca = s_e[par][2 + r2];
        cb = s_e[par][1 + r2];
    }

    void count(uint32_t r, uint32_t r2, uint32_t qc) {
        const E a = ca, b = cb;
        if (r2 <= r) {
            if (a.q == qc) ev[EV_CA_TIE]++;
            if (a.q > qc) ev[EV_CAND_STAYS]++;
            else {
                ev[b.q > qc ? EV_FRESH_AT_R2 : EV_DOWN_TO_R2]++;
                if (r2 == 0) ev[EV_SENTINEL_MOVE]++;
                else if (b.q == qc) ev[EV_CB_TIE]++;
            }
        }
        uint32_t nr = 0;  // the list is sorted by q (descending) and q[r] <= qc: the fresh entry lands at the first rank with q <= qc
        while (nr < r && Q[nr / S][nr % S] > qc) nr++;
        if (nr == 64 || nr == 128 || nr == 192) {
            ev[EV_INSERT_64 + nr / 64 - 1]++;
            if (nr < r && Q[nr / S][nr % S] == qc) ev[EV_INSERT_WARP_TIE]++;
        }
        for (uint32_t w = 1; w < 4; w++)
            if (nr < 64 * w && 64 * w <= r) ev[EV_CROSS_64 + w - 1]++;
    }

    // one step for every thread; x is the entry at rank r (the same in every thread), replaced by the entry at rank r2 after the step
    uint32_t step(uint32_t r, uint32_t r2, uint32_t i, int par, uint32_t& x) {
        E up[THREADS];
        for (int t = 0; t < THREADS; t++)
            up[t] = t & 31 ? E{Q[t - 1][S - 1], X[t - 1][S - 1]} : s_e[par ^ 1][1 + S * t];  // __shfl_up_sync(.., 1), lane 0 from the mirror
        const uint32_t e = x;
        const uint32_t qc = rank_mode ? (i + (e >> 8)) >> 1 : i;
        const uint32_t fresh = (i << 8) | (e & 0xFFu);
        if (ev) count(r, r2, qc);
        {  // the entry at rank r2 after this step
            const bool mv = r2 <= r && !(ca.q > qc);
            x = mv ? (cb.q > qc ? fresh : cb.x) : ca.x;
        }
        for (int t = 0; t < THREADS; t++) {
            const uint32_t base = uint32_t(S * t);
            uint32_t* q = Q[t];
            uint32_t* xx = X[t];
            bool gk = q[S - 1] > qc;
            for (int k = S - 1; k >= 1; k--) {
                const bool gk1 = q[k - 1] > qc;
                const bool mv = r >= base + k && !gk;
                const uint32_t xin = gk1 ? fresh : xx[k - 1];
                q[k] = mv ? (q[k - 1] < qc ? q[k - 1] : qc) : q[k];
                xx[k] = mv ? xin : xx[k];
                gk = gk1;
            }
            const bool mv = r >= base && !gk;
            q[0] = mv ? (up[t].q < qc ? up[t].q : qc) : q[0];
            xx[0] = mv ? (up[t].q > qc ? fresh : up[t].x) : xx[0];
        }
        for (int t = 0; t < THREADS; t++)
            for (int k = 0; k < S; k++) s_e[par][2 + S * t + k] = E{Q[t][k], X[t][k]};
        return e;
    }
};

}  // namespace

extern "C" const char* sbrt_inv_multi_event_names() { return kNames; }
extern "C" int sbrt_inv_multi_event_count() { return EV_COUNT; }

// mode: 1 = MTFT, 2 = RANK. events: EV_COUNT counters to add to, or null. n <= 2^24 (the kernel's 32-bit entries hold i << 8).
extern "C" int sbrt_inverse_multi_model(int mode, const uint8_t* src, uint32_t n, uint8_t* dst, uint64_t* events) {
    if (n == 0) return 0;
    if (n > (1u << 24)) return -1;
    Model m(mode == 2, events);
    uint8_t s_rk[2][32];  // the ranks of round k in s_rk[k & 1], 0 past the end of the block
    for (uint32_t l = 0; l < 32; l++) s_rk[0][l] = uint8_t(l < n ? src[l] : 0u), s_rk[1][l] = uint8_t(32 + l < n ? src[32 + l] : 0u);
    auto word = [&](int rb, uint32_t w) {  // little-endian, as the kernel's 16-byte loads of s_rk
        return uint32_t(s_rk[rb][4 * w]) | uint32_t(s_rk[rb][4 * w + 1]) << 8 | uint32_t(s_rk[rb][4 * w + 2]) << 16 | uint32_t(s_rk[rb][4 * w + 3]) << 24;
    };
    uint32_t r = s_rk[0][0], r2 = s_rk[0][1];
    uint32_t x = m.s_e[1][2 + r].x;
    m.load_candidates(r2, 1);
    uint32_t i0 = 0;
    for (; i0 + 32 <= n; i0 += 32) {
        const int rb = int(i0 >> 5) & 1;
        uint32_t mine[8], nn[32];
        for (uint32_t w = 0; w < 8; w++) mine[w] = word(rb, w);
        const uint32_t mine8 = word(rb ^ 1, 0);
        for (uint32_t l = 0; l < 32; l++) nn[l] = i0 + 64 + l < n ? src[i0 + 64 + l] : 0u;
        for (uint32_t j = 0; j < 32; j++) {
            const uint32_t r3 = ((j < 30 ? mine[(j + 2) >> 2] : mine8) >> (8 * ((j + 2) & 3))) & 0xFFu;
            dst[i0 + j] = uint8_t(m.step(r, r2, i0 + j, int(j & 1), x));
            m.load_candidates(r3, int(j & 1));
            if (j == 30)
                for (uint32_t l = 0; l < 32; l++) s_rk[rb][l] = uint8_t(nn[l]);
            r = r2;
            r2 = r3;
        }
    }
    if (i0 < n) {
        const uint8_t* rt = s_rk[(i0 >> 5) & 1];
        for (uint32_t j = 0; i0 + j < n; j++) {
            const uint32_t r3 = j < 30 ? rt[j + 2] : 0u;
            dst[i0 + j] = uint8_t(m.step(r, r2, i0 + j, int(j & 1), x));
            m.load_candidates(r3, int(j & 1));
            r = r2;
            r2 = r3;
        }
    }
    if (events) events[EV_TAIL0 + n % 32]++;
    return 0;
}
