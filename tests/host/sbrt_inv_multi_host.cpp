// CPU model of sbrt_inverse_multi_kernel (kanzi-go_b200/csrc/kz_sbrt.cu), the RANK / MTFT inverse for blocks of at most 16 MiB, written
// thread by thread the way the kernel moves data (tests/test_sbrt_inv_multi_host.py):
//   - 128 threads x 2 entries (q, x = p << 8 | symbol) in registers, thread t holding ranks 2 t and 2 t + 1;
//   - two mirror copies of the list, step j writing the copy of parity j & 1 and reading the other one;
//   - the candidates for step j + 1 (entries r2 and r2 - 1, with a sentinel q above position 0) loaded after step j;
//   - the decision of the entry at rank r2 after step j from the two candidates and qc;
//   - the entry above a thread's first one: a shuffle-up inside a warp, the mirror of the previous step across a warp boundary;
//   - the rounds of 32 ranks with r / r2 / r3 read from the round's ranks (mine), the next round's (nxt) and the one after (nn), then the tail.
// The model also counts the events that reach each of these, so that the test can assert that its corpus keeps reaching them.
#include <cstdint>
#include <cstring>

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
    E s_e[2][256];
    E ca, cb;  // the candidates: every thread loads the same two entries

    explicit Model(bool rm, uint64_t* events) : rank_mode(rm), ev(events) {
        for (int t = 0; t < THREADS; t++)
            for (int k = 0; k < S; k++) {
                Q[t][k] = 0;
                X[t][k] = uint32_t(S * t + k);
                s_e[0][S * t + k] = s_e[1][S * t + k] = E{0u, uint32_t(S * t + k)};
            }
    }

    void load_candidates(uint32_t r2, int par) {
        ca = s_e[par][r2];
        cb = r2 ? s_e[par][r2 - 1] : E{0xFFFFFFFFu, 0u};  // above position 0: a q larger than any qc
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
        uint32_t up_q[THREADS], up_x[THREADS];
        for (int t = 0; t < THREADS; t++) {
            const int lane = t & 31, warp = t >> 5;
            // __shfl_up_sync(.., 1): lane 0 gets its own value
            up_q[t] = lane ? Q[t - 1][S - 1] : Q[t][S - 1];
            up_x[t] = lane ? X[t - 1][S - 1] : X[t][S - 1];
            if (lane == 0 && warp > 0) {
                const E e = s_e[par ^ 1][S * t - 1];
                up_q[t] = e.q, up_x[t] = e.x;
            }
        }
        const uint32_t sym = x & 0xFFu;
        const uint32_t qc = rank_mode ? (i + (x >> 8)) >> 1 : i;
        const uint32_t fresh = (i << 8) | sym;
        if (ev) count(r, r2, qc);
        {  // the entry at rank r2 after this step
            const bool mv = r2 <= r && !(ca.q > qc);
            x = mv ? (cb.q > qc ? fresh : cb.x) : ca.x;
        }
        for (int t = 0; t < THREADS; t++) {
            const uint32_t base = uint32_t(S * t);
            const int d = int(r) - int(base);
            uint32_t* q = Q[t];
            uint32_t* xx = X[t];
            bool gk = q[S - 1] > qc;
            for (int k = S - 1; k >= 1; k--) {
                const bool gk1 = q[k - 1] > qc;
                const bool mv = k <= d && !gk;
                const uint32_t xin = gk1 ? fresh : xx[k - 1];
                q[k] = mv ? (q[k - 1] < qc ? q[k - 1] : qc) : q[k];
                xx[k] = mv ? xin : xx[k];
                gk = gk1;
            }
            const bool g_up = t == 0 ? true : up_q[t] > qc;
            const bool mv = 0 <= d && !gk;
            q[0] = mv ? (g_up ? qc : up_q[t]) : q[0];
            xx[0] = mv ? (g_up ? fresh : up_x[t]) : xx[0];
        }
        for (int t = 0; t < THREADS; t++)
            for (int k = 0; k < S; k++) s_e[par][S * t + k] = E{Q[t][k], X[t][k]};
        return sym;
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
    auto rk = [&](uint32_t k) -> uint32_t { return k < n ? src[k] : 0u; };  // ranks past the end load as 0
    uint32_t mine[32], nxt[32], nn[32];
    for (uint32_t l = 0; l < 32; l++) mine[l] = rk(l), nxt[l] = rk(32 + l);
    uint32_t x = m.s_e[1][mine[0]].x;
    m.load_candidates(mine[1], 1);
    uint32_t i0 = 0;
    for (; i0 + 32 <= n; i0 += 32) {
        for (uint32_t l = 0; l < 32; l++) nn[l] = rk(i0 + 64 + l);
        for (uint32_t j = 0; j < 32; j++) {
            const uint32_t r = mine[j];
            const uint32_t r2 = j < 31 ? mine[(j + 1) & 31] : nxt[0];
            const uint32_t r3 = j < 30 ? mine[(j + 2) & 31] : nxt[(j + 2) & 31];
            dst[i0 + j] = uint8_t(m.step(r, r2, i0 + j, int(j & 1), x));
            m.load_candidates(r3, int(j & 1));
        }
        memcpy(mine, nxt, sizeof mine);
        memcpy(nxt, nn, sizeof nxt);
    }
    for (uint32_t j = 0; i0 + j < n; j++) {
        const uint32_t r = mine[j];
        const uint32_t r2 = j < 31 ? mine[(j + 1) & 31] : 0u;
        const uint32_t r3 = j < 30 ? mine[(j + 2) & 31] : 0u;
        dst[i0 + j] = uint8_t(m.step(r, r2, i0 + j, int(j & 1), x));
        m.load_candidates(r3, int(j & 1));
    }
    if (events) events[EV_TAIL0 + n % 32]++;
    return 0;
}
