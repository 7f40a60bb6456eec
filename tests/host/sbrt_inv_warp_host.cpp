// CPU model of a warp-resident formulation of the RANK / MTFT inverse (tests/test_sbrt_inv_warp_host.py): 32 lanes x 8 consecutive ranks of
// 64-bit entries (q << 35 | p << 8 | symbol), the decoded symbol fetched with one shuffle, the new rank from a popc over "entry above rank r
// with a larger q" (valid because the list is always sorted by q), the move-up as a predicated register shift per lane plus one shuffle-up for
// the lane boundaries. sbrt_inverse_warp_kernel (kanzi-go_b200/csrc/kz_sbrt.cu) keeps the same list layout but decides the move-up locally
// per entry instead of counting the new rank, and takes a zero run in one step; this model checks the list rule they share.
// Reference: v2/transform/SBRT.go:177-226 (Inverse), modes :93-111.
#include <cstdint>

namespace {
inline uint64_t pack(int64_t q, int64_t p, uint32_t sym) { return (uint64_t(q) << 35) | (uint64_t(p) << 8) | sym; }  // q, p < 2^27
inline int64_t ent_q(uint64_t e) { return int64_t(e >> 35); }
inline int64_t ent_p(uint64_t e) { return int64_t((e >> 8) & ((1ull << 27) - 1)); }
}  // namespace

extern "C" int64_t sbrt_inverse_warp_model(int mode, const uint8_t* src, int64_t n, uint8_t* dst) {
    const bool rank_mode = mode == 2;  // MTFT: qc = i; RANK: qc = (i + p[c]) >> 1
    uint64_t e[32][8];
    for (int l = 0; l < 32; l++)
        for (int k = 0; k < 8; k++) e[l][k] = pack(0, 0, uint32_t(8 * l + k));
    for (int64_t i = 0; i < n; i++) {
        const int r = src[i];
        // shuffle: lane r >> 3 selects its register r & 7 and broadcasts it
        const uint64_t cur = e[r >> 3][r & 7];
        dst[i] = uint8_t(cur);
        const int64_t qc = rank_mode ? ((i + ent_p(cur)) >> 1) : i;
        // per lane: entries at ranks < r with q > qc; warp sum = new rank
        int nr = 0;
        for (int l = 0; l < 32; l++) {
            int c = 0;
            for (int k = 0; k < 8; k++)
                if (8 * l + k < r && ent_q(e[l][k]) > qc) c++;
            nr += c;
        }
        // per lane, in place: the last register of every lane before the shift (for the shuffle-up), then k = 7 .. 1, then k = 0
        uint64_t last[32];
        for (int l = 0; l < 32; l++) last[l] = e[l][7];
        const uint64_t fresh = pack(qc, i, uint32_t(cur & 0xFF));
        for (int l = 0; l < 32; l++) {
            for (int k = 7; k >= 1; k--) {
                const int rank = 8 * l + k;
                if (rank > nr && rank <= r) e[l][k] = e[l][k - 1];
            }
            const int rank0 = 8 * l;
            if (rank0 > nr && rank0 <= r) e[l][0] = last[l - 1];  // shuffle-up by one lane (lane 0 never takes this branch: rank0 = 0)
            for (int k = 0; k < 8; k++)
                if (8 * l + k == nr) e[l][k] = fresh;
        }
    }
    return n;
}
