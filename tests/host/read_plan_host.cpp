// CPU harness of the batched read plan and the index blob (kanzi-go_b200/csrc/kz_read_plan.h), for tests/test_read_plan_host.py. Built as a
// shared library for the plan checks, and as a program under ASan / UBSan for the blob fuzz (`read_plan_host <rounds>`).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_read_plan.h"

extern "C" {
static kz::ReadPlan PLAN;

// Plans the requests; the plan stays for the getters below. Returns the number of passes.
uint32_t plan_reads(uint64_t nblocks, uint32_t block_size, int64_t size, uint32_t nreq, const uint64_t* off, const uint64_t* len, uint64_t budget) {
    PLAN = kz::plan_reads(nblocks, block_size, size, nreq, off, len, budget);
    return PLAN.npasses();
}
uint64_t plan_nblocks() { return PLAN.blocks.size(); }
uint64_t plan_nslices() { return PLAN.slices.size(); }
// blocks (plan_nblocks), first (passes + 1), slice_of (plan_nblocks + 1), want (nreq), and the slices as 6 columns of u64
void plan_get(uint64_t* blocks, uint32_t* first, uint64_t* slice_of, uint64_t* want, uint64_t* slices) {
    for (size_t k = 0; k < PLAN.blocks.size(); k++) blocks[k] = PLAN.blocks[k];
    for (size_t p = 0; p < PLAN.first.size(); p++) first[p] = PLAN.first[p];
    for (size_t k = 0; k < PLAN.slice_of.size(); k++) slice_of[k] = PLAN.slice_of[k];
    for (size_t i = 0; i < PLAN.want.size(); i++) want[i] = PLAN.want[i];
    for (size_t s = 0; s < PLAN.slices.size(); s++) {
        const kz::ReadSlice& sl = PLAN.slices[s];
        const uint64_t row[6] = {sl.req, sl.block, sl.in_block, sl.len, sl.at, 0};
        for (int c = 0; c < 6; c++) slices[6 * s + c] = row[c];
    }
}
uint64_t read_cost(uint32_t block_size) { return kz::read_block_cost(block_size); }

// save(load(blob)) into out (cap bytes): the bytes written, 0 when load rejects the blob
uint64_t blob_roundtrip(const uint8_t* blob, uint64_t n, uint8_t* out, uint64_t cap) {
    kz::StreamIndex x;
    if (!kz::index_load(blob, (size_t)n, x)) return 0;
    const size_t need = kz::index_blob_bytes(x.nblocks());
    if (need <= cap) kz::index_save(x, out);
    return need;
}
uint64_t xxh64(const uint8_t* p, uint64_t n) { return kz::index_xxh64(p, (size_t)n); }
}

// Blob fuzz: valid blobs of random indexes, mutated (bytes, lengths, with and without a repaired hash). load must reject the blob or give
// an index that is consistent and saves to a blob of the same length; it must never read outside the n bytes it was given (each blob
// lives in a heap block of exactly n bytes, so the sanitizer sees any overrun).
static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd() {
    rng_state ^= rng_state << 13;
    rng_state ^= rng_state >> 7;
    rng_state ^= rng_state << 17;
    return rng_state;
}

int main(int argc, char** argv) {
    const int rounds = argc > 1 ? atoi(argv[1]) : 200;
    uint64_t accepted = 0, rejected = 0;
    for (int r = 0; r < rounds; r++) {
        kz::StreamIndex x;
        x.t48 = rnd() & ((1ull << 48) - 1);
        x.etype = rnd() % 10;
        x.block_size = 1024 + (uint32_t)(rnd() % 100000);
        x.checksum_bits = 32 * (uint32_t)(rnd() % 3);
        static const uint32_t HEADER_BITS[5] = {0, 160, 176, 192, 208};
        x.header_bits = HEADER_BITS[rnd() % 5];
        x.input_size = (int64_t)(rnd() % 100000);
        const uint32_t nb = (uint32_t)(rnd() % 40);
        uint64_t pos = x.header_bits;
        for (uint32_t b = 0; b < nb; b++) {
            x.start.push_back(pos + 8 + rnd() % 32);
            x.bits.push_back(1 + rnd() % 5000);
            pos = x.start.back() + x.bits.back();
        }
        x.stream_bytes = (pos + 8 + 7) / 8 + rnd() % 3;
        x.size = nb == 0 ? 0 : (rnd() & 1) ? -1 : (int64_t)((nb - 1) * (uint64_t)x.block_size + 1 + rnd() % x.block_size);
        for (size_t i = 0; i < kz::INDEX_HEAD; i++) x.head[i] = (uint8_t)rnd();
        if (!kz::index_consistent(x)) {
            printf("generated index not consistent\n");
            return 1;
        }
        std::vector<uint8_t> good(kz::index_blob_bytes(nb));
        kz::index_save(x, good.data());
        for (int m = 0; m < 64; m++) {
            size_t n = good.size();
            if (m % 8 == 1) n = rnd() % (good.size() + 1);                    // truncated
            if (m % 8 == 2) n = good.size() + 1 + rnd() % 40;                 // extended
            uint8_t* blob = (uint8_t*)malloc(n ? n : 1);
            for (size_t i = 0; i < n; i++) blob[i] = i < good.size() ? good[i] : (uint8_t)rnd();
            const int flips = m == 0 ? 0 : 1 + (int)(rnd() % 4);
            for (int f = 0; f < flips && n; f++) {
                const size_t at = (m % 4 == 3) ? rnd() % std::min<size_t>(n, kz::INDEX_FIXED) : rnd() % n;  // aim at the fixed fields
                blob[at] = (m % 2) ? (uint8_t)rnd() : (uint8_t)(blob[at] ^ (1u << (rnd() % 8)));
            }
            if (m % 3 == 0 && n >= 8) kz::index_put(blob + n - 8, kz::index_xxh64(blob, n - 8), 8);  // a damaged blob with a good hash
            kz::StreamIndex y;
            if (kz::index_load(blob, n, y)) {
                accepted++;
                if (!kz::index_consistent(y) || kz::index_blob_bytes(y.nblocks()) != n) {
                    printf("load accepted an inconsistent blob\n");
                    return 1;
                }
                std::vector<uint8_t> again(n);
                kz::index_save(y, again.data());
                if (memcmp(again.data(), blob, n)) {
                    printf("save(load(blob)) differs from the blob\n");
                    return 1;
                }
            } else {
                rejected++;
                if (m == 0) {
                    printf("load rejected a valid blob\n");
                    return 1;
                }
            }
            free(blob);
        }
    }
    printf("fuzz done: %llu accepted, %llu rejected\n", (unsigned long long)accepted, (unsigned long long)rejected);
    return 0;
}
