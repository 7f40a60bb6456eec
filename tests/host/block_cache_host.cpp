// CPU harness of the block cache bookkeeping (kanzi-go_b200/csrc/kz_block_cache.h) and the record hash (kz_xxh64_core.cuh), for
// tests/test_block_cache_host.py. Built as a shared library for the hash checks, and as a program under ASan / UBSan that holds the
// cache against a brute-force model (`block_cache_host <rounds>`).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_block_cache.h"
#include "../../kanzi-go_b200/csrc/kz_xxh64_core.cuh"

extern "C" {
// the record hash of bits [start, start + bits) of s (n bytes)
uint64_t record_hash(const uint8_t* s, uint64_t start, uint64_t bits) { return kz::record_hash_host(s, start, bits); }
uint64_t xxh64(const uint8_t* p, uint64_t n, uint64_t seed) { return kz::xxh64_bytes(p, n, seed); }
}

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd() {
    rng_state ^= rng_state << 13;
    rng_state ^= rng_state >> 7;
    rng_state ^= rng_state << 17;
    return rng_state;
}

#define CHECK(c)                                                         \
    do {                                                                 \
        if (!(c)) {                                                      \
            printf("check failed at line %d: %s\n", __LINE__, #c);       \
            exit(1);                                                     \
        }                                                                \
    } while (0)

// The model: entries most recently used first, each (key id, length).
struct Model {
    uint32_t npages;
    std::vector<std::pair<uint32_t, uint32_t>> lru;
    uint64_t hits = 0, misses = 0, inserts = 0, evictions = 0;
    int find(uint32_t id) const {
        for (size_t i = 0; i < lru.size(); i++)
            if (lru[i].first == id) return (int)i;
        return -1;
    }
    uint32_t used() const {
        uint32_t u = 0;
        for (auto& e : lru) u += kz::cache_pages(e.second);
        return u;
    }
    bool lookup(uint32_t id) {
        const int i = find(id);
        if (i < 0) return misses++, false;
        hits++;
        auto e = lru[i];
        lru.erase(lru.begin() + i);
        lru.insert(lru.begin(), e);
        return true;
    }
    // -1: refused, 0: already there, 1: made
    int insert(uint32_t id, uint32_t len) {
        const int i = find(id);
        if (i >= 0) {
            auto e = lru[i];
            lru.erase(lru.begin() + i);
            lru.insert(lru.begin(), e);
            return 0;
        }
        if (kz::cache_pages(len) > npages) return -1;
        while (used() + kz::cache_pages(len) > npages) lru.pop_back(), evictions++;
        lru.insert(lru.begin(), {id, len});
        inserts++;
        return 1;
    }
};

static kz::CacheKey key_of(uint32_t id) {
    kz::CacheKey k;
    k.hash = 0x1234567ull * (id / 2);  // pairs of ids share the hash and differ in another field of the key
    k.bits = 1000 + id / 2;
    k.last = id & 1;
    k.block_size = 65536;
    return k;
}

static void check_same(const kz::PageCache& c, const Model& m) {
    std::vector<std::pair<kz::CacheKey, uint32_t>> got;
    std::set<uint32_t> owned;
    uint64_t resident = 0;
    size_t npages_owned = 0;
    c.each_lru_first([&](const kz::CacheEntry& e) {
        got.push_back({e.key, e.len});
        CHECK(e.pages.size() == kz::cache_pages(e.len));
        for (uint32_t p : e.pages) {
            CHECK(p < c.npages());
            CHECK(owned.insert(p).second);  // no page owned twice
        }
        npages_owned += e.pages.size();
        resident += e.len;
    });
    CHECK(got.size() == m.lru.size());
    for (size_t i = 0; i < got.size(); i++) {  // got: least recently used first
        const auto& w = m.lru[m.lru.size() - 1 - i];
        CHECK(got[i].first == key_of(w.first) && got[i].second == w.second);
    }
    CHECK(npages_owned + c.free_pages() == c.npages());
    CHECK((uint64_t)npages_owned * kz::CACHE_PAGE <= c.stats().budget);
    const kz::CacheStats& st = c.stats();
    CHECK(st.entries == m.lru.size() && st.resident == resident && st.hits == m.hits && st.misses == m.misses && st.inserts == m.inserts &&
          st.evictions == m.evictions);
}

static void cache_fuzz(int rounds) {
    for (int r = 0; r < rounds; r++) {
        const uint64_t budget = r % 7 == 0 ? rnd() % kz::CACHE_PAGE : (rnd() % 12) * kz::CACHE_PAGE + rnd() % 3 * 1000;
        kz::PageCache c(budget);
        Model m{(uint32_t)(budget / kz::CACHE_PAGE)};
        CHECK(c.npages() == m.npages);
        const uint32_t nkeys = 2 + (uint32_t)(rnd() % 20);
        std::vector<uint32_t> len_of(nkeys);
        for (uint32_t& l : len_of) {
            const uint64_t kind = rnd() % 4;
            l = kind == 0 ? 0 : kind == 1 ? (uint32_t)(rnd() % kz::CACHE_PAGE) + 1 : (uint32_t)(rnd() % (5 * kz::CACHE_PAGE)) + 1;
        }
        for (int op = 0; op < 300; op++) {
            const uint32_t id = (uint32_t)(rnd() % nkeys);
            if (rnd() % 3) {
                const kz::CacheEntry* e = c.lookup(key_of(id));
                CHECK((e != nullptr) == m.lookup(id));
                if (e) {
                    // a slice of the entry as page-bounded copies: they tile it exactly
                    const uint64_t lo = e->len ? rnd() % e->len : 0, n = e->len ? rnd() % (e->len - lo + 1) : 0;
                    uint64_t next = 0;
                    kz::cache_slice_copies(*e, lo, n, [&](uint32_t page, uint64_t in_page, uint64_t at, uint64_t k) {
                        CHECK(at == next && k >= 1 && in_page + k <= kz::CACHE_PAGE);
                        CHECK(page == e->pages[(lo + at) / kz::CACHE_PAGE] && in_page == (lo + at) % kz::CACHE_PAGE);
                        next += k;
                    });
                    CHECK(next == n);
                }
            } else {
                bool fresh = false;
                const kz::CacheEntry* e = c.insert(key_of(id), len_of[id], &fresh);
                const int w = m.insert(id, len_of[id]);
                CHECK((e == nullptr) == (w < 0) && fresh == (w == 1));
                if (e) CHECK(c.peek(key_of(id), e->serial) == e);
            }
            check_same(c, m);
            if (op == 200 && r % 5 == 0) {
                c.clear();
                m.lru.clear();
                check_same(c, m);
            }
        }
    }
}

// The record at every bit offset 0..7 hashes alike, from a buffer that ends at the record's last byte (ASan sees any read past it).
static void hash_offsets(int rounds) {
    for (int r = 0; r < rounds; r++) {
        static const uint64_t SIZES[] = {1, 7, 8, 9, 63, 64, 65, 8 * 4096 - 1, 8 * 4096, 8 * 4096 + 1, 8 * 3 * 4096 + 13};
        const uint64_t bits = r < 11 ? SIZES[r] : 1 + rnd() % (8 * 3 * 4096);
        std::vector<uint8_t> rec((size_t)((bits + 7) / 8));
        for (uint8_t& b : rec) b = (uint8_t)rnd();
        uint64_t want = 0;
        for (uint32_t sh = 0; sh < 8; sh++) {
            const uint64_t lead = 8 * (rnd() % 3) + sh, nbytes = (lead + bits + 7) / 8;
            uint8_t* s = (uint8_t*)malloc(nbytes);
            for (uint64_t i = 0; i < nbytes; i++) s[i] = (uint8_t)rnd();  // bits around the record are noise
            for (uint64_t i = 0; i < bits; i++) {
                const uint64_t p = lead + i;
                const int bit = (rec[i / 8] >> (7 - i % 8)) & 1;
                s[p / 8] = (uint8_t)((s[p / 8] & ~(0x80 >> (p % 8))) | (bit << (7 - p % 8)));
            }
            const uint64_t h = kz::record_hash_host(s, lead, bits);
            if (sh == 0) want = h;
            CHECK(h == want);
            free(s);
        }
    }
}

int main(int argc, char** argv) {
    const int rounds = argc > 1 ? atoi(argv[1]) : 100;
    cache_fuzz(rounds);
    hash_offsets(11 + rounds / 10);
    printf("cache fuzz done\n");
    return 0;
}
