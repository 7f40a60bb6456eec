// The bookkeeping of the block cache (kz_cache_*, kz_read_ranges_cached[_device] in kz_api.cu): the page allocator, the key, the LRU and
// the split of a cached slice into page-sized copies. Pure host code: no CUDA types, so that tests/host/block_cache_host.cpp checks it
// under g++ (and under the sanitizers) against a brute-force model.
//
// The device memory of a cache is one allocation of npages pages of CACHE_PAGE bytes, made when the cache is created. An entry is one
// decoded block: its length and the list of pages that hold it, page i holding bytes [i * CACHE_PAGE, (i + 1) * CACHE_PAGE). Inserting
// takes free pages and evicts least recently used entries until enough are free; nothing is allocated per entry.
#pragma once
#include <algorithm>
#include <cstdint>
#include <list>
#include <unordered_map>
#include <vector>

namespace kz {

const uint64_t CACHE_PAGE = 64 * 1024;

// What a block record decodes to depends on its payload bits and on these header fields, and on nothing else: the key of an entry.
// `hash` is the record hash of kz_xxh64_core.cuh; TEXT sizes its hash map from block_size; `last` exempts NONE from its multiple-of-16
// rule (decode_walked's last flag).
struct CacheKey {
    uint64_t hash = 0, bits = 0, t48 = 0;
    uint32_t etype = 0, checksum_bits = 0, block_size = 0;
    uint8_t last = 0;
    bool operator==(const CacheKey& o) const {
        return hash == o.hash && bits == o.bits && t48 == o.t48 && etype == o.etype && checksum_bits == o.checksum_bits && block_size == o.block_size &&
               last == o.last;
    }
};
struct CacheKeyHash {
    size_t operator()(const CacheKey& k) const { return (size_t)(k.hash ^ (k.bits * 0x9E3779B97F4A7C15ull) ^ k.last); }
};

struct CacheEntry {
    CacheKey key;
    uint32_t len = 0;             // decoded bytes
    uint64_t serial = 0;          // unique per insert: tells an entry from a later one with the same key
    std::vector<uint32_t> pages;  // max(1, ceil(len / CACHE_PAGE)) pages
};

struct CacheStats {
    uint64_t entries = 0, resident = 0, budget = 0, hits = 0, misses = 0, inserts = 0, evictions = 0, served = 0;
};

inline uint32_t cache_pages(uint32_t len) { return len ? (uint32_t)((len + CACHE_PAGE - 1) / CACHE_PAGE) : 1u; }

class PageCache {
  public:
    // budget bytes, rounded down to whole pages
    explicit PageCache(uint64_t budget) : npages_((uint32_t)std::min<uint64_t>(budget / CACHE_PAGE, UINT32_MAX)) {
        stats_.budget = budget;
        clear();
    }
    uint32_t npages() const { return npages_; }

    // The entry of key, made the most recently used; nullptr when absent. Counts a hit or a miss.
    const CacheEntry* lookup(const CacheKey& key) {
        auto it = map_.find(key);
        if (it == map_.end()) {
            stats_.misses++;
            return nullptr;
        }
        stats_.hits++;
        lru_.splice(lru_.begin(), lru_, it->second);
        return &*it->second;
    }
    // The entry of key if it is resident and is the one inserted as `serial`; no use is recorded.
    const CacheEntry* peek(const CacheKey& key, uint64_t serial) const {
        auto it = map_.find(key);
        return it != map_.end() && it->second->serial == serial ? &*it->second : nullptr;
    }
    // A new most recently used entry of len bytes: its pages are taken from the free list, evicting from the least recently used end
    // until enough are free. nullptr, and nothing evicted, when the block needs more pages than the whole budget; an entry already
    // resident under key is only made the most recently used (and returned). *fresh: whether a new entry was made (its pages then
    // wait for the block's bytes).
    const CacheEntry* insert(const CacheKey& key, uint32_t len, bool* fresh) {
        *fresh = false;
        auto it = map_.find(key);
        if (it != map_.end()) {
            lru_.splice(lru_.begin(), lru_, it->second);
            return &*it->second;
        }
        const uint32_t need = cache_pages(len);
        if (need > npages_) return nullptr;
        while (free_.size() < need) evict_one();
        CacheEntry e;
        e.key = key;
        e.len = len;
        e.serial = ++serial_;
        e.pages.assign(free_.end() - need, free_.end());
        free_.resize(free_.size() - need);
        lru_.push_front(std::move(e));
        map_[key] = lru_.begin();
        stats_.inserts++;
        stats_.entries++;
        stats_.resident += len;
        *fresh = true;
        return &lru_.front();
    }
    void clear() {
        lru_.clear();
        map_.clear();
        free_.resize(npages_);
        for (uint32_t p = 0; p < npages_; p++) free_[p] = npages_ - 1 - p;  // page 0 is taken first
        stats_.entries = stats_.resident = 0;
    }
    void note_served(uint64_t bytes) { stats_.served += bytes; }
    const CacheStats& stats() const { return stats_; }
    // least recently used first (for the tests)
    template <class F>
    void each_lru_first(F&& f) const {
        for (auto it = lru_.rbegin(); it != lru_.rend(); ++it) f(*it);
    }
    size_t free_pages() const { return free_.size(); }

  private:
    void evict_one() {
        CacheEntry& e = lru_.back();
        free_.insert(free_.end(), e.pages.rbegin(), e.pages.rend());
        stats_.entries--;
        stats_.resident -= e.len;
        stats_.evictions++;
        map_.erase(e.key);
        lru_.pop_back();
    }
    uint32_t npages_;
    uint64_t serial_ = 0;
    std::list<CacheEntry> lru_;  // most recently used first
    std::unordered_map<CacheKey, std::list<CacheEntry>::iterator, CacheKeyHash> map_;
    std::vector<uint32_t> free_;  // taken from the back
    CacheStats stats_;
};

// Bytes [in_block, in_block + len) of a cached block as copies that stay inside one page each: f(page, offset in the page, offset from
// in_block, bytes). in_block + len must not pass the entry's length.
template <class F>
void cache_slice_copies(const CacheEntry& e, uint64_t in_block, uint64_t len, F&& f) {
    for (uint64_t done = 0; done < len;) {
        const uint64_t pos = in_block + done, in_page = pos % CACHE_PAGE;
        const uint64_t n = std::min<uint64_t>(len - done, CACHE_PAGE - in_page);
        f(e.pages[(size_t)(pos / CACHE_PAGE)], in_page, done, n);
        done += n;
    }
}

}  // namespace kz
