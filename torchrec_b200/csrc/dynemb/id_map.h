// Dynamic-embedding id transformer: global id -> cache slot with LFU/LRU eviction metadata.
//
// GPU-first host design (the table lives in HBM; the host only has to keep up with the KJT rate):
//  * flat open-addressing hash map (linear probing, tombstone-free backward-shift delete), 24 B / entry, one cache
//    line per probe on average — instead of the node-based std::unordered_map of the reference
//    (torchrec/csrc/dynamic_embedding/details/naive_id_transformer_impl.h);
//  * the map is split into P independent partitions (hash-routed, each owning a contiguous slot range and its own
//    free bitmap), so one transform() call fans out over P worker threads without locks on the hot path;
//  * eviction picks the globally smallest records with a bounded max-heap per partition, then merges.
// Parity: IDTransformer / NaiveIDTransformer / MixedLFULRUStrategy / Bitmap of the reference's `tde` ops.
#pragma once
#include <atomic>
#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <queue>
#include <random>
#include <vector>

namespace trb {

enum class Strategy : int { MIXED_LFU_LRU = 0, LRU = 1, LFU = 2, DISTANCE_LFU = 3 };

inline uint64_t mix64(uint64_t x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27; x *= 0x94d049bb133111ebULL;
  return x ^ (x >> 31);
}

// Free-slot bitmap with a rotating cursor (set bit = free).
class Bitmap {
 public:
  explicit Bitmap(int64_t n) : n_(n), words_((n + 63) / 64, ~0ULL), cursor_(0), free_(n) {
    if (n % 64) words_.back() = (1ULL << (n % 64)) - 1;
  }
  int64_t next_free() {
    if (free_ == 0) return -1;
    const size_t nw = words_.size();
    for (size_t k = 0; k < nw; ++k) {
      const size_t w = (cursor_ + k) % nw;
      if (words_[w]) {
        const int b = __builtin_ctzll(words_[w]);
        words_[w] &= words_[w] - 1;
        cursor_ = w;
        --free_;
        return (int64_t) w * 64 + b;
      }
    }
    return -1;
  }
  void release(int64_t i) { words_[i >> 6] |= 1ULL << (i & 63); ++free_; }
  bool full() const { return free_ == 0; }
  int64_t free_count() const { return free_; }

 private:
  int64_t n_;
  std::vector<uint64_t> words_;
  size_t cursor_;
  int64_t free_;
};

struct Entry {
  int64_t gid;
  int64_t slot;   // -1 = empty
  uint32_t lxu;   // eviction record (smaller = evicted earlier)
  uint32_t aux;   // LFU count / first-seen time (DISTANCE_LFU)
};

struct EvictItem {
  uint32_t key;
  int64_t gid;
  int64_t slot;
  bool operator<(const EvictItem& o) const { return key < o.key; }
};

class Partition {
 public:
  Partition(int64_t slot_base, int64_t n_slots) : slot_base_(slot_base), bitmap_(n_slots), size_(0) {
    cap_ = 16;
    while (cap_ < (uint64_t) n_slots * 2) cap_ <<= 1;
    table_.assign(cap_, Entry{0, -1, 0, 0});
  }
  Entry* find(int64_t gid) {
    uint64_t i = mix64((uint64_t) gid) >> 8 & (cap_ - 1);
    while (table_[i].slot >= 0) {
      if (table_[i].gid == gid) return &table_[i];
      i = (i + 1) & (cap_ - 1);
    }
    return nullptr;
  }
  // returns nullptr when no slot is free
  Entry* insert(int64_t gid) {
    const int64_t s = bitmap_.next_free();
    if (s < 0) return nullptr;
    uint64_t i = mix64((uint64_t) gid) >> 8 & (cap_ - 1);
    while (table_[i].slot >= 0) i = (i + 1) & (cap_ - 1);
    table_[i] = Entry{gid, slot_base_ + s, 0, 0};
    ++size_;
    return &table_[i];
  }
  void erase(int64_t gid) {
    uint64_t i = mix64((uint64_t) gid) >> 8 & (cap_ - 1);
    while (table_[i].slot >= 0 && table_[i].gid != gid) i = (i + 1) & (cap_ - 1);
    if (table_[i].slot < 0) return;
    bitmap_.release(table_[i].slot - slot_base_);
    --size_;
    // backward-shift deletion keeps probe sequences intact without tombstones
    uint64_t j = i;
    for (;;) {
      j = (j + 1) & (cap_ - 1);
      if (table_[j].slot < 0) break;
      const uint64_t home = mix64((uint64_t) table_[j].gid) >> 8 & (cap_ - 1);
      const bool between = (i <= j) ? (i < home && home <= j) : (i < home || home <= j);
      if (!between) { table_[i] = table_[j]; i = j; }
    }
    table_[i].slot = -1;
  }
  template <typename F>
  void for_each(F&& f) const {
    for (const Entry& e : table_) if (e.slot >= 0) f(e);
  }
  int64_t size() const { return size_; }
  bool full() const { return bitmap_.full(); }

 private:
  int64_t slot_base_;
  Bitmap bitmap_;
  uint64_t cap_;
  std::vector<Entry> table_;
  int64_t size_;
};

class IdTransformer {
 public:
  IdTransformer(int64_t num_embedding, Strategy strategy, int min_used_freq_power, int partitions);
  // Transform ids[0..n): writes cache slots. Ids that do not fit (cache full) get slot -1 and are counted in the
  // return value's complement: returns the number of ids resolved. New (gid, slot) pairs are appended to fetch_.
  int64_t transform(const int64_t* gids, int64_t n, int64_t* slots, int64_t time, int threads);
  // Evict up to `num` least valuable ids; writes (gid, slot) pairs.
  int64_t evict(int64_t num, int64_t* out_pairs);
  int64_t size() const;
  int64_t capacity() const { return num_embedding_; }
  int64_t take_fetch(int64_t* out_pairs, int64_t max_pairs);
  int64_t pending_fetch() const { return (int64_t) fetch_.size() / 2; }
  // dump all (gid, slot, record) triples
  int64_t save(int64_t* out_triples, int64_t max_entries) const;

 private:
  uint32_t update_record(Entry* e, bool fresh, uint32_t time, std::mt19937_64& rng) const;
  int64_t num_embedding_;
  Strategy strategy_;
  int min_power_;
  std::vector<std::unique_ptr<Partition>> parts_;
  std::vector<int64_t> fetch_;
  uint32_t now_ = 0;
  std::mutex mu_;
};

}  // namespace trb
