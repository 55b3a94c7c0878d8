// Multi-probe zero-collision hash (MPZCH): id -> slot of an open-addressing identity table, one thread per id.
//
// Table layout (modules/hash_mc_modules.py): `buckets` contiguous buckets of `bucket_size` slots; identities[slot] is the raw id owning the
// slot (-1 = free), metadata[slot] the hour it was last seen. An id hashes (splitmix64 finaliser, the same integer arithmetic as the
// PyTorch mirror so CPU- and GPU-built tables are interchangeable) to a bucket and a start slot inside it, and owns at most one of the
// `max_probe` slots after the start.
//
// Per id:  (1) scan the probe window for the id itself - a free slot ends the scan (slots are never freed, only re-owned), remembering
//              the first claimable slot: free, expired (TTL policy) or - LRU policy, no free slot in the window - the least recently seen;
//          (2) hit -> done;  training and a claimable slot -> atomicCAS(expected owner -> id). Losing the race to the SAME id (duplicates
//              inside the batch) is a hit; losing it to another id continues the scan behind that slot;
//          (3) nothing claimable -> collision: the id falls back to its start slot (or -1 when fallback is disabled).
// No host round trip per probe step (the PyTorch mirror synchronises every step); hit / insert / collision / evict counters are
// warp-reduced into 4 device integers; an evicted slot is reported in evicted[i] of the thread that took it.
//
// Replaces fbgemm `zero_collision_hash` (reference torchrec/modules/hash_mc_modules.py:460-520).
#include "common.cuh"

namespace {

__device__ __forceinline__ int64_t zch_mix64(int64_t x) {
  // arithmetic (sign-extending) shifts + wrap-around multiplies: bit-identical to the int64 tensor ops of the PyTorch mirror
  x = x ^ (x >> 30);
  x = (int64_t) ((uint64_t) x * 0xbf58476d1ce4e5b9ULL);
  x = x ^ (x >> 27);
  x = (int64_t) ((uint64_t) x * 0x94d049bb133111ebULL);
  return x ^ (x >> 31);
}

__device__ __forceinline__ int64_t zch_mod(int64_t a, int64_t m) {
  const int64_t r = a % m;
  return r < 0 ? r + m : r;
}

struct ZchParams {
  const int64_t* ids;
  int64_t n;
  unsigned long long* identities;
  int32_t* metadata;
  int64_t buckets, bucket_size;
  int max_probe;
  int readonly;
  int now;
  int ttl;       // hours; < 0 = never expires
  int policy;    // 0 none, 1 single TTL, 2 LRU
  int fallback;  // collision -> start slot (1) or -1 (0)
  int64_t* out;
  int64_t* evicted;
  int* counters;  // hit, insert, collision, evict
};

__global__ void __launch_bounds__(256) zch_probe_kernel(const ZchParams p) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  int hit = 0, ins = 0, col = 0, evi = 0;
  if (i < p.n) {
    const int64_t id = p.ids[i];
    const int64_t h = zch_mix64(id);
    const int64_t base = zch_mod(h, p.buckets) * p.bucket_size;
    const int64_t start = zch_mod(h >> 16, p.bucket_size);
    const int window = (int) min((int64_t) p.max_probe, p.bucket_size);
    int64_t res = -1, ev = -1;
    int from = 0;
    // every failed claim moves `from` past the slot that was lost (its new owner is fresh, so it stays unclaimable), so the loop ends
    // after at most `window` claims; LRU victims restart the scan and are bounded separately
    int lru_retries = 0;
    while (res < 0) {
      int64_t cand = -1;
      unsigned long long cand_owner = 0;
      int64_t lru_slot = -1;
      unsigned long long lru_owner = 0;
      int lru_seen = 0x7fffffff;
      int cand_probe = window;
      for (int q = from; q < window; ++q) {
        int64_t s = start + q;
        if (s >= p.bucket_size) s -= p.bucket_size;
        s += base;
        const unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(p.identities + s);
        if ((int64_t) cur == id) {
          res = s;
          hit = 1;
          break;
        }
        if ((int64_t) cur == -1) {  // free: the id cannot live further down the window
          if (cand < 0) { cand = s; cand_owner = cur; cand_probe = q; }
          break;
        }
        if (p.readonly) continue;
        // the owner's hour is stamped BEFORE its claim (below): read it after the identity, never older than that claim
        __threadfence();
        const int seen = *reinterpret_cast<volatile int*>(p.metadata + s);
        if (p.policy == 1 && p.ttl >= 0 && cand < 0 && seen + p.ttl < p.now) { cand = s; cand_owner = cur; cand_probe = q; }
        if (p.policy == 2 && seen < p.now && seen < lru_seen) { lru_seen = seen; lru_slot = s; lru_owner = cur; }
      }
      if (res >= 0 || p.readonly) break;
      bool lru_pick = false;
      if (cand < 0 && p.policy == 2 && lru_slot >= 0 && lru_retries < 8) { cand = lru_slot; cand_owner = lru_owner; lru_pick = true; ++lru_retries; }
      if (cand < 0) break;
      // stamp the hour first: a slot claimed in this batch must not look expired / least recently seen to the other threads of the
      // batch (they would take it over again). A lost claim leaves `now` on a slot its winner stamps with `now` as well.
      *reinterpret_cast<volatile int*>(p.metadata + cand) = p.now;
      __threadfence();
      const unsigned long long prev = atomicCAS(p.identities + cand, cand_owner, (unsigned long long) id);
      if (prev == cand_owner) {
        res = cand;
        ins = 1;
        if ((int64_t) cand_owner != -1) { ev = cand; evi = 1; }
      } else if ((int64_t) prev == id) {  // a duplicate of this id inside the batch took the slot first
        res = cand;
        hit = 1;
      } else {
        from = lru_pick ? 0 : cand_probe + 1;  // somebody else owns it now
      }
    }
    if (res >= 0) {
      if (!p.readonly) p.metadata[res] = p.now;
    } else {
      col = 1;
      res = p.fallback ? base + start : -1;
    }
    p.out[i] = res;
    if (p.evicted) p.evicted[i] = ev;
  }
  const int h_ = __reduce_add_sync(0xffffffffu, hit), i_ = __reduce_add_sync(0xffffffffu, ins);
  const int c_ = __reduce_add_sync(0xffffffffu, col), e_ = __reduce_add_sync(0xffffffffu, evi);
  if ((threadIdx.x & 31) == 0 && p.counters) {
    if (h_) atomicAdd(p.counters + 0, h_);
    if (i_) atomicAdd(p.counters + 1, i_);
    if (c_) atomicAdd(p.counters + 2, c_);
    if (e_) atomicAdd(p.counters + 3, e_);
  }
}

}  // namespace

TRB_API int trb_zch_probe(const int64_t* ids, int64_t n, int64_t* identities, int32_t* metadata, int64_t buckets, int64_t bucket_size, int max_probe, int readonly,
                          int now, int ttl, int policy, int fallback, int64_t* out, int64_t* evicted, int* counters, cudaStream_t stream) {
  if (n == 0) return 0;
  if (buckets < 1 || bucket_size < 1 || max_probe < 1) return -1;
  ZchParams p{ids, n, reinterpret_cast<unsigned long long*>(identities), metadata, buckets, bucket_size, max_probe, readonly, now, ttl, policy, fallback, out, evicted, counters};
  zch_probe_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(p);
  TRB_CHECK_LAUNCH();
  return 0;
}
