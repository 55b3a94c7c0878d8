// Training HBM row cache of fused_uvm_caching tables (ops/uvm.py: UvmCachedEmbeddingBags.prefetch), managed on the device.
//
// One prefetch makes every id of a batch resident in the cache of its table, for all tables at once, with a fixed sequence of
// launches and no host read:
//   memset  per-table distinct / miss counters
//   keys    (table, id) -> global row key (row_base[t] + id); ids outside the table and positions outside the batch get the sentinel
//   sort    cub::DeviceRadixSort::SortKeys over the keys (bits of the total row count only)
//   count   first key of each run: distinct rows per table (overflow check)
//   probe   first key of each run, tables that fit: hit -> score update (LRU tick / LFU +1) and stamp; miss -> flagged
//   select  cub::DeviceSelect::Flagged: the missing rows, ascending, grouped by table
//   victims one CTA per table: exact radix select of the n_miss lowest (score, slot) among the slots no protected batch uses
//   evict   live victims: weights + optimizer state back to host memory, slot_of_row cleared
//   fill    missing rows + state into the victim slots, maps / scores / stamps set
// With move_rows = 0 (host tables the GPU cannot address, e.g. an SSD-backed store) the kernels update only the maps and leave the
// victim / old-row / missing-row lists in the workspace for the caller's own row movement.
// Policy: victims are the lowest scores among unprotected slots, ties to the lower slot index; the k-th missing row (ascending id)
// takes the k-th victim (ascending slot). A table whose batch needs more distinct rows than it has slots (or, with a batch still in
// flight on another stream, more than the slots left unprotected) moves nothing and sets overflow[t] in mapped host memory.
#include "common.cuh"

#include <algorithm>

#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

// Mirrors ops/uvm.py `_PrefetchArgs` (pointers and int64 only: no padding).
struct UvmPrefetchArgs {
  const void* indices;
  const void* offsets;
  const int32_t* table_of_feature;  // [F]
  const int64_t* row_base;          // [T+1] first global row of table t (also the base of its slot_of_row entries)
  const int64_t* slot_base;         // [T+1] first global cache slot of table t
  const int64_t* host_elem_base;    // [T] first element of table t in the host weights / element-wise state
  const int64_t* cache_elem_base;   // [T] same in the cache
  const int64_t* dim;               // [T]
  int32_t* slot_of_row;             // [total rows]   local slot or -1
  int64_t* row_of_slot;             // [total slots]  local row or -1
  int64_t* score;                   // [total slots]
  int64_t* stamp;                   // [total slots]  tick of the last batch that used the slot
  uint8_t* host_w;
  uint8_t* cache_w;
  float* host_s1;
  float* cache_s1;
  float* host_s2;
  float* cache_s2;
  unsigned long long* stats;        // [T][3] hits, misses, evictions (cumulative)
  int32_t* overflow;                // [T] mapped host memory: distinct rows of a batch larger than the cache, -1 = too few unprotected slots
  void* workspace;
  int64_t workspace_bytes;
  int64_t n;                        // number of positions of `indices`
  int64_t total_rows;               // row_base[T]: the sort key of dropped positions
  int64_t idx64, off64;
  int64_t B, F, T;
  int64_t w_bytes;                  // element size of the weights
  int64_t s1_kind, s2_kind;         // 0 none, 1 one float per row, 2 one float per element
  int64_t tick;                     // this batch (>= 1, < 2^32)
  int64_t protect_from;             // slots with stamp >= protect_from are not victims
  int64_t lfu;
  int64_t move_rows;                // 1: the kernels move the rows zero-copy; 0: only the maps change, the caller moves the rows
};

namespace {

constexpr int kSelThreads = 1024;
constexpr int kDigitBits = 11;
constexpr int kBins = 1 << kDigitBits;

struct Ws {
  unsigned long long* keys_in;
  unsigned long long* keys;
  unsigned long long* miss;
  int64_t* victim;
  int64_t* old;        // row the victim held before (table-local, -1 = empty slot)
  uint8_t* flag;
  int32_t* distinct;   // [T]
  int32_t* n_miss;     // [T]
  int32_t* take;       // [T] 1 = the table's misses move
  int64_t* miss_base;  // [T+1]
  int32_t* n_sel;      // [1]
  void* tmp;
  size_t tmp_bytes;
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t) 255; }

int end_bit_of(int64_t sentinel) {
  int b = 1;
  while (b < 64 && (sentinel >> b) != 0) ++b;
  return b;
}

size_t cub_tmp_bytes(int64_t n, int end_bit) {
  // (the key count is < 2^31: checked by the entry point)
  size_t a = 0, b = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, a, (const unsigned long long*) nullptr, (unsigned long long*) nullptr, (int) n, 0, end_bit);
  cub::DeviceSelect::Flagged(nullptr, b, (const unsigned long long*) nullptr, (const uint8_t*) nullptr, (unsigned long long*) nullptr, (int32_t*) nullptr,
                             (int) n);
  return a > b ? a : b;
}

// Layout of the workspace; with base == nullptr only the size is computed.
size_t carve(uint8_t* base, int64_t n, int64_t T, int end_bit, Ws* w) {
  const int64_t m = n > 0 ? n : 1;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? base + o : nullptr;
    o += align256(bytes);
    return p;
  };
  w->keys_in = (unsigned long long*) take(m * 8);
  w->keys = (unsigned long long*) take(m * 8);
  w->miss = (unsigned long long*) take(m * 8);
  w->victim = (int64_t*) take(m * 8);
  w->old = (int64_t*) take(m * 8);
  w->flag = take(m);
  w->distinct = (int32_t*) take(T * 4);
  w->n_miss = (int32_t*) take(T * 4);
  w->take = (int32_t*) take(T * 4);
  w->miss_base = (int64_t*) take((T + 1) * 8);
  w->n_sel = (int32_t*) take(4);
  w->tmp_bytes = cub_tmp_bytes(m, end_bit);
  w->tmp = take(w->tmp_bytes);
  return o;
}

// last i in [0, cnt) with a[i] <= v (a ascending, a[0] <= v)
__device__ __forceinline__ int upper_index(const int64_t* a, int cnt, int64_t v) {
  int lo = 0, hi = cnt - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a[mid] <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ int64_t off_at(const UvmPrefetchArgs& a, int64_t i) { return trb_ld_idx(a.offsets, i, (int) a.off64); }

__global__ void __launch_bounds__(256) uvm_keys_kernel(UvmPrefetchArgs a, int64_t m, unsigned long long* keys, unsigned long long sentinel) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  unsigned long long k = sentinel;
  if (i < a.n && i >= off_at(a, 0) && i < off_at(a, a.F * a.B)) {
    int lo = 0, hi = (int) a.F - 1;  // feature owning position i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (off_at(a, (int64_t) mid * a.B) <= i) lo = mid; else hi = mid - 1;
    }
    const int t = a.table_of_feature[lo];
    const int64_t id = trb_ld_idx(a.indices, i, (int) a.idx64);
    const int64_t r0 = a.row_base[t];
    if (id >= 0 && id < a.row_base[t + 1] - r0) k = (unsigned long long) (r0 + id);
  }
  keys[i] = k;
}

__device__ __forceinline__ bool run_head(const unsigned long long* keys, int64_t j, unsigned long long sentinel) {
  const unsigned long long k = keys[j];
  return k != sentinel && (j == 0 || keys[j - 1] != k);
}

// warp-aggregated counter add: lanes with the same table add once
__device__ __forceinline__ void warp_add(int32_t* ctr, int t, bool active) {
  const unsigned mask = __ballot_sync(0xffffffffu, active);
  if (!active) return;
  const unsigned peers = __match_any_sync(mask, t);
  if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(ctr + t, __popc(peers));
}

__global__ void __launch_bounds__(256) uvm_count_kernel(UvmPrefetchArgs a, int64_t m, const unsigned long long* keys, unsigned long long sentinel, int32_t* distinct) {
  const int64_t j = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  const bool head = j < m && run_head(keys, j, sentinel);
  const int t = head ? upper_index(a.row_base, (int) a.T, (int64_t) keys[j]) : 0;
  warp_add(distinct, t, head);
}

__global__ void __launch_bounds__(256) uvm_probe_kernel(UvmPrefetchArgs a, int64_t m, const unsigned long long* keys, unsigned long long sentinel,
                                                        const int32_t* distinct, int32_t* n_miss, uint8_t* flag) {
  const int64_t j = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  bool hit = false, miss = false;
  int t = 0;
  if (j < m) {
    uint8_t f = 0;
    if (run_head(keys, j, sentinel)) {
      const int64_t k = (int64_t) keys[j];
      t = upper_index(a.row_base, (int) a.T, k);
      const int64_t sb = a.slot_base[t];
      if (distinct[t] > a.slot_base[t + 1] - sb) {
        a.overflow[t] = distinct[t];  // the distinct rows the batch needs: the host names them in the error
      } else {
        const int32_t s = a.slot_of_row[k];
        if (s >= 0) {
          const int64_t g = sb + s;
          a.score[g] = a.lfu ? a.score[g] + 1 : a.tick;  // one distinct id per slot: no race
          a.stamp[g] = a.tick;
          hit = true;
        } else {
          f = 1;
          miss = true;
        }
      }
    }
    flag[j] = f;
  }
  {
    const unsigned mask = __ballot_sync(0xffffffffu, hit);
    if (hit) {
      const unsigned peers = __match_any_sync(mask, t);
      if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(a.stats + 3 * t, (unsigned long long) __popc(peers));
    }
  }
  {
    const unsigned mask = __ballot_sync(0xffffffffu, miss);
    if (miss) {
      const unsigned peers = __match_any_sync(mask, t);
      if ((threadIdx.x & 31) == __ffs(peers) - 1) {
        atomicAdd(a.stats + 3 * t + 1, (unsigned long long) __popc(peers));
        atomicAdd(n_miss + t, __popc(peers));
      }
    }
  }
}

// One CTA per table: victims = the n_miss lowest (score, slot) among slots with stamp < protect_from, written in slot order to
// victim[miss_base[t] ...]. Scores are < 2^32 (ticks / counts bounded by the tick), so at most three 11-bit digit passes; a
// digit pass narrows `prefix` to the bucket that holds the n-th lowest, the last pass then takes every candidate below the
// prefix and the first `need` candidates equal to it in slot order.
__global__ void __launch_bounds__(kSelThreads) uvm_victim_kernel(UvmPrefetchArgs a, Ws w) {
  typedef cub::BlockScan<int, kSelThreads> Scan;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int hist[kBins];
  __shared__ int s_digit, s_below, s_total;
  const int t = blockIdx.x;
  const int tid = threadIdx.x;
  int64_t base = 0;
  for (int u = 0; u < t; ++u) base += w.n_miss[u];
  if (tid == 0) {
    w.miss_base[t] = base;
    if (t == a.T - 1) w.miss_base[a.T] = base + w.n_miss[t];
  }
  const int n = w.n_miss[t];
  if (n == 0) {
    if (tid == 0) w.take[t] = 0;
    return;
  }
  const int64_t sb = a.slot_base[t], C = a.slot_base[t + 1] - sb;
  const int64_t* score = a.score + sb;
  const int64_t* stamp = a.stamp + sb;
  int hi_bits = 0;
  while (hi_bits < 33 && (a.tick >> hi_bits) != 0) ++hi_bits;
  const int passes = (hi_bits + kDigitBits - 1) / kDigitBits;
  int64_t prefix = 0;
  int need = n;
  for (int p = 0; p < passes; ++p) {
    const int shift = (passes - 1 - p) * kDigitBits;
    for (int b = tid; b < kBins; b += kSelThreads) hist[b] = 0;
    __syncthreads();
    for (int64_t s = tid; s < C; s += kSelThreads) {
      if (stamp[s] >= a.protect_from) continue;
      const int64_t sc = score[s];
      if ((sc >> (shift + kDigitBits)) == prefix) atomicAdd(&hist[(sc >> shift) & (kBins - 1)], 1);
    }
    __syncthreads();
    int v[2] = {hist[2 * tid], hist[2 * tid + 1]}, ex[2], total;
    Scan(scan_tmp).ExclusiveSum(v, ex, total);
    for (int q = 0; q < 2; ++q)
      if (ex[q] < need && need <= ex[q] + v[q]) {
        s_digit = 2 * tid + q;
        s_below = ex[q];
      }
    if (tid == 0) s_total = total;
    __syncthreads();
    if (p == 0 && s_total < n) {  // a batch still in flight holds too many slots
      if (tid == 0) {
        a.overflow[t] = -1;
        w.take[t] = 0;
      }
      return;
    }
    need -= s_below;
    prefix = (prefix << kDigitBits) | s_digit;
    __syncthreads();
  }
  // in-order compaction over the slots
  int64_t* out = w.victim + base;
  int taken = 0, eq_seen = 0;
  for (int64_t s0 = 0; s0 < C && taken < n; s0 += kSelThreads) {
    const int64_t s = s0 + tid;
    int less = 0, eq = 0;
    if (s < C && stamp[s] < a.protect_from) {
      const int64_t sc = score[s];
      less = sc < prefix;
      eq = sc == prefix;
    }
    int eq_rank, eq_cnt;
    Scan(scan_tmp).ExclusiveSum(eq, eq_rank, eq_cnt);
    __syncthreads();
    const int pick = less || (eq && eq_seen + eq_rank < need);
    int pos, cnt;
    Scan(scan_tmp).ExclusiveSum(pick, pos, cnt);
    __syncthreads();
    if (pick) out[taken + pos] = sb + s;
    taken += cnt;
    eq_seen += eq_cnt;
  }
  if (tid == 0) w.take[t] = 1;
}

__device__ __forceinline__ void copy_row(uint8_t* dst, const uint8_t* src, int64_t bytes, int lane) {
  if (((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src) | (uintptr_t) bytes) & 15) == 0) {
    for (int64_t v = lane; v < bytes / 16; v += 32) reinterpret_cast<uint4*>(dst)[v] = reinterpret_cast<const uint4*>(src)[v];
  } else {
    for (int64_t v = lane; v < bytes / 4; v += 32) reinterpret_cast<uint32_t*>(dst)[v] = reinterpret_cast<const uint32_t*>(src)[v];
  }
}

// host row `row` <-> cache slot `slot` (both table-local) of table t: weights, then each optimizer state
__device__ __forceinline__ void move_row(const UvmPrefetchArgs& a, int t, int64_t row, int64_t slot, bool to_host, int lane) {
  const int64_t D = a.dim[t];
  const int64_t he = a.host_elem_base[t] + row * D, ce = a.cache_elem_base[t] + slot * D;
  const int64_t hr = a.row_base[t] + row, cr = a.slot_base[t] + slot;
  uint8_t* h = a.host_w + he * a.w_bytes;
  uint8_t* c = a.cache_w + ce * a.w_bytes;
  copy_row(to_host ? h : c, to_host ? c : h, D * a.w_bytes, lane);
  const int64_t kinds[2] = {a.s1_kind, a.s2_kind};
  float* hs[2] = {a.host_s1, a.host_s2};
  float* cs[2] = {a.cache_s1, a.cache_s2};
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    if (kinds[q] == 1) {
      if (lane == 0) {
        if (to_host) hs[q][hr] = cs[q][cr];
        else cs[q][cr] = hs[q][hr];
      }
    } else if (kinds[q] == 2) {
      uint8_t* hp = reinterpret_cast<uint8_t*>(hs[q] + he);
      uint8_t* cp = reinterpret_cast<uint8_t*>(cs[q] + ce);
      copy_row(to_host ? hp : cp, to_host ? cp : hp, D * 4, lane);
    }
  }
}

// One warp per missing row (grid-stride over the device-side count): evict = write the live victims back, fill = bring the rows in.
template <bool kEvict>
__global__ void __launch_bounds__(256) uvm_move_kernel(UvmPrefetchArgs a, Ws w) {
  const int lane = threadIdx.x & 31;
  const int64_t total = *w.n_sel;
  const int64_t warps = (int64_t) gridDim.x * (blockDim.x >> 5);
  for (int64_t m = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5; m < total; m += warps) {
    const int t = upper_index(w.miss_base, (int) a.T, m);
    if (!w.take[t]) continue;
    const int64_t g = w.victim[m];
    const int64_t slot = g - a.slot_base[t];
    if (kEvict) {
      const int64_t old = a.row_of_slot[g];
      if (lane == 0) w.old[m] = old;
      if (old < 0) continue;
      if (a.move_rows) move_row(a, t, old, slot, true, lane);
      if (lane == 0) {
        a.slot_of_row[a.row_base[t] + old] = -1;
        atomicAdd(a.stats + 3 * t + 2, 1ull);
      }
    } else {
      const int64_t row = (int64_t) w.miss[m] - a.row_base[t];
      if (a.move_rows) move_row(a, t, row, slot, false, lane);
      if (lane == 0) {
        a.slot_of_row[w.miss[m]] = (int32_t) slot;
        a.row_of_slot[g] = row;
        a.score[g] = a.lfu ? 1 : a.tick;
        a.stamp[g] = a.tick;
      }
    }
  }
}

}  // namespace

TRB_API int64_t trb_uvm_prefetch_ws_bytes(int64_t n, int64_t T, int64_t total_rows) {
  Ws w;
  return (int64_t) carve(nullptr, n, T, end_bit_of(total_rows), &w);
}

// Byte offsets in the workspace of what a caller that moves the rows itself (move_rows = 0) reads back after the prefetch:
// out = {n_sel (int32 [1]), miss_base (int64 [T+1]), take (int32 [T]), victim (int64 global slot), old (int64 table-local row),
// miss (int64 global row)}; entry m < n_sel of the last three belongs to table t with miss_base[t] <= m < miss_base[t+1].
TRB_API int trb_uvm_prefetch_ws_layout(int64_t n, int64_t T, int64_t total_rows, int64_t* out) {
  Ws w;
  uint8_t* const base = reinterpret_cast<uint8_t*>((uintptr_t) 256);  // any aligned base: only differences are reported
  carve(base, n, T, end_bit_of(total_rows), &w);
  const void* ptrs[6] = {w.n_sel, w.miss_base, w.take, w.victim, w.old, w.miss};
  for (int i = 0; i < 6; ++i) out[i] = (int64_t) ((const uint8_t*) ptrs[i] - base);
  return 0;
}

// `args`: host struct (ops/uvm.py `_PrefetchArgs`). The sequence of launches depends on the batch size only (CUB picks its sort passes by item count), never on the ids; nothing is read back to the host.
TRB_API int trb_uvm_prefetch(const UvmPrefetchArgs* args, cudaStream_t stream) {
  const UvmPrefetchArgs a = *args;
  if (a.T <= 0 || a.F <= 0 || a.B < 0 || a.tick < 1 || a.tick >= ((int64_t) 1 << 32) || a.n < 0 || a.n >= ((int64_t) 1 << 31)) return -2;
  const int end_bit = end_bit_of(a.total_rows);
  Ws w;
  if ((int64_t) carve(nullptr, a.n, a.T, end_bit, &w) > a.workspace_bytes) return -3;
  carve((uint8_t*) a.workspace, a.n, a.T, end_bit, &w);
  const int64_t m = a.n > 0 ? a.n : 1;  // an empty batch runs the same launches over one dropped key
  const unsigned long long sentinel = (unsigned long long) a.total_rows;
  const unsigned blocks = (unsigned) ((m + 255) / 256);
  TRB_CUDA(cudaMemsetAsync(w.distinct, 0, (size_t) (w.take - w.distinct) * sizeof(int32_t), stream));  // distinct + n_miss
  uvm_keys_kernel<<<blocks, 256, 0, stream>>>(a, m, w.keys_in, sentinel);
  TRB_CHECK_LAUNCH();
  size_t tmp = w.tmp_bytes;
  TRB_CUDA(cub::DeviceRadixSort::SortKeys(w.tmp, tmp, w.keys_in, w.keys, (int) m, 0, end_bit, stream));
  TRB_COUNT_LAUNCH();
  uvm_count_kernel<<<blocks, 256, 0, stream>>>(a, m, w.keys, sentinel, w.distinct);
  TRB_CHECK_LAUNCH();
  uvm_probe_kernel<<<blocks, 256, 0, stream>>>(a, m, w.keys, sentinel, w.distinct, w.n_miss, w.flag);
  TRB_CHECK_LAUNCH();
  tmp = w.tmp_bytes;
  TRB_CUDA(cub::DeviceSelect::Flagged(w.tmp, tmp, w.keys, w.flag, w.miss, w.n_sel, (int) m, stream));
  TRB_COUNT_LAUNCH();
  uvm_victim_kernel<<<(unsigned) a.T, kSelThreads, 0, stream>>>(a, w);
  TRB_CHECK_LAUNCH();
  const unsigned mv = (unsigned) std::min<int64_t>((m * 32 + 255) / 256, (int64_t) trb_num_sms() * 8);
  uvm_move_kernel<true><<<mv, 256, 0, stream>>>(a, w);
  TRB_CHECK_LAUNCH();
  uvm_move_kernel<false><<<mv, 256, 0, stream>>>(a, w);
  TRB_CHECK_LAUNCH();
  return 0;
}
