// Sparse-feature input dist as ONE device-side pass (hot path 1): bucketize + feature permute + peer write.
//
// Reference path (what this replaces): `block_bucketize_sparse_features` (embedding_sharding.py:268-353) -> feature
// `permute` (jagged_tensor.py:2816-2898) -> splits all-to-all -> D2H `.tolist()` host sync (dist_data.py:569-572) -> one NCCL
// all-to-all per tensor -> recat permute (dist_data.py:218-347) -> cumsum. That is ~30 kernels, 4 collectives and a host
// sync per step.
//
// Here every sharding type is described by ONE table of *lookup units* u = (input key, row range [lo, hi), destination rank,
// slot among the destination's units): TABLE_WISE / COLUMN_WISE units take the whole bag, ROW_WISE / TWRW / GRID units take the
// ids of their row range and rebase them (id - lo). Three launches, no host involvement:
//
//   A  route_len   len[u, b]   = #ids of bag (key(u), b) inside [lo, hi)
//   B  scan        exclusive prefix sum over len (cub::DeviceScan, one pass, decoupled look-back)
//   C  route_write per (u, b): offsets and (rebased) ids [+ per-id weights] are stored STRAIGHT INTO THE DESTINATION RANK's
//                  receive region for this source over NVLink (posted stores), already in the layout its lookup kernel consumes
//                  ([unit slot][sample] offsets relative to the region, see TrbSrcView in common.cuh) - no recat pass, no
//                  size exchange: regions have a fixed capacity, true sizes travel as the offsets themselves, an overflow
//                  raises a device flag that the host reads back asynchronously in the same step.
//
// With one destination pointing at local memory the same kernels produce the routed (unit-ordered) KJT for the NCCL / gloo
// fallback transport, plus the `unbucketize` permutation the sequence (unpooled) path needs. `trb_kjt_route_pos` adds a per-destination
// payload for the fused sequence inference path: next to every routed id, its position inside its feature's values (where its row goes).
#include "common.cuh"
#include <cub/device/device_scan.cuh>
#include <type_traits>

struct RouteParams {
  const void* in_off;       // [K * B + 1] offsets of the local KJT
  const void* in_val;       // ids
  const float* in_wgt;      // per-id weights or nullptr
  const int32_t* u_key;     // [U] position of the unit's feature among the input keys
  const int64_t* u_row_lo;  // [U]
  const int64_t* u_row_hi;  // [U] (full table: lo = 0, hi = INT64_MAX)
  const int32_t* u_dest;    // [U] destination index
  const int32_t* u_slot;    // [U] slot of the unit among the destination's units
  const int32_t* u_cslice;  // [U] column-slice index of the unit inside its feature (unbucketize only)
  const int32_t* dest_ustart;  // [n_dest + 1] first global unit of every destination
  int32_t* len;             // [U * B + 1] scratch (last entry 0)
  int32_t* scan;            // [U * B + 1] exclusive scan of len; scan[U * B] = total routed ids
  TrbPeerPtrs out_off;      // per destination: MY region's offsets [U_d * B + 1]
  TrbPeerPtrs out_val;      // per destination: MY region's ids [capacity]
  TrbPeerPtrs out_wgt;      // per destination: MY region's per-id weights (or nullptr)
  int64_t* unbucketize;     // optional [n_in * fc]: routed position of (input id j, column slice c)
  int64_t* pos_out;         // optional [capacity]: position of the id inside its ORIGINAL bag (single-destination / compact mode)
  const int64_t* u_wrap;    // optional [U]: ids >= u_wrap[u] (past the last block of the table) are dealt round-robin: kept by the unit
  const int32_t* u_wrap_rem;  //             whose remainder id % wrap_mod equals u_wrap_rem[u], with local id = id / wrap_mod
  int32_t wrap_mod;
  const int32_t* u_edge;    // optional [U]: bit 0 = the unit also keeps ids BELOW its range, bit 1 = ids ABOVE it (first / last row shard of a
                            // table: invalid ids are forwarded - the lookup kernel zeroes them - so every input id is routed exactly once)
  int32_t* overflow;        // set to 1 when a destination region would exceed `capacity`
  int64_t capacity;
  int32_t U, B, n_dest, fc;
  int32_t in_off64, val64, out_off64, out_val64;
};

// Route with a per-destination position payload (trb_kjt_route_pos): next to every routed id its position inside its feature's values,
// j - in_off[key(u) * B], as int32. A separate type, so the parameter block and the code of the plain route kernels stay as they were.
struct RoutePosParams : RouteParams {
  TrbPeerPtrs out_pos;      // per destination: MY region's positions [capacity]
};

template <class P> constexpr bool kRoutePos = std::is_same_v<P, RoutePosParams>;

// The position store of a writer: nothing for RouteParams.
template <class P> struct RoutePosOut {
  __device__ __forceinline__ void init(const P&, int, int) {}
  __device__ __forceinline__ void st(int64_t, int64_t) {}
};
template <> struct RoutePosOut<RoutePosParams> {
  int32_t* dst;
  int64_t fs;  // first value of the unit's feature
  __device__ __forceinline__ void init(const RoutePosParams& p, int u, int d) {
    dst = reinterpret_cast<int32_t*>(p.out_pos.p[d]);
    fs = trb_ld_idx(p.in_off, (int64_t) p.u_key[u] * p.B, p.in_off64);
  }
  __device__ __forceinline__ void st(int64_t k, int64_t j) { dst[k] = (int32_t) (j - fs); }
};

__device__ __forceinline__ bool route_full(const RouteParams& p, int u) { return p.u_row_lo[u] == 0 && p.u_row_hi[u] == INT64_MAX; }

// does unit u take this id, and as which local id? (row range, or the round-robin rule for ids past the table's last block)
__device__ __forceinline__ bool route_take(const RouteParams& p, int u, int64_t id, int64_t lo, int64_t hi, int64_t* local) {
  if (p.u_wrap != nullptr && id >= p.u_wrap[u]) {
    *local = id / p.wrap_mod;
    return (int32_t) (id % p.wrap_mod) == p.u_wrap_rem[u];
  }
  *local = id - lo;
  if (p.u_edge != nullptr) {
    const int e = p.u_edge[u];
    if (((e & 1) && id < lo) || ((e & 2) && id >= hi)) return true;
  }
  return id >= lo && id < hi;
}

// ---- A: per (unit, sample) lengths ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) kjt_route_len_kernel(const RouteParams p) {
  const int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = (int64_t) p.U * p.B;
  if (t == n) p.len[n] = 0;
  if (t >= n) return;
  const int u = (int) (t / p.B);
  const int b = (int) (t - (int64_t) u * p.B);
  const int64_t bag = (int64_t) p.u_key[u] * p.B + b;
  const int64_t s = trb_ld_idx(p.in_off, bag, p.in_off64), e = trb_ld_idx(p.in_off, bag + 1, p.in_off64);
  int32_t c;
  if (route_full(p, u)) {
    c = (int32_t) (e - s);
  } else {
    const int64_t lo = p.u_row_lo[u], hi = p.u_row_hi[u];
    c = 0;
    for (int64_t j = s; j < e; ++j) {
      const int64_t id = trb_ld_idx(p.in_val, j, p.val64);
      int64_t local;
      c += route_take(p, u, id, lo, hi, &local) ? 1 : 0;
    }
  }
  p.len[t] = c;
}

// ---- C: write offsets + ids into the destination regions -------------------------------------------------------------------
// One thread per (unit, sample): consecutive threads handle consecutive samples of one unit, i.e. consecutive source ids and
// consecutive destination positions for short bags (one-hot features: fully coalesced 8 B loads / peer stores).
template <class P>
__device__ __forceinline__ void route_write(const P p) {
  const int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = (int64_t) p.U * p.B;
  if (t >= n) return;
  const int u = (int) (t / p.B);
  const int b = (int) (t - (int64_t) u * p.B);
  const int d = p.u_dest[u];
  const int64_t seg0 = (int64_t) p.dest_ustart[d] * p.B;
  const int32_t base = p.scan[seg0];
  const int64_t o = (int64_t) p.scan[t] - base;  // position inside MY region at destination d
  const int64_t C = p.capacity;
  const int64_t oi = (int64_t) p.u_slot[u] * p.B + b;
  trb_st_idx(p.out_off.p[d], oi, p.out_off64, o < C ? o : C);
  if (u == p.dest_ustart[d + 1] - 1 && b == p.B - 1) {  // closing entry of the destination: total ids from this source
    const int64_t total = (int64_t) p.scan[(int64_t) p.dest_ustart[d + 1] * p.B] - base;
    trb_st_idx(p.out_off.p[d], oi + 1, p.out_off64, total < C ? total : C);
    if (total > C) *p.overflow = 1;
  }
  const int64_t bag = (int64_t) p.u_key[u] * p.B + b;
  const int64_t s = trb_ld_idx(p.in_off, bag, p.in_off64), e = trb_ld_idx(p.in_off, bag + 1, p.in_off64);
  const int64_t lo = p.u_row_lo[u], hi = p.u_row_hi[u];
  const bool full = route_full(p, u);  // whole-table units forward EVERY id (invalid ones are zeroed by the lookup kernel)
  float* const wdst = reinterpret_cast<float*>(p.out_wgt.p[d]);
  RoutePosOut<P> po;
  po.init(p, u, d);
  int64_t k = o;
  for (int64_t j = s; j < e; ++j) {
    const int64_t id = trb_ld_idx(p.in_val, j, p.val64);
    int64_t local = id - lo;
    if (!full && !route_take(p, u, id, lo, hi, &local)) continue;
    if (k < C) {
      trb_st_idx(p.out_val.p[d], k, p.out_val64, local);
      if (p.in_wgt != nullptr) wdst[k] = p.in_wgt[j];
      if (p.pos_out != nullptr) p.pos_out[k] = j - s;
      po.st(k, j);
    }
    if (p.unbucketize != nullptr) p.unbucketize[j * p.fc + p.u_cslice[u]] = k + base;
    ++k;
  }
}

__global__ void __launch_bounds__(256) kjt_route_write_kernel(const RouteParams p) { route_write(p); }
__global__ void __launch_bounds__(256) kjt_route_write_pos_kernel(const RoutePosParams p) { route_write(p); }

// Long bags: one warp per (unit, sample), lanes stride over the bag; row-range filtering keeps the source order through a
// ballot prefix (ids of one bag stay in input order, which the sequence path relies on).
template <class P>
__device__ __forceinline__ void route_write_warp(const P p) {
  const int lane = threadIdx.x & 31;
  const int64_t t = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n = (int64_t) p.U * p.B;
  if (t >= n) return;
  const int u = (int) (t / p.B);
  const int b = (int) (t - (int64_t) u * p.B);
  const int d = p.u_dest[u];
  const int64_t seg0 = (int64_t) p.dest_ustart[d] * p.B;
  const int32_t base = p.scan[seg0];
  const int64_t o = (int64_t) p.scan[t] - base;
  const int64_t C = p.capacity;
  const int64_t oi = (int64_t) p.u_slot[u] * p.B + b;
  if (lane == 0) {
    trb_st_idx(p.out_off.p[d], oi, p.out_off64, o < C ? o : C);
    if (u == p.dest_ustart[d + 1] - 1 && b == p.B - 1) {
      const int64_t total = (int64_t) p.scan[(int64_t) p.dest_ustart[d + 1] * p.B] - base;
      trb_st_idx(p.out_off.p[d], oi + 1, p.out_off64, total < C ? total : C);
      if (total > C) *p.overflow = 1;
    }
  }
  const int64_t bag = (int64_t) p.u_key[u] * p.B + b;
  const int64_t s = trb_ld_idx(p.in_off, bag, p.in_off64), e = trb_ld_idx(p.in_off, bag + 1, p.in_off64);
  const int64_t lo = p.u_row_lo[u], hi = p.u_row_hi[u];
  const bool full = route_full(p, u);
  float* const wdst = reinterpret_cast<float*>(p.out_wgt.p[d]);
  RoutePosOut<P> po;
  po.init(p, u, d);
  int64_t k0 = o;
  for (int64_t j0 = s; j0 < e; j0 += 32) {
    const int64_t j = j0 + lane;
    int64_t id = 0, local = 0;
    bool keep = false;
    if (j < e) {
      id = trb_ld_idx(p.in_val, j, p.val64);
      local = id - lo;
      keep = full || route_take(p, u, id, lo, hi, &local);
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int64_t k = k0 + __popc(m & ((1u << lane) - 1u));
      if (k < C) {
        trb_st_idx(p.out_val.p[d], k, p.out_val64, local);
        if (p.in_wgt != nullptr) wdst[k] = p.in_wgt[j];
        if (p.pos_out != nullptr) p.pos_out[k] = j - s;
        po.st(k, j);
      }
      if (p.unbucketize != nullptr) p.unbucketize[j * p.fc + p.u_cslice[u]] = k + base;
    }
    k0 += __popc(m);
  }
}

__global__ void __launch_bounds__(256) kjt_route_write_warp_kernel(const RouteParams p) { route_write_warp(p); }
__global__ void __launch_bounds__(256) kjt_route_write_warp_pos_kernel(const RoutePosParams p) { route_write_warp(p); }

static inline size_t route_align(size_t x) { return (x + 255) & ~(size_t) 255; }

static size_t route_scan_tmp_bytes(int64_t n) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const int32_t*) nullptr, (int32_t*) nullptr, (int) n);
  return bytes;
}

TRB_API int64_t trb_kjt_route_workspace_bytes(int U, int B) {
  const int64_t n = (int64_t) U * B + 1;
  return (int64_t) (2 * route_align(n * 4) + route_align(route_scan_tmp_bytes(n)) + 256);
}

// Fills the fields of RouteParams and launches the three passes with the writer of P.
template <class P>
static int route_run(P& p, const void* in_off, int in_off64, const void* in_val, int val64, const float* in_wgt, int B, const int32_t* u_key,
                     const int64_t* u_row_lo, const int64_t* u_row_hi, const int32_t* u_dest, const int32_t* u_slot,
                     const int32_t* u_cslice, const int32_t* dest_ustart, int U, int n_dest, void* const* out_off_ptrs, int out_off64,
                     void* const* out_val_ptrs, int out_val64, void* const* out_wgt_ptrs, int64_t capacity, int64_t* unbucketize, int fc,
                     int64_t* pos_out, const int64_t* u_wrap, const int32_t* u_wrap_rem, int wrap_mod, const int32_t* u_edge, int32_t* lengths_out,
                     int32_t* overflow, void* workspace, int64_t workspace_bytes, int avg_len_hint, cudaStream_t stream) {
  if (n_dest < 1 || n_dest > TRB_MAX_PEERS) return -1;
  if (U == 0 || B == 0) return 0;
  const int64_t n = (int64_t) U * B;
  if (n + 1 >= ((int64_t) 1 << 31)) return -6;
  if (workspace_bytes < trb_kjt_route_workspace_bytes(U, B)) return -7;
  p.in_off = in_off; p.in_val = in_val; p.in_wgt = in_wgt;
  p.u_key = u_key; p.u_row_lo = u_row_lo; p.u_row_hi = u_row_hi; p.u_dest = u_dest; p.u_slot = u_slot; p.u_cslice = u_cslice;
  p.dest_ustart = dest_ustart;
  char* ws = reinterpret_cast<char*>(workspace);
  p.len = lengths_out != nullptr ? lengths_out : reinterpret_cast<int32_t*>(ws);  // caller-owned [U * B + 1]: the routed lengths are an output
  p.scan = reinterpret_cast<int32_t*>(ws + route_align((n + 1) * 4));
  void* scan_tmp = ws + 2 * route_align((n + 1) * 4);
  size_t scan_tmp_bytes = route_scan_tmp_bytes(n + 1);
  for (int i = 0; i < TRB_MAX_PEERS; ++i) {
    p.out_off.p[i] = i < n_dest ? out_off_ptrs[i] : nullptr;
    p.out_val.p[i] = i < n_dest ? out_val_ptrs[i] : nullptr;
    p.out_wgt.p[i] = (i < n_dest && out_wgt_ptrs != nullptr) ? out_wgt_ptrs[i] : nullptr;
  }
  p.unbucketize = unbucketize; p.overflow = overflow; p.capacity = capacity;
  p.pos_out = pos_out; p.u_wrap = u_wrap; p.u_wrap_rem = u_wrap_rem; p.wrap_mod = wrap_mod > 0 ? wrap_mod : 1; p.u_edge = u_edge;
  p.U = U; p.B = B; p.n_dest = n_dest; p.fc = fc > 0 ? fc : 1;
  p.in_off64 = in_off64; p.val64 = val64; p.out_off64 = out_off64; p.out_val64 = out_val64;
  const int threads = 256;
  kjt_route_len_kernel<<<(unsigned) ((n + 1 + threads - 1) / threads), threads, 0, stream>>>(static_cast<const RouteParams&>(p));
  TRB_CHECK_LAUNCH();
  TRB_CUDA(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_tmp_bytes, (const int32_t*) p.len, p.scan, (int) (n + 1), stream));
  g_trb_launches += 1;
  if (avg_len_hint > 8) {
    const unsigned blocks = (unsigned) ((n * 32 + threads - 1) / threads);
    if constexpr (kRoutePos<P>) kjt_route_write_warp_pos_kernel<<<blocks, threads, 0, stream>>>(p);
    else kjt_route_write_warp_kernel<<<blocks, threads, 0, stream>>>(p);
  } else {
    const unsigned blocks = (unsigned) ((n + threads - 1) / threads);
    if constexpr (kRoutePos<P>) kjt_route_write_pos_kernel<<<blocks, threads, 0, stream>>>(p);
    else kjt_route_write_kernel<<<blocks, threads, 0, stream>>>(p);
  }
  TRB_CHECK_LAUNCH();
  return 0;
}

// Returns 0 on success. `avg_len_hint` (ids per bag, host estimate) picks the thread-per-bag or warp-per-bag writer.
TRB_API int trb_kjt_route_ex(const void* in_off, int in_off64, const void* in_val, int val64, const float* in_wgt, int B, const int32_t* u_key,
                             const int64_t* u_row_lo, const int64_t* u_row_hi, const int32_t* u_dest, const int32_t* u_slot,
                             const int32_t* u_cslice, const int32_t* dest_ustart, int U, int n_dest, void* const* out_off_ptrs, int out_off64,
                             void* const* out_val_ptrs, int out_val64, void* const* out_wgt_ptrs, int64_t capacity, int64_t* unbucketize, int fc,
                             int64_t* pos_out, const int64_t* u_wrap, const int32_t* u_wrap_rem, int wrap_mod, const int32_t* u_edge, int32_t* lengths_out,
                             int32_t* overflow, void* workspace, int64_t workspace_bytes, int avg_len_hint, cudaStream_t stream) {
  RouteParams p;
  return route_run(p, in_off, in_off64, in_val, val64, in_wgt, B, u_key, u_row_lo, u_row_hi, u_dest, u_slot, u_cslice, dest_ustart, U, n_dest,
                   out_off_ptrs, out_off64, out_val_ptrs, out_val64, out_wgt_ptrs, capacity, unbucketize, fc, pos_out, u_wrap, u_wrap_rem, wrap_mod,
                   u_edge, lengths_out, overflow, workspace, workspace_bytes, avg_len_hint, stream);
}

// The route of the sequence inference path: ids (no weights) plus, per destination, the int32 position of every routed id inside its
// feature's values (`out_pos_ptrs`, [capacity] each). `n_in` = number of input ids; more than INT32_MAX of them cannot be addressed by
// the int32 positions and returns -8. `u_edge` as in trb_kjt_route_ex (may be null).
TRB_API int trb_kjt_route_pos(const void* in_off, int in_off64, const void* in_val, int val64, int64_t n_in, int B, const int32_t* u_key,
                              const int64_t* u_row_lo, const int64_t* u_row_hi, const int32_t* u_dest, const int32_t* u_slot, const int32_t* dest_ustart,
                              const int32_t* u_edge, int U, int n_dest, void* const* out_off_ptrs, int out_off64, void* const* out_val_ptrs, int out_val64,
                              void* const* out_pos_ptrs, int64_t capacity, int32_t* overflow, void* workspace, int64_t workspace_bytes, int avg_len_hint,
                              cudaStream_t stream) {
  if (n_in > INT32_MAX) return -8;
  if (n_dest < 1 || n_dest > TRB_MAX_PEERS) return -1;
  RoutePosParams p;
  for (int i = 0; i < TRB_MAX_PEERS; ++i) p.out_pos.p[i] = i < n_dest ? out_pos_ptrs[i] : nullptr;
  return route_run(p, in_off, in_off64, in_val, val64, nullptr, B, u_key, u_row_lo, u_row_hi, u_dest, u_slot, nullptr, dest_ustart, U, n_dest,
                   out_off_ptrs, out_off64, out_val_ptrs, out_val64, nullptr, capacity, nullptr, 1, nullptr, nullptr, nullptr, 1, u_edge, nullptr,
                   overflow, workspace, workspace_bytes, avg_len_hint, stream);
}

TRB_API int trb_kjt_route(const void* in_off, int in_off64, const void* in_val, int val64, const float* in_wgt, int B, const int32_t* u_key,
                          const int64_t* u_row_lo, const int64_t* u_row_hi, const int32_t* u_dest, const int32_t* u_slot,
                          const int32_t* u_cslice, const int32_t* dest_ustart, int U, int n_dest, void* const* out_off_ptrs, int out_off64,
                          void* const* out_val_ptrs, int out_val64, void* const* out_wgt_ptrs, int64_t capacity, int64_t* unbucketize, int fc,
                          int32_t* overflow, void* workspace, int64_t workspace_bytes, int avg_len_hint, cudaStream_t stream) {
  return trb_kjt_route_ex(in_off, in_off64, in_val, val64, in_wgt, B, u_key, u_row_lo, u_row_hi, u_dest, u_slot, u_cslice, dest_ustart, U, n_dest, out_off_ptrs,
                          out_off64, out_val_ptrs, out_val64, out_wgt_ptrs, capacity, unbucketize, fc, nullptr, nullptr, nullptr, 1, nullptr, nullptr, overflow, workspace,
                          workspace_bytes, avg_len_hint, stream);
}
