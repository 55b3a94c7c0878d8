// Table-batched embedding backward fused with the sparse optimizer (sm_90a).
//
// Exact (deterministic, duplicate-safe) semantics like the reference's EXACT_* TBE optimizers
// (torchrec/distributed/embedding_types.py:57-72; fused backward reached through autograd at
// batched_embedding_kernel.py:3010-3058): the gradient of every *unique* row is summed over all
// of its occurrences first, then the optimizer is applied once to that row. No dense gradient is
// ever materialised.
//
// Pipeline (all stream-ordered, no host sync):
//   K0  build keys     key[i] = row_base(feature) + indices[i]   (invalid / padding -> sentinel)
//                      bag_of[i] = bag containing position i
//   K1  cub radix sort (key, i)
//   K2  chunk walk     one warp per 32 sorted positions: reduce each run of equal keys; runs that
//                      live inside the chunk get the optimizer applied immediately, runs that
//                      cross a chunk boundary leave a partial sum
//   K3  span combine   one CTA per boundary-crossing run sums the partials and applies
//
// The gradient rows are read through TrbPeerPtrs: with W peer pointers the kernel *pulls*
// grad[b_local, cols(f)] straight from the rank that owns sample b over NVLink — that is the
// backward all-to-all of the reference (comm_ops.py:1581-1646) fused into the optimizer kernel.
#include <cstdlib>

#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>

enum TrbOpt : int {
  OPT_SGD = 0,
  OPT_ROWWISE_ADAGRAD = 1,
  OPT_ADAGRAD = 2,
  OPT_ADAM = 3,
  OPT_PARTIAL_ROWWISE_ADAM = 4,
  OPT_LAMB = 5,
  OPT_PARTIAL_ROWWISE_LAMB = 6,
  OPT_LARS_SGD = 7,
  OPT_NONE = 8,  // accumulate summed gradient rows into a dense fp32 grad buffer (state1)
  OPT_LION = 9,  // sign(beta1 m + (1-beta1) g) update, momentum refreshed with beta2
};

// hyper[] slots (device memory, refreshed by the host each step; graph-capture friendly)
#define HP_LR 0
#define HP_EPS 1
#define HP_BETA1 2
#define HP_BETA2 3
#define HP_WD 4
#define HP_STEP 5
#define HP_MAXGRAD 6
#define HP_MOMENTUM 7

struct TbeBwdParams {
  void* weights;
  float* state1;  // rowwise: [total_rows]; elementwise: same layout as weights (fp32)
  float* state2;
  const float* hyper;
  const int64_t* feat_woff;     // [F]
  const int64_t* feat_rows;     // [F]
  const int64_t* feat_rowbase;  // [F] first global row id of feature f's table
  const int32_t* feat_dim;      // [F]
  const int32_t* feat_col;      // [F]
  TrbSrcView src;    // ids (one KJT or per-source regions)
  TrbPeerPtrs grad;  // gradient sources
  int64_t grad_stride;
  int64_t n;  // capacity of indices
  int64_t total_rows;
  int32_t B, B_local, F;
  int32_t mean;
  float grad_scale;  // multiplies every gradient row (1/W gradient division of the pooled output dist, folded into the kernel)
  int32_t wd_mode;  // 0 none, 1 L2, 2 decoupled
  // workspace
  void* keys;
  void* keys_sorted;
  int32_t* vals;
  int32_t* vals_sorted;
  int32_t* bag_of;
  float* partials;  // [chunks][2][max_dim]
  uint8_t* span_flags;
  uint8_t* chunk_done;  // [chunks] set by tbe_bwd_unique_kernel (nullptr: generic walk handles everything)
  int32_t* long_list;   // [chunks] first chunks of spans longer than kLongSpan pieces
  int32_t* long_count;  // zeroed by tbe_bwd_build_keys
  int sr;               // 1: stochastic rounding of the updated row when the table is bf16 / fp16 (unbiased low-precision training)
  unsigned long long sr_seed;
  int prefetch;         // 1: lanes prefetch their key's rows into L2 ahead of the walk (bit 1: also the gradient rows = local memory)
  int32_t max_dim;
  int32_t key64;
  int32_t opt;
  int32_t phase;        // 0: whole backward; 1: prepare only (keys + sort: depends on the ids alone, can run long before the gradient exists); 2: apply only
};

__device__ __forceinline__ uint64_t ld_key(const void* p, int64_t i, int key64) {
  return key64 ? reinterpret_cast<const uint64_t*>(p)[i] : (uint64_t) reinterpret_cast<const uint32_t*>(p)[i];
}

// number of ids in global bag (f * B + b)
__device__ __forceinline__ int64_t bag_len(const TbeBwdParams& p, int bag) {
  const int f = bag / p.B;
  int64_t pos_base;
  const int64_t oi = trb_src_off_index(p.src, f, bag - f * p.B, &pos_base);
  return trb_ld_idx(p.src.offsets, oi + 1, p.src.off64) - trb_ld_idx(p.src.offsets, oi, p.src.off64);
}

__global__ void __launch_bounds__(256) tbe_bwd_build_keys(const TbeBwdParams p) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *p.long_count = 0;
  if (i >= p.n) return;
  // position i lives in source region s (one region when n_src == 1); offsets of a region are relative to its start
  int s = 0;
  int64_t li = i;
  if (p.src.n_src > 1) {
    s = (int) (i / p.src.idx_stride);
    li = i - (int64_t) s * p.src.idx_stride;
  }
  const int64_t n_bags = (int64_t) p.F * p.src.src_B;
  const int64_t obase = (int64_t) s * p.src.off_stride;
  const int64_t total = trb_ld_idx(p.src.offsets, obase + n_bags, p.src.off64);
  uint64_t key = (uint64_t) p.total_rows;  // sentinel sorts last
  int32_t bag = 0;
  const int64_t first = trb_ld_idx(p.src.offsets, obase, p.src.off64);  // offsets may be a window into a larger id array
  if (s < p.src.n_src && li >= first && li < total) {
    // largest bag with offsets[bag] <= li  (bags may be empty -> take the last such bag)
    int64_t lo = 0, hi = n_bags - 1;
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (trb_ld_idx(p.src.offsets, obase + mid, p.src.off64) <= li) lo = mid; else hi = mid - 1;
    }
    const int f = (int) (lo / p.src.src_B);
    bag = (int32_t) ((int64_t) f * p.B + (int64_t) s * p.src.src_B + (lo - (int64_t) f * p.src.src_B));
    const int64_t idx = trb_ld_idx(p.src.indices, i, p.src.idx64);
    if (idx >= 0 && idx < p.feat_rows[f]) key = (uint64_t) (p.feat_rowbase[f] + idx);
  }
  if (p.key64) reinterpret_cast<uint64_t*>(p.keys)[i] = key;
  else reinterpret_cast<uint32_t*>(p.keys)[i] = (uint32_t) key;
  p.vals[i] = (int32_t) i;
  p.bag_of[i] = bag;
}

// ---- stochastic rounding (FBGEMM `stochastic_rounding=True` for FP16/BF16 tables) -------------------------------------------------
// Round-to-nearest loses every update smaller than half an ulp of the stored weight; rounding up with probability
// (x - lo) / (hi - lo) keeps the expected value exact. Random bits: splitmix64 of (seed, row key, vector index): one 64-bit hash =
// 4 x 16 bits for the 4 elements a lane stores; deterministic for a given (seed, step).
__device__ __forceinline__ unsigned long long trb_splitmix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__device__ __forceinline__ __nv_bfloat16 trb_sr_bf16(float x, unsigned r16) {
  unsigned b = __float_as_uint(x);
  if ((b & 0x7F800000u) != 0x7F800000u) b += r16;  // finite: add 16 random low bits, then truncate
  return __ushort_as_bfloat16((unsigned short) (b >> 16));
}

__device__ __forceinline__ __half trb_sr_half(float x, unsigned r16) {
  const __half lo = __float2half_rd(x), hi = __float2half_ru(x);
  const float flo = __half2float(lo), fhi = __half2float(hi);
  if (!(fhi > flo)) return lo;  // exactly representable, inf or nan
  const float pr = (x - flo) / (fhi - flo);
  return ((float) r16 * (1.f / 65536.f) < pr) ? hi : lo;
}

template <typename W>
__device__ __forceinline__ void trb_store_row4_sr(W* dst, float4 v, unsigned long long rnd) {
  Vec4<W>::st(dst, v);
}
template <>
__device__ __forceinline__ void trb_store_row4_sr<__nv_bfloat16>(__nv_bfloat16* dst, float4 v, unsigned long long rnd) {
  __nv_bfloat16 o[4] = {trb_sr_bf16(v.x, (unsigned) (rnd & 0xFFFF)), trb_sr_bf16(v.y, (unsigned) ((rnd >> 16) & 0xFFFF)),
                        trb_sr_bf16(v.z, (unsigned) ((rnd >> 32) & 0xFFFF)), trb_sr_bf16(v.w, (unsigned) ((rnd >> 48) & 0xFFFF))};
  *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(o);
}
template <>
__device__ __forceinline__ void trb_store_row4_sr<__half>(__half* dst, float4 v, unsigned long long rnd) {
  __half o[4] = {trb_sr_half(v.x, (unsigned) (rnd & 0xFFFF)), trb_sr_half(v.y, (unsigned) ((rnd >> 16) & 0xFFFF)),
                 trb_sr_half(v.z, (unsigned) ((rnd >> 32) & 0xFFFF)), trb_sr_half(v.w, (unsigned) ((rnd >> 48) & 0xFFFF))};
  *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(o);
}

// ---- optimizer application on one unique row ------------------------------------------------
// g[k] holds the summed gradient for elements (lane + 32k)*4 .. +3 of the row.
// PRE: the caller already issued the loads of the weight row (`wpre`) and, for row-wise Adagrad, of the row state (`spre`, lane 0)
// BEFORE it accumulated the gradient: the three round trips of a run (gradient rows, weight row, state) overlap instead of
// following each other.
template <typename W, int MAXV, bool PRE = false>
__device__ __forceinline__ void apply_row(const TbeBwdParams& p, int64_t key, int f, float4 (&g)[MAXV], int lane, const float4* wpre = nullptr,
                                          float spre = 0.f) {
  const int OPT = p.opt;
  const int D = p.feat_dim[f];
  const int nvec = D >> 2;
  const int64_t row = key - p.feat_rowbase[f];
  const int64_t eoff = p.feat_woff[f] + row * D;
  W* w = reinterpret_cast<W*>(p.weights) + eoff;
  const float lr = p.hyper[HP_LR], eps = p.hyper[HP_EPS], wd = p.hyper[HP_WD];
  const float maxg = p.hyper[HP_MAXGRAD];

  float4 wv[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = lane + k * 32;
    if constexpr (PRE) wv[k] = wpre[k];
    else wv[k] = (vi < nvec && OPT != OPT_NONE) ? Vec4<W>::ld(w + vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (maxg > 0.f) {
      g[k].x = fminf(fmaxf(g[k].x, -maxg), maxg);
      g[k].y = fminf(fmaxf(g[k].y, -maxg), maxg);
      g[k].z = fminf(fmaxf(g[k].z, -maxg), maxg);
      g[k].w = fminf(fmaxf(g[k].w, -maxg), maxg);
    }
    if (p.wd_mode == 1 && OPT != OPT_NONE) g[k] = f4_fma(wv[k], wd, g[k]);
    // decoupled decay for the non-Adam family (Adam/LAMB fold wd*w into their update below)
    if (p.wd_mode == 2 && (OPT == OPT_SGD || OPT == OPT_ROWWISE_ADAGRAD || OPT == OPT_ADAGRAD || OPT == OPT_LARS_SGD))
      wv[k] = f4_scale(wv[k], 1.f - lr * wd);
  }

  if (OPT == OPT_NONE) {
    float* gw = p.state1 + eoff;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = lane + k * 32;
      if (vi < nvec) {
        float4 o = *reinterpret_cast<float4*>(gw + vi * 4);
        *reinterpret_cast<float4*>(gw + vi * 4) = f4_add(o, g[k]);
      }
    }
    return;
  }

  if (OPT == OPT_SGD) {
#pragma unroll
    for (int k = 0; k < MAXV; ++k) wv[k] = f4_fma(g[k], -lr, wv[k]);
  } else if (OPT == OPT_ROWWISE_ADAGRAD) {
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) sq += f4_sq(g[k]);  // lanes beyond nvec hold zeros
    sq = warp_sum(sq) / (float) D;
    float st = PRE ? spre : ((lane == 0) ? p.state1[key] : 0.f);
    st = __shfl_sync(0xffffffffu, st, 0);
    const float ns = st + sq;
    if (lane == 0) p.state1[key] = ns;
    const float mult = lr / (sqrtf(ns) + eps);
#pragma unroll
    for (int k = 0; k < MAXV; ++k) wv[k] = f4_fma(g[k], -mult, wv[k]);
  } else if (OPT == OPT_ADAGRAD) {
    float* s = p.state1 + eoff;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = lane + k * 32;
      if (vi < nvec) {
        float4 sv = *reinterpret_cast<float4*>(s + vi * 4);
        sv.x += g[k].x * g[k].x; sv.y += g[k].y * g[k].y; sv.z += g[k].z * g[k].z; sv.w += g[k].w * g[k].w;
        *reinterpret_cast<float4*>(s + vi * 4) = sv;
        wv[k].x -= lr * g[k].x / (sqrtf(sv.x) + eps);
        wv[k].y -= lr * g[k].y / (sqrtf(sv.y) + eps);
        wv[k].z -= lr * g[k].z / (sqrtf(sv.z) + eps);
        wv[k].w -= lr * g[k].w / (sqrtf(sv.w) + eps);
      }
    }
  } else if (OPT == OPT_ADAM || OPT == OPT_PARTIAL_ROWWISE_ADAM || OPT == OPT_LAMB || OPT == OPT_PARTIAL_ROWWISE_LAMB) {
    const float b1 = p.hyper[HP_BETA1], b2 = p.hyper[HP_BETA2], step = p.hyper[HP_STEP];
    const float bc1 = 1.f - powf(b1, step), bc2 = 1.f - powf(b2, step);
    const bool ROWV = (OPT == OPT_PARTIAL_ROWWISE_ADAM || OPT == OPT_PARTIAL_ROWWISE_LAMB);
    const bool LAMB = (OPT == OPT_LAMB || OPT == OPT_PARTIAL_ROWWISE_LAMB);
    float* m = p.state1 + eoff;
    float vrow = 0.f;
    if (ROWV) {
      float sq = 0.f;
#pragma unroll
      for (int k = 0; k < MAXV; ++k) sq += f4_sq(g[k]);
      sq = warp_sum(sq) / (float) D;
      float st = (lane == 0) ? p.state2[key] : 0.f;
      st = __shfl_sync(0xffffffffu, st, 0);
      vrow = b2 * st + (1.f - b2) * sq;
      if (lane == 0) p.state2[key] = vrow;
    }
    float4 upd[MAXV];
    float un = 0.f, wn = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = lane + k * 32;
      upd[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (vi < nvec) {
        float4 mv = *reinterpret_cast<float4*>(m + vi * 4);
        mv.x = b1 * mv.x + (1.f - b1) * g[k].x; mv.y = b1 * mv.y + (1.f - b1) * g[k].y;
        mv.z = b1 * mv.z + (1.f - b1) * g[k].z; mv.w = b1 * mv.w + (1.f - b1) * g[k].w;
        *reinterpret_cast<float4*>(m + vi * 4) = mv;
        float4 vv;
        if (ROWV) {
          vv = make_float4(vrow, vrow, vrow, vrow);
        } else {
          float* v = p.state2 + eoff;
          vv = *reinterpret_cast<float4*>(v + vi * 4);
          vv.x = b2 * vv.x + (1.f - b2) * g[k].x * g[k].x; vv.y = b2 * vv.y + (1.f - b2) * g[k].y * g[k].y;
          vv.z = b2 * vv.z + (1.f - b2) * g[k].z * g[k].z; vv.w = b2 * vv.w + (1.f - b2) * g[k].w * g[k].w;
          *reinterpret_cast<float4*>(v + vi * 4) = vv;
        }
        upd[k].x = (mv.x / bc1) / (sqrtf(vv.x / bc2) + eps);
        upd[k].y = (mv.y / bc1) / (sqrtf(vv.y / bc2) + eps);
        upd[k].z = (mv.z / bc1) / (sqrtf(vv.z / bc2) + eps);
        upd[k].w = (mv.w / bc1) / (sqrtf(vv.w / bc2) + eps);
        if (LAMB || p.wd_mode == 2) upd[k] = f4_fma(wv[k], wd, upd[k]);
        un += f4_sq(upd[k]);
        wn += f4_sq(wv[k]);
      }
    }
    float ratio = 1.f;
    if (LAMB) {
      un = sqrtf(warp_sum(un));
      wn = sqrtf(warp_sum(wn));
      ratio = (wn > 0.f && un > 0.f) ? wn / un : 1.f;
    }
#pragma unroll
    for (int k = 0; k < MAXV; ++k) wv[k] = f4_fma(upd[k], -lr * ratio, wv[k]);
  } else if (OPT == OPT_LION) {
    const float b1 = p.hyper[HP_BETA1], b2 = p.hyper[HP_BETA2];
    float* m = p.state1 + eoff;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = lane + k * 32;
      if (vi < nvec) {
        float4 mv = *reinterpret_cast<float4*>(m + vi * 4);
        float4 c = make_float4(b1 * mv.x + (1.f - b1) * g[k].x, b1 * mv.y + (1.f - b1) * g[k].y, b1 * mv.z + (1.f - b1) * g[k].z, b1 * mv.w + (1.f - b1) * g[k].w);
        float4 u = make_float4((c.x > 0.f) - (c.x < 0.f), (c.y > 0.f) - (c.y < 0.f), (c.z > 0.f) - (c.z < 0.f), (c.w > 0.f) - (c.w < 0.f));
        if (p.wd_mode == 2) u = f4_fma(wv[k], wd, u);
        wv[k] = f4_fma(u, -lr, wv[k]);
        mv.x = b2 * mv.x + (1.f - b2) * g[k].x; mv.y = b2 * mv.y + (1.f - b2) * g[k].y;
        mv.z = b2 * mv.z + (1.f - b2) * g[k].z; mv.w = b2 * mv.w + (1.f - b2) * g[k].w;
        *reinterpret_cast<float4*>(m + vi * 4) = mv;
      }
    }
  } else if (OPT == OPT_LARS_SGD) {
    float gn = 0.f, wn = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) { gn += f4_sq(g[k]); wn += f4_sq(wv[k]); }
    gn = sqrtf(warp_sum(gn));
    wn = sqrtf(warp_sum(wn));
    const float eta = p.hyper[HP_MOMENTUM] > 0.f ? p.hyper[HP_MOMENTUM] : 0.001f;
    const float ratio = (wn > 0.f && gn > 0.f) ? eta * wn / (gn + wd * wn + eps) : 1.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) wv[k] = f4_fma(g[k], -lr * ratio, wv[k]);
  }
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nvec) {
      if (sizeof(W) == 2 && p.sr) trb_store_row4_sr<W>(w + vi * 4, wv[k], trb_splitmix64(p.sr_seed ^ ((unsigned long long) key * 0xD1B54A32D192ED03ull) ^ (unsigned long long) vi));
      else Vec4<W>::st(w + vi * 4, wv[k]);
    }
  }
}

template <typename G, int MAXV>
__device__ __forceinline__ void load_grad_row(const TbeBwdParams& p, int bag, float scale, int lane, float4 (&acc)[MAXV]) {
  const int f = bag / p.B;
  const int b = bag - f * p.B;
  const int s = b / p.B_local;
  const int bl = b - s * p.B_local;
  const int nvec = p.feat_dim[f] >> 2;
  const G* src = reinterpret_cast<const G*>(p.grad.p[s]) + (int64_t) bl * p.grad_stride + p.feat_col[f];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nvec) acc[k] = f4_fma(Vec4<G>::ld(src + vi * 4), scale, acc[k]);
  }
}


// ---- unique-rows kernel ------------------------------------------------------------------------------------------------
// Handles the chunks whose 32 sorted keys are distinct valid rows that do not continue into the neighbouring chunks (the
// common case for large tables) when the optimizer is SGD / row-wise Adagrad without clipping or decay; marks them in
// chunk_done so the generic walk (tbe_bwd_chunk_kernel, lighter on registers, higher occupancy) skips them. Per-lane geometry
// is computed ONCE in parallel (the generic walk re-derives it per row with integer divisions on every lane) and rows are
// processed U at a time with all of their gradient / weight / state loads in flight together. The generic path alone was
// instruction- and latency-bound: one row in flight per warp.
template <typename W, typename G, int MAXV>
__global__ void __launch_bounds__(256) tbe_bwd_unique_kernel(const TbeBwdParams p) {
  typedef uint64_t K;
  const int lane = threadIdx.x & 31;
  const int64_t chunk = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t base = chunk << 5;
  if (base >= p.n) return;
  const int cnt = (int) min((int64_t) 32, p.n - base);
  const void* keys = p.keys_sorted;
  const K sentinel = (K) p.total_rows;
  const K key = lane < cnt ? ld_key(keys, base + lane, p.key64) : sentinel;
  const bool has_prev = base > 0, has_next = base + 32 < p.n;
  const K prev_key = has_prev ? ld_key(keys, base - 1, p.key64) : sentinel;
  const K next_key = has_next ? ld_key(keys, base + 32, p.key64) : sentinel;
  constexpr int U = MAXV == 1 ? 4 : 2;  // rows in flight per warp (register budget: U x MAXV x 2 float4)
  const K down = __shfl_down_sync(0xffffffffu, key, 1);
  const bool lane_ok = lane >= cnt || (key != sentinel && (lane == cnt - 1 || key != down));
  const K key0 = __shfl_sync(0xffffffffu, key, 0), keyl = __shfl_sync(0xffffffffu, key, cnt - 1);
  const int OPT = p.opt;
  if (!__all_sync(0xffffffffu, lane_ok) || (has_prev && prev_key == key0) || (has_next && next_key == keyl) || p.hyper[HP_MAXGRAD] > 0.f) {
    if (lane == 0) p.chunk_done[chunk] = 0;
    return;
  }
  int bag = 0;
  float scale = 0.f;
  if (lane < cnt) {
    const int val = p.vals_sorted[base + lane];
    bag = p.bag_of[val];
    scale = (p.src.psw ? p.src.psw[val] : 1.f) * p.grad_scale;
    if (p.mean) {
      const int64_t L = bag_len(p, bag);
      scale /= (float) (L > 0 ? L : 1);
    }
  }
  int64_t goff = 0, woff = 0;
  int src_rank = 0, nvec_l = 0;
  if (lane < cnt) {
    const int f = bag / p.B;
    const int b = bag - f * p.B;
    src_rank = b / p.B_local;
    const int D = p.feat_dim[f];
    nvec_l = D >> 2;
    goff = (int64_t) (b - src_rank * p.B_local) * p.grad_stride + p.feat_col[f];
    woff = p.feat_woff[f] + ((int64_t) key - p.feat_rowbase[f]) * D;
  }
  const float lr = p.hyper[HP_LR], eps = p.hyper[HP_EPS];
  W* const wbase = reinterpret_cast<W*>(p.weights);
  for (int j = 0; j < cnt; j += U) {
    float4 g[U][MAXV], wv[U][MAXV];
    float st[U];
    int64_t wo[U], ky[U];
    int nv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int e = min(j + u, cnt - 1);
      const int64_t go = __shfl_sync(0xffffffffu, goff, e);
      wo[u] = __shfl_sync(0xffffffffu, woff, e);
      ky[u] = (int64_t) __shfl_sync(0xffffffffu, key, e);
      nv[u] = __shfl_sync(0xffffffffu, nvec_l, e);
      const float sc = __shfl_sync(0xffffffffu, scale, e);
      const int sr = __shfl_sync(0xffffffffu, src_rank, e);
      const G* gp = reinterpret_cast<const G*>(p.grad.p[sr]) + go;
      const W* wp = wbase + wo[u];
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        g[u][k] = (vi < nv[u]) ? f4_scale(Vec4<G>::ld(gp + vi * 4), sc) : make_float4(0.f, 0.f, 0.f, 0.f);
        wv[u][k] = (vi < nv[u]) ? Vec4<W>::ld(wp + vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      st[u] = (OPT == OPT_ROWWISE_ADAGRAD) ? p.state1[ky[u]] : 0.f;  // same address on every lane: one broadcast transaction
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (j + u >= cnt) break;
      float mult = lr;
      if (OPT == OPT_ROWWISE_ADAGRAD) {
        float sq = 0.f;
#pragma unroll
        for (int k = 0; k < MAXV; ++k) sq += f4_sq(g[u][k]);
        sq = warp_sum(sq) / (float) (nv[u] << 2);
        const float ns = st[u] + sq;
        if (lane == 0) p.state1[ky[u]] = ns;
        mult = lr / (sqrtf(ns) + eps);
      }
      W* wp = wbase + wo[u];
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        if (vi < nv[u]) Vec4<W>::st(wp + vi * 4, f4_fma(g[u][k], -mult, wv[u][k]));
      }
    }
  }
  if (lane == 0) {
    p.chunk_done[chunk] = 1;
    p.span_flags[chunk] = 0;
  }
}

// ---- multi-row walk ---------------------------------------------------------------------------------------------------
// The generic walk below handles one run of equal keys at a time: gradient rows -> weight row -> row state -> store is ONE dependent
// chain per warp, and every lane re-derives the row geometry (two integer divisions) for every gradient row. For SGD / row-wise Adagrad without clipping
// or weight decay this kernel walks the same 32 sorted keys U entries at a time instead:
//   * geometry (gradient offset, weight offset, scale, source rank) is computed once, one entry per lane, and broadcast by shuffles;
//   * the U gradient rows AND the weight rows / row states of the runs that end inside the group are all requested before any of
//     them is consumed (U x (256 B + 512 B) in flight per warp instead of one row);
//   * runs (duplicates) are handled by carrying the accumulator across entries - run boundaries are a ballot mask, so every branch
//     is warp-uniform. Accumulation order and fma contraction are those of the generic walk: results are bit-identical.
// Runs that continue into a neighbouring chunk leave partial rows exactly like the generic walk (span kernels combine them).
// Chunks it handled are marked in chunk_done; the generic kernel returns immediately for those.
template <typename W, typename G, int MAXV, int MINB, int UU = 0>
__global__ void __launch_bounds__(256, MINB) tbe_bwd_walk_kernel(const TbeBwdParams p) {
  typedef uint64_t K;
  const int lane = threadIdx.x & 31;
  const int64_t chunk = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t base = chunk << 5;
  if (base >= p.n) return;
  if (p.hyper[HP_MAXGRAD] > 0.f) {  // gradient clipping: generic path
    if (lane == 0) p.chunk_done[chunk] = 0;
    return;
  }
  const int cnt = (int) min((int64_t) 32, p.n - base);
  const void* keys = p.keys_sorted;
  const K sentinel = (K) p.total_rows;
  const K key = lane < cnt ? ld_key(keys, base + lane, p.key64) : sentinel;
  const bool valid = key != sentinel;  // padding / invalid ids sort last: the valid entries are a prefix of the chunk
  const int cnt_v = __popc(__ballot_sync(0xffffffffu, valid));
  const bool has_prev = base > 0, has_next = base + 32 < p.n;
  const K prev_key = has_prev ? ld_key(keys, base - 1, p.key64) : sentinel;
  const K next_key = has_next ? ld_key(keys, base + 32, p.key64) : sentinel;
  if (cnt_v == 0) {
    if (lane == 0) {
      p.chunk_done[chunk] = 1;
      p.span_flags[chunk] = 0;
    }
    return;
  }
  const K down = __shfl_down_sync(0xffffffffu, key, 1);
  const unsigned ends = __ballot_sync(0xffffffffu, lane < cnt_v && (lane == cnt_v - 1 || key != down));
  const K key0 = __shfl_sync(0xffffffffu, key, 0), keyl = __shfl_sync(0xffffffffu, key, cnt_v - 1);
  const bool head_open = has_prev && prev_key == key0;
  const bool tail_open = cnt_v == cnt && has_next && next_key == keyl;
  const int e_first_end = __ffs(ends) - 1;

  float scale = 0.f;
  int64_t goff = 0, woff = 0;
  int src_rank = 0, nvec_l = 0;
  if (lane < cnt_v) {
    const int val = p.vals_sorted[base + lane];
    const int bag = p.bag_of[val];
    scale = (p.src.psw ? p.src.psw[val] : 1.f) * p.grad_scale;
    if (p.mean) {
      const int64_t L = bag_len(p, bag);
      scale /= (float) (L > 0 ? L : 1);
    }
    const int f = bag / p.B;
    const int b = bag - f * p.B;
    src_rank = b / p.B_local;
    const int D = p.feat_dim[f];
    nvec_l = D >> 2;
    goff = (int64_t) (b - src_rank * p.B_local) * p.grad_stride + p.feat_col[f];
    woff = p.feat_woff[f] + ((int64_t) key - p.feat_rowbase[f]) * D;
  }
  constexpr int U = UU > 0 ? UU : (MAXV == 1 ? 4 : (MAXV == 2 ? 2 : 1));  // entries in flight per warp (register budget: U x MAXV x 2 float4)
  const int OPT = p.opt;
  if ((p.prefetch & 4) && lane < cnt_v) {
    // every lane pulls the lines of ITS entry (weight row, row state, gradient row) towards L2 now: the U-wide groups below then
    // find them on chip, and the whole chunk (32 rows) is in flight per warp instead of U rows
    const char* pw = reinterpret_cast<const char*>(reinterpret_cast<const W*>(p.weights) + woff);
    const int wbytes = nvec_l * 4 * (int) sizeof(W);
    for (int o = 0; o < wbytes; o += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pw + o));
    if (OPT == OPT_ROWWISE_ADAGRAD) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.state1 + key));
    if (p.prefetch & 2) {
      const char* pg = reinterpret_cast<const char*>(reinterpret_cast<const G*>(p.grad.p[src_rank]) + goff);
      const int gbytes = nvec_l * 4 * (int) sizeof(G);
      for (int o = 0; o < gbytes; o += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pg + o));
    }
  }
  const float lr = p.hyper[HP_LR], eps = p.hyper[HP_EPS];
  W* const wbase = reinterpret_cast<W*>(p.weights);
  float4 acc[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  bool wrote_slot1 = false;
  for (int j = 0; j < cnt_v; j += U) {
    typename Vec4<G>::raw g[U][MAXV];  // raw registers: converted when consumed, so all loads of the group are issued first
    typename Vec4<W>::raw wv[U][MAXV];
    float st[U], sc[U];
    int64_t wo[U], ky[U];
    int nv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int e = min(j + u, cnt_v - 1);
      const int64_t go = __shfl_sync(0xffffffffu, goff, e);
      const int sr = __shfl_sync(0xffffffffu, src_rank, e);
      sc[u] = __shfl_sync(0xffffffffu, scale, e);
      nv[u] = __shfl_sync(0xffffffffu, nvec_l, e);
      const G* gp = reinterpret_cast<const G*>(p.grad.p[sr]) + go;
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        // unconditional load from a clamped address (a predicated load + select made every load wait for the previous one)
        g[u][k] = Vec4<G>::ld_raw(gp + ((vi < nv[u]) ? vi * 4 : 0));
      }
      const bool fin = j + u < cnt_v && ((ends >> e) & 1u) && !(head_open && e == e_first_end) && !(tail_open && e == cnt_v - 1);
      wo[u] = 0;
      ky[u] = 0;
      st[u] = 0.f;
      if (fin) {  // this entry closes a run that lives entirely inside the chunk: fetch its row now, consume it below
        wo[u] = __shfl_sync(0xffffffffu, woff, e);
        ky[u] = (int64_t) __shfl_sync(0xffffffffu, key, e);
        const W* wp = wbase + wo[u];
#pragma unroll
        for (int k = 0; k < MAXV; ++k) {
          const int vi = lane + k * 32;
          wv[u][k] = Vec4<W>::ld_raw(wp + ((vi < nv[u]) ? vi * 4 : 0));
        }
        if (OPT == OPT_ROWWISE_ADAGRAD && !(p.prefetch & 8)) st[u] = p.state1[ky[u]];  // same address on every lane: one broadcast transaction
      }
    }
    // Group of U DISTINCT rows that all live inside the chunk (the common case for large tables): the U updates are independent, so
    // their square-sum reductions, square roots and divisions are interleaved instead of running as U dependent chains back to back
    // (with one warp per scheduler-slot nothing else hides that latency). Same arithmetic, same order per row as the sequential path below: bit-identical results.
    if constexpr (U > 1) {
      constexpr unsigned kAll = (1u << U) - 1u;
      const bool distinct = j + U <= cnt_v && ((ends >> j) & kAll) == kAll && (j == 0 || ((ends >> (j - 1)) & 1u)) &&
                            !(head_open && e_first_end >= j && e_first_end < j + U) && !(tail_open && cnt_v - 1 < j + U);
      if (distinct) {
        float4 a[U][MAXV];
        float sq[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          sq[u] = 0.f;
#pragma unroll
          for (int k = 0; k < MAXV; ++k) {
            a[u][k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (lane + k * 32 < nv[u]) a[u][k] = f4_fma(Vec4<G>::cvt(g[u][k]), sc[u], a[u][k]);
            sq[u] += f4_sq(a[u][k]);
          }
        }
        float mult[U];
        if (OPT == OPT_ROWWISE_ADAGRAD) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int u = 0; u < U; ++u) sq[u] += __shfl_xor_sync(0xffffffffu, sq[u], o);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const float ns = st[u] + sq[u] / (float) (nv[u] << 2);
            if (lane == 0 && !(p.prefetch & 8)) p.state1[ky[u]] = ns;
            mult[u] = lr / (sqrtf(ns) + eps);
          }
        } else {
#pragma unroll
          for (int u = 0; u < U; ++u) mult[u] = lr;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          W* wp = wbase + wo[u];
#pragma unroll
          for (int k = 0; k < MAXV; ++k) {
            const int vi = lane + k * 32;
            if (vi < nv[u]) Vec4<W>::st(wp + vi * 4, f4_fma(a[u][k], -mult[u], Vec4<W>::cvt(wv[u][k])));
          }
        }
        continue;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int e = j + u;
      if (e >= cnt_v) break;
#pragma unroll
      for (int k = 0; k < MAXV; ++k)
        if (lane + k * 32 < nv[u]) acc[k] = f4_fma(Vec4<G>::cvt(g[u][k]), sc[u], acc[k]);
      if (!((ends >> e) & 1u)) continue;
      const bool head_p = head_open && e == e_first_end, tail_p = tail_open && e == cnt_v - 1;
      if (!head_p && !tail_p) {
        float mult = lr;
        if (OPT == OPT_ROWWISE_ADAGRAD) {
          float sq = 0.f;
#pragma unroll
          for (int k = 0; k < MAXV; ++k) sq += f4_sq(acc[k]);
          sq = warp_sum(sq) / (float) (nv[u] << 2);
          const float ns = st[u] + sq;
          if (lane == 0 && !(p.prefetch & 8)) p.state1[ky[u]] = ns;
          mult = lr / (sqrtf(ns) + eps);
        }
        W* wp = wbase + wo[u];
#pragma unroll
        for (int k = 0; k < MAXV; ++k) {
          const int vi = lane + k * 32;
          if (vi < nv[u]) Vec4<W>::st(wp + vi * 4, f4_fma(acc[k], -mult, Vec4<W>::cvt(wv[u][k])));
        }
      } else {
        const int slot = head_p ? 0 : 1;
        if (!head_p) wrote_slot1 = true;
        float* dst = p.partials + ((chunk * 2 + slot) * (int64_t) p.max_dim);
#pragma unroll
        for (int k = 0; k < MAXV; ++k) {
          const int vi = lane + k * 32;
          if (vi < nv[u]) *reinterpret_cast<float4*>(dst + vi * 4) = acc[k];
        }
      }
#pragma unroll
      for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  if (lane == 0) {
    p.chunk_done[chunk] = 1;
    p.span_flags[chunk] = wrote_slot1 ? 1 : 0;
  }
}

template <typename W, typename G, int MAXV>
__global__ void __launch_bounds__(256) tbe_bwd_chunk_kernel(const TbeBwdParams p) {
  typedef uint64_t K;
  const int lane = threadIdx.x & 31;
  const int64_t chunk = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t base = chunk << 5;
  if (base >= p.n) return;
  if (p.chunk_done != nullptr && p.chunk_done[chunk]) return;  // already handled by tbe_bwd_walk_kernel / tbe_bwd_unique_kernel
  const int cnt = (int) min((int64_t) 32, p.n - base);
  const void* keys = p.keys_sorted;
  const K sentinel = (K) p.total_rows;
  const K key = lane < cnt ? ld_key(keys, base + lane, p.key64) : sentinel;
  const int val = lane < cnt ? p.vals_sorted[base + lane] : 0;
  int bag = 0;
  float scale = 0.f;
  if (lane < cnt && key != sentinel) {
    bag = p.bag_of[val];
    scale = (p.src.psw ? p.src.psw[val] : 1.f) * p.grad_scale;
    if (p.mean) {
      const int64_t L = bag_len(p, bag);
      scale /= (float) (L > 0 ? L : 1);
    }
  }
  const bool has_prev = base > 0, has_next = base + 32 < p.n;
  const K prev_key = has_prev ? ld_key(keys, base - 1, p.key64) : sentinel;
  const K next_key = has_next ? ld_key(keys, base + 32, p.key64) : sentinel;
  const K up = __shfl_up_sync(0xffffffffu, key, 1);
  const bool is_start = (lane == 0) || (key != up);
  unsigned starts = __ballot_sync(0xffffffffu, lane < cnt && is_start);
  // The walk below is one dependent chain per run (gradient rows -> weight row -> optimizer state -> store): ~3 DRAM round
  // trips per row with a single row in flight per warp made this kernel latency bound. Every lane therefore
  // software-prefetches the lines of ITS key (weight row, gradient row, row state) into L2 a few runs before the walk reaches
  // it, so the chain hits L2 (~250 cycles) instead of HBM. kPrefetchAhead keys in flight per warp keeps the footprint small.
  constexpr int kPrefetchAhead = 6;
  const char* pf_w = nullptr;
  const char* pf_g = nullptr;
  const char* pf_s = nullptr;
  int pf_wbytes = 0, pf_gbytes = 0;
  if (p.prefetch && lane < cnt && key != sentinel) {
    const int pf = bag / p.B;
    const int pb = bag - pf * p.B;
    const int ps = pb / p.B_local;
    const int pD = p.feat_dim[pf];
    pf_w = reinterpret_cast<const char*>(reinterpret_cast<const W*>(p.weights) + p.feat_woff[pf] + ((int64_t) key - p.feat_rowbase[pf]) * pD);
    pf_wbytes = p.opt == OPT_NONE ? 0 : pD * (int) sizeof(W);
    pf_g = reinterpret_cast<const char*>(reinterpret_cast<const G*>(p.grad.p[ps]) + (int64_t) (pb - ps * p.B_local) * p.grad_stride + p.feat_col[pf]);
    pf_gbytes = (p.prefetch & 2) ? pD * (int) sizeof(G) : 0;
    if (p.opt == OPT_ROWWISE_ADAGRAD) pf_s = reinterpret_cast<const char*>(p.state1 + key);
  }
  auto prefetch_mine = [&]() {
    for (int o = 0; o < pf_wbytes; o += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf_w + o));
    for (int o = 0; o < pf_gbytes; o += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf_g + o));
    if (pf_s != nullptr) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf_s));
  };
  int pf_upto = kPrefetchAhead < cnt ? kPrefetchAhead : cnt;
  if (lane < pf_upto && pf_w != nullptr) prefetch_mine();
  bool wrote_slot1 = false;
  while (starts) {
    const int a = __ffs(starts) - 1;
    starts &= starts - 1;
    const int bnd = starts ? (__ffs(starts) - 1) : cnt;
    {
      const int upto = (bnd + kPrefetchAhead) < cnt ? (bnd + kPrefetchAhead) : cnt;
      if (lane >= pf_upto && lane < upto && pf_w != nullptr) prefetch_mine();
      pf_upto = upto > pf_upto ? upto : pf_upto;
    }
    const K rk = __shfl_sync(0xffffffffu, key, a);
    if (rk == sentinel) break;  // padding / invalid ids sort last
    const int f = __shfl_sync(0xffffffffu, bag, a) / p.B;
    const bool head_open = (a == 0) && has_prev && (rk == prev_key);
    const bool tail_open = (bnd == cnt) && has_next && (rk == next_key);
    // (the weight row / row state are loaded after the gradient gather: with the L2 prefetch above the in-order loads of apply_row
    // already hit L2, and loading them here costs registers.)
    float4 acc[MAXV];
#pragma unroll
    for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int e = a; e < bnd; ++e) {
      const int ebag = __shfl_sync(0xffffffffu, bag, e);
      const float esc = __shfl_sync(0xffffffffu, scale, e);
      load_grad_row<G, MAXV>(p, ebag, esc, lane, acc);
    }
    if (!head_open && !tail_open) {
      apply_row<W, MAXV>(p, (int64_t) rk, f, acc, lane);
    } else {
      const int slot = head_open ? 0 : 1;
      if (!head_open) wrote_slot1 = true;
      float* dst = p.partials + ((chunk * 2 + slot) * (int64_t) p.max_dim);
      const int nvec = p.feat_dim[f] >> 2;
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        if (vi < nvec) *reinterpret_cast<float4*>(dst + vi * 4) = acc[k];
      }
    }
  }
  if (lane == 0) p.span_flags[chunk] = wrote_slot1 ? 1 : 0;
}

// One CTA per run that crosses chunk boundaries. blockDim = 256 (8 warps).
// ---- span combine ------------------------------------------------------------------------------------------------------
// A run of equal keys that crosses chunk boundaries left one partial row per chunk: slot 1 of its first chunk (flagged), slot 0
// of every following chunk. One WARP per flagged chunk sums the pieces and applies the optimizer (short spans are the common
// case: mid-size tables); spans longer than kLongSpan pieces (hot rows of tiny tables) are deferred to a worklist processed by
// whole blocks in tbe_bwd_span_long_kernel. (One 256-thread block per chunk would launch mostly-empty blocks; a compact grid would
// serialise neighbouring spans inside one block.)
constexpr int kLongSpan = 24;

template <int MAXV>
__device__ __forceinline__ void span_accumulate(const TbeBwdParams& p, int64_t c, int64_t j0, int64_t n_pieces, int64_t stride, int nvec, int lane, float4 (&acc)[MAXV]) {
  int64_t j = j0;
  for (; j + 3 * stride < n_pieces; j += 4 * stride) {
    float4 t[4][MAXV];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int64_t jj = j + q * stride;
      const float* src = p.partials + (((c + jj) * 2 + (jj == 0 ? 1 : 0)) * (int64_t) p.max_dim);
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        t[q][k] = *reinterpret_cast<const float4*>(src + ((vi < nvec) ? vi * 4 : 0));  // unconditional: all 4 pieces in flight
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int k = 0; k < MAXV; ++k)
        if (lane + k * 32 < nvec) acc[k] = f4_add(acc[k], t[q][k]);
  }
  for (; j < n_pieces; j += stride) {
    const float* src = p.partials + (((c + j) * 2 + (j == 0 ? 1 : 0)) * (int64_t) p.max_dim);
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = lane + k * 32;
      if (vi < nvec) acc[k] = f4_add(acc[k], *reinterpret_cast<const float4*>(src + vi * 4));
    }
  }
}

// Last chunk of the run of equal keys that leaves chunk c through its last entry. Called by whole warps: a 32-ary search (every lane
// probes one point per step, 4 steps over 1 M keys) instead of a 20-step binary search of dependent loads - the search was most of
// the latency of the span kernels.
__device__ __forceinline__ int64_t span_last_chunk(const TbeBwdParams& p, int64_t c, uint64_t* rk_out) {
  const int lane = threadIdx.x & 31;
  const int64_t last = c * 32 + 31;
  const uint64_t rk = ld_key(p.keys_sorted, last, p.key64);
  // invariant: keys[i] <= rk for i < lo, keys[i] > rk for i >= hi; result = upper bound of rk
  int64_t lo = last + 1, hi = p.n;
  while (hi - lo > 32) {
    const int64_t step = (hi - lo) >> 5;
    const int64_t pos = lo + step * (lane + 1) - 1;  // < hi
    const bool le = ld_key(p.keys_sorted, pos, p.key64) <= rk;
    const int cnt = __popc(__ballot_sync(0xffffffffu, le));  // keys are sorted: the predicate is a prefix of the lanes
    const int64_t nlo = cnt > 0 ? lo + step * cnt : lo;
    if (cnt < 32) hi = lo + step * (cnt + 1) - 1;
    lo = nlo;
  }
  {
    const int64_t pos = lo + lane;
    const bool le = pos < hi && ld_key(p.keys_sorted, pos, p.key64) <= rk;
    lo += __popc(__ballot_sync(0xffffffffu, le));
  }
  *rk_out = rk;
  return (lo - 1) >> 5;
}

template <typename W, int MAXV>
__global__ void __launch_bounds__(256) tbe_bwd_span_kernel(const TbeBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t c = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (c >= (p.n + 31) / 32 || !p.span_flags[c]) return;
  uint64_t rk;
  const int64_t c_end = span_last_chunk(p, c, &rk);
  const int64_t n_pieces = c_end - c + 1;
  if (n_pieces > kLongSpan) {
    if (lane == 0) p.long_list[atomicAdd(p.long_count, 1)] = (int32_t) c;
    return;
  }
  const int f = p.bag_of[p.vals_sorted[c * 32 + 31]] / p.B;
  const int nvec = p.feat_dim[f] >> 2;
  float4 acc[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  span_accumulate<MAXV>(p, c, 0, n_pieces, 1, nvec, lane, acc);
  apply_row<W, MAXV>(p, (int64_t) rk, f, acc, lane);
}

// kLongWarps warps per long span: at 8 GPUs the global batch makes the hot rows of the tiny tables 8x longer (a 3-row table: 87 k entries
// per row = 2730 partial rows), and this kernel runs at the very end of the step.
constexpr int kLongWarps = 32;

template <typename W, int MAXV>
__global__ void __launch_bounds__(kLongWarps * 32) tbe_bwd_span_long_kernel(const TbeBwdParams p) {
  extern __shared__ float smem[];  // [kLongWarps][max_dim]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_long = *p.long_count;
  for (int wi = blockIdx.x; wi < n_long; wi += gridDim.x) {
    const int64_t c = p.long_list[wi];
    uint64_t rk;
    const int64_t c_end = span_last_chunk(p, c, &rk);
    const int f = p.bag_of[p.vals_sorted[c * 32 + 31]] / p.B;
    const int nvec = p.feat_dim[f] >> 2;
    float4 acc[MAXV];
#pragma unroll
    for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    span_accumulate<MAXV>(p, c, warp, c_end - c + 1, kLongWarps, nvec, lane, acc);
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = lane + k * 32;
      if (vi < nvec) *reinterpret_cast<float4*>(smem + warp * p.max_dim + vi * 4) = acc[k];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (vi < nvec)
          for (int w8 = 0; w8 < kLongWarps; ++w8) s4 = f4_add(s4, *reinterpret_cast<const float4*>(smem + w8 * p.max_dim + vi * 4));
        acc[k] = s4;
      }
      apply_row<W, MAXV>(p, (int64_t) rk, f, acc, lane);
    }
    __syncthreads();
  }
}


static inline int bits_needed(int64_t v) {
  int b = 1;
  while (b < 64 && ((int64_t) 1 << b) <= v) ++b;
  return b;
}

template <typename K>
static size_t sort_temp_bytes(int64_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const K*) nullptr, (K*) nullptr, (const int32_t*) nullptr,
                                  (int32_t*) nullptr, n);
  return bytes;
}

static inline size_t align_up(size_t x) { return (x + 255) & ~(size_t) 255; }

struct BwdLayout {
  size_t keys, keys_sorted, vals, vals_sorted, bag_of, partials, flags, done, long_list, long_count, sort_tmp, total;
};

static BwdLayout bwd_layout(int64_t n, int max_dim, int key64) {
  BwdLayout L;
  const size_t ksz = key64 ? 8 : 4;
  const int64_t chunks = (n + 31) / 32;
  size_t o = 0;
  L.keys = o; o += align_up(n * ksz);
  L.keys_sorted = o; o += align_up(n * ksz);
  L.vals = o; o += align_up(n * 4);
  L.vals_sorted = o; o += align_up(n * 4);
  L.bag_of = o; o += align_up(n * 4);
  L.partials = o; o += align_up((size_t) chunks * 2 * max_dim * 4);
  L.flags = o; o += align_up(chunks);
  L.done = o; o += align_up(chunks);
  L.long_list = o; o += align_up((size_t) chunks * 4);
  L.long_count = o; o += align_up(16);
  L.sort_tmp = o;
  o += align_up(key64 ? sort_temp_bytes<uint64_t>(n) : sort_temp_bytes<uint32_t>(n));
  L.total = o;
  return L;
}

TRB_API int64_t trb_tbe_bwd_workspace_bytes(int64_t n, int max_dim, int64_t total_rows) {
  const int key64 = total_rows >= ((int64_t) 1 << 32) - 1;
  return (int64_t) bwd_layout(n > 0 ? n : 1, max_dim, key64).total;
}

template <typename W, typename G, int MAXV>
static int run_bwd(TbeBwdParams& p, char* ws, cudaStream_t stream) {
  const int key64 = p.key64;
  BwdLayout L = bwd_layout(p.n, p.max_dim, key64);
  p.keys = ws + L.keys;
  p.keys_sorted = ws + L.keys_sorted;
  p.vals = (int32_t*) (ws + L.vals);
  p.vals_sorted = (int32_t*) (ws + L.vals_sorted);
  p.bag_of = (int32_t*) (ws + L.bag_of);
  p.partials = (float*) (ws + L.partials);
  p.span_flags = (uint8_t*) (ws + L.flags);
  p.chunk_done = nullptr;
  p.long_list = (int32_t*) (ws + L.long_list);
  p.long_count = (int32_t*) (ws + L.long_count);
  const int threads = 256;
  if (p.phase != 2) {
    tbe_bwd_build_keys<<<(unsigned) ((p.n + threads - 1) / threads), threads, 0, stream>>>(p);
    TRB_CHECK_LAUNCH();
    size_t tmp_bytes = L.total - L.sort_tmp;
    const int end_bit = bits_needed(p.total_rows);
    if (key64) {
      TRB_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.sort_tmp, tmp_bytes, (const uint64_t*) p.keys,
                                               (uint64_t*) p.keys_sorted, (const int32_t*) p.vals, p.vals_sorted, p.n, 0,
                                               end_bit, stream));
    } else {
      TRB_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.sort_tmp, tmp_bytes, (const uint32_t*) p.keys,
                                               (uint32_t*) p.keys_sorted, (const int32_t*) p.vals, p.vals_sorted, p.n, 0,
                                               end_bit, stream));
    }
    g_trb_launches += 4;  // radix sort passes (library kernels, counted approximately)
  }
  if (p.phase == 1) return 0;
  const int64_t chunks = (p.n + 31) / 32;
  const int64_t blocks = (chunks + 7) / 8;
  // pass 1 (optional): chunks of distinct rows with a simple optimizer go through the high-MLP unique kernel
  static const int fast_enabled = getenv("TRB_BWD_UNIQUE") ? atoi(getenv("TRB_BWD_UNIQUE")) : 0;  // opt-in
  static const int walk_enabled = getenv("TRB_BWD_WALK") ? atoi(getenv("TRB_BWD_WALK")) : 1;
  const bool simple_opt = (p.opt == OPT_SGD || p.opt == OPT_ROWWISE_ADAGRAD) && p.wd_mode == 0 && !(sizeof(W) == 2 && p.sr);
  if constexpr (MAXV <= 4) {
    if (walk_enabled && simple_opt) {
      p.chunk_done = (uint8_t*) (ws + L.done);
      // entries in flight per warp vs CTAs per SM. One H100, 4 tables x 262144 distinct ids (tools/kernel_bench.py): =1 775 us,
      // =2 732 us, =3 814 us; =1 stays the default until the choice is re-measured on the whole step.
      // TRB_BWD_WALK=1 (default): D <= 128 -> 2 entries / 4 CTAs per SM; =3: 4 entries / 3 CTAs; =2: 4 entries / 2 CTAs
      if (walk_enabled == 2) tbe_bwd_walk_kernel<W, G, MAXV, 2><<<(unsigned) blocks, threads, 0, stream>>>(p);
      else if (walk_enabled == 3 && MAXV == 1) tbe_bwd_walk_kernel<W, G, MAXV, 3, 4><<<(unsigned) blocks, threads, 0, stream>>>(p);   // 4 entries in flight, 3 CTAs / SM
      else if (MAXV == 1) tbe_bwd_walk_kernel<W, G, MAXV, 4, 2><<<(unsigned) blocks, threads, 0, stream>>>(p);   // default: 2 entries in flight, 4 CTAs / SM
      else tbe_bwd_walk_kernel<W, G, MAXV, 3><<<(unsigned) blocks, threads, 0, stream>>>(p);
      TRB_CHECK_LAUNCH();
    } else if (fast_enabled && simple_opt) {
      p.chunk_done = (uint8_t*) (ws + L.done);
      tbe_bwd_unique_kernel<W, G, MAXV><<<(unsigned) blocks, threads, 0, stream>>>(p);
      TRB_CHECK_LAUNCH();
    }
  }
  // pass 2: generic run walk over the remaining chunks (duplicates, runs spanning chunks, other optimizers)
  tbe_bwd_chunk_kernel<W, G, MAXV><<<(unsigned) blocks, threads, 0, stream>>>(p);
  TRB_CHECK_LAUNCH();
  // pass 3: combine runs that span chunks (warp per flagged chunk), then the few long spans with whole blocks
  tbe_bwd_span_kernel<W, MAXV><<<(unsigned) blocks, threads, 0, stream>>>(p);
  TRB_CHECK_LAUNCH();
  const size_t smem = (size_t) kLongWarps * p.max_dim * sizeof(float);
  if (smem > 48 * 1024)
    TRB_CUDA(cudaFuncSetAttribute(tbe_bwd_span_long_kernel<W, MAXV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
  tbe_bwd_span_long_kernel<W, MAXV><<<trb_num_sms(), kLongWarps * 32, smem, stream>>>(p);
  TRB_CHECK_LAUNCH();
  return 0;
}

template <typename W, typename G>
static int dispatch_dim(TbeBwdParams& p, char* ws, cudaStream_t stream) {
  const int nvec = p.max_dim / 4;
  if (nvec <= 32) return run_bwd<W, G, 1>(p, ws, stream);
  if (nvec <= 128) return run_bwd<W, G, 4>(p, ws, stream);
  if (nvec <= 512) return run_bwd<W, G, 16>(p, ws, stream);
  return -2;
}

TRB_API int trb_tbe_bwd_fused_phase(void* weights, int w_dtype, float* state1, float* state2, const float* hyper, int opt,
                                    int wd_mode, const int64_t* feat_woff, const int64_t* feat_rows,
                                    const int64_t* feat_rowbase, const int32_t* feat_dim, const int32_t* feat_col,
                                    const void* indices, int idx64, const void* offsets, int off64, const float* psw,
                                    int n_src, int64_t idx_stride, int64_t off_stride,
                                    void* const* grad_ptrs, int n_grad, int grad_dtype, int64_t grad_stride, float grad_scale, int64_t n,
                                    int64_t total_rows, int B, int B_local, int F, int max_dim, int mean, void* workspace,
                                    int stochastic_rounding, unsigned long long sr_seed, int phase, cudaStream_t stream);

// Fused backward + optimizer. `workspace` must hold trb_tbe_bwd_workspace_bytes(n, max_dim, total_rows).
// `n` = number of id POSITIONS to scan (capacity of `indices`; with n_src > 1 it must equal n_src * idx_stride).
TRB_API int trb_tbe_bwd_fused_ms(void* weights, int w_dtype, float* state1, float* state2, const float* hyper, int opt,
                                 int wd_mode, const int64_t* feat_woff, const int64_t* feat_rows,
                                 const int64_t* feat_rowbase, const int32_t* feat_dim, const int32_t* feat_col,
                                 const void* indices, int idx64, const void* offsets, int off64, const float* psw,
                                 int n_src, int64_t idx_stride, int64_t off_stride,
                                 void* const* grad_ptrs, int n_grad, int grad_dtype, int64_t grad_stride, float grad_scale, int64_t n,
                                 int64_t total_rows, int B, int B_local, int F, int max_dim, int mean, void* workspace,
                                 int stochastic_rounding, unsigned long long sr_seed, cudaStream_t stream) {
  return trb_tbe_bwd_fused_phase(weights, w_dtype, state1, state2, hyper, opt, wd_mode, feat_woff, feat_rows, feat_rowbase, feat_dim, feat_col, indices, idx64,
                                 offsets, off64, psw, n_src, idx_stride, off_stride, grad_ptrs, n_grad, grad_dtype, grad_stride, grad_scale, n, total_rows, B,
                                 B_local, F, max_dim, mean, workspace, stochastic_rounding, sr_seed, 0, stream);
}

// phase 1 = prepare (keys + radix sort; needs only the ids: run it as soon as the ids exist, off the critical path);
// phase 2 = apply (run walk + optimizer; needs the gradient and the workspace filled by phase 1); phase 0 = both.
TRB_API int trb_tbe_bwd_fused_phase(void* weights, int w_dtype, float* state1, float* state2, const float* hyper, int opt,
                                    int wd_mode, const int64_t* feat_woff, const int64_t* feat_rows,
                                    const int64_t* feat_rowbase, const int32_t* feat_dim, const int32_t* feat_col,
                                    const void* indices, int idx64, const void* offsets, int off64, const float* psw,
                                    int n_src, int64_t idx_stride, int64_t off_stride,
                                    void* const* grad_ptrs, int n_grad, int grad_dtype, int64_t grad_stride, float grad_scale, int64_t n,
                                    int64_t total_rows, int B, int B_local, int F, int max_dim, int mean, void* workspace,
                                    int stochastic_rounding, unsigned long long sr_seed, int phase, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n_grad < 1 || n_grad > TRB_MAX_PEERS) return -1;
  if ((int64_t) B_local * n_grad != B) return -4;
  if (n_src < 1 || B % n_src != 0) return -4;
  if (n_src > 1 && n != (int64_t) n_src * idx_stride) return -4;
  if (phase < 0 || phase > 2) return -8;
  TbeBwdParams p;
  p.phase = phase;
  p.weights = weights;
  p.state1 = state1;
  p.state2 = state2;
  p.hyper = hyper;
  p.feat_woff = feat_woff;
  p.feat_rows = feat_rows;
  p.feat_rowbase = feat_rowbase;
  p.feat_dim = feat_dim;
  p.feat_col = feat_col;
  p.src.indices = indices;
  p.src.offsets = offsets;
  p.src.psw = psw;
  p.src.idx_stride = idx_stride;
  p.src.off_stride = off_stride;
  p.src.n_src = n_src;
  p.src.src_B = B / n_src;
  p.src.idx64 = idx64;
  p.src.off64 = off64;
  for (int i = 0; i < TRB_MAX_PEERS; ++i) p.grad.p[i] = i < n_grad ? grad_ptrs[i] : nullptr;
  p.grad_stride = grad_stride;
  p.grad_scale = grad_scale;
  p.n = n;
  p.total_rows = total_rows;
  p.B = B;
  p.B_local = B_local;
  p.F = F;
  p.mean = mean;
  p.wd_mode = wd_mode;
  p.max_dim = max_dim;
  p.key64 = total_rows >= ((int64_t) 1 << 32) - 1;
  p.opt = opt;
  p.sr = stochastic_rounding ? 1 : 0;
  p.sr_seed = sr_seed;
  {
    static const int pf = getenv("TRB_BWD_PREFETCH") ? atoi(getenv("TRB_BWD_PREFETCH")) : 1;
    static const int wpf = getenv("TRB_BWD_WALK_PF") ? atoi(getenv("TRB_BWD_WALK_PF")) : 1;
    p.prefetch = pf ? (1 | (n_grad <= 1 ? 2 : 0)) : 0;  // peer-resident gradient rows bypass the local L2: do not prefetch them
    if (wpf) p.prefetch |= 4 | (wpf >= 2 && n_grad <= 1 ? 2 : 0);
    static const int nostate = getenv("TRB_BWD_DEBUG_NOSTATE") ? atoi(getenv("TRB_BWD_DEBUG_NOSTATE")) : 0;  // measurement aid: skip the row-state memory traffic
    if (nostate) p.prefetch |= 8;
  }
  if (opt < 0 || opt > OPT_LION) return -5;
  char* ws = reinterpret_cast<char*>(workspace);
#define TRB_BWD_CASE(WC, WT, GC, GT) \
  if (w_dtype == WC && grad_dtype == GC) return dispatch_dim<WT, GT>(p, ws, stream)
  TRB_BWD_CASE(TRB_F32, float, TRB_F32, float);
  TRB_BWD_CASE(TRB_F32, float, TRB_BF16, __nv_bfloat16);
  TRB_BWD_CASE(TRB_BF16, __nv_bfloat16, TRB_F32, float);
  TRB_BWD_CASE(TRB_BF16, __nv_bfloat16, TRB_BF16, __nv_bfloat16);
  TRB_BWD_CASE(TRB_F16, __half, TRB_F32, float);
#undef TRB_BWD_CASE
  return -3;
}

TRB_API int trb_tbe_bwd_fused_ex(void* weights, int w_dtype, float* state1, float* state2, const float* hyper, int opt,
                                 int wd_mode, const int64_t* feat_woff, const int64_t* feat_rows,
                                 const int64_t* feat_rowbase, const int32_t* feat_dim, const int32_t* feat_col,
                                 const void* indices, int idx64, const void* offsets, int off64, const float* psw,
                                 void* const* grad_ptrs, int n_grad, int grad_dtype, int64_t grad_stride, int64_t n,
                                 int64_t total_rows, int B, int B_local, int F, int max_dim, int mean, void* workspace,
                                 int stochastic_rounding, unsigned long long sr_seed, cudaStream_t stream) {
  return trb_tbe_bwd_fused_ms(weights, w_dtype, state1, state2, hyper, opt, wd_mode, feat_woff, feat_rows, feat_rowbase, feat_dim, feat_col, indices,
                              idx64, offsets, off64, psw, 1, 0, 0, grad_ptrs, n_grad, grad_dtype, grad_stride, 1.f, n, total_rows, B, B_local, F,
                              max_dim, mean, workspace, stochastic_rounding, sr_seed, stream);
}

TRB_API int trb_tbe_bwd_fused(void* weights, int w_dtype, float* state1, float* state2, const float* hyper, int opt,
                              int wd_mode, const int64_t* feat_woff, const int64_t* feat_rows,
                              const int64_t* feat_rowbase, const int32_t* feat_dim, const int32_t* feat_col,
                              const void* indices, int idx64, const void* offsets, int off64, const float* psw,
                              void* const* grad_ptrs, int n_grad, int grad_dtype, int64_t grad_stride, int64_t n,
                              int64_t total_rows, int B, int B_local, int F, int max_dim, int mean, void* workspace,
                              cudaStream_t stream) {
  return trb_tbe_bwd_fused_ex(weights, w_dtype, state1, state2, hyper, opt, wd_mode, feat_woff, feat_rows, feat_rowbase, feat_dim, feat_col, indices,
                              idx64, offsets, off64, psw, grad_ptrs, n_grad, grad_dtype, grad_stride, n, total_rows, B, B_local, F, max_dim, mean,
                              workspace, 0, 0ull, stream);
}
