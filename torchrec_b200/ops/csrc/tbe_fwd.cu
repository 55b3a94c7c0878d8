// Table-batched embedding forward kernels (sm_90a).
//
// One launch covers every feature of a table group: bag n = f * B + b gathers rows
// indices[offsets[n] : offsets[n+1]] of feature f's table, pools them (SUM / MEAN, optional
// per-sample weights) and writes D_f values to the *destination rank's* output buffer:
//
//     s  = b / B_local               (source rank of the sample, == destination of the result)
//     bl = b % B_local
//     out_ptrs.p[s] + bl * out_stride + feat_col[f]
//
// With one pointer (B_local == B) this is a plain local lookup. With W peer pointers (buffers
// mapped over NVLink) it is the fused "lookup + pooled all-to-all": pooled rows are stored
// straight into the owner's [B_local, sum(D)] tensor, so the pack / all_to_all / cat / column
// permute kernels of the reference path (comm_ops.py:1390-1577, cw_sharding.py:294-317) vanish
// and the NVLink transfer overlaps the gathers bag by bag.  The row-wise (reduce-scatter) flavour
// points out_ptrs at per-source staging slabs that a tiny reduce kernel sums afterwards.
//
// Parity: replaces fbgemm SplitTableBatchedEmbeddingBagsCodegen forward
// (reference call site torchrec/distributed/batched_embedding_kernel.py:3010-3058).
//
// FP8 wire (trb_tbe_pooled_fwd_fp8, instances with Q = true): the pooled row, rounded to the wire dtype O, is stored as
// e4m3 groups of R = 4 * q_lanes columns plus one fp32 scale per group (qcomm_fp8.cuh). The R / 4 lanes that hold a group's
// float4 vectors take its amax with a shuffle; there is no extra pass over the pooled rows.
#include "common.cuh"
#include "qcomm_fp8.cuh"

unsigned long long g_trb_launches = 0;
TRB_API unsigned long long trb_launch_count() { return g_trb_launches; }
TRB_API void trb_launch_count_add(unsigned long long n) { g_trb_launches += n; }

struct TbeFwdParams {
  const void* weights;           // flat table storage (dtype W)
  const int64_t* feat_woff;      // [F] element offset of feature f's table in `weights`
  const int64_t* feat_rows;      // [F] rows of feature f's table (bounds check)
  const int32_t* feat_dim;       // [F] embedding dim of feature f
  const int32_t* feat_col;       // [F] output column offset
  TrbSrcView src;                // ids: indices [sum L], offsets [F*B + 1], per-sample weights (or per-source regions)
  TrbPeerPtrs out;               // destination buffers (dtype O)
  int64_t out_stride;            // elements between consecutive rows of a destination
  int32_t B;                     // total batch seen by this lookup (W_src * B_local)
  int32_t B_local;               // rows per destination
  int32_t F;
  int32_t mean;                  // 1 = MEAN pooling
};

// FP8 wire (Q = true instances only, so the other instances keep their parameter block): `out` points at uint8 payload rows,
// `q_scale` at fp32 rows of one scale per group of 4 * q_lanes columns
struct TbeFwdQParams : TbeFwdParams {
  TrbPeerPtrs q_scale;
  int64_t q_scale_stride;
  int32_t q_lanes;
};

template <bool Q>
struct TbeFwdParamsOf {
  using type = TbeFwdParams;
};
template <>
struct TbeFwdParamsOf<true> {
  using type = TbeFwdQParams;
};

// FP8 store of the 4 values of output columns [c, c + 4) of row `bl` of destination `s`. Every lane of the q_lanes-lane group
// that holds the R columns must call it (`ok` false for lanes past the row): the group amax is a shuffle across them.
template <typename O>
__device__ __forceinline__ void fp8_wire_store(const TbeFwdQParams& p, int s, int bl, int c, float4 v, bool ok, unsigned mask) {
  v = trb_round_to<O>(v);
  float amax = ok ? trb_fp8_abs_max4(v) : 0.f;
  for (int o = p.q_lanes >> 1; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(mask, amax, o));
  if (!ok) return;
  const float scale = trb_fp8_scale(amax);
  uint8_t* q = reinterpret_cast<uint8_t*>(p.out.p[s]) + (int64_t) bl * p.out_stride + c;
  *reinterpret_cast<uint32_t*>(q) = trb_fp8_encode4(v, 1.f / scale);
  const int R = p.q_lanes * 4;
  if (c % R == 0) reinterpret_cast<float*>(p.q_scale.p[s])[(int64_t) bl * p.q_scale_stride + c / R] = scale;
}

template <typename W, typename O, int LPB, int MAXV, bool Q = false>
__global__ void __launch_bounds__(256) tbe_pooled_fwd_kernel(const typename TbeFwdParamsOf<Q>::type p) {
  constexpr int UNROLL = (MAXV <= 2) ? 4 : (MAXV <= 4 ? 2 : 1);
  const int lig = threadIdx.x % LPB;  // lane in group
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) / LPB;
  const int64_t n_bags = (int64_t) p.F * p.B;
  if (group >= n_bags) return;  // whole groups exit together; shuffles below use the group mask
  const unsigned gmask = (LPB == 32) ? 0xffffffffu : (((1u << LPB) - 1u) << ((threadIdx.x % 32) / LPB * LPB));

  const int f = (int) (group / p.B);
  const int b = (int) (group - (int64_t) f * p.B);
  const int D = p.feat_dim[f];
  const int nvec = D >> 2;
  const int64_t rows = p.feat_rows[f];
  const W* __restrict__ wbase = reinterpret_cast<const W*>(p.weights) + p.feat_woff[f];

  int64_t pos_base;
  const int64_t oi = trb_src_off_index(p.src, f, b, &pos_base);
  const int64_t start = pos_base + trb_ld_idx(p.src.offsets, oi, p.src.off64);
  const int64_t end = pos_base + trb_ld_idx(p.src.offsets, oi + 1, p.src.off64);

  float4 acc[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);

  for (int64_t l0 = start; l0 < end; l0 += LPB) {
    const int n = (int) min((int64_t) LPB, end - l0);
    int64_t my_idx = -1;
    float my_w = 0.f;
    if (lig < n) {
      my_idx = trb_ld_idx(p.src.indices, l0 + lig, p.src.idx64);
      my_w = p.src.psw ? p.src.psw[l0 + lig] : 1.f;
      if (my_idx < 0 || my_idx >= rows) { my_idx = 0; my_w = 0.f; }  // out-of-range ids contribute zero
    }
    for (int j = 0; j < n; j += UNROLL) {
      float4 v[UNROLL][MAXV];
      float w[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int src = min(j + u, n - 1);
        const int64_t idx = __shfl_sync(gmask, my_idx, src, LPB);
        w[u] = __shfl_sync(gmask, my_w, src, LPB);
        if (j + u >= n) w[u] = 0.f;
        const W* row = wbase + idx * D;
#pragma unroll
        for (int k = 0; k < MAXV; ++k) {
          const int vi = lig + k * LPB;
          v[u][k] = (vi < nvec) ? Vec4<W>::ld_nc(row + vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u)
#pragma unroll
        for (int k = 0; k < MAXV; ++k) acc[k] = f4_fma(v[u][k], w[u], acc[k]);
    }
  }
  if (p.mean && end > start) {
    const float inv = 1.f / (float) (end - start);
#pragma unroll
    for (int k = 0; k < MAXV; ++k) acc[k] = f4_scale(acc[k], inv);
  }
  const int s = b / p.B_local;
  const int bl = b - s * p.B_local;
  if constexpr (Q) {
    const int col = p.feat_col[f];
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = lig + k * LPB;
      fp8_wire_store<O>(p, s, bl, col + vi * 4, acc[k], vi < nvec, gmask);
    }
  } else {
    O* dst = reinterpret_cast<O*>(p.out.p[s]) + (int64_t) bl * p.out_stride + p.feat_col[f];
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = lig + k * LPB;
      if (vi < nvec) Vec4<O>::st(dst + vi * 4, acc[k]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Wide-row variant (D >= 128): one warp walks 32 consecutive bags of a feature. The ids of those
// bags are contiguous, so they are fetched with coalesced loads and the row gathers of up to U
// ids are issued back to back (U independent 512 B requests in flight per warp) before any of
// them is consumed — with one id per bag (Criteo) this is what hides the HBM latency.
// ------------------------------------------------------------------------------------------------
template <typename W, typename O, int MAXV, int U, bool Q = false>
__global__ void __launch_bounds__(256) tbe_pooled_fwd_chunk_kernel(const typename TbeFwdParamsOf<Q>::type p) {
  const int lane = threadIdx.x & 31;
  const int64_t chunk = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  // chunks never straddle a source region or a destination: they tile the finer of the two partitions of the batch
  const int part = min(p.src.src_B, p.B_local);
  const int cpp = (part + 31) >> 5;             // chunks per partition
  const int cpf = cpp * (p.B / part);           // chunks per feature
  if (chunk >= (int64_t) p.F * cpf) return;
  const int f = (int) (chunk / cpf);
  const int rc = (int) (chunk - (int64_t) f * cpf);
  const int pi = rc / cpp;
  const int b0l = (rc - pi * cpp) << 5;
  const int b0 = pi * part + b0l;
  const int nb = min(32, part - b0l);
  const int D = p.feat_dim[f];
  const int nvec = D >> 2;
  const int64_t rows = p.feat_rows[f];
  const W* __restrict__ wbase = reinterpret_cast<const W*>(p.weights) + p.feat_woff[f];
  const int col = p.feat_col[f];

  int64_t pos_base;
  const int64_t bag0 = trb_src_off_index(p.src, f, b0, &pos_base);
  const void* const ids = p.src.idx64 ? (const void*) (reinterpret_cast<const int64_t*>(p.src.indices) + pos_base)
                                      : (const void*) (reinterpret_cast<const int32_t*>(p.src.indices) + pos_base);
  const float* const psw = p.src.psw ? p.src.psw + pos_base : nullptr;
  const int64_t my_start = trb_ld_idx(p.src.offsets, bag0 + min(lane, nb), p.src.off64);
  int64_t my_end = __shfl_down_sync(0xffffffffu, my_start, 1);
  const int64_t last_end = trb_ld_idx(p.src.offsets, bag0 + nb, p.src.off64);
  if (lane >= nb - 1) my_end = last_end;
  const int64_t e_begin = __shfl_sync(0xffffffffu, my_start, 0);
  const int64_t e_end = last_end;

  // ---- fast path: every bag of the chunk holds exactly ONE id (one-hot features, e.g. Criteo) and the 32 samples go to
  // one destination rank: no bag bookkeeping at all, ~20 instructions per row instead of ~125 (the generic walk below is
  // instruction-bound)
  {
    const bool unit = lane >= nb || (my_end - my_start) == 1;
    const int s0 = b0 / p.B_local;
    if (__all_sync(0xffffffffu, unit) && (b0 + nb - 1) / p.B_local == s0 && rows <= 0x7fffffffLL) {
      int my_idx = 0;
      float my_w = 0.f;
      if (lane < nb) {
        const int64_t id = trb_ld_idx(ids, e_begin + lane, p.src.idx64);
        my_w = psw ? psw[e_begin + lane] : 1.f;
        if (id < 0 || id >= rows) my_w = 0.f; else my_idx = (int) id;
      }
      O* dst0 = reinterpret_cast<O*>(p.out.p[s0]) + (int64_t) (b0 - s0 * p.B_local) * p.out_stride + col;
      for (int j = 0; j < nb; j += U) {
        float4 v[U][MAXV];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int idx = __shfl_sync(0xffffffffu, my_idx, min(j + u, nb - 1));
          const W* row = wbase + (int64_t) idx * D;
#pragma unroll
          for (int k = 0; k < MAXV; ++k) {
            const int vi = lane + k * 32;
            v[u][k] = (vi < nvec) ? Vec4<W>::ld_nc(row + vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (j + u < nb) {
            const float w = __shfl_sync(0xffffffffu, my_w, j + u);
            if constexpr (Q) {
#pragma unroll
              for (int k = 0; k < MAXV; ++k) {
                const int vi = lane + k * 32;
                fp8_wire_store<O>(p, s0, b0 - s0 * p.B_local + j + u, col + vi * 4, f4_scale(v[u][k], w), vi < nvec, 0xffffffffu);
              }
            } else {
              O* dst = dst0 + (int64_t) (j + u) * p.out_stride;
#pragma unroll
              for (int k = 0; k < MAXV; ++k) {
                const int vi = lane + k * 32;
                if (vi < nvec) Vec4<O>::st(dst + vi * 4, f4_scale(v[u][k], w));
              }
            }
          }
        }
      }
      return;
    }
  }

  float4 acc[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  int cur = 0;
  int64_t cur_start = e_begin;
  int64_t cur_end = __shfl_sync(0xffffffffu, my_end, 0);

  auto flush = [&](int bag_in_chunk, int64_t L) {
    if (p.mean && L > 0) {
      const float inv = 1.f / (float) L;
#pragma unroll
      for (int k = 0; k < MAXV; ++k) acc[k] = f4_scale(acc[k], inv);
    }
    const int b = b0 + bag_in_chunk;
    const int s = b / p.B_local;
    const int bl = b - s * p.B_local;
    if constexpr (Q) {
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        fp8_wire_store<O>(p, s, bl, col + vi * 4, acc[k], vi < nvec, 0xffffffffu);
        acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else {
      O* dst = reinterpret_cast<O*>(p.out.p[s]) + (int64_t) bl * p.out_stride + col;
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        if (vi < nvec) Vec4<O>::st(dst + vi * 4, acc[k]);
        acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };

  for (int64_t e0 = e_begin; e0 < e_end; e0 += 32) {
    const int n = (int) min((int64_t) 32, e_end - e0);
    int64_t my_idx = 0;
    float my_w = 0.f;
    if (lane < n) {
      my_idx = trb_ld_idx(ids, e0 + lane, p.src.idx64);
      my_w = psw ? psw[e0 + lane] : 1.f;
      if (my_idx < 0 || my_idx >= rows) { my_idx = 0; my_w = 0.f; }
    }
    for (int j = 0; j < n; j += U) {
      float4 v[U][MAXV];
      float w[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int src = min(j + u, n - 1);
        const int64_t idx = __shfl_sync(0xffffffffu, my_idx, src);
        w[u] = __shfl_sync(0xffffffffu, my_w, src);
        const W* row = wbase + idx * D;
#pragma unroll
        for (int k = 0; k < MAXV; ++k) {
          const int vi = lane + k * 32;
          v[u][k] = (vi < nvec && j + u < n) ? Vec4<W>::ld_nc(row + vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (j + u < n) {
          const int64_t e = e0 + j + u;
          while (e >= cur_end) {  // warp-uniform: close finished (possibly empty) bags
            flush(cur, cur_end - cur_start);
            ++cur;
            cur_start = cur_end;
            cur_end = __shfl_sync(0xffffffffu, my_end, min(cur, 31));
          }
#pragma unroll
          for (int k = 0; k < MAXV; ++k) acc[k] = f4_fma(v[u][k], w[u], acc[k]);
        }
      }
    }
  }
  // close the open bag and any trailing empty bags
  while (cur < nb) {
    flush(cur, cur_end - cur_start);
    ++cur;
    cur_start = cur_end;
    cur_end = __shfl_sync(0xffffffffu, my_end, min(cur, 31));
  }
}

template <typename W, typename O, int MAXV, int U, bool Q>
static int launch_pooled_chunk(const typename TbeFwdParamsOf<Q>::type& p, cudaStream_t stream) {
  if (p.B == 0 || p.F == 0) return 0;
  const int part = p.src.src_B < p.B_local ? p.src.src_B : p.B_local;
  const int64_t chunks = (int64_t) p.F * ((part + 31) / 32) * (p.B / part);
  if (chunks == 0) return 0;
  const int threads = 256;
  const int64_t blocks = (chunks + 7) / 8;
  tbe_pooled_fwd_chunk_kernel<W, O, MAXV, U, Q><<<(unsigned) blocks, threads, 0, stream>>>(p);
  TRB_CHECK_LAUNCH();
  return 0;
}

template <typename W, typename O, int LPB, int MAXV, bool Q>
static int launch_pooled(const typename TbeFwdParamsOf<Q>::type& p, cudaStream_t stream) {
  const int64_t n_bags = (int64_t) p.F * p.B;
  if (n_bags == 0) return 0;
  const int threads = 256;
  const int64_t groups_per_block = threads / LPB;
  const int64_t blocks = (n_bags + groups_per_block - 1) / groups_per_block;
  tbe_pooled_fwd_kernel<W, O, LPB, MAXV, Q><<<(unsigned) blocks, threads, 0, stream>>>(p);
  TRB_CHECK_LAUNCH();
  return 0;
}

template <typename W, typename O, bool Q = false>
static int dispatch_shape(const typename TbeFwdParamsOf<Q>::type& p, int max_dim, cudaStream_t stream) {
  const int nvec = max_dim / 4;
  if constexpr (Q) {
    if (p.q_lanes > (nvec <= 8 ? 8 : nvec <= 16 ? 16 : 32)) return -5;  // an FP8 group must lie inside the lanes of one row
  }
  if (nvec <= 8) return launch_pooled<W, O, 8, 1, Q>(p, stream);
  if (nvec <= 16) return launch_pooled<W, O, 16, 1, Q>(p, stream);
  if (nvec <= 32) return launch_pooled_chunk<W, O, 1, 8, Q>(p, stream);
  if (nvec <= 64) return launch_pooled_chunk<W, O, 2, 4, Q>(p, stream);
  if (nvec <= 128) return launch_pooled_chunk<W, O, 4, 2, Q>(p, stream);
  if (nvec <= 512) return launch_pooled<W, O, 32, 16, Q>(p, stream);
  return -2;  // dim > 2048 unsupported
}

template <typename W, bool Q = false>
static int dispatch_out(const typename TbeFwdParamsOf<Q>::type& p, int out_dtype, int max_dim, cudaStream_t stream) {
  switch (out_dtype) {
    case TRB_F32: return dispatch_shape<W, float, Q>(p, max_dim, stream);
    case TRB_BF16: return dispatch_shape<W, __nv_bfloat16, Q>(p, max_dim, stream);
  }
  return -3;
}

static int pooled_fwd_params(TbeFwdParams& p, const void* weights, const int64_t* feat_woff, const int64_t* feat_rows, const int32_t* feat_dim,
                             const int32_t* feat_col, const void* indices, int idx64, const void* offsets, int off64, const float* psw, int n_src,
                             int64_t idx_stride, int64_t off_stride, void* const* out_ptrs, int n_out, int64_t out_stride, int B, int B_local, int F,
                             int mean) {
  if (n_out < 1 || n_out > TRB_MAX_PEERS) return -1;
  if ((int64_t) B_local * n_out != B) return -4;
  if (n_src < 1 || B % n_src != 0) return -4;
  if (n_src > 1 && n_out > 1 && n_src != n_out) return -4;
  p.weights = weights;
  p.feat_woff = feat_woff;
  p.feat_rows = feat_rows;
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
  for (int i = 0; i < TRB_MAX_PEERS; ++i) p.out.p[i] = i < n_out ? out_ptrs[i] : nullptr;
  p.out_stride = out_stride;
  p.B = B;
  p.B_local = B_local;
  p.F = F;
  p.mean = mean;
  return 0;
}

// Pooled forward. Returns 0 on success, a cudaError_t (>0) or a negative library error.
// `n_src` > 1: ids arrive in per-source regions (see TrbSrcView); idx_stride / off_stride in elements.
TRB_API int trb_tbe_pooled_fwd(const void* weights, int w_dtype, const int64_t* feat_woff, const int64_t* feat_rows,
                               const int32_t* feat_dim, const int32_t* feat_col, const void* indices, int idx64,
                               const void* offsets, int off64, const float* psw, int n_src, int64_t idx_stride, int64_t off_stride,
                               void* const* out_ptrs, int n_out, int out_dtype, int64_t out_stride, int B, int B_local, int F,
                               int max_dim, int mean, cudaStream_t stream) {
  TbeFwdParams p;
  const int e = pooled_fwd_params(p, weights, feat_woff, feat_rows, feat_dim, feat_col, indices, idx64, offsets, off64, psw, n_src, idx_stride, off_stride,
                                  out_ptrs, n_out, out_stride, B, B_local, F, mean);
  if (e != 0) return e;
  switch (w_dtype) {
    case TRB_F32: return dispatch_out<float>(p, out_dtype, max_dim, stream);
    case TRB_F16: return dispatch_out<__half>(p, out_dtype, max_dim, stream);
    case TRB_BF16: return dispatch_out<__nv_bfloat16>(p, out_dtype, max_dim, stream);
  }
  return -3;
}

// Pooled forward with the FP8 wire: `out_ptrs` are uint8 payload rows [B_local, out_stride] per destination, `scale_ptrs` fp32
// rows [B_local, scale_stride] per destination, one scale per `row_dim` columns (32, 64 or 128). Every feature's output column
// and width must be multiples of row_dim. The groups are formed from the pooled values rounded to `wire_dtype` (fp32 | bf16).
TRB_API int trb_tbe_pooled_fwd_fp8(const void* weights, int w_dtype, const int64_t* feat_woff, const int64_t* feat_rows,
                                   const int32_t* feat_dim, const int32_t* feat_col, const void* indices, int idx64,
                                   const void* offsets, int off64, const float* psw, int n_src, int64_t idx_stride, int64_t off_stride,
                                   void* const* out_ptrs, void* const* scale_ptrs, int n_out, int wire_dtype, int64_t out_stride,
                                   int64_t scale_stride, int row_dim, int B, int B_local, int F, int max_dim, int mean, cudaStream_t stream) {
  if (row_dim != 32 && row_dim != 64 && row_dim != 128) return -5;
  TbeFwdQParams p;
  const int e = pooled_fwd_params(p, weights, feat_woff, feat_rows, feat_dim, feat_col, indices, idx64, offsets, off64, psw, n_src, idx_stride, off_stride,
                                  out_ptrs, n_out, out_stride, B, B_local, F, mean);
  if (e != 0) return e;
  for (int i = 0; i < TRB_MAX_PEERS; ++i) p.q_scale.p[i] = i < n_out ? scale_ptrs[i] : nullptr;
  p.q_scale_stride = scale_stride;
  p.q_lanes = row_dim / 4;
  switch (w_dtype) {
    case TRB_F32: return dispatch_out<float, true>(p, wire_dtype, max_dim, stream);
    case TRB_F16: return dispatch_out<__half, true>(p, wire_dtype, max_dim, stream);
    case TRB_BF16: return dispatch_out<__nv_bfloat16, true>(p, wire_dtype, max_dim, stream);
  }
  return -3;
}

// ------------------------------------------------------------------------------------------
// Sequence (unpooled) forward: out[i, :] = table(feature_of(i))[indices[i], :]
// All tables of an EmbeddingCollection group share one dim D. The feature of position i is
// found by binary search over per-feature value offsets (F+1 entries, tiny).
// Parity: BatchedFusedEmbedding forward (batched_embedding_kernel.py:1729-1915).
// ------------------------------------------------------------------------------------------
template <typename W, typename O, int LPB>
__global__ void __launch_bounds__(256)
tbe_seq_fwd_kernel(const W* __restrict__ weights, const int64_t* __restrict__ feat_woff,
                   const int64_t* __restrict__ feat_rows, const void* __restrict__ indices, int idx64,
                   const void* __restrict__ offsets, int off64, int F, int B, int D, O* __restrict__ out,
                   const int64_t* __restrict__ total_ptr) {
  const int lig = threadIdx.x % LPB;
  const int64_t r = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) / LPB;  // output row
  const int64_t total = trb_ld_idx(offsets, (int64_t) F * B, off64);
  const int64_t i = r + trb_ld_idx(offsets, 0, off64);  // offsets may be a window into a larger id array
  (void) total_ptr;
  if (i >= total) return;
  // binary search feature: largest f with offsets[f*B] <= i
  int lo = 0, hi = F - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (trb_ld_idx(offsets, (int64_t) mid * B, off64) <= i) lo = mid; else hi = mid - 1;
  }
  const int f = lo;
  int64_t idx = trb_ld_idx(indices, i, idx64);
  const bool ok = idx >= 0 && idx < feat_rows[f];
  const W* row = weights + feat_woff[f] + (ok ? idx : 0) * D;
  O* dst = out + r * D;
  const int nvec = D >> 2;
  for (int vi = lig; vi < nvec; vi += LPB) {
    float4 v = ok ? Vec4<W>::ld_nc(row + vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    Vec4<O>::st(dst + vi * 4, v);
  }
}

template <typename W, typename O>
static int launch_seq(const void* weights, const int64_t* feat_woff, const int64_t* feat_rows, const void* indices,
                      int idx64, const void* offsets, int off64, int F, int B, int D, void* out, int64_t max_total,
                      cudaStream_t stream) {
  if (max_total == 0) return 0;
  const int nvec = D / 4;
  const int threads = 256;
#define TRB_SEQ_LAUNCH(LPB)                                                                                   \
  {                                                                                                           \
    const int64_t gpb = threads / LPB;                                                                        \
    const int64_t blocks = (max_total + gpb - 1) / gpb;                                                       \
    tbe_seq_fwd_kernel<W, O, LPB><<<(unsigned) blocks, threads, 0, stream>>>(                                 \
        reinterpret_cast<const W*>(weights), feat_woff, feat_rows, indices, idx64, offsets, off64, F, B, D,  \
        reinterpret_cast<O*>(out), nullptr);                                                                  \
  }
  if (nvec <= 8) TRB_SEQ_LAUNCH(8)
  else if (nvec <= 16) TRB_SEQ_LAUNCH(16)
  else TRB_SEQ_LAUNCH(32)
#undef TRB_SEQ_LAUNCH
  TRB_CHECK_LAUNCH();
  return 0;
}

TRB_API int trb_tbe_seq_fwd(const void* weights, int w_dtype, const int64_t* feat_woff, const int64_t* feat_rows,
                            const void* indices, int idx64, const void* offsets, int off64, int F, int B, int D,
                            void* out, int out_dtype, int64_t max_total, cudaStream_t stream) {
#define TRB_SEQ_CASE(WT, OT) \
  return launch_seq<WT, OT>(weights, feat_woff, feat_rows, indices, idx64, offsets, off64, F, B, D, out, max_total, stream)
  if (w_dtype == TRB_F32 && out_dtype == TRB_F32) TRB_SEQ_CASE(float, float);
  if (w_dtype == TRB_F32 && out_dtype == TRB_BF16) TRB_SEQ_CASE(float, __nv_bfloat16);
  if (w_dtype == TRB_BF16 && out_dtype == TRB_F32) TRB_SEQ_CASE(__nv_bfloat16, float);
  if (w_dtype == TRB_BF16 && out_dtype == TRB_BF16) TRB_SEQ_CASE(__nv_bfloat16, __nv_bfloat16);
  if (w_dtype == TRB_F16 && out_dtype == TRB_F32) TRB_SEQ_CASE(__half, float);
#undef TRB_SEQ_CASE
  return -3;
}
