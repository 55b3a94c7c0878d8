// Inference table-batched lookup over quantized rows (sm_90a).
//
// Row formats (per table, mixed freely inside one launch):
//   FMT_FP32 / FMT_FP16 / FMT_BF16 : plain rows
//   FMT_INT8 / FMT_INT4 / FMT_INT2 : row-wise quantized, fused tail [scale fp16][bias fp16] after the packed
//                                    values (layout of fbgemm FloatOrHalfToFusedNBitRowwiseQuantizedSBHalf,
//                                    reference quant/embedding_modules.py:206-283)
//   FMT_FP8_BLOCK                  : e4m3 values + one fp16 scale per 32-element block ([D bytes][D/32 x fp16])
// One warp per bag; lane l dequantises elements 4l..4l+3 (+128k), accumulates in fp32, writes fp32/bf16/fp16.
// Parity: IntNBitTableBatchedEmbeddingBagsCodegen forward (reference quant_embedding_kernel.py:247-711).
#include "common.cuh"
#include <cuda_fp8.h>

enum QFmt : int { FMT_FP32 = 0, FMT_FP16 = 1, FMT_BF16 = 2, FMT_INT8 = 3, FMT_INT4 = 4, FMT_INT2 = 5, FMT_FP8_BLOCK = 6 };

struct QTbeParams {
  const uint8_t* weights;
  const int64_t* feat_woff;   // byte offset of the table
  const int64_t* feat_rows;
  const int32_t* feat_dim;
  const int32_t* feat_col;
  const int32_t* feat_fmt;
  const int32_t* feat_row_bytes;
  const void* indices;
  const void* offsets;
  const float* psw;
  void* out;
  int64_t out_stride;
  int32_t B, F, idx64, off64, mean, pooled;
};

__device__ __forceinline__ float4 dequant4(const uint8_t* row, int fmt, int D, int e) {
  // e = first element index (multiple of 4)
  switch (fmt) {
    case FMT_FP32: return *reinterpret_cast<const float4*>(row + e * 4);
    case FMT_FP16: return Vec4<__half>::ld(reinterpret_cast<const __half*>(row) + e);
    case FMT_BF16: return Vec4<__nv_bfloat16>::ld(reinterpret_cast<const __nv_bfloat16*>(row) + e);
    case FMT_INT8: {
      const uint32_t q = *reinterpret_cast<const uint32_t*>(row + e);
      const __half2 sb = *reinterpret_cast<const __half2*>(row + D);
      const float s = __low2float(sb), b = __high2float(sb);
      return make_float4((q & 0xff) * s + b, ((q >> 8) & 0xff) * s + b, ((q >> 16) & 0xff) * s + b, (q >> 24) * s + b);
    }
    case FMT_INT4: {
      const uint16_t q = *reinterpret_cast<const uint16_t*>(row + (e >> 1));
      const __half2 sb = *reinterpret_cast<const __half2*>(row + ((D + 1) >> 1));
      const float s = __low2float(sb), b = __high2float(sb);
      return make_float4((q & 0xf) * s + b, ((q >> 4) & 0xf) * s + b, ((q >> 8) & 0xf) * s + b, ((q >> 12) & 0xf) * s + b);
    }
    case FMT_INT2: {
      const uint8_t q = row[e >> 2];
      const __half2 sb = *reinterpret_cast<const __half2*>(row + ((D + 3) >> 2));
      const float s = __low2float(sb), b = __high2float(sb);
      return make_float4((q & 3) * s + b, ((q >> 2) & 3) * s + b, ((q >> 4) & 3) * s + b, ((q >> 6) & 3) * s + b);
    }
    case FMT_FP8_BLOCK: {
      const uint32_t q = *reinterpret_cast<const uint32_t*>(row + e);
      const float s = __half2float(*reinterpret_cast<const __half*>(row + D + (e >> 5) * 2));
      const __nv_fp8x4_e4m3 v = *reinterpret_cast<const __nv_fp8x4_e4m3*>(&q);
      const float4 f = static_cast<float4>(v);
      return make_float4(f.x * s, f.y * s, f.z * s, f.w * s);
    }
  }
  return make_float4(0.f, 0.f, 0.f, 0.f);
}

template <typename O, int MAXV>
__global__ void __launch_bounds__(256) qtbe_fwd_kernel(const QTbeParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t bag = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_bags = (int64_t) p.F * p.B;
  if (bag >= n_bags) return;
  const int f = (int) (bag / p.B);
  const int b = (int) (bag - (int64_t) f * p.B);
  const int D = p.feat_dim[f];
  const int nvec = D >> 2;
  const int fmt = p.feat_fmt[f];
  const int64_t rows = p.feat_rows[f];
  const int64_t rb = p.feat_row_bytes[f];
  const uint8_t* wbase = p.weights + p.feat_woff[f];
  const int64_t start = trb_ld_idx(p.offsets, bag, p.off64);
  const int64_t end = trb_ld_idx(p.offsets, bag + 1, p.off64);
  float4 acc[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t l0 = start; l0 < end; l0 += 32) {
    const int n = (int) min((int64_t) 32, end - l0);
    int64_t my_idx = 0;
    float my_w = 0.f;
    if (lane < n) {
      my_idx = trb_ld_idx(p.indices, l0 + lane, p.idx64);
      my_w = p.psw ? p.psw[l0 + lane] : 1.f;
      if (my_idx < 0 || my_idx >= rows) { my_idx = 0; my_w = 0.f; }
    }
    for (int j = 0; j < n; ++j) {
      const int64_t idx = __shfl_sync(0xffffffffu, my_idx, j);
      const float w = __shfl_sync(0xffffffffu, my_w, j);
      const uint8_t* row = wbase + idx * rb;
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        if (vi < nvec) acc[k] = f4_fma(dequant4(row, fmt, D, vi * 4), w, acc[k]);
      }
    }
  }
  if (p.mean && end > start) {
    const float inv = 1.f / (float) (end - start);
#pragma unroll
    for (int k = 0; k < MAXV; ++k) acc[k] = f4_scale(acc[k], inv);
  }
  O* dst = reinterpret_cast<O*>(p.out) + (int64_t) b * p.out_stride + p.feat_col[f];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nvec) Vec4<O>::st(dst + vi * 4, acc[k]);
  }
}

// ---- vector fast path (every table of the launch in ONE of INT8 / FP8 block-scaled / FP16 / BF16 / INT4) -----------------------------
// Serving batches are dominated by short bags (Criteo: one id per bag). The generic kernel above keeps ONE 4-byte-per-lane row in
// flight per warp (130-byte rows: ~5 % of the HBM rate). Here 8 lanes own a bag and read a row as 16 B vectors (EPV elements each: 16
// for the 8-bit formats, 8 for fp16 / bf16, 32 for int4 - a 128-element fp8 row is exactly one load per lane), every 8-lane group works on
// U bags at once with the first row of all of them in flight together, and a lane writes its EPV consecutive outputs.
template <int FMT> struct QVec;
template <> struct QVec<FMT_INT8> { static constexpr int EPV = 16; };
template <> struct QVec<FMT_FP8_BLOCK> { static constexpr int EPV = 16; };
template <> struct QVec<FMT_FP16> { static constexpr int EPV = 8; };
template <> struct QVec<FMT_BF16> { static constexpr int EPV = 8; };
template <> struct QVec<FMT_INT4> { static constexpr int EPV = 32; };

// scale word that belongs to the vector starting at element e: FP8_BLOCK = the fp16 scale of its 32-element block, INT8 / INT4 = the
// row's fp16 (scale, bias) behind the payload, fp16 / bf16 rows = none
template <int FMT>
__device__ __forceinline__ uint32_t load_scale_vec(const uint8_t* row, int D, int e) {
  if constexpr (FMT == FMT_FP8_BLOCK) return *reinterpret_cast<const uint16_t*>(row + D + (e >> 5) * 2);
  else if constexpr (FMT == FMT_INT8) return *reinterpret_cast<const uint32_t*>(row + D);
  else if constexpr (FMT == FMT_INT4) return *reinterpret_cast<const uint32_t*>(row + ((D + 1) >> 1));
  else return 0u;
}

template <int FMT>
__device__ __forceinline__ void dequant_vec(const uint4 q, const uint32_t sw, float (&v)[QVec<FMT>::EPV]) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
  if constexpr (FMT == FMT_FP8_BLOCK) {
    const float s = __half2float(__ushort_as_half((unsigned short) sw));
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const __nv_fp8x4_e4m3 x = *reinterpret_cast<const __nv_fp8x4_e4m3*>(&w[k]);
      const float4 f = static_cast<float4>(x);
      v[4 * k] = f.x * s; v[4 * k + 1] = f.y * s; v[4 * k + 2] = f.z * s; v[4 * k + 3] = f.w * s;
    }
  } else if constexpr (FMT == FMT_INT8) {  // value * scale + bias
    const __half2 sb = *reinterpret_cast<const __half2*>(&sw);
    const float s = __low2float(sb), b = __high2float(sb);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[4 * k] = (w[k] & 0xff) * s + b; v[4 * k + 1] = ((w[k] >> 8) & 0xff) * s + b;
      v[4 * k + 2] = ((w[k] >> 16) & 0xff) * s + b; v[4 * k + 3] = (w[k] >> 24) * s + b;
    }
  } else if constexpr (FMT == FMT_INT4) {  // low nibble first
    const __half2 sb = *reinterpret_cast<const __half2*>(&sw);
    const float s = __low2float(sb), b = __high2float(sb);
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int n = 0; n < 8; ++n) v[8 * k + n] = ((w[k] >> (4 * n)) & 0xf) * s + b;
  } else if constexpr (FMT == FMT_FP16) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[k]));
      v[2 * k] = f.x; v[2 * k + 1] = f.y;
    }
  } else {  // FMT_BF16
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[2 * k] = __uint_as_float(w[k] << 16); v[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u);
    }
  }
}

template <typename O, int N>
__device__ __forceinline__ void store_vec(O* dst, const float (&a)[N]) {
#pragma unroll
  for (int k = 0; k < N / 4; ++k) Vec4<O>::st(dst + 4 * k, make_float4(a[4 * k], a[4 * k + 1], a[4 * k + 2], a[4 * k + 3]));
}

template <typename O, int FMT, int MAXV, int U>
__global__ void __launch_bounds__(256, 3) qtbe_fwd_vec_kernel(const QTbeParams p) {
  constexpr int LPR = 8;
  constexpr int EPV = QVec<FMT>::EPV;
  const int lig = threadIdx.x & (LPR - 1);
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int64_t n_bags = (int64_t) p.F * p.B;
  const int64_t bag0 = group * U;
  if (bag0 >= n_bags) return;
  int64_t st[U], en[U];
  const uint8_t* wb[U];
  int64_t rb[U], rows[U];
  int D[U], col[U], b_of[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int64_t bag = bag0 + u < n_bags ? bag0 + u : n_bags - 1;
    const int f = (int) (bag / p.B);
    b_of[u] = (int) (bag - (int64_t) f * p.B);
    D[u] = p.feat_dim[f];
    col[u] = p.feat_col[f];
    rows[u] = p.feat_rows[f];
    rb[u] = p.feat_row_bytes[f];
    wb[u] = p.weights + p.feat_woff[f];
    st[u] = trb_ld_idx(p.offsets, bag, p.off64);
    en[u] = bag0 + u < n_bags ? trb_ld_idx(p.offsets, bag + 1, p.off64) : st[u];
  }
  // first id of every bag: all U x MAXV row vectors in flight before any is consumed
  uint4 q[U][MAXV];
  uint32_t sw[U][MAXV];
  float w0[U];
  const uint8_t* row0[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    w0[u] = 0.f;
    row0[u] = wb[u];
    if (en[u] > st[u]) {
      const int64_t idx = trb_ld_idx(p.indices, st[u], p.idx64);
      if (idx >= 0 && idx < rows[u]) {
        w0[u] = p.psw ? p.psw[st[u]] : 1.f;
        row0[u] = wb[u] + idx * rb[u];
      }
    }
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      // unconditional loads from clamped addresses, payload AND scale word: a predicated load + select (or a scale fetched when the
      // payload is consumed) made every row wait for the previous one (same finding as tbe_bwd_walk_kernel)
      const int vi = lig + k * LPR;
      const int vc = vi * EPV < D[u] ? vi : 0;
      q[u][k] = *reinterpret_cast<const uint4*>(row0[u] + vc * 16);
      sw[u][k] = load_scale_vec<FMT>(row0[u], D[u], vc * EPV);
    }
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    float acc1[MAXV][EPV];  // one bag's accumulator at a time (the loads of all U bags are already in flight)
#pragma unroll
    for (int k = 0; k < MAXV; ++k)
#pragma unroll
      for (int t = 0; t < EPV; ++t) acc1[k][t] = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int e = (lig + k * LPR) * EPV;
      if (e < D[u] && w0[u] != 0.f) {
        float v[EPV];
        dequant_vec<FMT>(q[u][k], sw[u][k], v);
#pragma unroll
        for (int t = 0; t < EPV; ++t) acc1[k][t] = v[t] * w0[u];
      }
    }
    // the rest of the bag (pooling factor > 1)
    for (int64_t j = st[u] + 1; j < en[u]; ++j) {
      const int64_t idx = trb_ld_idx(p.indices, j, p.idx64);
      if (idx < 0 || idx >= rows[u]) continue;
      const float w = p.psw ? p.psw[j] : 1.f;
      const uint8_t* row = wb[u] + idx * rb[u];
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lig + k * LPR;
        const int e = vi * EPV;
        if (e < D[u]) {
          float v[EPV];
          dequant_vec<FMT>(*reinterpret_cast<const uint4*>(row + vi * 16), load_scale_vec<FMT>(row, D[u], e), v);
#pragma unroll
          for (int t = 0; t < EPV; ++t) acc1[k][t] = fmaf(v[t], w, acc1[k][t]);
        }
      }
    }
    if (bag0 + u >= n_bags) continue;
    const float inv = (p.mean && en[u] > st[u]) ? 1.f / (float) (en[u] - st[u]) : 1.f;
    O* dst = reinterpret_cast<O*>(p.out) + (int64_t) b_of[u] * p.out_stride + col[u];
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int e = (lig + k * LPR) * EPV;
      if (e < D[u]) {
        if (inv != 1.f) {
#pragma unroll
          for (int t = 0; t < EPV; ++t) acc1[k][t] *= inv;
        }
        store_vec<O, EPV>(dst + e, acc1[k]);
      }
    }
  }
}

template <typename O, int FMT>
static int launch_q_vec(const QTbeParams& p, int max_dim, cudaStream_t stream) {
  const int64_t n_bags = (int64_t) p.F * p.B;
  if (n_bags == 0) return 0;
  const int threads = 256;
  const int vecs = (max_dim + QVec<FMT>::EPV - 1) / QVec<FMT>::EPV;  // 16 B vectors per row; 8 lanes per bag
#define TRB_QVEC(MAXV, U)                                                                                     \
  {                                                                                                           \
    const int64_t groups = (n_bags + U - 1) / U;                                                              \
    const unsigned blocks = (unsigned) ((groups * 8 + threads - 1) / threads);                                \
    qtbe_fwd_vec_kernel<O, FMT, MAXV, U><<<blocks, threads, 0, stream>>>(p);                                  \
  }
  if (vecs <= 8) TRB_QVEC(1, 4)
  else if (vecs <= 16) TRB_QVEC(2, 2)
  else if (vecs <= 32) TRB_QVEC(4, 1)
  else return -7;
#undef TRB_QVEC
  TRB_CHECK_LAUNCH();
  return 0;
}

// sequence (unpooled): one warp per id position
template <typename O>
__global__ void __launch_bounds__(256) qtbe_seq_kernel(const QTbeParams p, int64_t total) {
  const int lane = threadIdx.x & 31;
  const int64_t i = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= total) return;
  int lo = 0, hi = p.F - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (trb_ld_idx(p.offsets, (int64_t) mid * p.B, p.off64) <= i) lo = mid; else hi = mid - 1;
  }
  const int f = lo;
  const int D = p.feat_dim[f];
  const int nvec = D >> 2;
  int64_t idx = trb_ld_idx(p.indices, i, p.idx64);
  const bool ok = idx >= 0 && idx < p.feat_rows[f];
  const uint8_t* row = p.weights + p.feat_woff[f] + (ok ? idx : 0) * (int64_t) p.feat_row_bytes[f];
  O* dst = reinterpret_cast<O*>(p.out) + i * p.out_stride;
  for (int vi = lane; vi < nvec; vi += 32) {
    float4 v = ok ? dequant4(row, p.feat_fmt[f], D, vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    Vec4<O>::st(dst + vi * 4, v);
  }
}

template <typename O>
static int launch_q(const QTbeParams& p, int max_dim, int64_t total, int uniform_fmt, cudaStream_t stream) {
  const int threads = 256;
  if (p.pooled && uniform_fmt >= 0) {  // (the caller guarantees rows made of whole 16-byte vectors: quant_tbe.py _uniform_fmt)
    if (uniform_fmt == FMT_FP8_BLOCK && max_dim <= 512) return launch_q_vec<O, FMT_FP8_BLOCK>(p, max_dim, stream);
    if (uniform_fmt == FMT_INT8 && max_dim <= 512) return launch_q_vec<O, FMT_INT8>(p, max_dim, stream);
    if (uniform_fmt == FMT_FP16 && max_dim <= 256) return launch_q_vec<O, FMT_FP16>(p, max_dim, stream);
    if (uniform_fmt == FMT_BF16 && max_dim <= 256) return launch_q_vec<O, FMT_BF16>(p, max_dim, stream);
    if (uniform_fmt == FMT_INT4 && max_dim <= 1024) return launch_q_vec<O, FMT_INT4>(p, max_dim, stream);
  }
  if (!p.pooled) {
    if (total == 0) return 0;
    qtbe_seq_kernel<O><<<(unsigned) ((total * 32 + threads - 1) / threads), threads, 0, stream>>>(p, total);
    TRB_CHECK_LAUNCH();
    return 0;
  }
  const int64_t n_bags = (int64_t) p.F * p.B;
  if (n_bags == 0) return 0;
  const unsigned blocks = (unsigned) ((n_bags * 32 + threads - 1) / threads);
  const int nvec = max_dim / 4;
  if (nvec <= 32) qtbe_fwd_kernel<O, 1><<<blocks, threads, 0, stream>>>(p);
  else if (nvec <= 128) qtbe_fwd_kernel<O, 4><<<blocks, threads, 0, stream>>>(p);
  else if (nvec <= 512) qtbe_fwd_kernel<O, 16><<<blocks, threads, 0, stream>>>(p);
  else return -2;
  TRB_CHECK_LAUNCH();
  return 0;
}

TRB_API int trb_qtbe_fwd_ex(const void* weights, const int64_t* feat_woff, const int64_t* feat_rows, const int32_t* feat_dim, const int32_t* feat_col,
                            const int32_t* feat_fmt, const int32_t* feat_row_bytes, const void* indices, int idx64, const void* offsets, int off64,
                            const float* psw, void* out, int out_dtype, int64_t out_stride, int B, int F, int max_dim, int mean, int pooled,
                            int64_t total, int uniform_fmt, cudaStream_t stream);

TRB_API int trb_qtbe_fwd(const void* weights, const int64_t* feat_woff, const int64_t* feat_rows, const int32_t* feat_dim, const int32_t* feat_col,
                         const int32_t* feat_fmt, const int32_t* feat_row_bytes, const void* indices, int idx64, const void* offsets, int off64,
                         const float* psw, void* out, int out_dtype, int64_t out_stride, int B, int F, int max_dim, int mean, int pooled,
                         int64_t total, cudaStream_t stream) {
  return trb_qtbe_fwd_ex(weights, feat_woff, feat_rows, feat_dim, feat_col, feat_fmt, feat_row_bytes, indices, idx64, offsets, off64, psw, out, out_dtype,
                         out_stride, B, F, max_dim, mean, pooled, total, -1, stream);
}

// `uniform_fmt`: the row format shared by EVERY table of the launch with all dims % 16 == 0 (enables the vector fast path), or -1
TRB_API int trb_qtbe_fwd_ex(const void* weights, const int64_t* feat_woff, const int64_t* feat_rows, const int32_t* feat_dim, const int32_t* feat_col,
                            const int32_t* feat_fmt, const int32_t* feat_row_bytes, const void* indices, int idx64, const void* offsets, int off64,
                            const float* psw, void* out, int out_dtype, int64_t out_stride, int B, int F, int max_dim, int mean, int pooled,
                            int64_t total, int uniform_fmt, cudaStream_t stream) {
  QTbeParams p;
  p.weights = reinterpret_cast<const uint8_t*>(weights);
  p.feat_woff = feat_woff; p.feat_rows = feat_rows; p.feat_dim = feat_dim; p.feat_col = feat_col; p.feat_fmt = feat_fmt;
  p.feat_row_bytes = feat_row_bytes; p.indices = indices; p.offsets = offsets; p.psw = psw; p.out = out; p.out_stride = out_stride;
  p.B = B; p.F = F; p.idx64 = idx64; p.off64 = off64; p.mean = mean; p.pooled = pooled;
  switch (out_dtype) {
    case TRB_F32: return launch_q<float>(p, max_dim, total, uniform_fmt, stream);
    case TRB_F16: return launch_q<__half>(p, max_dim, total, uniform_fmt, stream);
    case TRB_BF16: return launch_q<__nv_bfloat16>(p, max_dim, total, uniform_fmt, stream);
  }
  return -3;
}
