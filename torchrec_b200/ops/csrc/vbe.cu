// Variable batch per feature (VBE) on the device.
//
// A VBE batch carries, for feature f, B_f <= B de-duplicated bags and a row inv[r(f), 0:B] that says which bag every sample uses.
// The lookup kernels see such a batch as an ordinary uniform one once every feature is padded with empty bags (trb_vbe_pad_offsets);
// the pooled rows [S, sum D] are expanded to the samples with out[b, c] = pooled[inv[r(c), b], c] (trb_vbe_expand), and the gradient
// of that expansion is a segmented sum over the samples that referenced each bag (trb_vbe_csr + trb_vbe_reduce).
//
// Columns are addressed in 16-byte vectors. col_row[v] is the inverse row of column vector v, or -1 when the vector's feature has no
// inverse row (identity). row_vec_off / row_vecs list the column vectors of every inverse row (the transpose of col_row).
//
// Determinism of the reduce: a segment lists its samples in ascending order (stable radix sort). A segment of at most
// VBE_LONG_SEG samples is summed in that order by one thread per column vector. A longer one is cut, from its own start, into slices of
// VBE_SLICE samples; a slice is summed by one block in an order fixed by the slice length and the feature width, and the slice sums
// are added in slice order. Nothing depends on the grid, the SM count or on scheduling; there are no floating-point atomics (the
// integer atomics of the long-segment list only decide where a slice's partial sum is parked).
#include "common.cuh"

#include <cub/cub.cuh>

#define VBE_LONG_SEG 256
#define VBE_SLICE 256

// ---------------------------------------------------------------------------------------------------------------
// pad_offsets: ragged offsets [sum_f B_f + 1] -> uniform offsets [F * B + 1]; bags u >= B_f of feature f are empty and point at the end
// of the feature's values.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vbe_pad_offsets_kernel(const void* __restrict__ off, int off64, const int32_t* __restrict__ bsz, int F, int64_t B,
                                                              void* __restrict__ out) {
  __shared__ int64_t s_base;
  const int f = blockIdx.y;
  if (threadIdx.x < 32) {
    int64_t s = 0;
    for (int g = threadIdx.x; g < f; g += 32) s += bsz[g];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) s_base = s;
  }
  __syncthreads();
  const int64_t u = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= B + (f == F - 1)) return;  // the last feature also writes the closing offset
  const int64_t bf = min((int64_t) bsz[f], B);
  trb_st_idx(out, (int64_t) f * B + u, off64, trb_ld_idx(off, s_base + min(u, bf), off64));
}

TRB_API int trb_vbe_pad_offsets(const void* offsets, int off64, const int32_t* batch_sizes, int F, int64_t B, void* out, cudaStream_t stream) {
  if (F < 0 || B < 0 || F > 65535) return -2;
  if (F == 0 || B == 0) return 0;
  dim3 grid((unsigned) ((B + 1 + 255) / 256), (unsigned) F);
  vbe_pad_offsets_kernel<<<grid, 256, 0, stream>>>(offsets, off64, batch_sizes, F, B, out);
  TRB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// expand: out[b, v] = pooled[inv[col_row[v], b], v] over 16-byte vectors (a copy: the element type does not matter). An inverse index
// outside [0, S) is not dereferenced: the address is clamped and the vector is written as zeros.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vbe_expand_kernel(const uint4* __restrict__ pooled, uint4* __restrict__ out, const int32_t* __restrict__ col_row,
                                                         const void* __restrict__ inv, int inv64, int64_t B, int64_t S, int cols_vec) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * cols_vec) return;
  const int v = (int) (i % cols_vec);
  const int64_t b = i / cols_vec;
  const int r = col_row[v];
  int64_t src = b;
  if (r >= 0) src = trb_ld_idx(inv, (int64_t) r * B + b, inv64);
  const bool ok = src >= 0 && src < S;
  uint4 x = pooled[(ok ? src : 0) * cols_vec + v];
  if (!ok) x = make_uint4(0u, 0u, 0u, 0u);
  out[i] = x;
}

TRB_API int trb_vbe_expand(const void* pooled, void* out, const int32_t* col_row, const void* inv, int inv64, int64_t B, int64_t S, int cols_vec,
                           cudaStream_t stream) {
  if (B < 0 || S < 0 || cols_vec < 0) return -2;
  const int64_t n = B * cols_vec;
  if (n == 0) return 0;
  if (S == 0) return -2;  // samples but no pooled row to read
  vbe_expand_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>((const uint4*) pooled, (uint4*) out, col_row, inv, inv64, B, S, cols_vec);
  TRB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// csr: the transpose of the inverse indices. Segment r * S + u lists, in ascending b, the samples with inv[r, b] == u:
// seg_b[seg_off[seg] : seg_off[seg + 1]]. Samples with an index outside [0, S) sort behind the last segment and belong to none.
// `lists` (int32, trb_vbe_long_list_elems) receives the segments longer than VBE_LONG_SEG and their slices:
//   [0] number of long segments, [1] number of slices, long_seg[maxL], long_base[maxL] (first slice of the segment),
//   slice_seg[maxS], slice_k[maxS].
// ---------------------------------------------------------------------------------------------------------------
static inline int64_t vbe_max_long(int64_t n) { return n / (VBE_LONG_SEG + 1) + 1; }
static inline int64_t vbe_max_slices(int64_t n) { return n / VBE_SLICE + vbe_max_long(n) + 1; }
static inline size_t vbe_align(size_t x) { return (x + 255) & ~(size_t) 255; }

static size_t vbe_sort_temp_bytes(int64_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*) nullptr, (uint32_t*) nullptr, (const int32_t*) nullptr, (int32_t*) nullptr, n);
  return bytes;
}

static inline bool vbe_shape_ok(int64_t R, int64_t B, int64_t S) {
  const int64_t lim = ((int64_t) 1 << 31) - 2;
  return R >= 0 && B >= 0 && S >= 0 && (R == 0 || (B <= lim / R && S <= lim / R));
}

TRB_API int64_t trb_vbe_csr_workspace_bytes(int64_t R, int64_t B) {
  if (!vbe_shape_ok(R, B, 0)) return -2;
  const int64_t n = R * B > 0 ? R * B : 1;
  return (int64_t) (3 * vbe_align(n * 4) + vbe_align(vbe_sort_temp_bytes(n)));
}

TRB_API int64_t trb_vbe_long_list_elems(int64_t R, int64_t B) {
  if (!vbe_shape_ok(R, B, 0)) return -2;
  const int64_t n = R * B;
  return 2 + 2 * vbe_max_long(n) + 2 * vbe_max_slices(n);
}

__global__ void __launch_bounds__(256) vbe_csr_keys_kernel(const void* __restrict__ inv, int inv64, int64_t n, int64_t B, int64_t S, uint32_t sentinel,
                                                           uint32_t* __restrict__ keys, int32_t* __restrict__ vals) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t r = i / B;
  const int64_t x = trb_ld_idx(inv, i, inv64);
  keys[i] = (x >= 0 && x < S) ? (uint32_t) (r * S + x) : sentinel;
  vals[i] = (int32_t) (i - r * B);
}

__device__ __forceinline__ int32_t vbe_lower_bound(const uint32_t* __restrict__ keys, int32_t n, uint32_t key) {
  int32_t lo = 0, hi = n;
  while (lo < hi) {
    const int32_t mid = lo + ((hi - lo) >> 1);
    if (keys[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(256) vbe_csr_offsets_kernel(const uint32_t* __restrict__ keys_sorted, int32_t n, int64_t n_seg, int32_t* __restrict__ seg_off,
                                                              int32_t* __restrict__ lists, int32_t max_long, int32_t max_slices) {
  const int64_t s = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (s > n_seg) return;
  const int32_t a = vbe_lower_bound(keys_sorted, n, (uint32_t) s);
  seg_off[s] = a;
  if (s == n_seg) return;
  const int32_t len = vbe_lower_bound(keys_sorted, n, (uint32_t) s + 1u) - a;
  if (len <= VBE_LONG_SEG) return;
  const int32_t n_sl = (len + VBE_SLICE - 1) / VBE_SLICE;
  const int32_t li = atomicAdd(&lists[0], 1);
  const int32_t base = atomicAdd(&lists[1], n_sl);
  int32_t* long_seg = lists + 2;
  int32_t* long_base = long_seg + max_long;
  int32_t* slice_seg = long_base + max_long;
  int32_t* slice_k = slice_seg + max_slices;
  long_seg[li] = (int32_t) s;
  long_base[li] = base;
  for (int32_t k = 0; k < n_sl; ++k) {
    slice_seg[base + k] = (int32_t) s;
    slice_k[base + k] = k;
  }
}

TRB_API int trb_vbe_csr(const void* inv, int inv64, int64_t R, int64_t B, int64_t S, int32_t* seg_off, int32_t* seg_b, int32_t* lists, void* workspace,
                        int64_t workspace_bytes, cudaStream_t stream) {
  if (!vbe_shape_ok(R, B, S)) return -2;
  const int64_t n = R * B, n_seg = R * S;
  if (workspace_bytes < trb_vbe_csr_workspace_bytes(R, B)) return -4;
  TRB_CUDA(cudaMemsetAsync(lists, 0, 2 * sizeof(int32_t), stream));
  char* ws = (char*) workspace;
  uint32_t* keys = (uint32_t*) ws;
  uint32_t* keys_sorted = (uint32_t*) (ws + vbe_align((n > 0 ? n : 1) * 4));
  int32_t* vals = (int32_t*) (ws + 2 * vbe_align((n > 0 ? n : 1) * 4));
  void* sort_tmp = ws + 3 * vbe_align((n > 0 ? n : 1) * 4);
  if (n > 0) {
    vbe_csr_keys_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(inv, inv64, n, B, S, (uint32_t) n_seg, keys, vals);
    TRB_CHECK_LAUNCH();
    size_t tmp_bytes = vbe_sort_temp_bytes(n);
    int end_bit = 1;
    while (end_bit < 32 && ((int64_t) 1 << end_bit) <= n_seg) ++end_bit;
    TRB_CUDA(cub::DeviceRadixSort::SortPairs(sort_tmp, tmp_bytes, (const uint32_t*) keys, keys_sorted, (const int32_t*) vals, seg_b, n, 0, end_bit, stream));
    g_trb_launches += 4;  // radix sort passes (library kernels, counted approximately)
  }
  vbe_csr_offsets_kernel<<<(unsigned) ((n_seg + 1 + 255) / 256), 256, 0, stream>>>(keys_sorted, (int32_t) n, n_seg, seg_off, lists, (int32_t) vbe_max_long(n),
                                                                                  (int32_t) vbe_max_slices(n));
  TRB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// reduce: gpooled[u, v] = sum over b in seg(col_row[v], u) of g[b, v], fp32 accumulation, output in the dtype of g.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
struct V16;

template <>
struct V16<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void add(float* a, uint4 u) {
    a[0] += __uint_as_float(u.x); a[1] += __uint_as_float(u.y); a[2] += __uint_as_float(u.z); a[3] += __uint_as_float(u.w);
  }
  static __device__ __forceinline__ uint4 pack(const float* a) {
    return make_uint4(__float_as_uint(a[0]), __float_as_uint(a[1]), __float_as_uint(a[2]), __float_as_uint(a[3]));
  }
};

template <>
struct V16<__nv_bfloat16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void add(float* a, uint4 u) {
    a[0] += __uint_as_float(u.x << 16); a[1] += __uint_as_float(u.x & 0xffff0000u);
    a[2] += __uint_as_float(u.y << 16); a[3] += __uint_as_float(u.y & 0xffff0000u);
    a[4] += __uint_as_float(u.z << 16); a[5] += __uint_as_float(u.z & 0xffff0000u);
    a[6] += __uint_as_float(u.w << 16); a[7] += __uint_as_float(u.w & 0xffff0000u);
  }
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&p);
  }
  static __device__ __forceinline__ uint4 pack(const float* a) {
    return make_uint4(pack2(a[0], a[1]), pack2(a[2], a[3]), pack2(a[4], a[5]), pack2(a[6], a[7]));
  }
};

// samples p, p + step, ... < e of seg_b, four gradient loads in flight, added in that order
template <typename T>
__device__ __forceinline__ void vbe_sum_rows(float* acc, const uint4* __restrict__ g, const int32_t* __restrict__ seg_b, int32_t p, int32_t e, int32_t step,
                                             int64_t cols_vec, int v) {
  for (; p + 3 * step < e; p += 4 * step) {
    const int32_t b0 = seg_b[p], b1 = seg_b[p + step], b2 = seg_b[p + 2 * step], b3 = seg_b[p + 3 * step];
    const uint4 x0 = g[b0 * cols_vec + v], x1 = g[b1 * cols_vec + v], x2 = g[b2 * cols_vec + v], x3 = g[b3 * cols_vec + v];
    V16<T>::add(acc, x0);
    V16<T>::add(acc, x1);
    V16<T>::add(acc, x2);
    V16<T>::add(acc, x3);
  }
  for (; p < e; p += step) V16<T>::add(acc, g[seg_b[p] * cols_vec + v]);
}

// one thread per (bag, column vector): the lanes of a feature's vectors form the lane group of (feature, bag)
template <typename T>
__global__ void __launch_bounds__(256) vbe_reduce_short_kernel(const uint4* __restrict__ g, uint4* __restrict__ out, const int32_t* __restrict__ col_row,
                                                               const int32_t* __restrict__ seg_off, const int32_t* __restrict__ seg_b, int64_t S, int cols_vec) {
  constexpr int N = V16<T>::N;
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S * cols_vec) return;
  const int v = (int) (i % cols_vec);
  const int64_t u = i / cols_vec;
  const int r = col_row[v];
  if (r < 0) {  // identity column: S == B, the gradient passes through
    out[i] = g[i];
    return;
  }
  const int32_t a = seg_off[r * S + u], e = seg_off[r * S + u + 1];
  if (e - a > VBE_LONG_SEG) return;  // written by vbe_reduce_combine_kernel
  float acc[N];
#pragma unroll
  for (int j = 0; j < N; ++j) acc[j] = 0.f;
  vbe_sum_rows<T>(acc, g, seg_b, a, e, 1, cols_vec, v);
  out[i] = V16<T>::pack(acc);
}

// one block per slice of a long segment. The block's threads form 256 / G groups of G lanes (G = the feature's vectors rounded up to a
// power of two, at most 32); group j sums samples j, j + 256 / G, ... of the slice in ascending order, then the group sums are added
// in group order.
template <typename T>
__global__ void __launch_bounds__(256) vbe_reduce_slice_kernel(const uint4* __restrict__ g, float* __restrict__ partial, const int32_t* __restrict__ lists,
                                                               int32_t max_long, int32_t max_slices, const int32_t* __restrict__ row_vec_off,
                                                               const int32_t* __restrict__ row_vecs, const int32_t* __restrict__ seg_off,
                                                               const int32_t* __restrict__ seg_b, int64_t S, int cols_vec, int max_nv) {
  constexpr int N = V16<T>::N;
  __shared__ float sm[N][256];
  const int32_t sidx = blockIdx.x;
  if (sidx >= lists[1]) return;
  const int32_t* slice_seg = lists + 2 + 2 * max_long;
  const int32_t seg = slice_seg[sidx], k = slice_seg[max_slices + sidx];
  const int r = (int) (seg / S);
  const int32_t a = seg_off[seg] + k * VBE_SLICE;
  const int32_t e = min(a + VBE_SLICE, seg_off[seg + 1]);
  const int v0 = row_vec_off[r], nv = row_vec_off[r + 1] - v0;
  int G = 4;
  while (G < nv && G < 32) G <<= 1;
  const int n_grp = 256 / G, lane = threadIdx.x & (G - 1), grp = threadIdx.x / G;
  for (int vb = 0; vb < nv; vb += G) {
    const int vi = vb + lane;
    float acc[N];
#pragma unroll
    for (int j = 0; j < N; ++j) acc[j] = 0.f;
    if (vi < nv) vbe_sum_rows<T>(acc, g, seg_b, a + grp, e, n_grp, cols_vec, row_vecs[v0 + vi]);
#pragma unroll
    for (int j = 0; j < N; ++j) sm[j][threadIdx.x] = acc[j];
    __syncthreads();
    if (threadIdx.x < G && vi < nv) {
#pragma unroll
      for (int j = 0; j < N; ++j) acc[j] = 0.f;
      for (int q = 0; q < n_grp; ++q) {
#pragma unroll
        for (int j = 0; j < N; ++j) acc[j] += sm[j][q * G + lane];
      }
      float* dst = partial + ((int64_t) sidx * max_nv + vi) * N;
#pragma unroll
      for (int j = 0; j < N; ++j) dst[j] = acc[j];
    }
    __syncthreads();
  }
}

// one block per long segment: slice sums added in slice order
template <typename T>
__global__ void __launch_bounds__(64) vbe_reduce_combine_kernel(const float* __restrict__ partial, uint4* __restrict__ out, const int32_t* __restrict__ lists,
                                                                int32_t max_long, const int32_t* __restrict__ row_vec_off, const int32_t* __restrict__ row_vecs,
                                                                const int32_t* __restrict__ seg_off, int64_t S, int cols_vec, int max_nv) {
  constexpr int N = V16<T>::N;
  const int32_t li = blockIdx.x;
  if (li >= lists[0]) return;
  const int32_t seg = lists[2 + li], base = lists[2 + max_long + li];
  const int32_t n_sl = (seg_off[seg + 1] - seg_off[seg] + VBE_SLICE - 1) / VBE_SLICE;
  const int r = (int) (seg / S);
  const int64_t u = seg - (int64_t) r * S;
  const int v0 = row_vec_off[r], nv = row_vec_off[r + 1] - v0;
  for (int vi = threadIdx.x; vi < nv; vi += blockDim.x) {
    float acc[N];
#pragma unroll
    for (int j = 0; j < N; ++j) acc[j] = 0.f;
    for (int32_t k = 0; k < n_sl; ++k) {
      const float* src = partial + ((int64_t) (base + k) * max_nv + vi) * N;
#pragma unroll
      for (int j = 0; j < N; ++j) acc[j] += src[j];
    }
    out[u * cols_vec + row_vecs[v0 + vi]] = V16<T>::pack(acc);
  }
}

TRB_API int64_t trb_vbe_reduce_workspace_bytes(int64_t R, int64_t B, int max_nv) {
  if (!vbe_shape_ok(R, B, 0) || max_nv < 0) return -2;
  return (int64_t) vbe_align((size_t) vbe_max_slices(R * B) * (max_nv > 0 ? max_nv : 1) * 8 * sizeof(float));
}

template <typename T>
static int vbe_run_reduce(const void* g, void* out, const int32_t* col_row, const int32_t* row_vec_off, const int32_t* row_vecs, int max_nv,
                          const int32_t* seg_off, const int32_t* seg_b, const int32_t* lists, int64_t n, int64_t S, int cols_vec, float* partial,
                          cudaStream_t stream) {
  const int64_t total = S * cols_vec;
  const int32_t max_long = (int32_t) vbe_max_long(n), max_slices = (int32_t) vbe_max_slices(n);
  vbe_reduce_short_kernel<T><<<(unsigned) ((total + 255) / 256), 256, 0, stream>>>((const uint4*) g, (uint4*) out, col_row, seg_off, seg_b, S, cols_vec);
  TRB_CHECK_LAUNCH();
  if (n <= VBE_LONG_SEG) return 0;  // no segment can be long
  // The numbers of long segments and slices live on the device (lists[0], lists[1]); reading them would synchronise the host and could
  // not be captured in a graph. Both kernels are launched over the bounds of those counts; a block past the count reads it and exits.
  vbe_reduce_slice_kernel<T><<<(unsigned) max_slices, 256, 0, stream>>>((const uint4*) g, partial, lists, max_long, max_slices, row_vec_off, row_vecs, seg_off,
                                                                      seg_b, S, cols_vec, max_nv);
  TRB_CHECK_LAUNCH();
  vbe_reduce_combine_kernel<T><<<(unsigned) max_long, 64, 0, stream>>>(partial, (uint4*) out, lists, max_long, row_vec_off, row_vecs, seg_off, S, cols_vec,
                                                                      max_nv);
  TRB_CHECK_LAUNCH();
  return 0;
}

TRB_API int trb_vbe_reduce(const void* g, void* out, int dtype, const int32_t* col_row, const int32_t* row_vec_off, const int32_t* row_vecs, int max_nv,
                           const int32_t* seg_off, const int32_t* seg_b, const int32_t* lists, int64_t R, int64_t B, int64_t S, int cols_vec, void* workspace,
                           int64_t workspace_bytes, cudaStream_t stream) {
  if (!vbe_shape_ok(R, B, S) || cols_vec < 0 || max_nv < 0) return -2;
  if (dtype != TRB_F32 && dtype != TRB_BF16) return -3;
  if (S * cols_vec == 0) return 0;
  if (workspace_bytes < trb_vbe_reduce_workspace_bytes(R, B, max_nv)) return -4;
  if (dtype == TRB_F32)
    return vbe_run_reduce<float>(g, out, col_row, row_vec_off, row_vecs, max_nv, seg_off, seg_b, lists, R * B, S, cols_vec, (float*) workspace, stream);
  return vbe_run_reduce<__nv_bfloat16>(g, out, col_row, row_vec_off, row_vecs, max_nv, seg_off, seg_b, lists, R * B, S, cols_vec, (float*) workspace, stream);
}
