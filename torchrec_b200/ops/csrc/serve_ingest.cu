// Server batch -> static inputs of a captured predict graph (inference/graphed.py).
//
// The serving core (csrc/serving) packs each batch into one slab: dense [B, num_float] fp32 | id_list lengths [F1 * B] int32 |
// id_list values int64 | id_score_list lengths [F2 * B] | values | weights fp32, every section 16-byte aligned. A CUDA graph needs
// fixed addresses and fixed shapes, so one launch turns the device copy of that slab into the buffers of a bucket (B_cap, nnz_cap):
//
//   dense   [B_cap, num_float]   rows >= B are zero
//   lengths [F * B_cap]          key-major, bags b >= B are empty: every feature keeps the stride B_cap
//   offsets [F * B_cap + 1]      block-level scan of the lengths, int32 or int64
//   values  [nnz_cap]            (and weights for id_score_list); nothing past nnz is written
//
// Every size comes from the device descriptor (inference/graphed.py: pack_desc), so one graph serves every batch that fits its bucket.
// A descriptor that does not fit (B > B_cap, nnz > nnz_cap, other feature counts, sections outside the slab) raises *error and the
// launch writes nothing. Lengths that are negative or do not sum to nnz also raise *error; the offsets are then clamped to
// [0, nnz], so the lookup behind them never reads past the values.
//
//   block 0      scan of the id_list lengths
//   block 1      scan of the id_score_list lengths
//   blocks 2..   dense rows, values and weights as 16-byte vectors (element-wise where a section is not 16-byte aligned)
#include "common.cuh"
#include <cub/block/block_scan.cuh>

namespace {

constexpr int kThreads = 512;
constexpr int kItems = 8;  // lengths per thread per scan tile

// descriptor fields (int64); keep in sync with inference/graphed.py: DESC_FIELDS
enum : int {
  D_B = 0, D_NUM_FLOAT, D_F_IDL, D_F_IDS, D_DENSE_OFF, D_IDL_LEN_OFF, D_IDL_VAL_OFF, D_IDL_NNZ, D_IDS_LEN_OFF, D_IDS_VAL_OFF,
  D_IDS_WGT_OFF, D_IDS_NNZ, D_TOTAL_BYTES, D_FIELDS
};

struct IngestParams {
  const uint8_t* slab;
  int64_t slab_bytes;
  const int64_t* desc;
  int B_cap;
  int64_t nnz_cap;
  int num_float, F_idl, F_ids;
  float* dense;
  int32_t* idl_len;
  void* idl_off;
  int64_t* idl_val;
  int32_t* ids_len;
  void* ids_off;
  int64_t* ids_val;
  float* ids_wgt;
  int off64;
  int32_t* error;
};

struct Desc {
  int64_t v[D_FIELDS];
};

// a present section [off, off + bytes) must lie inside the slab's used bytes
__device__ __forceinline__ bool section_ok(int64_t off, int64_t bytes, int64_t total) {
  return bytes == 0 || (off >= 0 && off <= total && bytes <= total - off);
}

__device__ __forceinline__ bool desc_ok(const IngestParams& p, const Desc& d) {
  const int64_t B = d.v[D_B], total = d.v[D_TOTAL_BYTES];
  if (B < 0 || B > p.B_cap || total < 0 || total > p.slab_bytes) return false;
  if (d.v[D_NUM_FLOAT] != p.num_float || d.v[D_F_IDL] != p.F_idl || d.v[D_F_IDS] != p.F_ids) return false;
  const int64_t n1 = p.F_idl ? d.v[D_IDL_NNZ] : 0, n2 = p.F_ids ? d.v[D_IDS_NNZ] : 0;
  if (n1 < 0 || n1 > p.nnz_cap || n2 < 0 || n2 > p.nnz_cap) return false;
  return section_ok(d.v[D_DENSE_OFF], B * p.num_float * 4, total) && section_ok(d.v[D_IDL_LEN_OFF], B * p.F_idl * 4, total) &&
         section_ok(d.v[D_IDL_VAL_OFF], n1 * 8, total) && section_ok(d.v[D_IDS_LEN_OFF], B * p.F_ids * 4, total) &&
         section_ok(d.v[D_IDS_VAL_OFF], n2 * 8, total) && section_ok(d.v[D_IDS_WGT_OFF], n2 * 4, total);
}

// lengths [F * B] (stride B) -> lengths / offsets of stride B_cap, one block, tiles of kThreads * kItems bags with a running carry
__device__ void scan_lengths(const int32_t* __restrict__ src, int64_t B, int B_cap, int F, int64_t nnz, int32_t* __restrict__ len_out,
                             void* off_out, int off64, int32_t* error) {
  typedef cub::BlockScan<int64_t, kThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const int64_t N = (int64_t) F * B_cap;
  int64_t carry = 0;
  bool bad = false;
  if (threadIdx.x == 0) trb_st_idx(off_out, 0, off64, 0);
  for (int64_t base = 0; base < N; base += (int64_t) kThreads * kItems) {
    int64_t v[kItems];
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
      const int64_t i = base + (int64_t) threadIdx.x * kItems + j;
      int32_t l = 0;
      if (i < N) {
        const int64_t f = i / B_cap, b = i - f * B_cap;
        if (b < B) l = src[f * B + b];
        if (l < 0) {
          bad = true;
          l = 0;
        }
        len_out[i] = l;
      }
      v[j] = l;
    }
    int64_t tile_sum;
    Scan(tmp).InclusiveSum(v, v, tile_sum);
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
      const int64_t i = base + (int64_t) threadIdx.x * kItems + j;
      if (i < N) {
        const int64_t o = carry + v[j];
        trb_st_idx(off_out, i + 1, off64, o < nnz ? o : nnz);
      }
    }
    carry += tile_sum;
    __syncthreads();  // tmp is reused by the next tile
  }
  if (bad || (threadIdx.x == 0 && carry != nnz)) *error = 1;
}

// dst[0, n_total) = src[0, n_copy) followed by zeros, 16-byte vectors of EPV elements where both pointers allow it
template <int EPV, typename T>
__device__ __forceinline__ void copy_vec(T* __restrict__ dst, const T* __restrict__ src, int64_t n_copy, int64_t n_total, int64_t v) {
  const int64_t e0 = v * EPV;
  const bool aligned = ((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 15) == 0;
  if (aligned && e0 + EPV <= n_copy) {
    *reinterpret_cast<uint4*>(dst + e0) = *reinterpret_cast<const uint4*>(src + e0);
  } else if (aligned && e0 >= n_copy && e0 + EPV <= n_total) {
    *reinterpret_cast<uint4*>(dst + e0) = make_uint4(0u, 0u, 0u, 0u);
  } else {
    const int64_t e1 = e0 + EPV < n_total ? e0 + EPV : n_total;
    for (int64_t e = e0; e < e1; ++e) dst[e] = e < n_copy ? src[e] : T(0);
  }
}

__global__ void __launch_bounds__(kThreads) serve_ingest_kernel(const IngestParams p) {
  Desc d;
#pragma unroll
  for (int k = 0; k < D_FIELDS; ++k) d.v[k] = p.desc[k];
  if (!desc_ok(p, d)) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *p.error = 1;
    return;
  }
  const int64_t B = d.v[D_B];
  if (blockIdx.x == 0) {
    if (p.F_idl)
      scan_lengths(reinterpret_cast<const int32_t*>(p.slab + d.v[D_IDL_LEN_OFF]), B, p.B_cap, p.F_idl, d.v[D_IDL_NNZ], p.idl_len, p.idl_off,
                   p.off64, p.error);
    return;
  }
  if (blockIdx.x == 1) {
    if (p.F_ids)
      scan_lengths(reinterpret_cast<const int32_t*>(p.slab + d.v[D_IDS_LEN_OFF]), B, p.B_cap, p.F_ids, d.v[D_IDS_NNZ], p.ids_len, p.ids_off,
                   p.off64, p.error);
    return;
  }
  // one index space over the vectors of the four copies
  const int64_t dn_total = (int64_t) p.B_cap * p.num_float, dn_copy = B * p.num_float;
  const int64_t n1 = p.F_idl ? d.v[D_IDL_NNZ] : 0, n2 = p.F_ids ? d.v[D_IDS_NNZ] : 0;
  const int64_t v0 = (dn_total + 3) / 4, v1 = (n1 + 1) / 2, v2 = (n2 + 1) / 2, v3 = (n2 + 3) / 4;
  const int64_t V = v0 + v1 + v2 + v3;
  const int64_t stride = (int64_t) (gridDim.x - 2) * blockDim.x;
  for (int64_t v = (int64_t) (blockIdx.x - 2) * blockDim.x + threadIdx.x; v < V; v += stride) {
    if (v < v0) {
      copy_vec<4>(p.dense, reinterpret_cast<const float*>(p.slab + (dn_copy ? d.v[D_DENSE_OFF] : 0)), dn_copy, dn_total, v);
    } else if (v < v0 + v1) {
      copy_vec<2>(p.idl_val, reinterpret_cast<const int64_t*>(p.slab + d.v[D_IDL_VAL_OFF]), n1, n1, v - v0);
    } else if (v < v0 + v1 + v2) {
      copy_vec<2>(p.ids_val, reinterpret_cast<const int64_t*>(p.slab + d.v[D_IDS_VAL_OFF]), n2, n2, v - v0 - v1);
    } else {
      copy_vec<4>(p.ids_wgt, reinterpret_cast<const float*>(p.slab + d.v[D_IDS_WGT_OFF]), n2, n2, v - v0 - v1 - v2);
    }
  }
}

}  // namespace

// Descriptor fields of one batch (int64 each).
TRB_API int trb_serve_ingest_desc_fields() { return D_FIELDS; }

// slab: device copy of the batch slab (slab_bytes usable); desc: device int64 [trb_serve_ingest_desc_fields()].
// Outputs for a list with F == 0, and dense with num_float == 0, may be null. off64 selects int64 offsets. error: int32 flag the kernel
// sets to 1 (never clears), device or mapped host memory.
TRB_API int trb_serve_ingest(const void* slab, int64_t slab_bytes, const int64_t* desc, int B_cap, int64_t nnz_cap, int num_float, int F_idl,
                             int F_ids, float* dense, int32_t* idl_len, void* idl_off, int64_t* idl_val, int32_t* ids_len, void* ids_off,
                             int64_t* ids_val, float* ids_wgt, int off64, int32_t* error, cudaStream_t stream) {
  if (B_cap < 0 || nnz_cap < 0 || num_float < 0 || F_idl < 0 || F_ids < 0 || error == nullptr || desc == nullptr) return -1;
  if ((num_float && dense == nullptr) || (F_idl && (idl_len == nullptr || idl_off == nullptr || idl_val == nullptr)) ||
      (F_ids && (ids_len == nullptr || ids_off == nullptr || ids_val == nullptr || ids_wgt == nullptr)))
    return -1;
  IngestParams p;
  p.slab = reinterpret_cast<const uint8_t*>(slab);
  p.slab_bytes = slab_bytes;
  p.desc = desc;
  p.B_cap = B_cap;
  p.nnz_cap = nnz_cap;
  p.num_float = num_float;
  p.F_idl = F_idl;
  p.F_ids = F_ids;
  p.dense = dense;
  p.idl_len = idl_len;
  p.idl_off = idl_off;
  p.idl_val = idl_val;
  p.ids_len = ids_len;
  p.ids_off = ids_off;
  p.ids_val = ids_val;
  p.ids_wgt = ids_wgt;
  p.off64 = off64;
  p.error = error;
  // copy blocks sized for the bucket's capacity (the launch shape is part of a captured graph, so it cannot follow the batch)
  const int64_t vmax = ((int64_t) B_cap * num_float + 3) / 4 + (F_idl ? (nnz_cap + 1) / 2 : 0) + (F_ids ? (nnz_cap + 1) / 2 + (nnz_cap + 3) / 4 : 0);
  int64_t copy_blocks = (vmax + kThreads - 1) / kThreads;
  const int64_t max_blocks = 2 * (int64_t) trb_num_sms();
  copy_blocks = copy_blocks < 1 ? 1 : (copy_blocks > max_blocks ? max_blocks : copy_blocks);
  serve_ingest_kernel<<<(unsigned) (2 + copy_blocks), kThreads, 0, stream>>>(p);
  TRB_CHECK_LAUNCH();
  return 0;
}
