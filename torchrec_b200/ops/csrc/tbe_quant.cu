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
//
// Placed launches (template PLACED = true, entry point trb_qtbe_fwd_placed): every feature has an absolute row base, so one launch mixes
// tables in HBM with tables in pinned host memory (UVA: the kernel dereferences the host pointer, zero-copy over the host link). A host
// table may sit behind an HBM row cache: the row address is `slot >= 0 ? cache + slot * rb : host + id * rb`. A miss is served from host
// memory in the same kernel and claims the row for admission (slot map ABSENT -> PENDING, one claimant per row, appended to a bounded
// miss list); trb_qcache_admit then copies the claimed rows into slots picked by CLOCK. Serving tables are read-only, so an eviction
// never writes back, and what the cache holds never changes a result. The all-HBM launch (trb_qtbe_fwd_ex) runs the PLACED = false
// instances, which compile to exactly the kernels without placement.
#include "common.cuh"
#include <cuda_fp8.h>
#include <cstring>
#include <type_traits>

enum QFmt : int { FMT_FP32 = 0, FMT_FP16 = 1, FMT_BF16 = 2, FMT_INT8 = 3, FMT_INT4 = 4, FMT_INT2 = 5, FMT_FP8_BLOCK = 6 };

constexpr int32_t QC_ABSENT = -1;   // slot map: row not cached
constexpr int32_t QC_PENDING = -2;  // slot map: row claimed for admission by a lookup of this call

// One cached table (an array of these lives in device memory; ops/quant_tbe.py packs it as int64 words, field order matters).
struct QCacheTab {
  int32_t* slot_of_row;        // [rows] cache slot of a row, QC_ABSENT or QC_PENDING
  int64_t* row_of_slot;        // [slots] row held by a slot, -1 when empty
  uint8_t* ref;                // [slots] CLOCK reference bits (set by hits and by admission)
  uint8_t* cache;              // [slots, rb] cached rows (HBM)
  const uint8_t* host;         // [rows, rb] the table (pinned host memory)
  int64_t* miss;               // [cap] rows claimed by the lookups of one call
  int64_t* victim;             // [cap] slot picked for miss[i]
  int32_t* ctr;                // [2] claims of the current call (may exceed cap), admissions of the last admission call
  int64_t* hand;               // [1] CLOCK hand
  unsigned long long* stats;   // [4] lookups, hits, admissions, evictions
  int64_t slots, cap, rb;
};

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

// Parameters of a placed launch (weights / feat_woff unused there). A separate type, so the parameter block of the all-HBM kernels stays
// as it was: growing it changed their register allocation and spills.
struct QTbePlaced : QTbeParams {
  const int64_t* feat_base;   // address of row 0 of the feature's table (HBM or pinned host)
  const int32_t* feat_ctab;    // cached table of the feature, -1 when its rows are not cached
  const QCacheTab* ctabs;
  const int32_t* no_slot;      // one QC_ABSENT word: the slot-map load of an uncached feature
};

template <bool PLACED> using QP = std::conditional_t<PLACED, QTbePlaced, QTbeParams>;

// Where a placed bag reads its rows from.
struct QPlace {
  const uint8_t* base;
  const uint8_t* cache;
  const int32_t* smap;
  int ct;
};

__device__ __forceinline__ QPlace qplace(const QTbePlaced& p, int f) {
  QPlace q;
  q.base = reinterpret_cast<const uint8_t*>(p.feat_base[f]);
  q.ct = p.feat_ctab[f];
  if (q.ct >= 0) {
    q.cache = p.ctabs[q.ct].cache;
    q.smap = p.ctabs[q.ct].slot_of_row;
  } else {
    q.cache = q.base;
    q.smap = p.no_slot;
  }
  return q;
}

// Row `idx` (already clamped into the table) of a placed bag. The slot is an unconditional load (an uncached feature reads the constant
// QC_ABSENT word) and the select is on the address, never on loaded row data.
__device__ __forceinline__ const uint8_t* qrow(const QPlace& q, int64_t idx, int64_t rb, int32_t& slot) {
  slot = q.smap[q.ct >= 0 ? idx : 0];
  return slot >= 0 ? q.cache + (int64_t) slot * rb : q.base + idx * rb;
}

// Cache bookkeeping of one valid lookup of a cached table: a hit sets the slot's reference bit; a miss on an absent row claims it and
// appends it to the miss list (a claim that does not fit returns the row to ABSENT, so a later call can admit it).
__device__ __forceinline__ void qcache_note(const QCacheTab& t, int64_t idx, int32_t slot) {
  if (slot >= 0) {
    if (!t.ref[slot]) t.ref[slot] = 1;
  } else if (slot == QC_ABSENT && atomicCAS(t.slot_of_row + idx, QC_ABSENT, QC_PENDING) == QC_ABSENT) {
    const int32_t pos = atomicAdd(t.ctr, 1);
    if (pos < t.cap) t.miss[pos] = idx;
    else atomicExch(t.slot_of_row + idx, QC_ABSENT);
  }
}

// Per-thread lookup / hit counts of the cached table being served, flushed when the table changes and when the thread ends.
struct QCount {
  int ct = -1;
  unsigned long long lookups = 0, hits = 0;
  __device__ __forceinline__ void flush(const QCacheTab* tabs) {
    if (ct >= 0 && lookups) {
      atomicAdd(tabs[ct].stats, lookups);
      if (hits) atomicAdd(tabs[ct].stats + 1, hits);
    }
    lookups = hits = 0;
  }
  __device__ __forceinline__ void add(const QCacheTab* tabs, int c, int32_t slot) {
    if (c != ct) {
      flush(tabs);
      ct = c;
    }
    ++lookups;
    hits += slot >= 0;
  }
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

template <typename O, int MAXV, bool PLACED>
__global__ void __launch_bounds__(256) qtbe_fwd_kernel(const QP<PLACED> p) {
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
  const uint8_t* wbase;
  QPlace pl;
  QCount cnt;
  if constexpr (PLACED) pl = qplace(p, f);
  else wbase = p.weights + p.feat_woff[f];
  const int64_t start = trb_ld_idx(p.offsets, bag, p.off64);
  const int64_t end = trb_ld_idx(p.offsets, bag + 1, p.off64);
  float4 acc[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t l0 = start; l0 < end; l0 += 32) {
    const int n = (int) min((int64_t) 32, end - l0);
    int64_t my_idx = 0;
    float my_w = 0.f;
    const uint8_t* my_row = nullptr;
    if (lane < n) {
      my_idx = trb_ld_idx(p.indices, l0 + lane, p.idx64);
      my_w = p.psw ? p.psw[l0 + lane] : 1.f;
      const bool ok = my_idx >= 0 && my_idx < rows;
      if (!ok) { my_idx = 0; my_w = 0.f; }
      if constexpr (PLACED) {  // every lane resolves the row of its own id; the bag loop below shuffles the address
        int32_t slot;
        my_row = qrow(pl, my_idx, rb, slot);
        if (ok && pl.ct >= 0) {
          qcache_note(p.ctabs[pl.ct], my_idx, slot);
          cnt.add(p.ctabs, pl.ct, slot);
        }
      }
    }
    for (int j = 0; j < n; ++j) {
      const uint8_t* row;
      float w;
      if constexpr (PLACED) {
        row = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(my_row), j));
        w = __shfl_sync(0xffffffffu, my_w, j);
      } else {
        const int64_t idx = __shfl_sync(0xffffffffu, my_idx, j);
        w = __shfl_sync(0xffffffffu, my_w, j);
        row = wbase + idx * rb;
      }
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
  if constexpr (PLACED) cnt.flush(p.ctabs);
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

template <typename O, int FMT, int MAXV, int U, bool PLACED>
__global__ void __launch_bounds__(256, 3) qtbe_fwd_vec_kernel(const QP<PLACED> p) {
  constexpr int LPR = 8;
  constexpr int EPV = QVec<FMT>::EPV;
  const int lig = threadIdx.x & (LPR - 1);
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int64_t n_bags = (int64_t) p.F * p.B;
  const int64_t bag0 = group * U;
  if (bag0 >= n_bags) return;
  int64_t st[U], en[U];
  const uint8_t* wb[U];
  QPlace pl[U];
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
    if constexpr (PLACED) {
      pl[u] = qplace(p, f);
      wb[u] = pl[u].base;
    } else {
      wb[u] = p.weights + p.feat_woff[f];
    }
    st[u] = trb_ld_idx(p.offsets, bag, p.off64);
    en[u] = bag0 + u < n_bags ? trb_ld_idx(p.offsets, bag + 1, p.off64) : st[u];
  }
  // first id of every bag: all U x MAXV row vectors in flight before any is consumed
  uint4 q[U][MAXV];
  uint32_t sw[U][MAXV];
  float w0[U];
  const uint8_t* row0[U];
  int64_t idx0[U];   // placed: the valid first id of the bag (-1: none) and its slot, noted after every load is issued
  int32_t slot0[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    w0[u] = 0.f;
    row0[u] = wb[u];
    if constexpr (PLACED) idx0[u] = -1;
    if (en[u] > st[u]) {
      const int64_t idx = trb_ld_idx(p.indices, st[u], p.idx64);
      if (idx >= 0 && idx < rows[u]) {
        w0[u] = p.psw ? p.psw[st[u]] : 1.f;
        if constexpr (PLACED) {
          row0[u] = qrow(pl[u], idx, rb[u], slot0[u]);
          idx0[u] = idx;
        } else {
          row0[u] = wb[u] + idx * rb[u];
        }
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
  QCount cnt;
  if constexpr (PLACED) {
    if (lig == 0) {  // one lane of the 8 owning a bag keeps its books
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (idx0[u] >= 0 && pl[u].ct >= 0) {
          qcache_note(p.ctabs[pl[u].ct], idx0[u], slot0[u]);
          cnt.add(p.ctabs, pl[u].ct, slot0[u]);
        }
      }
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
      const uint8_t* row;
      if constexpr (PLACED) {
        int32_t slot;
        row = qrow(pl[u], idx, rb[u], slot);
        if (lig == 0 && pl[u].ct >= 0) {
          qcache_note(p.ctabs[pl[u].ct], idx, slot);
          cnt.add(p.ctabs, pl[u].ct, slot);
        }
      } else {
        row = wb[u] + idx * rb[u];
      }
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
  if constexpr (PLACED) cnt.flush(p.ctabs);
}

template <typename O, int FMT, bool PLACED>
static int launch_q_vec(const QP<PLACED>& p, int max_dim, cudaStream_t stream) {
  const int64_t n_bags = (int64_t) p.F * p.B;
  if (n_bags == 0) return 0;
  const int threads = 256;
  const int vecs = (max_dim + QVec<FMT>::EPV - 1) / QVec<FMT>::EPV;  // 16 B vectors per row; 8 lanes per bag
#define TRB_QVEC(MAXV, U)                                                                                     \
  {                                                                                                           \
    const int64_t groups = (n_bags + U - 1) / U;                                                              \
    const unsigned blocks = (unsigned) ((groups * 8 + threads - 1) / threads);                                \
    qtbe_fwd_vec_kernel<O, FMT, MAXV, U, PLACED><<<blocks, threads, 0, stream>>>(p);                          \
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
template <typename O, bool PLACED>
__global__ void __launch_bounds__(256) qtbe_seq_kernel(const QP<PLACED> p, int64_t total) {
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
  const uint8_t* row;
  if constexpr (PLACED) {
    const QPlace pl = qplace(p, f);
    int32_t slot;
    row = qrow(pl, ok ? idx : 0, p.feat_row_bytes[f], slot);
    if (lane == 0 && ok && pl.ct >= 0) {
      qcache_note(p.ctabs[pl.ct], idx, slot);
      QCount cnt;
      cnt.add(p.ctabs, pl.ct, slot);
      cnt.flush(p.ctabs);
    }
  } else {
    row = p.weights + p.feat_woff[f] + (ok ? idx : 0) * (int64_t) p.feat_row_bytes[f];
  }
  O* dst = reinterpret_cast<O*>(p.out) + i * p.out_stride;
  for (int vi = lane; vi < nvec; vi += 32) {
    float4 v = ok ? dequant4(row, p.feat_fmt[f], D, vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    Vec4<O>::st(dst + vi * 4, v);
  }
}

// ---- sequence scatter (fused sharded sequence inference, trb_qtbe_seq_scatter) ---------------------------------------------------------
// The ids of a launch were routed by trb_kjt_route_pos: `offsets` ([F * B + 1], region-absolute, the first entry need not be 0) slice the
// routed ids into units f, and pos[k] is the position of routed id k inside its feature's values. The dequantized row of id k of unit f is
// stored at out + feat_obase[f] + pos[k] * feat_ostride[f] + feat_col[f] (out: the flat sequence output on the first device, so from any
// other device these are peer stores). Ids outside the unit's rows store zeros.
template <bool PLACED>
struct QTbeScatter : QP<PLACED> {  // derived, so the parameter block of the qtbe_* instances above stays as it was
  const int64_t* feat_obase;   // element offset of the unit's feature block in `out`
  const int32_t* feat_ostride; // the feature's full width D_f
  const int32_t* pos;          // [routed ids] position of the id inside its feature's values
};

// Routed id of thread group t (region-absolute index) and its unit; false past the last routed id (the grid covers a host-side bound).
template <bool PLACED>
__device__ __forceinline__ bool qscatter_id(const QTbeScatter<PLACED>& p, int64_t t, int64_t& i, int& f) {
  i = trb_ld_idx(p.offsets, 0, p.off64) + t;
  if (i >= trb_ld_idx(p.offsets, (int64_t) p.F * p.B, p.off64)) return false;
  int lo = 0, hi = p.F - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (trb_ld_idx(p.offsets, (int64_t) mid * p.B, p.off64) <= i) lo = mid; else hi = mid - 1;
  }
  f = lo;
  return true;
}

// Row of a routed id (clamped to row 0 when invalid) with the cache bookkeeping of qtbe_seq_kernel, kept by lane `keeper` only.
template <bool PLACED>
__device__ __forceinline__ const uint8_t* qscatter_row(const QTbeScatter<PLACED>& p, int f, int64_t idx, bool ok, bool keeper) {
  if constexpr (PLACED) {
    const QPlace pl = qplace(p, f);
    int32_t slot;
    const uint8_t* row = qrow(pl, ok ? idx : 0, p.feat_row_bytes[f], slot);
    if (keeper && ok && pl.ct >= 0) {
      qcache_note(p.ctabs[pl.ct], idx, slot);
      QCount cnt;
      cnt.add(p.ctabs, pl.ct, slot);
      cnt.flush(p.ctabs);
    }
    return row;
  } else {
    return p.weights + p.feat_woff[f] + (ok ? idx : 0) * (int64_t) p.feat_row_bytes[f];
  }
}

template <typename O, bool PLACED>
__device__ __forceinline__ O* qscatter_dst(const QTbeScatter<PLACED>& p, int f, int64_t i) {
  return reinterpret_cast<O*>(p.out) + p.feat_obase[f] + (int64_t) p.pos[i] * p.feat_ostride[f] + p.feat_col[f];
}

// any row formats: one warp per routed id, 4 elements per lane (as qtbe_seq_kernel)
template <typename O, bool PLACED>
__global__ void __launch_bounds__(256) qtbe_seq_scatter_kernel(const QTbeScatter<PLACED> p, int64_t bound) {
  const int lane = threadIdx.x & 31;
  const int64_t t = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int64_t i;
  int f;
  if (t >= bound || !qscatter_id(p, t, i, f)) return;
  const int D = p.feat_dim[f];
  const int fmt = p.feat_fmt[f];
  const int64_t idx = trb_ld_idx(p.indices, i, p.idx64);
  const bool ok = idx >= 0 && idx < p.feat_rows[f];
  const uint8_t* row = qscatter_row(p, f, idx, ok, lane == 0);
  O* dst = qscatter_dst<O>(p, f, i);
  for (int vi = lane; vi < (D >> 2); vi += 32) {
    const float4 v = ok ? dequant4(row, fmt, D, vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    Vec4<O>::st(dst + vi * 4, v);
  }
}

// one of INT8 / FP8 block-scaled / FP16 / BF16 / INT4 for every table of the launch, rows of whole 16-byte vectors: 8 lanes per routed
// id, one 16 B vector (EPV elements) per lane and step (the loads and the dequantization of qtbe_fwd_vec_kernel)
template <typename O, int FMT, bool PLACED>
__global__ void __launch_bounds__(256) qtbe_seq_scatter_vec_kernel(const QTbeScatter<PLACED> p, int64_t bound) {
  constexpr int LPR = 8;
  constexpr int EPV = QVec<FMT>::EPV;
  const int lig = threadIdx.x & (LPR - 1);
  const int64_t t = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  int64_t i;
  int f;
  if (t >= bound || !qscatter_id(p, t, i, f)) return;
  const int D = p.feat_dim[f];
  const int64_t idx = trb_ld_idx(p.indices, i, p.idx64);
  const bool ok = idx >= 0 && idx < p.feat_rows[f];
  const uint8_t* row = qscatter_row(p, f, idx, ok, lig == 0);
  O* dst = qscatter_dst<O>(p, f, i);
  for (int e = lig * EPV; e < D; e += LPR * EPV) {
    float v[EPV];
    if (ok) {
      dequant_vec<FMT>(*reinterpret_cast<const uint4*>(row + (e / EPV) * 16), load_scale_vec<FMT>(row, D, e), v);
    } else {
#pragma unroll
      for (int k = 0; k < EPV; ++k) v[k] = 0.f;
    }
    store_vec<O, EPV>(dst + e, v);
  }
}

template <typename O, bool PLACED>
static int launch_q_scatter(const QTbeScatter<PLACED>& p, int64_t bound, int uniform_fmt, cudaStream_t stream) {
  const int threads = 256;
  const unsigned vec_blocks = (unsigned) ((bound * 8 + threads - 1) / threads);
  switch (uniform_fmt) {  // (the caller guarantees rows made of whole 16-byte vectors: quant_tbe.py _uniform_fmt)
    case FMT_FP8_BLOCK: qtbe_seq_scatter_vec_kernel<O, FMT_FP8_BLOCK, PLACED><<<vec_blocks, threads, 0, stream>>>(p, bound); break;
    case FMT_INT8: qtbe_seq_scatter_vec_kernel<O, FMT_INT8, PLACED><<<vec_blocks, threads, 0, stream>>>(p, bound); break;
    case FMT_FP16: qtbe_seq_scatter_vec_kernel<O, FMT_FP16, PLACED><<<vec_blocks, threads, 0, stream>>>(p, bound); break;
    case FMT_BF16: qtbe_seq_scatter_vec_kernel<O, FMT_BF16, PLACED><<<vec_blocks, threads, 0, stream>>>(p, bound); break;
    case FMT_INT4: qtbe_seq_scatter_vec_kernel<O, FMT_INT4, PLACED><<<vec_blocks, threads, 0, stream>>>(p, bound); break;
    default: qtbe_seq_scatter_kernel<O, PLACED><<<(unsigned) ((bound * 32 + threads - 1) / threads), threads, 0, stream>>>(p, bound);
  }
  TRB_CHECK_LAUNCH();
  return 0;
}

template <bool PLACED>
static int launch_q_scatter_out(const QTbeScatter<PLACED>& p, int out_dtype, int64_t bound, int uniform_fmt, cudaStream_t stream) {
  if (bound <= 0 || p.F == 0 || p.B == 0) return 0;
  switch (out_dtype) {
    case TRB_F32: return launch_q_scatter<float, PLACED>(p, bound, uniform_fmt, stream);
    case TRB_F16: return launch_q_scatter<__half, PLACED>(p, bound, uniform_fmt, stream);
    case TRB_BF16: return launch_q_scatter<__nv_bfloat16, PLACED>(p, bound, uniform_fmt, stream);
  }
  return -3;
}

template <typename O, bool PLACED>
static int launch_q(const QP<PLACED>& p, int max_dim, int64_t total, int uniform_fmt, cudaStream_t stream) {
  const int threads = 256;
  if (p.pooled && uniform_fmt >= 0) {  // (the caller guarantees rows made of whole 16-byte vectors: quant_tbe.py _uniform_fmt)
    if (uniform_fmt == FMT_FP8_BLOCK && max_dim <= 512) return launch_q_vec<O, FMT_FP8_BLOCK, PLACED>(p, max_dim, stream);
    if (uniform_fmt == FMT_INT8 && max_dim <= 512) return launch_q_vec<O, FMT_INT8, PLACED>(p, max_dim, stream);
    if (uniform_fmt == FMT_FP16 && max_dim <= 256) return launch_q_vec<O, FMT_FP16, PLACED>(p, max_dim, stream);
    if (uniform_fmt == FMT_BF16 && max_dim <= 256) return launch_q_vec<O, FMT_BF16, PLACED>(p, max_dim, stream);
    if (uniform_fmt == FMT_INT4 && max_dim <= 1024) return launch_q_vec<O, FMT_INT4, PLACED>(p, max_dim, stream);
  }
  if (!p.pooled) {
    if (total == 0) return 0;
    qtbe_seq_kernel<O, PLACED><<<(unsigned) ((total * 32 + threads - 1) / threads), threads, 0, stream>>>(p, total);
    TRB_CHECK_LAUNCH();
    return 0;
  }
  const int64_t n_bags = (int64_t) p.F * p.B;
  if (n_bags == 0) return 0;
  const unsigned blocks = (unsigned) ((n_bags * 32 + threads - 1) / threads);
  const int nvec = max_dim / 4;
  if (nvec <= 32) qtbe_fwd_kernel<O, 1, PLACED><<<blocks, threads, 0, stream>>>(p);
  else if (nvec <= 128) qtbe_fwd_kernel<O, 4, PLACED><<<blocks, threads, 0, stream>>>(p);
  else if (nvec <= 512) qtbe_fwd_kernel<O, 16, PLACED><<<blocks, threads, 0, stream>>>(p);
  else return -2;
  TRB_CHECK_LAUNCH();
  return 0;
}

template <bool PLACED>
static int launch_q_out(const QP<PLACED>& p, int out_dtype, int max_dim, int64_t total, int uniform_fmt, cudaStream_t stream) {
  switch (out_dtype) {
    case TRB_F32: return launch_q<float, PLACED>(p, max_dim, total, uniform_fmt, stream);
    case TRB_F16: return launch_q<__half, PLACED>(p, max_dim, total, uniform_fmt, stream);
    case TRB_BF16: return launch_q<__nv_bfloat16, PLACED>(p, max_dim, total, uniform_fmt, stream);
  }
  return -3;
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
  QTbeParams p{};
  p.weights = reinterpret_cast<const uint8_t*>(weights);
  p.feat_woff = feat_woff; p.feat_rows = feat_rows; p.feat_dim = feat_dim; p.feat_col = feat_col; p.feat_fmt = feat_fmt;
  p.feat_row_bytes = feat_row_bytes; p.indices = indices; p.offsets = offsets; p.psw = psw; p.out = out; p.out_stride = out_stride;
  p.B = B; p.F = F; p.idx64 = idx64; p.off64 = off64; p.mean = mean; p.pooled = pooled;
  return launch_q_out<false>(p, out_dtype, max_dim, total, uniform_fmt, stream);
}

// The same lookup over placed tables: `feat_base` = absolute address of row 0 of each feature's table (HBM or pinned host memory),
// `feat_ctab` = index into `ctabs` of the feature's HBM row cache or -1, `no_slot` = one device word holding QC_ABSENT (-1).
TRB_API int trb_qtbe_fwd_placed(const int64_t* feat_base, const int32_t* feat_ctab, const void* ctabs, const int32_t* no_slot, const int64_t* feat_rows,
                                const int32_t* feat_dim, const int32_t* feat_col, const int32_t* feat_fmt, const int32_t* feat_row_bytes, const void* indices,
                                int idx64, const void* offsets, int off64, const float* psw, void* out, int out_dtype, int64_t out_stride, int B, int F,
                                int max_dim, int mean, int pooled, int64_t total, int uniform_fmt, cudaStream_t stream) {
  QTbePlaced p{};
  p.feat_base = feat_base; p.feat_ctab = feat_ctab; p.ctabs = reinterpret_cast<const QCacheTab*>(ctabs); p.no_slot = no_slot;
  p.feat_rows = feat_rows; p.feat_dim = feat_dim; p.feat_col = feat_col; p.feat_fmt = feat_fmt;
  p.feat_row_bytes = feat_row_bytes; p.indices = indices; p.offsets = offsets; p.psw = psw; p.out = out; p.out_stride = out_stride;
  p.B = B; p.F = F; p.idx64 = idx64; p.off64 = off64; p.mean = mean; p.pooled = pooled;
  return launch_q_out<true>(p, out_dtype, max_dim, total, uniform_fmt, stream);
}

// Sequence scatter lookup over F units of B bags (see QTbeScatter). HBM tables: `weights` + `feat_woff`, `feat_base` null; placed tables
// (any of them in host memory or behind an HBM row cache): `feat_base`, `feat_ctab`, `ctabs`, `no_slot` as in trb_qtbe_fwd_placed.
// `bound` >= the number of routed ids of the launch (sizes the grid; the kernels stop at offsets[F * B]). `uniform_fmt` as in trb_qtbe_fwd_ex.
TRB_API int trb_qtbe_seq_scatter(const void* weights, const int64_t* feat_woff, const int64_t* feat_base, const int32_t* feat_ctab, const void* ctabs,
                                 const int32_t* no_slot, const int64_t* feat_rows, const int32_t* feat_dim, const int32_t* feat_col, const int32_t* feat_fmt,
                                 const int32_t* feat_row_bytes, const int64_t* feat_obase, const int32_t* feat_ostride, const void* indices, int idx64,
                                 const void* offsets, int off64, const int32_t* pos, void* out, int out_dtype, int B, int F, int64_t bound, int uniform_fmt,
                                 cudaStream_t stream) {
  auto fill = [&](auto& p) {
    p.feat_rows = feat_rows; p.feat_dim = feat_dim; p.feat_col = feat_col; p.feat_fmt = feat_fmt; p.feat_row_bytes = feat_row_bytes;
    p.indices = indices; p.offsets = offsets; p.psw = nullptr; p.out = out; p.out_stride = 0;
    p.B = B; p.F = F; p.idx64 = idx64; p.off64 = off64; p.mean = 0; p.pooled = 0;
    p.feat_obase = feat_obase; p.feat_ostride = feat_ostride; p.pos = pos;
  };
  if (feat_base != nullptr) {
    QTbeScatter<true> p{};
    fill(p);
    p.feat_base = feat_base; p.feat_ctab = feat_ctab; p.ctabs = reinterpret_cast<const QCacheTab*>(ctabs); p.no_slot = no_slot;
    return launch_q_scatter_out<true>(p, out_dtype, bound, uniform_fmt, stream);
  }
  QTbeScatter<false> p{};
  fill(p);
  p.weights = reinterpret_cast<const uint8_t*>(weights); p.feat_woff = feat_woff;
  return launch_q_scatter_out<false>(p, out_dtype, bound, uniform_fmt, stream);
}

// ---- admission: claimed misses -> HBM slots ---------------------------------------------------------------------------------------------
// One block per cached table picks the victims with CLOCK (second chance; one hand per table): the hand sweeps windows of up to 256
// slots, a slot with a clear reference bit is a victim, a set bit is cleared as the hand passes it. Admitted slots get their bit set, so
// a second lap clears them instead of taking them again: with at most `slots` admissions per call (cap <= slots) no slot is taken twice.
__global__ void __launch_bounds__(256) qcache_pick_kernel(const QCacheTab* tabs) {
  const QCacheTab t = tabs[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ int s_n, s_wcnt[8], s_stop;
  __shared__ unsigned long long s_evict;
  if (tid == 0) {
    s_n = (int) min((int64_t) *t.ctr, t.cap);
    s_evict = 0;
  }
  __syncthreads();
  const int n = s_n;
  const int width = (int) min((int64_t) blockDim.x, t.slots);
  int64_t hand = *t.hand;
  int taken = 0;
  while (taken < n) {
    const int64_t s = (hand + tid) % t.slots;
    const bool active = tid < width;
    const bool cand = active && t.ref[s] == 0;
    const unsigned bal = __ballot_sync(0xffffffffu, cand);
    if (lane == 0) s_wcnt[warp] = __popc(bal);
    if (tid == 0) s_stop = width;
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < 8; ++w) {
      before += w < warp ? s_wcnt[w] : 0;
      total += s_wcnt[w];
    }
    const int rank = before + __popc(bal & ((1u << lane) - 1u));
    const int want = n - taken;
    if (cand && rank == want - 1) s_stop = tid + 1;  // the hand stops right after the last victim it needs
    __syncthreads();
    const int stop = s_stop;
    if (tid < stop) {
      if (cand) {
        t.victim[taken + rank] = s;
        t.ref[s] = 1;  // taken: a later window of this call (the hand can wrap) sees it as referenced
      } else if (active) {
        t.ref[s] = 0;
      }
    }
    taken += min(total, want);
    hand = (hand + stop) % t.slots;
    __syncthreads();
  }
  // retire the victims' rows, hand the slots to the claimed rows (the copy and the slot-map update follow in qcache_fill_kernel)
  unsigned long long ev = 0;
  for (int i = tid; i < n; i += blockDim.x) {
    const int64_t s = t.victim[i];
    const int64_t old = t.row_of_slot[s];
    if (old >= 0) {
      t.slot_of_row[old] = QC_ABSENT;
      ++ev;
    }
    t.row_of_slot[s] = t.miss[i];
    t.ref[s] = 1;
  }
  if (ev) atomicAdd(&s_evict, ev);
  __syncthreads();
  if (tid == 0) {
    *t.hand = hand;
    t.ctr[0] = 0;
    t.ctr[1] = n;
    t.stats[2] += (unsigned long long) n;
    t.stats[3] += s_evict;
  }
}

// One warp per admitted row: host row -> HBM slot in 16-byte vectors, then the row becomes visible to lookups.
__global__ void __launch_bounds__(256) qcache_fill_kernel(const QCacheTab* tabs) {
  const QCacheTab& t = tabs[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= t.ctr[1]) return;
  const int64_t row = t.miss[i], slot = t.victim[i];
  const uint4* src = reinterpret_cast<const uint4*>(t.host + row * t.rb);
  uint4* dst = reinterpret_cast<uint4*>(t.cache + slot * t.rb);
  for (int64_t v = lane; v < t.rb / 16; v += 32) dst[v] = src[v];
  __syncwarp();
  if (lane == 0) {
    __threadfence();
    t.slot_of_row[row] = (int32_t) slot;
  }
}

// `tabs`: device array of `n_tabs` QCacheTab; `max_cap`: the largest miss-list capacity among them (grid of the copy). Everything the
// admission needs stays on the device, so a lookup followed by its admission can be captured in a CUDA graph.
TRB_API int trb_qcache_admit(const void* tabs, int n_tabs, int64_t max_cap, cudaStream_t stream) {
  if (n_tabs <= 0 || max_cap <= 0) return 0;
  const QCacheTab* t = reinterpret_cast<const QCacheTab*>(tabs);
  qcache_pick_kernel<<<n_tabs, 256, 0, stream>>>(t);
  TRB_CHECK_LAUNCH();
  qcache_fill_kernel<<<dim3((unsigned) ((max_cap + 7) / 8), (unsigned) n_tabs), 256, 0, stream>>>(t);
  TRB_CHECK_LAUNCH();
  return 0;
}

// ---- host tables ------------------------------------------------------------------------------------------------------------------------
// Pinned, mapped, portable host memory of exactly `bytes` bytes (zeroed): the caching pinned allocator of PyTorch rounds a request up to a
// power of two, which for a 40 GB table pins 64 GB. With UVA the host pointer is also the device pointer on every device.
TRB_API int trb_host_alloc(int64_t bytes, void** out) {
  *out = nullptr;
  if (bytes <= 0) return 0;
  TRB_CUDA(cudaHostAlloc(out, (size_t) bytes, cudaHostAllocPortable | cudaHostAllocMapped));
  std::memset(*out, 0, (size_t) bytes);
  return 0;
}

TRB_API int trb_host_free(void* p) {
  if (p) TRB_CUDA(cudaFreeHost(p));
  return 0;
}
