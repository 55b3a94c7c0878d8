// Hand-written sm_90a GEMM for the dense DLRM arch: C[M,N] = act(alpha * A[M,K] . B[N,K]^T + bias) with
// bf16 operands staged by TMA (SWIZZLE_128B) into an mbarrier ring, wgmma (m64nNk16) accumulating in registers
// and a fused epilogue (bias, ReLU / sigmoid, ReLU-gradient mask, ReLU bit mask, bias-gradient column sums,
// bf16 / fp32 store or split-K fp32 reduction).
//
// Structure (one 128 x BN output tile per CTA, two CTAs per SM so that one CTA's epilogue overlaps the other's MMAs):
//   warps 0..3  consumer warpgroup 0   rows [0, 64) of the tile:   4 x wgmma m64nBNk16 per 64-wide k-block
//   warps 4..7  consumer warpgroup 1   rows [64, 128) of the tile
//   warp 8      TMA producer           cp.async.bulk.tensor.2d -> smem ring (kStages x (A 128x64, B BNx64))
// A consumer keeps one wgmma group in flight and releases the previous k-block's slot when it retires.
//
// Both operands may be K-major (row-major [rows, K], the natural layout of nn.Linear: x [M,K], weight [N,K]) or
// MN-major ([K, rows], consumed transposed by wgmma), so dgrad / wgrad need no transpose copies.
// Replaces the reference's cuBLAS nn.Linear + separate bias/ReLU kernels (modules/mlp.py:18-190).
#include <cstdlib>

#include "wgmma.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 B = one SWIZZLE_128B row
constexpr int WGMMA_K = 16;
constexpr int kConsumerThreads = 256;
constexpr int kNumThreads = kConsumerThreads + 32;
constexpr int kProducerWarp = 8;

using namespace trb;

enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_SIGMOID = 2, ACT_RELU_GRAD = 3 };

struct GemmParams {
  int M, N, K;
  const float* bias;            // [N] or nullptr
  const __nv_bfloat16* mask;    // ACT_RELU_GRAD: out *= (mask[m, n] > 0)
  int64_t ld_mask;
  void* out;
  int64_t ldo;
  int out_f32;                  // 1: fp32 output, 0: bf16
  int act;
  float alpha;                  // scale applied to the accumulator before bias
  int split_k;                  // >1: K range split over CTAs, fp32 atomic epilogue (out pre-zeroed)
  // 1 bit per element instead of re-reading the bf16 activation as the ReLU-gradient mask (67 MB -> 4 MB for 32768 x 1024):
  uint32_t* relu_bits_out;      // ACT_RELU: bit (n % 32) of word [m, n / 32] = (out[m, n] > 0); nullptr: not wanted
  const uint32_t* mask_bits;    // ACT_RELU_GRAD: the same words of the layer whose gradient this is; nullptr: use `mask`
  int64_t ld_bits;              // words per row of either bit matrix
  // bias gradient of the layer that produced this GEMM's input gradient, folded into the epilogue: the column sums of every
  // 32-row slab of the bf16 output go to colsum_ws[row0 / 32][n] ([ceil(M / 32), N], deterministic; reduced by
  // trb_colsum_partials). nullptr: not wanted.
  float* colsum_ws;
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int BN>
struct SmemLayout {
  static constexpr int kStages = BN == 128 ? 3 : 4;   // 96 KB of operand ring: two CTAs per SM
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BN * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kColsumOffset = kStages * kStageBytes;          // [2 warpgroups][2 slabs][BN] fp32
  static constexpr int kBarOffset = kColsumOffset + 4 * BN * 4;
  static constexpr int kTotal = kBarOffset + 2 * kStages * 8;
};

// Epilogue of one consumer warpgroup: rows [row0, row0 + 64) x cols [n0, n0 + BN) of the output.
// ACT / BIAS are compile-time so the unrolled loop carries no runtime branches on them.
template <int BN, int ACT, bool BIAS>
__device__ __forceinline__ void epilogue_impl(const GemmParams& p, float (&acc)[BN / 2], int row0, int n0, int wq, int lane, float* colsum_s) {
  const int q = lane & 3;
  const int rows[2] = {row0 + 16 * wq + (lane >> 2), row0 + 16 * wq + (lane >> 2) + 8};
  const bool row_ok[2] = {rows[0] < p.M, rows[1] < p.M};
  const bool want_colsum = p.colsum_ws != nullptr;
  const bool use_bits = (ACT == ACT_RELU_GRAD) && p.mask_bits != nullptr;
  uint32_t obits[2] = {0u, 0u};
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * q;
    const bool col_ok = col < p.N;  // N % 8 == 0: col + 1 < N as well
    float2 b2 = make_float2(0.f, 0.f);
    if constexpr (BIAS) {
      if (col_ok) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + col));
    }
    float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = acc[4 * j + 2 * h] * p.alpha, v1 = acc[4 * j + 2 * h + 1] * p.alpha;
      if constexpr (BIAS) {
        v0 += b2.x;
        v1 += b2.y;
      }
      const bool ok = row_ok[h] && col_ok;
      if constexpr (ACT == ACT_RELU) {
        v0 = fmaxf(v0, 0.f);
        v1 = fmaxf(v1, 0.f);
        obits[h] |= ((v0 > 0.f ? 1u : 0u) | (v1 > 0.f ? 2u : 0u)) << (8 * (j & 3) + 2 * q);
      } else if constexpr (ACT == ACT_SIGMOID) {
        v0 = 1.f / (1.f + __expf(-v0));
        v1 = 1.f / (1.f + __expf(-v1));
      } else if constexpr (ACT == ACT_RELU_GRAD) {
        if (ok) {
          if (use_bits) {
            const uint32_t w = __ldg(p.mask_bits + (int64_t) rows[h] * p.ld_bits + (col >> 5)) >> (col & 31);
            v0 = (w & 1u) ? v0 : 0.f;
            v1 = (w & 2u) ? v1 : 0.f;
          } else {
            const __nv_bfloat162 m2 = *reinterpret_cast<const __nv_bfloat162*>(p.mask + (int64_t) rows[h] * p.ld_mask + col);
            v0 = __bfloat162float(m2.x) > 0.f ? v0 : 0.f;
            v1 = __bfloat162float(m2.y) > 0.f ? v1 : 0.f;
          }
        }
      }
      if (ok) {
        if (p.split_k > 1) {
          float* o = reinterpret_cast<float*>(p.out) + (int64_t) rows[h] * p.ldo + col;
          atomicAdd(o, v0);
          atomicAdd(o + 1, v1);
        } else if (p.out_f32) {
          *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + (int64_t) rows[h] * p.ldo + col) = make_float2(v0, v1);
        } else {
          const uint32_t o = pack_bf16x2(v0, v1);
          *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (int64_t) rows[h] * p.ldo + col) = o;
          if (want_colsum) {  // sums of the stored bf16 values, so the result equals a column sum of the output tensor
            cs0 += __uint_as_float(o << 16);
            cs1 += __uint_as_float(o & 0xffff0000u);
          }
        }
      }
    }
    if constexpr (ACT == ACT_RELU) {
      if ((j & 3) == 3 && p.relu_bits_out != nullptr) {
        // the 4 lanes of a quad hold the 32 columns of one word of the same row
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          obits[h] |= __shfl_xor_sync(0xffffffffu, obits[h], 1);
          obits[h] |= __shfl_xor_sync(0xffffffffu, obits[h], 2);
          const int wcol = n0 + 8 * (j - 3);
          if (q == 0 && row_ok[h] && wcol < p.N) p.relu_bits_out[(int64_t) rows[h] * p.ld_bits + (wcol >> 5)] = obits[h];
          obits[h] = 0u;
        }
      }
    }
    if (want_colsum) {
      // this warp's 16 rows: fold the 8 lanes that share the columns (fixed order -> deterministic)
      float s0 = cs0, s1 = cs1;
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      }
      if (lane < 4 && (wq & 1)) *reinterpret_cast<float2*>(colsum_s + (wq >> 1) * BN + 8 * j + 2 * q) = make_float2(s0, s1);
      cs0 = s0;
      cs1 = s1;
      acc[4 * j] = s0;  // (the accumulator is dead after the store above: keep the 16-row sums for the pairing step below)
      acc[4 * j + 1] = s1;
    }
  }
  if (want_colsum) {
    // warps (0, 1) and (2, 3) of the warpgroup hold the two 16-row halves of a 32-row slab: the even warp adds the odd one's
    asm volatile("bar.sync %0, 128;" ::"r"(1 + (int) (threadIdx.x >> 7)) : "memory");  // named barrier of this warpgroup
    const int slab_row0 = row0 + 32 * (wq >> 1);
    if (!(wq & 1) && lane < 4 && slab_row0 < p.M) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + 2 * q;
        if (col < p.N) {
          const float2 o = *reinterpret_cast<const float2*>(colsum_s + (wq >> 1) * BN + 8 * j + 2 * q);
          *reinterpret_cast<float2*>(p.colsum_ws + (int64_t) (slab_row0 >> 5) * p.N + col) = make_float2(acc[4 * j] + o.x, acc[4 * j + 1] + o.y);
        }
      }
    }
  }
}

template <int BN>
__device__ __forceinline__ void epilogue(const GemmParams& p, float (&acc)[BN / 2], int row0, int n0, int wq, int lane, float* colsum_s) {
#define TRB_EPI(A, B) epilogue_impl<BN, A, B>(p, acc, row0, n0, wq, lane, colsum_s)
  const bool bias = p.bias != nullptr;
  switch (p.act) {
    case ACT_RELU: if (bias) TRB_EPI(ACT_RELU, true); else TRB_EPI(ACT_RELU, false); break;
    case ACT_SIGMOID: if (bias) TRB_EPI(ACT_SIGMOID, true); else TRB_EPI(ACT_SIGMOID, false); break;
    case ACT_RELU_GRAD: if (bias) TRB_EPI(ACT_RELU_GRAD, true); else TRB_EPI(ACT_RELU_GRAD, false); break;
    default: if (bias) TRB_EPI(ACT_NONE, true); else TRB_EPI(ACT_NONE, false); break;
  }
#undef TRB_EPI
}

template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint32_t a_addr, uint32_t b_addr) {
#pragma unroll
  for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
    // K-major: +32 B inside the 128 B swizzle row; MN-major: 16 reduction rows x 128 B = 2048 B
    const uint64_t ad = A_MN ? make_smem_desc(a_addr + k * 2048, 8192, 1024) : make_kmajor_desc(a_addr + k * 32);
    const uint64_t bd = B_MN ? make_smem_desc(b_addr + k * 2048, 8192, 1024) : make_kmajor_desc(b_addr + k * 32);
    if constexpr (BN == 128) wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, ad, bd);
    else wgmma_m64n64k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, ad, bd);
  }
}

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kNumThreads, 2)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const GemmParams p) {
  using L = SmemLayout<BN>;
  constexpr int kStages = L::kStages;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem is only guaranteed 16 B aligned: round up to 1024 B for SWIZZLE_128B
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = (p.N + BN - 1) / BN;
  const int k_blocks_total = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int splits = p.split_k > 1 ? p.split_k : 1;
  const int kb_per_split = (k_blocks_total + splits - 1) / splits;
  const int mn_tiles = m_tiles * n_tiles;
  const int mn = (int) blockIdx.x % mn_tiles, ks = (int) blockIdx.x / mn_tiles;
  const int m_blk = mn / n_tiles, n_blk = mn % n_tiles;
  const int kb0 = ks * kb_per_split, kb1 = min(k_blocks_total, kb0 + kb_per_split);

  if (warp_idx == kProducerWarp) {
    // ================= TMA producer =================
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_a)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_b)) : "memory");
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * L::kStageBytes;
        uint8_t* sb = sa + L::kABytes;
        mbar_arrive_expect_tx(&full_bar[stage], L::kStageBytes);
        if constexpr (A_MN) {
          // MN-major operand: the matrix is [reduction rows, MN cols]; one 64-column atom ([64 rows x 128 B]) per load
#pragma unroll
          for (int h = 0; h < BLOCK_M / 64; ++h) tma_load_2d(&tmap_a, &full_bar[stage], sa + h * 8192, m_blk * BLOCK_M + 64 * h, kb * BLOCK_K);
        } else {
          tma_load_2d(&tmap_a, &full_bar[stage], sa, kb * BLOCK_K, m_blk * BLOCK_M);
        }
        if constexpr (B_MN) {
#pragma unroll
          for (int h = 0; h < BN / 64; ++h) tma_load_2d(&tmap_b, &full_bar[stage], sb + h * 8192, n_blk * BN + 64 * h, kb * BLOCK_K);
        } else {
          tma_load_2d(&tmap_b, &full_bar[stage], sb, kb * BLOCK_K, n_blk * BN);
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ================= consumers =================
  const int wg = warp_idx >> 2;  // rows [64 wg, 64 wg + 64) of the tile
  const int wq = warp_idx & 3;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  // A rows of this warpgroup: K-major = 64 rows x 128 B further; MN-major = the second 64-column atom
  const uint32_t a_off = (uint32_t) wg * 8192u;
  int stage = 0, prev_stage = 0;
  uint32_t phase = 0;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a_addr = smem_u32(smem + stage * L::kStageBytes) + a_off;
    const uint32_t b_addr = smem_u32(smem + stage * L::kStageBytes + L::kABytes);
    wgmma_fence();
    mma_kblock<BN, A_MN, B_MN>(acc, a_addr, b_addr);
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's wgmmas retired: its smem slot is free
    wgmma_fence_regs(acc);
    if (kb > kb0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
    prev_stage = stage;
    if (++stage == kStages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  // (no arrival for the last slot: nothing is loaded after this tile's last k-block)
  epilogue<BN>(p, acc, m_blk * BLOCK_M + 64 * wg, n_blk * BN, wq, lane, reinterpret_cast<float*>(smem + L::kColsumOffset) + wg * 2 * BN);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// rows x K bf16 matrix, row pitch ld elements; box = [box_cols, box_rows], SWIZZLE_128B
int make_tmap(CUtensorMap* map, const void* ptr, int64_t rows, int64_t K, int64_t ld, int box_rows, int box_cols = BLOCK_K) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return -10;
  cuuint64_t dims[2] = {(cuuint64_t) K, (cuuint64_t) rows};
  cuuint64_t strides[1] = {(cuuint64_t) ld * 2};
  cuuint32_t box[2] = {(cuuint32_t) box_cols, (cuuint32_t) box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -11;
}

template <int BN, bool A_MN, bool B_MN>
int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  constexpr int smem_bytes = SmemLayout<BN>::kTotal + 1024;
  static bool configured = false;
  if (!configured) {
    TRB_CUDA(cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<BN, A_MN, B_MN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    configured = true;
  }
  const int64_t tiles = (int64_t) ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BN - 1) / BN) * (p.split_k > 1 ? p.split_k : 1);
  if (tiles > 0x7fffffff) return -12;
  gemm_bf16_wgmma_kernel<BN, A_MN, B_MN><<<(unsigned) tiles, kNumThreads, smem_bytes, stream>>>(ta, tb, p);
  TRB_CHECK_LAUNCH();
  return 0;
}

}  // namespace

// C[M,N] = act(alpha * op(A) . op(B)^T + bias), bf16 operands, fp32 accumulation.
//   a_mn == 0: A is [M, K] row-major (K-major operand)      a_mn == 1: A is [K, M] row-major (MN-major operand)
//   b_mn == 0: B is [N, K] row-major                        b_mn == 1: B is [K, N] row-major
// Pitches lda/ldb in elements (multiples of 8). out: bf16 or fp32 with pitch ldo.
template <bool A_MN, bool B_MN>
static int gemm_dispatch(const void* A, int64_t lda, const void* B, int64_t ldb, GemmParams& p, cudaStream_t stream) {
  CUtensorMap ta, tb;
  int rc = A_MN ? make_tmap(&ta, A, p.K, p.M, lda, 64, 64) : make_tmap(&ta, A, p.M, p.K, lda, BLOCK_M);
  if (rc) return rc;
  if (p.colsum_ws != nullptr && (p.out_f32 || p.split_k > 1)) return -14;  // column sums of a bf16 output without split-K only
  if (p.N <= 64) {
    rc = B_MN ? make_tmap(&tb, B, p.K, p.N, ldb, 64, 64) : make_tmap(&tb, B, p.N, p.K, ldb, 64);
    if (rc) return rc;
    return launch_gemm<64, A_MN, B_MN>(ta, tb, p, stream);
  }
  rc = B_MN ? make_tmap(&tb, B, p.K, p.N, ldb, 64, 64) : make_tmap(&tb, B, p.N, p.K, ldb, 128);
  if (rc) return rc;
  return launch_gemm<128, A_MN, B_MN>(ta, tb, p, stream);
}

TRB_API int trb_gemm_bf16_ex2(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* out, int64_t ldo, int out_f32, int M,
                              int N, int K, const float* bias, int act, const void* mask, int64_t ld_mask, float alpha, int split_k, int tile_n,
                              const void* mask_bits, void* relu_bits_out, int64_t ld_bits, cudaStream_t stream);

TRB_API int trb_gemm_bf16_ex(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* out, int64_t ldo, int out_f32, int M,
                             int N, int K, const float* bias, int act, const void* mask, int64_t ld_mask, float alpha, int split_k, int tile_n,
                             cudaStream_t stream) {
  return trb_gemm_bf16_ex2(A, lda, a_mn, B, ldb, b_mn, out, ldo, out_f32, M, N, K, bias, act, mask, ld_mask, alpha, split_k, tile_n, nullptr, nullptr, 0,
                           stream);
}

// mask_bits / relu_bits_out: int32 [M, ld_bits] bit matrices (bit n % 32 of word n / 32), see GemmParams
TRB_API int trb_gemm_bf16_ex3(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* out, int64_t ldo, int out_f32, int M,
                              int N, int K, const float* bias, int act, const void* mask, int64_t ld_mask, float alpha, int split_k, int tile_n,
                              const void* mask_bits, void* relu_bits_out, int64_t ld_bits, float* colsum_ws, cudaStream_t stream);

TRB_API int trb_gemm_bf16_ex2(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* out, int64_t ldo, int out_f32, int M,
                              int N, int K, const float* bias, int act, const void* mask, int64_t ld_mask, float alpha, int split_k, int tile_n,
                              const void* mask_bits, void* relu_bits_out, int64_t ld_bits, cudaStream_t stream) {
  return trb_gemm_bf16_ex3(A, lda, a_mn, B, ldb, b_mn, out, ldo, out_f32, M, N, K, bias, act, mask, ld_mask, alpha, split_k, tile_n, mask_bits, relu_bits_out,
                           ld_bits, nullptr, stream);
}

// colsum_ws: fp32 [ceil(M / 32), N] or nullptr, see GemmParams (bf16 output without split-K only: -14 otherwise).
// tile_n: tile-width hint of the caller's split-K plan; this kernel has one tile shape per N (128 x 64 or 128 x 128).
TRB_API int trb_gemm_bf16_ex3(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* out, int64_t ldo, int out_f32, int M,
                              int N, int K, const float* bias, int act, const void* mask, int64_t ld_mask, float alpha, int split_k, int tile_n,
                              const void* mask_bits, void* relu_bits_out, int64_t ld_bits, float* colsum_ws, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 8) || (ldb % 8) || (N % 8)) return -12;
  if ((!a_mn && (K % 8)) || (a_mn && (M % 8)) || (b_mn && (N % 8)) || (!b_mn && (K % 8))) return -12;
  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.bias = bias;
  p.mask = reinterpret_cast<const __nv_bfloat16*>(mask);
  p.ld_mask = ld_mask;
  p.out = out;
  p.ldo = ldo;
  p.out_f32 = out_f32;
  p.act = act;
  p.alpha = alpha;
  p.split_k = 1;
  p.mask_bits = reinterpret_cast<const uint32_t*>(mask_bits);
  p.relu_bits_out = reinterpret_cast<uint32_t*>(relu_bits_out);
  p.ld_bits = ld_bits;
  p.colsum_ws = colsum_ws;
  if ((mask_bits != nullptr || relu_bits_out != nullptr) && ld_bits * 32 < N) return -12;
  if (split_k > 1) {
    if (!out_f32 || bias != nullptr || act != ACT_NONE) return -13;  // split-K only for plain fp32 accumulation
    const int kb = (K + BLOCK_K - 1) / BLOCK_K;
    int s = split_k < kb ? split_k : kb;
    const int per = (kb + s - 1) / s;
    s = (kb + per - 1) / per;  // no empty splits
    p.split_k = s;
    if (s > 1) TRB_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * (size_t) M * (size_t) ldo, stream));
  }
  if (a_mn && b_mn) return gemm_dispatch<true, true>(A, lda, B, ldb, p, stream);
  if (a_mn) return gemm_dispatch<true, false>(A, lda, B, ldb, p, stream);
  if (b_mn) return gemm_dispatch<false, true>(A, lda, B, ldb, p, stream);
  return gemm_dispatch<false, false>(A, lda, B, ldb, p, stream);
}

TRB_API int trb_gemm_bf16(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* out, int64_t ldo, int out_f32, int M,
                          int N, int K, const float* bias, int act, const void* mask, int64_t ld_mask, float alpha, int split_k,
                          cudaStream_t stream) {
  return trb_gemm_bf16_ex(A, lda, a_mn, B, ldb, b_mn, out, ldo, out_f32, M, N, K, bias, act, mask, ld_mask, alpha, split_k, 0, stream);
}

TRB_API int trb_gemm_bf16_tn(const void* A, int64_t lda, const void* B, int64_t ldb, void* out, int64_t ldo, int out_f32, int M, int N, int K,
                             const float* bias, int act, const void* mask, int64_t ld_mask, float alpha, int split_k, cudaStream_t stream) {
  return trb_gemm_bf16(A, lda, 0, B, ldb, 0, out, ldo, out_f32, M, N, K, bias, act, mask, ld_mask, alpha, split_k, stream);
}

// ---- helpers used around the GEMM ----------------------------------------------------------------------
// bf16 transpose: out[c, r] = in[r, c]; 32x32 smem tiles, coalesced both ways.
__global__ void __launch_bounds__(256) trb_transpose_bf16_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int rows,
                                                                   int cols, int64_t ld_in, int64_t ld_out) {
  __shared__ __nv_bfloat16 tile[32][34];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int r = by + i, c = bx + tx;
    tile[i][tx] = (r < rows && c < cols) ? in[(int64_t) r * ld_in + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = bx + i, r = by + tx;
    if (c < cols && r < rows) out[(int64_t) c * ld_out + r] = tile[tx][i];
  }
}

TRB_API int trb_transpose_bf16(const void* in, void* out, int rows, int cols, int64_t ld_in, int64_t ld_out, cudaStream_t stream) {
  if (rows == 0 || cols == 0) return 0;
  dim3 grid((cols + 31) / 32, (rows + 31) / 32);
  trb_transpose_bf16_kernel<<<grid, 256, 0, stream>>>((const __nv_bfloat16*) in, (__nv_bfloat16*) out, rows, cols, ld_in, ld_out);
  TRB_CHECK_LAUNCH();
  return 0;
}

// column sums of a bf16 [rows, cols] matrix into fp32 (bias gradient). Each thread owns 8 columns
// (one 16 B load per row) and strides over rows; 8 row lanes per block are reduced through smem and
// the block result is added atomically (blocks tile the rows so the whole chip participates).
__global__ void __launch_bounds__(256) trb_colsum_bf16_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, int rows, int cols,
                                                                int64_t ld, int rows_per_block) {
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int vec = blockIdx.x * 32 + tx;  // 8-column group
  const int nvec = cols >> 3;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(rows, r0 + rows_per_block);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (vec < nvec) {
    for (int r = r0 + ty; r < r1; r += 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(in + (int64_t) r * ld + vec * 8);
      const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += __bfloat162float(b[j]);
    }
  }
  __shared__ float red[8][32][9];
#pragma unroll
  for (int j = 0; j < 8; ++j) red[ty][tx][j] = acc[j];
  __syncthreads();
  if (ty == 0 && vec < nvec) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += red[i][tx][j];
      atomicAdd(out + vec * 8 + j, s);
    }
  }
}

// v3: contended fp32 atomics were the bottleneck of v1 (every 128 B line of `out` took rows/256 x 32 serialized L2 atomics).
// Now: (a) ~4 blocks per SM, each walking a tall row slab with 8 independent 16 B loads in flight per
// thread, (b) narrow matrices fold several rows into one warp (vpr = lanes per row) so every lane loads, (c) block partials
// go to a workspace and the LAST block of a column group (ticket counter) sums them in a fixed order: no float atomics,
// deterministic result, one launch.
template <bool CLUSTER>
__device__ __forceinline__ void colsum_v3_body(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, int rows, int cols, int64_t ld,
                                               int rows_per_block, int vpr_log2, float* __restrict__ partial, unsigned int* __restrict__ tickets) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int vpr = 1 << vpr_log2, rpw = 32 >> vpr_log2;  // lanes per row, rows per warp
  const int sub = lane >> vpr_log2;
  const int vec = blockIdx.x * 32 + (lane & (vpr - 1));
  const int nvec = cols >> 3;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(rows, r0 + rows_per_block);
  const int step = 8 * rpw;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (vec < nvec) {
    const __nv_bfloat16* base = in + vec * 8;
    int r = r0 + warp * rpw + sub;
    constexpr int U = 8;  // independent 16 B loads in flight per thread
    for (; r + (U - 1) * step < r1; r += U * step) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(base + (int64_t) (r + u * step) * ld));
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&v[u]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __bfloat1622float2(b[j]);
          acc[2 * j] += f.x;
          acc[2 * j + 1] += f.y;
        }
      }
    }
    for (; r < r1; r += step) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(base + (int64_t) r * ld));
      const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __bfloat1622float2(b[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
  }
  // fold the row lanes of a warp, then the 8 warps through smem
  for (int o = vpr; o < 32; o <<= 1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
  }
  __shared__ float red[8][32][9];
  __shared__ unsigned int s_ticket;
  if (sub == 0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) red[warp][lane][j] = acc[j];
  }
  __syncthreads();
  // thread t owns column (blockIdx.x * 256 + t) of this block's 256-column group: vec lane t >> 3, element t & 7
  const int l = threadIdx.x >> 3, j = threadIdx.x & 7;
  const int col = blockIdx.x * 256 + threadIdx.x;
  const bool col_ok = l < vpr && col < cols;
  float s = 0.f;
  if (col_ok) {
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][l][j];
  }
  // CLUSTER: the 8 CTAs of a (1,8,1) cluster first fold their column sums through the leader's shared memory (DSMEM), so a
  // launch produces gridDim.y / 8 partials: short row slabs per thread (4 batches of 8 loads) AND a short last-block tail.
  int n_part = (int) gridDim.y, my_part = (int) blockIdx.y;
  if constexpr (CLUSTER) {
    __shared__ float cl[8][256];
    const uint32_t rank = cluster_ctarank();
    const uint32_t dst = mapa_shared(smem_u32(&cl[rank][threadIdx.x]), 0);
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(dst), "f"(s) : "memory");
    cluster_sync_all();
    if (rank != 0) return;
    s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += cl[i][threadIdx.x];
    n_part = (int) gridDim.y >> 3;
    my_part = (int) blockIdx.y >> 3;
  }
  if (n_part == 1) {
    if (col_ok) out[col] = s;
    return;
  }
  if (col_ok) partial[(int64_t) my_part * cols + col] = s;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_ticket = atomicAdd(&tickets[blockIdx.x], 1u);
  __syncthreads();
  if (s_ticket != (unsigned) n_part - 1) return;
  __threadfence();
  // last block of this column group: fixed-order sum of the partials. C = vpr * 8 columns; 256 / C thread groups split the
  // partial rows, 8 loads in flight each, then one smem pass over the groups
  {
    const int C = vpr * 8, G = 256 / C;
    const int c = threadIdx.x & (C - 1), g = threadIdx.x / C;
    const int gcol = blockIdx.x * 256 + c;
    float s = 0.f;
    if (gcol < cols) {
      const float* pc = partial + gcol;
      int y = g;
      for (; y + 7 * G < n_part; y += 8 * G) {
        float t[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) t[u] = __ldcg(pc + (int64_t) (y + u * G) * cols);
#pragma unroll
        for (int u = 0; u < 8; ++u) s += t[u];
      }
      for (; y < n_part; y += G) s += __ldcg(pc + (int64_t) y * cols);
    }
    float* fin = &red[0][0][0];  // 256 floats needed, 2304 available; all earlier reads of red are done (barriers above)
    fin[threadIdx.x] = s;
    __syncthreads();
    if (g == 0 && gcol < cols) {
      float tot = 0.f;
      for (int i = 0; i < G; ++i) tot += fin[i * C + c];
      out[gcol] = tot;
    }
  }
  if (threadIdx.x == 0) tickets[blockIdx.x] = 0;  // ready for the next launch on this stream
}

__global__ void __launch_bounds__(256) trb_colsum_bf16_v3_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, int rows, int cols,
                                                                   int64_t ld, int rows_per_block, int vpr_log2, float* __restrict__ partial,
                                                                   unsigned int* __restrict__ tickets) {
  colsum_v3_body<false>(in, out, rows, cols, ld, rows_per_block, vpr_log2, partial, tickets);
}

__global__ void __cluster_dims__(1, 8, 1) __launch_bounds__(256)
trb_colsum_bf16_v4_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, int rows, int cols, int64_t ld, int rows_per_block,
                          int vpr_log2, float* __restrict__ partial, unsigned int* __restrict__ tickets) {
  colsum_v3_body<true>(in, out, rows, cols, ld, rows_per_block, vpr_log2, partial, tickets);
}

// per-device workspace of the column-sum kernel (tickets + block partials); kernels that use it are stream ordered
size_t g_colsum_ws_bytes_dev[64] = {};
void* g_colsum_ws_dev[64] = {};

TRB_API int trb_colsum_bf16(const void* in, float* out, int rows, int cols, int64_t ld, cudaStream_t stream) {
  if (rows == 0 || cols == 0) return 0;
  if (cols % 8 || ld % 8) return -12;
  const int nvec = cols / 8;
  const int xblocks = (nvec + 31) / 32;
  static const int variant = [] { const char* e = getenv("TRB_COLSUM"); return e ? atoi(e) : 4; }();
  if (variant == 3 || variant == 4) {
    int vpr_log2 = 5;
    while (vpr_log2 > 0 && (1 << (vpr_log2 - 1)) >= nvec) --vpr_log2;
    const int rpw = 32 >> vpr_log2;
    int yblocks = (4 * trb_num_sms() + xblocks - 1) / xblocks;
    const bool clustered = variant == 4 && rows >= 2048;
    if (clustered) {
      if (yblocks > 256) yblocks = 256;  // 8-CTA clusters fold through DSMEM: 32 partials at most reach the last-block tail
    } else if (yblocks > 64) {
      yblocks = 64;  // the last block of a column group sums yblocks partials: keep that tail short
    }
    int rows_per_block = (rows + yblocks - 1) / yblocks;
    rows_per_block = (rows_per_block + 8 * rpw - 1) / (8 * rpw) * (8 * rpw);
    yblocks = (rows + rows_per_block - 1) / rows_per_block;
    if (clustered) yblocks = (yblocks + 7) / 8 * 8;  // trailing blocks past `rows` contribute zeros
    // workspace (per process, stream-ordered use: the dense backward runs on one stream): tickets then partial sums
    const size_t need = 4096 + sizeof(float) * (size_t) yblocks * (size_t) cols;
    int dev = 0;
    TRB_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) return -12;
    size_t& g_colsum_ws_bytes = g_colsum_ws_bytes_dev[dev];
    void*& g_colsum_ws = g_colsum_ws_dev[dev];
    if (need > g_colsum_ws_bytes) {
      if (g_colsum_ws) TRB_CUDA(cudaFree(g_colsum_ws));
      g_colsum_ws_bytes = need < (8u << 20) ? (8u << 20) : need;
      TRB_CUDA(cudaMalloc(&g_colsum_ws, g_colsum_ws_bytes));
      TRB_CUDA(cudaMemset(g_colsum_ws, 0, 4096));
    }
    if (xblocks > 1024) return -12;
    dim3 grid(xblocks, yblocks);
    if (clustered)
      trb_colsum_bf16_v4_kernel<<<grid, 256, 0, stream>>>((const __nv_bfloat16*) in, out, rows, cols, ld, rows_per_block, vpr_log2,
                                                          reinterpret_cast<float*>(static_cast<char*>(g_colsum_ws) + 4096),
                                                          reinterpret_cast<unsigned int*>(g_colsum_ws));
    else
      trb_colsum_bf16_v3_kernel<<<grid, 256, 0, stream>>>((const __nv_bfloat16*) in, out, rows, cols, ld, rows_per_block, vpr_log2,
                                                          reinterpret_cast<float*>(static_cast<char*>(g_colsum_ws) + 4096),
                                                          reinterpret_cast<unsigned int*>(g_colsum_ws));
    TRB_CHECK_LAUNCH();
    return 0;
  }
  TRB_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * cols, stream));
  int rows_per_block = 256;
  while ((int64_t) xblocks * ((rows + rows_per_block - 1) / rows_per_block) > 2048 && rows_per_block < 65536) rows_per_block *= 2;
  dim3 grid(xblocks, (rows + rows_per_block - 1) / rows_per_block);
  trb_colsum_bf16_kernel<<<grid, 256, 0, stream>>>((const __nv_bfloat16*) in, out, rows, cols, ld, rows_per_block);
  TRB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// fp32 master weights -> bf16 GEMM operands (K zero-padded to a multiple of 8) for ALL layers of an MLP in one launch. The per-layer
// `.to(bf16)` + `pad` pair cost 2-3 tiny kernels per layer in front of every GEMM of the captured forward (13 launch-latency-bound
// nodes on the critical chain of the DLRM step).
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int kMaxCastTensors = 16;
struct CastPadTable {
  const float* src[kMaxCastTensors];
  __nv_bfloat16* dst[kMaxCastTensors];
  int32_t rows[kMaxCastTensors], K[kMaxCastTensors], Kp[kMaxCastTensors];
};

__global__ void __launch_bounds__(256) multi_cast_pad_bf16_kernel(const CastPadTable t) {
  const int l = blockIdx.y;
  const int K = t.K[l], Kp = t.Kp[l];
  const int64_t total = (int64_t) t.rows[l] * (Kp >> 1);  // one bf16x2 per thread-iteration
  const float* __restrict__ src = t.src[l];
  __nv_bfloat162* __restrict__ dst = reinterpret_cast<__nv_bfloat162*>(t.dst[l]);
  const int half = Kp >> 1;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t) gridDim.x * blockDim.x) {
    const int r = (int) (i / half), c = (int) (i - (int64_t) r * half) * 2;
    const float a = c < K ? src[(int64_t) r * K + c] : 0.f;
    const float b = c + 1 < K ? src[(int64_t) r * K + c + 1] : 0.f;
    dst[i] = __floats2bfloat162_rn(a, b);
  }
}

TRB_API int trb_multi_cast_pad_bf16(const void* const* src, void* const* dst, const int32_t* rows, const int32_t* K, const int32_t* Kp, int n, cudaStream_t stream) {
  if (n < 1 || n > kMaxCastTensors) return -1;
  CastPadTable t;
  int64_t biggest = 0;
  for (int i = 0; i < n; ++i) {
    if (Kp[i] % 2 || Kp[i] < K[i]) return -2;
    t.src[i] = (const float*) src[i];
    t.dst[i] = (__nv_bfloat16*) dst[i];
    t.rows[i] = rows[i];
    t.K[i] = K[i];
    t.Kp[i] = Kp[i];
    const int64_t tot = (int64_t) rows[i] * (Kp[i] / 2);
    biggest = tot > biggest ? tot : biggest;
  }
  if (biggest == 0) return 0;
  int64_t bx = (biggest + 255) / 256;
  if (bx > trb_num_sms() * 4) bx = trb_num_sms() * 4;
  multi_cast_pad_bf16_kernel<<<dim3((unsigned) bx, (unsigned) n), 256, 0, stream>>>(t);
  TRB_CHECK_LAUNCH();
  return 0;
}

// ---- final reduction of the epilogue column sums: out[n] = sum_p ws[p][n], fixed order (deterministic) ---------------------------------
// grid.x = 64-column groups, 8 warps stride over the P partial rows, lanes read float2 (a warp reads 256 contiguous bytes per row).
__global__ void __launch_bounds__(256) colsum_partials_kernel(const float* __restrict__ ws, int P, int N, float* __restrict__ out) {
  __shared__ float2 part[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 64 + lane * 2;
  float2 acc = make_float2(0.f, 0.f);
  if (col < N) {
    int r = warp;
    for (; r + 24 < P; r += 32) {
      const float2 a = *reinterpret_cast<const float2*>(ws + (int64_t) r * N + col);
      const float2 b = *reinterpret_cast<const float2*>(ws + (int64_t) (r + 8) * N + col);
      const float2 c = *reinterpret_cast<const float2*>(ws + (int64_t) (r + 16) * N + col);
      const float2 d = *reinterpret_cast<const float2*>(ws + (int64_t) (r + 24) * N + col);
      acc.x += (a.x + b.x) + (c.x + d.x);
      acc.y += (a.y + b.y) + (c.y + d.y);
    }
    for (; r < P; r += 8) {
      const float2 a = *reinterpret_cast<const float2*>(ws + (int64_t) r * N + col);
      acc.x += a.x;
      acc.y += a.y;
    }
  }
  part[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && col < N) {
    float2 t = part[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) {
      t.x += part[w][lane].x;
      t.y += part[w][lane].y;
    }
    *reinterpret_cast<float2*>(out + col) = t;
  }
}

TRB_API int trb_colsum_partials(const float* ws, int P, int N, float* out, cudaStream_t stream) {
  if (P <= 0 || N <= 0) return 0;
  if (N % 2) return -1;
  colsum_partials_kernel<<<(unsigned) ((N + 63) / 64), 256, 0, stream>>>(ws, P, N, out);
  TRB_CHECK_LAUNCH();
  return 0;
}
