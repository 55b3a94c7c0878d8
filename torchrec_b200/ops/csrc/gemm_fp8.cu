// FP8 (e4m3) inference GEMM of the DLRM / DLRM-DCN dense arch, and the activation quantizer in front of it.
//
// Number format (CPU mirror, bit for bit: torchrec_b200/ops/fp8_dense.py):
//   values      e4m3, round to nearest even, saturating to +-448
//   activations one power-of-two scale per row per block of 128 consecutive columns (1 x 128; the last block may be partial)
//   weights     one power-of-two scale per output channel n ([N, K], nn.Linear layout)
//   scale       the smallest power of two s with amax <= 448 s (s = 1 for an all-zero block): dividing by s is exact, the e4m3
//               cast is the only rounding (pow2_block_scale in wgmma_fp8.cuh)
//   layout      values [M, Kp] row-major, Kp = K rounded up to 16 (16 B TMA rows), padding columns zero;
//               activation scales fp32 [ceil(Kp / 128), Mp] with Mp = M rounded up to 128 (the GEMM's BLOCK_M): the scales of one
//               K-block of one 128-row tile are 512 contiguous bytes, loaded by one bulk copy next to that K-block's operands.
//               Scales of the padding rows [M, Mp) are 1.
//
// trb_gemm_fp8: out = act(sw[n] * sum_kb sa[m, kb] * (A_q[m, kb] . W_q[n, kb]^T) + bias[n]), both operands K-major.
//   Persistent, warp-specialised (like gemm_bf16_wgmma_persistent_kernel in gemm_wgmma.cu), one CTA per SM walking a static tile list:
//     warps 0..3   consumer warpgroup 0   rows [0, 64) of the 128 x 128 tile
//     warps 4..7   consumer warpgroup 1   rows [64, 128)
//     warps 8..11  producer warpgroup     one thread issues the TMA loads (A 128 x 128 B, W 128 x 128 B, SWIZZLE_128B) and the bulk copy
//                                         of the K-block's 128 activation scales into a kStages-deep mbarrier ring
//   BLOCK_K = 128 e4m3 = one SWIZZLE_128B row: 4 x wgmma m64n128k32 per K-block, +32 B descriptor step as in the bf16 kernel.
//   Each K-block's product is accumulated in its own fp32 registers and then promoted into the running accumulator with that block's
//   activation scale (acc += sa[m, kb] * blk). That is where the per-block scales enter, and it bounds the error of the tensor core's
//   reduced-precision FP8 accumulation to one K-block. While one consumer warpgroup promotes, the other one's MMAs keep the tensor core busy.
//   Tile 128 x 128: the promotion needs two accumulator sets (64 + 64 fp32 per thread at BN = 128); a 128 x 256 tile would need 256
//   accumulator registers per thread, more than the 232 setmaxnreg leaves a consumer.
//   Epilogue: sw[n], fp32 bias, ACT_NONE / ACT_RELU, then either
//     bf16 output, or
//     e4m3 output plus the 1 x 128 block scales of the output itself (same layout as above, N / 16 = next layer's Kp): the input format
//     of the next fp8 layer, so an MLP chain never writes a bf16 activation. A 128-wide tile row lives in one lane quad: the row-block
//     amax is a per-thread max over 32 values plus two shfl_xor.
//   Limits: N % 16 == 0, K (the padded width) % 16 == 0, any M >= 1 (TMA clips the tails). Violations return -12.
//
// trb_fp8_quantize_rows: bf16 / fp32 [M, K] (any row pitch) -> e4m3 [M, Kp] + block scales, one pass (one warp per 1 x 128 block).
//
// Neither call synchronises the host: a predict forward built on them can be captured in a CUDA graph.
#include <cstring>

#include "wgmma_fp8.cuh"

namespace {

using namespace trb;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 128;
constexpr int BLOCK_K = 128;  // 128 e4m3 = 128 B = one SWIZZLE_128B row
constexpr int WGMMA_K = 32;
constexpr int kStages = 6;
constexpr int kThreads = 384;  // 2 consumer warpgroups + 1 producer warpgroup
constexpr int kConsumerWarps = 8;

constexpr int kABytes = BLOCK_M * BLOCK_K;
constexpr int kBBytes = BLOCK_N * BLOCK_K;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kScaleOffset = kStages * kStageBytes;             // [kStages][BLOCK_M] fp32 activation scales
constexpr int kBarOffset = kScaleOffset + kStages * BLOCK_M * 4;
constexpr int kSmemBytes = kBarOffset + 2 * kStages * 8 + 1024;  // + 1024: alignment of the dynamic smem base for SWIZZLE_128B
static_assert(kSmemBytes <= 227 * 1024, "shared memory of one CTA per SM");

enum Act : int { ACT_NONE = 0, ACT_RELU = 1 };

struct Fp8GemmParams {
  int M, N, K;
  const float* sa;      // [ceil(K / 128), ld_sa] activation block scales
  int64_t ld_sa;
  const float* sw;      // [N] weight channel scales
  const float* bias;    // [N] or nullptr
  int relu;
  void* out;            // bf16 or e4m3 [M, ldo]
  int64_t ldo;
  float* out_scales;    // e4m3 output: [N / 128 rounded up, ld_os] block scales of the output
  int64_t ld_os;
};

template <bool OUT_FP8>
__device__ __forceinline__ void epilogue(const Fp8GemmParams& p, float (&acc)[64], int row0, int n0, int wq, int lane) {
  const int q = lane & 3;
  const int rows[2] = {row0 + 16 * wq + (lane >> 2), row0 + 16 * wq + (lane >> 2) + 8};
  float amax[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = n0 + 8 * j + 2 * q;
    const bool col_ok = col < p.N;  // N % 16 == 0: col + 1 < N as well
    float2 s2 = make_float2(0.f, 0.f), b2 = make_float2(0.f, 0.f);
    if (col_ok) {
      s2 = __ldg(reinterpret_cast<const float2*>(p.sw + col));
      if (p.bias != nullptr) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + col));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = fmaf(acc[4 * j + 2 * h], s2.x, b2.x), v1 = fmaf(acc[4 * j + 2 * h + 1], s2.y, b2.y);
      if (p.relu) {
        v0 = fmaxf(v0, 0.f);
        v1 = fmaxf(v1, 0.f);
      }
      if constexpr (OUT_FP8) {
        acc[4 * j + 2 * h] = v0;  // (columns past N are 0: sw = bias = 0 there)
        acc[4 * j + 2 * h + 1] = v1;
        amax[h] = fmaxf(amax[h], fmaxf(fabsf(v0), fabsf(v1)));
      } else if (col_ok && rows[h] < p.M) {
        __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
        *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (int64_t) rows[h] * p.ldo + col) = o;
      }
    }
  }
  if constexpr (OUT_FP8) {
    // the 128 columns of this tile row = one output scale block, spread over the 4 lanes of a quad
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      amax[h] = fmaxf(amax[h], __shfl_xor_sync(0xffffffffu, amax[h], 1));
      amax[h] = fmaxf(amax[h], __shfl_xor_sync(0xffffffffu, amax[h], 2));
      float inv;
      const float s = pow2_block_scale(amax[h], &inv);
      // scales of every row of the tile (rows past M included: the next layer's bulk copy reads whole 128-row vectors)
      if (q == 0) p.out_scales[(int64_t) (n0 / BLOCK_N) * p.ld_os + rows[h]] = s;
      if (rows[h] < p.M) {
        uint8_t* orow = reinterpret_cast<uint8_t*>(p.out) + (int64_t) rows[h] * p.ldo;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = n0 + 8 * j + 2 * q;
          if (col < p.N) *reinterpret_cast<uint16_t*>(orow + col) = pack_e4m3x2(acc[4 * j + 2 * h] * inv, acc[4 * j + 2 * h + 1] * inv);
        }
      }
    }
  }
}

template <bool OUT_FP8>
__global__ void __launch_bounds__(kThreads, 1)
gemm_fp8_wgmma_persistent_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w, const Fp8GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  float* scale_ring = reinterpret_cast<float*>(smem + kScaleOffset);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kBarOffset);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumerWarps);  // one arrival per consumer warp, after it has read the slot's scales
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int tiles = m_tiles * n_tiles;

  if (warp_idx >= kConsumerWarps) {
    // ================= producer warpgroup =================
    setmaxnreg_dec<40>();
    if (warp_idx == kConsumerWarps && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_a)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_w)) : "memory");
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int m_blk = tile / n_tiles, n_blk = tile % n_tiles;
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * kStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes + BLOCK_M * 4);
          tma_load_2d(&tmap_a, &full_bar[stage], sa, kb * BLOCK_K, m_blk * BLOCK_M);
          tma_load_2d(&tmap_w, &full_bar[stage], sa + kABytes, kb * BLOCK_K, n_blk * BLOCK_N);
          bulk_load_1d(scale_ring + stage * BLOCK_M, p.sa + (int64_t) kb * p.ld_sa + (int64_t) m_blk * BLOCK_M, BLOCK_M * 4, &full_bar[stage]);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ================= consumers =================
  setmaxnreg_inc<232>();
  const int wg = warp_idx >> 2;  // rows [64 wg, 64 wg + 64) of the tile
  const int wq = warp_idx & 3;
  const int srow = 64 * wg + 16 * wq + (lane >> 2);  // this thread's two rows in the tile: srow, srow + 8
  int stage = 0;
  uint32_t phase = 0;
  float acc[64], blk[64];
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m_blk = tile / n_tiles, n_blk = tile % n_tiles;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const float s0 = scale_ring[stage * BLOCK_M + srow], s1 = scale_ring[stage * BLOCK_M + srow + 8];
      const uint32_t a_addr = smem_u32(smem + stage * kStageBytes) + (uint32_t) wg * 8192u;  // 64 rows x 128 B further
      const uint32_t b_addr = smem_u32(smem + stage * kStageBytes + kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
        wgmma_m64n128k32_e4m3(blk, make_kmajor_desc(a_addr + k * 32), make_kmajor_desc(b_addr + k * 32), k > 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(blk);
      if (lane == 0) mbar_arrive(&empty_bar[stage]);  // (release: orders this warp's scale reads before the slot is refilled)
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = fmaf((i & 2) ? s1 : s0, blk[i], acc[i]);
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    epilogue<OUT_FP8>(p, acc, m_blk * BLOCK_M + 64 * wg, n_blk * BLOCK_N, wq, lane);
  }
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

// rows x K e4m3 matrix, row pitch ld bytes; box = 128 columns x box_rows rows, SWIZZLE_128B, out-of-range elements read as zero
int make_tmap_e4m3(CUtensorMap* map, const void* ptr, int64_t rows, int64_t K, int64_t ld, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return -10;
  cuuint64_t dims[2] = {(cuuint64_t) K, (cuuint64_t) rows};
  cuuint64_t strides[1] = {(cuuint64_t) ld};
  cuuint32_t box[2] = {(cuuint32_t) BLOCK_K, (cuuint32_t) box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -11;
}

template <bool OUT_FP8>
int launch_gemm_fp8(const CUtensorMap& ta, const CUtensorMap& tw, const Fp8GemmParams& p, cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    TRB_CUDA(cudaFuncSetAttribute(gemm_fp8_wgmma_persistent_kernel<OUT_FP8>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    configured = true;
  }
  const int64_t tiles = (int64_t) ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N);
  if (tiles > 0x7fffffff) return -12;
  const int grid = (int) (tiles < trb_num_sms() ? tiles : trb_num_sms());
  gemm_fp8_wgmma_persistent_kernel<OUT_FP8><<<grid, kThreads, kSmemBytes, stream>>>(ta, tw, p);
  TRB_CHECK_LAUNCH();
  return 0;
}

// ---- activation quantizer: one warp per (row, 128-column block), 4 consecutive columns per lane ----
__global__ void __launch_bounds__(256) fp8_quantize_rows_kernel(const void* __restrict__ x, int64_t ldx, int x_bf16, int vec, int M, int Mp, int K,
                                                                  int Kp, uint8_t* __restrict__ q, int64_t ldq, float* __restrict__ s, int64_t lds) {
  const int lane = threadIdx.x & 31;
  const int kblocks = (Kp + BLOCK_K - 1) / BLOCK_K;
  const int64_t tasks = (int64_t) Mp * kblocks;
  const int64_t warps = (int64_t) gridDim.x * (blockDim.x >> 5);
  for (int64_t t = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < tasks; t += warps) {
    const int row = (int) (t / kblocks), kb = (int) (t - (int64_t) row * kblocks);
    if (row >= M) {
      if (lane == 0) s[(int64_t) kb * lds + row] = 1.f;
      continue;
    }
    const int c0 = kb * BLOCK_K + 4 * lane;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (x_bf16) {
      const __nv_bfloat16* xr = reinterpret_cast<const __nv_bfloat16*>(x) + (int64_t) row * ldx;
      if (vec && c0 + 3 < K) {
        const float4 f = Vec4<__nv_bfloat16>::ld(xr + c0);
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (c0 + i < K) v[i] = __bfloat162float(xr[c0 + i]);
      }
    } else {
      const float* xr = reinterpret_cast<const float*>(x) + (int64_t) row * ldx;
      if (vec && c0 + 3 < K) {
        const float4 f = *reinterpret_cast<const float4*>(xr + c0);
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (c0 + i < K) v[i] = xr[c0 + i];
      }
    }
    float amax = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    float inv;
    const float sc = pow2_block_scale(amax, &inv);
    if (c0 < Kp) {  // Kp % 16 == 0: the whole 4-column group is inside the padded row
      const uint32_t w = (uint32_t) pack_e4m3x2(v[0] * inv, v[1] * inv) | ((uint32_t) pack_e4m3x2(v[2] * inv, v[3] * inv) << 16);
      *reinterpret_cast<uint32_t*>(q + (int64_t) row * ldq + c0) = w;
    }
    if (lane == 0) s[(int64_t) kb * lds + row] = sc;
  }
}

}  // namespace

// x: bf16 (x_bf16 = 1) or fp32 [M, K] with row pitch ldx elements. q: e4m3 [M, ldq] (columns [0, Kp) written, Kp = K rounded up to 16).
// scales: fp32 [ceil(Kp / 128), lds], lds >= M rounded up to 128 (rows [M, Mp) get scale 1).
TRB_API int trb_fp8_quantize_rows(const void* x, int64_t ldx, int x_bf16, int M, int K, void* q, int64_t ldq, float* scales, int64_t lds,
                                  cudaStream_t stream) {
  if (M <= 0 || K <= 0) return 0;
  const int Kp = (K + 15) / 16 * 16;
  const int Mp = (M + BLOCK_M - 1) / BLOCK_M * BLOCK_M;
  if (ldx < K || ldq < Kp || ldq % 16 || lds < Mp || (reinterpret_cast<uintptr_t>(q) % 16)) return -12;
  const int esz = x_bf16 ? 2 : 4;
  const int vec = (ldx % 4 == 0) && (reinterpret_cast<uintptr_t>(x) % (4 * esz) == 0);
  const int64_t tasks = (int64_t) Mp * ((Kp + BLOCK_K - 1) / BLOCK_K);
  int64_t blocks = (tasks + 7) / 8;
  const int64_t cap = (int64_t) trb_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  fp8_quantize_rows_kernel<<<(unsigned) blocks, 256, 0, stream>>>(x, ldx, x_bf16, vec, M, Mp, K, Kp, reinterpret_cast<uint8_t*>(q), ldq, scales, lds);
  TRB_CHECK_LAUNCH();
  return 0;
}

// out = act(sw[n] * sum_kb sa[m, kb] * (A[m, kb] . W[n, kb]^T) + bias[n]).
//   A: e4m3 [M, lda] (K = padded width, K % 16 == 0), sa: fp32 [ceil(K / 128), ld_sa] (ld_sa >= M rounded up to 128, ld_sa % 4 == 0)
//   W: e4m3 [N, ldw], sw: fp32 [N], bias: fp32 [N] or nullptr, act: 0 none / 1 ReLU
//   out_fp8 = 0: out bf16 [M, ldo];  out_fp8 = 1: out e4m3 [M, ldo] + out_scales fp32 [ceil(N / 128), ld_os] (ld_os >= M rounded up to 128)
TRB_API int trb_gemm_fp8(const void* A, int64_t lda, const float* sa, int64_t ld_sa, const void* W, int64_t ldw, const float* sw, const float* bias,
                         int act, void* out, int64_t ldo, int out_fp8, float* out_scales, int64_t ld_os, int M, int N, int K, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  const int64_t Mp = (M + BLOCK_M - 1) / BLOCK_M * BLOCK_M;
  if ((N % 16) || (K % 16) || (lda % 16) || (ldw % 16) || lda < K || ldw < K) return -12;
  if (ld_sa < Mp || (ld_sa % 4) || (reinterpret_cast<uintptr_t>(sa) % 16)) return -12;
  if (ldo < N || (ldo % 2) || (act != ACT_NONE && act != ACT_RELU) || sw == nullptr) return -12;
  if (out_fp8 && (out_scales == nullptr || ld_os < Mp)) return -12;
  Fp8GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.sa = sa;
  p.ld_sa = ld_sa;
  p.sw = sw;
  p.bias = bias;
  p.relu = act == ACT_RELU;
  p.out = out;
  p.ldo = ldo;
  p.out_scales = out_scales;
  p.ld_os = ld_os;
  CUtensorMap ta, tw;
  int rc = make_tmap_e4m3(&ta, A, M, K, lda, BLOCK_M);
  if (rc) return rc;
  rc = make_tmap_e4m3(&tw, W, N, K, ldw, BLOCK_N);
  if (rc) return rc;
  return out_fp8 ? launch_gemm_fp8<true>(ta, tw, p, stream) : launch_gemm_fp8<false>(ta, tw, p, stream);
}
