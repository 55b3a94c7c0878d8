// e4m3 wgmma, 1-D bulk copy and e4m3 conversion wrappers of the FP8 dense kernels (gemm_fp8.cu).
// The block-scale rule lives here once for every kernel; its CPU mirror is torchrec_b200/ops/fp8_dense.py (pow2_scale).
#pragma once
#include "wgmma.cuh"

namespace trb {

constexpr float kE4m3Max = 448.f;

// D[64 x 128] (+)= A[64 x 32] . B[128 x 32]^T, e4m3 operands (both K-major: FP8 wgmma has no transposed-operand form) from shared
// memory, fp32 accumulators. scale_d = 0 overwrites D. Same fragment layout as the bf16 m64n128k16 (wgmma.cuh): thread t (warp
// w = (t / 32) % 4, lane l) holds d[4 j + 2 h + c] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + c].
__device__ __forceinline__ void wgmma_m64n128k32_e4m3(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

// Non-tensor bulk copy global -> shared completing on an mbarrier (bytes and both addresses multiples of 16).
__device__ __forceinline__ void bulk_load_1d(void* smem, const void* gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(gmem)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Two fp32 values -> two e4m3 bytes (round to nearest even, saturating to +-448); `lo` lands in the low byte.
__device__ __forceinline__ uint16_t pack_e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

// Block scale of a block whose largest magnitude is `amax`: the smallest power of two s with amax <= 448 s, s = 1 for an all-zero
// block, s clamped to >= 2^-126 so that 1 / s is a finite fp32 power of two. With amax = f 2^E (1 <= f < 2), 448 = 1.75 2^8: the
// answer is 2^(E - 8) when f <= 1.75 (one exact comparison), else 2^(E - 7). Returns s; *inv = 1 / s (exact).
__device__ __forceinline__ float pow2_block_scale(float amax, float* inv) {
  if (!(amax > 0.f)) {
    *inv = 1.f;
    return 1.f;
  }
  int e = (int) ((__float_as_uint(amax) >> 23) & 0xffu) - 127 - 8;
  if (e < -126) e = -126;
  if (!(amax <= kE4m3Max * __uint_as_float((uint32_t) (e + 127) << 23))) ++e;
  *inv = __uint_as_float((uint32_t) (127 - e) << 23);
  return __uint_as_float((uint32_t) (e + 127) << 23);
}

}  // namespace trb
