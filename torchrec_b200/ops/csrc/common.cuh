// Common helpers for the torchrec_b200 sm_90a kernel library.
//
// The library is a plain C ABI (.so loaded with ctypes): every entry point takes raw device
// pointers + a cudaStream_t, so it builds in seconds with nvcc alone (no torch headers) and the
// same object works from Python, from the C++ serving runtime and from tests.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define TRB_API extern "C" __attribute__((visibility("default")))

// dtype codes shared with python (torchrec_b200/ops/_lib.py)
enum TrbDType : int { TRB_F32 = 0, TRB_F16 = 1, TRB_BF16 = 2, TRB_U8 = 3, TRB_I32 = 4, TRB_I64 = 5, TRB_FP8 = 6 };

// Max ranks of one NVLink domain we address with peer pointers passed by value.
#define TRB_MAX_PEERS 16

struct TrbPeerPtrs {
  void* p[TRB_MAX_PEERS];
};

// SM count of the current device: grid size of the persistent / grid-stride kernels
inline int trb_num_sms() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 1;
}

// ---- launch accounting ------------------------------------------------------------------
// Every kernel launch of this library bumps a host-side counter so bench.py can report
// "gpu_launches" truthfully (see trb_launch_count()).
extern unsigned long long g_trb_launches;
#define TRB_COUNT_LAUNCH() (++g_trb_launches)

#define TRB_CHECK_LAUNCH()                                  \
  do {                                                      \
    TRB_COUNT_LAUNCH();                                     \
    cudaError_t e__ = cudaPeekAtLastError();                \
    if (e__ != cudaSuccess) return (int)e__;                \
  } while (0)

#define TRB_CUDA(x)                                         \
  do {                                                      \
    cudaError_t e__ = (x);                                  \
    if (e__ != cudaSuccess) return (int)e__;                \
  } while (0)

// ---- small device helpers ---------------------------------------------------------------
__device__ __forceinline__ int64_t trb_ld_idx(const void* p, int64_t i, int is64) {
  return is64 ? reinterpret_cast<const int64_t*>(p)[i] : (int64_t) reinterpret_cast<const int32_t*>(p)[i];
}

__device__ __forceinline__ void trb_st_idx(void* p, int64_t i, int is64, int64_t v) {
  if (is64) reinterpret_cast<int64_t*>(p)[i] = v;
  else reinterpret_cast<int32_t*>(p)[i] = (int32_t) v;
}


// ---- multi-source id views ----------------------------------------------------------------
// A table-batched kernel sees B = n_src * src_B samples per feature. With n_src == 1 the ids are one KJT (offsets
// [F*B + 1] over one indices array). With n_src > 1 (NVLink input dist, csrc/kjt_route.cu) every source rank s wrote
// ITS samples into a private fixed-capacity region of the receive slot:
//     offsets_s = offsets + s * off_stride   ([F * src_B + 1], relative to the start of the region)
//     indices_s = indices + s * idx_stride   (per-sample weights use the same stride)
// so the lookup / backward kernels consume the received regions in place (no recat / compaction pass).
struct TrbSrcView {
  const void* indices;
  const void* offsets;
  const float* psw;
  int64_t idx_stride;
  int64_t off_stride;
  int32_t n_src;
  int32_t src_B;
  int32_t idx64, off64;
};

// element index (into offsets) of bag (f, b) and the position base of its source region
__device__ __forceinline__ int64_t trb_src_off_index(const TrbSrcView& v, int f, int b, int64_t* pos_base) {
  if (v.n_src <= 1) {
    *pos_base = 0;
    return (int64_t) f * v.src_B + b;
  }
  const int s = b / v.src_B;
  *pos_base = (int64_t) s * v.idx_stride;
  return (int64_t) s * v.off_stride + (int64_t) f * v.src_B + (b - s * v.src_B);
}

// 4-element vector load/store with conversion to/from float4. Rows are 4-element aligned
// (embedding dims are multiples of 4, same constraint as the reference TBE).
template <typename T>
struct Vec4;

template <>
struct Vec4<float> {
  // raw = the registers a 4-element load lands in; cvt(raw) -> float4. Kernels that want several rows in flight load raw values for all
  // of them first and convert later: a load fused with its conversion makes the compiler wait for each load before issuing the next
  // (measured in tbe_bwd_walk_kernel: the 4 gradient loads of a group shared one destination register and ran back to back).
  typedef float4 raw;
  static __device__ __forceinline__ raw ld_raw(const float* p) { return *reinterpret_cast<const float4*>(p); }
  static __device__ __forceinline__ raw zero_raw() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  static __device__ __forceinline__ float4 cvt(raw r) { return r; }
  static __device__ __forceinline__ float4 ld(const float* p) { return *reinterpret_cast<const float4*>(p); }
  static __device__ __forceinline__ float4 ld_nc(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
  }
  static __device__ __forceinline__ void st(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
};

template <>
struct Vec4<__nv_bfloat16> {
  typedef uint2 raw;
  static __device__ __forceinline__ raw ld_raw(const __nv_bfloat16* p) { return *reinterpret_cast<const uint2*>(p); }
  static __device__ __forceinline__ raw zero_raw() { return make_uint2(0u, 0u); }
  static __device__ __forceinline__ float4 cvt(uint2 u) {
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&u.x);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&u.y);
    float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
    return make_float4(fa.x, fa.y, fb.x, fb.y);
  }
  static __device__ __forceinline__ float4 ld(const __nv_bfloat16* p) { return cvt(*reinterpret_cast<const uint2*>(p)); }
  static __device__ __forceinline__ float4 ld_nc(const __nv_bfloat16* p) {
    uint2 u;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(u.x), "=r"(u.y) : "l"(p));
    return cvt(u);
  }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, float4 v) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&a);
    u.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = u;
  }
};

template <>
struct Vec4<__half> {
  typedef uint2 raw;
  static __device__ __forceinline__ raw ld_raw(const __half* p) { return *reinterpret_cast<const uint2*>(p); }
  static __device__ __forceinline__ raw zero_raw() { return make_uint2(0u, 0u); }
  static __device__ __forceinline__ float4 cvt(uint2 u) {
    __half2 a = *reinterpret_cast<__half2*>(&u.x);
    __half2 b = *reinterpret_cast<__half2*>(&u.y);
    float2 fa = __half22float2(a), fb = __half22float2(b);
    return make_float4(fa.x, fa.y, fb.x, fb.y);
  }
  static __device__ __forceinline__ float4 ld(const __half* p) { return cvt(*reinterpret_cast<const uint2*>(p)); }
  static __device__ __forceinline__ float4 ld_nc(const __half* p) {
    uint2 u;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(u.x), "=r"(u.y) : "l"(p));
    return cvt(u);
  }
  static __device__ __forceinline__ void st(__half* p, float4 v) {
    __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&a);
    u.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = u;
  }
};

__device__ __forceinline__ float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 f4_fma(float4 a, float s, float4 c) {
  return make_float4(fmaf(a.x, s, c.x), fmaf(a.y, s, c.y), fmaf(a.z, s, c.z), fmaf(a.w, s, c.w));
}
__device__ __forceinline__ float4 f4_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float f4_sq(float4 a) { return a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// system-scope release / acquire used by cross-GPU signalling over NVLink
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
