// Shared helpers for the lav_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/lav_b200.h"

namespace lavb {

void set_error(const char* fmt, ...);

#define LAVB_CHECK_ARG(cond, ...)            \
  do {                                       \
    if (!(cond)) {                           \
      lavb::set_error(__VA_ARGS__);          \
      return 1;                              \
    }                                        \
  } while (0)

#define LAVB_CUDA_OK(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      lavb::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));  \
      return 2;                                                                              \
    }                                                                                        \
  } while (0)

#define LAVB_LAUNCH_OK()                                                                     \
  do {                                                                                       \
    cudaError_t _e = cudaGetLastError();                                                     \
    if (_e != cudaSuccess) {                                                                 \
      lavb::set_error("%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e));     \
      return 3;                                                                              \
    }                                                                                        \
  } while (0)

constexpr int kNumSMsH100 = 132;   // fallback only; grids are sized from num_sms()
int num_sms();
cudaError_t ensure_dyn_smem(const void* kernel, int bytes);
#define kNumSMs (lavb::num_sms())

// ---- the 16-bit storage type of the tensor-core path ------------------------------------------------------------------------
// IEEE half (11-bit significand, fp32 accumulation everywhere): through the 12 chained Conv-ReLU-BN layers of the BEV stack its
// rounding error stays at 1-2e-3 of the tensor scale where bfloat16 (8-bit significand) measures 1.0-1.7e-2 — outside the
// 1e-2 the 16-bit path is held to.  The range (65504) is guarded: every fp32 -> h16 conversion SATURATES (one F2FP.SATFINITE).
// -DLAVB_H16_BF16 builds the bfloat16 variant of the same kernels (error studies only).
#ifdef LAVB_H16_BF16
using h16 = __nv_bfloat16;
using h162 = __nv_bfloat162;
#define LAVB_H16_PTX "bf16"
#define LAVB_H16 LAVB_BF16
#define LAVB_TMAP_H16 CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
__device__ __forceinline__ uint32_t pack_h16(float a, float b) {            // (a -> low half, b -> high half)
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_h16(uint32_t u) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u)); }
__device__ __forceinline__ h16 float2h16(float v) { return __float2bfloat16_rn(v); }
__device__ __forceinline__ float h162float(h16 v) { return __bfloat162float(v); }
#else
using h16 = __half;
using h162 = __half2;
#define LAVB_H16_PTX "f16"
#define LAVB_H16 LAVB_F16
#define LAVB_TMAP_H16 CU_TENSOR_MAP_DATA_TYPE_FLOAT16
__device__ __forceinline__ uint32_t pack_h16(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ float2 unpack_h16(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); }
__device__ __forceinline__ h16 float2h16(float v) {
  unsigned short r;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(r) : "f"(v));
  return __ushort_as_half(r);
}
__device__ __forceinline__ float h162float(h16 v) { return __half2float(v); }
#endif
__device__ __forceinline__ h162 floats2h162(float a, float b) {
  const uint32_t u = pack_h16(a, b);
  return *reinterpret_cast<const h162*>(&u);
}
__device__ __forceinline__ float2 h1622float2(h162 v) { return unpack_h16(*reinterpret_cast<const uint32_t*>(&v)); }

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// host-side argument checks: pointer alignment, and whether the byte ranges [a, a + na) and [b, b + nb) share a byte
static inline bool is_aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }
static inline bool ranges_overlap(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return na > 0 && nb > 0 && x < y + nb && y < x + na;
}

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<h16>(h16 v) { return h162float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ h16 from_f32<h16>(float v) { return float2h16(v); }

// 4 consecutive elements -> float4 (pointer must be 16 B aligned for float, 8 B for h16)
template <typename T> __device__ __forceinline__ float4 load4(const T* p);
template <> __device__ __forceinline__ float4 load4<float>(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}
template <> __device__ __forceinline__ float4 load4<h16>(const h16* p) {
  const uint2 r = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 fa = unpack_h16(r.x), fb = unpack_h16(r.y);
  return make_float4(fa.x, fa.y, fb.x, fb.y);
}
template <typename T> __device__ __forceinline__ void store4(T* p, float4 v);
template <> __device__ __forceinline__ void store4<float>(float* p, float4 v) {
  *reinterpret_cast<float4*>(p) = v;
}
template <> __device__ __forceinline__ void store4<h16>(h16* p, float4 v) {
  *reinterpret_cast<uint2*>(p) = make_uint2(pack_h16(v.x, v.y), pack_h16(v.z, v.w));
}

// 2 consecutive elements (pointer 8 B aligned for float, 4 B for h16)
template <typename T> __device__ __forceinline__ float2 load2(const T* p);
template <> __device__ __forceinline__ float2 load2<float>(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
template <> __device__ __forceinline__ float2 load2<h16>(const h16* p) {
  return unpack_h16(__ldg(reinterpret_cast<const uint32_t*>(p)));
}
template <typename T> __device__ __forceinline__ void store2(T* p, float a, float b);
template <> __device__ __forceinline__ void store2<float>(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
template <> __device__ __forceinline__ void store2<h16>(h16* p, float a, float b) {
  *reinterpret_cast<uint32_t*>(p) = pack_h16(a, b);
}

}  // namespace lavb
