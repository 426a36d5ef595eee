// common.cuh -- error plumbing and small device helpers shared by every kernel in libfpd_b200 (built for sm_90a:
//   -gencode arch=compute_90a,code=sm_90a)
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdio>
#include <type_traits>

#include "../../include/fpd_b200.h"

namespace fpd {

// ------------------------------------------------------------------------------------------------
// error plumbing (thread-local last-error string, return codes of fpd_b200.h; see elementwise.cu)
// ------------------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);

#define FPD_CUDA_CHECK(expr)                                                                       \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      fpd::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));   \
      return FPD_ERR_CUDA;                                                                         \
    }                                                                                              \
  } while (0)

#define FPD_REQUIRE(cond, ...)                                                                     \
  do {                                                                                             \
    if (!(cond)) {                                                                                 \
      fpd::set_last_error(__VA_ARGS__);                                                            \
      return FPD_ERR_INVALID;                                                                      \
    }                                                                                              \
  } while (0)

// every kernel launch in the library is followed by exactly one FPD_LAUNCH_CHECK: it doubles as the launch counter
// behind fpd_launch_count() (what bench.py reports as gpu_launches).
void count_launch();
#define FPD_LAUNCH_CHECK()                  \
  do {                                      \
    fpd::count_launch();                    \
    FPD_CUDA_CHECK(cudaPeekAtLastError());  \
  } while (0)

// Grid sizes of the bandwidth-bound kernels are multiples of the H100 SXM's 132 SMs (a few waves keep enough bytes in
// flight for HBM; fixed caps keep the reductions' partial buffers, and so their summation order, independent of the
// device they run on).
constexpr int kNumSMs = 132;
// SMs of the current device (kNumSMs when it cannot be queried): the persistent grids of the tensor-core kernels
int device_sm_count();

// 3xFP16 and single-pass FP16 weights are stored as __half of w * 2^kF16WeightScaleLog2 (fpd_weight_prep_f16); the
// convolution epilogues multiply by 2^-kF16WeightScaleLog2
constexpr int kF16WeightScaleLog2 = 8;

// ------------------------------------------------------------------------------------------------
// numeric helpers
// ------------------------------------------------------------------------------------------------
// Round-to-nearest (ties away) fp32 -> tf32, result kept in an fp32 container (low 13 bits zero).
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// hi/lo split used by the 3xTF32 scheme: x ~= hi + lo with both exactly representable in tf32.
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - hi);
}

// Same split with the rounding done in integer arithmetic (2 ALU ops instead of the multi-instruction emulation ptxas
// emits for cvt.rna.tf32): adding half an ulp of the 13 dropped bits and truncating is round-to-nearest,
// ties away from zero, i.e. exactly cvt.rna for finite inputs. Used inside the tensor-core pipelines where the
// transform competes with the MMA issue for scheduler slots.
__device__ __forceinline__ void split_tf32_fast(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
  const float r = x - hi;
  lo = __uint_as_float((__float_as_uint(r) + 0x1000u) & 0xFFFFE000u);
}

// ---- fp16 activation storage (inference precision "fp16_act"): kernels compute in fp32 from float(x) and store
// fp16_rn of the result saturated to +-65504, so NaN stays NaN and no finite value becomes infinite.
__device__ __forceinline__ float sat_f16(float v) { return fabsf(v) > 65504.f ? copysignf(65504.f, v) : v; }
__device__ __forceinline__ uint32_t f16x2_sat_bits(float a, float b) {
  const __half2 h = __floats2half2_rn(sat_f16(a), sat_f16(b));
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float2 f16x2_bits_to_float2(uint32_t u) {
  return __half22float2(*reinterpret_cast<const __half2*>(&u));
}

// Four consecutive activations (element offset 4 i) of an fp32 or fp16 tensor, as fp32 / stored from fp32.
template <typename T>
__device__ __forceinline__ float4 ld_act4(const T* p, int64_t i) {
  if constexpr (std::is_same<T, float>::value) {
    return __ldg(reinterpret_cast<const float4*>(p) + i);
  } else {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p) + i);
    const float2 a = f16x2_bits_to_float2(u.x), b = f16x2_bits_to_float2(u.y);
    return make_float4(a.x, a.y, b.x, b.y);
  }
}
template <typename T>
__device__ __forceinline__ void st_act4(T* p, int64_t i, float4 v) {
  if constexpr (std::is_same<T, float>::value) {
    reinterpret_cast<float4*>(p)[i] = v;
  } else {
    reinterpret_cast<uint2*>(p)[i] = make_uint2(f16x2_sat_bits(v.x, v.y), f16x2_sat_bits(v.z, v.w));
  }
}
// Two consecutive activations at element offset `off` (even).
template <typename T>
__device__ __forceinline__ float2 ld_act2(const T* p, size_t off) {
  if constexpr (std::is_same<T, float>::value) {
    return __ldg(reinterpret_cast<const float2*>(p + off));
  } else {
    return f16x2_bits_to_float2(__ldg(reinterpret_cast<const unsigned int*>(p + off)));
  }
}
template <typename T>
__device__ __forceinline__ void st_act2(T* p, size_t off, float2 v) {
  if constexpr (std::is_same<T, float>::value) {
    *reinterpret_cast<float2*>(p + off) = v;
  } else {
    *reinterpret_cast<uint32_t*>(p + off) = f16x2_sat_bits(v.x, v.y);
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// generic-proxy smem writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

}  // namespace fpd
