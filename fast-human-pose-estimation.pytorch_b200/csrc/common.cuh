// common.cuh -- error plumbing and small device helpers shared by every kernel in libfpd_b200 (built for sm_90a:
//   -gencode arch=compute_90a,code=sm_90a)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdio>

namespace fpd {

// ------------------------------------------------------------------------------------------------
// error plumbing (thread-local last-error string; see api.cu)
// ------------------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);
#define FPD_OK 0
#define FPD_ERR_INVALID -1
#define FPD_ERR_CUDA -2
#define FPD_ERR_UNSUPPORTED -3

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
