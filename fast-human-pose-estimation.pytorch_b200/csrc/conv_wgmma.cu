// conv_wgmma.cu -- implicit-GEMM convolution and convolution weight gradient on the sm_90a warpgroup tensor cores
// (wgmma.mma_async), operand preparation fused in.
//
// Forward (fpd_conv2d_tc_ts, fpd_conv2d_tc_h*): y = conv(relu?((x - mean) * scale + shift)) (+ bias, + residual, ReLU
// mask), stride 1, "same" padding, NHWC activations, weights [tap][Cout][Cin] as hi/lo pairs (3xTF32: fp32 containers
// from fpd_weight_prep; 3xFP16: __half from fpd_weight_prep_f16, pre-scaled by 2^kF16WeightScaleLog2). BatchNorm2d-apply
// + ReLU + Conv2d of lib/models/hourglass.py:34-44: padding positions are zero AFTER the affine.
//   GEMM: M = 128 output pixels (two warpgroups x 64 rows), N = one Cout slice (<= 128), K = taps x Cin in steps of one
//   128-byte operand row (32 tf32 or 64 fp16 channels of one tap). Every thread loads its share of the raw x rows into
//   registers one K step ahead, applies the affine + ReLU + hi/lo split and stores the result into the swizzled
//   K-major A tile; the weight tiles arrive by cp.async. Three pipeline stages: a stage is rewritten only after every
//   warpgroup has retired the wgmma group that read it (wait_group<0> + the per-step CTA barrier); each step's
//   products are summed into the fp32 accumulators outside the tensor core (see mma_row).
//   Split operands: acc += A_lo * B_hi + A_hi * B_lo + A_hi * B_hi (the lo * lo term is below fp32 rounding).
//   Optional epilogue statistics: per output channel {sum (y - pivot), sum (y - pivot)^2} in fp64, per-warp shared
//   accumulators merged in a fixed order (deterministic), one [Cout][2] block per CTA for fpd_bn_finalize_sums.
//   3x3 with 3xFP16 operands (conv_halo_kernel, where conv_plan finds it fits in shared memory): the same GEMM
//   with the A operand of a tile loaded and transformed once into a halo in shared memory and fed from registers.
//   Single-pass FP16 (fpd_conv2d_tc_f16x1*): the halo and 1x1 weight-resident kernels with kSplit = false
//   (conv_halo_f16x1_kernel, pw_conv_f16x1_kernel), one MMA per k16 straight into the accumulators. Inference calls,
//   and the training precision "fp16": forward calls with epilogue statistics, data gradients with in_scale. Their
//   TIn / TOut template parameters (float or __half) are the activation types of x and of y with the residual: the
//   inference precision "fp16_act" (fpd_conv2d_tc_f16x1_io) stores activations in fp16.
//
// Weight gradient (fpd_conv2d_wgrad_tc*):
//   dW[co][ci][tap] = scale * sum_{pixels p} dY[p][co] * A[p (+) tap][ci],  A = relu?((x - mean) * scale + shift)
//   GEMM: M = 128 output channels, N = one input-channel tile, K = pixels in steps of 32, one tap per CTA, split-K over
//   pixel ranges. tf32 wgmma takes K-major operands only, so the transform threads write both operands transposed
//   (channel rows of 32 pixels). Each CTA stores an fp32 partial; a second kernel reduces the partials in a fixed
//   order (deterministic) into the OIHW gradient.
//   Every 3x3 shape and the 1x1 shapes with Cout <= 64 run the same plan on wgrad_halo_kernel instead (input channels
//   on M, x from registers, one staged pixel step for the three taps of a kernel row), bit-identical to it.
#include <cuda.h>
#include <cuda_fp16.h>

#include <atomic>
#include <mutex>
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"

namespace fpd {
namespace {

constexpr int kTileM = 128;                 // GEMM rows per CTA: two warpgroups x 64
constexpr int kThreads = 256;
constexpr int kStages = 3;
constexpr int kATileBytes = kTileM * 128;   // one [128 rows x 128 B] operand tile
constexpr int kMaxCinTs = 512;
constexpr int kMaxCinH = 2048;              // pose_resnet's layer4 / first deconv
constexpr int kMaxStatCout = 256;           // epilogue statistics: [8 warps][Cout][2] fp64 in shared memory
constexpr int kSmemLimit = 227 * 1024;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void sts128u(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

// (v0, v1) -> packed fp16 hi pair and lo pair: v ~= hi + lo. v0 goes to the low half (even k).
__device__ __forceinline__ void split_f16x2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  v0 = fminf(fmaxf(v0, -65504.f), 65504.f);   // saturate instead of producing inf (never hit by sane activations)
  v1 = fminf(fmaxf(v1, -65504.f), 65504.f);
  const __half2 h = __floats2half2_rn(v0, v1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

__device__ __forceinline__ float4 affine_relu4(float4 v, const float* mean, const float* scale, const float* shift,
                                               int c, int relu) {
  if (scale) {
    const float4 mu = mean ? __ldg(reinterpret_cast<const float4*>(mean + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 sc = __ldg(reinterpret_cast<const float4*>(scale + c));
    const float4 sh = __ldg(reinterpret_cast<const float4*>(shift + c));
    v.x = fmaf(v.x - mu.x, sc.x, sh.x); v.y = fmaf(v.y - mu.y, sc.y, sh.y);
    v.z = fmaf(v.z - mu.z, sc.z, sh.z); v.w = fmaf(v.w - mu.w, sc.w, sh.w);
  }
  if (relu) {
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
  }
  return v;
}

// Raw load of the 8 activations at element offset `off` of x (fp32 or fp16 NHWC): fp32 into v[0], v[1]; fp16 as its
// 16 bytes in v[0], kept as bits until cvt_raw8 widens them (so the load stays in flight like the fp32 one).
template <typename TIn>
__device__ __forceinline__ void ld_raw8(const float* x, size_t off, float4 (&v)[2]) {
  if constexpr (std::is_same<TIn, float>::value) {
    const float4* src = reinterpret_cast<const float4*>(x + off);
    v[0] = __ldg(src);
    v[1] = __ldg(src + 1);
  } else {
    const uint4 h = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(x) + off));
    v[0] = make_float4(__uint_as_float(h.x), __uint_as_float(h.y), __uint_as_float(h.z), __uint_as_float(h.w));
  }
}
template <typename TIn>
__device__ __forceinline__ void cvt_raw8(const float4 (&v)[2], float4& a0, float4& a1) {
  if constexpr (std::is_same<TIn, float>::value) {
    a0 = v[0];
    a1 = v[1];
  } else {
    const float2 p0 = f16x2_bits_to_float2(__float_as_uint(v[0].x)), p1 = f16x2_bits_to_float2(__float_as_uint(v[0].y));
    const float2 p2 = f16x2_bits_to_float2(__float_as_uint(v[0].z)), p3 = f16x2_bits_to_float2(__float_as_uint(v[0].w));
    a0 = make_float4(p0.x, p0.y, p1.x, p1.y);
    a1 = make_float4(p2.x, p2.y, p3.x, p3.y);
  }
}

__device__ __forceinline__ void split_tf32x4(float4 v, float4& h, float4& l) {
  split_tf32_fast(v.x, h.x, l.x); split_tf32_fast(v.y, h.y, l.y);
  split_tf32_fast(v.z, h.z, l.z); split_tf32_fast(v.w, h.w, l.w);
}

template <int N>
__device__ __forceinline__ void zero_acc(float (&acc)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.f;
}

// One 128-byte K row of MMAs (4 x k8 tf32 or 4 x k16 fp16) of this warpgroup: hi * hi products into `part`, the two
// cross terms of split operands into `part_x` (2^-11 smaller, so they no longer lengthen the chain that carries the
// large values) or, without kSepCross (part_x aliases part), into the same fragment; the first MMA into a fragment
// overwrites it: +32 bytes along K inside the swizzled row = +2 in the (address >> 4) start field of both descriptors.
// The caller adds `part` into its fp32 accumulators with ordinary (round-to-nearest) additions once the group has
// retired: the tensor core's own accumulation truncates, and over a K of thousands (3x3 convolutions over 512
// channels, weight gradients over ~1000 pixels per split) that drifts to many times the error of an fp32 sum.
// acc0 = 1 makes the first MMA accumulate too (the single-pass kernels accumulate straight into `acc`).
template <bool kF16, int kN, bool kSepCross>
__device__ __forceinline__ void mma_row(float (&part)[kN / 2], float (&part_x)[kN / 2], uint32_t a_hi, uint32_t a_lo,
                                        uint32_t b_hi, uint32_t b_lo, bool split, int acc0 = 0) {
  const uint64_t dah = gmma_desc_sw128(a_hi), dal = gmma_desc_sw128(a_lo);
  const uint64_t dbh = gmma_desc_sw128(b_hi), dbl = gmma_desc_sw128(b_lo);
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t o = (uint64_t)(kk * 2);
    const int acc = kk > 0 ? 1 : acc0;
    if (split) {
      if (kF16) {
        Wgmma<kN>::f16(part_x, dal + o, dbh + o, acc);
        Wgmma<kN>::f16(part_x, dah + o, dbl + o, 1);
      } else {
        Wgmma<kN>::tf32(part_x, dal + o, dbh + o, acc);
        Wgmma<kN>::tf32(part_x, dah + o, dbl + o, 1);
      }
    }
    const int acc_hh = (acc || (split && !kSepCross)) ? 1 : 0;   // one shared fragment: keep the cross terms
    if (kF16) Wgmma<kN>::f16(part, dah + o, dbh + o, acc_hh);
    else Wgmma<kN>::tf32(part, dah + o, dbh + o, acc_hh);
  }
}

template <int N>
__device__ __forceinline__ void add_part(float (&acc)[N], const float (&part)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] += part[i];
}
template <int N>
__device__ __forceinline__ void add_part(float (&acc)[N], const float (&part)[N], const float (&part_x)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] += part[i] + part_x[i];
}

// ===================================================== forward =====================================================

struct ConvParams {
  int B, H, W, Cin, Cout, ksize, P;
  int passes;
  int nt, n_tiles, num_tiles;
  int ncb, ksteps;             // channel blocks per tap, taps * ncb
  int b_tile_bytes, stage_bytes;
  const float* x;
  const void* w_hi;
  const void* w_lo;
  const float* pre_mean;
  const float* pre_scale;
  const float* pre_shift;
  int pre_relu;
  const float* bias;
  const float* residual;       // x, residual and y point to __half where the kernel's TIn / TOut is __half
  const float* relu_mask;
  float* y;
  float out_scale;
  const float* in_scale;       // nullable device float[2] {S, 1/S}: operands are x * S, the epilogue multiplies by 1/S
  double* stat_part;           // nullable [gridDim.x][Cout][2] = {sum (y - pivot), sum (y - pivot)^2}
  const float* stat_pivot;     // nullable [Cout]
  int halo_rows;               // conv_halo_kernel: kTileM + 2 W + 2 pixel rows + one zero row per channel block
  int halo_stages;             // conv_halo_kernel: weight stages in the TMA ring (2 or 3)
};

// Weights of K step ks for output columns [n0, n0 + nt): nt K-major rows of 128 bytes (one tap, kCB input channels)
// under the 128-byte swizzle, hi at `b`, lo at `b + b_lo_off`, by cp.async (one commit group); channels >= Cin are zeros.
template <bool kF16>
__device__ __forceinline__ void conv_load_b(const ConvParams& p, int ks, int n0, uint32_t b, uint32_t b_lo_off) {
  constexpr int kCB = kF16 ? 64 : 32;
  constexpr int kChunkEl = kF16 ? 8 : 4;    // weight elements per 16-byte chunk
  constexpr int kEl = kF16 ? 2 : 4;
  const bool split = p.passes == 3;
  const char* wh = reinterpret_cast<const char*>(p.w_hi);
  const char* wl = reinterpret_cast<const char*>(p.w_lo ? p.w_lo : p.w_hi);
  const int tap = ks / p.ncb, cb = ks - tap * p.ncb;
  for (int idx = threadIdx.x; idx < p.nt * 8; idx += kThreads) {
    const int n = idx >> 3, jj = idx & 7;
    const int c = cb * kCB + jj * kChunkEl;
    const bool ok = c < p.Cin;
    const size_t off = ((((size_t)tap * p.Cout + n0 + n) * p.Cin) + (ok ? c : 0)) * kEl;
    const uint32_t dst = b + (uint32_t)n * 128u + ((uint32_t)(jj ^ (n & 7)) << 4);
    cp_async16(dst, wh + off, ok);
    if (split) cp_async16(dst + b_lo_off, wl + off, ok);
  }
  cp_async_commit();
}

__device__ __forceinline__ void conv_stats_init(const ConvParams& p, double* s_stat) {
  if (p.stat_part) {
    for (int i = threadIdx.x; i < 8 * p.Cout * 2; i += kThreads) s_stat[i] = 0.0;
  }
}

// Epilogue of one 128 x kN tile: y = acc * oscale (+ bias) (+ residual) (ReLU mask), and the per-warp fp64 statistics.
// Fragment row g (+8), columns 8 i + 2 t (+1) of this warp's 16 rows. TOut: the type of y and the residual (__half:
// the same fp32 expression from float(residual), stored as a saturated fp16_rn).
template <int kN, typename TOut = float>
__device__ __forceinline__ void conv_epilogue(const ConvParams& p, const float (&acc)[kN / 2], int m0, int n0,
                                              float oscale, double* s_stat) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const bool stats = p.stat_part != nullptr;
  const int g = lane >> 2, t = lane & 3;
  const int mrow = m0 + wg * 64 + (warp & 3) * 16 + g;
  double* my_stat = s_stat + (size_t)warp * p.Cout * 2;
#pragma unroll
  for (int i = 0; i < kN / 8; ++i) {
    const int col = n0 + i * 8 + 2 * t;
    float2 b2 = make_float2(0.f, 0.f), pv = make_float2(0.f, 0.f);
    if (p.bias) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + col));
    if (stats && p.stat_pivot) pv = __ldg(reinterpret_cast<const float2*>(p.stat_pivot + col));
    double s1a = 0.0, s1b = 0.0, s2a = 0.0, s2b = 0.0;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int m = mrow + rr * 8;
      if (m >= p.P) continue;
      const size_t off = (size_t)m * p.Cout + col;
      float2 o = make_float2(acc[4 * i + 2 * rr] * oscale + b2.x, acc[4 * i + 2 * rr + 1] * oscale + b2.y);
      if (p.residual) {
        const float2 r2 = ld_act2(reinterpret_cast<const TOut*>(p.residual), off);
        o.x += r2.x; o.y += r2.y;
      }
      if (p.relu_mask) {
        const float2 k = __ldg(reinterpret_cast<const float2*>(p.relu_mask + off));
        o.x = k.x > 0.f ? o.x : 0.f; o.y = k.y > 0.f ? o.y : 0.f;
      }
      st_act2(reinterpret_cast<TOut*>(p.y), off, o);
      if (stats) {
        const double d0 = (double)(o.x - pv.x), d1 = (double)(o.y - pv.y);
        s1a += d0; s2a += d0 * d0; s1b += d1; s2b += d1 * d1;
      }
    }
    if (stats) {
#pragma unroll
      for (int sh = 4; sh < 32; sh <<= 1) {
        s1a += __shfl_xor_sync(0xffffffffu, s1a, sh); s2a += __shfl_xor_sync(0xffffffffu, s2a, sh);
        s1b += __shfl_xor_sync(0xffffffffu, s1b, sh); s2b += __shfl_xor_sync(0xffffffffu, s2b, sh);
      }
      if (g == 0) {   // lanes 0..3 own two distinct columns each: no conflicts, no atomics
        my_stat[(size_t)col * 2 + 0] += s1a; my_stat[(size_t)col * 2 + 1] += s2a;
        my_stat[(size_t)col * 2 + 2] += s1b; my_stat[(size_t)col * 2 + 3] += s2b;
      }
    }
  }
}

// One [Cout][2] statistics block per CTA: the eight per-warp accumulators merged in a fixed order (deterministic).
__device__ __forceinline__ void conv_stats_flush(const ConvParams& p, const double* s_stat) {
  if (p.stat_part) {
    __syncthreads();
    for (int i = threadIdx.x; i < p.Cout * 2; i += kThreads) {
      double v = 0.0;
      for (int w8 = 0; w8 < 8; ++w8) v += s_stat[(size_t)w8 * p.Cout * 2 + i];   // fixed order
      p.stat_part[(size_t)blockIdx.x * p.Cout * 2 + i] = v;
    }
  }
}

template <bool kF16, int kN>
__global__ void __launch_bounds__(kThreads, 1) conv_wgmma_kernel(const ConvParams p) {
  constexpr int kCB = kF16 ? 64 : 32;       // input channels per K step (one 128-byte operand row)
  constexpr int kV = kF16 ? 2 : 1;          // raw float4 per thread, row and K step
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  double* s_stat = reinterpret_cast<double*>(smem + (size_t)kStages * p.stage_bytes);
  const uint32_t smem_a = smem_u32(smem);
  const int tid = threadIdx.x, wg = tid >> 7;
  const bool split = p.passes == 3;
  const float in_s = p.in_scale ? __ldg(p.in_scale) : 1.f;
  const float oscale = p.in_scale ? p.out_scale * __ldg(p.in_scale + 1) : p.out_scale;
  const uint32_t a_lo_off = split ? (uint32_t)kATileBytes : 0u;
  const uint32_t b_off = (split ? 2u : 1u) * (uint32_t)kATileBytes;
  const uint32_t b_lo_off = split ? (uint32_t)p.b_tile_bytes : 0u;
  conv_stats_init(p, s_stat);
  __syncthreads();

  // A tile: thread -> 16-byte chunk j of rows r0 + 32 i
  const int j = tid & 7, r0 = tid >> 3;
  const int HW = p.H * p.W;

  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int m0 = (tile / p.n_tiles) * kTileM;
    const int n0 = (tile % p.n_tiles) * p.nt;
    int pn[4], ph[4], pw[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + r0 + 32 * i;
      pn[i] = m < p.P ? m / HW : p.B;   // pn == B marks a row past the last pixel
      ph[i] = (m % HW) / p.W;
      pw[i] = m % p.W;
    }
    float4 ra[4][kV];
    uint32_t okm = 0;
    auto load_a = [&](int ks) {
      const int tap = ks / p.ncb, cb = ks - tap * p.ncb;
      const int dh = p.ksize == 3 ? tap / 3 - 1 : 0, dw = p.ksize == 3 ? tap % 3 - 1 : 0;
      const int c = cb * kCB + j * 4 * kV;
      okm = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int hh = ph[i] + dh, ww = pw[i] + dw;
        const bool ok = pn[i] < p.B && hh >= 0 && hh < p.H && ww >= 0 && ww < p.W && c < p.Cin;
#pragma unroll
        for (int v = 0; v < kV; ++v) ra[i][v] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok) {
          okm |= 1u << i;
          const float* src = p.x + (((size_t)pn[i] * p.H + hh) * p.W + ww) * (size_t)p.Cin + c;
#pragma unroll
          for (int v = 0; v < kV; ++v) ra[i][v] = __ldg(reinterpret_cast<const float4*>(src) + v);
        }
      }
    };
    auto store_a = [&](int ks, uint32_t st) {
      const int cb = ks % p.ncb;
      const int c = cb * kCB + j * 4 * kV;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = r0 + 32 * i;
        const uint32_t dst = st + (uint32_t)r * 128u + ((uint32_t)(j ^ (r & 7)) << 4);
        uint4 oh = make_uint4(0u, 0u, 0u, 0u), ol = make_uint4(0u, 0u, 0u, 0u);
        if (okm & (1u << i)) {
          float4 v[kV];
#pragma unroll
          for (int u = 0; u < kV; ++u) {
            v[u] = affine_relu4(ra[i][u], p.pre_mean, p.pre_scale, p.pre_shift, c + 4 * u, p.pre_relu);
            v[u].x *= in_s; v[u].y *= in_s; v[u].z *= in_s; v[u].w *= in_s;
          }
          if (kF16) {
            split_f16x2(v[0].x, v[0].y, oh.x, ol.x);
            split_f16x2(v[0].z, v[0].w, oh.y, ol.y);
            split_f16x2(v[kV - 1].x, v[kV - 1].y, oh.z, ol.z);
            split_f16x2(v[kV - 1].z, v[kV - 1].w, oh.w, ol.w);
          } else {
            float4 h, l;
            split_tf32x4(v[0], h, l);
            oh = make_uint4(__float_as_uint(h.x), __float_as_uint(h.y), __float_as_uint(h.z), __float_as_uint(h.w));
            ol = make_uint4(__float_as_uint(l.x), __float_as_uint(l.y), __float_as_uint(l.z), __float_as_uint(l.w));
          }
        }
        sts128u(dst, oh);
        if (split) sts128u(dst + a_lo_off, ol);
      }
    };
    // one partial for all terms here: a separate cross-term partial would push the fp16 N = 128 form past 255 registers
    float acc[kN / 2], part[kN / 2];
    zero_acc(acc);
    zero_acc(part);
    conv_load_b<kF16>(p, 0, n0, smem_a + b_off, b_lo_off);
    load_a(0);
    for (int ks = 0; ks < p.ksteps; ++ks) {
      const uint32_t st = smem_a + (uint32_t)((ks % kStages) * p.stage_bytes);
      store_a(ks, st);   // overlaps the MMAs of step ks - 1
      if (ks > 0) {
        wgmma_wait<0>();
        add_part(acc, part);
      }
      cp_async_wait_all();
      fence_proxy_async_smem();
      __syncthreads();
      if (ks + 1 < p.ksteps) {
        conv_load_b<kF16>(p, ks + 1, n0, smem_a + (uint32_t)(((ks + 1) % kStages) * p.stage_bytes) + b_off, b_lo_off);
        load_a(ks + 1);
      }
      wgmma_fence();
      const uint32_t a_hi = st + (uint32_t)wg * 64u * 128u;
      mma_row<kF16, kN, false>(part, part, a_hi, a_hi + a_lo_off, st + b_off, st + b_off + b_lo_off, split);
      wgmma_commit();
    }
    wgmma_wait<0>();
    add_part(acc, part);
    __syncthreads();   // every warpgroup is done with every stage: the next tile may refill them

    conv_epilogue<kN>(p, acc, m0, n0, oscale, s_stat);
  }
  conv_stats_flush(p, s_stat);
}

// ================================================ forward, 3x3 halo ================================================
// conv_halo_kernel: the 3x3, 3xFP16 case of conv_wgmma_kernel<true, kN> with the A operand prepared once per tile instead
// of once per K step. Tiles, K order (tap-major, then channel block) and products are those of conv_wgmma_kernel, so every
// output is bit-identical to it; only where A comes from differs.
//   Halo: the tile's nine taps read pixels [m0 - W - 1, m0 + 128 + W + 1) of the flattened B*H*W sequence, one contiguous
//   NHWC range. Every thread loads its share once per tile, applies the affine + ReLU, in_scale and the fp16 hi/lo split
//   exactly as store_a does, and stores fp16 hi and lo planes in shared memory: [channel block][row][128 B], 16-byte
//   chunks XOR-swizzled by row & 7 (ldmatrix over 8 consecutive rows is conflict-free). Pixels outside [0, P) and
//   channels >= Cin are zeros; row halo_rows - 1 of every channel block is all zero.
//   Step ks (tap = ks / ncb, cb = ks % ncb): output pixel m reads the halo row of pixel m + dh W + dw, or the zero row when
//   that neighbour lies outside m's image (or m >= P). ldmatrix.x4 loads each warp's 16 rows x k16 (hi and lo) straight
//   into the register-A fragment of wgmma; B comes from the swizzled weight stage as before. (Shifted shared-memory A
//   descriptors cannot do this: at dw = +-1 the pixel past a row end is a real pixel of the next image row, not zero, and
//   an odd row shift breaks the 128-byte swizzle phase.)
//   Per k16: lo * hi, hi * lo, hi * hi into `part` (mma_row's order), `acc += part` once per step. The A registers are
//   rewritten only after wgmma_wait<0>.
//   Weights: a ring of S = halo_stages (2 or 3) stages, each {B hi, B lo} of one K step, filled by TMA from two 2-D tensor
//   maps over the [tap][Cout][Cin] fp16 weights (rows of Cin, box 64 channels x nt rows, 128-byte swizzle: the layout
//   mma_row's B descriptors read; channels >= Cin are zero-filled). The CTA's (tile, K step) sequence is one stream of
//   steps s = 0, 1, ...; step s uses stage s % S, and its fill is phase s / S of full[s % S] (one arrive with expect_tx
//   for the two boxes) and its release phase s / S of empty[s % S] (one arrive per warp, after that warp's
//   wgmma_wait<0> has retired the step's MMAs: 8 arrivals). The ring runs across tiles, so the first S - 1 steps of the
//   CTA's next tile load during the epilogue and the halo fill.
//   Ping-pong: the warpgroups take turns to issue their MMAs of a step, warpgroup 0 first, through two named barriers
//   (turn[wg] = kTurnBar + wg; a warpgroup syncs on its own turn, then arrives on the other's once its MMAs are issued;
//   warpgroup 0 does not wait before the CTA's first step, warpgroup 1 does not hand over after the CTA's last). The
//   tensor cores run each warpgroup's 12 MMAs of a step in issue order, so warpgroup 0's drain, accumulator adds and
//   ldmatrix of the next step overlap warpgroup 1's MMAs and the other way round; without the turns both warpgroups
//   stay in step (they start every tile together) and drain at the same time. A warpgroup can arrive on a turn barrier
//   again only after the other has synced on it, so no turn phase is skipped.
//   Producer: thread kTileM (warpgroup 1, the second to issue) fills step s + S - 1 into the stage of step s - 1 right
//   after its warpgroup has issued the MMAs of step s. Its wait on empty[(s - 1) % S] never blocks: its own warpgroup
//   released step s - 1 before issuing step s, and warpgroup 0 released it before issuing step s, which came before
//   warpgroup 1's turn. So the producer never holds back a warpgroup's MMA issue, and waits on full never depend on a
//   warpgroup the waiter is itself holding. Parity waits are unambiguous: a stage is refilled only after both
//   warpgroups released its previous step, so no barrier runs two phases ahead of a waiter. Two CTA barriers per tile
//   remain, around the halo fill that both warpgroups read.
constexpr int kHaloBatch = 8;   // halo chunks per thread in flight (2 x float4 each)
constexpr int kTurnBar = 1;     // named barriers kTurnBar + wg: warpgroup wg may issue its MMAs (0 is __syncthreads)

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@!p bra WAIT;\n}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}

// conv_halo_f16x1_kernel: the single-pass form (kSplit = false) of the same body. Activation operand fp16_rn(x), the
// hi plane alone (half the halo, half the ldmatrix), weights the one box of w * 2^8 per stage. One register-A MMA per k16
// straight into `acc` for the whole K loop: with fp16-rounded operands (relative 2^-11) the tensor core's accumulation
// drift no longer matters, so no per-step fragment. The A fragments are double-buffered (step parity) and every step
// ends with wgmma_wait<1>, so step s + 1 issues while step s is still in the tensor core; that wait retires step s - 1,
// whose stage the warp releases then. The producer therefore fills step s + S - 2 into the stage of step s - 2 (both
// warpgroups released it during step s - 1, before warpgroup 0's turn for step s), and the ring has S >= 3 stages.
//   Half-precision activations (TIn / TOut = __half, single-pass only): the halo fill reads 16 bytes per 8 channels
// instead of 32 and applies the same fp32 transform to float(x); the epilogue is conv_epilogue<kN, TOut>.
template <int kN, bool kSplit, typename TIn = float, typename TOut = float>
__device__ __forceinline__ void conv_halo_body(const ConvParams& p, const CUtensorMap& w_hi_map,
                                               const CUtensorMap& w_lo_map) {
  static_assert(!kSplit || (std::is_same<TIn, float>::value && std::is_same<TOut, float>::value),
                "half-precision activations only on the single-pass kernel");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int R = p.halo_rows;
  const uint32_t S = (uint32_t)p.halo_stages;
  const uint32_t ahead = kSplit ? S - 1u : S - 2u;                 // steps in the ring ahead of the one being issued
  const uint32_t lo_plane = (uint32_t)p.ncb * (uint32_t)R * 128u;
  const uint32_t smem_b = smem_u32(smem);                          // S x {B hi, B lo}
  const uint32_t halo = smem_b + S * (uint32_t)p.stage_bytes;      // hi plane, then lo plane
  double* s_stat = reinterpret_cast<double*>(smem + (size_t)S * p.stage_bytes + (kSplit ? 2 : 1) * (size_t)lo_plane);
  const uint32_t full = smem_u32(s_stat) + (p.stat_part ? 16u * 8u * (uint32_t)p.Cout : 0u);   // S mbarriers
  const uint32_t empty = full + 8u * S;                                                         // S mbarriers
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const float in_s = p.in_scale ? __ldg(p.in_scale) : 1.f;
  const float oscale = p.in_scale ? p.out_scale * __ldg(p.in_scale + 1) : p.out_scale;
  const uint32_t b_lo_off = (uint32_t)p.b_tile_bytes;
  // fill of stream step s = (tile, ks): thread 0 for the first `ahead` steps (after the barrier init), then thread kTileM
  auto load_b = [&](uint32_t s, int tile, int ks) {
    const uint32_t st = s % S;
    if (s >= S) mbar_wait(empty + 8u * st, (s / S - 1u) & 1u);
    const uint32_t bar = full + 8u * st, dst = smem_b + st * (uint32_t)p.stage_bytes;
    const int tap = ks / p.ncb, cb = ks - tap * p.ncb;
    const int row = tap * p.Cout + (tile % p.n_tiles) * p.nt;
    mbar_arrive_expect_tx(bar, (kSplit ? 2u : 1u) * (uint32_t)p.b_tile_bytes);
    tma_load_2d(dst, &w_hi_map, cb * 64, row, bar);
    if (kSplit) tma_load_2d(dst + b_lo_off, &w_lo_map, cb * 64, row, bar);
  };
  if (tid == 0) {
    for (uint32_t i = 0; i < S; ++i) {
      mbar_init(full + 8u * i, 1);
      mbar_init(empty + 8u * i, kThreads / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (uint32_t s = 0; s < ahead; ++s) load_b(s, blockIdx.x, (int)s);   // ksteps >= 9 > ahead
  }
  conv_stats_init(p, s_stat);
  for (int i = tid; i < p.ncb * 8; i += kThreads) {   // the zero rows: never overwritten by the halo loads
    const uint32_t dst = halo + (uint32_t)((i >> 3) * R + R - 1) * 128u + ((uint32_t)(i & 7) << 4);
    sts128u(dst, make_uint4(0u, 0u, 0u, 0u));
    if (kSplit) sts128u(dst + lo_plane, make_uint4(0u, 0u, 0u, 0u));
  }

  const int HW = p.H * p.W;
  // this lane's ldmatrix.x4 row among the tile's 128 and its k half: matrices {rows 0-7, rows 8-15} x {k 0-7, k 8-15}
  // of the warp's 16 rows, in the order of the A fragment registers
  const int lr = wg * 64 + (warp & 3) * 16 + (lane & 7) + (lane & 8);
  const uint32_t khalf = (uint32_t)(lane >> 4);
  const int items = p.ncb * (R - 1) * 8;   // 16-byte chunks of one halo plane, zero rows excluded
  uint32_t s = 0;                          // stream step

  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int m0 = (tile / p.n_tiles) * kTileM;
    const int n0 = (tile % p.n_tiles) * p.nt;
    const int hs = m0 - p.W - 1;   // pixel of halo row 0

    // ---- halo: chunk idx = (row * ncb + cb) * 8 + jj covers channels cb * 64 + 8 jj .. + 7 of pixel hs + row, so
    // consecutive threads read consecutive 32-byte pieces of the NHWC span
    for (int base = tid; base < items; base += kThreads * kHaloBatch) {
      float4 v[kHaloBatch][2];
#pragma unroll
      for (int u = 0; u < kHaloBatch; ++u) {
        const int idx = base + u * kThreads;
        const int jj = idx & 7, rc = idx >> 3;
        const int r = rc / p.ncb, cb = rc - r * p.ncb;
        const int q = hs + r, c = cb * 64 + jj * 8;
        v[u][0] = v[u][1] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (idx < items && q >= 0 && q < p.P && c < p.Cin) ld_raw8<TIn>(p.x, (size_t)q * p.Cin + c, v[u]);
      }
#pragma unroll
      for (int u = 0; u < kHaloBatch; ++u) {
        const int idx = base + u * kThreads;
        if (idx >= items) continue;
        const int jj = idx & 7, rc = idx >> 3;
        const int r = rc / p.ncb, cb = rc - r * p.ncb;
        const int q = hs + r, c = cb * 64 + jj * 8;
        uint4 oh = make_uint4(0u, 0u, 0u, 0u), ol = make_uint4(0u, 0u, 0u, 0u);
        if (q >= 0 && q < p.P && c < p.Cin) {
          float4 a0, a1;
          cvt_raw8<TIn>(v[u], a0, a1);
          a0 = affine_relu4(a0, p.pre_mean, p.pre_scale, p.pre_shift, c, p.pre_relu);
          a1 = affine_relu4(a1, p.pre_mean, p.pre_scale, p.pre_shift, c + 4, p.pre_relu);
          a0.x *= in_s; a0.y *= in_s; a0.z *= in_s; a0.w *= in_s;
          a1.x *= in_s; a1.y *= in_s; a1.z *= in_s; a1.w *= in_s;
          split_f16x2(a0.x, a0.y, oh.x, ol.x);
          split_f16x2(a0.z, a0.w, oh.y, ol.y);
          split_f16x2(a1.x, a1.y, oh.z, ol.z);
          split_f16x2(a1.z, a1.w, oh.w, ol.w);
        }
        const uint32_t dst = halo + (uint32_t)(cb * R + r) * 128u + ((uint32_t)(jj ^ (r & 7)) << 4);
        sts128u(dst, oh);
        if (kSplit) sts128u(dst + lo_plane, ol);
      }
    }

    __syncthreads();   // the halo is visible

    const int m = m0 + lr;
    const int pn = m < p.P ? m / HW : p.B;   // pn == B marks a row past the last pixel
    const int ph = (m % HW) / p.W, pw = m % p.W;
    float acc[kN / 2];
    zero_acc(acc);
    if constexpr (!kSplit) {
      uint32_t ah[2][4][4];   // A fragments of steps of even / odd parity
      // step s = (tile, ks) of the stream; `buf` (a compile-time step parity) selects its A fragments
      auto step = [&](int ks, auto buf) {
        constexpr int kb = decltype(buf)::value;
        const uint32_t st = s % S;
        const int tap = ks / p.ncb, cb = ks - tap * p.ncb;
        const int dh = tap / 3 - 1, dw = tap % 3 - 1;
        const int hh = ph + dh, ww = pw + dw;
        const bool ok = pn < p.B && hh >= 0 && hh < p.H && ww >= 0 && ww < p.W;
        const int hr = ok ? lr + (dh + 1) * p.W + dw + 1 : R - 1;
        const uint32_t row = halo + (uint32_t)(cb * R + hr) * 128u;
        const uint32_t sw = (uint32_t)(hr & 7);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) ldsm_x4(ah[kb][kk], row + (((2u * kk + khalf) ^ sw) << 4));
        mbar_wait(full + 8u * st, (s / S) & 1u);   // the weights of step s have landed
        if (wg == 1 || s > 0) named_bar_sync(kTurnBar + wg, kThreads);   // this warpgroup's turn to issue
        wgmma_fence();
        const uint64_t db = gmma_desc_sw128(smem_b + st * (uint32_t)p.stage_bytes);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) WgmmaRA<kN>::f16(acc, ah[kb][kk], db + (uint64_t)(kk * 2), 1);
        wgmma_commit();
        if (wg == 0 || ks + 1 < p.ksteps || tile + (int)gridDim.x < p.num_tiles)
          named_bar_arrive(kTurnBar + 1 - wg, kThreads);   // the other warpgroup's turn (none after the CTA's last step)
        wgmma_wait<1>();   // step s - 1 has retired: its A fragments and its weight stage are free
        if (ks > 0 && lane == 0) mbar_arrive(empty + 8u * ((s - 1u) % S));
        if (tid == kTileM) {   // fill step s + S - 2 into the stage of step s - 2
          int lt = tile, lks = ks + (int)ahead;
          if (lks >= p.ksteps) {
            lks -= p.ksteps;
            lt += gridDim.x;
          }
          if (lt < p.num_tiles) load_b(s + ahead, lt, lks);
        }
        __syncwarp();
        ++s;
      };
      int ks = 0;
      for (; ks + 1 < p.ksteps; ks += 2) {
        step(ks, std::integral_constant<int, 0>());
        step(ks + 1, std::integral_constant<int, 1>());
      }
      if (ks < p.ksteps) step(ks, std::integral_constant<int, 0>());
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(empty + 8u * ((s - 1u) % S));
      __syncthreads();   // every warpgroup is done with the halo: the next tile may refill it
      conv_epilogue<kN, TOut>(p, acc, m0, n0, oscale, s_stat);
      continue;
    }
    float part[kN / 2];
    zero_acc(part);
    for (int ks = 0; ks < p.ksteps; ++ks, ++s) {
      const uint32_t st = s % S;
      if (ks > 0) {
        wgmma_wait<0>();
        add_part(acc, part);
        if (lane == 0) mbar_arrive(empty + 8u * ((s - 1u) % S));   // this warp is done with step s - 1
      }
      const int tap = ks / p.ncb, cb = ks - tap * p.ncb;
      const int dh = tap / 3 - 1, dw = tap % 3 - 1;
      const int hh = ph + dh, ww = pw + dw;
      const bool ok = pn < p.B && hh >= 0 && hh < p.H && ww >= 0 && ww < p.W;
      const int hr = ok ? lr + (dh + 1) * p.W + dw + 1 : R - 1;
      const uint32_t row = halo + (uint32_t)(cb * R + hr) * 128u;
      const uint32_t sw = (uint32_t)(hr & 7);
      uint32_t ah[4][4], al[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t a = row + (((2u * kk + khalf) ^ sw) << 4);
        ldsm_x4(ah[kk], a);
        ldsm_x4(al[kk], a + lo_plane);
      }
      mbar_wait(full + 8u * st, (s / S) & 1u);   // the weights of step s have landed
      if (wg == 1 || s > 0) named_bar_sync(kTurnBar + wg, kThreads);   // this warpgroup's turn to issue
      wgmma_fence();
      const uint32_t b = smem_b + st * (uint32_t)p.stage_bytes;
      const uint64_t dbh = gmma_desc_sw128(b), dbl = gmma_desc_sw128(b + b_lo_off);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t o = (uint64_t)(kk * 2);
        WgmmaRA<kN>::f16(part, al[kk], dbh + o, kk > 0 ? 1 : 0);
        WgmmaRA<kN>::f16(part, ah[kk], dbl + o, 1);
        WgmmaRA<kN>::f16(part, ah[kk], dbh + o, 1);
      }
      wgmma_commit();
      if (wg == 0 || ks + 1 < p.ksteps || tile + (int)gridDim.x < p.num_tiles)
        named_bar_arrive(kTurnBar + 1 - wg, kThreads);   // the other warpgroup's turn (none after the CTA's last step)
      if (tid == kTileM) {   // fill step s + S - 1 into the stage of step s - 1
        int lt = tile, lks = ks + (int)S - 1;
        if (lks >= p.ksteps) {
          lks -= p.ksteps;
          lt += gridDim.x;
        }
        if (lt < p.num_tiles) load_b(s + S - 1u, lt, lks);
      }
      __syncwarp();
    }
    wgmma_wait<0>();
    add_part(acc, part);
    if (lane == 0) mbar_arrive(empty + 8u * ((s - 1u) % S));
    __syncthreads();   // every warpgroup is done with the halo: the next tile may refill it

    conv_epilogue<kN>(p, acc, m0, n0, oscale, s_stat);
  }
  conv_stats_flush(p, s_stat);
}

template <int kN>
__global__ void __launch_bounds__(kThreads, 1)
    conv_halo_kernel(const __grid_constant__ ConvParams p, const __grid_constant__ CUtensorMap w_hi_map,
                     const __grid_constant__ CUtensorMap w_lo_map) {
  conv_halo_body<kN, true>(p, w_hi_map, w_lo_map);
}

template <int kN, typename TIn = float, typename TOut = float>
__global__ void __launch_bounds__(kThreads, 1)
    conv_halo_f16x1_kernel(const __grid_constant__ ConvParams p, const __grid_constant__ CUtensorMap w_map) {
  conv_halo_body<kN, false, TIn, TOut>(p, w_map, w_map);
}

// ============================================ forward, 1x1 resident weights ============================================
// pw_conv_wgmma_kernel: the 1x1, 3xFP16 case of conv_wgmma_kernel<true, kN> (without statistics) for shapes whose
// weight slice fits in shared memory. Grid, tiles (m = tile / n_tiles, n = tile % n_tiles), K order, the A transform
// (store_a) and the MMAs (mma_row: per k16 lo * hi, hi * lo, hi * hi into `part`, then acc += part once per K step) are
// those of conv_wgmma_kernel, and the epilogue evaluates the same expression per element, so every output is
// bit-identical to it. (The name keeps the conv_wgmma_kernel family name that the profiling tools match on.)
//   Resident weights: the hi/lo weights of the CTA's output slice, all ncb channel blocks, are loaded once under the
//   128-byte swizzle and stay in shared memory; they are reloaded only when the CTA's next tile belongs to another slice
//   (never when gridDim.x is a multiple of n_tiles, as it is for every Cout these models use on 132 SMs).
//   Loads that cross tiles: the CTA's (tile, K step) sequence is one stream. The raw NHWC rows of the next step in the
//   stream, including step 0 of the CTA's next tile, are requested right after the step's barrier, so they are in flight
//   during the MMAs and the epilogue. Two A stages: stage s % 2 is rewritten by step s only after the step s - 1 barrier,
//   which follows every warpgroup's wgmma_wait<0> for step s - 2, the last reader of that stage.
//   Epilogue inputs: the tile's residual and ReLU-mask rows are prefetched into L2 (one bulk prefetch per row) before its
//   MMAs, and the epilogue reads them in batches of kPwEpiCols fragment columns before computing any of those outputs.
//   (Prefetching the next tile's input rows into L2 the same way made most shapes slower on the H100, and was dropped.)
constexpr int kPwStages = 2;
constexpr int kPwEpiCols = 8;

__device__ __forceinline__ void prefetch_l2(const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}

template <int kN, typename TOut = float>
__device__ __forceinline__ void pw_epilogue(const ConvParams& p, const float (&acc)[kN / 2], int m0, int n0,
                                            float oscale) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int g = lane >> 2, t = lane & 3;
  const int mrow = m0 + wg * 64 + (warp & 3) * 16 + g;
#pragma unroll
  for (int i0 = 0; i0 < kN / 8; i0 += kPwEpiCols) {
    float2 r2[kPwEpiCols][2], k2[kPwEpiCols][2];
#pragma unroll
    for (int u = 0; u < kPwEpiCols; ++u) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = mrow + rr * 8;
        r2[u][rr] = k2[u][rr] = make_float2(0.f, 0.f);
        if (i0 + u >= kN / 8 || m >= p.P) continue;
        const size_t off = (size_t)m * p.Cout + n0 + (i0 + u) * 8 + 2 * t;
        if (p.residual) r2[u][rr] = ld_act2(reinterpret_cast<const TOut*>(p.residual), off);
        if (p.relu_mask) k2[u][rr] = __ldg(reinterpret_cast<const float2*>(p.relu_mask + off));
      }
    }
#pragma unroll
    for (int u = 0; u < kPwEpiCols; ++u) {
      const int i = i0 + u;
      if (i >= kN / 8) continue;
      const int col = n0 + i * 8 + 2 * t;
      float2 b2 = make_float2(0.f, 0.f);
      if (p.bias) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = mrow + rr * 8;
        if (m >= p.P) continue;
        float2 o = make_float2(acc[4 * i + 2 * rr] * oscale + b2.x, acc[4 * i + 2 * rr + 1] * oscale + b2.y);
        if (p.residual) {
          o.x += r2[u][rr].x; o.y += r2[u][rr].y;
        }
        if (p.relu_mask) {
          o.x = k2[u][rr].x > 0.f ? o.x : 0.f; o.y = k2[u][rr].y > 0.f ? o.y : 0.f;
        }
        st_act2(reinterpret_cast<TOut*>(p.y), (size_t)m * p.Cout + col, o);
      }
    }
  }
}

// pw_conv_f16x1_kernel: the single-pass form (kSplit = false): hi-only A stages and weights (16 KB per stage, so the
// slice fits up to Cin = 640 at 128 columns), one MMA per k16 straight into `acc`. Three A stages and wgmma_wait<1>
// before each step's barrier keep one step's MMAs in flight across it: stage s % 3 is rewritten by step s after the
// barrier of step s - 1, which follows every warpgroup's retirement of step s - 3.
//   Optional epilogue statistics (training calls): the [8 warps][Cout][2] fp64 accumulators follow the resident
// weights; tiles with statistics take conv_epilogue (same outputs as pw_epilogue, plus the per-warp sums) and the CTA
// flushes one block at the end, merged in the fixed order of conv_stats_flush. The 3-pass kernel has no statistics.
//   Half-precision activations (TIn / TOut = __half, single-pass only): the A staging loads 16 bytes per row and K step
// instead of 32 and transforms float(x) as before; the epilogue is pw_epilogue<kN, TOut>.
constexpr int kPwStages1 = 3;

size_t pw_smem_bytes(bool split, int ncb, int nt) {
  return 1024 + (size_t)(split ? kPwStages : kPwStages1) * (split ? 2 : 1) * kATileBytes +
         (size_t)ncb * (split ? 2 : 1) * nt * 128;
}

template <int kN, bool kSplit, typename TIn = float, typename TOut = float>
__device__ __forceinline__ void pw_conv_body(const ConvParams& p) {
  static_assert(!kSplit || (std::is_same<TIn, float>::value && std::is_same<TOut, float>::value),
                "half-precision activations only on the single-pass kernel");
  constexpr uint32_t kAStage = (kSplit ? 2u : 1u) * kATileBytes;   // A hi, then A lo
  constexpr uint32_t kNumStages = kSplit ? kPwStages : kPwStages1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t smem_a = smem_u32(smem);                        // kNumStages x {A hi, A lo}
  const uint32_t smem_w = smem_a + kNumStages * kAStage;         // ncb x {B hi, B lo}
  const uint32_t w_step = (kSplit ? 2u : 1u) * (uint32_t)p.b_tile_bytes;
  const int tid = threadIdx.x, wg = tid >> 7;
  const float in_s = p.in_scale ? __ldg(p.in_scale) : 1.f;
  const float oscale = p.in_scale ? p.out_scale * __ldg(p.in_scale + 1) : p.out_scale;
  double* s_stat = reinterpret_cast<double*>(smem + (size_t)kNumStages * kAStage + (size_t)p.ncb * w_step);
  if constexpr (!kSplit) conv_stats_init(p, s_stat);   // visible after the first K step's barrier

  // A tile: thread -> 16-byte chunk j (channels 8 j .. 8 j + 7 of the block) of rows r0 + 32 i
  const int j = tid & 7, r0 = tid >> 3;
  float4 ra[4][2];
  uint32_t okm = 0;
  auto load_a = [&](int m0, int cb) {
    const int c = cb * 64 + j * 8;
    okm = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + r0 + 32 * i;
      ra[i][0] = ra[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < p.P && c < p.Cin) {
        okm |= 1u << i;
        ld_raw8<TIn>(p.x, (size_t)m * p.Cin + c, ra[i]);
      }
    }
  };
  auto store_a = [&](int cb, uint32_t st) {   // conv_wgmma_kernel's store_a for kF16
    const int c = cb * 64 + j * 8;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = r0 + 32 * i;
      const uint32_t dst = st + (uint32_t)r * 128u + ((uint32_t)(j ^ (r & 7)) << 4);
      uint4 oh = make_uint4(0u, 0u, 0u, 0u), ol = make_uint4(0u, 0u, 0u, 0u);
      if (okm & (1u << i)) {
        float4 v[2];
        cvt_raw8<TIn>(ra[i], v[0], v[1]);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          v[u] = affine_relu4(v[u], p.pre_mean, p.pre_scale, p.pre_shift, c + 4 * u, p.pre_relu);
          v[u].x *= in_s; v[u].y *= in_s; v[u].z *= in_s; v[u].w *= in_s;
        }
        split_f16x2(v[0].x, v[0].y, oh.x, ol.x);
        split_f16x2(v[0].z, v[0].w, oh.y, ol.y);
        split_f16x2(v[1].x, v[1].y, oh.z, ol.z);
        split_f16x2(v[1].z, v[1].w, oh.w, ol.w);
      }
      sts128u(dst, oh);
      if (kSplit) sts128u(dst + (uint32_t)kATileBytes, ol);
    }
  };

  int w_n0 = -1;       // output slice whose weights are resident
  uint32_t s = 0;      // step of the CTA's stream: selects the A stage
  load_a((blockIdx.x / p.n_tiles) * kTileM, 0);
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int m0 = (tile / p.n_tiles) * kTileM;
    const int n0 = (tile % p.n_tiles) * p.nt;
    if (n0 != w_n0) {
      __syncthreads();   // every warpgroup has retired the MMAs that read the previous slice
      for (int ks = 0; ks < p.ncb; ++ks) conv_load_b<true>(p, ks, n0, smem_w + (uint32_t)ks * w_step, p.b_tile_bytes);
      w_n0 = n0;
    }
    if (tid < kTileM) {   // the epilogue inputs of this tile: row m0 + tid, columns [n0, n0 + nt)
      const int m = m0 + tid;
      const size_t off = (size_t)m * p.Cout + n0;
      if (m < p.P && p.residual)
        prefetch_l2(reinterpret_cast<const TOut*>(p.residual) + off, (uint32_t)p.nt * (uint32_t)sizeof(TOut));
      if (m < p.P && p.relu_mask) prefetch_l2(p.relu_mask + off, (uint32_t)p.nt * 4u);
    }
    float acc[kN / 2], part[kN / 2];
    zero_acc(acc);
    zero_acc(part);
    for (int ks = 0; ks < p.ncb; ++ks, ++s) {
      const uint32_t st = smem_a + (s % kNumStages) * kAStage;
      store_a(ks, st);   // overlaps the MMAs of step ks - 1
      if (!kSplit) {
        wgmma_wait<1>();   // step ks - 2 has retired
      } else if (ks > 0) {
        wgmma_wait<0>();
        add_part(acc, part);
      }
      cp_async_wait_all();   // resident weights (after a slice change)
      fence_proxy_async_smem();
      __syncthreads();
      if (ks + 1 < p.ncb) load_a(m0, ks + 1);
      else if (tile + (int)gridDim.x < p.num_tiles) load_a(((tile + gridDim.x) / p.n_tiles) * kTileM, 0);
      wgmma_fence();
      const uint32_t a_hi = st + (uint32_t)wg * 64u * 128u;
      const uint32_t b = smem_w + (uint32_t)ks * w_step;
      if (kSplit) mma_row<true, kN, false>(part, part, a_hi, a_hi + kATileBytes, b, b + p.b_tile_bytes, true);
      else mma_row<true, kN, false>(acc, acc, a_hi, a_hi, b, b, false, 1);
      wgmma_commit();
    }
    wgmma_wait<0>();
    if (kSplit) add_part(acc, part);
    if constexpr (!kSplit) {
      if (p.stat_part) {
        conv_epilogue<kN, TOut>(p, acc, m0, n0, oscale, s_stat);
        continue;
      }
    }
    pw_epilogue<kN, TOut>(p, acc, m0, n0, oscale);
  }
  if constexpr (!kSplit) conv_stats_flush(p, s_stat);
}

template <int kN>
__global__ void __launch_bounds__(kThreads, 1) pw_conv_wgmma_kernel(const __grid_constant__ ConvParams p) {
  pw_conv_body<kN, true>(p);
}

template <int kN, typename TIn = float, typename TOut = float>
__global__ void __launch_bounds__(kThreads, 1) pw_conv_f16x1_kernel(const __grid_constant__ ConvParams p) {
  pw_conv_body<kN, false, TIn, TOut>(p);
}

// Output channels are processed in slices of nt columns: the widest divisor of Cout that is a multiple of 16 and at
// most 128 (one wgmma N per slice; the accumulators of a 64 x 128 warpgroup tile take 64 registers per thread).
int conv_tc_ts_slice(int Cout) {
  if (Cout <= 128) return Cout % 16 == 0 ? Cout : 0;
  for (int nt = 128; nt >= 16; nt -= 16)
    if (Cout % nt == 0) return nt;
  return 0;
}

bool conv_shape_ok(int Cin, int Cout, int ksize, int f16, int max_cin, int max_cout) {
  return (ksize == 1 || ksize == 3) && Cin >= 4 && Cin <= max_cin && Cin % (f16 ? 8 : 4) == 0 && Cout >= 16 &&
         Cout <= max_cout && Cout % 16 == 0 && conv_tc_ts_slice(Cout) > 0;
}

int conv_num_tiles(int B, int H, int W, int Cout) {
  const long long P = (long long)B * H * W;
  return (int)((P + kTileM - 1) / kTileM) * (Cout / conv_tc_ts_slice(Cout));
}

// Raises a kernel's dynamic shared-memory limit once per device (the attribute is per device; `done` holds one bit per
// device ordinal). Concurrent first calls may both set it, which is harmless: the call is idempotent.
template <typename Kernel>
int allow_smem(Kernel kernel, std::atomic<uint64_t>& done) {
  int dev = 0;
  FPD_CUDA_CHECK(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (!(done.load(std::memory_order_acquire) & bit)) {
    FPD_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    done.fetch_or(bit, std::memory_order_release);
  }
  return FPD_OK;
}

// Launches kKernel, with its dynamic shared-memory limit raised first (once per device).
template <auto kKernel, typename... Args>
int launch(int grid, int threads, size_t smem, cudaStream_t stream, const Args&... args) {
  static std::atomic<uint64_t> done{0};
  if (int rc = allow_smem(kKernel, done)) return rc;
  kKernel<<<grid, threads, smem, stream>>>(args...);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

// The weights [taps][Cout][Cin] (fp16) as a 2-D tensor of taps * Cout rows of Cin channels, loaded in boxes of 64
// channels x nt rows under the 128-byte swizzle; channels >= Cin read as zero. TMA needs a 16-byte row pitch, which
// conv_shape_ok guarantees for fp16 (Cin % 8 == 0). cuTensorMapEncodeTiled is a driver API entry point; the library
// links only the runtime, so it is looked up once through cudaGetDriverEntryPoint.
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// A map depends only on (address, Cin, rows, nt), so the last kMapCache maps are kept and reused: a training step
// launches the same weights many times, and reuse keeps driver calls out of the launch path.
constexpr int kMapCache = 64;
struct MapEntry {
  const void* w;
  int cin, rows, nt;
  CUtensorMap map;
};

int halo_weight_map(CUtensorMap* map, const void* w, const ConvParams& p) {
  static std::mutex mu;
  static MapEntry cache[kMapCache];
  static int cached = 0, next = 0;
  const int rows = p.ksize * p.ksize * p.Cout;
  std::lock_guard<std::mutex> lock(mu);
  for (int i = 0; i < cached; ++i) {
    const MapEntry& e = cache[i];
    if (e.w == w && e.cin == p.Cin && e.rows == rows && e.nt == p.nt) {
      *map = e.map;
      return FPD_OK;
    }
  }
  static std::atomic<EncodeTiledFn> encode{nullptr};
  EncodeTiledFn fn = encode.load(std::memory_order_acquire);
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    FPD_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q));
    FPD_REQUIRE(q == cudaDriverEntryPointSuccess && f, "conv_halo: the driver has no cuTensorMapEncodeTiled");
    fn = reinterpret_cast<EncodeTiledFn>(f);
    encode.store(fn, std::memory_order_release);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)p.Cin, (cuuint64_t)p.ksize * p.ksize * p.Cout};
  const cuuint64_t pitch[1] = {(cuuint64_t)p.Cin * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)p.nt};
  const cuuint32_t elem_strides[2] = {1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(w), dims, pitch, box, elem_strides,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  FPD_REQUIRE(r == CUDA_SUCCESS, "conv_halo: cuTensorMapEncodeTiled failed (%d) for Cin=%d Cout=%d nt=%d", (int)r,
              p.Cin, p.Cout, p.nt);
  cache[next] = MapEntry{w, p.Cin, rows, p.nt, *map};
  next = (next + 1) % kMapCache;
  if (cached < kMapCache) ++cached;
  return FPD_OK;
}

// f(std::integral_constant<int, kN>{}) for an output slice of nt columns: the kN of every forward-convolution kernel.
template <typename F>
int with_slice(int nt, F&& f) {
  switch (nt) {
    case 16: return f(std::integral_constant<int, 16>{});
    case 32: return f(std::integral_constant<int, 32>{});
    case 48: return f(std::integral_constant<int, 48>{});
    case 64: return f(std::integral_constant<int, 64>{});
    case 80: return f(std::integral_constant<int, 80>{});
    case 96: return f(std::integral_constant<int, 96>{});
    case 112: return f(std::integral_constant<int, 112>{});
    case 128: return f(std::integral_constant<int, 128>{});
  }
  set_last_error("conv_wgmma: no kernel for a %d-column slice", nt);
  return FPD_ERR_UNSUPPORTED;
}

std::atomic<int> g_conv1x1{1};
std::atomic<int> g_conv_halo{1};

// The shape part of a launch's parameters, staged-kernel layout (passes 3: hi and lo tiles per stage).
ConvParams conv_shape_params(int B, int H, int W, int Cin, int Cout, int ksize, int f16, int passes) {
  ConvParams p{};
  p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.ksize = ksize; p.P = B * H * W;
  p.passes = passes;
  p.nt = conv_tc_ts_slice(Cout);
  p.n_tiles = Cout / p.nt;
  p.num_tiles = conv_num_tiles(B, H, W, Cout);
  p.ncb = (Cin + (f16 ? 63 : 31)) / (f16 ? 64 : 32);
  p.ksteps = ksize * ksize * p.ncb;
  p.b_tile_bytes = p.nt * 128;
  p.stage_bytes = (p.passes == 3 ? 2 : 1) * (kATileBytes + p.b_tile_bytes);
  return p;
}

// The forward-convolution kernels, numbered as conv_f16x1_kernel reports them.
enum ConvKernel { kConvNone = 0, kConvStaged = 1, kConvHalo = 2, kConvPw = 3 };

struct ConvPlan {
  int kernel;    // ConvKernel
  int grid;      // persistent CTAs; a launch with statistics writes one partial block per CTA
  size_t smem;
};

// Which kernel runs a forward convolution. p: conv_shape_params of the call (passes 3: hi and lo operands); the halo
// kernel's ring goes into p. kConvNone only where the staged kernel's shared memory does not fit.
//   3x3: the halo kernel (conv_halo_kernel, conv_halo_f16x1_kernel) wherever the halo (one copy per operand half), the
//   statistics scratch and a ring of weight stages with two mbarriers each fit: 3, else 2 stages with hi and lo
//   operands; 4, else 3 single-pass.
//   1x1: the weight-resident kernel (pw_conv_wgmma_kernel, pw_conv_f16x1_kernel) wherever the slice's weights, the A
//   stages and the statistics scratch fit; only the single-pass kernel carries statistics.
//   Everything else: the staged conv_wgmma_kernel.
// The halo and 1x1 kernels take the 3xFP16 calls (f16 with w_lo), under the fpd_set_conv_halo / fpd_set_conv1x1 toggles,
// and the single-pass calls (fpd_conv2d_tc_f16x1*), regardless of the toggles. TF32 calls and fpd_conv2d_tc_h's fp16
// calls without w_lo stay on the staged kernel.
ConvPlan conv_plan(ConvParams& p, bool f16, bool single_pass, bool stats, int num_sms) {
  const bool split = p.passes == 3;
  const bool fast = single_pass || (f16 && split);
  const int copies = split ? 2 : 1;
  const size_t stat_bytes = stats ? (size_t)8 * p.Cout * 2 * sizeof(double) : 0;
  ConvPlan pl{kConvStaged, p.num_tiles < num_sms ? p.num_tiles : num_sms, 0};
  if (fast && p.ksize == 3 && (single_pass || g_conv_halo.load(std::memory_order_relaxed))) {
    const int max_stages = split ? 3 : 4;
    ConvParams h = p;
    h.halo_rows = kTileM + 2 * p.W + 3;
    h.stage_bytes = copies * p.b_tile_bytes;
    for (int stages = max_stages; stages >= max_stages - 1; --stages) {
      h.halo_stages = stages;
      pl.smem = 1024 + (size_t)stages * h.stage_bytes + (size_t)copies * h.ncb * h.halo_rows * 128 + stat_bytes +
                (size_t)stages * 2 * 8;
      if (pl.smem <= (size_t)kSmemLimit) {
        p = h;
        pl.kernel = kConvHalo;
        return pl;
      }
    }
  }
  if (fast && p.ksize == 1 && (single_pass || (!stats && g_conv1x1.load(std::memory_order_relaxed)))) {
    pl.smem = pw_smem_bytes(split, p.ncb, p.nt) + stat_bytes;
    if (pl.smem <= (size_t)kSmemLimit) {
      pl.kernel = kConvPw;
      return pl;
    }
  }
  pl.smem = 1024 + (size_t)kStages * p.stage_bytes + stat_bytes;
  if (pl.smem > (size_t)kSmemLimit) pl.kernel = kConvNone;
  return pl;
}

template <typename T>
struct TypeTag {
  using type = T;
};

// f(TypeTag<TIn>{}, TypeTag<TOut>{}) for the activation types of a single-pass call (__half where the flag is set).
template <typename F>
int with_act_types(bool x_f16, bool y_f16, F&& f) {
  if (x_f16) return y_f16 ? f(TypeTag<__half>{}, TypeTag<__half>{}) : f(TypeTag<__half>{}, TypeTag<float>{});
  return y_f16 ? f(TypeTag<float>{}, TypeTag<__half>{}) : f(TypeTag<float>{}, TypeTag<float>{});
}

// Every forward convolution: checks the call, plans it and launches the planned kernel. w_lo == nullptr: hi operands
// only; single_pass: an fpd_conv2d_tc_f16x1* call. x_f16 / y_f16: x, or y and the residual, are __half (single-pass
// calls on the halo and 1x1 kernels without statistics only).
int conv_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift, int pre_relu,
                const void* w_hi, const void* w_lo, int f16, bool single_pass, const float* bias,
                const float* residual, const float* relu_mask, float* y, float out_scale, const float* in_scale, int B,
                int H, int W, int Cin, int Cout, int ksize, cudaStream_t stream, double* stat_part,
                const float* stat_pivot, bool x_f16 = false, bool y_f16 = false) {
  FPD_REQUIRE(x && w_hi && y, "conv_wgmma: null operand");
  FPD_REQUIRE((double)B * H * W * Cout < 4294967296.0, "conv_wgmma: output has 2^32 or more elements");
  FPD_REQUIRE((pre_scale == nullptr) == (pre_shift == nullptr), "conv_wgmma: pre_scale/pre_shift come in pairs");
  FPD_REQUIRE(pre_scale != nullptr || pre_mean == nullptr, "conv_wgmma: pre_mean needs pre_scale/pre_shift");
  FPD_REQUIRE(stat_part == nullptr || Cout <= kMaxStatCout, "conv_wgmma: statistics need Cout <= %d", kMaxStatCout);
  ConvParams p = conv_shape_params(B, H, W, Cin, Cout, ksize, f16, w_lo ? 3 : 1);
  const ConvPlan pl = conv_plan(p, f16, single_pass, stat_part != nullptr, device_sm_count());
  FPD_REQUIRE(pl.kernel != kConvNone, "conv_wgmma: shared memory plan %zu B too large", pl.smem);
  FPD_REQUIRE(!(x_f16 || y_f16) || (single_pass && !w_lo && !stat_part && (pl.kernel == kConvHalo || pl.kernel == kConvPw)),
              "conv_wgmma: half-precision activations need a single-pass halo or 1x1 launch without statistics");
  p.x = x; p.w_hi = w_hi; p.w_lo = w_lo;
  p.pre_mean = pre_mean; p.pre_scale = pre_scale; p.pre_shift = pre_shift; p.pre_relu = pre_relu;
  p.bias = bias; p.residual = residual; p.relu_mask = relu_mask; p.y = y;
  p.out_scale = f16 ? out_scale * (1.0f / (float)(1 << kF16WeightScaleLog2)) : out_scale;
  p.in_scale = in_scale;
  p.stat_part = stat_part; p.stat_pivot = stat_pivot;
  const bool split = p.passes == 3;
  CUtensorMap hi, lo;
  if (pl.kernel == kConvHalo) {
    if (int rc = halo_weight_map(&hi, w_hi, p)) return rc;
    if (split) {
      if (int rc = halo_weight_map(&lo, w_lo, p)) return rc;
    }
  }
  return with_slice(p.nt, [&](auto n) {
    constexpr int kN = decltype(n)::value;
    if (pl.kernel == kConvHalo && split) return launch<conv_halo_kernel<kN>>(pl.grid, kThreads, pl.smem, stream, p, hi, lo);
    if (pl.kernel == kConvPw && split) return launch<pw_conv_wgmma_kernel<kN>>(pl.grid, kThreads, pl.smem, stream, p);
    if (pl.kernel == kConvHalo || pl.kernel == kConvPw)
      return with_act_types(x_f16, y_f16, [&](auto ti, auto to) {
        using TIn = typename decltype(ti)::type;
        using TOut = typename decltype(to)::type;
        return pl.kernel == kConvHalo
                   ? launch<conv_halo_f16x1_kernel<kN, TIn, TOut>>(pl.grid, kThreads, pl.smem, stream, p, hi)
                   : launch<pw_conv_f16x1_kernel<kN, TIn, TOut>>(pl.grid, kThreads, pl.smem, stream, p);
      });
    return f16 ? launch<conv_wgmma_kernel<true, kN>>(pl.grid, kThreads, pl.smem, stream, p)
               : launch<conv_wgmma_kernel<false, kN>>(pl.grid, kThreads, pl.smem, stream, p);
  });
}

// The single-pass FP16 calls' shapes (also: statistics need Cout <= kMaxStatCout).
bool conv_f16x1_supported(int B, int H, int W, int Cin, int Cout, int ksize, bool stats) {
  return conv_shape_ok(Cin, Cout, ksize, 1, kMaxCinH, 2048) && B >= 1 && H >= 1 && W >= 1 &&
         (double)B * H * W * Cout < 4294967296.0 && (!stats || Cout <= kMaxStatCout);
}

// The checked 3xTF32 / 3xFP16 forward of fpd_conv2d_tc_h and fpd_conv2d_tc_h_stats.
int conv_tc_h_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                     int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                     const float* residual, const float* relu_mask, float* y, float out_scale, const float* in_scale,
                     int B, int H, int W, int Cin, int Cout, int ksize, cudaStream_t stream, double* stat_part,
                     const float* stat_pivot) {
  FPD_REQUIRE(fpd_conv2d_tc_h_supported(Cin, Cout, ksize, H, W, f16),
              "conv_tc_h: unsupported shape Cin=%d Cout=%d k=%d H=%d W=%d f16=%d", Cin, Cout, ksize, H, W, f16);
  return conv_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, f16, false, bias, residual, relu_mask,
                     y, out_scale, in_scale, B, H, W, Cin, Cout, ksize, stream, stat_part, stat_pivot);
}

// The kernel (ConvKernel) a single-pass call with (stats != 0) or without statistics runs on, and in *stat_blocks
// (nullable) the partial blocks a statistics launch writes: 0 without statistics or when unsupported.
int conv_f16x1_kernel(int B, int H, int W, int Cin, int Cout, int ksize, int stats, int num_sms, int* stat_blocks) {
  if (stat_blocks) *stat_blocks = 0;
  if (!conv_f16x1_supported(B, H, W, Cin, Cout, ksize, stats != 0)) return 0;
  ConvParams p = conv_shape_params(B, H, W, Cin, Cout, ksize, 1, 1);
  const ConvPlan pl = conv_plan(p, true, true, stats != 0, num_sms);
  if (pl.kernel != kConvNone && stats && stat_blocks) *stat_blocks = pl.grid;
  return pl.kernel;
}

// The checked single-pass FP16 forward of fpd_conv2d_tc_f16x1 and fpd_conv2d_tc_f16x1_train.
int conv_f16x1_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                      int pre_relu, const void* w, const float* bias, const float* residual, const float* relu_mask,
                      float* y, float out_scale, const float* in_scale, int B, int H, int W, int Cin, int Cout,
                      int ksize, cudaStream_t stream, double* stat_part, const float* stat_pivot) {
  FPD_REQUIRE(conv_f16x1_supported(B, H, W, Cin, Cout, ksize, stat_part != nullptr),
              "conv_f16x1: unsupported shape B=%d H=%d W=%d Cin=%d Cout=%d k=%d (statistics: %d, Cout <= %d)", B, H,
              W, Cin, Cout, ksize, stat_part != nullptr, kMaxStatCout);
  return conv_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w, nullptr, 1, true, bias, residual, relu_mask, y,
                     out_scale, in_scale, B, H, W, Cin, Cout, ksize, stream, stat_part, stat_pivot);
}

// ================================================= weight gradient =================================================

constexpr int kKp = 32;   // pixels (K) per pipeline stage: one 128-byte tf32 operand row

struct WgradParams {
  int B, H, W, Cin, Cout, ksize, taps, P, passes;
  int co_tiles, ci_tiles, num_kt, kt_per_split;
  int b_tile_bytes, stage_bytes;
  const float* x;
  const float* dy;
  const float* pre_mean;
  const float* pre_scale;
  const float* pre_shift;
  int pre_relu;
  float* partial;   // [split][tap][Cout][Cin]
  // wgrad_halo_kernel only
  int h_ci, h_co_tiles, h_ci_tiles, h_rows, h_halo, h_win, h_xstride, h_stage_bytes;
};

template <int kN>
__global__ void __launch_bounds__(kThreads, 1) wgrad_wgmma_kernel(const WgradParams p) {
  constexpr int kGq = kTileM / 4 / 8;   // dY channel-quad groups per warp and stage (4)
  constexpr int kXq = kN / 4 / 8;       // x channel-quad groups per warp and stage (1, 2 or 4)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t smem_a = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const bool split = p.passes == 3;
  int bid = blockIdx.x;
  const int ct = bid % p.co_tiles; bid /= p.co_tiles;
  const int it = bid % p.ci_tiles; bid /= p.ci_tiles;
  const int tap = bid % p.taps;
  const int sp = bid / p.taps;
  const int co0 = ct * kTileM, ci0 = it * kN;
  const int dh = p.ksize == 3 ? tap / 3 - 1 : 0, dw = p.ksize == 3 ? tap % 3 - 1 : 0;
  const int kt0 = sp * p.kt_per_split, kt1 = min(kt0 + p.kt_per_split, p.num_kt);
  const uint32_t a_lo_off = split ? (uint32_t)kATileBytes : 0u;
  const uint32_t b_off = (split ? 2u : 1u) * (uint32_t)kATileBytes;
  const uint32_t b_lo_off = split ? (uint32_t)p.b_tile_bytes : 0u;
  const int HW = p.H * p.W;

  // loads: a warp covers 8 pixels x 4 channel quads per instruction (64 contiguous bytes per pixel in global memory);
  // group q of warp w: pixels 8 (q & 3) + (lane & 7), quad 4 (q >> 2) + (lane >> 3)
  float4 rg[kGq], rx[kXq];
  uint32_t okg = 0, okx = 0;
  auto pix_of = [&](int q) { return ((q & 3) << 3) + (lane & 7); };
  auto quad_of = [&](int q) { return ((q >> 2) << 2) + (lane >> 3); };
  auto load = [&](int kt) {
    okg = okx = 0;
#pragma unroll
    for (int u = 0; u < kGq; ++u) {
      const int q = warp * kGq + u;
      const int m = kt * kKp + pix_of(q), co = co0 + 4 * quad_of(q);
      rg[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < p.P && co < p.Cout) {
        okg |= 1u << u;
        rg[u] = __ldg(reinterpret_cast<const float4*>(p.dy + (size_t)m * p.Cout + co));
      }
    }
#pragma unroll
    for (int u = 0; u < kXq; ++u) {
      const int q = warp * kXq + u;
      const int m = kt * kKp + pix_of(q), ci = ci0 + 4 * quad_of(q);
      rx[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < p.P && ci < p.Cin) {
        const int n = m / HW, hh = (m % HW) / p.W + dh, ww = m % p.W + dw;
        if (hh >= 0 && hh < p.H && ww >= 0 && ww < p.W) {
          okx |= 1u << u;
          rx[u] = __ldg(reinterpret_cast<const float4*>(p.x + (((size_t)n * p.H + hh) * p.W + ww) * p.Cin + ci));
        }
      }
    }
  };
  // transposed store: element (channel row ch, pixel k) of a K-major tile with 128-byte rows under the 128-byte swizzle
  auto put4 = [&](uint32_t base, int ch, int k, float4 v, uint32_t lo_off) {
    float4 h, l;
    split_tf32x4(v, h, l);
    const float hv[4] = {h.x, h.y, h.z, h.w}, lv[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = ch + e;
      const uint32_t a = base + (uint32_t)c * 128u + ((uint32_t)((k >> 2) ^ (c & 7)) << 4) + (uint32_t)(k & 3) * 4u;
      sts32(a, hv[e]);
      if (split) sts32(a + lo_off, lv[e]);
    }
  };
  auto store = [&](uint32_t st) {
#pragma unroll
    for (int u = 0; u < kGq; ++u) {
      const int q = warp * kGq + u;
      put4(st, 4 * quad_of(q), pix_of(q), rg[u], a_lo_off);
    }
#pragma unroll
    for (int u = 0; u < kXq; ++u) {
      const int q = warp * kXq + u;
      const int ci = ci0 + 4 * quad_of(q);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (okx & (1u << u)) v = affine_relu4(rx[u], p.pre_mean, p.pre_scale, p.pre_shift, ci, p.pre_relu);
      put4(st + b_off, 4 * quad_of(q), pix_of(q), v, b_lo_off);
    }
  };

  float acc[kN / 2], part[kN / 2], part_x[kN / 2];
  zero_acc(acc);
  zero_acc(part);
  zero_acc(part_x);
  if (kt0 < kt1) load(kt0);
  for (int kt = kt0; kt < kt1; ++kt) {
    const uint32_t st = smem_a + (uint32_t)(((kt - kt0) % kStages) * p.stage_bytes);
    store(st);   // overlaps the MMAs of step kt - 1
    if (kt > kt0) {
      wgmma_wait<0>();
      add_part(acc, part, part_x);
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (kt + 1 < kt1) load(kt + 1);
    wgmma_fence();
    const uint32_t a_hi = st + (uint32_t)wg * 64u * 128u;
    mma_row<false, kN, true>(part, part_x, a_hi, a_hi + a_lo_off, st + b_off, st + b_off + b_lo_off, split);
    wgmma_commit();
  }
  wgmma_wait<0>();
  if (kt1 > kt0) add_part(acc, part, part_x);

  const int g = lane >> 2, t = lane & 3;
  float* out = p.partial + ((size_t)sp * p.taps + tap) * p.Cout * p.Cin;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int co = co0 + wg * 64 + (warp & 3) * 16 + g + rr * 8;
    if (co >= p.Cout) continue;
#pragma unroll
    for (int i = 0; i < kN / 8; ++i) {
      const int ci = ci0 + i * 8 + 2 * t;
      if (ci < p.Cin)
        *reinterpret_cast<float2*>(out + (size_t)co * p.Cin + ci) = make_float2(acc[4 * i + 2 * rr], acc[4 * i + 2 * rr + 1]);
    }
  }
}

// ============================================ weight gradient, tap rows ============================================
// wgrad_halo_kernel: the weight gradient of wgrad_wgmma_kernel with the roles of the operands swapped, so that M is
// filled for every Cout, and with one staged pixel step serving every tap of a kernel row. Same plan (splits,
// kt_per_split, K steps of 32 pixels, partial layout), and per output element the same chain: per K step the same
// hi / lo values, per k8 dY_lo x_hi then dY_hi x_lo into `part_x` and dY_hi x_hi into `part` (the products are the
// same numbers as wgrad_wgmma_kernel's, A and B only trade places), then acc += part + part_x.
//   GEMM: M = (tap, input channel) rows, 64 per warpgroup, one tap and 16 channels per warp; N = a kN-wide slice of the
//   output channels; one CTA = one split x one row of the 3x3 kernel (three taps; the 1x1 tap alone) x one input-channel
//   tile of h_ci (<= 64) x one output slice. With h_ci = 32 two taps share a warpgroup; rows past the CTA's last tap
//   (the fourth warpgroup half at h_ci = 32) compute a duplicate and are not written.
//   Per K step (pixels p0 .. p0 + 31) the CTA stages, double-buffered:
//     - dY as the B operand: kN K-major rows of 128 bytes under the 128-byte swizzle, hi and lo. Each thread loads 4
//       pixels x 4 channels, transposes them in registers and writes one 16-byte chunk per channel row (8 consecutive
//       threads write 8 chunks of one row: conflict-free).
//     - x after the BN affine + ReLU, fp32, in its natural [pixel][channel] layout: the h_win = 32 + 2 h_halo
//       flattened pixels p0 + dh W - h_halo .. of the kernel row dh, rows padded to h_xstride = h_ci + 8 floats so that
//       the four k columns of a fragment load fall in distinct banks.
//     - one word per pixel of the step: bit j set if tap j of the row reads a pixel inside the image (and p < P).
//   Every lane then reads its A fragment for its tap from the shifted rows (zero where the mask bit is clear, the rule
//   of wgrad_wgmma_kernel's loads), splits hi / lo in registers and issues the MMAs from registers.
//   Stage s % 2 is rewritten at step s after the step s - 1 barrier, which follows every warpgroup's wgmma_wait<0> for
//   step s - 2 (the last reader of that stage); the next step's global loads are in flight during the MMAs.
constexpr int kWhMaxThreads = 384;
constexpr int kWhXChunks = 4;   // staged x float4 chunks per thread and step, at most

template <int kN, bool kSplit>
__global__ void __launch_bounds__(kWhMaxThreads, 1) wgrad_halo_kernel(const WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t smem_s = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nthr = blockDim.x;
  int bid = blockIdx.x;
  const int ct = bid % p.h_co_tiles; bid /= p.h_co_tiles;
  const int it = bid % p.h_ci_tiles; bid /= p.h_ci_tiles;
  const int trow = bid % p.h_rows;
  const int sp = bid / p.h_rows;
  const int co0 = ct * kN, ci0 = it * p.h_ci;
  const int row_taps = p.ksize == 3 ? 3 : 1;
  const int dh = p.ksize == 3 ? trow - 1 : 0;
  const int kt0 = sp * p.kt_per_split, kt1 = min(kt0 + p.kt_per_split, p.num_kt);
  const uint32_t dy_lo_off = (uint32_t)kN * 128u;
  const uint32_t x_off = 2u * dy_lo_off;
  const uint32_t mask_off = x_off + (uint32_t)(p.h_win * p.h_xstride) * 4u;
  const int HW = p.H * p.W;

  // this warp's 16 rows: tap tl of the row, input channels cb .. cb + 15 of the tile
  const int r0 = warp * 16;
  int tl = r0 / p.h_ci;
  const bool active = tl < row_taps;
  if (!active) tl = row_taps - 1;
  const int cb = r0 % p.h_ci;
  const int tap = trow * row_taps + tl;
  const int dw = p.ksize == 3 ? tl - 1 : 0;
  const int g = lane >> 2, t = lane & 3;

  // loads, one step ahead: dY item (pixel quad dq, channel quad dc) into registers for threads < 2 kN; the raw x window
  // by cp.async straight into the stage; the tap mask
  const int dq = tid & 7, dc = tid >> 3;
  const bool dy_thread = tid < 2 * kN;
  const int xq = p.h_ci / 4;                 // float4 chunks per staged pixel
  const int x_items = p.h_win * xq;
  const uint32_t dy_raw = mask_off + kKp * 4u + (uint32_t)((4 * dq * kN + 4 * dc) * 4);   // this thread's raw dY
  uint32_t mbits = 0;
  auto load = [&](int kt, uint32_t st) {
    if (dy_thread) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int m = kt * kKp + 4 * dq + r;
        cp_async16(st + dy_raw + (uint32_t)(r * kN * 4), p.dy + (size_t)(m < p.P ? m : 0) * p.Cout + co0 + 4 * dc,
                   m < p.P);
      }
    }
    const int qs = kt * kKp + dh * p.W - p.h_halo;
#pragma unroll
    for (int u = 0; u < kWhXChunks; ++u) {
      const int idx = tid + u * nthr;
      if (idx >= x_items) break;
      const int j = idx / xq, c = (idx - j * xq) * 4;
      const int q = qs + j;
      const bool ok = q >= 0 && q < p.P;   // rows outside [0, P) are never read unmasked: zero-filled
      cp_async16(st + x_off + (uint32_t)(j * p.h_xstride + c) * 4u, p.x + (size_t)(ok ? q : 0) * p.Cin + ci0 + c, ok);
    }
    cp_async_commit();
    if (tid < kKp) {
      const int m = kt * kKp + tid;
      mbits = 0;
      if (m < p.P) {
        const int hh = (m % HW) / p.W + dh, w0 = m % p.W;
        if (hh >= 0 && hh < p.H) {
          for (int k = 0; k < row_taps; ++k) {
            const int ww = w0 + (p.ksize == 3 ? k - 1 : 0);
            if (ww >= 0 && ww < p.W) mbits |= 1u << k;
          }
        }
      }
    }
  };
  auto store = [&](uint32_t st) {   // after cp_async_wait_all: this thread's own raw dY copies have landed
    if (dy_thread) {
      float v[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(v[r][0]), "=f"(v[r][1]), "=f"(v[r][2]), "=f"(v[r][3])
                     : "r"(st + dy_raw + (uint32_t)(r * kN * 4))
                     : "memory");
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = 4 * dc + e;   // output channel co0 + row, pixels 4 dq .. 4 dq + 3
        float4 h, l;
        split_tf32x4(make_float4(v[0][e], v[1][e], v[2][e], v[3][e]), h, l);
        const uint32_t a = st + (uint32_t)row * 128u + ((uint32_t)(dq ^ (row & 7)) << 4);
        sts128u(a, make_uint4(__float_as_uint(h.x), __float_as_uint(h.y), __float_as_uint(h.z), __float_as_uint(h.w)));
        if (kSplit)
          sts128u(a + dy_lo_off,
                  make_uint4(__float_as_uint(l.x), __float_as_uint(l.y), __float_as_uint(l.z), __float_as_uint(l.w)));
      }
    }
    if (tid < kKp) asm volatile("st.shared.u32 [%0], %1;" ::"r"(st + mask_off + (uint32_t)tid * 4u), "r"(mbits) : "memory");
  };

  float acc[kN / 2], part[kN / 2], part_x[kN / 2];
  zero_acc(acc);
  zero_acc(part);
  zero_acc(part_x);
  if (kt0 < kt1) load(kt0, smem_s);
  for (int kt = kt0; kt < kt1; ++kt) {
    const uint32_t st = smem_s + (uint32_t)(((kt - kt0) & 1) * p.h_stage_bytes);
    cp_async_wait_all();
    store(st);   // overlaps the MMAs of step kt - 1
    if (kt > kt0) {
      wgmma_wait<0>();
      add_part(acc, part, part_x);
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (kt + 1 < kt1) load(kt + 1, smem_s + (uint32_t)(((kt + 1 - kt0) & 1) * p.h_stage_bytes));
    // A fragments: k = 8 kk + t (+ 4), rows cb + g (+ 8); pixel k of the step reads staged row k + dw + h_halo
    // the BN affine of this lane's two fragment channels, affine_relu4's expression applied per element
    const int c_lane = ci0 + cb + g;
    float mu[2] = {0.f, 0.f}, sc[2] = {1.f, 1.f}, sh[2] = {0.f, 0.f};
    if (p.pre_scale) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        mu[hr] = p.pre_mean ? __ldg(p.pre_mean + c_lane + 8 * hr) : 0.f;
        sc[hr] = __ldg(p.pre_scale + c_lane + 8 * hr);
        sh[hr] = __ldg(p.pre_shift + c_lane + 8 * hr);
      }
    }
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int hk = 0; hk < 2; ++hk) {
        const int k = 8 * kk + t + 4 * hk;
        uint32_t mk;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(mk) : "r"(st + mask_off + (uint32_t)k * 4u));
        const bool ok = (mk >> tl) & 1u;
        const uint32_t src = st + x_off + (uint32_t)((k + dw + p.h_halo) * p.h_xstride + cb + g) * 4u;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          float v;
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(src + (uint32_t)hr * 32u));
          if (p.pre_scale) v = fmaf(v - mu[hr], sc[hr], sh[hr]);
          if (p.pre_relu) v = fmaxf(v, 0.f);
          if (!ok) v = 0.f;
          float h, l;
          split_tf32_fast(v, h, l);
          // volatile moves keep the fragment writes ahead of wgmma_fence (no warpgroup.arrive between the MMAs)
          asm volatile("mov.b32 %0, %1;" : "=r"(ah[kk][2 * hk + hr]) : "r"(__float_as_uint(h)));
          asm volatile("mov.b32 %0, %1;" : "=r"(al[kk][2 * hk + hr]) : "r"(__float_as_uint(l)));
        }
      }
    }
    wgmma_fence();
    const uint64_t dbh = gmma_desc_sw128(st), dbl = gmma_desc_sw128(st + dy_lo_off);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint64_t o = (uint64_t)(kk * 2);
      const int accum = kk > 0 ? 1 : 0;
      if (kSplit) {
        WgmmaRATf32<kN>::mma(part_x, ah[kk], dbl + o, accum);   // dY_lo x_hi
        WgmmaRATf32<kN>::mma(part_x, al[kk], dbh + o, 1);       // dY_hi x_lo
      }
      WgmmaRATf32<kN>::mma(part, ah[kk], dbh + o, accum);
    }
    wgmma_commit();
  }
  wgmma_wait<0>();
  if (kt1 > kt0) add_part(acc, part, part_x);

  if (!active) return;
  float* out = p.partial + ((size_t)sp * p.taps + tap) * p.Cout * p.Cin;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int ci = ci0 + cb + g + rr * 8;
#pragma unroll
    for (int i = 0; i < kN / 8; ++i) {
      const int co = co0 + i * 8 + 2 * t;
      out[(size_t)co * p.Cin + ci] = acc[4 * i + 2 * rr];
      out[(size_t)(co + 1) * p.Cin + ci] = acc[4 * i + 2 * rr + 1];
    }
  }
}

// dw[co][ci][tap] = scale * sum_splits partial[split][tap][co][ci]
// Block = 32 consecutive partial elements (coalesced along ci) x 8 split groups: every thread sums splits sg, sg+8, ...
// and the eight group sums are added in a fixed order (deterministic).
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dw, float scale, int Cin, int Cout, int taps,
                    int splits) {
  __shared__ float red[8][32];
  const int64_t total = (int64_t)taps * Cin * Cout;
  const int lane = threadIdx.x & 31, sg = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * 32 + lane;   // index into [tap][co][ci]
  float acc = 0.f;
  if (i < total) {
#pragma unroll 4
    for (int s = sg; s < splits; s += 8) acc += partial[(size_t)s * total + i];
  }
  red[sg][lane] = acc;
  __syncthreads();
  if (sg != 0 || i >= total) return;
  float t = red[0][lane];
#pragma unroll
  for (int k = 1; k < 8; ++k) t += red[k][lane];
  const int ci = (int)(i % Cin);
  const int co = (int)((i / Cin) % Cout);
  const int tap = (int)(i / ((int64_t)Cout * Cin));
  dw[((size_t)co * Cin + ci) * taps + tap] = t * scale;
}

int wgrad_n(int Cin) { return Cin <= 32 ? 32 : Cin <= 64 ? 64 : 128; }

struct WgradPlan {
  int n, co_tiles, ci_tiles, taps, num_kt, splits, kt_per_split;
};

WgradPlan wgrad_plan(int B, int H, int W, int Cin, int Cout, int ksize, int num_sms) {
  WgradPlan pl{};
  pl.n = wgrad_n(Cin);
  pl.co_tiles = (Cout + kTileM - 1) / kTileM;
  pl.ci_tiles = (Cin + pl.n - 1) / pl.n;
  pl.taps = ksize * ksize;
  pl.num_kt = (int)(((long long)B * H * W + kKp - 1) / kKp);
  const int per_split = pl.co_tiles * pl.ci_tiles * pl.taps;
  int s = (2 * num_sms + per_split - 1) / per_split;   // about two CTAs per SM
  if (s < 1) s = 1;
  if (s > pl.num_kt) s = pl.num_kt;
  pl.kt_per_split = (pl.num_kt + s - 1) / s;
  pl.splits = (pl.num_kt + pl.kt_per_split - 1) / pl.kt_per_split;   // every split gets at least one K step
  return pl;
}

std::atomic<int> g_wgrad_halo{1};

// wgrad_halo_kernel takes every 3x3 shape of fpd_conv2d_wgrad_tc_supported, and the 1x1 shapes whose input channels
// fill whole 64-row warpgroups and whose Cout is 32 or 64, where wgrad_wgmma_kernel's 128-row tile is at most half
// used. (At Cout >= 128 that tile is full, and the per-tap kernel was faster on the H100: 128 -> 128 at 64x64, batch
// 32, 128.5 against 151.9 µs.)
bool wgrad_halo_ok(int Cin, int Cout, int ksize) {
  if (!g_wgrad_halo.load(std::memory_order_relaxed)) return false;
  if (ksize == 3) return true;
  return Cin % 64 == 0 && (Cout == 32 || Cout == 64);
}

// The tap-row kernel for a plan of wgrad_plan (the splits are the plan's; only the CTA decomposition differs).
int wgrad_halo_launch(WgradParams p, const WgradPlan& pl, cudaStream_t stream) {
  const int n = p.Cout % 64 == 0 ? 64 : 32;
  p.h_ci = p.Cin < 64 ? p.Cin : 64;
  p.h_co_tiles = p.Cout / n;
  p.h_ci_tiles = p.Cin / p.h_ci;
  p.h_rows = p.ksize == 3 ? 3 : 1;
  p.h_halo = p.ksize == 3 ? 1 : 0;
  p.h_win = kKp + 2 * p.h_halo;
  p.h_xstride = p.h_ci + 8;
  const int row_taps = p.ksize == 3 ? 3 : 1;
  const int threads = (row_taps * p.h_ci + 63) / 64 * 128;
  // dY hi / lo tiles, the x window, the tap mask, raw dY
  const size_t stage = 2 * (size_t)n * 128 + (size_t)p.h_win * p.h_xstride * 4 + kKp * 4 + (size_t)kKp * n * 4;
  p.h_stage_bytes = (int)((stage + 1023) / 1024 * 1024);
  FPD_REQUIRE(threads <= kWhMaxThreads && p.h_win * (p.h_ci / 4) <= kWhXChunks * threads,
              "wgrad_halo: no plan for Cin=%d k=%d", p.Cin, p.ksize);
  const size_t smem = 1024 + 2 * (size_t)p.h_stage_bytes;
  const int grid = pl.splits * p.h_rows * p.h_ci_tiles * p.h_co_tiles;
  if (p.passes == 3)
    return n == 64 ? launch<wgrad_halo_kernel<64, true>>(grid, threads, smem, stream, p)
                   : launch<wgrad_halo_kernel<32, true>>(grid, threads, smem, stream, p);
  return n == 64 ? launch<wgrad_halo_kernel<64, false>>(grid, threads, smem, stream, p)
                 : launch<wgrad_halo_kernel<32, false>>(grid, threads, smem, stream, p);
}

}  // namespace
}  // namespace fpd

using namespace fpd;

extern "C" {

// ------------------------------------------------- forward entry points -------------------------------------------------

int fpd_conv2d_tc_ts_supported(int Cin, int Cout, int ksize) {
  return conv_shape_ok(Cin, Cout, ksize, 0, kMaxCinTs, 1024);
}

int fpd_conv2d_tc_ts(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                     int pre_relu, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                     const float* relu_mask, float* y, float out_scale, int B, int H, int W, int Cin, int Cout,
                     int ksize, fpd_stream_t stream) {
  FPD_REQUIRE(fpd_conv2d_tc_ts_supported(Cin, Cout, ksize), "conv_tc_ts: unsupported shape Cin=%d Cout=%d k=%d", Cin,
              Cout, ksize);
  return conv_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, 0, false, bias, residual, relu_mask, y,
                     out_scale, nullptr, B, H, W, Cin, Cout, ksize, stream, nullptr, nullptr);
}

int fpd_set_conv1x1(int enabled) { return g_conv1x1.exchange(enabled ? 1 : 0); }
int fpd_set_conv_halo(int enabled) { return g_conv_halo.exchange(enabled ? 1 : 0); }

int fpd_conv2d_tc_h_supported(int Cin, int Cout, int ksize, int H, int W, int f16) {
  (void)H; (void)W;
  return conv_shape_ok(Cin, Cout, ksize, f16, kMaxCinH, 2048);
}

int fpd_conv2d_tc_h_stats_blocks(int B, int H, int W, int Cin, int Cout, int ksize, int f16) {
  if (!fpd_conv2d_tc_h_supported(Cin, Cout, ksize, H, W, f16) || Cout > kMaxStatCout) return 0;
  ConvParams p = conv_shape_params(B, H, W, Cin, Cout, ksize, f16, 3);   // the grid is the same with hi operands only
  const ConvPlan pl = conv_plan(p, f16, false, true, device_sm_count());
  return pl.kernel != kConvNone ? pl.grid : 0;
}

int fpd_conv2d_tc_h(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                    int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                    const float* residual, const float* relu_mask, float* y, float out_scale, const float* in_scale,
                    int B, int H, int W, int Cin, int Cout, int ksize, fpd_stream_t stream) {
  return conv_tc_h_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, f16, bias, residual, relu_mask, y,
                          out_scale, in_scale, B, H, W, Cin, Cout, ksize, stream, nullptr, nullptr);
}

int fpd_conv2d_tc_h_stats(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                          int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                          const float* residual, float* y, float out_scale, int B, int H, int W, int Cin, int Cout,
                          int ksize, double* stat_part, const float* stat_pivot, fpd_stream_t stream) {
  FPD_REQUIRE(stat_part != nullptr, "fpd_conv2d_tc_h_stats: stat_part is NULL (use fpd_conv2d_tc_h)");
  return conv_tc_h_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, f16, bias, residual, nullptr, y,
                          out_scale, nullptr, B, H, W, Cin, Cout, ksize, stream, stat_part, stat_pivot);
}

int fpd_conv2d_tc_f16x1_kernel(int B, int H, int W, int Cin, int Cout, int ksize) {
  return conv_f16x1_kernel(B, H, W, Cin, Cout, ksize, 0, 0, nullptr);
}

int fpd_conv2d_tc_f16x1_train_plan(int B, int H, int W, int Cin, int Cout, int ksize, int stats, int* stat_blocks) {
  return conv_f16x1_kernel(B, H, W, Cin, Cout, ksize, stats, device_sm_count(), stat_blocks);
}

int fpd_conv2d_tc_f16x1(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                        int pre_relu, const void* w, const float* bias, const float* residual, const float* relu_mask,
                        float* y, float out_scale, int B, int H, int W, int Cin, int Cout, int ksize,
                        fpd_stream_t stream) {
  return conv_f16x1_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w, bias, residual, relu_mask, y, out_scale,
                           nullptr, B, H, W, Cin, Cout, ksize, stream, nullptr, nullptr);
}

int fpd_conv2d_tc_f16x1_train(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                              int pre_relu, const void* w, const float* bias, const float* residual,
                              const float* relu_mask, float* y, float out_scale, const float* in_scale, int B, int H,
                              int W, int Cin, int Cout, int ksize, double* stat_part, const float* stat_pivot,
                              fpd_stream_t stream) {
  return conv_f16x1_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w, bias, residual, relu_mask, y, out_scale,
                           in_scale, B, H, W, Cin, Cout, ksize, stream, stat_part, stat_pivot);
}

int fpd_conv2d_tc_f16x1_io(const void* x, int x_f16, const float* pre_mean, const float* pre_scale,
                           const float* pre_shift, int pre_relu, const void* w, const float* bias, const void* residual,
                           void* y, int y_f16, float out_scale, int B, int H, int W, int Cin, int Cout, int ksize,
                           fpd_stream_t stream) {
  FPD_REQUIRE(conv_f16x1_supported(B, H, W, Cin, Cout, ksize, false),
              "conv_f16x1_io: unsupported shape B=%d H=%d W=%d Cin=%d Cout=%d k=%d", B, H, W, Cin, Cout, ksize);
  const int kind = fpd_conv2d_tc_f16x1_kernel(B, H, W, Cin, Cout, ksize);
  if (kind != kConvHalo && kind != kConvPw) {
    set_last_error("conv_f16x1_io: B=%d H=%d W=%d Cin=%d Cout=%d k=%d runs on the staged kernel, which has no "
                   "half-precision activation form", B, H, W, Cin, Cout, ksize);
    return FPD_ERR_UNSUPPORTED;
  }
  return conv_launch(static_cast<const float*>(x), pre_mean, pre_scale, pre_shift, pre_relu, w, nullptr, 1, true, bias,
                     static_cast<const float*>(residual), nullptr, static_cast<float*>(y), out_scale, nullptr, B, H, W,
                     Cin, Cout, ksize, stream, nullptr, nullptr, x_f16 != 0, y_f16 != 0);
}

// ---------------------------------------------- weight-gradient entry points ----------------------------------------------

// Shapes taken per launch: 3x3 with Cin in {32, 64, 128} and Cout a multiple of 32 up to 256; 1x1 with Cin <= 256 and
// any Cout % 4 == 0. Wider layers go through ops.conv2d_wgrad_tc_chunked in channel chunks of these sizes, which keeps
// the per-launch partial-sum workspace (splits x taps x Cin x Cout) small.
int fpd_conv2d_wgrad_tc_supported(int Cin, int Cout, int ksize) {
  if (ksize == 3) return (Cin == 32 || Cin == 64 || Cin == 128) && Cout % 32 == 0 && Cout >= 32 && Cout <= 256;
  return ksize == 1 && Cout % 4 == 0 && Cin % 4 == 0 && Cin >= 4 && Cin <= 256;
}

int fpd_set_wgrad_halo(int enabled) { return g_wgrad_halo.exchange(enabled ? 1 : 0); }

int fpd_conv2d_wgrad_tc3_supported(int H, int W, int Cin, int Cout, int ksize) {
  (void)H; (void)W;
  return ksize == 3 && fpd_conv2d_wgrad_tc_supported(Cin, Cout, ksize);
}

size_t fpd_conv2d_wgrad_tc_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize) {
  if (!fpd_conv2d_wgrad_tc_supported(Cin, Cout, ksize)) return 0;
  const WgradPlan pl = wgrad_plan(B, H, W, Cin, Cout, ksize, device_sm_count());
  return (size_t)pl.splits * pl.taps * Cin * Cout * sizeof(float);
}

int fpd_conv2d_wgrad_tc_fused(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                              int pre_relu, const float* dy, int passes, float* dw_oihw, float scale, int B, int H,
                              int W, int Cin, int Cout, int ksize, void* workspace, size_t workspace_bytes,
                              fpd_stream_t stream) {
  FPD_REQUIRE(fpd_conv2d_wgrad_tc_supported(Cin, Cout, ksize), "wgrad_tc: unsupported shape Cin=%d Cout=%d k=%d", Cin,
              Cout, ksize);
  FPD_REQUIRE(x && dy && dw_oihw, "wgrad_tc: null operand");
  FPD_REQUIRE(passes == 1 || passes == 3, "wgrad_tc_fused: passes must be 1 or 3");
  FPD_REQUIRE((pre_scale == nullptr) == (pre_shift == nullptr), "wgrad_tc_fused: pre_scale/pre_shift come in pairs");
  const WgradPlan pl = wgrad_plan(B, H, W, Cin, Cout, ksize, device_sm_count());
  WgradParams p{};
  p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.ksize = ksize; p.taps = pl.taps; p.P = B * H * W;
  p.passes = passes;
  p.co_tiles = pl.co_tiles; p.ci_tiles = pl.ci_tiles; p.num_kt = pl.num_kt; p.kt_per_split = pl.kt_per_split;
  p.b_tile_bytes = pl.n * 128;
  p.stage_bytes = (passes == 3 ? 2 : 1) * (kATileBytes + p.b_tile_bytes);
  p.x = x; p.dy = dy;
  p.pre_mean = pre_mean; p.pre_scale = pre_scale; p.pre_shift = pre_shift; p.pre_relu = pre_relu;
  const size_t need = (size_t)pl.splits * pl.taps * Cin * Cout * sizeof(float);
  FPD_REQUIRE(workspace && workspace_bytes >= need, "wgrad_tc: workspace too small (%zu < %zu)", workspace_bytes, need);
  p.partial = (float*)workspace;
  const size_t smem = 1024 + (size_t)kStages * p.stage_bytes;
  const int grid = pl.splits * pl.taps * pl.co_tiles * pl.ci_tiles;
  int rc = wgrad_halo_ok(Cin, Cout, ksize) ? wgrad_halo_launch(p, pl, stream)
         : pl.n == 32 ? launch<wgrad_wgmma_kernel<32>>(grid, kThreads, smem, stream, p)
         : pl.n == 64 ? launch<wgrad_wgmma_kernel<64>>(grid, kThreads, smem, stream, p)
                      : launch<wgrad_wgmma_kernel<128>>(grid, kThreads, smem, stream, p);
  if (rc) return rc;
  const int64_t total = (int64_t)pl.taps * Cin * Cout;
  wgrad_reduce_kernel<<<(int)((total + 31) / 32), 256, 0, stream>>>(p.partial, dw_oihw, scale, Cin, Cout, pl.taps,
                                                                    pl.splits);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // extern "C"
