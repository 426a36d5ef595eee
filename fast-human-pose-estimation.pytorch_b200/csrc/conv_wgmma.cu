// conv_wgmma.cu -- implicit-GEMM convolution and convolution weight gradient on the sm_90a warpgroup tensor cores
// (wgmma.mma_async), operand preparation fused in.
//
// Forward (conv_tc_ts_* and conv_tc_h_*): y = conv(relu?((x - mean) * scale + shift)) (+ bias, + residual, ReLU mask),
// stride 1, "same" padding, NHWC activations, weights [tap][Cout][Cin] as hi/lo pairs (3xTF32: fp32 containers from
// weight_prep; 3xFP16: __half from weight_prep_f16, pre-scaled by 2^kF16WeightScaleLog2). BatchNorm2d-apply + ReLU +
// Conv2d of lib/models/hourglass.py:34-44: padding positions are zero AFTER the affine.
//   GEMM: M = 128 output pixels (two warpgroups x 64 rows), N = one Cout slice (<= 128), K = taps x Cin in steps of one
//   128-byte operand row (32 tf32 or 64 fp16 channels of one tap). Every thread loads its share of the raw x rows into
//   registers one K step ahead, applies the affine + ReLU + hi/lo split and stores the result into the swizzled
//   K-major A tile; the weight tiles arrive by cp.async. Three pipeline stages: a stage is rewritten only after every
//   warpgroup has retired the wgmma group that read it (wait_group<0> + the per-step CTA barrier); each step's
//   products are summed into the fp32 accumulators outside the tensor core (see mma_row).
//   Split operands: acc += A_lo * B_hi + A_hi * B_lo + A_hi * B_hi (the lo * lo term is below fp32 rounding).
//   Optional epilogue statistics: per output channel {sum (y - pivot), sum (y - pivot)^2} in fp64, per-warp shared
//   accumulators merged in a fixed order (deterministic), one [Cout][2] block per CTA for bn_finalize_sums.
//
// Weight gradient (wgrad_tc_*):
//   dW[co][ci][tap] = scale * sum_{pixels p} dY[p][co] * A[p (+) tap][ci],  A = relu?((x - mean) * scale + shift)
//   GEMM: M = 128 output channels, N = one input-channel tile, K = pixels in steps of 32, one tap per CTA, split-K over
//   pixel ranges. tf32 wgmma takes K-major operands only, so the transform threads write both operands transposed
//   (channel rows of 32 pixels). Each CTA stores an fp32 partial; a second kernel reduces the partials in a fixed
//   order (deterministic) into the OIHW gradient.
#include <cuda_fp16.h>

#include <atomic>

#include "common.cuh"
#include "kernels.h"
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
template <bool kF16, int kN, bool kSepCross>
__device__ __forceinline__ void mma_row(float (&part)[kN / 2], float (&part_x)[kN / 2], uint32_t a_hi, uint32_t a_lo,
                                        uint32_t b_hi, uint32_t b_lo, bool split) {
  const uint64_t dah = gmma_desc_sw128(a_hi), dal = gmma_desc_sw128(a_lo);
  const uint64_t dbh = gmma_desc_sw128(b_hi), dbl = gmma_desc_sw128(b_lo);
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t o = (uint64_t)(kk * 2);
    const int acc = kk > 0 ? 1 : 0;
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
  const float* residual;
  const float* relu_mask;
  float* y;
  float out_scale;
  const float* in_scale;       // nullable device float[2] {S, 1/S}: operands are x * S, the epilogue multiplies by 1/S
  double* stat_part;           // nullable [gridDim.x][Cout][2] = {sum (y - pivot), sum (y - pivot)^2}
  const float* stat_pivot;     // nullable [Cout]
};

template <bool kF16, int kN>
__global__ void __launch_bounds__(kThreads, 1) conv_wgmma_kernel(const ConvParams p) {
  constexpr int kCB = kF16 ? 64 : 32;       // input channels per K step (one 128-byte operand row)
  constexpr int kV = kF16 ? 2 : 1;          // raw float4 per thread, row and K step
  constexpr int kChunkEl = kF16 ? 8 : 4;    // weight elements per 16-byte chunk
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  double* s_stat = reinterpret_cast<double*>(smem + (size_t)kStages * p.stage_bytes);
  const uint32_t smem_a = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const bool split = p.passes == 3;
  const bool stats = p.stat_part != nullptr;
  const float in_s = p.in_scale ? __ldg(p.in_scale) : 1.f;
  const float oscale = p.in_scale ? p.out_scale * __ldg(p.in_scale + 1) : p.out_scale;
  const uint32_t a_lo_off = split ? (uint32_t)kATileBytes : 0u;
  const uint32_t b_off = (split ? 2u : 1u) * (uint32_t)kATileBytes;
  const uint32_t b_lo_off = split ? (uint32_t)p.b_tile_bytes : 0u;
  const char* wh = reinterpret_cast<const char*>(p.w_hi);
  const char* wl = reinterpret_cast<const char*>(p.w_lo ? p.w_lo : p.w_hi);
  constexpr int kEl = kF16 ? 2 : 4;
  if (stats) {
    for (int i = tid; i < 8 * p.Cout * 2; i += kThreads) s_stat[i] = 0.0;
  }
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
    auto load_b = [&](int ks, uint32_t st) {
      const int tap = ks / p.ncb, cb = ks - tap * p.ncb;
      for (int idx = tid; idx < p.nt * 8; idx += kThreads) {
        const int n = idx >> 3, jj = idx & 7;
        const int c = cb * kCB + jj * kChunkEl;
        const bool ok = c < p.Cin;
        const size_t off = ((((size_t)tap * p.Cout + n0 + n) * p.Cin) + (ok ? c : 0)) * kEl;
        const uint32_t dst = st + b_off + (uint32_t)n * 128u + ((uint32_t)(jj ^ (n & 7)) << 4);
        cp_async16(dst, wh + off, ok);
        if (split) cp_async16(dst + b_lo_off, wl + off, ok);
      }
      cp_async_commit();
    };

    // one partial for all terms here: a separate cross-term partial would push the fp16 N = 128 form past 255 registers
    float acc[kN / 2], part[kN / 2];
    zero_acc(acc);
    zero_acc(part);
    load_b(0, smem_a);
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
        load_b(ks + 1, smem_a + (uint32_t)(((ks + 1) % kStages) * p.stage_bytes));
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

    // ---- epilogue: fragment row g (+8), columns 8 i + 2 t (+1) of this warp's 16 rows ----
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
          const float2 r2 = __ldg(reinterpret_cast<const float2*>(p.residual + off));
          o.x += r2.x; o.y += r2.y;
        }
        if (p.relu_mask) {
          const float2 k = __ldg(reinterpret_cast<const float2*>(p.relu_mask + off));
          o.x = k.x > 0.f ? o.x : 0.f; o.y = k.y > 0.f ? o.y : 0.f;
        }
        *reinterpret_cast<float2*>(p.y + off) = o;
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
  if (stats) {
    __syncthreads();
    for (int i = tid; i < p.Cout * 2; i += kThreads) {
      double v = 0.0;
      for (int w8 = 0; w8 < 8; ++w8) v += s_stat[(size_t)w8 * p.Cout * 2 + i];   // fixed order
      p.stat_part[(size_t)blockIdx.x * p.Cout * 2 + i] = v;
    }
  }
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

template <bool kF16, int kN>
int launch_n(const ConvParams& p, int grid, size_t smem, cudaStream_t stream) {
  static std::atomic<uint64_t> done{0};
  if (int rc = allow_smem(conv_wgmma_kernel<kF16, kN>, done)) return rc;
  conv_wgmma_kernel<kF16, kN><<<grid, kThreads, smem, stream>>>(p);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

template <bool kF16>
int launch_f(const ConvParams& p, int grid, size_t smem, cudaStream_t stream) {
  switch (p.nt) {
    case 16: return launch_n<kF16, 16>(p, grid, smem, stream);
    case 32: return launch_n<kF16, 32>(p, grid, smem, stream);
    case 48: return launch_n<kF16, 48>(p, grid, smem, stream);
    case 64: return launch_n<kF16, 64>(p, grid, smem, stream);
    case 80: return launch_n<kF16, 80>(p, grid, smem, stream);
    case 96: return launch_n<kF16, 96>(p, grid, smem, stream);
    case 112: return launch_n<kF16, 112>(p, grid, smem, stream);
    case 128: return launch_n<kF16, 128>(p, grid, smem, stream);
  }
  set_last_error("conv_wgmma: no kernel for a %d-column slice", p.nt);
  return FPD_ERR_UNSUPPORTED;
}

int conv_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift, int pre_relu,
                const void* w_hi, const void* w_lo, int f16, const float* bias, const float* residual,
                const float* relu_mask, float* y, float out_scale, const float* in_scale, int B, int H, int W, int Cin,
                int Cout, int ksize, int num_sms, cudaStream_t stream, double* stat_part, const float* stat_pivot) {
  FPD_REQUIRE(x && w_hi && y, "conv_wgmma: null operand");
  FPD_REQUIRE((double)B * H * W * Cout < 4294967296.0, "conv_wgmma: output has 2^32 or more elements");
  FPD_REQUIRE((pre_scale == nullptr) == (pre_shift == nullptr), "conv_wgmma: pre_scale/pre_shift come in pairs");
  FPD_REQUIRE(pre_scale != nullptr || pre_mean == nullptr, "conv_wgmma: pre_mean needs pre_scale/pre_shift");
  FPD_REQUIRE(stat_part == nullptr || Cout <= kMaxStatCout, "conv_wgmma: statistics need Cout <= %d", kMaxStatCout);
  ConvParams p{};
  p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.ksize = ksize; p.P = B * H * W;
  p.passes = w_lo ? 3 : 1;
  p.nt = conv_tc_ts_slice(Cout);
  p.n_tiles = Cout / p.nt;
  p.num_tiles = conv_num_tiles(B, H, W, Cout);
  p.ncb = (Cin + (f16 ? 63 : 31)) / (f16 ? 64 : 32);
  p.ksteps = ksize * ksize * p.ncb;
  p.b_tile_bytes = p.nt * 128;
  p.stage_bytes = (p.passes == 3 ? 2 : 1) * (kATileBytes + p.b_tile_bytes);
  p.x = x; p.w_hi = w_hi; p.w_lo = w_lo;
  p.pre_mean = pre_mean; p.pre_scale = pre_scale; p.pre_shift = pre_shift; p.pre_relu = pre_relu;
  p.bias = bias; p.residual = residual; p.relu_mask = relu_mask; p.y = y;
  p.out_scale = f16 ? out_scale * (1.0f / (float)(1 << kF16WeightScaleLog2)) : out_scale;
  p.in_scale = in_scale;
  p.stat_part = stat_part; p.stat_pivot = stat_pivot;
  const size_t smem = 1024 + (size_t)kStages * p.stage_bytes + (stat_part ? (size_t)8 * Cout * 2 * sizeof(double) : 0);
  FPD_REQUIRE(smem <= (size_t)kSmemLimit, "conv_wgmma: shared memory plan %zu B too large", smem);
  const int grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
  return f16 ? launch_f<true>(p, grid, smem, stream) : launch_f<false>(p, grid, smem, stream);
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

template <int kN>
int wgrad_launch_n(const WgradParams& p, int grid, size_t smem, cudaStream_t stream) {
  static std::atomic<uint64_t> done{0};
  if (int rc = allow_smem(wgrad_wgmma_kernel<kN>, done)) return rc;
  wgrad_wgmma_kernel<kN><<<grid, kThreads, smem, stream>>>(p);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // namespace

// ------------------------------------------------- forward entry points -------------------------------------------------

// Output channels are processed in slices of nt columns: the widest divisor of Cout that is a multiple of 16 and at
// most 128 (one wgmma N per slice; the accumulators of a 64 x 128 warpgroup tile take 64 registers per thread).
int conv_tc_ts_slice(int Cout) {
  if (Cout <= 128) return Cout % 16 == 0 ? Cout : 0;
  for (int nt = 128; nt >= 16; nt -= 16)
    if (Cout % nt == 0) return nt;
  return 0;
}

bool conv_tc_ts_supported(int Cin, int Cout, int ksize) { return conv_shape_ok(Cin, Cout, ksize, 0, kMaxCinTs, 1024); }

int conv_tc_ts_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                      int pre_relu, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                      const float* relu_mask, float* y, float out_scale, int B, int H, int W, int Cin, int Cout,
                      int ksize, int num_sms, cudaStream_t stream) {
  FPD_REQUIRE(conv_tc_ts_supported(Cin, Cout, ksize), "conv_tc_ts: unsupported shape Cin=%d Cout=%d k=%d", Cin, Cout,
              ksize);
  return conv_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, 0, bias, residual, relu_mask, y,
                     out_scale, nullptr, B, H, W, Cin, Cout, ksize, num_sms, stream, nullptr, nullptr);
}

bool conv_tc_h_supported(int Cin, int Cout, int ksize, int H, int W, int f16) {
  (void)H; (void)W;
  return conv_shape_ok(Cin, Cout, ksize, f16, kMaxCinH, 2048);
}

int conv_tc_h_stats_grid(int B, int H, int W, int Cin, int Cout, int ksize, int f16, int num_sms) {
  if (!conv_tc_h_supported(Cin, Cout, ksize, H, W, f16) || Cout > kMaxStatCout) return 0;
  const int tiles = conv_num_tiles(B, H, W, Cout);
  return tiles < num_sms ? tiles : num_sms;
}

int conv_tc_h_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                     int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                     const float* residual, const float* relu_mask, float* y, float out_scale, const float* in_scale,
                     int B, int H, int W, int Cin, int Cout, int ksize, int num_sms, cudaStream_t stream,
                     double* stat_part, const float* stat_pivot) {
  FPD_REQUIRE(conv_tc_h_supported(Cin, Cout, ksize, H, W, f16),
              "conv_tc_h: unsupported shape Cin=%d Cout=%d k=%d H=%d W=%d f16=%d", Cin, Cout, ksize, H, W, f16);
  return conv_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, f16, bias, residual, relu_mask, y,
                     out_scale, in_scale, B, H, W, Cin, Cout, ksize, num_sms, stream, stat_part, stat_pivot);
}

// ---------------------------------------------- weight-gradient entry points ----------------------------------------------

// Shapes taken per launch: 3x3 with Cin in {32, 64, 128} and Cout a multiple of 32 up to 256; 1x1 with Cin <= 256 and
// any Cout % 4 == 0. Wider layers go through ops.conv2d_wgrad_tc_chunked in channel chunks of these sizes, which keeps
// the per-launch partial-sum workspace (splits x taps x Cin x Cout) small.
bool wgrad_tc_supported(int Cin, int Cout, int ksize) {
  if (ksize == 3) return (Cin == 32 || Cin == 64 || Cin == 128) && Cout % 32 == 0 && Cout >= 32 && Cout <= 256;
  return ksize == 1 && Cout % 4 == 0 && Cin % 4 == 0 && Cin >= 4 && Cin <= 256;
}

bool wgrad_tc3_supported(int H, int W, int Cin, int Cout, int ksize) {
  (void)H; (void)W;
  return ksize == 3 && wgrad_tc_supported(Cin, Cout, ksize);
}

size_t wgrad_tc_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, int num_sms) {
  if (!wgrad_tc_supported(Cin, Cout, ksize)) return 0;
  const WgradPlan pl = wgrad_plan(B, H, W, Cin, Cout, ksize, num_sms);
  return (size_t)pl.splits * pl.taps * Cin * Cout * sizeof(float);
}

int wgrad_tc_fused_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                          int pre_relu, const float* dy, int passes, float* dw_oihw, float scale, int B, int H, int W,
                          int Cin, int Cout, int ksize, void* workspace, size_t workspace_bytes, int num_sms,
                          cudaStream_t stream) {
  FPD_REQUIRE(wgrad_tc_supported(Cin, Cout, ksize), "wgrad_tc: unsupported shape Cin=%d Cout=%d k=%d", Cin, Cout, ksize);
  FPD_REQUIRE(x && dy && dw_oihw, "wgrad_tc: null operand");
  FPD_REQUIRE(passes == 1 || passes == 3, "wgrad_tc_fused: passes must be 1 or 3");
  FPD_REQUIRE((pre_scale == nullptr) == (pre_shift == nullptr), "wgrad_tc_fused: pre_scale/pre_shift come in pairs");
  const WgradPlan pl = wgrad_plan(B, H, W, Cin, Cout, ksize, num_sms);
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
  int rc = pl.n == 32 ? wgrad_launch_n<32>(p, grid, smem, stream)
         : pl.n == 64 ? wgrad_launch_n<64>(p, grid, smem, stream)
                      : wgrad_launch_n<128>(p, grid, smem, stream);
  if (rc) return rc;
  const int64_t total = (int64_t)pl.taps * Cin * Cout;
  wgrad_reduce_kernel<<<(int)((total + 31) / 32), 256, 0, stream>>>(p.partial, dw_oihw, scale, Cin, Cout, pl.taps,
                                                                    pl.splits);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // namespace fpd
