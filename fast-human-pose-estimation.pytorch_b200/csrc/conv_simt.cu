// conv_simt.cu -- fp32 CUDA-core convolution on NHWC activations with OIHW weights, for the shapes the
// tensor-core kernels do not take: the 7x7 stride-2 stem (reference lib/models/hourglass.py:116, Cin=3),
// the 16-channel score / score_ 1x1 convs (hourglass.py:135-137), stride-2 3x3 convs (pose_hrnet.py:205-239)
// and odd shapes. Also the on-device cross-check the tests use for conv_tc / wgrad_tc.
// fp32 FFMA accumulation throughout, so results track the fp32 reference to round-off.
//
// Design: the (small) weight tensor is staged once per CTA in shared memory, re-laid out so the inner loop reads
// it as conflict-free float4 broadcasts; each thread owns one pixel x 4 channels; activations come through the
// read-only path (neighbouring threads share pixels, so they hit L1). The weight gradient is a two-stage,
// fixed-order (deterministic) reduction: per-CTA partials over a pixel chunk, then a sum over chunks.
#include "common.cuh"

namespace fpd {
namespace {

constexpr int kMaxSmemWeights = 24 * 1024;  // floats (96 KB)

// ------------------------------------------------------------------------------------------------ forward
// smem weights: ws[(tap*Cin + ci) * CoutP + co], CoutP = Cout rounded up to 4
__global__ void __launch_bounds__(256)
conv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                const float* __restrict__ residual, float* __restrict__ y, int B, int H, int W, int Cin, int Cout,
                int k, int stride, int pad, int Ho, int Wo, int use_smem) {
  extern __shared__ float ws[];
  const int taps = k * k;
  const int CoutP = (Cout + 3) & ~3;
  if (use_smem) {
    const int n = taps * Cin * CoutP;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int co = i % CoutP;
      const int kc = i / CoutP;  // tap*Cin + ci
      const int ci = kc % Cin, tap = kc / Cin;
      ws[i] = co < Cout ? __ldg(w + ((int64_t)co * Cin + ci) * taps + tap) : 0.f;
    }
    __syncthreads();
  }
  const int cq = CoutP / 4;
  const int64_t n = (int64_t)B * Ho * Wo * cq;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % cq) * 4;
    int64_t t = i / cq;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int kh = 0; kh < k; ++kh) {
      const int hi = ho * stride + kh - pad;
      if (hi < 0 || hi >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int wi = wo * stride + kw - pad;
        if (wi < 0 || wi >= W) continue;
        const float* xp = x + (((int64_t)b * H + hi) * W + wi) * Cin;
        const int tap = kh * k + kw;
        if (use_smem) {
          const float* wp = ws + (size_t)tap * Cin * CoutP + c4;
#pragma unroll 4
          for (int ci = 0; ci < Cin; ++ci) {
            const float xv = __ldg(xp + ci);
            const float4 wv = *reinterpret_cast<const float4*>(wp + (size_t)ci * CoutP);
            acc[0] = fmaf(xv, wv.x, acc[0]);
            acc[1] = fmaf(xv, wv.y, acc[1]);
            acc[2] = fmaf(xv, wv.z, acc[2]);
            acc[3] = fmaf(xv, wv.w, acc[3]);
          }
        } else {
          for (int ci = 0; ci < Cin; ++ci) {
            const float xv = __ldg(xp + ci);
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (c4 + j < Cout) acc[j] = fmaf(xv, __ldg(w + ((int64_t)(c4 + j) * Cin + ci) * taps + tap), acc[j]);
          }
        }
      }
    }
    const int64_t o = (((int64_t)b * Ho + ho) * Wo + wo) * Cout + c4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c4 + j < Cout) {
        float v = acc[j];
        if (bias) v += __ldg(bias + c4 + j);
        if (residual) v += __ldg(residual + o + j);
        y[o + j] = v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ dgrad
// dx[b,hi,wi,ci] = sum_{co,kh,kw} dy[b,ho,wo,co] * w[co,ci,kh,kw];   smem weights: ws[(tap*Cout + co)*CinP + ci]
__global__ void __launch_bounds__(256)
conv_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx, int B, int H,
                  int W, int Cin, int Cout, int k, int stride, int pad, int Ho, int Wo, int use_smem) {
  extern __shared__ float ws[];
  const int taps = k * k;
  const int CinP = (Cin + 3) & ~3;
  if (use_smem) {
    const int n = taps * Cout * CinP;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int ci = i % CinP;
      const int kc = i / CinP;  // tap*Cout + co
      const int co = kc % Cout, tap = kc / Cout;
      ws[i] = ci < Cin ? __ldg(w + ((int64_t)co * Cin + ci) * taps + tap) : 0.f;
    }
    __syncthreads();
  }
  const int cq = CinP / 4;
  const int64_t n = (int64_t)B * H * W * cq;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % cq) * 4;
    int64_t t = i / cq;
    const int wi = (int)(t % W); t /= W;
    const int hi = (int)(t % H);
    const int b = (int)(t / H);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int kh = 0; kh < k; ++kh) {
      const int hn = hi + pad - kh;
      if (hn < 0 || hn % stride != 0) continue;
      const int ho = hn / stride;
      if (ho >= Ho) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int wn = wi + pad - kw;
        if (wn < 0 || wn % stride != 0) continue;
        const int wo = wn / stride;
        if (wo >= Wo) continue;
        const float* gp = dy + (((int64_t)b * Ho + ho) * Wo + wo) * Cout;
        const int tap = kh * k + kw;
        if (use_smem) {
          const float* wp = ws + (size_t)tap * Cout * CinP + c4;
#pragma unroll 4
          for (int co = 0; co < Cout; ++co) {
            const float g = __ldg(gp + co);
            const float4 wv = *reinterpret_cast<const float4*>(wp + (size_t)co * CinP);
            acc[0] = fmaf(g, wv.x, acc[0]);
            acc[1] = fmaf(g, wv.y, acc[1]);
            acc[2] = fmaf(g, wv.z, acc[2]);
            acc[3] = fmaf(g, wv.w, acc[3]);
          }
        } else {
          for (int co = 0; co < Cout; ++co) {
            const float g = __ldg(gp + co);
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (c4 + j < Cin) acc[j] = fmaf(g, __ldg(w + ((int64_t)co * Cin + c4 + j) * taps + tap), acc[j]);
          }
        }
      }
    }
    const int64_t o = (((int64_t)b * H + hi) * W + wi) * Cin + c4;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (c4 + j < Cin) dx[o + j] = acc[j];
  }
}

// ------------------------------------------------------------------------------------------------ wgrad
// Stage 1: CTA c owns output pixels [c*chunk, (c+1)*chunk). Work item = (kc = tap*Cin+ci, group of 8 output
// channels); each thread keeps 8 partial sums in registers over the chunk. dy rows are staged in shared memory
// in sub-chunks of kSub pixels; x is gathered through L1. partial[c][kc][co].
constexpr int kSub = 64;

__global__ void __launch_bounds__(256)
conv_wgrad_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ partial,
                          int B, int H, int W, int Cin, int Cout, int k, int stride, int pad, int Ho, int Wo,
                          int chunk) {
  extern __shared__ float sdy[];  // [kSub][CoutP8]
  const int taps = k * k;
  const int K = taps * Cin;
  const int CoutP8 = (Cout + 7) & ~7;
  const int cg = CoutP8 / 8;
  const int items = K * cg;
  const int64_t P = (int64_t)B * Ho * Wo;
  const int64_t p0 = (int64_t)blockIdx.x * chunk;
  int64_t p1 = p0 + chunk;
  if (p1 > P) p1 = P;
  float* out = partial + (size_t)blockIdx.x * K * CoutP8;
  for (int it0 = 0; it0 < items; it0 += blockDim.x) {
    const int it = it0 + threadIdx.x;
    const bool active = it < items;
    const int kc = active ? it / cg : 0;
    const int co0 = active ? (it % cg) * 8 : 0;
    const int tap = kc / Cin, ci = kc % Cin;
    const int kh = tap / k, kw = tap % k;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int64_t s0 = p0; s0 < p1; s0 += kSub) {
      const int ns = (int)min((int64_t)kSub, p1 - s0);
      __syncthreads();
      for (int i = threadIdx.x; i < ns * CoutP8; i += blockDim.x) {
        const int pp = i / CoutP8, c = i % CoutP8;
        sdy[i] = c < Cout ? __ldg(dy + (s0 + pp) * Cout + c) : 0.f;
      }
      __syncthreads();
      if (active) {
        for (int pp = 0; pp < ns; ++pp) {
          const int64_t p = s0 + pp;
          const int wo = (int)(p % Wo);
          const int ho = (int)((p / Wo) % Ho);
          const int b = (int)(p / ((int64_t)Wo * Ho));
          const int hi = ho * stride + kh - pad, wi = wo * stride + kw - pad;
          if (hi < 0 || hi >= H || wi < 0 || wi >= W) continue;
          const float xv = __ldg(x + (((int64_t)b * H + hi) * W + wi) * Cin + ci);
          const float4 g0 = *reinterpret_cast<const float4*>(sdy + pp * CoutP8 + co0);
          const float4 g1 = *reinterpret_cast<const float4*>(sdy + pp * CoutP8 + co0 + 4);
          acc[0] = fmaf(xv, g0.x, acc[0]); acc[1] = fmaf(xv, g0.y, acc[1]);
          acc[2] = fmaf(xv, g0.z, acc[2]); acc[3] = fmaf(xv, g0.w, acc[3]);
          acc[4] = fmaf(xv, g1.x, acc[4]); acc[5] = fmaf(xv, g1.y, acc[5]);
          acc[6] = fmaf(xv, g1.z, acc[6]); acc[7] = fmaf(xv, g1.w, acc[7]);
        }
      }
    }
    if (active) {
#pragma unroll
      for (int j = 0; j < 8; ++j) out[(size_t)kc * CoutP8 + co0 + j] = acc[j];
    }
  }
}

// one warp per weight element; lanes sum a strided subset of the chunk partials, then a fixed-order shuffle tree
__global__ void conv_wgrad_final_kernel(const float* __restrict__ partial, float* __restrict__ dw, float scale,
                                        int nchunks, int Cin, int Cout, int taps) {
  const int CoutP8 = (Cout + 7) & ~7;
  const int K = taps * Cin;
  const int64_t total = (int64_t)Cout * Cin * taps;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= total) return;
  const int tap = (int)(i % taps);
  const int ci = (int)((i / taps) % Cin);
  const int co = (int)(i / ((int64_t)taps * Cin));
  const size_t off = (size_t)(tap * Cin + ci) * CoutP8 + co;
  double s = 0.0;
  for (int c = lane; c < nchunks; c += 32) s += (double)partial[(size_t)c * K * CoutP8 + off];
  s = warp_sum(s);
  if (lane == 0) dw[i] = (float)(s * (double)scale);
}

inline int grid_for(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  const int64_t cap = kNumSMs * 16;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

struct WgradGeom {
  int chunk, nchunks;
  size_t bytes;
};
inline WgradGeom wgrad_geom(int64_t P, int Cin, int Cout, int k) {
  WgradGeom g;
  const int CoutP8 = (Cout + 7) & ~7;
  const size_t per_chunk = (size_t)k * k * Cin * CoutP8 * sizeof(float);
  // aim for ~2 waves of CTAs but keep the partial buffer under ~64 MB
  int64_t nch = kNumSMs * 4;
  const int64_t cap = (int64_t)((64u << 20) / per_chunk);
  if (nch > cap) nch = cap < 1 ? 1 : cap;
  int64_t chunk = (P + nch - 1) / nch;
  chunk = (chunk + kSub - 1) / kSub * kSub;
  g.chunk = (int)chunk;
  g.nchunks = (int)((P + chunk - 1) / chunk);
  g.bytes = (size_t)g.nchunks * per_chunk;
  return g;
}

}  // namespace
}  // namespace fpd

using namespace fpd;

extern "C" {

int fpd_conv2d_simt_fwd(const float* x, const float* w_oihw, const float* bias, const float* residual, float* y,
                        int B, int H, int W, int Cin, int Cout, int k, int stride, int pad, fpd_stream_t stream) {
  FPD_REQUIRE(k >= 1 && stride >= 1 && pad >= 0, "conv_simt_fwd: bad geometry");
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const int CoutP = (Cout + 3) & ~3;
  const int64_t n = (int64_t)B * Ho * Wo * (CoutP / 4);
  const int wfloats = k * k * Cin * CoutP;
  const int use_smem = wfloats <= kMaxSmemWeights;
  const size_t smem = use_smem ? (size_t)wfloats * sizeof(float) : 0;
  static bool attr = false;
  if (!attr) {
    FPD_CUDA_CHECK(cudaFuncSetAttribute(conv_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        kMaxSmemWeights * (int)sizeof(float)));
    attr = true;
  }
  int grid = grid_for(n, 256);
  if (use_smem && grid > kNumSMs * 4) grid = kNumSMs * 4;  // amortise the weight staging over a grid-stride loop
  conv_fwd_kernel<<<grid, 256, smem, stream>>>(x, w_oihw, bias, residual, y, B, H, W, Cin, Cout, k, stride, pad, Ho,
                                               Wo, use_smem);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_conv2d_simt_dgrad(const float* dy, const float* w_oihw, float* dx, int B, int H, int W, int Cin, int Cout,
                          int k, int stride, int pad, fpd_stream_t stream) {
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const int CinP = (Cin + 3) & ~3;
  const int64_t n = (int64_t)B * H * W * (CinP / 4);
  const int wfloats = k * k * Cout * CinP;
  const int use_smem = wfloats <= kMaxSmemWeights;
  const size_t smem = use_smem ? (size_t)wfloats * sizeof(float) : 0;
  static bool attr = false;
  if (!attr) {
    FPD_CUDA_CHECK(cudaFuncSetAttribute(conv_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        kMaxSmemWeights * (int)sizeof(float)));
    attr = true;
  }
  int grid = grid_for(n, 256);
  if (use_smem && grid > kNumSMs * 4) grid = kNumSMs * 4;
  conv_dgrad_kernel<<<grid, 256, smem, stream>>>(dy, w_oihw, dx, B, H, W, Cin, Cout, k, stride, pad, Ho, Wo,
                                                 use_smem);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

size_t fpd_conv2d_simt_wgrad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k, int stride, int pad) {
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  return wgrad_geom((int64_t)B * Ho * Wo, Cin, Cout, k).bytes;
}

int fpd_conv2d_simt_wgrad(const float* x, const float* dy, float* dw_oihw, float scale, int B, int H, int W,
                          int Cin, int Cout, int k, int stride, int pad, void* workspace, size_t ws_bytes,
                          fpd_stream_t stream) {
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const int64_t P = (int64_t)B * Ho * Wo;
  const WgradGeom g = wgrad_geom(P, Cin, Cout, k);
  FPD_REQUIRE(workspace && ws_bytes >= g.bytes, "conv_simt_wgrad: workspace too small (%zu < %zu)", ws_bytes, g.bytes);
  const int CoutP8 = (Cout + 7) & ~7;
  const size_t smem = (size_t)kSub * CoutP8 * sizeof(float);
  FPD_REQUIRE(smem <= 192 * 1024, "conv_simt_wgrad: Cout=%d too wide for the CUDA-core path", Cout);
  static bool wattr = false;
  if (!wattr) {   // dy sub-chunk tile [64][Cout]: opt in beyond 48 KB for the wide HRNet stride-2 convs (Cout 256 / 384)
    FPD_CUDA_CHECK(cudaFuncSetAttribute(conv_wgrad_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 192 * 1024));
    wattr = true;
  }
  conv_wgrad_partial_kernel<<<g.nchunks, 256, smem, stream>>>(x, dy, (float*)workspace, B, H, W, Cin, Cout, k, stride,
                                                              pad, Ho, Wo, g.chunk);
  FPD_LAUNCH_CHECK();
  const int64_t total = (int64_t)Cout * Cin * k * k;
  conv_wgrad_final_kernel<<<(unsigned)((total * 32 + 127) / 128), 128, 0, stream>>>((const float*)workspace, dw_oihw,
                                                                                    scale, g.nchunks, Cin, Cout, k * k);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // extern "C"
