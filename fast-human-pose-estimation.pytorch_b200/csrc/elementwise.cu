// elementwise.cu -- the HBM-bound glue of the hourglass / HRNet hot path on NHWC fp32 tensors:
// BatchNorm batch statistics (reference: nn.BatchNorm2d in train mode, lib/models/hourglass.py:18-26,117),
// BN+ReLU apply fused with the tf32 hi/lo operand split, BN backward, 2x2 max-pool fwd/bwd
// (hourglass.py:82,124), nearest-2x upsample + add (hourglass.py:60,90-91), layout converts, weight
// re-layout. All kernels are vectorised (float4 along the channel axis = the contiguous NHWC axis) and
// sized for >= 2 waves of the H100's 132 SMs (kNumSMs); reductions are deterministic (fixed-order partial buffers, no atomics).
// Also the library's state behind fpd_last_error, fpd_launch_count and fpd_sm_count.
#include <cuda_fp16.h>

#include <atomic>
#include <cstdarg>

#include "common.cuh"

namespace fpd {

namespace {

constexpr int kRedThreads = 256;
constexpr int kMaxRedBlocks = 4 * kNumSMs;   // enough bytes in flight for HBM, and a short second stage

struct RedGeom {
  int L;       // float4 lanes across channels (C/4)
  int R;       // pixel rows handled per block iteration
  int nblocks;
  int64_t rows_per_block;
};

inline RedGeom red_geom(int64_t P, int C, int max_blocks = kMaxRedBlocks);
// the single-launch (last block finishes) forms keep the second stage short: one wave of blocks
constexpr int kMaxFusedRedBlocks = kNumSMs;
inline RedGeom red_geom(int64_t P, int C, int max_blocks) {
  RedGeom g;
  g.L = C / 4;
  g.R = kRedThreads / g.L;
  if (g.R < 1) g.R = 1;
  int64_t want = (P + (int64_t)g.R * 4 - 1) / ((int64_t)g.R * 4);
  if (want < 1) want = 1;
  g.nblocks = (int)(want < max_blocks ? want : max_blocks);
  g.rows_per_block = (P + g.nblocks - 1) / g.nblocks;
  // round rows_per_block up to a multiple of R so chunk boundaries are uniform
  g.rows_per_block = (g.rows_per_block + g.R - 1) / g.R * g.R;
  g.nblocks = (int)((P + g.rows_per_block - 1) / g.rows_per_block);
  return g;
}

// -------------------------------------------------------------------------------------------------
// BN statistics: per block -> (n, mean, M2) per channel, merged with Chan's parallel formula in fp64.
// -------------------------------------------------------------------------------------------------
template <bool kWide>   // kWide: more than 1024 channels (the common narrow form keeps its single-trip code)
__global__ void __launch_bounds__(kRedThreads)
bn_stats_partial_kernel(const float* __restrict__ x, int64_t P, int C, int L, int R, int64_t rows_per_block,
                        double* __restrict__ part /*[nblocks][C][2]*/) {
  extern __shared__ double sm[];  // [R][C][2] (mean, M2) + counts [R]
  const int tid = threadIdx.x;
  // more than 4 x 256 channels (pose_resnet's 2048-channel layer4): the block walks the channel lanes in segments of 256
  const int Lc = L < kRedThreads ? L : kRedThreads;
  const int ry = tid / Lc;
  const int64_t row0 = (int64_t)blockIdx.x * rows_per_block;
  int64_t row1 = row0 + rows_per_block;
  if (row1 > P) row1 = P;
  const int cx0 = tid % Lc;
  if (ry < R)
  for (int cx = cx0; kWide ? cx < L : cx == cx0; cx += kRedThreads) {
    float piv[4] = {0, 0, 0, 0}, s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
    int n = 0;
    for (int64_t r = row0 + ry; r < row1; r += R) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * C) + cx);
      const float e[4] = {v.x, v.y, v.z, v.w};
      if (n == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) piv[j] = e[j];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float d = e[j] - piv[j];
        s1[j] += d;
        s2[j] = fmaf(d, d, s2[j]);
      }
      ++n;
    }
    double* cnt = sm + (size_t)R * C * 2;
    if (cx == 0) cnt[ry] = (double)n;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double mean = 0.0, m2 = 0.0;
      if (n > 0) {
        const double ds1 = (double)s1[j], ds2 = (double)s2[j];
        mean = (double)piv[j] + ds1 / n;
        m2 = ds2 - ds1 * ds1 / n;
        if (m2 < 0.0) m2 = 0.0;
      }
      sm[((size_t)ry * C + cx * 4 + j) * 2 + 0] = mean;
      sm[((size_t)ry * C + cx * 4 + j) * 2 + 1] = m2;
    }
  }
  __syncthreads();
  for (int c = tid; c < C; c += kRedThreads) {
    const double* cnt = sm + (size_t)R * C * 2;
    double na = 0.0, ma = 0.0, m2a = 0.0;
    for (int r = 0; r < R; ++r) {
      const double nb = cnt[r];
      if (nb == 0.0) continue;
      const double mb = sm[((size_t)r * C + c) * 2 + 0];
      const double m2b = sm[((size_t)r * C + c) * 2 + 1];
      const double nt = na + nb;
      const double delta = mb - ma;
      ma += delta * (nb / nt);
      m2a += m2b + delta * delta * (na * nb / nt);
      na = nt;
    }
    part[((size_t)blockIdx.x * C + c) * 2 + 0] = ma;
    part[((size_t)blockIdx.x * C + c) * 2 + 1] = m2a;
  }
}

// one warp per channel: each lane Chan-merges a strided subset of the block partials, then the lanes merge by
// shuffle (fixed order -> deterministic).
__global__ void bn_stats_final_kernel(const double* __restrict__ part, int nblocks, int64_t rows_per_block,
                                      int64_t P, int C, float* __restrict__ mean, float* __restrict__ var) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  double na = 0.0, ma = 0.0, m2a = 0.0;
  for (int b = lane; b < nblocks; b += 32) {
    int64_t r0 = (int64_t)b * rows_per_block, r1 = r0 + rows_per_block;
    if (r1 > P) r1 = P;
    const double nb = (double)(r1 - r0);
    if (nb <= 0.0) continue;
    const double mb = part[((size_t)b * C + c) * 2 + 0];
    const double m2b = part[((size_t)b * C + c) * 2 + 1];
    const double nt = na + nb;
    const double delta = mb - ma;
    ma += delta * (nb / nt);
    m2a += m2b + delta * delta * (na * nb / nt);
    na = nt;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double nb = __shfl_xor_sync(0xffffffffu, na, o);
    const double mb = __shfl_xor_sync(0xffffffffu, ma, o);
    const double m2b = __shfl_xor_sync(0xffffffffu, m2a, o);
    const double nt = na + nb;
    if (nt > 0.0) {
      // symmetric form so both partners compute the identical merged triple
      const double mean_t = (na * ma + nb * mb) / nt;
      const double delta = mb - ma;
      m2a = m2a + m2b + delta * delta * (na * nb / nt);
      ma = mean_t;
      na = nt;
    }
  }
  if (lane == 0) {
    mean[c] = (float)ma;
    var[c] = (float)(m2a / (double)P);
  }
}

__global__ void bn_finalize_kernel(const float* __restrict__ mean, const float* __restrict__ var,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   int64_t count, float* __restrict__ scale, float* __restrict__ shift,
                                   float* __restrict__ invstd_out, float* __restrict__ rmean,
                                   float* __restrict__ rvar, float momentum, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float m = mean[c], v = var[c];
  const float invstd = (float)(1.0 / sqrt((double)v + (double)eps));
  const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  const float sc = g * invstd;
  scale[c] = sc;
  shift[c] = b;  // centred form: y = (x - mean) * scale + shift
  if (invstd_out) invstd_out[c] = invstd;
  if (rmean) {
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * m;
    const float unbiased = count > 1 ? v * ((float)count / (float)(count - 1)) : v;
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * unbiased;
  }
}

// "Last block finishes" form of a two-stage reduction: every block publishes its partial, takes a ticket, and the
// block that draws the last ticket runs the (fixed-order, hence deterministic) second stage. One launch instead of two
// or three; the ticket counter must be zero on entry and is left zero (self-resetting, CUDA-graph safe). Returns true in
// the finishing block only.
__device__ __forceinline__ bool last_block_ticket(unsigned int* counter) {
  __shared__ bool s_last;
  __threadfence();   // release this block's partials
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (s_last) __threadfence();   // acquire the other blocks' partials
  return s_last;
}

struct BnFinalize {
  const float* gamma; const float* beta; float eps; float momentum;
  float* mean; float* var; float* scale; float* shift; float* invstd; float* rmean; float* rvar;
};

// Second stage of the BN statistics + the BatchNorm finalize of one consuming module in ONE kernel (was two): per
// channel, mean = sum_b n_b mean_b / P, then M2 = sum_b M2_b + n_b (mean_b - mean)^2 over the block partials of
// bn_stats_partial_kernel, in fp64 and a fixed order (deterministic; no division inside the loops, unlike the sequential
// Chan merge of bn_stats_final_kernel whose fp64 divide chain cost ~7 us per launch). One 256-thread block per 4 channels.
// Reference semantics: nn.BatchNorm2d in train mode incl. the running-statistics update (lib/models/hourglass.py:18-26).
__global__ void __launch_bounds__(256)
bn_stats_final_finalize_kernel(const double* __restrict__ part, int nblocks, int64_t rows_per_block, int64_t P, int C,
                               BnFinalize fz) {
  // one 256-thread block per 4 channels: every thread takes <= ceil(nblocks/256) partial blocks, so each of the two
  // passes costs about one load round trip + a block reduction (the one-warp-per-channel form walked 19 dependent
  // round trips per pass: 12 us per launch)
  __shared__ double red[8][4];
  __shared__ double s_mu[4];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int c0 = blockIdx.x * 4;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int b = tid; b < nblocks; b += 256) {
    int64_t r0 = (int64_t)b * rows_per_block, r1 = r0 + rows_per_block;
    if (r1 > P) r1 = P;
    const double nb = (double)(r1 > r0 ? r1 - r0 : 0);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (c0 + k < C) acc[k] += nb * part[((size_t)b * C + c0 + k) * 2 + 0];
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double w = warp_sum(acc[k]);
    if (lane == 0) red[wid][k] = w;
  }
  __syncthreads();
  if (tid < 4) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w][tid];
    s_mu[tid] = t / (double)P;
  }
  __syncthreads();
  double mu[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) { mu[k] = s_mu[k]; acc[k] = 0.0; }
  for (int b = tid; b < nblocks; b += 256) {
    int64_t r0 = (int64_t)b * rows_per_block, r1 = r0 + rows_per_block;
    if (r1 > P) r1 = P;
    const double nb = (double)(r1 > r0 ? r1 - r0 : 0);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (c0 + k < C) {
        const double d = part[((size_t)b * C + c0 + k) * 2 + 0] - mu[k];
        acc[k] += part[((size_t)b * C + c0 + k) * 2 + 1] + nb * d * d;
      }
  }
  __syncthreads();   // red[] is reused
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double w = warp_sum(acc[k]);
    if (lane == 0) red[wid][k] = w;
  }
  __syncthreads();
  if (tid < 4 && c0 + tid < C) {
    double m2t = 0.0;
    for (int w = 0; w < 8; ++w) m2t += red[w][tid];
    const int c = c0 + tid;
    const float m = (float)mu[tid], v = (float)(m2t / (double)P);
    fz.mean[c] = m;
    fz.var[c] = v;
    const float invstd = (float)(1.0 / sqrt((double)v + (double)fz.eps));
    const float g = fz.gamma ? fz.gamma[c] : 1.f, b = fz.beta ? fz.beta[c] : 0.f;
    fz.scale[c] = g * invstd;
    fz.shift[c] = b;   // centred form: y = (x - mean) * scale + shift
    if (fz.invstd) fz.invstd[c] = invstd;
    if (fz.rmean) {
      fz.rmean[c] = (1.f - fz.momentum) * fz.rmean[c] + fz.momentum * m;
      const float unbiased = P > 1 ? v * ((float)P / (float)(P - 1)) : v;
      fz.rvar[c] = (1.f - fz.momentum) * fz.rvar[c] + fz.momentum * unbiased;
    }
  }
}

// BatchNorm finalize from per-CTA column SUMS written by a producing kernel's epilogue (conv_tc_h_kernel<.., kStats>:
// part[b][c] = {sum (y - pivot_c), sum (y - pivot_c)^2} over the pixels CTA b wrote): mean = pivot + S1 / P,
// var = S2 / P - (S1 / P)^2, all in fp64, CTAs merged in a fixed order (one warp per channel: lane-strided partial sums,
// then the shuffle tree). Then exactly the finalize of bn_stats_final_finalize_kernel.
__global__ void __launch_bounds__(256)
bn_sums_finalize_kernel(const double* __restrict__ part, int nblocks, const float* __restrict__ pivot, int64_t P, int C,
                        BnFinalize fz) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  double s1 = 0.0, s2 = 0.0;
  for (int b = lane; b < nblocks; b += 32) {
    s1 += part[((size_t)b * C + c) * 2 + 0];
    s2 += part[((size_t)b * C + c) * 2 + 1];
  }
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  if (lane != 0) return;
  const double inv = 1.0 / (double)P;
  const double dm = s1 * inv;
  double vv = s2 * inv - dm * dm;
  if (vv < 0.0) vv = 0.0;
  const float m = (float)((pivot ? (double)pivot[c] : 0.0) + dm), v = (float)vv;
  fz.mean[c] = m;
  fz.var[c] = v;
  const float invstd = (float)(1.0 / sqrt((double)v + (double)fz.eps));
  const float g = fz.gamma ? fz.gamma[c] : 1.f, b = fz.beta ? fz.beta[c] : 0.f;
  fz.scale[c] = g * invstd;
  fz.shift[c] = b;   // centred form: y = (x - mean) * scale + shift
  if (fz.invstd) fz.invstd[c] = invstd;
  if (fz.rmean) {
    fz.rmean[c] = (1.f - fz.momentum) * fz.rmean[c] + fz.momentum * m;
    const float unbiased = P > 1 ? v * ((float)P / (float)(P - 1)) : v;
    fz.rvar[c] = (1.f - fz.momentum) * fz.rvar[c] + fz.momentum * unbiased;
  }
}

// -------------------------------------------------------------------------------------------------
// generic per-channel sum reductions (NV sums per element), deterministic two-stage
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void write_amax_scale(float m, float* amax_scale) {
  // power-of-two scale that puts max|v| into [2^14, 2^15): fp16 hi/lo operands of v * S then keep every element to within
  // 2^-39 of the largest one (csrc/conv_wgmma.cu in_scale). Zero, non-finite and >= 3e38 maxima -> no scaling. S is at most 2^126,
  // so that S and 1/S are both normal floats: maxima below 2^-112 (which would need S >= 2^127, and below 2^-113 an
  // infinite S) get S = 2^126 and land below 2^14, still exact powers of two apart from v.
  float S = 1.f;
  if (m > 0.f && m < 3.0e38f) {
    int e;
    frexpf(m, &e);                              // m = f * 2^e, f in [0.5, 1)
    S = ldexpf(1.f, min(15 - e, 126));          // m * S in [2^14, 2^15) for m >= 2^-112
  }
  amax_scale[0] = S;
  amax_scale[1] = 1.f / S;
}

template <int NV, class F, bool kWide = false>
__global__ void __launch_bounds__(kRedThreads)
channel_reduce_partial_kernel(F f, int64_t P, int C, int L, int R, int64_t rows_per_block,
                              double* __restrict__ part /*[nblocks][NV][C]*/, unsigned int* counter = nullptr,
                              float out_scale = 1.f, float* __restrict__ out = nullptr,
                              float* __restrict__ amax_scale /*[2] or null*/ = nullptr) {
  extern __shared__ double sm[];  // [R][NV][C]
  const int tid = threadIdx.x;
  const int Lc = L < kRedThreads ? L : kRedThreads;   // > 1024 channels: channel lanes in segments of 256 (see bn_stats)
  const int ry = tid / Lc;
  const int64_t row0 = (int64_t)blockIdx.x * rows_per_block;
  int64_t row1 = row0 + rows_per_block;
  if (row1 > P) row1 = P;
  float tmax = 0.f;   // max |v[0]| seen by this thread (used by the fused form's amax output)
  const int cx0 = tid % Lc;
  if (ry < R)
  for (int cx = cx0; kWide ? cx < L : cx == cx0; cx += kRedThreads) {
    double acc[NV][4];
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[k][j] = 0.0;
    float facc[NV][4];
    int inner = 0;
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) facc[k][j] = 0.f;
    for (int64_t r = row0 + ry; r < row1; r += R) {
      float v[NV][4];
      f(r, cx, v);
#pragma unroll
      for (int j = 0; j < 4; ++j) tmax = fmaxf(tmax, fabsf(v[0][j]));
#pragma unroll
      for (int k = 0; k < NV; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) facc[k][j] += v[k][j];
      if (++inner == 16) {  // short fp32 runs, fp64 across runs
        inner = 0;
#pragma unroll
        for (int k = 0; k < NV; ++k)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[k][j] += (double)facc[k][j];
            facc[k][j] = 0.f;
          }
      }
    }
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) sm[((size_t)ry * NV + k) * C + cx * 4 + j] = acc[k][j] + (double)facc[k][j];
  }
  __syncthreads();
  for (int i = tid; i < NV * C; i += kRedThreads) {
    double s = 0.0;
    for (int r = 0; r < R; ++r) s += sm[(size_t)r * NV * C + i];
    part[(size_t)blockIdx.x * NV * C + i] = s;
  }
  // optional max |v| of the first value plane (block maxima live behind the partial sums)
  float* pmax = reinterpret_cast<float*>(part + (size_t)gridDim.x * NV * C);
  if (amax_scale) {
    __shared__ float s_max[kRedThreads / 32];
    float mx = tmax;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((tid & 31) == 0) s_max[tid >> 5] = mx;
    __syncthreads();
    if (tid == 0) {
      float m = s_max[0];
      for (int w = 1; w < kRedThreads / 32; ++w) m = fmaxf(m, s_max[w]);
      pmax[blockIdx.x] = m;
    }
  }
  if (counter == nullptr) return;   // two-stage form (the default): channel_reduce_final_kernel follows
  if (!last_block_ticket(counter)) return;
  const int nblocks = gridDim.x, n = NV * C, lane = tid & 31;
  for (int i0 = (tid >> 5) * 4; i0 < n; i0 += (kRedThreads / 32) * 4) {   // 4 outputs per warp iteration: loads in flight
    double s4[4] = {0.0, 0.0, 0.0, 0.0};
    for (int b = lane; b < nblocks; b += 32) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (i0 + k < n) s4[k] += __ldcg(&part[(size_t)b * n + i0 + k]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double t = warp_sum(s4[k]);
      if (lane == 0 && i0 + k < n) out[i0 + k] = (float)(t * (double)out_scale);
    }
  }
  if (amax_scale && tid < 32) {
    float m = 0.f;
    for (int b = lane; b < nblocks; b += 32) m = fmaxf(m, __ldcg(&pmax[b]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) write_amax_scale(m, amax_scale);
  }
  if (tid == 0) *counter = 0u;
}

// one warp per output value; lanes sum a strided subset of the block partials, then a fixed-order shuffle tree
__global__ void channel_reduce_final_kernel(const double* __restrict__ part, int nblocks, int n /*NV*C*/,
                                            float scale, float* __restrict__ out,
                                            float* __restrict__ amax_scale = nullptr) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (amax_scale && i == n) {   // one extra warp: block maxima -> operand scale
    const float* pmax = reinterpret_cast<const float*>(part + (size_t)nblocks * n);
    float m = 0.f;
    for (int b = lane; b < nblocks; b += 32) m = fmaxf(m, pmax[b]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) write_amax_scale(m, amax_scale);
    return;
  }
  if (i >= n) return;
  double s = 0.0;
  for (int b = lane; b < nblocks; b += 32) s += part[(size_t)b * n + i];
  s = warp_sum(s);
  if (lane == 0) out[i] = (float)(s * (double)scale);
}

struct SumFunctor {
  const float* dy;
  int C;
  __device__ void operator()(int64_t r, int cx, float (&v)[1][4]) const {
    const float4 a = __ldg(reinterpret_cast<const float4*>(dy + r * C) + cx);
    v[0][0] = a.x; v[0][1] = a.y; v[0][2] = a.z; v[0][3] = a.w;
  }
};

struct BnBwdFunctor {
  const float* da; const float* x; const float* mean; const float* invstd; const float* scale; const float* shift;
  int relu; int C;
  __device__ void operator()(int64_t r, int cx, float (&v)[2][4]) const {
    const float4 g = __ldg(reinterpret_cast<const float4*>(da + r * C) + cx);
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x + r * C) + cx);
    const float4 m = __ldg(reinterpret_cast<const float4*>(mean) + cx);
    const float4 is = __ldg(reinterpret_cast<const float4*>(invstd) + cx);
    const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + cx);
    const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + cx);
    const float ge[4] = {g.x, g.y, g.z, g.w}, xe[4] = {xv.x, xv.y, xv.z, xv.w}, me[4] = {m.x, m.y, m.z, m.w},
                ie[4] = {is.x, is.y, is.z, is.w}, se[4] = {sc.x, sc.y, sc.z, sc.w}, he[4] = {sh.x, sh.y, sh.z, sh.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool on = !relu || (fmaf(xe[j] - me[j], se[j], he[j]) > 0.f);
      const float dz = on ? ge[j] : 0.f;
      v[0][j] = dz;
      v[1][j] = dz * ((xe[j] - me[j]) * ie[j]);
    }
  }
};

// BatchNorm-backward apply that ALSO reduces its own output: dx = gamma*invstd*(dz - mean(dz) - xhat*mean(dz*xhat)) is
// written and, in the same pass, summed per channel (= the bias gradient of the convolution that produced x) with its
// max |dx| (= the power-of-two operand scale of that convolution's 3xFP16 data gradient). Replaces bn_bwd_apply +
// channel_sum (one read of dx less, one partial-reduction launch less per conv whose output feeds exactly one BN).
struct BnBwdApplySumFunctor {
  const float* da; const float* x; const float* mean; const float* invstd; const float* scale; const float* shift;
  const float* gamma; const float* sums; float* dx; int relu; int C; float inv_count;
  __device__ void operator()(int64_t r, int cx, float (&v)[1][4]) const {
    const float4 g = __ldg(reinterpret_cast<const float4*>(da + r * C) + cx);
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x + r * C) + cx);
    const float4 m = __ldg(reinterpret_cast<const float4*>(mean) + cx);
    const float4 is = __ldg(reinterpret_cast<const float4*>(invstd) + cx);
    const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + cx);
    const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + cx);
    const float4 gm = gamma ? __ldg(reinterpret_cast<const float4*>(gamma) + cx) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(sums) + cx);
    const float4 s1 = __ldg(reinterpret_cast<const float4*>(sums + C) + cx);
    const float ge[4] = {g.x, g.y, g.z, g.w}, xe[4] = {xv.x, xv.y, xv.z, xv.w}, me[4] = {m.x, m.y, m.z, m.w},
                ie[4] = {is.x, is.y, is.z, is.w}, se[4] = {sc.x, sc.y, sc.z, sc.w}, he[4] = {sh.x, sh.y, sh.z, sh.w},
                ga[4] = {gm.x, gm.y, gm.z, gm.w}, a0[4] = {s0.x, s0.y, s0.z, s0.w}, a1[4] = {s1.x, s1.y, s1.z, s1.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {   // same expression as bn_bwd_apply_kernel: bit-identical dx
      const bool on = !relu || (fmaf(xe[j] - me[j], se[j], he[j]) > 0.f);
      const float dz = on ? ge[j] : 0.f;
      const float xh = (xe[j] - me[j]) * ie[j];
      v[0][j] = ga[j] * ie[j] * (dz - a0[j] * inv_count - xh * a1[j] * inv_count);
    }
    *(reinterpret_cast<float4*>(dx + r * C) + cx) = make_float4(v[0][0], v[0][1], v[0][2], v[0][3]);
  }
};

// -------------------------------------------------------------------------------------------------
// pointwise kernels
// -------------------------------------------------------------------------------------------------
__global__ void affine_act_split_kernel(const float4* __restrict__ x, const float* __restrict__ mean,
                                        const float* __restrict__ scale,
                                        const float* __restrict__ shift, int relu, float4* __restrict__ hi,
                                        float4* __restrict__ lo, int64_t n4, int L, int round,
                                        const float4* __restrict__ residual = nullptr) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = __ldg(x + i);
    if (scale) {
      const int cx = (int)(i % L);
      const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + cx);
      const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + cx);
      const float4 mu = mean ? __ldg(reinterpret_cast<const float4*>(mean) + cx) : make_float4(0.f, 0.f, 0.f, 0.f);
      v.x = fmaf(v.x - mu.x, sc.x, sh.x); v.y = fmaf(v.y - mu.y, sc.y, sh.y);
      v.z = fmaf(v.z - mu.z, sc.z, sh.z); v.w = fmaf(v.w - mu.w, sc.w, sh.w);
    }
    if (residual) {
      const float4 r = __ldg(residual + i);
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (relu) {
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    }
    if (!round) {
      hi[i] = v;
      continue;
    }
    float4 h, l;
    split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y);
    split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}

__global__ void bn_bwd_apply_kernel(const float4* __restrict__ da, const float4* __restrict__ x,
                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                    const float* __restrict__ scale, const float* __restrict__ shift,
                                    const float* __restrict__ gamma, int relu, const float* __restrict__ sums,
                                    int accumulate, float4* __restrict__ dx, int64_t n4, int L, float inv_count) {
  const int C = L * 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    const float4 g = __ldg(da + i);
    const float4 xv = __ldg(x + i);
    const float4 m = __ldg(reinterpret_cast<const float4*>(mean) + cx);
    const float4 is = __ldg(reinterpret_cast<const float4*>(invstd) + cx);
    const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + cx);
    const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + cx);
    const float4 gm = gamma ? __ldg(reinterpret_cast<const float4*>(gamma) + cx) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(sums) + cx);
    const float4 s1 = __ldg(reinterpret_cast<const float4*>(sums + C) + cx);
    const float ge[4] = {g.x, g.y, g.z, g.w}, xe[4] = {xv.x, xv.y, xv.z, xv.w}, me[4] = {m.x, m.y, m.z, m.w},
                ie[4] = {is.x, is.y, is.z, is.w}, se[4] = {sc.x, sc.y, sc.z, sc.w}, he[4] = {sh.x, sh.y, sh.z, sh.w},
                ga[4] = {gm.x, gm.y, gm.z, gm.w}, a0[4] = {s0.x, s0.y, s0.z, s0.w}, a1[4] = {s1.x, s1.y, s1.z, s1.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool on = !relu || (fmaf(xe[j] - me[j], se[j], he[j]) > 0.f);
      const float dz = on ? ge[j] : 0.f;
      const float xh = (xe[j] - me[j]) * ie[j];
      o[j] = ga[j] * ie[j] * (dz - a0[j] * inv_count - xh * a1[j] * inv_count);
    }
    float4 r = make_float4(o[0], o[1], o[2], o[3]);
    if (accumulate) {
      const float4 p = dx[i];
      r.x += p.x; r.y += p.y; r.z += p.z; r.w += p.w;
    }
    dx[i] = r;
  }
}

__global__ void affine_act_bwd_kernel(const float4* __restrict__ da, const float4* __restrict__ x,
                                      const float* __restrict__ mean, const float* __restrict__ scale, const float* __restrict__ shift, int relu,
                                      int accumulate, float4* __restrict__ dx, int64_t n4, int L) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    const float4 g = __ldg(da + i);
    float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f), mu = sh;
    if (scale) {
      sc = __ldg(reinterpret_cast<const float4*>(scale) + cx);
      sh = __ldg(reinterpret_cast<const float4*>(shift) + cx);
      if (mean) mu = __ldg(reinterpret_cast<const float4*>(mean) + cx);
    }
    float4 r = make_float4(g.x * sc.x, g.y * sc.y, g.z * sc.z, g.w * sc.w);
    if (relu) {
      const float4 xv = __ldg(x + i);
      if (!(fmaf(xv.x - mu.x, sc.x, sh.x) > 0.f)) r.x = 0.f;
      if (!(fmaf(xv.y - mu.y, sc.y, sh.y) > 0.f)) r.y = 0.f;
      if (!(fmaf(xv.z - mu.z, sc.z, sh.z) > 0.f)) r.z = 0.f;
      if (!(fmaf(xv.w - mu.w, sc.w, sh.w) > 0.f)) r.w = 0.f;
    }
    if (accumulate) {
      const float4 p = dx[i];
      r.x += p.x; r.y += p.y; r.z += p.z; r.w += p.w;
    }
    dx[i] = r;
  }
}

// T: the activation type (float, or __half for the fp16 activation storage of inference precision "fp16_act": loads
// widen to fp32, stores are one saturating fp16_rn, ld_act4 / st_act4 of common.cuh). Vectors of 4 channels.
template <typename T>
__global__ void maxpool2x2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int B, int Ho, int Wo, int L) {
  const int64_t n = (int64_t)B * Ho * Wo * L;
  const int W = Wo * 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    const int64_t base = (((int64_t)b * Ho * 2 + ho * 2) * W + wo * 2) * L + cx;
    const float4 a = ld_act4(x, base), bb = ld_act4(x, base + L), c = ld_act4(x, base + (int64_t)W * L),
                 d = ld_act4(x, base + (int64_t)W * L + L);
    float4 r;
    r.x = fmaxf(fmaxf(a.x, bb.x), fmaxf(c.x, d.x));
    r.y = fmaxf(fmaxf(a.y, bb.y), fmaxf(c.y, d.y));
    r.z = fmaxf(fmaxf(a.z, bb.z), fmaxf(c.z, d.z));
    r.w = fmaxf(fmaxf(a.w, bb.w), fmaxf(c.w, d.w));
    st_act4(y, i, r);
  }
}

// y = relu?((x - mean) * scale + shift (+ residual)) with fp16 x, residual and y: the expression of
// affine_act_split_kernel's unrounded form, in fp32 from float(x), float(residual).
__global__ void affine_act_f16_kernel(const __half* __restrict__ x, const float* __restrict__ mean,
                                      const float* __restrict__ scale, const float* __restrict__ shift, int relu,
                                      const __half* __restrict__ residual, __half* __restrict__ y, int64_t n4, int L) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = ld_act4(x, i);
    if (scale) {
      const int cx = (int)(i % L);
      const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + cx);
      const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + cx);
      const float4 mu = mean ? __ldg(reinterpret_cast<const float4*>(mean) + cx) : make_float4(0.f, 0.f, 0.f, 0.f);
      v.x = fmaf(v.x - mu.x, sc.x, sh.x); v.y = fmaf(v.y - mu.y, sc.y, sh.y);
      v.z = fmaf(v.z - mu.z, sc.z, sh.z); v.w = fmaf(v.w - mu.w, sc.w, sh.w);
    }
    if (residual) {
      const float4 r = ld_act4(residual, i);
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (relu) {
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    }
    st_act4(y, i, v);
  }
}

// The explicit widening of fp16 activations for the calls that have no half-precision form (CUDA-core convolutions,
// the staged tensor-core kernel): y = float(x), n4 vectors of 4.
__global__ void half_to_float_kernel(const __half* __restrict__ x, float* __restrict__ y, int64_t n4) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
    st_act4(y, i, ld_act4(x, i));
}

// gradient goes to the first maximum in window scan order (row-major), like ATen's max_pool2d backward
__device__ __forceinline__ void pool_route(float a, float b, float c, float d, float g, float& oa, float& ob,
                                           float& oc, float& od) {
  int k = 0;
  float m = a;
  if (b > m) { m = b; k = 1; }
  if (c > m) { m = c; k = 2; }
  if (d > m) { m = d; k = 3; }
  oa = k == 0 ? g : 0.f; ob = k == 1 ? g : 0.f; oc = k == 2 ? g : 0.f; od = k == 3 ? g : 0.f;
}

__global__ void maxpool2x2_bwd_kernel(const float4* __restrict__ x, const float4* __restrict__ dy,
                                      float4* __restrict__ dx, int accumulate, int B, int Ho, int Wo, int L) {
  const int64_t n = (int64_t)B * Ho * Wo * L;
  const int W = Wo * 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    const int64_t base = (((int64_t)b * Ho * 2 + ho * 2) * W + wo * 2) * L + cx;
    const int64_t i00 = base, i01 = base + L, i10 = base + (int64_t)W * L, i11 = i10 + L;
    const float4 a = __ldg(x + i00), bb = __ldg(x + i01), c = __ldg(x + i10), d = __ldg(x + i11);
    const float4 g = __ldg(dy + i);
    float4 ra, rb, rc, rd;
    pool_route(a.x, bb.x, c.x, d.x, g.x, ra.x, rb.x, rc.x, rd.x);
    pool_route(a.y, bb.y, c.y, d.y, g.y, ra.y, rb.y, rc.y, rd.y);
    pool_route(a.z, bb.z, c.z, d.z, g.z, ra.z, rb.z, rc.z, rd.z);
    pool_route(a.w, bb.w, c.w, d.w, g.w, ra.w, rb.w, rc.w, rd.w);
    if (accumulate) {
      float4 p;
      p = dx[i00]; ra.x += p.x; ra.y += p.y; ra.z += p.z; ra.w += p.w;
      p = dx[i01]; rb.x += p.x; rb.y += p.y; rb.z += p.z; rb.w += p.w;
      p = dx[i10]; rc.x += p.x; rc.y += p.y; rc.z += p.z; rc.w += p.w;
      p = dx[i11]; rd.x += p.x; rd.y += p.y; rd.z += p.z; rd.w += p.w;
    }
    dx[i00] = ra; dx[i01] = rb; dx[i10] = rc; dx[i11] = rd;
  }
}

template <typename T>
__global__ void upsample2x_add_kernel(const T* __restrict__ up1, const T* __restrict__ low, T* __restrict__ out, int B,
                                      int H, int W, int L) {
  const int64_t n = (int64_t)B * H * W * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int w = (int)(t % W); t /= W;
    const int h = (int)(t % H);
    const int b = (int)(t / H);
    const float4 a = ld_act4(up1, i);
    const float4 l = ld_act4(low, (((int64_t)b * (H / 2) + h / 2) * (W / 2) + w / 2) * L + cx);
    st_act4(out, i, make_float4(a.x + l.x, a.y + l.y, a.z + l.z, a.w + l.w));
  }
}

__global__ void upsample2x_bwd_kernel(const float4* __restrict__ dout, float4* __restrict__ dlow, int B, int Ho,
                                      int Wo, int L) {  // Ho,Wo = low-res size
  const int64_t n = (int64_t)B * Ho * Wo * L;
  const int W = Wo * 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    const int64_t base = (((int64_t)b * Ho * 2 + ho * 2) * W + wo * 2) * L + cx;
    const float4 a = __ldg(dout + base), bb = __ldg(dout + base + L), c = __ldg(dout + base + (int64_t)W * L),
                 d = __ldg(dout + base + (int64_t)W * L + L);
    dlow[i] = make_float4((a.x + bb.x) + (c.x + d.x), (a.y + bb.y) + (c.y + d.y), (a.z + bb.z) + (c.z + d.z),
                          (a.w + bb.w) + (c.w + d.w));
  }
}

// Stride-2 convolutions on the stride-1 tensor-core kernels: y_s2[ho, wo] = y_s1[2 ho, 2 wo] (k = 3, pad = 1), so the
// forward is the stride-1 convolution followed by this even-position pick, and the backward feeds the stride-1 data /
// weight gradient kernels with dY scattered back to the even positions of a zero tensor.
template <typename T>
__global__ void subsample2_kernel(const T* __restrict__ x, T* __restrict__ y, int B, int Ho, int Wo, int L) {
  const int64_t n = (int64_t)B * Ho * Wo * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int64_t b = t / Ho;
    st_act4(y, i, ld_act4(x, ((b * (2 * Ho) + 2 * ho) * (2 * Wo) + 2 * wo) * L + cx));
  }
}
__global__ void upsample_zero2_kernel(const float4* __restrict__ dy, float4* __restrict__ dx, int B, int Ho, int Wo, int L) {
  const int64_t n = (int64_t)B * (2 * Ho) * (2 * Wo) * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int w = (int)(t % (2 * Wo)); t /= (2 * Wo);
    const int h = (int)(t % (2 * Ho));
    const int64_t b = t / (2 * Ho);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (((w | h) & 1) == 0) v = __ldg(dy + ((b * Ho + (h >> 1)) * Wo + (w >> 1)) * L + cx);
    dx[i] = v;
  }
}

// ---- pose_resnet (reference lib/models/pose_resnet.py:107,230-233): nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
// after the stem, NHWC. Padding counts as -inf; the FIRST maximum in window scan order (kh, then kw) wins, like ATen.
__device__ __forceinline__ bool pool_takes(float v, float m) { return v > m || v != v; }

__global__ void maxpool3x3s2_fwd_kernel(const float4* __restrict__ x, float4* __restrict__ y, int B, int H, int W, int Ho,
                                        int Wo, int L) {
  const int64_t n = (int64_t)B * Ho * Wo * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int64_t b = t / Ho;
    const float ninf = __int_as_float(0xff800000);
    float4 m = make_float4(ninf, ninf, ninf, ninf);
    for (int kh = 0; kh < 3; ++kh) {
      const int h = 2 * ho - 1 + kh;
      if (h < 0 || h >= H) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int w = 2 * wo - 1 + kw;
        if (w < 0 || w >= W) continue;
        const float4 v = __ldg(x + ((b * H + h) * W + w) * L + cx);
        if (pool_takes(v.x, m.x)) m.x = v.x;
        if (pool_takes(v.y, m.y)) m.y = v.y;
        if (pool_takes(v.z, m.z)) m.z = v.z;
        if (pool_takes(v.w, m.w)) m.w = v.w;
      }
    }
    y[i] = m;
  }
}

// Gather form of the backward (windows overlap, so a scatter would need atomics): every input position looks at the up to
// four windows that contain it, re-derives each window's winner from x and takes that window's dY where it IS the winner.
// Deterministic; x is 4 x re-read through L1/L2 (one stem tensor per network).
__global__ void maxpool3x3s2_bwd_kernel(const float4* __restrict__ x, const float4* __restrict__ dy,
                                        float4* __restrict__ dx, int accumulate, int B, int H, int W, int Ho, int Wo,
                                        int L) {
  const int64_t n = (int64_t)B * H * W * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int w = (int)(t % W); t /= W;
    const int h = (int)(t % H);
    const int64_t b = t / H;
    float4 r = accumulate ? dx[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const int ho0 = h >> 1, ho1 = (h + 1) >> 1, wo0 = w >> 1, wo1 = (w + 1) >> 1;   // 2 ho - 1 <= h <= 2 ho + 1
    for (int ho = ho0; ho <= ho1; ++ho) {
      if (ho >= Ho) continue;
      for (int wo = wo0; wo <= wo1; ++wo) {
        if (wo >= Wo) continue;
        const int me = (h - (2 * ho - 1)) * 3 + (w - (2 * wo - 1));   // my position in this window
        const float ninf = __int_as_float(0xff800000);
        float4 m = make_float4(ninf, ninf, ninf, ninf);
        int kx = -1, ky = -1, kz = -1, kw_ = -1;
        for (int kh = 0; kh < 3; ++kh) {
          const int hh = 2 * ho - 1 + kh;
          if (hh < 0 || hh >= H) continue;
          for (int kw = 0; kw < 3; ++kw) {
            const int ww = 2 * wo - 1 + kw;
            if (ww < 0 || ww >= W) continue;
            const float4 v = __ldg(x + ((b * H + hh) * W + ww) * L + cx);
            const int k = kh * 3 + kw;
            if (kx < 0 || pool_takes(v.x, m.x)) { m.x = v.x; kx = k; }
            if (ky < 0 || pool_takes(v.y, m.y)) { m.y = v.y; ky = k; }
            if (kz < 0 || pool_takes(v.z, m.z)) { m.z = v.z; kz = k; }
            if (kw_ < 0 || pool_takes(v.w, m.w)) { m.w = v.w; kw_ = k; }
          }
        }
        const float4 g = __ldg(dy + ((b * Ho + ho) * Wo + wo) * L + cx);
        if (kx == me) r.x += g.x;
        if (ky == me) r.y += g.y;
        if (kz == me) r.z += g.z;
        if (kw_ == me) r.w += g.w;
      }
    }
    dx[i] = r;
  }
}

// ---- ConvTranspose2d(k, stride 2) of pose_resnet's deconv head (pose_resnet.py:176-204) as a stride-1 3x3 convolution to
// 4 x Cout channels (one group of Cout per output parity (rh, rw)) followed by this depth-to-space shuffle:
//   out[b, 2a + rh, 2c + rw, co] = y[b, a, c, (2 rh + rw) Cout + co]
// dir = 0: y [B,H,W,4C] -> out [B,2H,2W,C];  dir = 1: the inverse (= adjoint: a permutation), for the gradient.
__global__ void depth_space2_kernel(const float4* __restrict__ src, float4* __restrict__ dst, int B, int H, int W, int L,
                                    int dir) {
  const int64_t n = (int64_t)B * H * W * 4 * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    // i runs over the depth layout [b][a][c][r][co4]
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int r = (int)(t & 3); t >>= 2;
    const int c = (int)(t % W); t /= W;
    const int a = (int)(t % H);
    const int64_t b = t / H;
    const int64_t j = ((b * (2 * H) + 2 * a + (r >> 1)) * (2 * W) + 2 * c + (r & 1)) * L + cx;
    if (dir == 0) dst[j] = __ldg(src + i);
    else dst[i] = __ldg(src + j);
  }
}

// Weights of that equivalent convolution. Transposed convolution: out[oh] += x[ih] Wd[kh] with oh = 2 ih - pad + kh; for
// oh = 2a + rh and ih = a + dh this is kh = rh + pad - 2 dh, i.e. tap th = dh + 1 of a 3x3 kernel (zero where kh falls
// outside [0, k)). Wd: [Cin][Cout][k][k] (torch layout), W3: OIHW [4 Cout][Cin][3][3].
// dir = 0 builds W3 from Wd; dir = 1 gathers dWd from dW3 (every Wd element appears in exactly one place of W3).
__global__ void deconv_weight_map_kernel(const float* __restrict__ src, float* __restrict__ dst, int Cin, int Cout, int k,
                                         int pad, int dir) {
  if (dir == 0) {
    const int64_t n = (int64_t)4 * Cout * Cin * 9;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
      const int tw = (int)(i % 3), th = (int)((i / 3) % 3);
      int64_t t = i / 9;
      const int ci = (int)(t % Cin); t /= Cin;
      const int co = (int)(t % Cout);
      const int r = (int)(t / Cout);
      const int kh = (r >> 1) + pad - 2 * (th - 1), kw = (r & 1) + pad - 2 * (tw - 1);
      float v = 0.f;
      if (kh >= 0 && kh < k && kw >= 0 && kw < k) v = __ldg(src + (((int64_t)ci * Cout + co) * k + kh) * k + kw);
      dst[i] = v;
    }
  } else {
    const int64_t n = (int64_t)Cin * Cout * k * k;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
      const int kw = (int)(i % k), kh = (int)((i / k) % k);
      int64_t t = i / (k * k);
      const int co = (int)(t % Cout);
      const int ci = (int)(t / Cout);
      const int rh = (kh - pad) & 1, rw = (kw - pad) & 1;
      const int th = (rh + pad - kh) / 2 + 1, tw = (rw + pad - kw) / 2 + 1;   // exact divisions
      dst[i] = __ldg(src + ((((int64_t)(2 * rh + rw) * Cout + co) * Cin + ci) * 3 + th) * 3 + tw);
    }
  }
}

// NCHW <-> NHWC through a 32x33 shared-memory transpose tile (coalesced on both sides)
__global__ void transpose_cs_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols, int flip_w) {
  // in: [batch][rows][cols] -> out: [batch][cols][rows]; flip_w > 0 (NCHW -> NHWC only): cols = H * flip_w pixels and the
  // output pixel of input pixel (h, w) is (h, flip_w - 1 - w) -- the W-mirrored image of the flip test (function.py:220)
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const float* src = in + (size_t)b * rows * cols;
  float* dst = out + (size_t)b * rows * cols;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < rows && c < cols) tile[j][threadIdx.x] = src[(size_t)r * cols + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < rows && c < cols) {
      const int co = flip_w > 0 ? (c / flip_w) * flip_w + (flip_w - 1 - c % flip_w) : c;
      dst[(size_t)co * rows + r] = tile[threadIdx.x][j];
    }
  }
}

__global__ void add_kernel(const float4* __restrict__ a, const float4* __restrict__ b, float4* __restrict__ o,
                           int64_t n4) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 x = __ldg(a + i), y = __ldg(b + i);
    o[i] = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
  }
}

__global__ void weight_prep_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo,
                                   int O, int I, int k, int for_dgrad) {
  const int taps = k * k;
  const int64_t n = (int64_t)O * I * taps;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    // destination index i -> (tap, row, col)
    int64_t t = i;
    int col, row, tap;
    if (!for_dgrad) {  // [tap][O][I]
      col = (int)(t % I); t /= I; row = (int)(t % O); tap = (int)(t / O);
      const float v = w[((size_t)row * I + col) * taps + tap];
      float h, l; split_tf32(v, h, l);
      hi[i] = h; if (lo) lo[i] = l;
    } else {  // [tap'][I][O] with tap' = taps-1-tap (180-degree flip)
      col = (int)(t % O); t /= O; row = (int)(t % I); tap = (int)(t / I);
      const float v = w[((size_t)col * I + row) * taps + (taps - 1 - tap)];
      float h, l; split_tf32(v, h, l);
      hi[i] = h; if (lo) lo[i] = l;
    }
  }
}

// fp16 hi/lo operand form of the weights for the 3xFP16 convolution (conv_wgmma.cu): w * 2^scale_log2 = hi + lo with
// hi = fp16(w'), lo = fp16(w' - hi); the power-of-two pre-scale keeps lo out of the fp16 subnormal range for ordinary
// weight magnitudes (|w| ~ 1e-2) and is undone exactly in the convolution epilogue. Saturates at +-65504.
__global__ void weight_prep_f16_kernel(const float* __restrict__ w, __half* __restrict__ hi, __half* __restrict__ lo,
                                       int O, int I, int k, int for_dgrad, float scale) {
  const int taps = k * k;
  const int64_t n = (int64_t)O * I * taps;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t t = i;
    int col, row, tap;
    float v;
    if (!for_dgrad) {  // [tap][O][I]
      col = (int)(t % I); t /= I; row = (int)(t % O); tap = (int)(t / O);
      v = w[((size_t)row * I + col) * taps + tap];
    } else {           // [tap'][I][O] with tap' = taps-1-tap (180-degree flip)
      col = (int)(t % O); t /= O; row = (int)(t % I); tap = (int)(t / I);
      v = w[((size_t)col * I + row) * taps + (taps - 1 - tap)];
    }
    v = fminf(fmaxf(v * scale, -65504.f), 65504.f);
    const __half h = __float2half_rn(v);
    hi[i] = h;
    if (lo) lo[i] = __float2half_rn(v - __half2float(h));
  }
}

// Forward AND data-gradient operand forms from one read of the weights (one launch per convolution instead of two):
// fwd [tap][O][I], dgrad [taps-1-tap][I][O], both as fp16 hi/lo of w * scale (hi only when the lo pointers are null).
__global__ void weight_prep_f16_both_kernel(const float* __restrict__ w, __half* __restrict__ f_hi,
                                            __half* __restrict__ f_lo, __half* __restrict__ d_hi,
                                            __half* __restrict__ d_lo, int O, int I, int k, float scale) {
  const int taps = k * k;
  const int64_t n = (int64_t)O * I * taps;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    // i indexes the forward layout [tap][o][c]
    const int c = (int)(i % I);
    const int o = (int)((i / I) % O);
    const int tap = (int)(i / ((int64_t)I * O));
    float v = w[((size_t)o * I + c) * taps + tap];
    v = fminf(fmaxf(v * scale, -65504.f), 65504.f);
    const __half h = __float2half_rn(v);
    const __half l = __float2half_rn(v - __half2float(h));
    const size_t di = ((size_t)(taps - 1 - tap) * I + c) * O + o;
    f_hi[i] = h;
    d_hi[di] = h;
    if (f_lo) {
      f_lo[i] = l;
      d_lo[di] = l;
    }
  }
}

// ---- HRNet glue (reference lib/models/pose_hrnet.py:256-263 fuse, :41-57 BasicBlock tail) -------------------
struct FuseTerms {
  const void* t[4];   // float or __half, as the kernel's T
  int shift[4];  // log2 of the nearest-neighbour upsampling factor of each term
  int n;
};

// out[b,h,w,:] = relu?( sum_j t_j[b, h >> s_j, w >> s_j, :] ), summed in term order like the reference's
// `y = y + fuse_layers[i][j](x[j])` loop (in fp32 for both activation types T)
template <typename T>
__global__ void fuse_sum_kernel(FuseTerms ft, int relu, T* __restrict__ out, int B, int H, int W, int L) {
  const int64_t n = (int64_t)B * H * W * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int w = (int)(t % W); t /= W;
    const int h = (int)(t % H);
    const int b = (int)(t / H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < ft.n; ++j) {
      const int s = ft.shift[j];
      const int hs = H >> s, wsz = W >> s;
      const float4 v = ld_act4(static_cast<const T*>(ft.t[j]), (((int64_t)b * hs + (h >> s)) * wsz + (w >> s)) * L + cx);
      if (j == 0) acc = v;
      else { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
    }
    if (relu) { acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f); }
    st_act4(out, i, acc);
  }
}

// dlow[b,ho,wo,:] = sum over the f x f block of dout (f = 1 << shift); Ho,Wo = low-res size
__global__ void upsample_bwd_kernel(const float4* __restrict__ dout, float4* __restrict__ dlow, int shift, int B,
                                    int Ho, int Wo, int L) {
  const int64_t n = (int64_t)B * Ho * Wo * L;
  const int f = 1 << shift;
  const int W = Wo << shift, H = Ho << shift;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = (int)(i % L);
    int64_t t = i / L;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int dy = 0; dy < f; ++dy)
      for (int dx = 0; dx < f; ++dx) {
        const float4 v = __ldg(dout + (((int64_t)b * H + (ho * f + dy)) * W + (wo * f + dx)) * L + cx);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    dlow[i] = acc;
  }
}


// ---- im2col for the few-input-channel stem convs (hourglass 7x7 s2, reference hourglass.py:116; HRNet 3x3 s2,
//      pose_hrnet.py:281): cols[b,ho,wo, (kh*k+kw)*Cin + ci] = x[b, ho*s+kh-p, wo*s+kw-p, ci], zero outside the image and
//      for the K padding. The result is an ordinary NHWC tensor with Kpad channels, so the stem becomes a 1x1
//      convolution on the tensor-core path (forward and weight gradient).
// KK / CIN > 0: compile-time kernel size and channel count (the two stems that exist: 7x7x3 and 3x3x3) -- the four
// divisions / modulos per element become multiply-shifts (the generic form spent most of its 350 us on them).
template <int KK, int CIN>
__global__ void im2col_kernel(const float* __restrict__ x, float4* __restrict__ cols, int B, int H, int W, int Cin_rt,
                              int k_rt, int stride, int pad, int Ho, int Wo, int Kpad) {
  const int Cin = CIN > 0 ? CIN : Cin_rt;
  const int k = KK > 0 ? KK : k_rt;
  const int K = k * k * Cin;
  const int kq = Kpad / 4;
  const int64_t n = (int64_t)B * Ho * Wo * kq;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int k4 = (int)(i % kq) * 4;
    int64_t t = i / kq;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int kk = k4 + j;
      float val = 0.f;
      if (kk < K) {
        const int ci = kk % Cin, tap = kk / Cin;
        const int hi = ho * stride + tap / k - pad, wi = wo * stride + tap % k - pad;
        if (hi >= 0 && hi < H && wi >= 0 && wi < W) val = __ldg(x + (((int64_t)b * H + hi) * W + wi) * Cin + ci);
      }
      v[j] = val;
    }
    cols[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

inline int grid_for(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  const int64_t cap = kNumSMs * 16;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

}  // namespace

// =================================================================================================
// library state: the calling thread's last error, the launch counter and the device's SM count
// =================================================================================================
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int device_sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return kNumSMs;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kNumSMs;
  }
  return n;
}

// =================================================================================================
// launch helpers shared by several entry points
// =================================================================================================
template <int NV, class F>
static int run_channel_reduce_fused(F f, int64_t P, int C, float scale, float* out, float* amax_scale, void* workspace,
                                    size_t ws_bytes, unsigned int* counter, cudaStream_t stream) {
  // Two launches (partial + final). A single-launch "last block finishes" form exists behind counter != null in the
  // kernel, but measured ~2x slower on an earlier GPU (one wave of blocks starves the main pass of memory parallelism, many blocks
  // make the one-CTA tail long), so the counter is accepted for ABI stability and ignored.
  (void)counter;
  FPD_REQUIRE(C % 4 == 0 && C >= 4 && C <= 4096, "channel reduce: C=%d must be a multiple of 4 in [4,4096]", C);
  RedGeom g = red_geom(P, C);
  FPD_REQUIRE(ws_bytes >= (size_t)g.nblocks * NV * C * sizeof(double) + (size_t)g.nblocks * sizeof(float),
              "channel reduce: workspace too small");
  const size_t smem = (size_t)g.R * NV * C * sizeof(double);
  static bool attr = false;
  if (!attr) {
    FPD_CUDA_CHECK(cudaFuncSetAttribute(channel_reduce_partial_kernel<NV, F, false>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    FPD_CUDA_CHECK(cudaFuncSetAttribute(channel_reduce_partial_kernel<NV, F, true>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr = true;
  }
  if (C > 4 * kRedThreads)
    channel_reduce_partial_kernel<NV, F, true><<<g.nblocks, kRedThreads, smem, stream>>>(
        f, P, C, g.L, g.R, g.rows_per_block, (double*)workspace, nullptr, scale, out, amax_scale);
  else
    channel_reduce_partial_kernel<NV, F, false><<<g.nblocks, kRedThreads, smem, stream>>>(
        f, P, C, g.L, g.R, g.rows_per_block, (double*)workspace, nullptr, scale, out, amax_scale);
  FPD_LAUNCH_CHECK();
  const int warps = NV * C + (amax_scale ? 1 : 0);
  channel_reduce_final_kernel<<<(warps * 32 + 127) / 128, 128, 0, stream>>>((const double*)workspace, g.nblocks, NV * C,
                                                                       scale, out, amax_scale);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

template <int NV, class F>
static int run_channel_reduce(F f, int64_t P, int C, float scale, float* out, void* workspace, size_t ws_bytes,
                              cudaStream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && C >= 4 && C <= 4096, "channel reduce: C=%d must be a multiple of 4 in [4,4096]", C);
  RedGeom g = red_geom(P, C);
  FPD_REQUIRE(ws_bytes >= (size_t)g.nblocks * NV * C * sizeof(double), "channel reduce: workspace too small");
  const size_t smem = (size_t)g.R * NV * C * sizeof(double);
  static bool attr = false;
  if (!attr) {
    FPD_CUDA_CHECK(cudaFuncSetAttribute(channel_reduce_partial_kernel<NV, F, false>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    FPD_CUDA_CHECK(cudaFuncSetAttribute(channel_reduce_partial_kernel<NV, F, true>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr = true;
  }
  if (C > 4 * kRedThreads)
    channel_reduce_partial_kernel<NV, F, true><<<g.nblocks, kRedThreads, smem, stream>>>(f, P, C, g.L, g.R,
                                                                                          g.rows_per_block,
                                                                                          (double*)workspace);
  else
    channel_reduce_partial_kernel<NV, F, false><<<g.nblocks, kRedThreads, smem, stream>>>(f, P, C, g.L, g.R,
                                                                                           g.rows_per_block,
                                                                                           (double*)workspace);
  FPD_LAUNCH_CHECK();
  channel_reduce_final_kernel<<<(NV * C * 32 + 127) / 128, 128, 0, stream>>>((const double*)workspace, g.nblocks, NV * C,
                                                                        scale, out);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

// channel counts that are not a multiple of 4 (the 17-joint HRNet head): one CTA per channel, fixed-order tree
__global__ void channel_sum_generic_kernel(const float* __restrict__ dy, int64_t P, int C, float scale,
                                           float* __restrict__ out) {
  const int c = blockIdx.x;
  double s = 0.0;
  for (int64_t r = threadIdx.x; r < P; r += blockDim.x) s += (double)__ldg(dy + r * C + c);
  __shared__ double red[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[i];
    out[c] = (float)(t * (double)scale);
  }
}

template <typename T>
static int fuse_sum_t(const void* const* terms, const int* shifts, int n, int relu, T* out, int B, int H, int W, int C,
                      cudaStream_t stream) {
  FPD_REQUIRE(n >= 1 && n <= 4, "fuse_sum: 1..4 terms, got %d", n);
  FPD_REQUIRE(C % 4 == 0, "fuse_sum: C=%d must be a multiple of 4", C);
  FuseTerms ft{};
  ft.n = n;
  for (int j = 0; j < n; ++j) {
    FPD_REQUIRE(shifts[j] >= 0 && (H % (1 << shifts[j])) == 0 && (W % (1 << shifts[j])) == 0,
                "fuse_sum: term %d upsampling factor does not divide the output size", j);
    ft.t[j] = terms[j];
    ft.shift[j] = shifts[j];
  }
  const int64_t n4 = (int64_t)B * H * W * (C / 4);
  fuse_sum_kernel<<<grid_for(n4, 256), 256, 0, stream>>>(ft, relu, out, B, H, W, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

// fp16-in / fp16-out affine_act, and affine_add_act where residual is not NULL
static int affine_act_f16(const void* x, const float* mean, const float* scale, const float* shift,
                          const void* residual, int relu, void* y, int64_t P, int C, cudaStream_t stream) {
  FPD_REQUIRE(C % 4 == 0, "affine_act_f16: C=%d must be a multiple of 4", C);
  FPD_REQUIRE((scale == nullptr) == (shift == nullptr), "affine_act_f16: scale/shift must come in pairs");
  const int64_t n4 = P * C / 4;
  affine_act_f16_kernel<<<grid_for(n4, 256), 256, 0, stream>>>((const __half*)x, mean, scale, shift, relu,
                                                               (const __half*)residual, (__half*)y, n4, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // namespace fpd

using namespace fpd;

// =================================================================================================
// entry points
// =================================================================================================
extern "C" {

size_t fpd_bn_stats_workspace_bytes(int64_t P, int C) {
  RedGeom g = red_geom(P, C);
  return (size_t)g.nblocks * C * 2 * sizeof(double);
}

int fpd_bn_stats(const float* x, int64_t P, int C, float* mean, float* var_biased, void* workspace, size_t ws_bytes,
                 fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && C >= 4 && C <= 4096, "bn_stats: C=%d must be a multiple of 4 in [4,4096]", C);
  FPD_REQUIRE(P > 0, "bn_stats: empty tensor");
  RedGeom g = red_geom(P, C);
  FPD_REQUIRE(ws_bytes >= (size_t)g.nblocks * C * 2 * sizeof(double), "bn_stats: workspace too small");
  const size_t smem = ((size_t)g.R * C * 2 + g.R) * sizeof(double);
  static bool attr = false;
  if (!attr) {
    FPD_CUDA_CHECK(cudaFuncSetAttribute(bn_stats_partial_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        160 * 1024));
    FPD_CUDA_CHECK(cudaFuncSetAttribute(bn_stats_partial_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        160 * 1024));
    attr = true;
  }
  if (C > 4 * kRedThreads)
    bn_stats_partial_kernel<true><<<g.nblocks, kRedThreads, smem, stream>>>(x, P, C, g.L, g.R, g.rows_per_block,
                                                                            (double*)workspace);
  else
    bn_stats_partial_kernel<false><<<g.nblocks, kRedThreads, smem, stream>>>(x, P, C, g.L, g.R, g.rows_per_block,
                                                                             (double*)workspace);
  FPD_LAUNCH_CHECK();
  bn_stats_final_kernel<<<(C * 32 + 127) / 128, 128, 0, stream>>>((const double*)workspace, g.nblocks,
                                                             g.rows_per_block, P, C, mean, var_biased);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_bn_finalize(const float* mean, const float* var_biased, const float* gamma, const float* beta, float eps,
                    int64_t count, float* scale, float* shift, float* invstd, float* running_mean, float* running_var,
                    float momentum, int C, fpd_stream_t stream) {
  FPD_REQUIRE((running_mean == nullptr) == (running_var == nullptr), "bn_finalize: running stats must come in pairs");
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, stream>>>(mean, var_biased, gamma, beta, eps, count, scale, shift,
                                                          invstd, running_mean, running_var, momentum, C);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_affine_act_split(const float* x, const float* mean, const float* scale, const float* shift, int relu,
                         float* a_hi, float* a_lo, int64_t P, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0, "affine_act_split: C=%d must be a multiple of 4", C);
  FPD_REQUIRE((scale == nullptr) == (shift == nullptr), "affine_act_split: scale/shift must come in pairs");
  const int64_t n4 = P * C / 4;
  affine_act_split_kernel<<<grid_for(n4, 256), 256, 0, stream>>>((const float4*)x, mean, scale, shift, relu,
                                                                 (float4*)a_hi, (float4*)a_lo, n4, C / 4, 1);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_affine_act(const float* x, const float* mean, const float* scale, const float* shift, int relu, float* y,
                   int64_t P, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0, "affine_act: C=%d must be a multiple of 4", C);
  FPD_REQUIRE((scale == nullptr) == (shift == nullptr), "affine_act: scale/shift must come in pairs");
  const int64_t n4 = P * C / 4;
  affine_act_split_kernel<<<grid_for(n4, 256), 256, 0, stream>>>((const float4*)x, mean, scale, shift, relu,
                                                                 (float4*)y, nullptr, n4, C / 4, 0);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_affine_act_f16(const void* x, const float* mean, const float* scale, const float* shift, int relu, void* y,
                       int64_t P, int C, fpd_stream_t stream) {
  return affine_act_f16(x, mean, scale, shift, nullptr, relu, y, P, C, stream);
}

int fpd_affine_add_act_f16(const void* x, const float* mean, const float* scale, const float* shift,
                           const void* residual, int relu, void* y, int64_t P, int C, fpd_stream_t stream) {
  FPD_REQUIRE(residual, "fpd_affine_add_act_f16: NULL residual");
  return affine_act_f16(x, mean, scale, shift, residual, relu, y, P, C, stream);
}

int fpd_half_to_float(const void* x, float* y, int64_t n, fpd_stream_t stream) {
  FPD_REQUIRE(n % 4 == 0, "half_to_float: n=%lld must be a multiple of 4", (long long)n);
  half_to_float_kernel<<<grid_for(n / 4, 256), 256, 0, stream>>>((const __half*)x, y, n / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_maxpool2x2_fwd(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "maxpool2x2: bad shape H=%d W=%d C=%d", H, W, C);
  const int64_t n = (int64_t)B * (H / 2) * (W / 2) * (C / 4);
  maxpool2x2_fwd_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, y, B, H / 2, W / 2, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_maxpool2x2_fwd_f16(const void* x, void* y, int B, int H, int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "maxpool2x2_f16: bad shape H=%d W=%d C=%d", H, W, C);
  const int64_t n = (int64_t)B * (H / 2) * (W / 2) * (C / 4);
  maxpool2x2_fwd_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const __half*)x, (__half*)y, B, H / 2, W / 2, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_maxpool2x2_bwd(const float* x, const float* dy, float* dx, int accumulate, int B, int H, int W, int C,
                       fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "maxpool2x2_bwd: bad shape H=%d W=%d C=%d", H, W, C);
  const int64_t n = (int64_t)B * (H / 2) * (W / 2) * (C / 4);
  maxpool2x2_bwd_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const float4*)x, (const float4*)dy, (float4*)dx,
                                                              accumulate, B, H / 2, W / 2, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_upsample2x_add(const float* up1, const float* low, float* out, int B, int H, int W, int C,
                       fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "upsample2x_add: bad shape H=%d W=%d C=%d", H, W, C);
  const int64_t n = (int64_t)B * H * W * (C / 4);
  upsample2x_add_kernel<<<grid_for(n, 256), 256, 0, stream>>>(up1, low, out, B, H, W, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_upsample2x_add_f16(const void* up1, const void* low, void* out, int B, int H, int W, int C,
                           fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "upsample2x_add_f16: bad shape H=%d W=%d C=%d", H, W, C);
  const int64_t n = (int64_t)B * H * W * (C / 4);
  upsample2x_add_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const __half*)up1, (const __half*)low, (__half*)out, B,
                                                              H, W, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_upsample2x_bwd(const float* dout, float* dlow, int B, int H, int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "upsample2x_bwd: bad shape H=%d W=%d C=%d", H, W, C);
  const int64_t n = (int64_t)B * (H / 2) * (W / 2) * (C / 4);
  upsample2x_bwd_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const float4*)dout, (float4*)dlow, B, H / 2, W / 2,
                                                              C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_subsample2(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "subsample2: need C %% 4 == 0 and even H, W (C=%d H=%d W=%d)", C, H, W);
  const int64_t n = (int64_t)B * (H / 2) * (W / 2) * (C / 4);
  subsample2_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, y, B, H / 2, W / 2, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_subsample2_f16(const void* x, void* y, int B, int H, int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "subsample2_f16: need C %% 4 == 0 and even H, W (C=%d H=%d W=%d)",
              C, H, W);
  const int64_t n = (int64_t)B * (H / 2) * (W / 2) * (C / 4);
  subsample2_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const __half*)x, (__half*)y, B, H / 2, W / 2, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_upsample_zero2(const float* dy, float* dx, int B, int Ho, int Wo, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0, "upsample_zero2: C=%d must be a multiple of 4", C);
  const int64_t n = (int64_t)B * (2 * Ho) * (2 * Wo) * (C / 4);
  upsample_zero2_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const float4*)dy, (float4*)dx, B, Ho, Wo, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_maxpool3x3s2_fwd(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H >= 1 && W >= 1, "maxpool3x3s2: bad shape H=%d W=%d C=%d", H, W, C);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int64_t n = (int64_t)B * Ho * Wo * (C / 4);
  maxpool3x3s2_fwd_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const float4*)x, (float4*)y, B, H, W, Ho, Wo, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_maxpool3x3s2_bwd(const float* x, const float* dy, float* dx, int accumulate, int B, int H, int W, int C,
                         fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && H >= 1 && W >= 1, "maxpool3x3s2_bwd: bad shape H=%d W=%d C=%d", H, W, C);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int64_t n = (int64_t)B * H * W * (C / 4);
  maxpool3x3s2_bwd_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const float4*)x, (const float4*)dy, (float4*)dx,
                                                                accumulate, B, H, W, Ho, Wo, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_depth_space2(const float* src, float* dst, int B, int H, int W, int C, int to_depth, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && C > 0, "depth_space2: C=%d must be a positive multiple of 4", C);
  const int64_t n = (int64_t)B * H * W * 4 * (C / 4);
  depth_space2_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const float4*)src, (float4*)dst, B, H, W, C / 4,
                                                            to_depth ? 1 : 0);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_deconv_weight_map(const float* src, float* dst, int Cin, int Cout, int k, int pad, int to_deconv,
                          fpd_stream_t stream) {
  FPD_REQUIRE((k == 4 && pad == 1) || (k == 3 && pad == 1) || (k == 2 && pad == 0),
              "deconv_weight_map: (kernel, padding) = (%d, %d) is not one of pose_resnet's (4,1) (3,1) (2,0)", k, pad);
  FPD_REQUIRE(src && dst && Cin > 0 && Cout > 0, "deconv_weight_map: bad argument");
  const int64_t n = to_deconv ? (int64_t)Cin * Cout * k * k : (int64_t)4 * Cout * Cin * 9;
  deconv_weight_map_kernel<<<grid_for(n, 256), 256, 0, stream>>>(src, dst, Cin, Cout, k, pad, to_deconv ? 1 : 0);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, fpd_stream_t stream) {
  // per image: [C][HW] -> [HW][C]
  dim3 grid((H * W + 31) / 32, (C + 31) / 32, B), block(32, 8);
  transpose_cs_kernel<<<grid, block, 0, stream>>>(x, y, C, H * W, 0);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_nchw_to_nhwc_flipw(const float* x, float* y, int B, int C, int H, int W, fpd_stream_t stream) {
  dim3 grid((H * W + 31) / 32, (C + 31) / 32, B), block(32, 8);
  transpose_cs_kernel<<<grid, block, 0, stream>>>(x, y, C, H * W, W);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_nhwc_to_nchw(const float* x, float* y, int B, int C, int H, int W, fpd_stream_t stream) {
  dim3 grid((C + 31) / 32, (H * W + 31) / 32, B), block(32, 8);
  transpose_cs_kernel<<<grid, block, 0, stream>>>(x, y, H * W, C, 0);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_add(const float* a, const float* b, float* out, int64_t n, fpd_stream_t stream) {
  FPD_REQUIRE(n % 4 == 0, "add_tensors: n must be a multiple of 4");
  add_kernel<<<grid_for(n / 4, 256), 256, 0, stream>>>((const float4*)a, (const float4*)b, (float4*)out, n / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

size_t fpd_channel_reduce_workspace_bytes(int64_t P, int C) {
  RedGeom g = red_geom(P, C);
  return (size_t)g.nblocks * 2 * C * sizeof(double) + (size_t)g.nblocks * sizeof(float);   // + block maxima (fused form)
}

int fpd_channel_sum(const float* dy, int64_t P, int C, float scale, float* out, void* workspace, size_t ws_bytes,
                    fpd_stream_t stream) {
  if (C % 4 != 0) {
    channel_sum_generic_kernel<<<C, 256, 0, stream>>>(dy, P, C, scale, out);
    FPD_LAUNCH_CHECK();
    return FPD_OK;
  }
  SumFunctor f{dy, C};
  return run_channel_reduce<1>(f, P, C, scale, out, workspace, ws_bytes, stream);
}

int fpd_channel_sum_fused(const float* dy, int64_t P, int C, float scale, float* out, float* amax_scale,
                          void* workspace, size_t ws_bytes, unsigned int* counter, fpd_stream_t stream) {
  SumFunctor f{dy, C};
  return run_channel_reduce_fused<1>(f, P, C, scale, out, amax_scale, workspace, ws_bytes, counter, stream);
}

int fpd_bn_bwd_reduce_fused(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                            const float* shift, int relu, int64_t P, int C, float* sums, void* workspace,
                            size_t ws_bytes, unsigned int* counter, fpd_stream_t stream) {
  BnBwdFunctor f{da, x, mean, invstd, scale, shift, relu, C};
  return run_channel_reduce_fused<2>(f, P, C, 1.f, sums, nullptr, workspace, ws_bytes, counter, stream);
}

int fpd_bn_stats_fused(const float* x, int64_t P, int C, const float* gamma, const float* beta, float eps,
                       float momentum, float* rmean, float* rvar, float* mean, float* var, float* scale, float* shift,
                       float* invstd, void* workspace, size_t ws_bytes, unsigned int* counter, fpd_stream_t stream) {
  (void)counter;   // see run_channel_reduce_fused: two launches (partial + final/finalize) instead of three
  FPD_REQUIRE(C % 4 == 0 && C >= 4 && C <= 4096, "bn_stats_fused: C=%d must be a multiple of 4 in [4,4096]", C);
  FPD_REQUIRE(P > 0 && mean && var && scale && shift, "bn_stats_fused: bad argument");
  FPD_REQUIRE((rmean == nullptr) == (rvar == nullptr), "bn_stats_fused: running stats come in pairs");
  RedGeom g = red_geom(P, C);
  FPD_REQUIRE(ws_bytes >= (size_t)g.nblocks * C * 2 * sizeof(double), "bn_stats_fused: workspace too small");
  const size_t smem = ((size_t)g.R * C * 2 + g.R) * sizeof(double);
  static bool attr = false;
  if (!attr) {
    FPD_CUDA_CHECK(cudaFuncSetAttribute(bn_stats_partial_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        160 * 1024));
    FPD_CUDA_CHECK(cudaFuncSetAttribute(bn_stats_partial_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        160 * 1024));
    attr = true;
  }
  if (C > 4 * kRedThreads)
    bn_stats_partial_kernel<true><<<g.nblocks, kRedThreads, smem, stream>>>(x, P, C, g.L, g.R, g.rows_per_block,
                                                                            (double*)workspace);
  else
    bn_stats_partial_kernel<false><<<g.nblocks, kRedThreads, smem, stream>>>(x, P, C, g.L, g.R, g.rows_per_block,
                                                                             (double*)workspace);
  FPD_LAUNCH_CHECK();
  BnFinalize fz{gamma, beta, eps, momentum, mean, var, scale, shift, invstd, rmean, rvar};
  bn_stats_final_finalize_kernel<<<(C + 3) / 4, 256, 0, stream>>>((const double*)workspace, g.nblocks,
                                                                  g.rows_per_block, P, C, fz);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_bn_finalize_sums(const double* part, int nblocks, const float* pivot, int64_t P, int C, const float* gamma,
                         const float* beta, float eps, float momentum, float* rmean, float* rvar, float* mean,
                         float* var, float* scale, float* shift, float* invstd, fpd_stream_t stream) {
  FPD_REQUIRE(part && nblocks > 0 && P > 0 && C > 0 && mean && var && scale && shift, "bn_finalize_sums: bad argument");
  FPD_REQUIRE((rmean == nullptr) == (rvar == nullptr), "bn_finalize_sums: running stats come in pairs");
  BnFinalize fz{gamma, beta, eps, momentum, mean, var, scale, shift, invstd, rmean, rvar};
  bn_sums_finalize_kernel<<<(C * 32 + 255) / 256, 256, 0, stream>>>(part, nblocks, pivot, P, C, fz);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_bn_bwd_reduce(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                      const float* shift, int relu, int64_t P, int C, float* sums, void* workspace, size_t ws_bytes,
                      fpd_stream_t stream) {
  BnBwdFunctor f{da, x, mean, invstd, scale, shift, relu, C};
  return run_channel_reduce<2>(f, P, C, 1.f, sums, workspace, ws_bytes, stream);
}

int fpd_bn_bwd_apply(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                     const float* shift, const float* gamma, int relu, const float* sums, int accumulate, float* dx,
                     int64_t P, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0, "bn_bwd_apply: C=%d must be a multiple of 4", C);
  const int64_t n4 = P * C / 4;
  bn_bwd_apply_kernel<<<grid_for(n4, 256), 256, 0, stream>>>((const float4*)da, (const float4*)x, mean, invstd,
                                                             scale, shift, gamma, relu, sums, accumulate,
                                                             (float4*)dx, n4, C / 4, 1.f / (float)P);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_bn_bwd_apply_sum(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                         const float* shift, const float* gamma, int relu, const float* sums, float* dx, float* dx_sum,
                         float* amax_scale, int64_t P, int C, void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  FPD_REQUIRE(da && x && mean && invstd && scale && shift && sums && dx && dx_sum, "bn_bwd_apply_sum: null pointer");
  BnBwdApplySumFunctor f{da, x, mean, invstd, scale, shift, gamma, sums, dx, relu, C, 1.f / (float)P};
  return run_channel_reduce_fused<1>(f, P, C, 1.f, dx_sum, amax_scale, workspace, ws_bytes, nullptr, stream);
}

int fpd_affine_act_bwd(const float* da, const float* x, const float* mean, const float* scale, const float* shift,
                       int relu, int accumulate, float* dx, int64_t P, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0, "affine_act_bwd: C=%d must be a multiple of 4", C);
  const int64_t n4 = P * C / 4;
  affine_act_bwd_kernel<<<grid_for(n4, 256), 256, 0, stream>>>((const float4*)da, (const float4*)x, mean, scale,
                                                               shift, relu, accumulate, (float4*)dx, n4, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_weight_prep(const float* w_oihw, float* w_hi, float* w_lo, int O, int I, int k, int for_dgrad,
                    fpd_stream_t stream) {
  const int64_t n = (int64_t)O * I * k * k;
  weight_prep_kernel<<<grid_for(n, 256), 256, 0, stream>>>(w_oihw, w_hi, w_lo, O, I, k, for_dgrad);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_weight_prep_f16(const float* w_oihw, void* w_hi, void* w_lo, int O, int I, int k, int for_dgrad,
                        fpd_stream_t stream) {
  const int64_t n = (int64_t)O * I * k * k;
  weight_prep_f16_kernel<<<grid_for(n, 256), 256, 0, stream>>>(w_oihw, (__half*)w_hi, (__half*)w_lo, O, I, k, for_dgrad,
                                                               (float)(1 << kF16WeightScaleLog2));
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_weight_prep_f16_both(const float* w_oihw, void* f_hi, void* f_lo, void* d_hi, void* d_lo, int O, int I, int k,
                             fpd_stream_t stream) {
  FPD_REQUIRE(w_oihw && f_hi && d_hi, "weight_prep_f16_both: null operand");
  FPD_REQUIRE((f_lo == nullptr) == (d_lo == nullptr), "weight_prep_f16_both: f_lo and d_lo are both set or both NULL");
  const int64_t n = (int64_t)O * I * k * k;
  weight_prep_f16_both_kernel<<<grid_for(n, 256), 256, 0, stream>>>(w_oihw, (__half*)f_hi, (__half*)f_lo, (__half*)d_hi,
                                                                    (__half*)d_lo, O, I, k,
                                                                    (float)(1 << kF16WeightScaleLog2));
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_affine_add_act(const float* x, const float* mean, const float* scale, const float* shift, const float* residual,
                       int relu, float* y, int64_t P, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0, "affine_add_act: C=%d must be a multiple of 4", C);
  FPD_REQUIRE((scale == nullptr) == (shift == nullptr), "affine_add_act: scale/shift must come in pairs");
  const int64_t n4 = P * C / 4;
  affine_act_split_kernel<<<grid_for(n4, 256), 256, 0, stream>>>((const float4*)x, mean, scale, shift, relu,
                                                                 (float4*)y, nullptr, n4, C / 4, 0,
                                                                 (const float4*)residual);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_fuse_sum(const float* const* terms, const int* shifts, int n, int relu, float* out, int B, int H, int W, int C,
                 fpd_stream_t stream) {
  FPD_REQUIRE(terms && shifts, "fpd_fuse_sum: NULL term table");
  return fuse_sum_t(reinterpret_cast<const void* const*>(terms), shifts, n, relu, out, B, H, W, C, stream);
}

int fpd_fuse_sum_f16(const void* const* terms, const int* shifts, int n, int relu, void* out, int B, int H, int W,
                     int C, fpd_stream_t stream) {
  FPD_REQUIRE(terms && shifts, "fpd_fuse_sum_f16: NULL term table");
  return fuse_sum_t(terms, shifts, n, relu, (__half*)out, B, H, W, C, stream);
}

int fpd_upsample_bwd(const float* dout, float* dlow, int shift, int B, int H, int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(C % 4 == 0 && shift >= 0 && H % (1 << shift) == 0 && W % (1 << shift) == 0,
              "upsample_bwd: bad shape H=%d W=%d C=%d shift=%d", H, W, C, shift);
  const int Ho = H >> shift, Wo = W >> shift;
  const int64_t n = (int64_t)B * Ho * Wo * (C / 4);
  upsample_bwd_kernel<<<grid_for(n, 256), 256, 0, stream>>>((const float4*)dout, (float4*)dlow, shift, B, Ho, Wo, C / 4);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_im2col(const float* x, float* cols, int B, int H, int W, int Cin, int k, int stride, int pad, int Kpad,
               fpd_stream_t stream) {
  FPD_REQUIRE(Kpad % 4 == 0 && Kpad >= k * k * Cin, "im2col: Kpad=%d must be a multiple of 4 and >= k*k*Cin", Kpad);
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const int64_t n = (int64_t)B * Ho * Wo * (Kpad / 4);
  if (k == 7 && Cin == 3)
    im2col_kernel<7, 3><<<grid_for(n, 256), 256, 0, stream>>>(x, (float4*)cols, B, H, W, Cin, k, stride, pad, Ho, Wo, Kpad);
  else if (k == 3 && Cin == 3)
    im2col_kernel<3, 3><<<grid_for(n, 256), 256, 0, stream>>>(x, (float4*)cols, B, H, W, Cin, k, stride, pad, Ho, Wo, Kpad);
  else
    im2col_kernel<0, 0><<<grid_for(n, 256), 256, 0, stream>>>(x, (float4*)cols, B, H, W, Cin, k, stride, pad, Ho, Wo, Kpad);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

const char* fpd_last_error(void) { return g_err; }
int fpd_version(void) { return 100; }
int fpd_sm_count(void) { return device_sm_count(); }
long long fpd_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
