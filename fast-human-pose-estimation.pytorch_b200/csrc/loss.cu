// loss.cu -- fused Fast-Pose-Distillation loss + gradient in ONE pass over the heat-maps.
//
// Reference semantics (lib/core/loss.py:21-39 JointsMSELoss, lib/core/function.py:127-134 fpd_train):
//   L(out, ref) = 1/J * sum_j 0.5 * mean_{b,hw} ( w[b,j]*out - w[b,j]*ref )^2
//               = 0.5/(J*B*hw) * sum (w*(out-ref))^2                      (weights enter squared)
//   pose = sum_s L(out_s, target);  kd = sum_s L(out_s, teacher_last);  loss = (1-a)*pose + a*kd
//   dloss/dout_s = w^2 * ((1-a)*(out_s-target) + a*(out_s-teacher)) / (J*B*hw)
// The reference launches ~6 tiny kernels per joint per stack per term (~770 launches for the 4-stack
// student); here every stack's loss terms and gradient come out of one HBM pass, with a deterministic
// two-stage fp64 reduction (no atomics).
//
// Layouts: student / teacher heat-maps are the network-internal NHWC [B,h,w,J]; `target` is the caller's
// NCHW [B,J,h,w] tensor (lib/dataset/JointsDataset.py target layout), staged through shared memory.
#include <cooperative_groups.h>

#include "common.cuh"

namespace fpd {
namespace {

constexpr int kPix = 64;       // pixels per block
constexpr int kThreads = 256;
constexpr int kMaxStacks = 8;

struct StackPtrs {
  const float* out[kMaxStacks];
  float* grad[kMaxStacks];
};

// KD_W: the kd term has its own weights kw (the pose term keeps tw). Where kw == tw the gradient is the expression of
// the single-weight form, so equal weights give that form's bits.
template <bool KD_W>
__global__ void __launch_bounds__(kThreads)
fpd_loss_kernel(StackPtrs sp, int S, const float* __restrict__ target, const float* __restrict__ teacher,
                const float* __restrict__ tw, const float* __restrict__ kw, float alpha, float inv_norm,
                float grad_scale, int B, int J, int hw, double* __restrict__ part /*[nblocks][2]*/) {
  extern __shared__ float tgt[];  // [J][kPix+1]
  const int blocks_per_img = hw / kPix;
  const int b = blockIdx.x / blocks_per_img;
  const int p0 = (blockIdx.x % blocks_per_img) * kPix;
  for (int i = threadIdx.x; i < J * kPix; i += kThreads) {
    const int j = i / kPix, px = i % kPix;
    tgt[j * (kPix + 1) + px] = __ldg(target + ((int64_t)b * J + j) * hw + p0 + px);
  }
  __syncthreads();
  float pose = 0.f, kd = 0.f;
  const int64_t base = ((int64_t)b * hw + p0) * J;
  for (int i = threadIdx.x; i < J * kPix; i += kThreads) {
    const int px = i / J, j = i % J;
    const float w = __ldg(tw + b * J + j);
    const float w2 = w * w;
    const float k = KD_W ? __ldg(kw + b * J + j) : w;
    const float k2 = k * k;
    const float g = tgt[j * (kPix + 1) + px];
    const float t = teacher ? __ldg(teacher + base + i) : 0.f;
    for (int s = 0; s < S; ++s) {
      const float o = __ldg(sp.out[s] + base + i);
      const float dp = o - g;
      const float dk = o - t;
      pose = fmaf(w2 * dp, dp, pose);
      if (teacher) kd = fmaf(k2 * dk, dk, kd);
      if (sp.grad[s]) {
        if (!KD_W || k == w) {
          const float gr = teacher ? ((1.f - alpha) * dp + alpha * dk) : dp;
          sp.grad[s][base + i] = grad_scale * w2 * gr * inv_norm;
        } else {
          sp.grad[s][base + i] = grad_scale * ((1.f - alpha) * w2 * dp + alpha * k2 * dk) * inv_norm;
        }
      }
    }
  }
  __shared__ double red[2][kThreads / 32];
  double dpose = warp_sum((double)pose), dkd = warp_sum((double)kd);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { red[0][wid] = dpose; red[1][wid] = dkd; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, c = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) { a += red[0][i]; c += red[1][i]; }
    part[(size_t)blockIdx.x * 2 + 0] = a;
    part[(size_t)blockIdx.x * 2 + 1] = c;
  }
}

__global__ void fpd_loss_final_kernel(const double* __restrict__ part, int nblocks, double half_inv_norm,
                                      float alpha, int has_teacher, float* __restrict__ losses) {
  __shared__ double red[2][8];
  double a = 0.0, c = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) { a += part[(size_t)i * 2]; c += part[(size_t)i * 2 + 1]; }
  a = warp_sum(a); c = warp_sum(c);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { red[0][wid] = a; red[1][wid] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sc = 0.0;
    for (int i = 0; i < (int)(blockDim.x / 32); ++i) { sa += red[0][i]; sc += red[1][i]; }
    const double pose = sa * half_inv_norm, kd = sc * half_inv_norm;
    losses[0] = (float)pose;
    losses[1] = (float)kd;
    losses[2] = has_teacher ? (float)((1.0 - (double)alpha) * pose + (double)alpha * kd) : (float)pose;
  }
}

// single-term JointsMSELoss on NCHW tensors (the reference module's own signature)
__global__ void __launch_bounds__(kThreads)
joints_mse_kernel(const float* __restrict__ out, const float* __restrict__ target, const float* __restrict__ tw,
                  float inv_norm, float* __restrict__ grad, int64_t n, int hw, double* __restrict__ part) {
  float acc = 0.f;
  double dacc = 0.0;
  int inner = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float w = tw ? __ldg(tw + i / hw) : 1.f;
    const float d = __ldg(out + i) - __ldg(target + i);
    acc = fmaf(w * w * d, d, acc);
    if (grad) grad[i] = w * w * d * inv_norm;
    if (++inner == 32) { dacc += (double)acc; acc = 0.f; inner = 0; }
  }
  dacc += (double)acc;
  __shared__ double red[kThreads / 32];
  dacc = warp_sum(dacc);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = dacc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) s += red[i];
    part[(size_t)blockIdx.x * 2] = s;
    part[(size_t)blockIdx.x * 2 + 1] = 0.0;
  }
}

}  // namespace
}  // namespace fpd

using namespace fpd;

extern "C" {

size_t fpd_loss_workspace_bytes(int B, int J, int h, int w) {
  const int64_t hw = (int64_t)h * w;
  int64_t nblocks = (int64_t)B * ((hw + kPix - 1) / kPix);
  if (nblocks < 2048) nblocks = 2048;
  return (size_t)nblocks * 2 * sizeof(double);
}

}  // extern "C"

namespace fpd {
namespace {

// kw: the kd term's weights, or NULL for tw (the single-weight kernel)
int loss_mse_launch(const float* const* outs, int S, const float* target_nchw, const float* teacher_nhwc,
                    const float* tw, const float* kw, float alpha, float* const* grads, float grad_scale, float* losses,
                    int B, int J, int h, int w, void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  FPD_REQUIRE(outs != nullptr, "fpd_loss_fused: outs_host is NULL");
  const int hw = h * w;
  FPD_REQUIRE(S >= 1 && S <= kMaxStacks, "fpd_loss: S=%d out of range [1,%d]", S, kMaxStacks);
  FPD_REQUIRE(hw % kPix == 0, "fpd_loss: h*w=%d must be a multiple of %d", hw, kPix);
  FPD_REQUIRE(J >= 1 && J <= 64, "fpd_loss: J=%d out of range", J);
  FPD_REQUIRE(tw != nullptr, "fpd_loss: target_weight is required (pass ones for use_target_weight=False)");
  const int nblocks = B * (hw / kPix);
  FPD_REQUIRE(ws_bytes >= (size_t)nblocks * 2 * sizeof(double), "fpd_loss: workspace too small");
  StackPtrs sp{};
  for (int s = 0; s < S; ++s) {
    sp.out[s] = outs[s];
    sp.grad[s] = grads ? grads[s] : nullptr;
  }
  const double norm = (double)J * (double)B * (double)hw;
  const size_t smem = (size_t)J * (kPix + 1) * sizeof(float);
  if (kw)
    fpd_loss_kernel<true><<<nblocks, kThreads, smem, stream>>>(sp, S, target_nchw, teacher_nhwc, tw, kw, alpha,
                                                                (float)(1.0 / norm), grad_scale, B, J, hw,
                                                                (double*)workspace);
  else
    fpd_loss_kernel<false><<<nblocks, kThreads, smem, stream>>>(sp, S, target_nchw, teacher_nhwc, tw, nullptr, alpha,
                                                                 (float)(1.0 / norm), grad_scale, B, J, hw,
                                                                 (double*)workspace);
  FPD_LAUNCH_CHECK();
  fpd_loss_final_kernel<<<1, 256, 0, stream>>>((const double*)workspace, nblocks, 0.5 / norm, alpha,
                                               teacher_nhwc != nullptr, losses);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // namespace
}  // namespace fpd

extern "C" {

int fpd_loss_fused(const float* const* outs, int S, const float* target_nchw, const float* teacher_nhwc, const float* tw,
                   float alpha, float* const* grads, float grad_scale, float* losses, int B, int J, int h, int w,
                   void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  return loss_mse_launch(outs, S, target_nchw, teacher_nhwc, tw, nullptr, alpha, grads, grad_scale, losses, B, J, h, w,
                         workspace, ws_bytes, stream);
}

int fpd_joints_mse(const float* out_nchw, const float* target_nchw, const float* tw, float* loss, float* grad_out, int B,
                   int J, int hw, void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  const int64_t n = (int64_t)B * J * hw;
  int nblocks = (int)((n + kThreads * 8 - 1) / (kThreads * 8));
  if (nblocks > 2048) nblocks = 2048;
  if (nblocks < 1) nblocks = 1;
  FPD_REQUIRE(ws_bytes >= (size_t)nblocks * 2 * sizeof(double), "joints_mse: workspace too small");
  const double norm = (double)J * (double)B * (double)hw;
  joints_mse_kernel<<<nblocks, kThreads, 0, stream>>>(out_nchw, target_nchw, tw, (float)(1.0 / norm), grad_out, n, hw,
                                                      (double*)workspace);
  FPD_LAUNCH_CHECK();
  fpd_loss_final_kernel<<<1, 256, 0, stream>>>((const double*)workspace, nblocks, 0.5 / norm, 0.f, 0, loss);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Online hard keypoint mining (reference lib/core/loss.py:42-87, JointsOHKMMSELoss):
//   l[b,j] = 0.5 * mean_p (w[b,j]*o - w[b,j]*g)^2 ;  L = 1/B * sum_b 1/topk * sum_{j in S_b} l[b,j]
//   S_b = the topk joints with the largest fp32-rounded l[b,.]; on exact ties the lower joint index wins
//   dL/do = [j in S_b] * w^2 * (o - g) / (B * topk * hw)
// The gradient depends on a per-sample selection, so the heat-maps are read twice: (1) per-(stack, sample, joint)
// sums of squares, fp32 partials added in fp64 in a fixed order; (2) one warp per (stack, term, sample) ranks the J
// values and turns the selection into per-(s, b, j) gradient coefficients (zero for joints left out); (3) one pass
// writes every gradient element. A topk of 0 makes a term plain JointsMSELoss (coefficient 1/(J*B*hw) for every
// joint), so the fused FPD form covers all four pose / kd combinations. No floating-point atomics: deterministic and
// graph-capturable.
//
// Workspace: part double [B][nch][S][2][J] | contrib double [B][S][2] | coef float [B][S][2][J]
// (nch = 64-pixel chunks per sample on the fused NHWC form, 1 on the NCHW module form).
namespace fpd {
namespace {

constexpr int kMaxJ = 64;

// a ranks ahead of b: larger value first (NaN above everything, as torch.topk orders it), then the lower index
__device__ __forceinline__ bool ohkm_ahead(float a, int ia, float b, int ib) {
  const bool an = isnan(a), bn = isnan(b);
  if (an || bn) return an && (!bn || ia < ib);
  return a > b || (a == b && ia < ib);
}

// Bit j set <=> joint j is among the k first of v[0..J) in ohkm_ahead order. One warp, J <= 64; every lane gets the
// same mask. Ranking by counting is a total order, so exactly min(k, J) bits are set.
__device__ __forceinline__ unsigned long long warp_topk_mask(const float* v, int J, int k, int lane) {
  bool sel[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int j = lane + 32 * h;
    sel[h] = false;
    if (j < J) {
      const float x = v[j];
      int rank = 0;
      for (int jj = 0; jj < J; ++jj) rank += ohkm_ahead(v[jj], jj, x, j) ? 1 : 0;
      sel[h] = rank < k;
    }
  }
  const unsigned lo = __ballot_sync(0xffffffffu, sel[0]);
  const unsigned hi = __ballot_sync(0xffffffffu, sel[1]);
  return (unsigned long long)lo | ((unsigned long long)hi << 32);
}

// (1) fused form: per (sample, 64-pixel chunk) block, sums over the chunk of (o_s - g)^2 and (o_s - t)^2 for every
// (s, j). Thread (pl, j) owns joint j and pixels pl, pl + L, ... (L = pixel lanes), so the reduction needs no atomics.
__global__ void __launch_bounds__(kThreads)
ohkm_sums_nhwc_kernel(StackPtrs sp, int S, const float* __restrict__ target, const float* __restrict__ teacher, int J,
                      int hw, double* __restrict__ part) {
  extern __shared__ float sm[];
  float* tgt = sm;                        // [J][kPix+1]
  float* red = sm + J * (kPix + 1);       // [S*2][L*J]
  const int nch = hw / kPix;
  const int b = blockIdx.x / nch;
  const int p0 = (blockIdx.x % nch) * kPix;
  for (int i = threadIdx.x; i < J * kPix; i += kThreads) {
    const int j = i / kPix, px = i % kPix;
    tgt[j * (kPix + 1) + px] = __ldg(target + ((int64_t)b * J + j) * hw + p0 + px);
  }
  __syncthreads();
  const int L = min(kPix, kThreads / J);
  const int active = L * J;
  if (threadIdx.x < active) {
    const int j = threadIdx.x % J, pl = threadIdx.x / J;
    float ap[kMaxStacks], ak[kMaxStacks];
#pragma unroll
    for (int s = 0; s < kMaxStacks; ++s) ap[s] = ak[s] = 0.f;
    const int64_t base = ((int64_t)b * hw + p0) * J + j;
    for (int px = pl; px < kPix; px += L) {
      const int64_t e = base + (int64_t)px * J;
      const float g = tgt[j * (kPix + 1) + px];
      const float t = teacher ? __ldg(teacher + e) : 0.f;
#pragma unroll
      for (int s = 0; s < kMaxStacks; ++s) {
        if (s < S) {
          const float o = __ldg(sp.out[s] + e);
          const float dp = o - g, dk = o - t;
          ap[s] = fmaf(dp, dp, ap[s]);
          ak[s] = fmaf(dk, dk, ak[s]);
        }
      }
    }
#pragma unroll
    for (int s = 0; s < kMaxStacks; ++s) {
      if (s < S) {
        red[(2 * s) * active + threadIdx.x] = ap[s];
        red[(2 * s + 1) * active + threadIdx.x] = teacher ? ak[s] : 0.f;
      }
    }
  }
  __syncthreads();
  double* dst = part + (size_t)blockIdx.x * S * 2 * J;
  for (int q = threadIdx.x; q < S * 2 * J; q += kThreads) {
    const int st = q / J, j = q % J;
    double acc = 0.0;
    for (int pl = 0; pl < L; ++pl) acc += (double)red[st * active + pl * J + j];
    dst[q] = acc;
  }
}

// (1) module form: one block per NCHW (b, j) map; part[b][0][0][0][j] = sum_p (o - g)^2, the kd slot is zero
__global__ void __launch_bounds__(kThreads)
ohkm_sums_nchw_kernel(const float* __restrict__ out, const float* __restrict__ target, int J, int hw,
                      double* __restrict__ part) {
  const int b = blockIdx.x / J, j = blockIdx.x % J;
  const float* o = out + (int64_t)blockIdx.x * hw;
  const float* g = target + (int64_t)blockIdx.x * hw;
  float acc = 0.f;
  double dacc = 0.0;
  int inner = 0;
  for (int p = threadIdx.x; p < hw; p += kThreads) {
    const float d = __ldg(o + p) - __ldg(g + p);
    acc = fmaf(d, d, acc);
    if (++inner == 32) { dacc += (double)acc; acc = 0.f; inner = 0; }
  }
  dacc += (double)acc;
  __shared__ double red[kThreads / 32];
  dacc = warp_sum(dacc);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = dacc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) s += red[i];
    part[(size_t)b * 2 * J + j] = s;
    part[(size_t)b * 2 * J + J + j] = 0.0;
  }
}

// (2) one block per sample: per-(s, term, j) losses l = 0.5 * w^2 * sum / hw, then one warp per (s, term) selects and
// writes the sample's share of the term (selected sum / topk, or sum / J for plain MSE) and the gradient
// coefficients grad_scale * {1-alpha | alpha | 1} * w^2 / (B * {topk | J} * hw) of the selected joints. w is tw for the
// pose term and kw for the kd term.
__global__ void __launch_bounds__(kThreads)
ohkm_select_kernel(const double* __restrict__ part, int nch, int S, int J, int hw, int B, const float* __restrict__ tw,
                   const float* __restrict__ kw, int has_teacher, int pose_topk, int kd_topk, float alpha, float grad_scale,
                   double* __restrict__ contrib, float* __restrict__ coef) {
  __shared__ double ld[kMaxStacks * 2][kMaxJ];
  __shared__ float lf[kMaxStacks * 2][kMaxJ];
  const int b = blockIdx.x;
  const int SJ2 = S * 2 * J;
  for (int q = threadIdx.x; q < SJ2; q += kThreads) {
    const int st = q / J, j = q % J;
    double acc = 0.0;
    for (int c = 0; c < nch; ++c) acc += part[((size_t)b * nch + c) * SJ2 + q];
    const float* wt = (st & 1) ? kw : tw;
    const double w = wt ? (double)__ldg(wt + (size_t)b * J + j) : 1.0;
    const double l = 0.5 * (w * w) * acc / (double)hw;
    ld[st][j] = l;
    lf[st][j] = (float)l;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int st = wid; st < S * 2; st += kThreads / 32) {
    const int s = st >> 1, term = st & 1;
    float* cf = coef + (((size_t)b * S + s) * 2 + term) * J;
    double* ct = contrib + ((size_t)b * S + s) * 2 + term;
    if (term == 1 && !has_teacher) {
      for (int j = lane; j < J; j += 32) cf[j] = 0.f;
      if (lane == 0) *ct = 0.0;
      continue;
    }
    const int k = term ? kd_topk : pose_topk;
    const unsigned long long mask = k > 0 ? warp_topk_mask(lf[st], J, k, lane)
                                          : (J == 64 ? ~0ull : ((1ull << J) - 1ull));
    const int cnt = k > 0 ? k : J;
    const double factor = has_teacher ? (term ? (double)alpha : 1.0 - (double)alpha) : 1.0;
    const double scale = (double)grad_scale * factor / ((double)B * (double)cnt * (double)hw);
    const float* wt = term ? kw : tw;
    for (int j = lane; j < J; j += 32) {
      const double w = wt ? (double)__ldg(wt + (size_t)b * J + j) : 1.0;
      cf[j] = ((mask >> j) & 1ull) ? (float)(scale * w * w) : 0.f;
    }
    if (lane == 0) {
      double sum = 0.0;
      for (int j = 0; j < J; ++j)
        if ((mask >> j) & 1ull) sum += ld[st][j];
      *ct = sum / (double)cnt;
    }
  }
}

// (2') losses[3] = {pose, kd, total}: term_s = 1/B sum_b share[b][s][term], pose / kd = sum over stacks in order
__global__ void ohkm_final_kernel(const double* __restrict__ contrib, int B, int S, int has_teacher, float alpha,
                                  float* __restrict__ losses) {
  __shared__ double crit[kMaxStacks * 2];
  const int st = threadIdx.x;
  if (st < S * 2) {
    double a = 0.0;
    for (int b = 0; b < B; ++b) a += contrib[(size_t)b * S * 2 + st];
    crit[st] = a / (double)B;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double pose = 0.0, kd = 0.0;
    for (int s = 0; s < S; ++s) { pose += crit[2 * s]; kd += crit[2 * s + 1]; }
    losses[0] = (float)pose;
    losses[1] = (float)kd;
    losses[2] = has_teacher ? (float)((1.0 - (double)alpha) * pose + (double)alpha * kd) : (float)pose;
  }
}

// (3) fused form: grad_s = c_pose[s,b,j] * (o_s - g) + c_kd[s,b,j] * (o_s - t) for every element
__global__ void __launch_bounds__(kThreads)
ohkm_grad_nhwc_kernel(StackPtrs sp, int S, const float* __restrict__ target, const float* __restrict__ teacher,
                      const float* __restrict__ coef, int J, int hw) {
  extern __shared__ float sm[];
  float* tgt = sm;                        // [J][kPix+1]
  float* cs = sm + J * (kPix + 1);        // [S][2][J] of this sample
  const int nch = hw / kPix;
  const int b = blockIdx.x / nch;
  const int p0 = (blockIdx.x % nch) * kPix;
  for (int i = threadIdx.x; i < J * kPix; i += kThreads) {
    const int j = i / kPix, px = i % kPix;
    tgt[j * (kPix + 1) + px] = __ldg(target + ((int64_t)b * J + j) * hw + p0 + px);
  }
  for (int i = threadIdx.x; i < S * 2 * J; i += kThreads) cs[i] = __ldg(coef + (size_t)b * S * 2 * J + i);
  __syncthreads();
  const int64_t base = ((int64_t)b * hw + p0) * J;
  for (int i = threadIdx.x; i < J * kPix; i += kThreads) {
    const int px = i / J, j = i % J;
    const float g = tgt[j * (kPix + 1) + px];
    const float t = teacher ? __ldg(teacher + base + i) : 0.f;
#pragma unroll
    for (int s = 0; s < kMaxStacks; ++s) {
      if (s < S) {
        // each term rounded on its own, then added (no FMA), as autograd adds the gradients of the two module-form
        // criteria: the same bits whenever alpha and 1 - alpha are powers of two (alpha = 0.5)
        const float o = __ldg(sp.out[s] + base + i);
        float gr = __fmul_rn(cs[(2 * s) * J + j], o - g);
        if (teacher) gr = __fadd_rn(gr, __fmul_rn(cs[(2 * s + 1) * J + j], o - t));
        sp.grad[s][base + i] = gr;
      }
    }
  }
}

// (3) module form: one block per NCHW (b, j) map; joints left out (coefficient 0) get zeros without reading the maps
__global__ void __launch_bounds__(kThreads)
ohkm_grad_nchw_kernel(const float* __restrict__ out, const float* __restrict__ target, const float* __restrict__ coef,
                      int J, int hw, float* __restrict__ grad) {
  const int b = blockIdx.x / J, j = blockIdx.x % J;
  const float c = __ldg(coef + (size_t)b * 2 * J + j);
  const int64_t off = (int64_t)blockIdx.x * hw;
  if (c == 0.f) {
    for (int p = threadIdx.x; p < hw; p += kThreads) grad[off + p] = 0.f;
    return;
  }
  for (int p = threadIdx.x; p < hw; p += kThreads) grad[off + p] = c * (__ldg(out + off + p) - __ldg(target + off + p));
}

size_t ohkm_ws_bytes(int64_t B, int64_t nch, int64_t S, int64_t J) {
  return (size_t)((B * nch * S * 2 * J + B * S * 2) * (int64_t)sizeof(double) + B * S * 2 * J * (int64_t)sizeof(float));
}

struct OhkmWs {
  double* part;
  double* contrib;
  float* coef;
};

OhkmWs ohkm_ws_split(void* ws, int64_t B, int64_t nch, int64_t S, int64_t J) {
  OhkmWs r;
  r.part = (double*)ws;
  r.contrib = r.part + B * nch * S * 2 * J;
  r.coef = (float*)(r.contrib + B * S * 2);
  return r;
}

}  // namespace
}  // namespace fpd

extern "C" {

size_t fpd_loss_ohkm_workspace_bytes(int S, int B, int J, int h, int w) {
  const int64_t hw = (int64_t)h * w;
  if (S < 1 || B < 1 || J < 1 || hw < 1) return 0;
  return ohkm_ws_bytes(B, (hw + kPix - 1) / kPix, S, J);
}

size_t fpd_joints_ohkm_workspace_bytes(int B, int J) {
  if (B < 1 || J < 1) return 0;
  return ohkm_ws_bytes(B, 1, 1, J);
}

}  // extern "C"

namespace fpd {
namespace {

int loss_ohkm_launch(const float* const* outs, int S, const float* target_nchw, const float* teacher_nhwc,
                     const float* tw, const float* kw, float alpha, float* const* grads, float grad_scale,
                     float* losses, int B, int J, int h, int w, int pose_topk, int kd_topk, void* workspace,
                     size_t ws_bytes, fpd_stream_t stream) {
  FPD_REQUIRE(outs != nullptr, "fpd_loss_ohkm_fused: outs_host is NULL");
  FPD_REQUIRE(S >= 1 && S <= kMaxStacks, "fpd_loss_ohkm: S=%d out of range [1,%d]", S, kMaxStacks);
  FPD_REQUIRE(B >= 1, "fpd_loss_ohkm: B=%d (an empty batch has no loss)", B);
  FPD_REQUIRE(h >= 1 && w >= 1, "fpd_loss_ohkm: empty heat-map %dx%d", h, w);
  const int64_t hw64 = (int64_t)h * w;
  FPD_REQUIRE(hw64 % kPix == 0 && hw64 <= (1 << 30), "fpd_loss_ohkm: h*w=%lld must be a multiple of %d",
              (long long)hw64, kPix);
  const int hw = (int)hw64;
  FPD_REQUIRE(J >= 1 && J <= kMaxJ, "fpd_loss_ohkm: J=%d out of range [1,%d]", J, kMaxJ);
  FPD_REQUIRE(pose_topk >= 0 && pose_topk <= J, "fpd_loss_ohkm: pose_topk=%d out of range [0,J=%d]", pose_topk, J);
  FPD_REQUIRE(kd_topk >= 0 && kd_topk <= J, "fpd_loss_ohkm: kd_topk=%d out of range [0,J=%d]", kd_topk, J);
  FPD_REQUIRE(teacher_nhwc != nullptr || kd_topk == 0, "fpd_loss_ohkm: kd_topk=%d without a teacher", kd_topk);
  FPD_REQUIRE(target_nchw != nullptr && losses != nullptr, "fpd_loss_ohkm: target or losses is NULL");
  FPD_REQUIRE(tw != nullptr, "fpd_loss_ohkm: target_weight is required (pass ones for use_target_weight=False)");
  const int64_t nch = hw / kPix;
  FPD_REQUIRE((int64_t)B * nch <= 0x7fffffff, "fpd_loss_ohkm: B * h*w/%d too large", kPix);
  FPD_REQUIRE(workspace != nullptr && ws_bytes >= ohkm_ws_bytes(B, nch, S, J), "fpd_loss_ohkm: workspace too small");
  StackPtrs sp{};
  for (int s = 0; s < S; ++s) {
    FPD_REQUIRE(outs[s] != nullptr, "fpd_loss_ohkm: outs[%d] is NULL", s);
    sp.out[s] = outs[s];
    sp.grad[s] = grads ? grads[s] : nullptr;
    FPD_REQUIRE(grads == nullptr || grads[s] != nullptr, "fpd_loss_ohkm: grads[%d] is NULL", s);
  }
  const OhkmWs ws = ohkm_ws_split(workspace, B, nch, S, J);
  const int L = kThreads / J < kPix ? kThreads / J : kPix;
  const size_t smem1 = ((size_t)J * (kPix + 1) + (size_t)S * 2 * L * J) * sizeof(float);
  ohkm_sums_nhwc_kernel<<<(int)(B * nch), kThreads, smem1, stream>>>(sp, S, target_nchw, teacher_nhwc, J, hw, ws.part);
  FPD_LAUNCH_CHECK();
  const int has_teacher = teacher_nhwc != nullptr;
  ohkm_select_kernel<<<B, kThreads, 0, stream>>>(ws.part, (int)nch, S, J, hw, B, tw, kw, has_teacher, pose_topk,
                                                 kd_topk, alpha, grad_scale, ws.contrib, ws.coef);
  FPD_LAUNCH_CHECK();
  ohkm_final_kernel<<<1, 32, 0, stream>>>(ws.contrib, B, S, has_teacher, alpha, losses);
  FPD_LAUNCH_CHECK();
  if (grads) {
    const size_t smem3 = ((size_t)J * (kPix + 1) + (size_t)S * 2 * J) * sizeof(float);
    ohkm_grad_nhwc_kernel<<<(int)(B * nch), kThreads, smem3, stream>>>(sp, S, target_nchw, teacher_nhwc, ws.coef, J, hw);
    FPD_LAUNCH_CHECK();
  }
  return FPD_OK;
}

}  // namespace
}  // namespace fpd

extern "C" {

int fpd_loss_ohkm_fused(const float* const* outs, int S, const float* target_nchw, const float* teacher_nhwc,
                        const float* tw, float alpha, float* const* grads, float grad_scale, float* losses, int B, int J,
                        int h, int w, int pose_topk, int kd_topk, void* workspace, size_t ws_bytes,
                        fpd_stream_t stream) {
  return loss_ohkm_launch(outs, S, target_nchw, teacher_nhwc, tw, tw, alpha, grads, grad_scale, losses, B, J, h, w,
                          pose_topk, kd_topk, workspace, ws_bytes, stream);
}

int fpd_joints_ohkm(const float* out_nchw, const float* target_nchw, const float* tw, int topk, float* loss3,
                    float* grad_out, int B, int J, int hw, void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  FPD_REQUIRE(out_nchw != nullptr && target_nchw != nullptr && loss3 != nullptr,
              "joints_ohkm: out, target or loss3 is NULL");
  FPD_REQUIRE(B >= 1, "joints_ohkm: B=%d (an empty batch has no loss)", B);
  FPD_REQUIRE(hw >= 1, "joints_ohkm: hw=%d (empty heat-map)", hw);
  FPD_REQUIRE(J >= 1 && J <= kMaxJ, "joints_ohkm: J=%d out of range [1,%d]", J, kMaxJ);
  FPD_REQUIRE(topk >= 1 && topk <= J, "joints_ohkm: topk=%d out of range [1,J=%d]", topk, J);
  FPD_REQUIRE((int64_t)B * J <= 0x7fffffff, "joints_ohkm: B*J too large");
  FPD_REQUIRE(workspace != nullptr && ws_bytes >= ohkm_ws_bytes(B, 1, 1, J), "joints_ohkm: workspace too small");
  const OhkmWs ws = ohkm_ws_split(workspace, B, 1, 1, J);
  ohkm_sums_nchw_kernel<<<B * J, kThreads, 0, stream>>>(out_nchw, target_nchw, J, hw, ws.part);
  FPD_LAUNCH_CHECK();
  ohkm_select_kernel<<<B, kThreads, 0, stream>>>(ws.part, 1, 1, J, hw, B, tw, tw, 0, topk, 0, 0.f, 1.f, ws.contrib,
                                                 ws.coef);
  FPD_LAUNCH_CHECK();
  ohkm_final_kernel<<<1, 32, 0, stream>>>(ws.contrib, B, 1, 0, 0.f, loss3);
  FPD_LAUNCH_CHECK();
  if (grad_out) {
    ohkm_grad_nchw_kernel<<<B * J, kThreads, 0, stream>>>(out_nchw, target_nchw, ws.coef, J, hw, grad_out);
    FPD_LAUNCH_CHECK();
  }
  return FPD_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Channel-wise distillation (Shu et al., ICCV 2021) per joint heat-map, JointsKLDLoss: each (b, j) map is a
// distribution over its P = h*w pixels at temperature T,
//   p = softmax(r / T) (reference: target or teacher),  q = softmax(o / T) (student),  KL = sum_p p (log p - log q)
//   L = T^2 / (B*J) * sum_{b,j} w[b,j] KL[b,j]          dL/do = T * w * (q - p) / (B*J)
// With m = max r, S = sum exp((r - m)/T) and C = sum exp((r - m)/T) (r - o) (and m', S' for o):
//   KL = C / (T S) + (m' - m) / T + log(S' / S)
// Three passes, like the hard keypoint mining above: (1) per (sample, 64-pixel chunk) block, each map's chunk maximum,
// then the chunk's exp-sums and cross sums relative to it (fp32 within a thread, lanes added in fp64); (2) one block
// per sample merges the chunks in fp64 (rescaling by exp((m_c - m)/T)), forms KL (or the sums of squares of an MSE /
// OHKM term, with the same selection), the sample's share of each term and the gradient constants; (3) one pass writes
// every gradient element. The reference's statistics are computed once and shared by all stacks. Student and reference
// probabilities come out of the same arithmetic, so a student equal to its reference gives exactly zero loss and
// gradient. No floating-point atomics: deterministic and graph-capturable.
//
// The module form (NCHW student) runs the same three kernels with S = 1 and the reference in the pose slot, chunk by
// chunk; for h*w % 64 == 0 it therefore gives the fused form's bits term by term.
//
// Workspace: part double [B][nch][S+1][2][J][3] (slot S: the reference; {max, exp-sum, cross sum} or {-, sum of
// squares, -}) | contrib double [B][S][2] | coef float4 [B][S+1][2][J] ({coefficient, max, 1/exp-sum, -}).
namespace fpd {
namespace {

enum { kKindSq = 0, kKindKl = 1 };

struct KlTerms {
  int kind[2];      // pose, kd: kKindSq (MSE / OHKM) or kKindKl
  float t[2];       // T of a KL term
  float inv_t[2];   // its 1/T, the scale every exponent uses
};

// exp((x - m) / T): the one expression both the student's and the reference's statistics and probabilities use
__device__ __forceinline__ float kl_exp(float x, float m, float inv_t) {
  return expf(__fmul_rn(__fsub_rn(x, m), inv_t));
}

// (1) one block per (sample, 64-pixel chunk); thread (pl, j) owns joint j and pixels pl, pl + L, ... of the chunk.
// NCHW_OUT: the student is NCHW (module form; the chunk may be partial), else NHWC with h*w % 64 == 0.
template <bool NCHW_OUT>
__global__ void __launch_bounds__(kThreads, 1)
kl_stats_kernel(StackPtrs sp, int S, const float* __restrict__ target, const float* __restrict__ teacher, int J, int hw,
                KlTerms tm, double* __restrict__ part) {
  extern __shared__ float sm[];
  float* tgt = sm;                          // [J][kPix+1]
  float* red = sm + J * (kPix + 1);         // [max(S+2, 4)][L*J] lane partials
  float* cmax = red + (S + 2 > 4 ? S + 2 : 4) * kThreads;   // [S+2][J] chunk maxima: stacks, target, teacher
  const int nch = (hw + kPix - 1) / kPix;
  const int b = blockIdx.x / nch;
  const int p0 = (blockIdx.x % nch) * kPix;
  const int np = min(kPix, hw - p0);
  for (int i = threadIdx.x; i < J * kPix; i += kThreads) {
    const int j = i / kPix, px = i % kPix;
    if (px < np) tgt[j * (kPix + 1) + px] = __ldg(target + ((int64_t)b * J + j) * hw + p0 + px);
  }
  __syncthreads();
  const int L = min(kPix, kThreads / J);
  const int active = L * J;
  const int j = threadIdx.x % J, pl = threadIdx.x / J;
  const bool kl_p = tm.kind[0] == kKindKl, kl_k = tm.kind[1] == kKindKl;
  const bool any_kl = kl_p || kl_k;
  auto out_at = [&](int s, int px) -> float {
    return NCHW_OUT ? __ldg(sp.out[s] + ((int64_t)b * J + j) * hw + p0 + px)
                    : __ldg(sp.out[s] + ((int64_t)b * hw + p0 + px) * J + j);
  };
  auto teacher_at = [&](int px) -> float { return __ldg(teacher + ((int64_t)b * hw + p0 + px) * J + j); };
  // chunk maxima (fmaxf passes a NaN over; the exp-sums below carry it into the loss)
  if (any_kl) {
    if (threadIdx.x < active) {
      float mo[kMaxStacks], mg = -INFINITY, mt = -INFINITY;
#pragma unroll
      for (int s = 0; s < kMaxStacks; ++s) mo[s] = -INFINITY;
      for (int px = pl; px < np; px += L) {
        if (kl_p) mg = fmaxf(mg, tgt[j * (kPix + 1) + px]);
        if (kl_k) mt = fmaxf(mt, teacher_at(px));
#pragma unroll
        for (int s = 0; s < kMaxStacks; ++s)
          if (s < S) mo[s] = fmaxf(mo[s], out_at(s, px));
      }
#pragma unroll
      for (int s = 0; s < kMaxStacks; ++s)
        if (s < S) red[s * active + threadIdx.x] = mo[s];
      red[S * active + threadIdx.x] = mg;
      red[(S + 1) * active + threadIdx.x] = mt;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < (S + 2) * J; q += kThreads) {
      const int slot = q / J, jj = q % J;
      float m = -INFINITY;
      for (int l = 0; l < L; ++l) m = fmaxf(m, red[slot * active + l * J + jj]);
      cmax[q] = m;
    }
    __syncthreads();
  }
  // exp-sums, cross sums and sums of squares; per stack: {A_pose, C_pose, A_kd, C_kd}
  float ap[kMaxStacks], cp[kMaxStacks], ak[kMaxStacks], ck[kMaxStacks], sg = 0.f, st = 0.f;
#pragma unroll
  for (int s = 0; s < kMaxStacks; ++s) ap[s] = cp[s] = ak[s] = ck[s] = 0.f;
  if (threadIdx.x < active) {
    const float mg = any_kl ? cmax[S * J + j] : 0.f, mt = any_kl ? cmax[(S + 1) * J + j] : 0.f;
    for (int px = pl; px < np; px += L) {
      const float g = tgt[j * (kPix + 1) + px];
      const float t = teacher ? teacher_at(px) : 0.f;
      const float eg = kl_p ? kl_exp(g, mg, tm.inv_t[0]) : 0.f;
      const float et = kl_k ? kl_exp(t, mt, tm.inv_t[1]) : 0.f;
      sg = __fadd_rn(sg, eg);
      st = __fadd_rn(st, et);
#pragma unroll
      for (int s = 0; s < kMaxStacks; ++s) {
        if (s < S) {
          const float o = out_at(s, px);
          const float mo = any_kl ? cmax[s * J + j] : 0.f;
          if (kl_p) {
            ap[s] = __fadd_rn(ap[s], kl_exp(o, mo, tm.inv_t[0]));
            cp[s] = fmaf(eg, __fsub_rn(g, o), cp[s]);
          } else {
            const float d = o - g;
            ap[s] = fmaf(d, d, ap[s]);
          }
          if (teacher) {
            if (kl_k) {
              ak[s] = __fadd_rn(ak[s], kl_exp(o, mo, tm.inv_t[1]));
              ck[s] = fmaf(et, __fsub_rn(t, o), ck[s]);
            } else {
              const float d = o - t;
              ak[s] = fmaf(d, d, ak[s]);
            }
          }
        }
      }
    }
  }
  // lanes added in fp64 in lane order, one stack at a time (the shared buffer holds four slots)
  const size_t J3 = (size_t)J * 3;
  double* dst = part + (size_t)blockIdx.x * (S + 1) * 2 * J3;     // [S+1][2][J][3]
  for (int s = 0; s <= S; ++s) {
    __syncthreads();
    if (threadIdx.x < active) {
      float v[4] = {sg, 0.f, st, 0.f};       // slot S: the references
#pragma unroll
      for (int ss = 0; ss < kMaxStacks; ++ss)
        if (ss == s && s < S) { v[0] = ap[ss]; v[1] = cp[ss]; v[2] = ak[ss]; v[3] = ck[ss]; }
#pragma unroll
      for (int k = 0; k < 4; ++k) red[k * active + threadIdx.x] = v[k];
    }
    __syncthreads();
    for (int q = threadIdx.x; q < 2 * J; q += kThreads) {
      const int term = q / J, jj = q % J;
      double a = 0.0, c = 0.0;
      for (int l = 0; l < L; ++l) {
        a += (double)red[(2 * term) * active + l * J + jj];
        c += (double)red[(2 * term + 1) * active + l * J + jj];
      }
      const int mslot = s < S ? s : S + term;       // the student's or this term's reference's maximum
      double* r = dst + ((size_t)s * 2 + term) * J3 + (size_t)jj * 3;
      r[0] = any_kl ? (double)cmax[mslot * J + jj] : 0.0;
      r[1] = a;
      r[2] = c;
    }
  }
}

// (2) one block per sample: merge the chunks, per-(s, term, j) losses, the sample's share of each term (losses as
// ohkm_final_kernel sums them) and the gradient constants. For a KL term l = T^2 w KL and every joint counts (1/J).
__global__ void __launch_bounds__(kThreads)
kl_select_kernel(const double* __restrict__ part, int nch, int S, int J, int hw, int B, const float* __restrict__ tw,
                 const float* __restrict__ kw, int has_teacher, int pose_topk, int kd_topk, KlTerms tm, float alpha, float grad_scale,
                 double* __restrict__ contrib, float4* __restrict__ coef) {
  __shared__ double ld[kMaxStacks * 2][kMaxJ];
  __shared__ float lf[kMaxStacks * 2][kMaxJ];
  __shared__ double rm[2][kMaxJ], rs[2][kMaxJ];
  const int b = blockIdx.x;
  const size_t rec = (size_t)(S + 1) * 2 * J * 3;        // one chunk's record
  const double* pb = part + (size_t)b * nch * rec;
  float4* cb = coef + (size_t)b * (S + 1) * 2 * J;
  // the references' maxima and exp-sums
  for (int q = threadIdx.x; q < 2 * J; q += kThreads) {
    const int term = q / J, j = q % J;
    if (tm.kind[term] != kKindKl || (term == 1 && !has_teacher)) continue;
    const double it = (double)tm.inv_t[term];
    const size_t off = ((size_t)S * 2 + term) * J * 3 + (size_t)j * 3;
    double m = -INFINITY;
    for (int c = 0; c < nch; ++c) m = fmax(m, pb[c * rec + off]);
    double s = 0.0;
    for (int c = 0; c < nch; ++c) s += pb[c * rec + off + 1] * exp((pb[c * rec + off] - m) * it);
    rm[term][j] = m;
    rs[term][j] = s;
    cb[((size_t)S * 2 + term) * J + j] = make_float4(0.f, (float)m, (float)(1.0 / s), 0.f);
  }
  __syncthreads();
  for (int q = threadIdx.x; q < S * 2 * J; q += kThreads) {
    const int stt = q / J, j = q % J, term = stt & 1;
    const float* wt = term ? kw : tw;
    const double w = wt ? (double)__ldg(wt + (size_t)b * J + j) : 1.0;
    const size_t off = (size_t)q * 3;
    double l = 0.0;
    if (term == 1 && !has_teacher) {
      l = 0.0;
    } else if (tm.kind[term] == kKindKl) {
      const double it = (double)tm.inv_t[term];
      const size_t roff = ((size_t)S * 2 + term) * J * 3 + (size_t)j * 3;
      double m = -INFINITY;
      for (int c = 0; c < nch; ++c) m = fmax(m, pb[c * rec + off]);
      double a = 0.0, x = 0.0;
      for (int c = 0; c < nch; ++c) {
        a += pb[c * rec + off + 1] * exp((pb[c * rec + off] - m) * it);
        x += pb[c * rec + off + 2] * exp((pb[c * rec + roff] - rm[term][j]) * it);
      }
      const double kl = x * it / rs[term][j] + (m - rm[term][j]) * it + log(a / rs[term][j]);
      l = w * kl * (double)tm.t[term] * (double)tm.t[term];
      cb[(size_t)q] = make_float4(0.f, (float)m, (float)(1.0 / a), 0.f);
    } else {
      double a = 0.0;
      for (int c = 0; c < nch; ++c) a += pb[c * rec + off + 1];
      l = 0.5 * (w * w) * a / (double)hw;
    }
    ld[stt][j] = l;
    lf[stt][j] = (float)l;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int stt = wid; stt < S * 2; stt += kThreads / 32) {
    const int s = stt >> 1, term = stt & 1;
    float4* cf = cb + ((size_t)s * 2 + term) * J;
    double* ct = contrib + ((size_t)b * S + s) * 2 + term;
    if (term == 1 && !has_teacher) {
      for (int j = lane; j < J; j += 32) cf[j].x = 0.f;
      if (lane == 0) *ct = 0.0;
      continue;
    }
    const bool kl = tm.kind[term] == kKindKl;
    const int k = kl ? 0 : (term ? kd_topk : pose_topk);
    const unsigned long long mask = k > 0 ? warp_topk_mask(lf[stt], J, k, lane)
                                          : (J == 64 ? ~0ull : ((1ull << J) - 1ull));
    const int cnt = k > 0 ? k : J;
    const double factor = has_teacher ? (term ? (double)alpha : 1.0 - (double)alpha) : 1.0;
    const double scale = kl ? (double)grad_scale * factor * (double)tm.t[term] / ((double)B * (double)J)
                            : (double)grad_scale * factor / ((double)B * (double)cnt * (double)hw);
    const float* wt = term ? kw : tw;
    for (int j = lane; j < J; j += 32) {
      const double w = wt ? (double)__ldg(wt + (size_t)b * J + j) : 1.0;
      cf[j].x = ((mask >> j) & 1ull) ? (float)(kl ? scale * w : scale * w * w) : 0.f;
    }
    if (lane == 0) {
      double sum = 0.0;
      for (int j = 0; j < J; ++j)
        if ((mask >> j) & 1ull) sum += ld[stt][j];
      *ct = sum / (double)cnt;
    }
  }
}

// one term's gradient at one element: c (q - p) for KL, c (o - ref) otherwise; rounded on its own
__device__ __forceinline__ float kl_term_grad(bool kl, float4 c, float o, float ref, float p, float inv_t) {
  if (!kl) return __fmul_rn(c.x, o - ref);
  const float q = __fmul_rn(kl_exp(o, c.y, inv_t), c.z);
  return __fmul_rn(c.x, __fsub_rn(q, p));
}

// (3) fused form: grad_s = pose term + kd term for every element
__global__ void __launch_bounds__(kThreads)
kl_grad_nhwc_kernel(StackPtrs sp, int S, const float* __restrict__ target, const float* __restrict__ teacher,
                    const float4* __restrict__ coef, int J, int hw, KlTerms tm) {
  extern __shared__ float sm[];
  float* tgt = sm;                                      // [J][kPix+1]
  float4* cs = (float4*)(sm + ((J * (kPix + 1) + 3) & ~3));   // [S+1][2][J] of this sample
  const int nch = hw / kPix;
  const int b = blockIdx.x / nch;
  const int p0 = (blockIdx.x % nch) * kPix;
  for (int i = threadIdx.x; i < J * kPix; i += kThreads) {
    const int j = i / kPix, px = i % kPix;
    tgt[j * (kPix + 1) + px] = __ldg(target + ((int64_t)b * J + j) * hw + p0 + px);
  }
  const int n = (S + 1) * 2 * J;
  for (int i = threadIdx.x; i < n; i += kThreads) cs[i] = __ldg(coef + (size_t)b * n + i);
  __syncthreads();
  const bool kl_p = tm.kind[0] == kKindKl, kl_k = tm.kind[1] == kKindKl;
  const int64_t base = ((int64_t)b * hw + p0) * J;
  for (int i = threadIdx.x; i < J * kPix; i += kThreads) {
    const int px = i / J, j = i % J;
    const float g = tgt[j * (kPix + 1) + px];
    const float t = teacher ? __ldg(teacher + base + i) : 0.f;
    float pg = 0.f, pt = 0.f;
    if (kl_p) { const float4 r = cs[(S * 2) * J + j]; pg = __fmul_rn(kl_exp(g, r.y, tm.inv_t[0]), r.z); }
    if (kl_k && teacher) { const float4 r = cs[(S * 2 + 1) * J + j]; pt = __fmul_rn(kl_exp(t, r.y, tm.inv_t[1]), r.z); }
#pragma unroll
    for (int s = 0; s < kMaxStacks; ++s) {
      if (s < S) {
        const float o = __ldg(sp.out[s] + base + i);
        float gr = kl_term_grad(kl_p, cs[(2 * s) * J + j], o, g, pg, tm.inv_t[0]);
        if (teacher) gr = __fadd_rn(gr, kl_term_grad(kl_k, cs[(2 * s + 1) * J + j], o, t, pt, tm.inv_t[1]));
        sp.grad[s][base + i] = gr;
      }
    }
  }
}

// (3) module form: one element per thread over the NCHW tensor
__global__ void __launch_bounds__(kThreads)
kl_grad_nchw_kernel(const float* __restrict__ out, const float* __restrict__ ref, const float4* __restrict__ coef,
                    int J, int hw, float inv_t, int64_t n, float* __restrict__ grad) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bj = i / hw;
    const int b = (int)(bj / J), j = (int)(bj % J);
    const float4* cb = coef + (size_t)b * 2 * 2 * J;      // [S+1 = 2][2][J]
    const float4 rr = cb[2 * J + j];
    const float r = __ldg(ref + i);
    const float p = __fmul_rn(kl_exp(r, rr.y, inv_t), rr.z);
    grad[i] = kl_term_grad(true, cb[j], __ldg(out + i), r, p, inv_t);
  }
}

size_t kl_ws_bytes(int64_t B, int64_t nch, int64_t S, int64_t J) {
  return (size_t)((B * nch * (S + 1) * 2 * J * 3 + B * S * 2) * (int64_t)sizeof(double) +
                  B * (S + 1) * 2 * J * (int64_t)sizeof(float4));
}

struct KlWs {
  double* part;
  double* contrib;
  float4* coef;
};

KlWs kl_ws_split(void* ws, int64_t B, int64_t nch, int64_t S, int64_t J) {
  KlWs r;
  r.part = (double*)ws;
  r.contrib = r.part + B * nch * (S + 1) * 2 * J * 3;
  r.coef = (float4*)(r.contrib + B * S * 2);     // an even number of doubles before it: 16-byte aligned
  return r;
}

size_t kl_stats_smem(int S, int J) {
  return ((size_t)J * (kPix + 1) + (size_t)(S + 2 > 4 ? S + 2 : 4) * kThreads + (size_t)(S + 2) * J) * sizeof(float);
}

// 0: not KL; else a finite T > 0
bool kl_temperature_ok(float t) { return t == 0.f || (isfinite(t) && t > 0.f); }

}  // namespace
}  // namespace fpd

extern "C" {

size_t fpd_loss_kl_workspace_bytes(int S, int B, int J, int h, int w) {
  const int64_t hw = (int64_t)h * w;
  if (S < 1 || B < 1 || J < 1 || hw < 1) return 0;
  return kl_ws_bytes(B, (hw + kPix - 1) / kPix, S, J) + 16;
}

size_t fpd_joints_kld_workspace_bytes(int B, int J, int hw) {
  if (B < 1 || J < 1 || hw < 1) return 0;
  return kl_ws_bytes(B, ((int64_t)hw + kPix - 1) / kPix, 1, J) + 16;
}

}  // extern "C"

namespace fpd {
namespace {

int loss_kl_launch(const float* const* outs, int S, const float* target_nchw, const float* teacher_nhwc,
                   const float* tw, const float* kw, float alpha, float* const* grads, float grad_scale, float* losses,
                   int B, int J, int h, int w, int pose_topk, int kd_topk, float pose_temperature,
                   float kd_temperature, void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  FPD_REQUIRE(outs != nullptr, "fpd_loss_kl_fused: outs_host is NULL");
  FPD_REQUIRE(S >= 1 && S <= kMaxStacks, "fpd_loss_kl: S=%d out of range [1,%d]", S, kMaxStacks);
  FPD_REQUIRE(B >= 1, "fpd_loss_kl: B=%d (an empty batch has no loss)", B);
  FPD_REQUIRE(h >= 1 && w >= 1, "fpd_loss_kl: empty heat-map %dx%d", h, w);
  const int64_t hw64 = (int64_t)h * w;
  FPD_REQUIRE(hw64 % kPix == 0 && hw64 <= (1 << 30), "fpd_loss_kl: h*w=%lld must be a multiple of %d",
              (long long)hw64, kPix);
  const int hw = (int)hw64;
  FPD_REQUIRE(J >= 1 && J <= kMaxJ, "fpd_loss_kl: J=%d out of range [1,%d]", J, kMaxJ);
  FPD_REQUIRE(kl_temperature_ok(pose_temperature), "fpd_loss_kl: pose_temperature=%g must be 0 (not KL) or finite > 0",
              (double)pose_temperature);
  FPD_REQUIRE(kl_temperature_ok(kd_temperature), "fpd_loss_kl: kd_temperature=%g must be 0 (not KL) or finite > 0",
              (double)kd_temperature);
  FPD_REQUIRE(pose_topk >= 0 && pose_topk <= J, "fpd_loss_kl: pose_topk=%d out of range [0,J=%d]", pose_topk, J);
  FPD_REQUIRE(kd_topk >= 0 && kd_topk <= J, "fpd_loss_kl: kd_topk=%d out of range [0,J=%d]", kd_topk, J);
  FPD_REQUIRE(!(pose_topk > 0 && pose_temperature > 0.f), "fpd_loss_kl: pose term has both topk=%d and temperature=%g",
              pose_topk, (double)pose_temperature);
  FPD_REQUIRE(!(kd_topk > 0 && kd_temperature > 0.f), "fpd_loss_kl: kd term has both topk=%d and temperature=%g",
              kd_topk, (double)kd_temperature);
  FPD_REQUIRE(teacher_nhwc != nullptr || (kd_topk == 0 && kd_temperature == 0.f),
              "fpd_loss_kl: a kd topk or temperature without a teacher");
  FPD_REQUIRE(target_nchw != nullptr && losses != nullptr, "fpd_loss_kl: target or losses is NULL");
  FPD_REQUIRE(tw != nullptr, "fpd_loss_kl: target_weight is required (pass ones for use_target_weight=False)");
  const int64_t nch = hw / kPix;
  FPD_REQUIRE((int64_t)B * nch <= 0x7fffffff, "fpd_loss_kl: B * h*w/%d too large", kPix);
  FPD_REQUIRE(workspace != nullptr && ws_bytes >= kl_ws_bytes(B, nch, S, J) + 16, "fpd_loss_kl: workspace too small");
  StackPtrs sp{};
  for (int s = 0; s < S; ++s) {
    FPD_REQUIRE(outs[s] != nullptr, "fpd_loss_kl: outs[%d] is NULL", s);
    sp.out[s] = outs[s];
    sp.grad[s] = grads ? grads[s] : nullptr;
    FPD_REQUIRE(grads == nullptr || grads[s] != nullptr, "fpd_loss_kl: grads[%d] is NULL", s);
  }
  KlTerms tm;
  tm.kind[0] = pose_temperature > 0.f ? kKindKl : kKindSq;
  tm.kind[1] = kd_temperature > 0.f ? kKindKl : kKindSq;
  tm.t[0] = pose_temperature;
  tm.t[1] = kd_temperature;
  tm.inv_t[0] = pose_temperature > 0.f ? (float)(1.0 / (double)pose_temperature) : 0.f;
  tm.inv_t[1] = kd_temperature > 0.f ? (float)(1.0 / (double)kd_temperature) : 0.f;
  void* aligned = (void*)(((uintptr_t)workspace + 15) & ~(uintptr_t)15);
  const KlWs ws = kl_ws_split(aligned, B, nch, S, J);
  kl_stats_kernel<false><<<(int)(B * nch), kThreads, kl_stats_smem(S, J), stream>>>(sp, S, target_nchw, teacher_nhwc,
                                                                                    J, hw, tm, ws.part);
  FPD_LAUNCH_CHECK();
  const int has_teacher = teacher_nhwc != nullptr;
  kl_select_kernel<<<B, kThreads, 0, stream>>>(ws.part, (int)nch, S, J, hw, B, tw, kw, has_teacher, pose_topk, kd_topk,
                                               tm, alpha, grad_scale, ws.contrib, ws.coef);
  FPD_LAUNCH_CHECK();
  ohkm_final_kernel<<<1, 32, 0, stream>>>(ws.contrib, B, S, has_teacher, alpha, losses);
  FPD_LAUNCH_CHECK();
  if (grads) {
    const size_t smem3 = ((size_t)((J * (kPix + 1) + 3) & ~3)) * sizeof(float) + (size_t)(S + 1) * 2 * J * sizeof(float4);
    kl_grad_nhwc_kernel<<<(int)(B * nch), kThreads, smem3, stream>>>(sp, S, target_nchw, teacher_nhwc, ws.coef, J, hw,
                                                                     tm);
    FPD_LAUNCH_CHECK();
  }
  return FPD_OK;
}

}  // namespace
}  // namespace fpd

extern "C" {

int fpd_loss_kl_fused(const float* const* outs, int S, const float* target_nchw, const float* teacher_nhwc,
                      const float* tw, float alpha, float* const* grads, float grad_scale, float* losses, int B, int J,
                      int h, int w, int pose_topk, int kd_topk, float pose_temperature, float kd_temperature,
                      void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  return loss_kl_launch(outs, S, target_nchw, teacher_nhwc, tw, tw, alpha, grads, grad_scale, losses, B, J, h, w,
                        pose_topk, kd_topk, pose_temperature, kd_temperature, workspace, ws_bytes, stream);
}

int fpd_joints_kld(const float* out_nchw, const float* target_nchw, const float* tw, float temperature, float* loss3,
                   float* grad_out, int B, int J, int hw, void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  FPD_REQUIRE(out_nchw != nullptr && target_nchw != nullptr && loss3 != nullptr,
              "joints_kld: out, target or loss3 is NULL");
  FPD_REQUIRE(B >= 1, "joints_kld: B=%d (an empty batch has no loss)", B);
  FPD_REQUIRE(hw >= 1 && hw <= (1 << 30), "joints_kld: hw=%d out of range", hw);
  FPD_REQUIRE(J >= 1 && J <= kMaxJ, "joints_kld: J=%d out of range [1,%d]", J, kMaxJ);
  FPD_REQUIRE(isfinite(temperature) && temperature > 0.f, "joints_kld: temperature=%g must be finite and > 0",
              (double)temperature);
  const int64_t nch = ((int64_t)hw + kPix - 1) / kPix;
  FPD_REQUIRE((int64_t)B * nch <= 0x7fffffff, "joints_kld: B * ceil(hw/%d) too large", kPix);
  FPD_REQUIRE(workspace != nullptr && ws_bytes >= kl_ws_bytes(B, nch, 1, J) + 16, "joints_kld: workspace too small");
  KlTerms tm;
  tm.kind[0] = kKindKl;
  tm.kind[1] = kKindSq;
  tm.t[0] = temperature;
  tm.t[1] = 0.f;
  tm.inv_t[0] = (float)(1.0 / (double)temperature);
  tm.inv_t[1] = 0.f;
  void* aligned = (void*)(((uintptr_t)workspace + 15) & ~(uintptr_t)15);
  const KlWs ws = kl_ws_split(aligned, B, nch, 1, J);
  StackPtrs sp{};
  sp.out[0] = out_nchw;
  kl_stats_kernel<true><<<(int)(B * nch), kThreads, kl_stats_smem(1, J), stream>>>(sp, 1, target_nchw, nullptr, J, hw,
                                                                                  tm, ws.part);
  FPD_LAUNCH_CHECK();
  kl_select_kernel<<<B, kThreads, 0, stream>>>(ws.part, (int)nch, 1, J, hw, B, tw, tw, 0, 0, 0, tm, 0.f, 1.f,
                                               ws.contrib, ws.coef);
  FPD_LAUNCH_CHECK();
  ohkm_final_kernel<<<1, 32, 0, stream>>>(ws.contrib, B, 1, 0, 0.f, loss3);
  FPD_LAUNCH_CHECK();
  if (grad_out) {
    const int64_t n = (int64_t)B * J * hw;
    int64_t nb = (n + kThreads - 1) / kThreads;
    if (nb > 132 * 64) nb = 132 * 64;
    kl_grad_nchw_kernel<<<(int)nb, kThreads, 0, stream>>>(out_nchw, target_nchw, ws.coef, J, hw, tm.inv_t[0], n,
                                                          grad_out);
    FPD_LAUNCH_CHECK();
  }
  return FPD_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Distillation from unlabeled samples. A sample is unlabeled when all J of its target weights are exactly 0; its kd
// weight for joint j is 1 when the teacher's map [b, :, :, j] has a maximum strictly above `thre` (a map holding a NaN
// has a NaN maximum: weight 0), else 0. A labeled sample's kd weights are its target weights.
//
// fpd_kd_weights: one cluster of kKdSplit blocks per sample, each block takes the per-joint maxima of 1/kKdSplit of the
// sample's pixels; block 0 of the cluster reads the others' maxima from their shared memory and writes the weights.
// Maxima are exact, so the result does not depend on the order; no atomics, graph-capturable.
//
// fpd_loss_kdw_fused: the fused loss with the kd term weighted by kd_weight instead of target_weight. It runs the
// launcher fpd_loss_fused / fpd_loss_ohkm_fused / fpd_loss_kl_fused would run for the same topks and temperatures.
namespace fpd {
namespace {

namespace cg = cooperative_groups;

constexpr int kKdSplit = 8;     // blocks per sample: one cluster
constexpr int kKdUnroll = 8;    // loads in flight per thread

// the larger of a and b; a NaN on either side wins
__device__ __forceinline__ float max_nan(float a, float b) { return (isnan(a) || a > b) ? a : b; }

__global__ void __cluster_dims__(kKdSplit, 1, 1) __launch_bounds__(kThreads)
kd_weights_kernel(const float* __restrict__ teacher, const float* __restrict__ tw, float thre, int J, int hw,
                  float* __restrict__ kdw) {
  __shared__ float red[kThreads];
  __shared__ float bmax[kMaxJ];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int b = blockIdx.y;
  const int t = threadIdx.x;
  const int L = kThreads / J;     // pixel lanes: thread (pl, j) owns joint j, pixels p0 + pl, p0 + pl + L, ...
  float m = -INFINITY;
  if (t < L * J) {
    const int j = t % J, pl = t / J;
    const int64_t p1 = (int64_t)hw * (rank + 1) / kKdSplit;
    const float* src = teacher + (int64_t)b * hw * J + j;
    int64_t px = (int64_t)hw * rank / kKdSplit + pl;
    for (; px + (kKdUnroll - 1) * L < p1; px += kKdUnroll * L) {
      float v[kKdUnroll];
#pragma unroll
      for (int u = 0; u < kKdUnroll; ++u) v[u] = __ldg(src + (px + u * L) * J);
#pragma unroll
      for (int u = 0; u < kKdUnroll; ++u) m = max_nan(m, v[u]);
    }
    for (; px < p1; px += L) m = max_nan(m, __ldg(src + px * J));
  }
  red[t] = m;
  __syncthreads();
  if (t < J) {
    float r = -INFINITY;
    for (int l = 0; l < L; ++l) r = max_nan(r, red[l * J + t]);
    bmax[t] = r;
  }
  cluster.sync();
  if (rank == 0) {
    const float w = t < J ? __ldg(tw + (size_t)b * J + t) : 0.f;
    const int labeled = __syncthreads_or(w != 0.f);
    if (t < J) {
      float r = -INFINITY;
      for (int q = 0; q < kKdSplit; ++q) r = max_nan(r, cluster.map_shared_rank(bmax, q)[t]);
      kdw[(size_t)b * J + t] = labeled ? w : (r > thre ? 1.f : 0.f);
    }
  }
  cluster.sync();   // every block's maxima stay in its shared memory until block 0 has read them
}

}  // namespace
}  // namespace fpd

extern "C" {

int fpd_kd_weights(const float* teacher_nhwc, const float* tw, float thre, float* kd_weight, int B, int J, int h, int w,
                   fpd_stream_t stream) {
  FPD_REQUIRE(teacher_nhwc != nullptr && tw != nullptr && kd_weight != nullptr,
              "kd_weights: teacher, target_weight or kd_weight is NULL");
  FPD_REQUIRE(B >= 1 && B <= 65535, "kd_weights: B=%d out of range [1,65535]", B);
  FPD_REQUIRE(J >= 1 && J <= kMaxJ, "kd_weights: J=%d out of range [1,%d]", J, kMaxJ);
  FPD_REQUIRE(h >= 1 && w >= 1 && (int64_t)h * w <= (1 << 30), "kd_weights: heat-map %dx%d out of range", h, w);
  FPD_REQUIRE(isfinite(thre), "kd_weights: thre=%g must be finite", (double)thre);
  kd_weights_kernel<<<dim3(kKdSplit, B), kThreads, 0, stream>>>(teacher_nhwc, tw, thre, J, h * w, kd_weight);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_loss_kdw_fused(const float* const* outs, int S, const float* target_nchw, const float* teacher_nhwc,
                       const float* tw, const float* kd_weight, float alpha, float* const* grads, float grad_scale,
                       float* losses, int B, int J, int h, int w, int pose_topk, int kd_topk, float pose_temperature,
                       float kd_temperature, void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  FPD_REQUIRE(outs != nullptr, "fpd_loss_kdw: outs_host is NULL");
  FPD_REQUIRE(S >= 1 && S <= kMaxStacks, "fpd_loss_kdw: S=%d out of range [1,%d]", S, kMaxStacks);
  FPD_REQUIRE(B >= 1, "fpd_loss_kdw: B=%d (an empty batch has no loss)", B);
  FPD_REQUIRE(h >= 1 && w >= 1, "fpd_loss_kdw: empty heat-map %dx%d", h, w);
  FPD_REQUIRE(target_nchw != nullptr && losses != nullptr && tw != nullptr,
              "fpd_loss_kdw: target, losses or target_weight is NULL");
  FPD_REQUIRE(teacher_nhwc != nullptr && kd_weight != nullptr, "fpd_loss_kdw: kd_weight and a teacher are required");
  FPD_REQUIRE(workspace != nullptr, "fpd_loss_kdw: workspace is NULL");
  for (int s = 0; s < S; ++s) {
    FPD_REQUIRE(outs[s] != nullptr, "fpd_loss_kdw: outs[%d] is NULL", s);
    FPD_REQUIRE(grads == nullptr || grads[s] != nullptr, "fpd_loss_kdw: grads[%d] is NULL", s);
  }
  if (pose_temperature != 0.f || kd_temperature != 0.f)
    return loss_kl_launch(outs, S, target_nchw, teacher_nhwc, tw, kd_weight, alpha, grads, grad_scale, losses, B, J, h,
                          w, pose_topk, kd_topk, pose_temperature, kd_temperature, workspace, ws_bytes, stream);
  if (pose_topk != 0 || kd_topk != 0)
    return loss_ohkm_launch(outs, S, target_nchw, teacher_nhwc, tw, kd_weight, alpha, grads, grad_scale, losses, B, J,
                            h, w, pose_topk, kd_topk, workspace, ws_bytes, stream);
  return loss_mse_launch(outs, S, target_nchw, teacher_nhwc, tw, kd_weight, alpha, grads, grad_scale, losses, B, J, h, w,
                         workspace, ws_bytes, stream);
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Feature distillation, a hint term in the FitNets sense (Romero et al., ICLR 2015). With a = A(s) the student's head
// feature through the 1x1 adapter and t the teacher's head feature, both NHWC with n elements,
//   L_feat = (1/n) * sum (a - t)^2,   grad = (2 * weight / n) * (a - t),   losses[2] += weight * L_feat.
// One pass: each thread reads 4 consecutive elements of a and of t per step (t in fp32, or in fp16 widened on load),
// writes the gradient and adds (a - t)^2 in fp64; each block writes one fp64 partial, and a one-block kernel adds the
// partials in index order. No atomics and a grid that depends on n alone: runs and graph replays are bit-identical, and
// an fp16 teacher gives the bits of the same teacher widened to fp32 (widening is exact). A NaN anywhere in a or t makes
// L_feat NaN.
namespace fpd {
namespace {

constexpr int kFeatBlocks = kNumSMs * 4;   // grid cap
constexpr int kFeatUnroll = 4;             // 4-element steps in flight per thread

__device__ __forceinline__ float4 feat_load4(const float* t, int64_t g) {
  return __ldg(reinterpret_cast<const float4*>(t) + g);
}
__device__ __forceinline__ float4 feat_load4(const __half* t, int64_t g) {
  const uint2 r = __ldg(reinterpret_cast<const uint2*>(t) + g);
  const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
  const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
__device__ __forceinline__ float feat_load1(const float* t, int64_t i) { return __ldg(t + i); }
__device__ __forceinline__ float feat_load1(const __half* t, int64_t i) { return __half2float(t[i]); }

// VEC: n % 4 == 0 and every pointer aligned to its 4-element access (the host checks)
template <typename T, bool VEC>
__global__ void __launch_bounds__(kThreads)
feature_mse_kernel(const float* __restrict__ a, const T* __restrict__ t, float coef, int64_t n,
                   float* __restrict__ grad, double* __restrict__ part) {
  double acc = 0.0;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int64_t first = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (VEC) {
    const int64_t ng = n / 4;
    for (int64_t g0 = first; g0 < ng; g0 += stride * kFeatUnroll) {
      float4 av[kFeatUnroll], tv[kFeatUnroll];
#pragma unroll
      for (int u = 0; u < kFeatUnroll; ++u) {
        const int64_t g = g0 + u * stride;
        if (g < ng) {
          av[u] = __ldg(reinterpret_cast<const float4*>(a) + g);
          tv[u] = feat_load4(t, g);
        }
      }
#pragma unroll
      for (int u = 0; u < kFeatUnroll; ++u) {
        const int64_t g = g0 + u * stride;
        if (g < ng) {
          const float d0 = av[u].x - tv[u].x, d1 = av[u].y - tv[u].y, d2 = av[u].z - tv[u].z, d3 = av[u].w - tv[u].w;
          acc = fma((double)d0, (double)d0, acc);
          acc = fma((double)d1, (double)d1, acc);
          acc = fma((double)d2, (double)d2, acc);
          acc = fma((double)d3, (double)d3, acc);
          reinterpret_cast<float4*>(grad)[g] = make_float4(coef * d0, coef * d1, coef * d2, coef * d3);
        }
      }
    }
  } else {
    for (int64_t i = first; i < n; i += stride) {
      const float d = __ldg(a + i) - feat_load1(t, i);
      acc = fma((double)d, (double)d, acc);
      grad[i] = coef * d;
    }
  }
  __shared__ double red[kThreads / 32];
  acc = warp_sum(acc);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) s += red[i];
    part[blockIdx.x] = s;
  }
}

__global__ void __launch_bounds__(kThreads)
feature_mse_final_kernel(const double* __restrict__ part, int nblocks, double inv_n, float weight,
                         float* __restrict__ feat_loss, float* __restrict__ losses) {
  __shared__ double red[kThreads / 32];
  double s = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += kThreads) s += part[i];
  s = warp_sum(s);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) tot += red[i];
    const double L = tot * inv_n;
    feat_loss[0] = (float)L;
    if (losses) losses[2] = (float)((double)losses[2] + (double)weight * L);
  }
}

bool feature_vec_ok(const void* p, int64_t n, int align) {
  return n % 4 == 0 && (reinterpret_cast<uintptr_t>(p) % align) == 0;
}

int feature_blocks(int64_t n, bool vec) {
  const int64_t units = vec ? n / 4 : n;
  int64_t nb = (units + (int64_t)kThreads * kFeatUnroll - 1) / ((int64_t)kThreads * kFeatUnroll);
  if (nb > kFeatBlocks) nb = kFeatBlocks;
  return nb < 1 ? 1 : (int)nb;
}

}  // namespace
}  // namespace fpd

extern "C" {

size_t fpd_feature_mse_workspace_bytes(int64_t n) {
  return (size_t)feature_blocks(n, false) * sizeof(double);
}

int fpd_feature_mse(const float* student, const void* teacher, int teacher_f16, float weight, float* grad,
                    float* feat_loss, float* losses, int64_t n, void* workspace, size_t workspace_bytes,
                    fpd_stream_t stream) {
  FPD_REQUIRE(student != nullptr && teacher != nullptr && grad != nullptr && feat_loss != nullptr,
              "fpd_feature_mse: student, teacher, grad or feat_loss is NULL");
  FPD_REQUIRE(workspace != nullptr, "fpd_feature_mse: workspace is NULL");
  FPD_REQUIRE(n >= 1, "fpd_feature_mse: n=%lld (an empty feature has no loss)", (long long)n);
  FPD_REQUIRE(teacher_f16 == 0 || teacher_f16 == 1, "fpd_feature_mse: teacher_f16=%d must be 0 or 1", teacher_f16);
  FPD_REQUIRE(isfinite(weight) && weight >= 0.f, "fpd_feature_mse: weight=%g must be finite and >= 0", (double)weight);
  const bool vec = feature_vec_ok(student, n, 16) && feature_vec_ok(grad, n, 16) &&
                   feature_vec_ok(teacher, n, teacher_f16 ? 8 : 16);
  const int nblocks = feature_blocks(n, vec);
  FPD_REQUIRE(workspace_bytes >= (size_t)nblocks * sizeof(double), "fpd_feature_mse: workspace too small");
  const float coef = (float)(2.0 * (double)weight / (double)n);
  double* part = (double*)workspace;
  if (teacher_f16) {
    const __half* t = (const __half*)teacher;
    if (vec) feature_mse_kernel<__half, true><<<nblocks, kThreads, 0, stream>>>(student, t, coef, n, grad, part);
    else feature_mse_kernel<__half, false><<<nblocks, kThreads, 0, stream>>>(student, t, coef, n, grad, part);
  } else {
    const float* t = (const float*)teacher;
    if (vec) feature_mse_kernel<float, true><<<nblocks, kThreads, 0, stream>>>(student, t, coef, n, grad, part);
    else feature_mse_kernel<float, false><<<nblocks, kThreads, 0, stream>>>(student, t, coef, n, grad, part);
  }
  FPD_LAUNCH_CHECK();
  feature_mse_final_kernel<<<1, kThreads, 0, stream>>>(part, nblocks, 1.0 / (double)n, weight, feat_loss, losses);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // extern "C"
