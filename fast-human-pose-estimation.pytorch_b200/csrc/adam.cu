// adam.cu -- fused Adam over one flat fp32 parameter buffer (one launch instead of ~750 per-tensor
// updates). Matches torch.optim.Adam (non-amsgrad) as the reference configures it in
// lib/utils/utils.py:69-73 (Adam(lr) -- TRAIN.WD is ignored for adam) stepped at lib/core/function.py:147.
//   m = b1*m + (1-b1)*g ; v = b2*v + (1-b2)*g*g
//   p -= (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
#include "common.cuh"

namespace fpd {
namespace {
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, int64_t n, float lr, float b1, float b2, float eps, float wd,
                            float bc1, float rsqrt_bc2, float gscale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float grad = g[i] * gscale;
    const float pv = p[i];
    if (wd != 0.f) grad = fmaf(wd, pv, grad);
    const float mi = b1 * m[i] + (1.f - b1) * grad;
    const float vi = b2 * v[i] + (1.f - b2) * grad * grad;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) * rsqrt_bc2 + eps;
    p[i] = pv - (lr / bc1) * (mi / denom);
  }
}
}  // namespace
}  // namespace fpd

using namespace fpd;

extern "C" {

int fpd_adam_flat(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float beta1,
                  float beta2, float eps, float weight_decay, int step, float grad_scale, fpd_stream_t stream) {
  FPD_REQUIRE(step >= 1, "adam_flat: step must be >= 1");
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  int64_t blocks = (n + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  if (blocks < 1) blocks = 1;
  adam_kernel<<<(int)blocks, 256, 0, stream>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps,
                                               weight_decay, (float)bc1, (float)(1.0 / sqrt(bc2)), grad_scale);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // extern "C"
