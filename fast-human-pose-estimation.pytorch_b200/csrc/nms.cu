// nms.cu -- greedy box NMS for sm_90a, entirely on the device.
//
// What it replaces: reference lib/nms/nms_kernel.cu:33-77 (pairwise-IoU bit-mask kernel) and the host
// driver `_nms` :90-143 (cudaMalloc/cudaFree per call, full-mask D2H, serial host sweep).
// Same arithmetic contract: boxes pre-sorted by score, IoU with the "+1 pixel" convention, a box is
// suppressed when IoU > thresh (strict), result = indices (into the sorted list) that survive.
//
// Design:
//  * pass 1 (HBM/L2-bound, embarrassingly parallel): only the upper triangle of 64x64 tiles is launched
//    (the reference computes both triangles and throws the lower away); box tiles are staged as SoA in
//    shared memory so the inner loop is bank-conflict free; each thread owns one row box and emits one
//    uint64 suppression word per column tile.
//  * pass 2 (latency-bound, serial by nature): one CTA sweeps the mask on the device, 64 boxes at a
//    time: the 64 diagonal words are staged to shared memory, one thread resolves the chunk with register
//    bit-ops, then the whole CTA ORs the kept rows into the running "removed" bitmap (coalesced reads).
//    Only the keep list (<= n ints) and its length ever cross PCIe.
#include <mutex>

#include "common.cuh"

namespace fpd {
namespace {

constexpr int kT = 64;

__device__ __forceinline__ float iou_p1(float ax1, float ay1, float ax2, float ay2, float bx1, float by1, float bx2,
                                        float by2) {
  const float left = fmaxf(ax1, bx1), right = fminf(ax2, bx2);
  const float top = fmaxf(ay1, by1), bottom = fminf(ay2, by2);
  const float width = fmaxf(right - left + 1.f, 0.f), height = fmaxf(bottom - top + 1.f, 0.f);
  const float inter = width * height;
  const float sa = (ax2 - ax1 + 1.f) * (ay2 - ay1 + 1.f);
  const float sb = (bx2 - bx1 + 1.f) * (by2 - by1 + 1.f);
  return inter / (sa + sb - inter);
}

// linear block id -> (row_tile, col_tile) with col_tile >= row_tile
__global__ void __launch_bounds__(kT)
nms_mask_kernel(const float* __restrict__ boxes, int n, int box_dim, float thresh, int col_blocks,
                unsigned long long* __restrict__ mask) {
  // decode triangular index
  int t = blockIdx.x;
  int row = 0;
  int rem = col_blocks;
  while (t >= rem) { t -= rem; ++row; --rem; }
  const int col = row + t;

  __shared__ float cx1[kT], cy1[kT], cx2[kT], cy2[kT];
  const int cj = col * kT + threadIdx.x;
  if (cj < n) {
    const float* b = boxes + (size_t)cj * box_dim;
    cx1[threadIdx.x] = b[0]; cy1[threadIdx.x] = b[1]; cx2[threadIdx.x] = b[2]; cy2[threadIdx.x] = b[3];
  }
  __syncthreads();
  const int ri = row * kT + threadIdx.x;
  if (ri >= n) return;
  const float* a = boxes + (size_t)ri * box_dim;
  const float ax1 = a[0], ay1 = a[1], ax2 = a[2], ay2 = a[3];
  const int col_size = min(kT, n - col * kT);
  unsigned long long bits = 0ull;
  const int start = (row == col) ? threadIdx.x + 1 : 0;
  for (int i = start; i < col_size; ++i) {
    if (iou_p1(ax1, ay1, ax2, ay2, cx1[i], cy1[i], cx2[i], cy2[i]) > thresh) bits |= 1ull << i;
  }
  mask[(size_t)ri * col_blocks + col] = bits;
}

__global__ void __launch_bounds__(1024)
nms_sweep_kernel(const unsigned long long* __restrict__ mask, int n, int col_blocks, int* __restrict__ keep,
                 int* __restrict__ num_keep) {
  extern __shared__ unsigned long long sm[];
  unsigned long long* remv = sm;               // [col_blocks]
  unsigned long long* diag = sm + col_blocks;  // [64]
  __shared__ unsigned long long kept_bits;
  __shared__ int count;
  for (int j = threadIdx.x; j < col_blocks; j += blockDim.x) remv[j] = 0ull;
  if (threadIdx.x == 0) count = 0;
  __syncthreads();
  for (int c = 0; c < col_blocks; ++c) {
    const int base = c * kT;
    const int csize = min(kT, n - base);
    if (threadIdx.x < kT) diag[threadIdx.x] = threadIdx.x < csize ? mask[(size_t)(base + threadIdx.x) * col_blocks + c] : 0ull;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long cur = remv[c];
      unsigned long long kb = 0ull;
      int cnt = count;
      for (int b = 0; b < csize; ++b) {
        if (!((cur >> b) & 1ull)) {
          keep[cnt++] = base + b;
          kb |= 1ull << b;
          cur |= diag[b];
        }
      }
      count = cnt;
      kept_bits = kb;
    }
    __syncthreads();
    const unsigned long long kb = kept_bits;
    for (int j = c + 1 + threadIdx.x; j < col_blocks; j += blockDim.x) {
      unsigned long long acc = remv[j];
      unsigned long long bits = kb;
      while (bits) {
        const int b = __ffsll((long long)bits) - 1;
        bits &= bits - 1;
        acc |= mask[(size_t)(base + b) * col_blocks + j];
      }
      remv[j] = acc;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *num_keep = count;
}

// ------------------------------------------------------------------------------------------------
// OKS-NMS (reference lib/nms/nms.py:75-124) and the person rescoring that precedes it (lib/dataset/coco.py:346-357).
// Same two-pass structure as the box NMS: pass 1 fills the upper-triangle suppression mask (bit j of row i = "person j
// is suppressed once person i is kept", i.e. oks(g = i, d = j) > thresh), pass 2 is the shared greedy sweep above.
// Arithmetic follows numpy: coordinate differences and dx^2 + dy^2 in the key points' own type T (the reference's
// arrays are float32 from coco.py:283 or float64), everything after the division by the float64 variances in double,
// and the sum over joints in numpy's pairwise order for n <= 128 (8 interleaved partial sums, then a tree, then the
// tail) so that the result is bit-identical up to exp()'s last bit. The visibility mask is the CANDIDATE's alone
// (`list(vg > t) and list(vd > t)` in nms.py:91 evaluates to the second list).
// ------------------------------------------------------------------------------------------------
constexpr int kMaxJ = 32;

__device__ __forceinline__ double np_sum_small(const double* a, int n) {
  if (n < 8) {
    double r = 0.;
    for (int i = 0; i < n; ++i) r += a[i];
    return r;
  }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = a[j];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] += a[i + j];
  double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) res += a[i];
  return res;
}

__device__ __forceinline__ float sq_sum(float a, float b) { return __fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)); }
__device__ __forceinline__ double sq_sum(double a, double b) { return __dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)); }

template <typename T>
__global__ void __launch_bounds__(kT)
oks_mask_kernel(const T* __restrict__ kpts, const double* __restrict__ areas, const double* __restrict__ vars_, int n, int J,
                double thresh, int use_vis, double in_vis_thre, int col_blocks, unsigned long long* __restrict__ mask) {
  int t = blockIdx.x;
  int row = 0;
  int rem = col_blocks;
  while (t >= rem) { t -= rem; ++row; --rem; }
  const int col = row + t;
  const int ri = row * kT + threadIdx.x;
  if (ri >= n) return;
  const T* g = kpts + (size_t)ri * J * 3;
  const double a_g = areas[ri];
  const int col_size = min(kT, n - col * kT);
  unsigned long long bits = 0ull;
  const int start = (row == col) ? threadIdx.x + 1 : 0;
  for (int i = start; i < col_size; ++i) {
    const int cj = col * kT + i;
    const T* d = kpts + (size_t)cj * J * 3;
    const double den = (a_g + areas[cj]) / 2 + 2.220446049250313e-16;   // np.spacing(1)
    double e[kMaxJ];
    int m = 0;
    for (int j = 0; j < J; ++j) {
      const T dx = d[3 * j] - g[3 * j];
      const T dy = d[3 * j + 1] - g[3 * j + 1];
      const T d2 = sq_sum(dx, dy);          // no FMA contraction: numpy rounds dx^2, dy^2 and the sum separately
      if (use_vis && !((double)d[3 * j + 2] > in_vis_thre)) continue;
      e[m++] = exp(-((double)d2 / vars_[j] / den / 2));
    }
    const double oks = m ? np_sum_small(e, m) / m : 0.0;
    if (oks > thresh) bits |= 1ull << i;
  }
  mask[(size_t)ri * col_blocks + col] = bits;
}

template <typename T>
__global__ void oks_rescore_kernel(const T* __restrict__ kpts, const double* __restrict__ box_score, int n, int J,
                                   double in_vis_thre, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double ks = 0;
  int vn = 0;
  for (int j = 0; j < J; ++j) {
    const double s = (double)kpts[((size_t)i * J + j) * 3 + 2];
    if (s > in_vis_thre) { ks = ks + s; ++vn; }
  }
  if (vn) ks = ks / vn;
  out[i] = ks * box_score[i];
}

// Gaussian heat-map targets (reference lib/dataset/JointsDataset.py:233-289): one CTA per (sample, joint) map. `gauss` is
// the (6 sigma + 1)^2 table the host computed with the reference's own float32 numpy expression, so the stamped values
// are bit-identical; mu = int(x / stride + 0.5) in double, truncation toward zero like Python's int().
__global__ void __launch_bounds__(256)
gaussian_target_kernel(const float* __restrict__ joints, const float* __restrict__ joints_vis, const float* __restrict__ joints_weight,
                       const float* __restrict__ gauss, float* __restrict__ target, float* __restrict__ target_weight,
                       int J, int H, int W, double stride_x, double stride_y, int tmp) {
  const int nj = blockIdx.x;
  const int j = nj % J;
  const float* jt = joints + (size_t)nj * 3;
  const int mu_x = (int)((double)jt[0] / stride_x + 0.5);
  const int mu_y = (int)((double)jt[1] / stride_y + 0.5);
  const int ulx = mu_x - tmp, uly = mu_y - tmp, brx = mu_x + tmp + 1, bry = mu_y + tmp + 1;
  float v = joints_vis[(size_t)nj * 3];
  const bool oob = ulx >= W || uly >= H || brx < 0 || bry < 0;
  if (oob) v = 0.f;
  const bool stamp = !oob && v > 0.5f;
  const int size = 2 * tmp + 1;
  float* tg = target + (size_t)nj * H * W;
  for (int p = threadIdx.x; p < H * W; p += blockDim.x) {
    const int y = p / W, x = p - y * W;
    float o = 0.f;
    if (stamp && x >= ulx && x < brx && y >= uly && y < bry) o = gauss[(y - uly) * size + (x - ulx)];
    tg[p] = o;
  }
  if (threadIdx.x == 0) target_weight[nj] = joints_weight ? v * joints_weight[j] : v;
}

// Unbiased targets (DARK, Zhang et al., CVPR 2020): the Gaussian on the sub-pixel centre mu = joint * (W / image_w,
// H / image_h), evaluated in double at every pixel of the map. Visibility as gaussian_target_kernel, on the unrounded
// window ul = mu - 3 sigma, br = mu + 3 sigma + 1.
__global__ void __launch_bounds__(256)
gaussian_target_unbiased_kernel(const float* __restrict__ joints, const float* __restrict__ joints_vis,
                                const float* __restrict__ joints_weight, float* __restrict__ target,
                                float* __restrict__ target_weight, int J, int H, int W, double scale_x, double scale_y,
                                double sigma) {
  const int nj = blockIdx.x;
  const int j = nj % J;
  const float* jt = joints + (size_t)nj * 3;
  const double mu_x = (double)jt[0] * scale_x, mu_y = (double)jt[1] * scale_y;
  const double rad = 3.0 * sigma, den = 2.0 * sigma * sigma;
  float v = joints_vis[(size_t)nj * 3];
  const bool oob = mu_x - rad >= W || mu_y - rad >= H || mu_x + rad + 1.0 < 0.0 || mu_y + rad + 1.0 < 0.0;
  if (oob) v = 0.f;
  const bool stamp = !oob && v > 0.5f;
  float* tg = target + (size_t)nj * H * W;
  for (int p = threadIdx.x; p < H * W; p += blockDim.x) {
    const int y = p / W, x = p - y * W;
    float o = 0.f;
    if (stamp) {
      const double dx = x - mu_x, dy = y - mu_y;
      o = (float)exp(-(dx * dx + dy * dy) / den);
    }
    tg[p] = o;
  }
  if (threadIdx.x == 0) target_weight[nj] = joints_weight ? v * joints_weight[j] : v;
}

// UDP targets (unbiased data processing, Huang et al., CVPR 2020). Sizes are pixel spacings, so the stride is
// (image - 1) / (map - 1) per axis and the centre mu = joint / stride is not rounded. The window and the visibility
// rule are gaussian_target_kernel's, around the rounded centre int(mu + 0.5); inside the window the Gaussian on the
// unrounded centre is evaluated in double.
__global__ void __launch_bounds__(256)
gaussian_target_udp_kernel(const float* __restrict__ joints, const float* __restrict__ joints_vis,
                           const float* __restrict__ joints_weight, float* __restrict__ target,
                           float* __restrict__ target_weight, int J, int H, int W, double stride_x, double stride_y,
                           int tmp, double sigma) {
  const int nj = blockIdx.x;
  const int j = nj % J;
  const float* jt = joints + (size_t)nj * 3;
  const double mu_x = (double)jt[0] / stride_x, mu_y = (double)jt[1] / stride_y;
  const int cx = (int)(mu_x + 0.5), cy = (int)(mu_y + 0.5);
  const int ulx = cx - tmp, uly = cy - tmp, brx = cx + tmp + 1, bry = cy + tmp + 1;
  const double den = 2.0 * sigma * sigma;
  float v = joints_vis[(size_t)nj * 3];
  const bool oob = ulx >= W || uly >= H || brx < 0 || bry < 0;
  if (oob) v = 0.f;
  const bool stamp = !oob && v > 0.5f;
  float* tg = target + (size_t)nj * H * W;
  for (int p = threadIdx.x; p < H * W; p += blockDim.x) {
    const int y = p / W, x = p - y * W;
    float o = 0.f;
    if (stamp && x >= ulx && x < brx && y >= uly && y < bry) {
      const double dx = x - mu_x, dy = y - mu_y;
      o = (float)exp(-(dx * dx + dy * dy) / den);
    }
    tg[p] = o;
  }
  if (threadIdx.x == 0) target_weight[nj] = joints_weight ? v * joints_weight[j] : v;
}

template <typename T>
int oks_nms_device_t(const T* kpts, const double* areas, const double* vars_, int n, int J, double thresh, int use_vis,
                     double in_vis_thre, int* keep_dev, int* num_keep_dev, void* workspace, size_t ws_bytes,
                     cudaStream_t stream) {
  FPD_REQUIRE(J >= 1 && J <= kMaxJ, "oks_nms: J=%d must be in [1, %d]", J, kMaxJ);
  if (n <= 0) {
    FPD_CUDA_CHECK(cudaMemsetAsync(num_keep_dev, 0, sizeof(int), stream));
    return FPD_OK;
  }
  FPD_REQUIRE(kpts && areas && vars_, "oks_nms: null input");
  FPD_REQUIRE(ws_bytes >= fpd_nms_workspace_bytes(n), "oks_nms: workspace too small");
  const int col_blocks = (n + kT - 1) / kT;
  FPD_REQUIRE(col_blocks <= 4096, "oks_nms: n=%d too large", n);
  unsigned long long* mask = (unsigned long long*)workspace;
  const int tri = col_blocks * (col_blocks + 1) / 2;
  oks_mask_kernel<T><<<tri, kT, 0, stream>>>(kpts, areas, vars_, n, J, thresh, use_vis, in_vis_thre, col_blocks, mask);
  FPD_LAUNCH_CHECK();
  const size_t smem = (size_t)(col_blocks + kT) * sizeof(unsigned long long);
  nms_sweep_kernel<<<1, 1024, smem, stream>>>(mask, n, col_blocks, keep_dev, num_keep_dev);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // namespace
}  // namespace fpd

using namespace fpd;

extern "C" {

size_t fpd_nms_workspace_bytes(int n) {
  const size_t col_blocks = (size_t)(n + kT - 1) / kT;
  return (size_t)n * col_blocks * sizeof(unsigned long long) + 256;
}

int fpd_nms_device(const float* boxes_sorted_dev, int n, int box_dim, float thresh, int* keep_dev, int* num_keep_dev,
                   void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  FPD_REQUIRE(box_dim >= 4, "nms: box_dim=%d must be >= 4 (x1,y1,x2,y2[,score])", box_dim);
  if (n <= 0) {
    FPD_CUDA_CHECK(cudaMemsetAsync(num_keep_dev, 0, sizeof(int), stream));
    return FPD_OK;
  }
  FPD_REQUIRE(ws_bytes >= fpd_nms_workspace_bytes(n), "nms: workspace too small");
  const int col_blocks = (n + kT - 1) / kT;
  FPD_REQUIRE(col_blocks <= 4096, "nms: n=%d too large", n);
  unsigned long long* mask = (unsigned long long*)workspace;
  const int tri = col_blocks * (col_blocks + 1) / 2;
  nms_mask_kernel<<<tri, kT, 0, stream>>>(boxes_sorted_dev, n, box_dim, thresh, col_blocks, mask);
  FPD_LAUNCH_CHECK();
  const size_t smem = (size_t)(col_blocks + kT) * sizeof(unsigned long long);
  nms_sweep_kernel<<<1, 1024, smem, stream>>>(mask, n, col_blocks, keep_dev, num_keep_dev);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_oks_nms_device(const void* kpts_sorted, int kpt_f64, const double* areas_sorted, const double* vars_, int n,
                       int J, double thresh, int use_vis, double in_vis_thre, int* keep_dev, int* num_keep_dev,
                       void* workspace, size_t ws_bytes, fpd_stream_t stream) {
  return kpt_f64 ? oks_nms_device_t<double>((const double*)kpts_sorted, areas_sorted, vars_, n, J, thresh, use_vis,
                                            in_vis_thre, keep_dev, num_keep_dev, workspace, ws_bytes, stream)
                 : oks_nms_device_t<float>((const float*)kpts_sorted, areas_sorted, vars_, n, J, thresh, use_vis,
                                           in_vis_thre, keep_dev, num_keep_dev, workspace, ws_bytes, stream);
}

int fpd_oks_rescore(const void* kpts, int kpt_f64, const double* box_score, int n, int J, double in_vis_thre,
                    double* out, fpd_stream_t stream) {
  if (n <= 0) return FPD_OK;
  FPD_REQUIRE(kpts && box_score && out && J >= 1, "oks_rescore: bad arguments");
  if (kpt_f64) oks_rescore_kernel<double><<<(n + 127) / 128, 128, 0, stream>>>((const double*)kpts, box_score, n, J, in_vis_thre, out);
  else oks_rescore_kernel<float><<<(n + 127) / 128, 128, 0, stream>>>((const float*)kpts, box_score, n, J, in_vis_thre, out);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_gaussian_targets(const float* joints, const float* joints_vis, const float* joints_weight,
                         const float* gauss_table, float* target, float* target_weight, int N, int J, int H, int W,
                         int image_w, int image_h, int sigma, fpd_stream_t stream) {
  FPD_REQUIRE(joints && joints_vis && gauss_table && target && target_weight, "gaussian_targets: null pointer");
  FPD_REQUIRE(N >= 0 && J >= 1 && H >= 1 && W >= 1 && sigma >= 1, "gaussian_targets: bad sizes");
  if (N == 0) return FPD_OK;
  gaussian_target_kernel<<<N * J, 256, 0, stream>>>(joints, joints_vis, joints_weight, gauss_table, target, target_weight, J,
                                                    H, W, (double)image_w / W, (double)image_h / H, sigma * 3);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_gaussian_targets_unbiased(const float* joints, const float* joints_vis, const float* joints_weight, float* target,
                                  float* target_weight, int N, int J, int H, int W, int image_w, int image_h, int sigma,
                                  fpd_stream_t stream) {
  FPD_REQUIRE(joints && joints_vis && target && target_weight, "gaussian_targets_unbiased: null pointer");
  FPD_REQUIRE(N >= 0 && J >= 1 && H >= 1 && W >= 1 && image_w >= 1 && image_h >= 1 && sigma >= 1,
              "gaussian_targets_unbiased: bad sizes");
  if (N == 0) return FPD_OK;
  gaussian_target_unbiased_kernel<<<N * J, 256, 0, stream>>>(joints, joints_vis, joints_weight, target, target_weight, J,
                                                             H, W, (double)W / image_w, (double)H / image_h,
                                                             (double)sigma);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_gaussian_targets_udp(const float* joints, const float* joints_vis, const float* joints_weight, float* target,
                             float* target_weight, int N, int J, int H, int W, int image_w, int image_h, int sigma,
                             fpd_stream_t stream) {
  FPD_REQUIRE(joints && joints_vis && target && target_weight, "gaussian_targets_udp: null pointer");
  FPD_REQUIRE(N >= 0 && J >= 1 && H >= 2 && W >= 2 && image_w >= 2 && image_h >= 2 && sigma >= 1,
              "gaussian_targets_udp: bad sizes");
  if (N == 0) return FPD_OK;
  gaussian_target_udp_kernel<<<N * J, 256, 0, stream>>>(joints, joints_vis, joints_weight, target, target_weight, J, H,
                                                        W, (image_w - 1.0) / (W - 1), (image_h - 1.0) / (H - 1),
                                                        sigma * 3, (double)sigma);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_nms_host(int* keep_out, int* num_out, const float* boxes_host, int boxes_num, int boxes_dim, float thresh,
                 int device_id) {
  FPD_REQUIRE(keep_out && num_out, "fpd_nms_host: NULL output pointer");
  if (boxes_num <= 0) {
    *num_out = 0;
    return FPD_OK;
  }
  FPD_REQUIRE(boxes_host != nullptr, "fpd_nms_host: boxes_host is NULL");
  int cur = -1;
  FPD_CUDA_CHECK(cudaGetDevice(&cur));
  if (cur != device_id) FPD_CUDA_CHECK(cudaSetDevice(device_id));
  // grow-only scratch (the reference signature has no workspace argument)
  static std::mutex mu;
  static void* scratch = nullptr;
  static size_t scratch_bytes = 0;
  static int scratch_dev = -1;
  std::lock_guard<std::mutex> lock(mu);
  const size_t boxes_bytes = (size_t)boxes_num * boxes_dim * sizeof(float);
  const size_t boxes_pad = (boxes_bytes + 255) / 256 * 256;
  const size_t keep_pad = ((size_t)boxes_num * sizeof(int) + 255) / 256 * 256;
  const size_t need = boxes_pad + keep_pad + 256 + fpd_nms_workspace_bytes(boxes_num);
  if (need > scratch_bytes || scratch_dev != device_id) {
    if (scratch) cudaFree(scratch);
    scratch = nullptr;
    scratch_bytes = 0;
    FPD_CUDA_CHECK(cudaMalloc(&scratch, need));
    scratch_bytes = need;
    scratch_dev = device_id;
  }
  char* base = (char*)scratch;
  float* boxes_dev = (float*)base;
  int* keep_dev = (int*)(base + boxes_pad);
  int* num_dev = (int*)(base + boxes_pad + keep_pad);
  void* ws = base + boxes_pad + keep_pad + 256;
  cudaStream_t st = 0;
  FPD_CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  int rc = FPD_OK;
  do {
    if (cudaMemcpyAsync(boxes_dev, boxes_host, boxes_bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = FPD_ERR_CUDA; break; }
    rc = fpd_nms_device(boxes_dev, boxes_num, boxes_dim, thresh, keep_dev, num_dev, ws,
                        fpd_nms_workspace_bytes(boxes_num), st);
    if (rc) break;
    if (cudaMemcpyAsync(num_out, num_dev, sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess) { rc = FPD_ERR_CUDA; break; }
    if (cudaStreamSynchronize(st) != cudaSuccess) { rc = FPD_ERR_CUDA; break; }
    if (*num_out > 0 &&
        cudaMemcpy(keep_out, keep_dev, (size_t)(*num_out) * sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) {
      rc = FPD_ERR_CUDA;
      break;
    }
  } while (0);
  if (rc == FPD_ERR_CUDA) set_last_error("fpd_nms_host: CUDA failure: %s", cudaGetErrorString(cudaGetLastError()));
  cudaStreamDestroy(st);
  if (cur != device_id && cur >= 0) cudaSetDevice(cur);
  return rc;
}

}  // extern "C"
