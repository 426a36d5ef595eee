// decode.cu -- device-side flip-test merge and heat-map arg-max.
//
// Reference (host numpy, three host round-trips per batch):
//   lib/core/function.py:218-240  flip the input, second forward, flip_back, 1-px shift, average
//   lib/utils/transforms.py:15-29 flip_back: reverse W, swap left/right joint channels
//   lib/core/inference.py:18-46   get_max_preds: flat arg-max per (b,j) (first maximum wins), max value
// Here one kernel reads both NHWC heat-maps, emits the averaged map and the per-(b,j) arg-max.
// The average is computed as (a + f) * 0.5f exactly like the reference's fp32 torch expression, so
// arg-max indices are bit-exact given bit-identical heat-maps.
// final_preds / pck_counts continue from those arg-maxes on the device:
//   lib/core/inference.py:49-79  get_final_preds: quarter-pixel nudge toward the higher neighbour, heat-map -> image
//   lib/core/evaluate.py:16-71   accuracy: PCK@0.5 against the arg-max of the target heat-maps
// Every floating-point step is an explicitly rounded intrinsic in the order the host (numpy / torch) evaluates it, so
// the results are bit-identical to lib/core/inference.py::get_final_preds and lib/core/evaluate.py::accuracy.
// final_preds_dark is the opt-in alternative to the quarter-pixel nudge: DARK's Taylor step on the log of the blurred
// map (Zhang et al., "Distribution-Aware Coordinate Representation for Human Pose Estimation", CVPR 2020).
// heatmap_resample carries a teacher's heat-maps from its own crop size onto the student's heat-map grid.
#include "common.cuh"

namespace fpd {
namespace {

struct Best {
  float v;
  int i;
};
// numpy semantics: NaN counts as the maximum (np.argmax returns the first NaN, np.amax NaN), otherwise the first
// occurrence of the largest value
__device__ __forceinline__ bool beats(float v, float best) { return v > best || (v != v && best == best); }
__device__ __forceinline__ Best better(Best a, Best b) {
  const bool an = a.v != a.v, bn = b.v != b.v;
  if (an || bn) {
    if (an && bn) return b.i < a.i ? b : a;
    return bn ? b : a;
  }
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}

// grid: B blocks; thread t -> joint j = t % J, pixel lane = t / J, stepping blockDim/J pixels.
__global__ void flip_merge_argmax_kernel(const float* __restrict__ hm, const float* __restrict__ hm_flip,
                                         const int* __restrict__ perm, int shift, float* __restrict__ avg_nhwc,
                                         int* __restrict__ idx, float* __restrict__ maxval, int J, int h, int w) {
  extern __shared__ unsigned char smraw[];
  Best* sbest = reinterpret_cast<Best*>(smraw);
  const int b = blockIdx.x;
  const int lanes = blockDim.x / J;
  const int j = threadIdx.x % J, pl = threadIdx.x / J;
  const int hw = h * w;
  const float* a = hm + (int64_t)b * hw * J;
  const float* f = hm_flip ? hm_flip + (int64_t)b * hw * J : nullptr;
  const int pj = (f && perm) ? perm[j] : j;
  Best best{-INFINITY, 0x7fffffff};
  if (pl < lanes) {
    for (int p = pl; p < hw; p += lanes) {
      float v = __ldg(a + (int64_t)p * J + j);
      if (f) {
        const int y = p / w, x = p % w;
        // flipped-back value at x comes from mirrored column; with the 1-px shift column x reads x-1 (x>=1)
        const int xs = (shift && x >= 1) ? x - 1 : x;
        const float fv = __ldg(f + ((int64_t)y * w + (w - 1 - xs)) * J + pj);
        v = (v + fv) * 0.5f;
      }
      if (avg_nhwc) avg_nhwc[((int64_t)b * hw + p) * J + j] = v;
      if (beats(v, best.v)) { best.v = v; best.i = p; }
    }
    sbest[pl * J + j] = best;
  }
  __syncthreads();
  if (threadIdx.x < J) {
    Best r = sbest[threadIdx.x];
    for (int l = 1; l < lanes; ++l) r = better(r, sbest[l * J + threadIdx.x]);
    idx[b * J + threadIdx.x] = r.i == 0x7fffffff ? 0 : r.i;
    maxval[b * J + threadIdx.x] = r.v;
  }
}

// arg-max of one contiguous map by a full warp; every lane returns the result (index 0 for an all -inf map)
__device__ __forceinline__ Best warp_argmax(const float* __restrict__ p, int hw, int lane) {
  Best best{-INFINITY, 0x7fffffff};
  for (int i = lane; i < hw; i += 32) {
    const float v = __ldg(p + i);
    if (beats(v, best.v)) { best.v = v; best.i = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Best other;
    other.v = __shfl_xor_sync(0xffffffffu, best.v, o);
    other.i = __shfl_xor_sync(0xffffffffu, best.i, o);
    best = better(best, other);
  }
  if (best.i == 0x7fffffff) best.i = 0;
  return best;
}

// plain NCHW arg-max: one warp per (b,j) map
__global__ void argmax_nchw_kernel(const float* __restrict__ hm, int* __restrict__ idx, float* __restrict__ maxval,
                                   int BJ, int hw) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= BJ) return;
  const Best best = warp_argmax(hm + (int64_t)warp * hw, hw, lane);
  if (lane == 0) {
    idx[warp] = best.i;
    maxval[warp] = best.v;
  }
}

// preds_from_argmax (lib/core/inference.py) in float32 like numpy: x = idx % w, y = floor(idx / w), both zeroed unless
// maxval > 0 (a NaN maximum zeroes them too)
__device__ __forceinline__ void coords_from_argmax(int idx, float maxval, int w, float& x, float& y) {
  const float fi = (float)idx, fw = (float)w;
  x = fmodf(fi, fw);
  y = floorf(__fdiv_rn(fi, fw));
  if (!(maxval > 0.f)) x = y = 0.f;
}

// torch.sign: NaN -> 0
__device__ __forceinline__ float sign_of(float d) { return (float)((0.f < d) - (d < 0.f)); }

// preds[t] = (x, y) mapped by the heat-map -> image matrix T, and maxval.
// transform_preds evaluates coords @ t[:, :2].T + t[:, 2] through numpy's matmul, whose OpenBLAS dgemm rounds x*t0,
// adds y*t1 in one fused multiply-add, then adds t2. Plain multiply-then-add differs in the last double bit, and
// now and then in the float32 result.
__device__ __forceinline__ void store_pred(float* __restrict__ preds, int t, const double* __restrict__ T, float x,
                                           float y, float mv) {
  const double xd = x, yd = y;
  preds[(int64_t)t * 3 + 0] = (float)__dadd_rn(__fma_rn(yd, T[1], __dmul_rn(xd, T[0])), T[2]);
  preds[(int64_t)t * 3 + 1] = (float)__dadd_rn(__fma_rn(yd, T[4], __dmul_rn(xd, T[3])), T[5]);
  preds[(int64_t)t * 3 + 2] = mv;
}

// get_final_preds: one thread per (b,j)
__global__ void final_preds_kernel(const float* __restrict__ avg_nhwc, const int* __restrict__ idx,
                                   const float* __restrict__ maxval, const double* __restrict__ inv, int post_process,
                                   float* __restrict__ preds, int BJ, int J, int h, int w) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= BJ) return;
  const int b = t / J, j = t % J;
  const float mv = maxval[t];
  float x, y;
  coords_from_argmax(idx[t], mv, w, x, y);
  if (post_process) {
    // the host gathers from clamped cells and multiplies the sign by the in-range mask, so a NaN neighbour
    // difference contributes sign 0 whether or not the cell is in range
    const int px = (int)floorf(__fadd_rn(x, 0.5f)), py = (int)floorf(__fadd_rn(y, 0.5f));
    const float ok = (px > 1 && px < w - 1 && py > 1 && py < h - 1) ? 1.f : 0.f;
    const int cx = min(max(px, 1), w - 2), cy = min(max(py, 1), h - 2);
    const float* m = avg_nhwc + (int64_t)b * h * w * J + j;
    const float dx = sign_of(__fsub_rn(m[((int64_t)cy * w + cx + 1) * J], m[((int64_t)cy * w + cx - 1) * J]));
    const float dy = sign_of(__fsub_rn(m[((int64_t)(cy + 1) * w + cx) * J], m[((int64_t)(cy - 1) * w + cx) * J]));
    x = __fadd_rn(x, __fmul_rn(__fmul_rn(dx, ok), 0.25f));
    y = __fadd_rn(y, __fmul_rn(__fmul_rn(dy, ok), 0.25f));
  }
  store_pred(preds, t, inv + (int64_t)b * 6, x, y, mv);
}

// ---- DARK decode (distribution-aware coordinates, Zhang et al., CVPR 2020): a second-order Taylor step on the log of
// the Gaussian-blurred map at the arg-max. One CTA per (b,j) map, which it holds in shared memory with its blur along x.
constexpr int kDarkThreads = 256;
constexpr int kDarkMaxKernel = 15;
// dynamic shared memory per block: sm_90's 227 KB opt-in less room for the kernel's static arrays (352 bytes), which
// count against the same limit
constexpr size_t kDarkSmemLimit = 226 * 1024;

// np.max semantics (a NaN anywhere makes the result NaN); exact, so the reduction order cannot change the result
__device__ __forceinline__ float nan_max(float m, float v) { return (v > m || v != v) ? v : m; }

__device__ float block_nan_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < kDarkThreads / 32; ++i) r = nan_max(r, red[i]);
  return r;
}

// The 13 cells the derivatives read, as (dx, dy) around the arg-max, each offset + 2 in 3 bits:
// 0 (0,0), 1 (+1,0), 2 (-1,0), 3 (+2,0), 4 (-2,0), 5 (0,+1), 6 (0,-1), 7 (0,+2), 8 (0,-2),
// 9 (+1,+1), 10 (+1,-1), 11 (-1,+1), 12 (-1,-1)
constexpr uint64_t kDarkCellX = 01133222204132ull;   // octal digits, cell 0 last
constexpr uint64_t kDarkCellY = 01313041322222ull;

__global__ void __launch_bounds__(kDarkThreads)
final_preds_dark_kernel(const float* __restrict__ avg_nhwc, const int* __restrict__ idx, const float* __restrict__ maxval,
                        const double* __restrict__ inv, int ksize, float* __restrict__ preds, int J, int h, int w) {
  extern __shared__ float dark_sm[];
  float* m = dark_sm;               // [h*w] the map
  float* hb = dark_sm + h * w;      // [h*w] the map blurred along x
  __shared__ double wk64[kDarkMaxKernel];
  __shared__ float wk32[kDarkMaxKernel];
  __shared__ float red[2][kDarkThreads / 32];
  __shared__ double gwin[13];
  const int t = blockIdx.x;
  const int b = t / J, j = t - b * J;
  const int hw = h * w, r = ksize / 2;
  const float* src = avg_nhwc + (int64_t)b * hw * J + j;
  float mmax = -INFINITY;
  for (int p = threadIdx.x; p < hw; p += kDarkThreads) {
    const float v = __ldg(src + (int64_t)p * J);
    m[p] = v;
    mmax = nan_max(mmax, v);
  }
  if (threadIdx.x == 0) {
    // sigma_b = 0.3 ((k - 1) / 2 - 1) + 0.8, weights normalised to sum to 1
    const double sigma = 0.3 * ((ksize - 1) * 0.5 - 1.0) + 0.8;
    double sum = 0.0;
    for (int i = 0; i < ksize; ++i) {
      const double d = i - r;
      wk64[i] = exp(-(d * d) / (2.0 * sigma * sigma));
      sum += wk64[i];
    }
    for (int i = 0; i < ksize; ++i) {
      wk64[i] /= sum;
      wk32[i] = (float)wk64[i];
    }
  }
  __syncthreads();
  // max G over the whole map enters only through the 1e-10 clamp: fp32 is enough there
  for (int p = threadIdx.x; p < hw; p += kDarkThreads) {
    const int y = p / w, x = p - y * w;
    float a = 0.f;
    for (int i = 0; i < ksize; ++i) {
      const int xx = x + i - r;
      if (xx >= 0 && xx < w) a = fmaf(wk32[i], m[y * w + xx], a);
    }
    hb[p] = a;
  }
  __syncthreads();
  float gmax = -INFINITY;
  for (int p = threadIdx.x; p < hw; p += kDarkThreads) {
    const int y = p / w, x = p - y * w;
    float a = 0.f;
    for (int i = 0; i < ksize; ++i) {
      const int yy = y + i - r;
      if (yy >= 0 && yy < h) a = fmaf(wk32[i], hb[yy * w + x], a);
    }
    gmax = nan_max(gmax, a);
  }
  mmax = block_nan_max(mmax, red[0]);
  gmax = block_nan_max(gmax, red[1]);

  const float mv = maxval[t];
  float x, y;
  coords_from_argmax(idx[t], mv, w, x, y);
  const int x0 = (int)x, y0 = (int)y;
  if (!(x0 >= 2 && x0 <= w - 3 && y0 >= 2 && y0 <= h - 3)) {
    if (threadIdx.x == 0) store_pred(preds, t, inv + (int64_t)b * 6, x, y, mv);
    return;
  }
  // G at the 13 cells in fp64, straight from the map (zero outside it), in a fixed order
  if (threadIdx.x < 13) {
    const int px = x0 + (int)((kDarkCellX >> (3 * threadIdx.x)) & 7) - 2;
    const int py = y0 + (int)((kDarkCellY >> (3 * threadIdx.x)) & 7) - 2;
    double g = 0.0;
    for (int u = 0; u < ksize; ++u) {
      const int yy = py + u - r;
      if (yy < 0 || yy >= h) continue;
      double row = 0.0;
      for (int v = 0; v < ksize; ++v) {
        const int xx = px + v - r;
        if (xx >= 0 && xx < w) row = fma(wk64[v], (double)m[yy * w + xx], row);
      }
      g = fma(wk64[u], row, g);
    }
    gwin[threadIdx.x] = g;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  // G *= max(M) / max(G) when max(G) > 0; L = log(max(G, 1e-10)), a NaN staying NaN
  const double scale = gmax > 0.f ? (double)mmax / (double)gmax : 1.0;
  double L[13];
#pragma unroll
  for (int i = 0; i < 13; ++i) {
    const double g = gwin[i] * scale;
    L[i] = log(g > 1e-10 || g != g ? g : 1e-10);
  }
  const double dx = 0.5 * (L[1] - L[2]), dy = 0.5 * (L[5] - L[6]);
  const double dxx = 0.25 * (L[3] - 2.0 * L[0] + L[4]), dyy = 0.25 * (L[7] - 2.0 * L[0] + L[8]);
  const double dxy = 0.25 * (L[9] - L[10] - L[11] + L[12]);
  const double det = dxx * dyy - dxy * dxy;
  if (det != 0.0) {
    // offset = -H^-1 (dx, dy), H = [[dxx, dxy], [dxy, dyy]]
    const double ox = -(dyy * dx - dxy * dy) / det, oy = -(dxx * dy - dxy * dx) / det;
    if (isfinite(ox) && isfinite(oy)) {
      x = (float)(x0 + ox);
      y = (float)(y0 + oy);
    }
  }
  store_pred(preds, t, inv + (int64_t)b * 6, x, y, mv);
}

// accuracy(): one warp per (b,j) takes the target's arg-max, lane 0 compares it with the prediction's and adds the
// joint's valid / hit counts. counts must be zero on entry.
__global__ void pck_counts_kernel(const int* __restrict__ idx, const float* __restrict__ maxval,
                                  const float* __restrict__ target, int* __restrict__ counts,
                                  float* __restrict__ pred_hm, int BJ, int J, int h, int w) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= BJ) return;
  const Best tb = warp_argmax(target + (int64_t)warp * h * w, h * w, lane);
  if (lane != 0) return;
  float px, py, tx, ty;
  coords_from_argmax(idx[warp], maxval[warp], w, px, py);
  coords_from_argmax(tb.i, tb.v, w, tx, ty);
  if (pred_hm) {
    pred_hm[(int64_t)warp * 2] = px;
    pred_hm[(int64_t)warp * 2 + 1] = py;
  }
  if (!(tx > 1.f && ty > 1.f)) return;
  // pck_from_preds: float32 differences, normalised in double by (h, w) / 10 -- x by h, y by w, as the reference does
  const double dx = __ddiv_rn((double)__fsub_rn(px, tx), __ddiv_rn((double)h, 10.0));
  const double dy = __ddiv_rn((double)__fsub_rn(py, ty), __ddiv_rn((double)w, 10.0));
  const double d = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
  const int j = warp % J;
  atomicAdd(counts + j * 2, 1);
  if (d < 0.5) atomicAdd(counts + j * 2 + 1, 1);
}

// (1 - f) a + f b with explicit roundings; f == 0 returns a itself (an equal-size resample is an exact copy even next to
// an infinite or NaN neighbour)
__device__ __forceinline__ float lerp_rn(float a, float b, float f) {
  return f == 0.f ? a : __fadd_rn(__fmul_rn(__fsub_rn(1.f, f), a), __fmul_rn(f, b));
}

// heatmap_resample: one thread per output element of an NHWC map; the source position is one fp32 multiply of the
// output pixel index by the host's ratio, clamped to the input (replicate edge), then bilinear
__global__ void heatmap_resample_kernel(const float* __restrict__ in, float* __restrict__ out, int Hi, int Wi, int Ho,
                                        int Wo, int C, float ry, float rx, int64_t total) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int c = (int)(t % C);
  const int64_t p = t / C;
  const int u = (int)(p % Wo);
  const int64_t q = p / Wo;
  const int v = (int)(q % Ho);
  const int64_t b = q / Ho;
  const float x = fminf(fmaxf(__fmul_rn((float)u, rx), 0.f), (float)(Wi - 1));
  const float y = fminf(fmaxf(__fmul_rn((float)v, ry), 0.f), (float)(Hi - 1));
  const int x0 = (int)x, y0 = (int)y;
  const int x1 = min(x0 + 1, Wi - 1), y1 = min(y0 + 1, Hi - 1);
  const float fx = __fsub_rn(x, (float)x0), fy = __fsub_rn(y, (float)y0);
  const float* m = in + b * Hi * Wi * C + c;
  const float top = lerp_rn(__ldg(m + ((int64_t)y0 * Wi + x0) * C), __ldg(m + ((int64_t)y0 * Wi + x1) * C), fx);
  const float bot = lerp_rn(__ldg(m + ((int64_t)y1 * Wi + x0) * C), __ldg(m + ((int64_t)y1 * Wi + x1) * C), fx);
  out[t] = lerp_rn(top, bot, fy);
}

}  // namespace
}  // namespace fpd

using namespace fpd;

extern "C" {

int fpd_flip_merge_argmax(const float* hm, const float* hm_flip, const int* flip_perm, int shift, float* avg_nhwc,
                          int* idx, float* maxval, int B, int J, int h, int w, fpd_stream_t stream) {
  FPD_REQUIRE(J >= 1 && J <= 64, "flip_merge_argmax: J=%d out of range", J);
  const int threads = (512 / J) * J;
  const size_t smem = (size_t)threads * sizeof(Best);
  flip_merge_argmax_kernel<<<B, threads, smem, stream>>>(hm, hm_flip, flip_perm, shift, avg_nhwc, idx, maxval, J, h,
                                                         w);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_argmax_nchw(const float* hm, int* idx, float* maxval, int BJ, int hw, fpd_stream_t stream) {
  const int threads = 256;
  const int blocks = (BJ * 32 + threads - 1) / threads;
  argmax_nchw_kernel<<<blocks, threads, 0, stream>>>(hm, idx, maxval, BJ, hw);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_final_preds(const float* avg_nhwc, const int* idx, const float* maxval, const double* inv, int post_process,
                    float* preds, int B, int J, int h, int w, fpd_stream_t stream) {
  FPD_REQUIRE(B >= 0 && J >= 1 && J <= 64, "final_preds: B=%d J=%d out of range", B, J);
  FPD_REQUIRE(h >= 1 && w >= 1, "final_preds: empty %dx%d heat-map", h, w);
  FPD_REQUIRE(!post_process || (h >= 3 && w >= 3), "final_preds: post_process needs a heat-map of at least 3x3, got %dx%d",
              h, w);
  FPD_REQUIRE(idx && maxval && inv && preds && (avg_nhwc || !post_process), "final_preds: null pointer");
  if (B == 0) return FPD_OK;
  const int BJ = B * J, threads = 128;
  final_preds_kernel<<<(BJ + threads - 1) / threads, threads, 0, stream>>>(avg_nhwc, idx, maxval, inv, post_process,
                                                                           preds, BJ, J, h, w);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_final_preds_dark(const float* avg_nhwc, const int* idx, const float* maxval, const double* inv, int blur_kernel,
                         float* preds, int B, int J, int h, int w, fpd_stream_t stream) {
  FPD_REQUIRE(B >= 0 && J >= 1 && J <= 64, "final_preds_dark: B=%d J=%d out of range", B, J);
  FPD_REQUIRE(h >= 5 && w >= 5, "final_preds_dark: needs a heat-map of at least 5x5, got %dx%d", h, w);
  FPD_REQUIRE(blur_kernel >= 3 && blur_kernel <= kDarkMaxKernel && blur_kernel % 2 == 1,
              "final_preds_dark: blur_kernel=%d must be odd and in [3, %d]", blur_kernel, kDarkMaxKernel);
  FPD_REQUIRE(avg_nhwc && idx && maxval && inv && preds, "final_preds_dark: null pointer");
  const size_t smem = (size_t)2 * h * w * sizeof(float);
  FPD_REQUIRE(smem <= kDarkSmemLimit, "final_preds_dark: a %dx%d heat-map does not fit in shared memory", h, w);
  if (B == 0) return FPD_OK;
  if (smem > 48 * 1024)
    FPD_CUDA_CHECK(cudaFuncSetAttribute(final_preds_dark_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)kDarkSmemLimit));
  final_preds_dark_kernel<<<B * J, kDarkThreads, smem, stream>>>(avg_nhwc, idx, maxval, inv, blur_kernel, preds, J, h, w);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_pck_counts(const int* idx, const float* maxval, const float* target_nchw, int* counts, float* pred_hm, int B,
                   int J, int h, int w, fpd_stream_t stream) {
  FPD_REQUIRE(B >= 0 && J >= 1 && J <= 64, "pck_counts: B=%d J=%d out of range", B, J);
  FPD_REQUIRE(h >= 1 && w >= 1, "pck_counts: empty %dx%d heat-map", h, w);
  FPD_REQUIRE(idx && maxval && target_nchw && counts, "pck_counts: null pointer");
  FPD_CUDA_CHECK(cudaMemsetAsync(counts, 0, (size_t)J * 2 * sizeof(int), stream));
  if (B == 0) return FPD_OK;
  const int BJ = B * J, threads = 256;
  pck_counts_kernel<<<(BJ * 32 + threads - 1) / threads, threads, 0, stream>>>(idx, maxval, target_nchw, counts, pred_hm,
                                                                              BJ, J, h, w);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

int fpd_heatmap_resample(const float* in, float* out, int B, int Hi, int Wi, int Ho, int Wo, int C, int udp,
                         fpd_stream_t stream) {
  FPD_REQUIRE(B >= 0 && C >= 1 && C <= 64, "heatmap_resample: B=%d C=%d out of range", B, C);
  FPD_REQUIRE(Hi >= 1 && Wi >= 1 && Ho >= 1 && Wo >= 1, "heatmap_resample: empty map %dx%d -> %dx%d", Hi, Wi, Ho, Wo);
  FPD_REQUIRE(in && out, "heatmap_resample: null pointer");
  if (B == 0) return FPD_OK;
  // reference crops: output pixel u is the box fraction u / Wo, so u_in = u * Wi / Wo; UDP crops measure sizes in pixel
  // spacings, so u_in = u * (Wi - 1) / (Wo - 1). The ratio is rounded to fp32 once, here.
  const float rx = udp ? (Wo > 1 ? (float)((double)(Wi - 1) / (Wo - 1)) : 0.f) : (float)((double)Wi / Wo);
  const float ry = udp ? (Ho > 1 ? (float)((double)(Hi - 1) / (Ho - 1)) : 0.f) : (float)((double)Hi / Ho);
  const int64_t total = (int64_t)B * Ho * Wo * C;
  const int threads = 256;
  heatmap_resample_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, stream>>>(in, out, Hi, Wi, Ho, Wo, C,
                                                                                              ry, rx, total);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // extern "C"
