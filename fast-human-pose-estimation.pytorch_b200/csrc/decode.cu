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
  // transform_preds evaluates coords @ t[:, :2].T + t[:, 2] through numpy's matmul, whose OpenBLAS dgemm rounds x*t0,
  // adds y*t1 in one fused multiply-add, then adds t2. Plain multiply-then-add differs in the last double bit, and
  // now and then in the float32 result.
  const double* T = inv + (int64_t)b * 6;
  const double xd = x, yd = y;
  preds[(int64_t)t * 3 + 0] = (float)__dadd_rn(__fma_rn(yd, T[1], __dmul_rn(xd, T[0])), T[2]);
  preds[(int64_t)t * 3 + 1] = (float)__dadd_rn(__fma_rn(yd, T[4], __dmul_rn(xd, T[3])), T[5]);
  preds[(int64_t)t * 3 + 2] = mv;
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

}  // extern "C"
