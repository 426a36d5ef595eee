// augment.cu -- batched affine crop + normalisation of training images: cv2.warpAffine(INTER_LINEAR, BORDER_CONSTANT=0) on
// 8-bit 3-channel images followed by torchvision ToTensor + Normalize, bit for bit (lib/dataset/JointsDataset.py:177-184 of
// the reference). The source of each sample is the uint8 HWC region of its (already mirrored / colour-converted) image that
// the crop reads; taps outside that region lie outside the image and contribute 0.
//
// Fixed-point model of cv2 4.x (imgwarp.cpp, 8-bit INTER_LINEAR): coordinates in 1/1024 pixel rounded half to even
// (cvRound), then 1/32-pixel bilinear weights with 15 fractional bits.
#include <cmath>

#include "common.cuh"

namespace fpd {
namespace {

constexpr int kThreads = 256;
constexpr int kAbBits = 10;                                     // cv2 AB_BITS
constexpr int kInterBits = 5;                                   // cv2 INTER_BITS: 32 sub-pixel phases per axis
constexpr int kRoundDelta = (1 << kAbBits) / (1 << kInterBits) / 2;
constexpr double kAbScale = 1 << kAbBits;
constexpr int kMaxImageSide = 32767;                            // cv2 keeps integer tap positions in int16
constexpr int kCropDescLen = 7;                                 // byte offset, region x, y, w, h, image w, h

struct Norm {
  float mean[3], std[3];
};

__global__ void __launch_bounds__(kThreads)
crop_affine_normalize_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ desc,
                             const double* __restrict__ inv, Norm norm, float* __restrict__ out, int oh, int ow) {
  const int n = blockIdx.y;
  const int p = blockIdx.x * kThreads + threadIdx.x;
  if (p >= oh * ow) return;
  const int y = p / ow, x = p - y * ow;
  const int64_t* d = desc + (size_t)n * kCropDescLen;
  const uint8_t* reg = src + d[0];
  const int rx = (int)d[1], ry = (int)d[2], rw = (int)d[3], rh = (int)d[4];
  const double* m = inv + (size_t)n * 6;
  // explicit round-to-nearest products and sums: no FMA contraction, as in the host build of cv2
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], (double)y), m[2]), kAbScale)) + kRoundDelta;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], (double)y), m[5]), kAbScale)) + kRoundDelta;
  const int X = (X0 + __double2int_rn(__dmul_rn(__dmul_rn(m[0], (double)x), kAbScale))) >> (kAbBits - kInterBits);
  const int Y = (Y0 + __double2int_rn(__dmul_rn(__dmul_rn(m[3], (double)x), kAbScale))) >> (kAbBits - kInterBits);
  const int ax = X & ((1 << kInterBits) - 1), ay = Y & ((1 << kInterBits) - 1);
  const int xi = (X >> kInterBits) - rx, yi = (Y >> kInterBits) - ry;
  const int w[4] = {(32 - ax) * (32 - ay) * 32, ax * (32 - ay) * 32, (32 - ax) * ay * 32, ax * ay * 32};
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int tx = xi + (t & 1), ty = yi + (t >> 1);
    if (tx >= 0 && tx < rw && ty >= 0 && ty < rh) {
      const uint8_t* s = reg + ((size_t)ty * rw + tx) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] += (int)s[c] * w[t];
    }
  }
  float* o = out + (size_t)n * 3 * oh * ow + p;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int u8 = min(max((acc[c] + (1 << 14)) >> 15, 0), 255);
    // ToTensor divides by 255, Normalize subtracts the mean and divides by the deviation: two IEEE divisions
    o[(size_t)c * oh * ow] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)u8, 255.0f), norm.mean[c]), norm.std[c]);
  }
}

// largest |rne(v * 1024)| over the end points of v = a * t + b, t in {0, tmax} (affine, so they bound every t between)
double fixed_extent(double a, double b, int tmax) {
  return fmax(fabs(b), fabs(a * tmax + b)) * kAbScale + 1.0;
}

}  // namespace
}  // namespace fpd

using namespace fpd;

extern "C" {

int fpd_crop_affine_normalize(const uint8_t* src, size_t src_bytes, const int64_t* desc, const double* inv,
                              const int64_t* desc_host, const double* inv_host, const float* mean_std_host, float* out,
                              int N, int out_h, int out_w, fpd_stream_t stream) {
  FPD_REQUIRE(N >= 0, "crop_affine_normalize: N=%d < 0", N);
  FPD_REQUIRE(out_h >= 1 && out_w >= 1, "crop_affine_normalize: empty output %dx%d", out_h, out_w);
  FPD_REQUIRE(N <= 65535 && (int64_t)out_h * out_w <= (1 << 24),
              "crop_affine_normalize: N=%d / output %dx%d too large", N, out_h, out_w);
  if (N == 0) return FPD_OK;
  FPD_REQUIRE(desc && inv && desc_host && inv_host && mean_std_host && out && (src || src_bytes == 0),
              "crop_affine_normalize: null pointer");
  Norm norm;
  for (int c = 0; c < 3; ++c) {
    norm.mean[c] = mean_std_host[c];
    norm.std[c] = mean_std_host[3 + c];
  }
  const double limit = 2147483647.0 - kRoundDelta;
  for (int n = 0; n < N; ++n) {
    const int64_t* d = desc_host + (size_t)n * kCropDescLen;
    const int64_t off = d[0], rx = d[1], ry = d[2], rw = d[3], rh = d[4], iw = d[5], ih = d[6];
    FPD_REQUIRE(iw >= 1 && ih >= 1 && iw <= kMaxImageSide && ih <= kMaxImageSide,
                "crop_affine_normalize: sample %d: image %lldx%lld outside [1, %d]", n, (long long)iw, (long long)ih,
                kMaxImageSide);
    FPD_REQUIRE(rx >= 0 && ry >= 0 && rw >= 0 && rh >= 0 && rx + rw <= iw && ry + rh <= ih,
                "crop_affine_normalize: sample %d: region (%lld,%lld) %lldx%lld not inside the %lldx%lld image", n,
                (long long)rx, (long long)ry, (long long)rw, (long long)rh, (long long)iw, (long long)ih);
    FPD_REQUIRE(off >= 0 && (uint64_t)off + (uint64_t)(rw * rh * 3) <= (uint64_t)src_bytes,
                "crop_affine_normalize: sample %d: region bytes [%lld, +%lld) outside the %zu-byte buffer", n,
                (long long)off, (long long)(rw * rh * 3), src_bytes);
    const double* m = inv_host + (size_t)n * 6;
    bool finite = true;
    for (int k = 0; k < 6; ++k) finite = finite && std::isfinite(m[k]);
    FPD_REQUIRE(finite, "crop_affine_normalize: sample %d: inverse matrix is not finite", n);
    // X =(rne((A12 y + b1) 1024) + 16 + rne(A11 x 1024)) >> 5 must not overflow int32 anywhere on the output (same for Y)
    const double ex = fixed_extent(m[1], m[2], out_h - 1) + fixed_extent(m[0], 0.0, out_w - 1);
    const double ey = fixed_extent(m[4], m[5], out_h - 1) + fixed_extent(m[3], 0.0, out_w - 1);
    FPD_REQUIRE(ex < limit && ey < limit,
                "crop_affine_normalize: sample %d: inverse matrix [%g %g %g; %g %g %g] overflows the fixed-point "
                "coordinates", n, m[0], m[1], m[2], m[3], m[4], m[5]);
  }
  const dim3 grid((unsigned)((out_h * out_w + kThreads - 1) / kThreads), (unsigned)N);
  crop_affine_normalize_kernel<<<grid, kThreads, 0, stream>>>(src, desc, inv, norm, out, out_h, out_w);
  FPD_LAUNCH_CHECK();
  return FPD_OK;
}

}  // extern "C"
