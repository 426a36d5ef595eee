// api.cu -- the extern "C" surface declared in include/fpd_b200.h: thin argument-checking wrappers over
// the launchers in kernels.h, the thread-local error string and the `_nms`-compatible host entry point.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <atomic>
#include <mutex>

#include "../../include/fpd_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace fpd {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

}  // namespace fpd

using namespace fpd;
#define S(x) reinterpret_cast<cudaStream_t>(x)

extern "C" {

const char* fpd_last_error(void) { return fpd::g_err; }
int fpd_version(void) { return 100; }
int fpd_sm_count(void) { return device_sm_count(); }
long long fpd_launch_count(void) { return fpd::g_launches.load(std::memory_order_relaxed); }




int fpd_conv2d_tc_ts_supported(int Cin, int Cout, int ksize) { return conv_tc_ts_supported(Cin, Cout, ksize) ? 1 : 0; }

int fpd_conv2d_tc_ts(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                     int pre_relu, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                     const float* relu_mask, float* y, float out_scale, int B, int H, int W, int Cin, int Cout,
                     int ksize, fpd_stream_t stream) {
  return conv_tc_ts_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, bias, residual, relu_mask, y,
                           out_scale, B, H, W, Cin, Cout, ksize, device_sm_count(), S(stream));
}


int fpd_conv2d_tc_h_supported(int Cin, int Cout, int ksize, int H, int W, int f16) {
  return conv_tc_h_supported(Cin, Cout, ksize, H, W, f16) ? 1 : 0;
}

int fpd_conv2d_tc_h(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                    int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                    const float* residual, const float* relu_mask, float* y, float out_scale, const float* in_scale,
                    int B, int H, int W, int Cin, int Cout, int ksize, fpd_stream_t stream) {
  return conv_tc_h_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, f16, bias, residual, relu_mask, y,
                          out_scale, in_scale, B, H, W, Cin, Cout, ksize, device_sm_count(), S(stream));
}

int fpd_conv2d_tc_f16x1_kernel(int B, int H, int W, int Cin, int Cout, int ksize) {
  return conv_f16x1_kernel(B, H, W, Cin, Cout, ksize, 0, 0, nullptr);
}

int fpd_conv2d_tc_f16x1(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                        int pre_relu, const void* w, const float* bias, const float* residual, const float* relu_mask,
                        float* y, float out_scale, int B, int H, int W, int Cin, int Cout, int ksize,
                        fpd_stream_t stream) {
  return conv_f16x1_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w, bias, residual, relu_mask, y, out_scale,
                           nullptr, B, H, W, Cin, Cout, ksize, device_sm_count(), S(stream), nullptr, nullptr);
}

int fpd_conv2d_tc_f16x1_io(const void* x, int x_f16, const float* pre_mean, const float* pre_scale,
                           const float* pre_shift, int pre_relu, const void* w, const float* bias, const void* residual,
                           void* y, int y_f16, float out_scale, int B, int H, int W, int Cin, int Cout, int ksize,
                           fpd_stream_t stream) {
  return conv_f16x1_io_launch(x, x_f16, pre_mean, pre_scale, pre_shift, pre_relu, w, bias, residual, y, y_f16,
                              out_scale, B, H, W, Cin, Cout, ksize, device_sm_count(), S(stream));
}

int fpd_conv2d_tc_f16x1_train_plan(int B, int H, int W, int Cin, int Cout, int ksize, int stats, int* stat_blocks) {
  return conv_f16x1_kernel(B, H, W, Cin, Cout, ksize, stats, device_sm_count(), stat_blocks);
}

int fpd_conv2d_tc_f16x1_train(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                              int pre_relu, const void* w, const float* bias, const float* residual,
                              const float* relu_mask, float* y, float out_scale, const float* in_scale, int B, int H,
                              int W, int Cin, int Cout, int ksize, double* stat_part, const float* stat_pivot,
                              fpd_stream_t stream) {
  return conv_f16x1_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w, bias, residual, relu_mask, y, out_scale,
                           in_scale, B, H, W, Cin, Cout, ksize, device_sm_count(), S(stream), stat_part, stat_pivot);
}

int fpd_set_conv1x1(int enabled) { return set_conv1x1(enabled); }
int fpd_set_conv_halo(int enabled) { return set_conv_halo(enabled); }
int fpd_set_wgrad_halo(int enabled) { return set_wgrad_halo(enabled); }

int fpd_conv2d_tc_h_stats_blocks(int B, int H, int W, int Cin, int Cout, int ksize, int f16) {
  return conv_tc_h_stats_grid(B, H, W, Cin, Cout, ksize, f16, device_sm_count());
}
int fpd_conv2d_tc_h_stats(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                          int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                          const float* residual, float* y, float out_scale, int B, int H, int W, int Cin, int Cout,
                          int ksize, double* stat_part, const float* stat_pivot, fpd_stream_t stream) {
  FPD_REQUIRE(stat_part != nullptr, "fpd_conv2d_tc_h_stats: stat_part is NULL (use fpd_conv2d_tc_h)");
  return conv_tc_h_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, w_hi, w_lo, f16, bias, residual, nullptr, y,
                          out_scale, nullptr, B, H, W, Cin, Cout, ksize, device_sm_count(), S(stream), stat_part,
                          stat_pivot);
}
int fpd_bn_finalize_sums(const double* part, int nblocks, const float* pivot, int64_t P, int C, const float* gamma,
                         const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                         float* mean, float* var_biased, float* scale, float* shift, float* invstd,
                         fpd_stream_t stream) {
  return bn_finalize_sums(part, nblocks, pivot, P, C, gamma, beta, eps, momentum, running_mean, running_var, mean,
                          var_biased, scale, shift, invstd, S(stream));
}

int fpd_channel_sum_fused(const float* dy, int64_t P, int C, float scale, float* out, float* amax_scale,
                          void* workspace, size_t workspace_bytes, unsigned int* counter, fpd_stream_t stream) {
  return channel_sum_fused(dy, P, C, scale, out, amax_scale, workspace, workspace_bytes, counter, S(stream));
}
int fpd_bn_bwd_reduce_fused(const float* da, const float* x, const float* mean, const float* invstd,
                            const float* scale, const float* shift, int relu, int64_t P, int C, float* sums,
                            void* workspace, size_t workspace_bytes, unsigned int* counter, fpd_stream_t stream) {
  return bn_bwd_reduce_fused(da, x, mean, invstd, scale, shift, relu, P, C, sums, workspace, workspace_bytes, counter,
                             S(stream));
}
int fpd_bn_stats_fused(const float* x, int64_t P, int C, const float* gamma, const float* beta, float eps,
                       float momentum, float* running_mean, float* running_var, float* mean, float* var_biased,
                       float* scale, float* shift, float* invstd, void* workspace, size_t workspace_bytes,
                       unsigned int* counter, fpd_stream_t stream) {
  return bn_stats_fused(x, P, C, gamma, beta, eps, momentum, running_mean, running_var, mean, var_biased, scale, shift,
                        invstd, workspace, workspace_bytes, counter, S(stream));
}

int fpd_weight_prep_f16(const float* w, void* w_hi, void* w_lo, int O, int I, int k, int for_dgrad,
                        fpd_stream_t stream) {
  return weight_prep_f16(w, w_hi, w_lo, O, I, k, for_dgrad, S(stream));
}

int fpd_weight_prep_f16_both(const float* w, void* f_hi, void* f_lo, void* d_hi, void* d_lo, int O, int I, int k,
                             fpd_stream_t stream) {
  return weight_prep_f16_both(w, f_hi, f_lo, d_hi, d_lo, O, I, k, S(stream));
}

int fpd_conv2d_wgrad_tc3_supported(int H, int W, int Cin, int Cout, int ksize) {
  return wgrad_tc3_supported(H, W, Cin, Cout, ksize) ? 1 : 0;
}
int fpd_conv2d_wgrad_tc_supported(int Cin, int Cout, int ksize) {
  return wgrad_tc_supported(Cin, Cout, ksize) ? 1 : 0;
}
size_t fpd_conv2d_wgrad_tc_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize) {
  return wgrad_tc_workspace_bytes(B, H, W, Cin, Cout, ksize, device_sm_count());
}

int fpd_conv2d_wgrad_tc_fused(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                              int pre_relu, const float* dy, int passes, float* dw_oihw, float scale, int B, int H,
                              int W, int Cin, int Cout, int ksize, void* workspace, size_t workspace_bytes,
                              fpd_stream_t stream) {
  return wgrad_tc_fused_launch(x, pre_mean, pre_scale, pre_shift, pre_relu, dy, passes, dw_oihw, scale, B, H, W, Cin,
                               Cout, ksize, workspace, workspace_bytes, device_sm_count(), S(stream));
}

int fpd_conv2d_simt_fwd(const float* x, const float* w, const float* bias, const float* residual, float* y, int B,
                        int H, int W, int Cin, int Cout, int k, int stride, int pad, fpd_stream_t stream) {
  return conv_simt_fwd(x, w, bias, residual, y, B, H, W, Cin, Cout, k, stride, pad, S(stream));
}
int fpd_conv2d_simt_dgrad(const float* dy, const float* w, float* dx, int B, int H, int W, int Cin, int Cout, int k,
                          int stride, int pad, fpd_stream_t stream) {
  return conv_simt_dgrad(dy, w, dx, B, H, W, Cin, Cout, k, stride, pad, S(stream));
}
size_t fpd_conv2d_simt_wgrad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k, int stride, int pad) {
  return conv_simt_wgrad_workspace_bytes(B, H, W, Cin, Cout, k, stride, pad);
}
int fpd_conv2d_simt_wgrad(const float* x, const float* dy, float* dw, float scale, int B, int H, int W, int Cin,
                          int Cout, int k, int stride, int pad, void* workspace, size_t workspace_bytes,
                          fpd_stream_t stream) {
  return conv_simt_wgrad(x, dy, dw, scale, B, H, W, Cin, Cout, k, stride, pad, workspace, workspace_bytes, S(stream));
}
int fpd_weight_prep(const float* w, float* w_hi, float* w_lo, int O, int I, int k, int for_dgrad,
                    fpd_stream_t stream) {
  return weight_prep(w, w_hi, w_lo, O, I, k, for_dgrad, S(stream));
}

size_t fpd_bn_stats_workspace_bytes(int64_t P, int C) { return bn_stats_workspace_bytes(P, C); }
int fpd_bn_stats(const float* x, int64_t P, int C, float* mean, float* var, void* ws, size_t wsb,
                 fpd_stream_t stream) {
  return bn_stats(x, P, C, mean, var, ws, wsb, S(stream));
}
int fpd_bn_finalize(const float* mean, const float* var, const float* gamma, const float* beta, float eps,
                    int64_t count, float* scale, float* shift, float* invstd, float* rmean, float* rvar,
                    float momentum, int C, fpd_stream_t stream) {
  return bn_finalize(mean, var, gamma, beta, eps, count, scale, shift, invstd, rmean, rvar, momentum, C, S(stream));
}
int fpd_affine_act_split(const float* x, const float* mean, const float* scale, const float* shift, int relu,
                         float* a_hi, float* a_lo, int64_t P, int C, fpd_stream_t stream) {
  return affine_act_split(x, mean, scale, shift, relu, a_hi, a_lo, P, C, S(stream));
}
int fpd_affine_act(const float* x, const float* mean, const float* scale, const float* shift, int relu, float* y,
                   int64_t P, int C, fpd_stream_t stream) {
  return affine_act(x, mean, scale, shift, relu, y, P, C, S(stream));
}
int fpd_affine_add_act(const float* x, const float* mean, const float* scale, const float* shift,
                       const float* residual, int relu, float* y, int64_t P, int C, fpd_stream_t stream) {
  return affine_add_act(x, mean, scale, shift, residual, relu, y, P, C, S(stream));
}
int fpd_fuse_sum(const float* const* terms_host, const int* shifts_host, int n, int relu, float* out, int B, int H,
                 int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(terms_host && shifts_host, "fpd_fuse_sum: NULL term table");
  return fuse_sum(terms_host, shifts_host, n, relu, out, B, H, W, C, S(stream));
}
int fpd_upsample_bwd(const float* dout, float* dlow, int shift, int B, int H, int W, int C, fpd_stream_t stream) {
  return upsample_bwd(dout, dlow, shift, B, H, W, C, S(stream));
}
int fpd_im2col(const float* x, float* cols, int B, int H, int W, int Cin, int k, int stride, int pad, int Kpad,
               fpd_stream_t stream) {
  return im2col(x, cols, B, H, W, Cin, k, stride, pad, Kpad, S(stream));
}
size_t fpd_channel_reduce_workspace_bytes(int64_t P, int C) { return channel_reduce_workspace_bytes(P, C); }
int fpd_channel_sum(const float* dy, int64_t P, int C, float scale, float* out, void* ws, size_t wsb,
                    fpd_stream_t stream) {
  return channel_sum(dy, P, C, scale, out, ws, wsb, S(stream));
}
int fpd_bn_bwd_reduce(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                      const float* shift, int relu, int64_t P, int C, float* sums, void* ws, size_t wsb,
                      fpd_stream_t stream) {
  return bn_bwd_reduce(da, x, mean, invstd, scale, shift, relu, P, C, sums, ws, wsb, S(stream));
}
int fpd_bn_bwd_apply_sum(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                         const float* shift, const float* gamma, int relu, const float* sums, float* dx, float* dx_sum,
                         float* amax_scale, int64_t P, int C, void* ws, size_t wsb, fpd_stream_t stream) {
  return bn_bwd_apply_sum(da, x, mean, invstd, scale, shift, gamma, relu, sums, dx, dx_sum, amax_scale, P, C, ws, wsb,
                          S(stream));
}
int fpd_bn_bwd_apply(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                     const float* shift, const float* gamma, int relu, const float* sums, int accumulate, float* dx,
                     int64_t P, int C, fpd_stream_t stream) {
  return bn_bwd_apply(da, x, mean, invstd, scale, shift, gamma, relu, sums, accumulate, dx, P, C, S(stream));
}
int fpd_affine_act_bwd(const float* da, const float* x, const float* mean, const float* scale, const float* shift,
                       int relu, int accumulate, float* dx, int64_t P, int C, fpd_stream_t stream) {
  return affine_act_bwd(da, x, mean, scale, shift, relu, accumulate, dx, P, C, S(stream));
}
int fpd_maxpool2x2_fwd(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream) {
  return maxpool2x2_fwd(x, y, B, H, W, C, S(stream));
}
int fpd_maxpool2x2_bwd(const float* x, const float* dy, float* dx, int accumulate, int B, int H, int W, int C,
                       fpd_stream_t stream) {
  return maxpool2x2_bwd(x, dy, dx, accumulate, B, H, W, C, S(stream));
}
int fpd_upsample2x_add(const float* up1, const float* low, float* out, int B, int H, int W, int C,
                       fpd_stream_t stream) {
  return upsample2x_add(up1, low, out, B, H, W, C, S(stream));
}
int fpd_upsample2x_bwd(const float* dout, float* dlow, int B, int H, int W, int C, fpd_stream_t stream) {
  return upsample2x_bwd(dout, dlow, B, H, W, C, S(stream));
}
int fpd_maxpool3x3s2_fwd(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream) {
  return maxpool3x3s2_fwd(x, y, B, H, W, C, S(stream));
}
int fpd_maxpool3x3s2_bwd(const float* x, const float* dy, float* dx, int accumulate, int B, int H, int W, int C,
                         fpd_stream_t stream) {
  return maxpool3x3s2_bwd(x, dy, dx, accumulate, B, H, W, C, S(stream));
}
int fpd_depth_space2(const float* src, float* dst, int B, int H, int W, int C, int to_depth, fpd_stream_t stream) {
  return depth_space2(src, dst, B, H, W, C, to_depth, S(stream));
}
int fpd_deconv_weight_map(const float* src, float* dst, int Cin, int Cout, int k, int pad, int to_deconv,
                          fpd_stream_t stream) {
  return deconv_weight_map(src, dst, Cin, Cout, k, pad, to_deconv, S(stream));
}
int fpd_subsample2(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream) {
  return subsample2(x, y, B, H, W, C, S(stream));
}
int fpd_upsample_zero2(const float* dy, float* dx, int B, int Ho, int Wo, int C, fpd_stream_t stream) {
  return upsample_zero2(dy, dx, B, Ho, Wo, C, S(stream));
}
int fpd_affine_act_f16(const void* x, const float* mean, const float* scale, const float* shift, int relu, void* y,
                       int64_t P, int C, fpd_stream_t stream) {
  return affine_act_f16(x, mean, scale, shift, nullptr, relu, y, P, C, S(stream));
}
int fpd_affine_add_act_f16(const void* x, const float* mean, const float* scale, const float* shift,
                           const void* residual, int relu, void* y, int64_t P, int C, fpd_stream_t stream) {
  FPD_REQUIRE(residual, "fpd_affine_add_act_f16: NULL residual");
  return affine_act_f16(x, mean, scale, shift, residual, relu, y, P, C, S(stream));
}
int fpd_fuse_sum_f16(const void* const* terms_host, const int* shifts_host, int n, int relu, void* out, int B, int H,
                     int W, int C, fpd_stream_t stream) {
  FPD_REQUIRE(terms_host && shifts_host, "fpd_fuse_sum_f16: NULL term table");
  return fuse_sum_f16(terms_host, shifts_host, n, relu, out, B, H, W, C, S(stream));
}
int fpd_maxpool2x2_fwd_f16(const void* x, void* y, int B, int H, int W, int C, fpd_stream_t stream) {
  return maxpool2x2_fwd_f16(x, y, B, H, W, C, S(stream));
}
int fpd_upsample2x_add_f16(const void* up1, const void* low, void* out, int B, int H, int W, int C,
                           fpd_stream_t stream) {
  return upsample2x_add_f16(up1, low, out, B, H, W, C, S(stream));
}
int fpd_subsample2_f16(const void* x, void* y, int B, int H, int W, int C, fpd_stream_t stream) {
  return subsample2_f16(x, y, B, H, W, C, S(stream));
}
int fpd_half_to_float(const void* x, float* y, int64_t n, fpd_stream_t stream) {
  return half_to_float(x, y, n, S(stream));
}
int fpd_nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, fpd_stream_t stream) {
  return nchw_to_nhwc(x, y, B, C, H, W, S(stream));
}
int fpd_nchw_to_nhwc_flipw(const float* x, float* y, int B, int C, int H, int W, fpd_stream_t stream) {
  return nchw_to_nhwc_flipw(x, y, B, C, H, W, S(stream));
}
int fpd_nhwc_to_nchw(const float* x, float* y, int B, int C, int H, int W, fpd_stream_t stream) {
  return nhwc_to_nchw(x, y, B, C, H, W, S(stream));
}
int fpd_add(const float* a, const float* b, float* out, int64_t n, fpd_stream_t stream) {
  return add_tensors(a, b, out, n, S(stream));
}

size_t fpd_loss_workspace_bytes(int B, int J, int h, int w) { return fpd::fpd_loss_workspace_bytes(B, J, h, w); }
int fpd_loss_fused(const float* const* outs_host, int Sn, const float* target_nchw, const float* teacher_nhwc,
                   const float* tw, float alpha, float* const* grads_host, float grad_scale, float* losses, int B,
                   int J, int h, int w, void* ws, size_t wsb, fpd_stream_t stream) {
  FPD_REQUIRE(outs_host != nullptr, "fpd_loss_fused: outs_host is NULL");
  return fpd::fpd_loss(outs_host, Sn, target_nchw, teacher_nhwc, tw, alpha, grads_host, grad_scale, losses, B, J, h,
                       w, ws, wsb, S(stream));
}
int fpd_joints_mse(const float* out, const float* target, const float* tw, float* loss3, float* grad, int B, int J,
                   int hw, void* ws, size_t wsb, fpd_stream_t stream) {
  return joints_mse(out, target, tw, loss3, grad, 1.f, B, J, hw, ws, wsb, S(stream));
}
size_t fpd_loss_ohkm_workspace_bytes(int Sn, int B, int J, int h, int w) {
  return fpd::fpd_loss_ohkm_workspace_bytes(Sn, B, J, h, w);
}
int fpd_loss_ohkm_fused(const float* const* outs_host, int Sn, const float* target_nchw, const float* teacher_nhwc,
                        const float* tw, float alpha, float* const* grads_host, float grad_scale, float* losses, int B,
                        int J, int h, int w, int pose_topk, int kd_topk, void* ws, size_t wsb, fpd_stream_t stream) {
  FPD_REQUIRE(outs_host != nullptr, "fpd_loss_ohkm_fused: outs_host is NULL");
  return fpd::fpd_loss_ohkm(outs_host, Sn, target_nchw, teacher_nhwc, tw, alpha, grads_host, grad_scale, losses, B, J,
                            h, w, pose_topk, kd_topk, ws, wsb, S(stream));
}
size_t fpd_joints_ohkm_workspace_bytes(int B, int J) { return joints_ohkm_workspace_bytes(B, J); }
int fpd_joints_ohkm(const float* out, const float* target, const float* tw, int topk, float* loss3, float* grad, int B,
                    int J, int hw, void* ws, size_t wsb, fpd_stream_t stream) {
  return joints_ohkm(out, target, tw, topk, loss3, grad, B, J, hw, ws, wsb, S(stream));
}

int fpd_flip_merge_argmax(const float* hm, const float* hm_flip, const int* perm, int shift, float* avg_nhwc,
                          int* idx, float* maxval, int B, int J, int h, int w, fpd_stream_t stream) {
  return flip_merge_argmax(hm, hm_flip, perm, shift, avg_nhwc, idx, maxval, B, J, h, w, S(stream));
}
int fpd_argmax_nchw(const float* hm, int* idx, float* maxval, int BJ, int hw, fpd_stream_t stream) {
  return argmax_nchw(hm, idx, maxval, BJ, hw, S(stream));
}
int fpd_final_preds(const float* avg_nhwc, const int* idx, const float* maxval, const double* inv, int post_process,
                    float* preds, int B, int J, int h, int w, fpd_stream_t stream) {
  return final_preds(avg_nhwc, idx, maxval, inv, post_process, preds, B, J, h, w, S(stream));
}
int fpd_pck_counts(const int* idx, const float* maxval, const float* target_nchw, int* counts, float* pred_hm, int B,
                   int J, int h, int w, fpd_stream_t stream) {
  return pck_counts(idx, maxval, target_nchw, counts, pred_hm, B, J, h, w, S(stream));
}

size_t fpd_nms_workspace_bytes(int n) { return nms_workspace_bytes(n); }
int fpd_nms_device(const float* boxes, int n, int box_dim, float thresh, int* keep, int* num_keep, void* ws,
                   size_t wsb, fpd_stream_t stream) {
  return nms_device(boxes, n, box_dim, thresh, keep, num_keep, ws, wsb, S(stream));
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
  const size_t need = boxes_pad + keep_pad + 256 + nms_workspace_bytes(boxes_num);
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
    rc = nms_device(boxes_dev, boxes_num, boxes_dim, thresh, keep_dev, num_dev, ws, nms_workspace_bytes(boxes_num), st);
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

int fpd_oks_nms_device(const void* kpts_sorted, int kpt_f64, const double* areas_sorted, const double* vars_, int n, int J,
                       double thresh, int use_vis, double in_vis_thre, int* keep, int* num_keep, void* ws, size_t wsb,
                       fpd_stream_t stream) {
  return oks_nms_device(kpts_sorted, kpt_f64, areas_sorted, vars_, n, J, thresh, use_vis, in_vis_thre, keep, num_keep, ws,
                        wsb, S(stream));
}
int fpd_oks_rescore(const void* kpts, int kpt_f64, const double* box_score, int n, int J, double in_vis_thre, double* out,
                    fpd_stream_t stream) {
  return oks_rescore(kpts, kpt_f64, box_score, n, J, in_vis_thre, out, S(stream));
}
int fpd_gaussian_targets(const float* joints, const float* joints_vis, const float* joints_weight, const float* gauss_table,
                         float* target, float* target_weight, int N, int J, int H, int W, int image_w, int image_h,
                         int sigma, fpd_stream_t stream) {
  return gaussian_targets(joints, joints_vis, joints_weight, gauss_table, target, target_weight, N, J, H, W, image_w,
                          image_h, sigma, S(stream));
}

int fpd_crop_affine_normalize(const uint8_t* src, size_t src_bytes, const int64_t* desc, const double* inv,
                              const int64_t* desc_host, const double* inv_host, const float* mean_std_host, float* out,
                              int N, int out_h, int out_w, fpd_stream_t stream) {
  return crop_affine_normalize(src, src_bytes, desc, inv, desc_host, inv_host, mean_std_host, out, N, out_h, out_w,
                               S(stream));
}

int fpd_adam_flat(float* param, const float* grad, float* m, float* v, int64_t n, float lr, float b1, float b2,
                  float eps, float wd, int step, float grad_scale, fpd_stream_t stream) {
  return adam_flat(param, grad, m, v, n, lr, b1, b2, eps, wd, step, grad_scale, S(stream));
}

}  // extern "C"
