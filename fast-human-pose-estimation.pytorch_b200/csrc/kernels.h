// kernels.h -- internal launcher declarations (C++), one per kernel family. The public C ABI that
// wraps these lives in api.cu / include/fpd_b200.h. Every launcher: launches only on `stream`, never
// allocates or frees device memory, never synchronises, returns FPD_OK or a negative error code.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fpd {

// ---- conv_wgmma.cu : warpgroup-MMA implicit-GEMM convolution (3xTF32, Cin <= 512) ----
bool conv_tc_ts_supported(int Cin, int Cout, int ksize);   // Cout up to 1024 in slices of <= 128 columns
int conv_tc_ts_slice(int Cout);
int conv_tc_ts_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                      int pre_relu, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                      const float* relu_mask, float* y, float out_scale, int B, int H, int W, int Cin, int Cout,
                      int ksize, int num_sms, cudaStream_t stream);

// ---- conv_wgmma.cu : the same kernel with Cin up to 2048, optional epilogue statistics and optional 3xFP16 operands (f16 = 1: w_hi / w_lo are __half [tap][Cout][Cin] from weight_prep_f16, pre-scaled
//      by 2^kF16WeightScaleLog2; f16 = 0: fp32 containers from weight_prep, 3xTF32) ----
constexpr int kF16WeightScaleLog2 = 8;
bool conv_tc_h_supported(int Cin, int Cout, int ksize, int H, int W, int f16);
int conv_tc_h_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                     int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                     const float* residual, const float* relu_mask, float* y, float out_scale, const float* in_scale,
                     int B, int H, int W, int Cin, int Cout, int ksize, int num_sms, cudaStream_t stream,
                     double* stat_part = nullptr, const float* stat_pivot = nullptr);
// BatchNorm statistics of the OUTPUT from the epilogue: number of per-CTA partial blocks the launch writes to
// stat_part[blocks][Cout][2] (0: this shape cannot carry the statistics, e.g. Cout > 256)
int conv_tc_h_stats_grid(int B, int H, int W, int Cin, int Cout, int ksize, int f16, int num_sms);

// ---- conv_wgmma.cu : warpgroup-MMA weight-gradient GEMM (K = pixels) reading RAW x and dY; BN-apply + ReLU + tf32 split
//      fused into the operand staging ----
bool wgrad_tc_supported(int Cin, int Cout, int ksize);
size_t wgrad_tc_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, int num_sms);
int wgrad_tc_fused_launch(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                          int pre_relu, const float* dy, int passes, float* dw_oihw, float scale, int B, int H, int W,
                          int Cin, int Cout, int ksize, void* workspace, size_t workspace_bytes, int num_sms,
                          cudaStream_t stream);

// the 3x3 shape rule of wgrad_tc_supported (fpd_conv2d_wgrad_tc3_supported)
bool wgrad_tc3_supported(int H, int W, int Cin, int Cout, int ksize);

// ---- conv_simt.cu : generic fp32 CUDA-core convolution (any k / stride / pad, NHWC activations,
//      OIHW weights). Used for the shapes the tensor-core kernels do not take (7x7 stem, 16-channel
//      score convs) and as the on-device cross-check in tests. ----
int conv_simt_fwd(const float* x, const float* w_oihw, const float* bias, const float* residual, float* y, int B,
                  int H, int W, int Cin, int Cout, int k, int stride, int pad, cudaStream_t stream);
int conv_simt_dgrad(const float* dy, const float* w_oihw, float* dx, int B, int H, int W, int Cin, int Cout, int k,
                    int stride, int pad, cudaStream_t stream);  // H,W = input size; dx[B,H,W,Cin]
size_t conv_simt_wgrad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k, int stride, int pad);
int conv_simt_wgrad(const float* x, const float* dy, float* dw_oihw, float scale, int B, int H, int W, int Cin,
                    int Cout, int k, int stride, int pad, void* workspace, size_t ws_bytes, cudaStream_t stream);

// ---- elementwise.cu ----
// Per-channel batch statistics of x[P,C] (numerically robust: per-chunk shifted sums, Chan merge in fp64).
size_t bn_stats_workspace_bytes(int64_t P, int C);
int bn_stats(const float* x, int64_t P, int C, float* mean, float* var_biased, void* workspace, size_t ws_bytes,
             cudaStream_t stream);
// centred affine y = (x-mean)*scale + shift: scale = gamma*rsqrt(var+eps), shift = beta ; optional running-stat update (momentum, unbiased var)
int bn_finalize(const float* mean, const float* var_biased, const float* gamma, const float* beta, float eps,
                int64_t count, float* scale, float* shift, float* invstd, float* running_mean, float* running_var,
                float momentum, int C, cudaStream_t stream);
// a = act((x-mean)*scale+shift) (mean/scale/shift may be null = identity; relu optional); hi = tf32(a), lo = tf32(a-hi)
int affine_act_split(const float* x, const float* mean, const float* scale, const float* shift, int relu,
                     float* a_hi, float* a_lo, int64_t P, int C, cudaStream_t stream);
// y = act(x*scale+shift), full fp32 (no operand rounding)
int affine_act(const float* x, const float* mean, const float* scale, const float* shift, int relu, float* y,
               int64_t P, int C, cudaStream_t stream);
// y = act((x-mean)*scale+shift + residual): tail of the post-activation residual blocks (pose_hrnet.py:48-55)
int affine_add_act(const float* x, const float* mean, const float* scale, const float* shift, const float* residual,
                   int relu, float* y, int64_t P, int C, cudaStream_t stream);
// out = relu?(sum_j nearest_up_{2^shift_j}(term_j)) (HRNet fuse, pose_hrnet.py:256-263); terms/shifts: host arrays
int fuse_sum(const float* const* terms, const int* shifts, int n, int relu, float* out, int B, int H, int W, int C,
             cudaStream_t stream);
// dlow = sum over (2^shift)^2 blocks of dout [B,H,W,C]
int upsample_bwd(const float* dout, float* dlow, int shift, int B, int H, int W, int C, cudaStream_t stream);
// cols[B,Ho,Wo,Kpad] = im2col(x[B,H,W,Cin]) with K index (kh*k+kw)*Cin+ci, zero padded to Kpad channels
int im2col(const float* x, float* cols, int B, int H, int W, int Cin, int k, int stride, int pad, int Kpad,
           cudaStream_t stream);
int maxpool2x2_fwd(const float* x, float* y, int B, int H, int W, int C, cudaStream_t stream);
int maxpool2x2_bwd(const float* x, const float* dy, float* dx, int accumulate, int B, int H, int W, int C,
                   cudaStream_t stream);
int upsample2x_add(const float* up1, const float* low, float* out, int B, int H, int W, int C,
                   cudaStream_t stream);  // H,W = output size
int upsample2x_bwd(const float* dout, float* dlow, int B, int H, int W, int C, cudaStream_t stream);
// pose_resnet stem pool: 3x3, stride 2, padding 1 ([B,H,W,C] -> [B,(H-1)/2+1,(W-1)/2+1,C]); first maximum wins
int maxpool3x3s2_fwd(const float* x, float* y, int B, int H, int W, int C, cudaStream_t stream);
int maxpool3x3s2_bwd(const float* x, const float* dy, float* dx, int accumulate, int B, int H, int W, int C,
                     cudaStream_t stream);
// depth [B,H,W,4C] <-> space [B,2H,2W,C] shuffle and the ConvTranspose2d -> 3x3-conv weight map (see elementwise.cu)
int depth_space2(const float* src, float* dst, int B, int H, int W, int C, int to_depth, cudaStream_t stream);
int deconv_weight_map(const float* src, float* dst, int Cin, int Cout, int k, int pad, int to_deconv, cudaStream_t stream);
int subsample2(const float* x, float* y, int B, int H, int W, int C, cudaStream_t stream);        // y[ho,wo] = x[2ho,2wo]
int upsample_zero2(const float* dy, float* dx, int B, int Ho, int Wo, int C, cudaStream_t stream);  // adjoint of subsample2
int nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, cudaStream_t stream);
int nchw_to_nhwc_flipw(const float* x, float* y, int B, int C, int H, int W, cudaStream_t stream);   // + W mirror
int nhwc_to_nchw(const float* x, float* y, int B, int C, int H, int W, cudaStream_t stream);
int add_tensors(const float* a, const float* b, float* out, int64_t n, cudaStream_t stream);  // out = a + b
size_t channel_reduce_workspace_bytes(int64_t P, int C);
// sum over pixels of dy[P,C] -> out[C] (out = scale*sum)
int channel_sum(const float* dy, int64_t P, int C, float scale, float* out, void* workspace, size_t ws_bytes,
                cudaStream_t stream);
// BN(+ReLU) backward, phase 1: dz = da * (relu ? (x*scale+shift > 0) : 1); sums[0:C] = sum dz,
// sums[C:2C] = sum dz * xhat  where xhat = (x-mean)*invstd.
int bn_bwd_reduce(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                  const float* shift, int relu, int64_t P, int C, float* sums, void* workspace, size_t ws_bytes,
                  cudaStream_t stream);
// phase 2: dx (=|+=) gamma*invstd*(dz - sum_dz/P - xhat*sum_dzx/P); also writes dgamma = sum_dzx, dbeta = sum_dz
// bn_bwd_apply + per-channel sum of dx (-> dx_sum[C]) + power-of-two operand scale of dx (-> amax_scale[2], nullable);
// workspace as channel reduce
int bn_bwd_apply_sum(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                     const float* shift, const float* gamma, int relu, const float* sums, float* dx, float* dx_sum,
                     float* amax_scale, int64_t P, int C, void* workspace, size_t ws_bytes, cudaStream_t stream);
int bn_bwd_apply(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                 const float* shift, const float* gamma, int relu, const float* sums, int accumulate, float* dx,
                 int64_t P, int C, cudaStream_t stream);
// eval-mode / no-stat variant: dx (=|+=) da * mask * scale
int affine_act_bwd(const float* da, const float* x, const float* mean, const float* scale, const float* shift,
                   int relu, int accumulate, float* dx, int64_t P, int C, cudaStream_t stream);
// OIHW fp32 -> [tap][O][I] (fwd) or [flipped tap][I][O] (dgrad), split into tf32 hi/lo
int weight_prep(const float* w_oihw, float* w_hi, float* w_lo, int O, int I, int k, int for_dgrad,
                cudaStream_t stream);
// same layouts as __half hi/lo of w * 2^kF16WeightScaleLog2 (3xFP16 operands of conv_wgmma.cu)
int weight_prep_f16(const float* w_oihw, void* w_hi, void* w_lo, int O, int I, int k, int for_dgrad,
                    cudaStream_t stream);
// forward [tap][O][I] and data-gradient [taps-1-tap][I][O] forms in one launch
int weight_prep_f16_both(const float* w_oihw, void* f_hi, void* f_lo, void* d_hi, void* d_lo, int O, int I, int k,
                         cudaStream_t stream);

// Leaner forms of the reductions above (see include/fpd_b200.h): BN statistics second stage + finalize in one kernel,
// channel sum with the optional 3xFP16 operand scale amax_scale = {S, 1/S}. `counter` is reserved (ignored).
int channel_sum_fused(const float* dy, int64_t P, int C, float scale, float* out, float* amax_scale, void* workspace,
                      size_t ws_bytes, unsigned int* counter, cudaStream_t stream);
int bn_bwd_reduce_fused(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                        const float* shift, int relu, int64_t P, int C, float* sums, void* workspace, size_t ws_bytes,
                        unsigned int* counter, cudaStream_t stream);
// batch statistics + BatchNorm finalize (affine for the consumers, running-stat update) in one launch
// finalize from per-CTA column sums {sum (y - pivot), sum (y - pivot)^2} (conv_tc_h epilogue statistics)
int bn_finalize_sums(const double* part, int nblocks, const float* pivot, int64_t P, int C, const float* gamma,
                     const float* beta, float eps, float momentum, float* rmean, float* rvar, float* mean, float* var,
                     float* scale, float* shift, float* invstd, cudaStream_t stream);
int bn_stats_fused(const float* x, int64_t P, int C, const float* gamma, const float* beta, float eps, float momentum,
                   float* rmean, float* rvar, float* mean, float* var, float* scale, float* shift, float* invstd,
                   void* workspace, size_t ws_bytes, unsigned int* counter, cudaStream_t stream);

// ---- loss.cu : fused FPD loss + gradient ----
// out_s: S pointers to NHWC [B,h,w,J] student heat-maps; target NCHW [B,J,h,w]; teacher NHWC [B,h,w,J] or null;
// tw [B,J]; losses[3] = {pose, kd, total}; grads: S pointers (NHWC) or null.
size_t fpd_loss_workspace_bytes(int B, int J, int h, int w);
int fpd_loss(const float* const* outs_dev_ptrs_host, int S, const float* target_nchw, const float* teacher_nhwc,
             const float* tw, float alpha, float* const* grads_host, float grad_scale, float* losses, int B, int J,
             int h, int w, void* workspace, size_t ws_bytes, cudaStream_t stream);
// reference-compatible single JointsMSELoss on NCHW tensors (lib/core/loss.py:21-39)
int joints_mse(const float* out_nchw, const float* target_nchw, const float* tw, float* loss, float* grad_out,
               float grad_scale_unused, int B, int J, int hw, void* workspace, size_t ws_bytes, cudaStream_t stream);

// ---- decode.cu ----
// flip-test merge + arg-max: hm/hm_flip NHWC [B,h,w,J]; out avg NCHW (optional), idx[B,J] int32, maxval[B,J]
int flip_merge_argmax(const float* hm, const float* hm_flip, const int* flip_perm, int shift, float* avg_nchw,
                      int* idx, float* maxval, int B, int J, int h, int w, cudaStream_t stream);
int argmax_nchw(const float* hm, int* idx, float* maxval, int BJ, int hw, cudaStream_t stream);

// ---- nms.cu ----
size_t nms_workspace_bytes(int n);
int nms_device(const float* boxes_sorted_dev, int n, int box_dim, float thresh, int* keep_dev, int* num_keep_dev,
               void* workspace, size_t ws_bytes, cudaStream_t stream);

// OKS-NMS (lib/nms/nms.py:75-124): kpts [n,J,3] (x,y,score; float or double) sorted by person score descending,
// areas [n], vars_[J] = (2 sigma_j)^2 as float64; keep/num_keep as nms_device. use_vis: mask joints by the candidate's
// score > in_vis_thre.
int oks_nms_device(const void* kpts_sorted, int kpt_f64, const double* areas_sorted, const double* vars_, int n, int J,
                   double thresh, int use_vis, double in_vis_thre, int* keep_dev, int* num_keep_dev, void* workspace,
                   size_t ws_bytes, cudaStream_t stream);
// person rescoring (lib/dataset/coco.py:346-357): out[i] = box_score[i] * mean(score_j | score_j > in_vis_thre)
int oks_rescore(const void* kpts, int kpt_f64, const double* box_score, int n, int J, double in_vis_thre, double* out,
                cudaStream_t stream);
// Gaussian heat-map targets (lib/dataset/JointsDataset.py:233-289) for N samples
int gaussian_targets(const float* joints, const float* joints_vis, const float* joints_weight, const float* gauss_table,
                     float* target, float* target_weight, int N, int J, int H, int W, int image_w, int image_h, int sigma,
                     cudaStream_t stream);

// ---- adam.cu ----
int adam_flat(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float beta1,
              float beta2, float eps, float weight_decay, int step, float grad_scale, cudaStream_t stream);

int device_sm_count();

}  // namespace fpd
