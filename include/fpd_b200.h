/* fpd_b200.h -- C ABI of libfpd_b200.so: the H100 (sm_90a) kernels behind the reference's hot path
 * (ilovepose/fast-human-pose-estimation.pytorch: stacked-hourglass / HRNet heat-map regression with the
 * Fast-Pose-Distillation loss, flip-test decode, box NMS).
 *
 * Conventions (all entry points):
 *  - plain pointers and sizes, no torch types; every tensor is caller-owned DEVICE memory unless the
 *    parameter name ends in `_host`; the library never allocates or frees device memory at call time
 *    (scratch comes in through `workspace`, sized by the matching *_workspace_bytes query). The one
 *    exception is fpd_nms_host, which keeps the reference `_nms` signature (no workspace argument) and
 *    therefore owns a grow-only scratch buffer.
 *  - work is enqueued on `stream` only (pass torch.cuda.current_stream().cuda_stream); no implicit
 *    device synchronisation, no default-stream use, safe under CUDA-graph capture.
 *  - return 0 on success, a negative FPD_ERR_* code otherwise; fpd_last_error() gives the message of the
 *    last failure on the calling thread. Nothing prints-and-continues (contrast the reference's
 *    CUDA_CHECK, lib/nms/nms_kernel.cu:11-18).
 *  - activations are NHWC fp32 ("[B,H,W,C]", C contiguous); conv weights are the reference's OIHW fp32
 *    unless stated; heat-maps handed to/from callers are NCHW like the reference's.
 *
 * Each group cites the reference interface it replaces (paths relative to the reference repo).
 */
#ifndef FPD_B200_H_
#define FPD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* fpd_stream_t;

#define FPD_OK 0
#define FPD_ERR_INVALID (-1)
#define FPD_ERR_CUDA (-2)
#define FPD_ERR_UNSUPPORTED (-3)

const char* fpd_last_error(void);
int fpd_version(void);
int fpd_sm_count(void);
/* number of kernels this library has launched in this process (monotonic) */
long long fpd_launch_count(void);

/* ---------------------------------------------------------------------------------------------------
 * Convolution. Replaces nn.Conv2d -> cuDNN/oneDNN as used by lib/models/hourglass.py:20-27 (Bottleneck
 * conv1/conv2/conv3), :116 (7x7 stem), :134-137,149,163 (fc / score / fc_ / score_ / downsample) and
 * lib/models/pose_hrnet.py:23-25 (conv3x3), :33-37,66-74.
 * ------------------------------------------------------------------------------------------------- */

/* Tensor-core implicit GEMM with the operand preparation fused in, forward or data-gradient (dgrad = same call on dY with
 * weights prepared by fpd_weight_prep(for_dgrad=1)): x is the RAW fp32 NHWC activation and the kernel applies
 * a = relu?((x - pre_mean) * pre_scale + pre_shift) (pre_scale/pre_shift NULL = identity, pre_mean NULL = 0) and the tf32
 * hi/lo split on chip -- i.e. conv(relu(bn(x))) of lib/models/hourglass.py:34-44 in one kernel.
 *   y[B,H,W,Cout] = out_scale * conv(a, w) (+ bias[Cout]) (+ residual[B,H,W,Cout]); if relu_mask is given (same shape as
 *   y) elements with relu_mask <= 0 are written as 0 (ReLU backward fused).
 *   w_hi/w_lo : [ksize*ksize][Cout][Cin] fp32 containers holding tf32 values from fpd_weight_prep (w_lo NULL => single-pass
 *               TF32; both non-NULL => 3xTF32, fp32-grade accuracy)
 * Runs on the warpgroup-MMA implicit-GEMM kernel of csrc/conv_wgmma.cu (3xTF32 operands), Cin up to 512. */
int fpd_conv2d_tc_ts_supported(int Cin, int Cout, int ksize); /* Cout up to 1024, processed in <=128-column slices */
int fpd_conv2d_tc_ts(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                     int pre_relu, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                     const float* relu_mask, float* y, float out_scale, int B, int H, int W, int Cin, int Cout,
                     int ksize, fpd_stream_t stream);

/* Fused convolution (csrc/conv_wgmma.cu), same contract as fpd_conv2d_tc_ts, Cin up to 2048 and Cout up to 2048.
 * f16 = 1 selects 3xFP16 operands (x = hi + lo in fp16, fp16 wgmma, fp32 accumulate): w_hi / w_lo
 * are then the __half arrays of fpd_weight_prep_f16; f16 = 0: fp32 containers of fpd_weight_prep (3xTF32).
 * w_lo NULL => single pass. in_scale (nullable, device float[2] {S, 1/S}, e.g. from fpd_channel_sum_fused): the operand
 * is x * S and the result is multiplied by 1/S -- exact powers of two that bring small-magnitude gradients into the fp16
 * range for the data-gradient convolution. Replaces nn.Conv2d after BatchNorm2d + ReLU (and its data gradient),
 * lib/models/hourglass.py:34-44. */
int fpd_conv2d_tc_h_supported(int Cin, int Cout, int ksize, int H, int W, int f16);
int fpd_conv2d_tc_h(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                    int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                    const float* residual, const float* relu_mask, float* y, float out_scale, const float* in_scale,
                    int B, int H, int W, int Cin, int Cout, int ksize, fpd_stream_t stream);
/* Forward ([tap][O][I]) and data-gradient ([taps-1-tap][I][O]) __half hi/lo forms of w * 2^8 from one read of the
 * weights: one launch per convolution and training step instead of two. */
int fpd_weight_prep_f16_both(const float* w_oihw, void* f_hi, void* f_lo, void* d_hi, void* d_lo, int O, int I, int k,
                             fpd_stream_t stream);
/* OIHW fp32 -> __half hi/lo of w * 2^8 in the layouts of fpd_weight_prep (w_lo may be NULL); the 2^-8 is applied by
 * fpd_conv2d_tc_h. */
int fpd_weight_prep_f16(const float* w_oihw, void* w_hi, void* w_lo, int O, int I, int k, int for_dgrad,
                        fpd_stream_t stream);

/* Forward convolution that also produces the BatchNorm batch statistics of its OUTPUT (train mode): the per-channel sums
 * come out of the epilogue (per-CTA partial blocks, merged by fpd_bn_finalize_sums), so the separate statistics pass
 * over the tensor that nn.BatchNorm2d (lib/models/hourglass.py:18-26) implies disappears. Arguments as fpd_conv2d_tc_h
 * (no relu_mask / in_scale: forward only); stat_part: device double[fpd_conv2d_tc_h_stats_blocks(...)][Cout][2];
 * stat_pivot: device float[Cout] or NULL, any per-channel value near the expected mean (improves conditioning only). */
int fpd_conv2d_tc_h_stats_blocks(int B, int H, int W, int Cin, int Cout, int ksize, int f16);   /* 0 = shape not supported */
int fpd_conv2d_tc_h_stats(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                          int pre_relu, const void* w_hi, const void* w_lo, int f16, const float* bias,
                          const float* residual, float* y, float out_scale, int B, int H, int W, int Cin, int Cout,
                          int ksize, double* stat_part, const float* stat_pivot, fpd_stream_t stream);
/* mean = pivot + S1/P, var = S2/P - (S1/P)^2 from those partial sums, then the BatchNorm finalize (scale = gamma * invstd,
 * shift = beta, running statistics update with `momentum`); outputs as fpd_bn_stats_fused. */
int fpd_bn_finalize_sums(const double* part, int nblocks, const float* pivot, int64_t P, int C, const float* gamma,
                         const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                         float* mean, float* var_biased, float* scale, float* shift, float* invstd, fpd_stream_t stream);
/* Leaner forms of fpd_channel_sum / fpd_bn_bwd_reduce / (fpd_bn_stats + fpd_bn_finalize): the BatchNorm statistics'
 * second stage and the module's finalize (affine + running statistics) run as one kernel (division-free fp64 merge), and
 * the channel sum can also return the operand scale of the 3xFP16 gradient convolutions: amax_scale (nullable float[2])
 * receives {S, 1/S} with S the power of two that puts max|dy| into [2^14, 2^15). `counter` is reserved (a single-launch
 * "last block finishes" variant measured slower and is disabled); pass a zeroed unsigned int or NULL.
 * Workspace sizes: fpd_channel_reduce_workspace_bytes / fpd_bn_stats_workspace_bytes.
 * Replace the per-channel sums of Conv2d bias backward, BatchNorm2d backward and BatchNorm2d train-mode forward
 * (lib/models/hourglass.py:18-26 modules under loss.backward(), lib/core/function.py:146). */
int fpd_channel_sum_fused(const float* dy, int64_t P, int C, float scale, float* out, float* amax_scale,
                          void* workspace, size_t workspace_bytes, unsigned int* counter, fpd_stream_t stream);
int fpd_bn_bwd_reduce_fused(const float* da, const float* x, const float* mean, const float* invstd,
                            const float* scale, const float* shift, int relu, int64_t P, int C, float* sums,
                            void* workspace, size_t workspace_bytes, unsigned int* counter, fpd_stream_t stream);
int fpd_bn_stats_fused(const float* x, int64_t P, int C, const float* gamma, const float* beta, float eps,
                       float momentum, float* running_mean, float* running_var, float* mean, float* var_biased,
                       float* scale, float* shift, float* invstd, void* workspace, size_t workspace_bytes,
                       unsigned int* counter, fpd_stream_t stream);

/* Tensor-core weight gradient: dw_oihw[Cout,Cin,k,k] = scale * sum_pixels dy (x) a(tap-shifted). */
int fpd_conv2d_wgrad_tc_supported(int Cin, int Cout, int ksize);
size_t fpd_conv2d_wgrad_tc_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize);

/* Weight gradient with the operand preparation fused in: x and dy are RAW fp32 NHWC tensors; the kernel applies
 * a = relu?((x - pre_mean) * pre_scale + pre_shift) (NULLs = identity), zeroes the 3x3 padding positions and does the
 * tf32 split on chip. passes = 3 (3xTF32) or 1. Workspace: fpd_conv2d_wgrad_tc_workspace_bytes. */
int fpd_conv2d_wgrad_tc_fused(const float* x, const float* pre_mean, const float* pre_scale, const float* pre_shift,
                              int pre_relu, const float* dy, int passes, float* dw_oihw, float scale, int B, int H,
                              int W, int Cin, int Cout, int ksize, void* workspace, size_t workspace_bytes,
                              fpd_stream_t stream);

/* 1 if fpd_conv2d_wgrad_tc_fused takes this 3x3 shape in one launch (the same rule as fpd_conv2d_wgrad_tc_supported). */
int fpd_conv2d_wgrad_tc3_supported(int H, int W, int Cin, int Cout, int ksize);

/* Generic fp32 CUDA-core convolution (any k/stride/pad): x NHWC [B,H,W,Cin], w OIHW. */
int fpd_conv2d_simt_fwd(const float* x, const float* w_oihw, const float* bias, const float* residual, float* y,
                        int B, int H, int W, int Cin, int Cout, int k, int stride, int pad, fpd_stream_t stream);
int fpd_conv2d_simt_dgrad(const float* dy, const float* w_oihw, float* dx, int B, int H, int W, int Cin, int Cout,
                          int k, int stride, int pad, fpd_stream_t stream);
size_t fpd_conv2d_simt_wgrad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k, int stride, int pad);
int fpd_conv2d_simt_wgrad(const float* x, const float* dy, float* dw_oihw, float scale, int B, int H, int W,
                          int Cin, int Cout, int k, int stride, int pad, void* workspace, size_t workspace_bytes,
                          fpd_stream_t stream);

/* OIHW fp32 -> tensor-core operand layout, split into tf32 hi/lo (w_lo may be NULL).
 * for_dgrad=0: [tap][O][I]; for_dgrad=1: [taps-1-tap][I][O] (180-degree flipped, transposed). */
int fpd_weight_prep(const float* w_oihw, float* w_hi, float* w_lo, int O, int I, int k, int for_dgrad,
                    fpd_stream_t stream);

/* ---------------------------------------------------------------------------------------------------
 * BatchNorm / ReLU / pooling glue. Replaces nn.BatchNorm2d (train + eval), nn.ReLU, F.max_pool2d,
 * nn.Upsample(scale_factor=2) + add: lib/models/hourglass.py:18-28,34-50,60,82-91,117-124.
 * ------------------------------------------------------------------------------------------------- */
size_t fpd_bn_stats_workspace_bytes(int64_t P, int C);
/* per-channel batch mean and biased variance of x[P,C] */
int fpd_bn_stats(const float* x, int64_t P, int C, float* mean, float* var_biased, void* workspace,
                 size_t workspace_bytes, fpd_stream_t stream);
/* Centred affine form used by every consumer: y = (x - mean) * scale + shift with
 * scale = gamma/sqrt(var+eps), shift = beta (no cancellation when |mean| >> std); invstd optional;
 * running stats (optional, both or neither) updated with `momentum` and the unbiased variance like
 * nn.BatchNorm2d. */
int fpd_bn_finalize(const float* mean, const float* var_biased, const float* gamma, const float* beta, float eps,
                    int64_t count, float* scale, float* shift, float* invstd, float* running_mean,
                    float* running_var, float momentum, int C, fpd_stream_t stream);
/* a = relu?((x-mean)*scale+shift) (scale/shift NULL = identity, mean NULL = 0)
 * -> a_hi = tf32(a), a_lo = tf32(a - a_hi) (optional) */
int fpd_affine_act_split(const float* x, const float* mean, const float* scale, const float* shift, int relu,
                         float* a_hi, float* a_lo, int64_t P, int C, fpd_stream_t stream);
/* y = relu?((x-mean)*scale+shift) in full fp32 (materialised activations: stem output, fc output) */
int fpd_affine_act(const float* x, const float* mean, const float* scale, const float* shift, int relu, float* y,
                   int64_t P, int C, fpd_stream_t stream);
/* HRNet glue (lib/models/pose_hrnet.py:41-57,78-98 block tails; :256-263 multi-resolution fuse):
 * y = relu?((x-mean)*scale+shift + residual);  out = relu?(sum_j nearest_up_{2^shift_j}(term_j)) with
 * terms_host/shifts_host HOST arrays of n<=4 device pointers / log2 factors, summed in order;
 * dlow = (2^shift)^2 block sums of dout[B,H,W,C]. */
int fpd_affine_add_act(const float* x, const float* mean, const float* scale, const float* shift,
                       const float* residual, int relu, float* y, int64_t P, int C, fpd_stream_t stream);
int fpd_fuse_sum(const float* const* terms_host, const int* shifts_host, int n, int relu, float* out, int B, int H,
                 int W, int C, fpd_stream_t stream);
int fpd_upsample_bwd(const float* dout, float* dlow, int shift, int B, int H, int W, int C, fpd_stream_t stream);
/* Stem convs with very few input channels (hourglass.py:116 7x7 s2 Cin=3; pose_hrnet.py:281 3x3 s2 Cin=3):
 * cols[B,Ho,Wo,Kpad] with channel index (kh*k+kw)*Cin+ci (zero outside the image / beyond k*k*Cin), which turns the
 * stem into a 1x1 convolution for the tensor-core kernels. */
int fpd_im2col(const float* x, float* cols, int B, int H, int W, int Cin, int k, int stride, int pad, int Kpad,
               fpd_stream_t stream);
size_t fpd_channel_reduce_workspace_bytes(int64_t P, int C);
int fpd_channel_sum(const float* dy, int64_t P, int C, float scale, float* out, void* workspace,
                    size_t workspace_bytes, fpd_stream_t stream);
/* BN(+ReLU) backward: phase 1 reduces sums[0:C]=sum dz, sums[C:2C]=sum dz*xhat; phase 2 writes
 * dx (= or +=) gamma*invstd*(dz - sum_dz/P - xhat*sum_dzxhat/P). dbeta = sums[0:C], dgamma = sums[C:2C]. */
int fpd_bn_bwd_reduce(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                      const float* shift, int relu, int64_t P, int C, float* sums, void* workspace,
                      size_t workspace_bytes, fpd_stream_t stream);
/* fpd_bn_bwd_apply (fresh dx, no accumulation) that also reduces its output in the same pass: dx_sum[C] = per-channel sum
 * of dx -- the bias gradient of the convolution whose output this BatchNorm consumed (hourglass.py:20-27) -- and
 * amax_scale[2] = {S, 1/S}, the power-of-two operand scale of that convolution's 3xFP16 data gradient (as
 * fpd_channel_sum_fused; nullable). workspace: fpd_channel_reduce_workspace_bytes(P, C). */
int fpd_bn_bwd_apply_sum(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                         const float* shift, const float* gamma, int relu, const float* sums, float* dx, float* dx_sum,
                         float* amax_scale, int64_t P, int C, void* workspace, size_t workspace_bytes, fpd_stream_t stream);
int fpd_bn_bwd_apply(const float* da, const float* x, const float* mean, const float* invstd, const float* scale,
                     const float* shift, const float* gamma, int relu, const float* sums, int accumulate, float* dx,
                     int64_t P, int C, fpd_stream_t stream);
int fpd_affine_act_bwd(const float* da, const float* x, const float* mean, const float* scale, const float* shift,
                       int relu, int accumulate, float* dx, int64_t P, int C, fpd_stream_t stream);
int fpd_maxpool2x2_fwd(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream);
int fpd_maxpool2x2_bwd(const float* x, const float* dy, float* dx, int accumulate, int B, int H, int W, int C,
                       fpd_stream_t stream);
int fpd_upsample2x_add(const float* up1, const float* low, float* out, int B, int H, int W, int C,
                       fpd_stream_t stream); /* H,W = output size */
int fpd_upsample2x_bwd(const float* dout, float* dlow, int B, int H, int W, int C, fpd_stream_t stream);
/* pose_resnet (lib/models/pose_resnet.py). Stem pool nn.MaxPool2d(3, 2, 1) (:107,233), NHWC: x [B,H,W,C] ->
 * y [B,(H-1)/2+1,(W-1)/2+1,C], padding = -inf, first maximum in window scan order wins (ATen); the backward is a
 * deterministic gather (accumulate != 0: dx += ...). C % 4 == 0. */
int fpd_maxpool3x3s2_fwd(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream);
int fpd_maxpool3x3s2_bwd(const float* x, const float* dy, float* dx, int accumulate, int B, int H, int W, int C,
                         fpd_stream_t stream);
/* The deconv head nn.ConvTranspose2d(Cin, Cout, k, stride=2, padding=pad) (:176-204; (k,pad) in (4,1) (3,1) (2,0)) runs as
 * a stride-1 3x3 convolution to 4*Cout channels on the tensor-core kernels + a depth-to-space shuffle:
 * fpd_deconv_weight_map(to_deconv=0) builds the OIHW [4*Cout,Cin,3,3] weights from the module's [Cin,Cout,k,k] ones,
 * (to_deconv=1) gathers the module's weight gradient back out of the convolution's; fpd_depth_space2(to_depth=0) maps
 * src [B,H,W,4C] -> dst [B,2H,2W,C], dst[b,2a+rh,2c+rw,co] = src[b,a,c,(2rh+rw)C+co]; (to_depth=1) is the inverse, src
 * [B,2H,2W,C] -> dst [B,H,W,4C] (B, H, W, C always name the DEPTH side's [B,H,W,4C]). */
int fpd_depth_space2(const float* src, float* dst, int B, int H, int W, int C, int to_depth, fpd_stream_t stream);
int fpd_deconv_weight_map(const float* src, float* dst, int Cin, int Cout, int k, int pad, int to_deconv,
                          fpd_stream_t stream);

/* Stride-2 3x3 convolutions (HRNet stem / transition / fuse down paths, lib/models/pose_hrnet.py:213-239,281-284,355-370)
 * on the stride-1 tensor-core kernels: y = subsample2(conv_s1(x)) picks the even positions (x: [B,H,W,C] -> y:
 * [B,H/2,W/2,C]); upsample_zero2 is its adjoint (dY scattered to the even positions of a zero [B,2Ho,2Wo,C] tensor), which
 * then feeds the stride-1 data- and weight-gradient kernels. */
int fpd_subsample2(const float* x, float* y, int B, int H, int W, int C, fpd_stream_t stream);
int fpd_upsample_zero2(const float* dy, float* dx, int B, int Ho, int Wo, int C, fpd_stream_t stream);
int fpd_nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, fpd_stream_t stream);
/* Same, with the image mirrored along W on the way (the flipped input of the flip test, lib/core/function.py:218-221:
 * np.flip(input, 3)), so the second forward needs no separate flip pass. */
int fpd_nchw_to_nhwc_flipw(const float* x_nchw, float* y_nhwc, int B, int C, int H, int W, fpd_stream_t stream);
int fpd_nhwc_to_nchw(const float* x, float* y, int B, int C, int H, int W, fpd_stream_t stream);
int fpd_add(const float* a, const float* b, float* out, int64_t n, fpd_stream_t stream);

/* ---------------------------------------------------------------------------------------------------
 * Loss. Replaces lib/core/loss.py:21-39 (JointsMSELoss) and the FPD combination in
 * lib/core/function.py:127-134: loss = (1-alpha)*sum_s L(out_s,target) + alpha*sum_s L(out_s,teacher).
 * ------------------------------------------------------------------------------------------------- */
size_t fpd_loss_workspace_bytes(int B, int J, int h, int w);
/* outs_host / grads_host: HOST arrays of S device pointers (NHWC [B,h,w,J]); grads_host or its entries
 * may be NULL. target: NCHW [B,J,h,w]; teacher: NHWC or NULL (plain sum-of-stacks MSE, function.py:44-55);
 * target_weight [B,J]; losses[3] (device) = {pose, kd, total}; grads = grad_scale * dtotal/dout_s. */
int fpd_loss_fused(const float* const* outs_host, int S, const float* target_nchw, const float* teacher_nhwc,
                   const float* target_weight, float alpha, float* const* grads_host, float grad_scale,
                   float* losses, int B, int J, int h, int w, void* workspace, size_t workspace_bytes,
                   fpd_stream_t stream);
/* single JointsMSELoss on NCHW tensors; loss3 (device, 3 floats, [0] is the loss); grad (optional) =
 * dloss/dout; target_weight NULL = use_target_weight False. */
int fpd_joints_mse(const float* out_nchw, const float* target_nchw, const float* target_weight, float* loss3,
                   float* grad, int B, int J, int hw, void* workspace, size_t workspace_bytes, fpd_stream_t stream);

/* ---------------------------------------------------------------------------------------------------
 * Decode. Replaces the numpy round-trips of lib/core/function.py:218-240 (flip test),
 * lib/utils/transforms.py:15-29 (flip_back) and lib/core/inference.py:18-46 (get_max_preds).
 * ------------------------------------------------------------------------------------------------- */
/* hm, hm_flip: NHWC [B,h,w,J] (hm_flip NULL = no flip test); flip_perm[J] device int32 (joint j of the
 * flipped map comes from channel flip_perm[j]); avg_nhwc optional output; idx[B*J] flat arg-max
 * (first maximum), maxval[B*J]. */
int fpd_flip_merge_argmax(const float* hm, const float* hm_flip, const int* flip_perm, int shift, float* avg_nhwc,
                          int* idx, float* maxval, int B, int J, int h, int w, fpd_stream_t stream);
int fpd_argmax_nchw(const float* hm_nchw, int* idx, float* maxval, int BJ, int hw, fpd_stream_t stream);

/* ---------------------------------------------------------------------------------------------------
 * NMS. Replaces lib/nms/nms_kernel.cu:33-77 (nms_kernel) and :90-143 (_nms), declared in
 * lib/nms/gpu_nms.hpp:1-2.
 * ------------------------------------------------------------------------------------------------- */
size_t fpd_nms_workspace_bytes(int n);
/* boxes: device [n,box_dim] sorted by score descending; keep/num_keep: device outputs */
int fpd_nms_device(const float* boxes_sorted, int n, int box_dim, float thresh, int* keep, int* num_keep,
                   void* workspace, size_t workspace_bytes, fpd_stream_t stream);
/* Drop-in for `void _nms(int* keep_out, int* num_out, const float* boxes_host, int boxes_num,
 * int boxes_dim, float nms_overlap_thresh, int device_id)` (host pointers, synchronous) -- but it
 * returns an error code instead of printing. */
int fpd_nms_host(int* keep_out_host, int* num_out_host, const float* boxes_host, int boxes_num, int boxes_dim,
                 float nms_overlap_thresh, int device_id);

/* OKS-NMS. Replaces the host numpy loops of lib/nms/nms.py:75-96 (oks_iou) and :99-124 (oks_nms), called from
 * lib/dataset/coco.py:359-369. kpts_sorted: device [n,J,3] (x, y, score), float32 (kpt_f64 = 0, what coco.py:283 holds)
 * or float64, persons sorted by score descending; areas_sorted: device double[n]; vars: device double[J] = (2 sigma_j)^2;
 * a person j is suppressed when oks(kept i, j) > thresh; use_vis != 0 masks joints by the candidate's score >
 * in_vis_thre (nms.py:90-92). keep / num_keep / workspace as fpd_nms_device (fpd_nms_workspace_bytes(n)). */
int fpd_oks_nms_device(const void* kpts_sorted, int kpt_f64, const double* areas_sorted, const double* vars, int n, int J,
                       double thresh, int use_vis, double in_vis_thre, int* keep, int* num_keep, void* workspace,
                       size_t workspace_bytes, fpd_stream_t stream);
/* Person rescoring before OKS-NMS, lib/dataset/coco.py:346-357: out[i] = box_score[i] * mean of the joint scores above
 * in_vis_thre (0 if none). kpts: device [n,J,3]; box_score, out: device double[n]. */
int fpd_oks_rescore(const void* kpts, int kpt_f64, const double* box_score, int n, int J, double in_vis_thre, double* out,
                    fpd_stream_t stream);

/* ---------------------------------------------------------------------------------------------------
 * Target generation. Replaces JointsDataset.generate_target, lib/dataset/JointsDataset.py:233-289, for a whole batch:
 * joints, joints_vis: device float[N,J,3]; joints_weight: device float[J] or NULL (USE_DIFFERENT_JOINTS_WEIGHT);
 * gauss_table: device float[(6 sigma + 1)^2], the reference's un-normalised Gaussian patch; outputs target
 * float[N,J,H,W] (fully written) and target_weight float[N,J]. image_w/h and W/H give feat_stride.
 * ------------------------------------------------------------------------------------------------- */
int fpd_gaussian_targets(const float* joints, const float* joints_vis, const float* joints_weight, const float* gauss_table,
                         float* target, float* target_weight, int N, int J, int H, int W, int image_w, int image_h,
                         int sigma, fpd_stream_t stream);

/* ---------------------------------------------------------------------------------------------------
 * Optimizer. Replaces torch.optim.Adam as configured by lib/utils/utils.py:69-73, stepped at
 * lib/core/function.py:147, over one flat parameter buffer.
 * ------------------------------------------------------------------------------------------------- */
int fpd_adam_flat(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                  float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                  fpd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* FPD_B200_H_ */
