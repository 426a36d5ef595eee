"""Tensor-level wrappers over the C ABI: torch is used only for device memory and streams.

Every function takes contiguous fp32 CUDA tensors, enqueues on torch's current stream and returns
(or fills) tensors. Activations are NHWC ([B,H,W,C]) unless a name says otherwise.
"""
import ctypes
import os

import torch

from . import _native as N


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk(t, name):
    if t is None:
        return
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise ValueError("%s must be a contiguous fp32 CUDA tensor (got %s %s %s)" % (name, t.device, t.dtype,
                                                                                 t.is_contiguous()))


class Workspace:
    """Grow-only scratch buffers handed to the kernels that need one (no allocation at call time once warm).
    One buffer per CUDA stream: kernels enqueued on different streams (teacher / weight-gradient side streams) may run
    concurrently and must not share reduction scratch."""

    def __init__(self):
        self.bufs = {}

    def get(self, nbytes, device):
        nbytes = int(nbytes)
        key = (device, torch.cuda.current_stream(device).cuda_stream)
        buf = self.bufs.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
            self.bufs[key] = buf
        return buf


_ws = Workspace()
_counters = {}


def _counter(device):
    """Zero-initialised ticket counter for the single-launch reductions (one per device and stream; the kernels leave it
    zero)."""
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    c = _counters.get(key)
    if c is None:
        c = torch.zeros(16, dtype=torch.int32, device=device)
        _counters[key] = c
    return c


FUSED_REDUCE = os.environ.get("FPD_FUSED_REDUCE", "1") != "0"   # single-launch reductions (A/B switch)


def conv2d_tc_supported(cin, cout, k, fused=True):
    """Does a tensor-core convolution kernel take these channel counts (the TS kernel takes Cout > 256 in slices)?"""
    return bool(N.lib().fpd_conv2d_tc_ts_supported(cin, cout, k))


def weight_prep(w_oihw, for_dgrad=False, split=True):
    _chk(w_oihw, "w")
    O, I, k, _ = w_oihw.shape
    shape = (k * k, I, O) if for_dgrad else (k * k, O, I)
    hi = torch.empty(shape, dtype=torch.float32, device=w_oihw.device)
    lo = torch.empty_like(hi) if split else None
    N.check(N.lib().fpd_weight_prep(_p(w_oihw), _p(hi), _p(lo), O, I, k, int(for_dgrad), _stream()), "weight_prep")
    return hi, lo


def affine_act_split(x, scale=None, shift=None, relu=False, split=True, out_hi=None, out_lo=None, mean=None):
    _chk(x, "x")
    C = x.shape[-1]
    P = x.numel() // C
    hi = out_hi if out_hi is not None else torch.empty_like(x)
    lo = (out_lo if out_lo is not None else torch.empty_like(x)) if split else None
    N.check(N.lib().fpd_affine_act_split(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(hi), _p(lo), P, C,
                                         _stream()),
            "affine_act_split")
    return hi, lo


def affine_act(x, scale=None, shift=None, relu=False, out=None, mean=None):
    _chk(x, "x")
    C = x.shape[-1]
    P = x.numel() // C
    y = out if out is not None else torch.empty_like(x)
    N.check(N.lib().fpd_affine_act(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(y), P, C, _stream()),
            "affine_act")
    return y


def affine_add_act(x, residual, scale=None, shift=None, relu=True, mean=None, out=None):
    C = x.shape[-1]
    P = x.numel() // C
    y = out if out is not None else torch.empty_like(x)
    N.check(N.lib().fpd_affine_add_act(_p(x), _p(mean), _p(scale), _p(shift), _p(residual), int(relu), _p(y), P, C,
                                       _stream()), "affine_add_act")
    return y


def fuse_sum(terms, shifts, relu=True, out=None):
    """out = relu?(sum_j nearest-upsample_{2^shift_j}(terms[j])); terms[j] is [B, H>>s, W>>s, C]."""
    n = len(terms)
    B, C = terms[0].shape[0], terms[0].shape[-1]
    H, W = terms[0].shape[1] << shifts[0], terms[0].shape[2] << shifts[0]
    y = out if out is not None else torch.empty((B, H, W, C), dtype=torch.float32, device=terms[0].device)
    arr = (ctypes.c_void_p * n)(*[t.data_ptr() for t in terms])
    sh = (ctypes.c_int * n)(*[int(s) for s in shifts])
    N.check(N.lib().fpd_fuse_sum(arr, sh, n, int(relu), _p(y), B, H, W, C, _stream()), "fuse_sum")
    return y


def upsample_bwd(dout, shift, out=None):
    B, H, W, C = dout.shape
    d = out if out is not None else torch.empty((B, H >> shift, W >> shift, C), dtype=torch.float32,
                                                device=dout.device)
    N.check(N.lib().fpd_upsample_bwd(_p(dout), _p(d), int(shift), B, H, W, C, _stream()), "upsample_bwd")
    return d


def im2col(x, k, stride, pad, kpad, out=None):
    B, H, W, Cin = x.shape
    Ho = (H + 2 * pad - k) // stride + 1
    Wo = (W + 2 * pad - k) // stride + 1
    cols = out if out is not None else torch.empty((B, Ho, Wo, kpad), dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_im2col(_p(x), _p(cols), B, H, W, Cin, k, stride, pad, kpad, _stream()), "im2col")
    return cols


def conv2d_tc_fused(x, w_hi, w_lo, ksize, mean=None, scale=None, shift=None, relu=False, bias=None, residual=None,
                    relu_mask=None, out=None, out_scale=1.0):
    """y = conv(relu?((x-mean)*scale+shift)) on the tensor cores (csrc/conv_wgmma.cu,
    3xTF32) -- the fallback for the shapes conv2d_tc_h declines."""
    B, H, W, Cin = x.shape
    Cout = w_hi.shape[1]
    y = out if out is not None else torch.empty((B, H, W, Cout), dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_conv2d_tc_ts(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(w_hi), _p(w_lo), _p(bias),
                                     _p(residual), _p(relu_mask), _p(y), float(out_scale), B, H, W, Cin, Cout, ksize,
                                     _stream()), "conv2d_tc_ts")
    return y


CONV_H = os.environ.get("FPD_CONV_H", "1") != "0"          # conv2d_tc_h (3xFP16 capable, Cin up to 2048) where it supports the shape
CONV_F16 = os.environ.get("FPD_CONV_F16", "1") != "0"      # 3xFP16 operands for the forward convolutions
CONV_F16_DGRAD = os.environ.get("FPD_CONV_F16_DGRAD", "1") != "0"   # ... and for the data-gradient convolutions (dY * 2^k)


def conv2d_tc_h_supported(cin, cout, k, H, W, f16):
    return CONV_H and bool(N.lib().fpd_conv2d_tc_h_supported(cin, cout, k, H, W, int(f16)))


def weight_prep_f16(w_oihw, for_dgrad=False, split=True):
    """__half hi/lo of w * 2^8 (3xFP16 operands of conv2d_tc_h(f16=True)); layouts as weight_prep."""
    _chk(w_oihw, "w")
    O, I, k, _ = w_oihw.shape
    shape = (k * k, I, O) if for_dgrad else (k * k, O, I)
    hi = torch.empty(shape, dtype=torch.float16, device=w_oihw.device)
    lo = torch.empty_like(hi) if split else None
    N.check(N.lib().fpd_weight_prep_f16(_p(w_oihw), _p(hi), _p(lo), O, I, k, int(for_dgrad), _stream()),
            "weight_prep_f16")
    return hi, lo


def weight_prep_f16_both(w_oihw):
    """-> ((fwd_hi, fwd_lo), (dgrad_hi, dgrad_lo)) in one launch."""
    _chk(w_oihw, "w")
    O, I, k, _ = w_oihw.shape
    f_hi = torch.empty((k * k, O, I), dtype=torch.float16, device=w_oihw.device)
    f_lo = torch.empty_like(f_hi)
    d_hi = torch.empty((k * k, I, O), dtype=torch.float16, device=w_oihw.device)
    d_lo = torch.empty_like(d_hi)
    N.check(N.lib().fpd_weight_prep_f16_both(_p(w_oihw), _p(f_hi), _p(f_lo), _p(d_hi), _p(d_lo), O, I, k, _stream()),
            "weight_prep_f16_both")
    return (f_hi, f_lo), (d_hi, d_lo)


# BatchNorm statistics of conv outputs from the conv epilogue: "0" off, "1" every tensor-core conv, "3x3" only the 3x3
# convolutions. On the bench configuration (hg_fpd, one H100 SXM at 700 W, two runs each) the three settings are within
# noise of each other: 3x3 83.9 / 84.0 ms/step, off 84.0 / 83.9, every conv 83.9 / 83.9. "3x3" is kept: it saves the
# separate statistics pass over the largest tensors without adding epilogue work to the 1x1 convolutions.
CONV_STATS = os.environ.get("FPD_CONV_STATS", "3x3").lower()


def conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, k, f16):
    """Number of per-CTA partial blocks conv2d_tc_h(..., stats_part=) writes; 0 if the shape cannot carry statistics."""
    if CONV_STATS == "0" or (CONV_STATS == "3x3" and k != 3):
        return 0
    return int(N.lib().fpd_conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, k, int(f16)))


def bn_finalize_sums(part, nblocks, pivot, P, gamma, beta, eps, running_mean=None, running_var=None, momentum=0.1):
    """BatchNorm finalize from the per-CTA column sums of a producing conv's epilogue (conv2d_tc_h(stats_part=...)).
    Returns (mean, var_biased, scale, shift, invstd); updates the running statistics like nn.BatchNorm2d."""
    C = part.shape[1]
    dev = part.device
    mean = torch.empty(C, dtype=torch.float32, device=dev)
    var, scale, shift, invstd = (torch.empty_like(mean) for _ in range(4))
    N.check(N.lib().fpd_bn_finalize_sums(_p(part), int(nblocks), _p(pivot), int(P), C, _p(gamma), _p(beta), float(eps),
                                         float(momentum), _p(running_mean), _p(running_var), _p(mean), _p(var), _p(scale),
                                         _p(shift), _p(invstd), _stream()), "bn_finalize_sums")
    return mean, var, scale, shift, invstd


def conv2d_tc_h(x, w_hi, w_lo, ksize, mean=None, scale=None, shift=None, relu=False, bias=None, residual=None,
                relu_mask=None, out=None, out_scale=1.0, in_scale=None, stats_part=None, stats_pivot=None):
    """y = conv(relu?((x-mean)*scale+shift)) on the fused tensor-core kernel (csrc/conv_wgmma.cu). The operand precision
    follows the weight dtype: float16 hi/lo -> 3xFP16 (kind::f16), float32 containers -> 3xTF32."""
    B, H, W, Cin = x.shape
    Cout = w_hi.shape[1]
    f16 = w_hi.dtype == torch.float16
    y = out if out is not None else torch.empty((B, H, W, Cout), dtype=torch.float32, device=x.device)
    if stats_part is not None:
        # forward convolution + per-channel sums of its output (the next BatchNorm's batch statistics) from the epilogue
        assert relu_mask is None and in_scale is None and stats_part.dtype == torch.float64
        N.check(N.lib().fpd_conv2d_tc_h_stats(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(w_hi), _p(w_lo),
                                              int(f16), _p(bias), _p(residual), _p(y), float(out_scale), B, H, W, Cin,
                                              Cout, ksize, _p(stats_part), _p(stats_pivot), _stream()), "conv2d_tc_h_stats")
        return y
    N.check(N.lib().fpd_conv2d_tc_h(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(w_hi), _p(w_lo), int(f16),
                                    _p(bias), _p(residual), _p(relu_mask), _p(y), float(out_scale), _p(in_scale), B, H,
                                    W, Cin, Cout, ksize, _stream()), "conv2d_tc_h")
    return y


def conv2d_simt_fwd(x, w_oihw, bias=None, residual=None, stride=1, pad=0, out=None):
    B, H, W, Cin = x.shape
    Cout, _, k, _ = w_oihw.shape
    Ho = (H + 2 * pad - k) // stride + 1
    Wo = (W + 2 * pad - k) // stride + 1
    y = out if out is not None else torch.empty((B, Ho, Wo, Cout), dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_conv2d_simt_fwd(_p(x), _p(w_oihw), _p(bias), _p(residual), _p(y), B, H, W, Cin, Cout, k, stride,
                                        pad, _stream()), "conv2d_simt_fwd")
    return y


def conv2d_simt_dgrad(dy, w_oihw, in_hw, stride=1, pad=0, out=None):
    B = dy.shape[0]
    H, W = in_hw
    Cout, Cin, k, _ = w_oihw.shape
    dx = out if out is not None else torch.empty((B, H, W, Cin), dtype=torch.float32, device=dy.device)
    N.check(N.lib().fpd_conv2d_simt_dgrad(_p(dy), _p(w_oihw), _p(dx), B, H, W, Cin, Cout, k, stride, pad, _stream()),
            "conv2d_simt_dgrad")
    return dx


def conv2d_simt_wgrad(x, dy, k, stride=1, pad=0, scale=1.0, out=None):
    B, H, W, Cin = x.shape
    Cout = dy.shape[-1]
    dw = out if out is not None else torch.empty((Cout, Cin, k, k), dtype=torch.float32, device=x.device)
    ws = _ws.get(N.lib().fpd_conv2d_simt_wgrad_workspace_bytes(B, H, W, Cin, Cout, k, stride, pad), x.device)
    N.check(N.lib().fpd_conv2d_simt_wgrad(_p(x), _p(dy), _p(dw), float(scale), B, H, W, Cin, Cout, k, stride, pad,
                                          _p(ws), ws.numel(), _stream()), "conv2d_simt_wgrad")
    return dw


def conv2d_wgrad_tc_supported(cin, cout, k):
    return bool(N.lib().fpd_conv2d_wgrad_tc_supported(cin, cout, k))


def conv2d_wgrad_tc_fused(x, dy, ksize, mean=None, scale=None, shift=None, relu=False, passes=3, out_scale=1.0,
                          out=None):
    """dW for y = conv(relu?((x-mean)*scale+shift)) given raw x and raw dy (operand transform inside the kernel)."""
    B, H, W, Cin = x.shape
    Cout = dy.shape[-1]
    dw = out if out is not None else torch.empty((Cout, Cin, ksize, ksize), dtype=torch.float32, device=x.device)
    nb = N.lib().fpd_conv2d_wgrad_tc_workspace_bytes(B, H, W, Cin, Cout, ksize)
    ws = _ws.get(nb, x.device)
    N.check(N.lib().fpd_conv2d_wgrad_tc_fused(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(dy), int(passes),
                                              _p(dw), float(out_scale), B, H, W, Cin, Cout, ksize, _p(ws), ws.numel(),
                                              _stream()), "conv2d_wgrad_tc_fused")
    return dw


def wgrad_channel_chunks(cin, cout, k):
    """(input-channel chunk, output-channel chunk) widths the tensor-core weight-gradient kernels take, for convolutions
    that are too wide for one launch (HRNet's 256-channel 3x3, pose_resnet's 512..2048-channel layers); the largest
    supported pair of divisors. None if there is none."""
    for co in (cout, 256, 128, 64, 32):
        if co > cout or cout % co:
            continue
        for ci in (cin, 256, 128, 64, 32):
            if ci > cin or cin % ci:
                continue
            if conv2d_wgrad_tc_supported(ci, co, k):
                return ci, co
    return None


def conv2d_wgrad_tc_chunked(x, dy, ksize, chunks, mean=None, scale=None, shift=None, relu=False, passes=3):
    """dW of a wide convolution as one tensor-core weight-gradient launch per (input-channel, output-channel) chunk: the
    chunks of x / dY are made contiguous (strided copies -- these are the low-resolution, many-channel tensors), the BN
    parameters are slices."""
    Cin = x.shape[-1]
    Cout = dy.shape[-1]
    ci, co = chunks
    dw = torch.empty((Cout, Cin, ksize, ksize), dtype=torch.float32, device=x.device)
    dys = [dy if co == Cout else dy[..., o0:o0 + co].contiguous() for o0 in range(0, Cout, co)]
    for c0 in range(0, Cin, ci):
        sl = slice(c0, c0 + ci)
        xs = x if ci == Cin else x[..., sl].contiguous()
        for j, o0 in enumerate(range(0, Cout, co)):
            dws = conv2d_wgrad_tc_fused(xs, dys[j], ksize, mean=None if mean is None else mean[sl],
                                        scale=None if scale is None else scale[sl],
                                        shift=None if shift is None else shift[sl], relu=relu, passes=passes)
            dw[o0:o0 + co, sl] = dws
    return dw


def bn_stats(x):
    C = x.shape[-1]
    P = x.numel() // C
    mean = torch.empty(C, dtype=torch.float32, device=x.device)
    var = torch.empty_like(mean)
    ws = _ws.get(N.lib().fpd_bn_stats_workspace_bytes(P, C), x.device)
    N.check(N.lib().fpd_bn_stats(_p(x), P, C, _p(mean), _p(var), _p(ws), ws.numel(), _stream()), "bn_stats")
    return mean, var


def bn_finalize(mean, var, gamma, beta, eps, count, running_mean=None, running_var=None, momentum=0.1):
    C = mean.numel()
    scale = torch.empty_like(mean)
    shift = torch.empty_like(mean)
    invstd = torch.empty_like(mean)
    N.check(N.lib().fpd_bn_finalize(_p(mean), _p(var), _p(gamma), _p(beta), float(eps), int(count), _p(scale),
                                    _p(shift), _p(invstd), _p(running_mean), _p(running_var), float(momentum), C,
                                    _stream()), "bn_finalize")
    return scale, shift, invstd


def channel_sum(dy, scale=1.0, want_amax=False):
    """Per-channel sum of dy (bias gradient). want_amax=True also returns the float[2] device tensor {S, 1/S} with S the
    power of two that puts max|dy| into [2^14, 2^15) (operand scale of the 3xFP16 gradient convolutions), or None when
    the fused reduction is unavailable (C % 4 != 0)."""
    C = dy.shape[-1]
    P = dy.numel() // C
    out = torch.empty(C, dtype=torch.float32, device=dy.device)
    ws = _ws.get(N.lib().fpd_channel_reduce_workspace_bytes(P, C), dy.device)
    if FUSED_REDUCE and C % 4 == 0:
        amax = torch.empty(2, dtype=torch.float32, device=dy.device) if want_amax else None
        N.check(N.lib().fpd_channel_sum_fused(_p(dy), P, C, float(scale), _p(out), _p(amax), _p(ws), ws.numel(),
                                              _p(_counter(dy.device)), _stream()), "channel_sum_fused")
        return (out, amax) if want_amax else out
    N.check(N.lib().fpd_channel_sum(_p(dy), P, C, float(scale), _p(out), _p(ws), ws.numel(), _stream()), "channel_sum")
    return (out, None) if want_amax else out


def bn_stats_finalize(x, gamma, beta, eps, running_mean=None, running_var=None, momentum=0.1):
    """Train-mode BatchNorm2d statistics of x plus the finalize step of one consuming BN, in ONE launch.
    Returns (mean, var_biased, scale, shift, invstd)."""
    C = x.shape[-1]
    P = x.numel() // C
    mean = torch.empty(C, dtype=torch.float32, device=x.device)
    var, scale, shift, invstd = (torch.empty_like(mean) for _ in range(4))
    ws = _ws.get(N.lib().fpd_bn_stats_workspace_bytes(P, C), x.device)
    N.check(N.lib().fpd_bn_stats_fused(_p(x), P, C, _p(gamma), _p(beta), float(eps), float(momentum),
                                       _p(running_mean), _p(running_var), _p(mean), _p(var), _p(scale), _p(shift),
                                       _p(invstd), _p(ws), ws.numel(), _p(_counter(x.device)), _stream()),
            "bn_stats_fused")
    return mean, var, scale, shift, invstd


def bn_bwd_reduce(da, x, mean, invstd, scale, shift, relu):
    """sums[0:C] = sum dz (= dbeta), sums[C:2C] = sum dz*xhat (= dgamma), dz = da masked by the ReLU."""
    C = x.shape[-1]
    P = x.numel() // C
    sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
    ws = _ws.get(N.lib().fpd_channel_reduce_workspace_bytes(P, C), x.device)
    if FUSED_REDUCE:
        N.check(N.lib().fpd_bn_bwd_reduce_fused(_p(da), _p(x), _p(mean), _p(invstd), _p(scale), _p(shift), int(relu), P,
                                                C, _p(sums), _p(ws), ws.numel(), _p(_counter(x.device)), _stream()),
                "bn_bwd_reduce_fused")
        return sums
    N.check(N.lib().fpd_bn_bwd_reduce(_p(da), _p(x), _p(mean), _p(invstd), _p(scale), _p(shift), int(relu), P, C,
                                      _p(sums), _p(ws), ws.numel(), _stream()), "bn_bwd_reduce")
    return sums


# bias-gradient sums + dY operand scale out of the BN-backward apply pass (one launch and one read of dx less per conv);
# not a measurable gain on the bench configuration (hg_fpd, one H100 SXM at 700 W: 83.9 / 83.3 ms/step on, 83.9 / 84.0
# off -- within the run-to-run spread), so off by default
BN_APPLY_SUM = os.environ.get("FPD_BN_APPLY_SUM", "0") != "0"


def bn_bwd(da, x, mean, invstd, scale, shift, gamma, relu, accumulate_into=None, sync_mean=None, want_dx_sum=False):
    """Returns (dx, dgamma, dbeta) for y = relu?(bn(x)) given da = dL/dy (train-mode batch statistics).
    sync_mean: optional callable sums[2C] -> the MEAN over ranks of the per-rank sums (SyncBN, parallel.allreduce_avg):
    the batch-statistics terms of dx then use the statistics of the global batch (global sum / global count =
    rank-mean of the sums / local count), while dgamma / dbeta stay this rank's sums (the gradient all-reduce averages
    them like every other parameter gradient)."""
    C = x.shape[-1]
    P = x.numel() // C
    sums = bn_bwd_reduce(da, x, mean, invstd, scale, shift, relu)
    apply_sums = sums if sync_mean is None else sync_mean(sums)
    dx = accumulate_into if accumulate_into is not None else torch.empty_like(x)
    if (want_dx_sum and accumulate_into is None and FUSED_REDUCE and (BN_APPLY_SUM or want_dx_sum == "force")
            and C % 4 == 0):
        # the same pass also yields sum_pixels(dx) per channel and the operand scale of dx: what channel_sum(dx,
        # want_amax=True) would compute for the bias gradient / 3xFP16 data gradient of the conv that produced x
        dx_sum = torch.empty(C, dtype=torch.float32, device=x.device)
        amax = torch.empty(2, dtype=torch.float32, device=x.device)
        ws = _ws.get(N.lib().fpd_channel_reduce_workspace_bytes(P, C), x.device)
        N.check(N.lib().fpd_bn_bwd_apply_sum(_p(da), _p(x), _p(mean), _p(invstd), _p(scale), _p(shift), _p(gamma), int(relu),
                                             _p(apply_sums), _p(dx), _p(dx_sum), _p(amax), P, C, _p(ws), ws.numel(),
                                             _stream()), "bn_bwd_apply_sum")
        return dx, sums[C:], sums[:C], (dx_sum, amax)
    N.check(N.lib().fpd_bn_bwd_apply(_p(da), _p(x), _p(mean), _p(invstd), _p(scale), _p(shift), _p(gamma), int(relu),
                                     _p(apply_sums), int(accumulate_into is not None), _p(dx), P, C, _stream()),
            "bn_bwd_apply")
    if want_dx_sum:
        return dx, sums[C:], sums[:C], None
    return dx, sums[C:], sums[:C]


def affine_act_bwd(da, x, scale, shift, relu, accumulate_into=None, mean=None):
    C = x.shape[-1]
    P = x.numel() // C
    dx = accumulate_into if accumulate_into is not None else torch.empty_like(x)
    N.check(N.lib().fpd_affine_act_bwd(_p(da), _p(x), _p(mean), _p(scale), _p(shift), int(relu),
                                       int(accumulate_into is not None), _p(dx), P, C, _stream()), "affine_act_bwd")
    return dx


def maxpool2x2(x, out=None):
    B, H, W, C = x.shape
    y = out if out is not None else torch.empty((B, H // 2, W // 2, C), dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_maxpool2x2_fwd(_p(x), _p(y), B, H, W, C, _stream()), "maxpool2x2_fwd")
    return y


def maxpool2x2_bwd(x, dy, accumulate_into=None):
    B, H, W, C = x.shape
    dx = accumulate_into if accumulate_into is not None else torch.empty_like(x)
    N.check(N.lib().fpd_maxpool2x2_bwd(_p(x), _p(dy), _p(dx), int(accumulate_into is not None), B, H, W, C, _stream()),
            "maxpool2x2_bwd")
    return dx


def upsample2x_add(up1, low, out=None):
    B, H, W, C = up1.shape
    y = out if out is not None else torch.empty_like(up1)
    N.check(N.lib().fpd_upsample2x_add(_p(up1), _p(low), _p(y), B, H, W, C, _stream()), "upsample2x_add")
    return y


def upsample2x_bwd(dout, out=None):
    B, H, W, C = dout.shape
    d = out if out is not None else torch.empty((B, H // 2, W // 2, C), dtype=torch.float32, device=dout.device)
    N.check(N.lib().fpd_upsample2x_bwd(_p(dout), _p(d), B, H, W, C, _stream()), "upsample2x_bwd")
    return d


def maxpool3x3s2(x):
    """nn.MaxPool2d(3, stride=2, padding=1) on NHWC (pose_resnet stem, reference pose_resnet.py:107)."""
    B, H, W, C = x.shape
    y = torch.empty((B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C), dtype=x.dtype, device=x.device)
    N.check(N.lib().fpd_maxpool3x3s2_fwd(_p(x), _p(y), B, H, W, C, _stream()), "maxpool3x3s2_fwd")
    return y


def maxpool3x3s2_bwd(x, dy, accumulate_into=None):
    B, H, W, C = x.shape
    dx = accumulate_into if accumulate_into is not None else torch.empty_like(x)
    N.check(N.lib().fpd_maxpool3x3s2_bwd(_p(x), _p(dy), _p(dx), int(accumulate_into is not None), B, H, W, C, _stream()),
            "maxpool3x3s2_bwd")
    return dx


def depth_to_space2(y):
    """[B,H,W,4C] -> [B,2H,2W,C]: out[b,2a+rh,2c+rw,co] = y[b,a,c,(2rh+rw)C+co] (tail of the deconv-as-3x3-conv)."""
    B, H, W, C4 = y.shape
    C = C4 // 4
    out = torch.empty((B, 2 * H, 2 * W, C), dtype=y.dtype, device=y.device)
    N.check(N.lib().fpd_depth_space2(_p(y), _p(out), B, H, W, C, 0, _stream()), "depth_to_space2")
    return out


def space_to_depth2(g):
    """Inverse (= adjoint) of depth_to_space2: [B,2H,2W,C] -> [B,H,W,4C]."""
    B, H2, W2, C = g.shape
    out = torch.empty((B, H2 // 2, W2 // 2, 4 * C), dtype=g.dtype, device=g.device)
    N.check(N.lib().fpd_depth_space2(_p(g), _p(out), B, H2 // 2, W2 // 2, C, 1, _stream()), "space_to_depth2")
    return out


def deconv_weight_to_conv3(wd, pad):
    """ConvTranspose2d weight [Cin,Cout,k,k] (stride 2) -> OIHW [4*Cout,Cin,3,3] of the equivalent stride-1 convolution."""
    Cin, Cout, k, _ = wd.shape
    w3 = torch.empty((4 * Cout, Cin, 3, 3), dtype=torch.float32, device=wd.device)
    N.check(N.lib().fpd_deconv_weight_map(_p(wd), _p(w3), Cin, Cout, k, int(pad), 0, _stream()), "deconv_weight_map")
    return w3


def conv3_grad_to_deconv(dw3, k, pad):
    """Gradient of the ConvTranspose2d weight out of the equivalent convolution's [4*Cout,Cin,3,3] weight gradient."""
    Cout, Cin = dw3.shape[0] // 4, dw3.shape[1]
    dwd = torch.empty((Cin, Cout, k, k), dtype=torch.float32, device=dw3.device)
    N.check(N.lib().fpd_deconv_weight_map(_p(dw3), _p(dwd), Cin, Cout, int(k), int(pad), 1, _stream()),
            "deconv_weight_map")
    return dwd


def subsample2(x, out=None):
    """y[b, ho, wo] = x[b, 2 ho, 2 wo]: the stride-2 pick after a stride-1 3x3 convolution (pad 1)."""
    B, H, W, C = x.shape
    y = out if out is not None else torch.empty((B, H // 2, W // 2, C), dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_subsample2(_p(x), _p(y), B, H, W, C, _stream()), "subsample2")
    return y


def upsample_zero2(dy, out=None):
    """Adjoint of subsample2: dy scattered to the even positions of a zero [B, 2Ho, 2Wo, C] tensor."""
    B, Ho, Wo, C = dy.shape
    dx = out if out is not None else torch.empty((B, 2 * Ho, 2 * Wo, C), dtype=torch.float32, device=dy.device)
    N.check(N.lib().fpd_upsample_zero2(_p(dy), _p(dx), B, Ho, Wo, C, _stream()), "upsample_zero2")
    return dx


def nchw_to_nhwc(x, out=None):
    B, C, H, W = x.shape
    y = out if out is not None else torch.empty((B, H, W, C), dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_nchw_to_nhwc(_p(x), _p(y), B, C, H, W, _stream()), "nchw_to_nhwc")
    return y


def nchw_to_nhwc_flipw(x, out=None):
    """NHWC copy of the W-mirrored image (flip-test input, function.py:218-221) in the same single pass."""
    B, C, H, W = x.shape
    y = out if out is not None else torch.empty((B, H, W, C), dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_nchw_to_nhwc_flipw(_p(x), _p(y), B, C, H, W, _stream()), "nchw_to_nhwc_flipw")
    return y


def nhwc_to_nchw(x, out=None):
    B, H, W, C = x.shape
    y = out if out is not None else torch.empty((B, C, H, W), dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_nhwc_to_nchw(_p(x), _p(y), B, C, H, W, _stream()), "nhwc_to_nchw")
    return y


def add(a, b, out=None):
    o = out if out is not None else torch.empty_like(a)
    N.check(N.lib().fpd_add(_p(a), _p(b), _p(o), a.numel(), _stream()), "add")
    return o


def fpd_loss(outs_nhwc, target_nchw, teacher_nhwc, target_weight, alpha, want_grads=True, grad_scale=1.0,
             grads_out=None, losses_out=None):
    """Fused FPD loss. outs_nhwc: list of [B,h,w,J]; returns (losses[3] device tensor, grads list or None)."""
    S = len(outs_nhwc)
    B, h, w, J = outs_nhwc[0].shape
    dev = outs_nhwc[0].device
    tw = target_weight.reshape(B, J).contiguous()
    losses = losses_out if losses_out is not None else torch.empty(3, dtype=torch.float32, device=dev)
    grads = None
    if want_grads:
        grads = grads_out if grads_out is not None else [torch.empty_like(o) for o in outs_nhwc]
    outs_arr = (ctypes.c_void_p * S)(*[o.data_ptr() for o in outs_nhwc])
    grads_arr = (ctypes.c_void_p * S)(*[g.data_ptr() for g in grads]) if grads is not None else None
    ws = _ws.get(N.lib().fpd_loss_workspace_bytes(B, J, h, w), dev)
    N.check(N.lib().fpd_loss_fused(outs_arr, S, _p(target_nchw), _p(teacher_nhwc), _p(tw), float(alpha), grads_arr,
                                   float(grad_scale), _p(losses), B, J, h, w, _p(ws), ws.numel(), _stream()),
            "loss_fused")
    return losses, grads


def joints_mse(out_nchw, target_nchw, target_weight=None, want_grad=True):
    B, J = out_nchw.shape[:2]
    hw = out_nchw.numel() // (B * J)
    dev = out_nchw.device
    loss3 = torch.empty(3, dtype=torch.float32, device=dev)
    grad = torch.empty_like(out_nchw) if want_grad else None
    tw = None if target_weight is None else target_weight.reshape(B, J).contiguous()
    ws = _ws.get(1 << 16, dev)
    N.check(N.lib().fpd_joints_mse(_p(out_nchw), _p(target_nchw), _p(tw), _p(loss3), _p(grad), B, J, hw, _p(ws),
                                   ws.numel(), _stream()), "joints_mse")
    return loss3, grad


def flip_merge_argmax(hm_nhwc, hm_flip_nhwc=None, flip_perm=None, shift=False, want_avg=True):
    B, h, w, J = hm_nhwc.shape
    dev = hm_nhwc.device
    avg = torch.empty_like(hm_nhwc) if want_avg else None
    idx = torch.empty((B, J), dtype=torch.int32, device=dev)
    maxval = torch.empty((B, J), dtype=torch.float32, device=dev)
    N.check(N.lib().fpd_flip_merge_argmax(_p(hm_nhwc), _p(hm_flip_nhwc), _p(flip_perm), int(shift), _p(avg), _p(idx),
                                          _p(maxval), B, J, h, w, _stream()), "flip_merge_argmax")
    return avg, idx, maxval


def argmax_nchw(hm):
    B, J = hm.shape[:2]
    hw = hm.numel() // (B * J)
    idx = torch.empty((B, J), dtype=torch.int32, device=hm.device)
    maxval = torch.empty((B, J), dtype=torch.float32, device=hm.device)
    N.check(N.lib().fpd_argmax_nchw(_p(hm), _p(idx), _p(maxval), B * J, hw, _stream()), "argmax_nchw")
    return idx, maxval


def nms_device(boxes_sorted, thresh):
    n, d = boxes_sorted.shape
    dev = boxes_sorted.device
    keep = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    num = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = _ws.get(N.lib().fpd_nms_workspace_bytes(n), dev)
    N.check(N.lib().fpd_nms_device(_p(boxes_sorted), n, d, float(thresh), _p(keep), _p(num), _p(ws), ws.numel(),
                                   _stream()), "nms_device")
    return keep, num


def adam_flat(param, grad, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0):
    N.check(N.lib().fpd_adam_flat(_p(param), _p(grad), _p(exp_avg), _p(exp_avg_sq), param.numel(), float(lr),
                                  float(beta1), float(beta2), float(eps), float(weight_decay), int(step),
                                  float(grad_scale), _stream()), "adam_flat")


def oks_nms_device(kpts_sorted, areas_sorted, thresh, sigmas=None, in_vis_thre=None):
    """OKS-NMS on the device (csrc/nms.cu; reference lib/nms/nms.py:75-124). kpts_sorted: CUDA [n,J,3] float32 or float64
    (x, y, score), persons sorted by score descending; areas_sorted: CUDA float64 [n]. Returns (keep int32[n], num int32[1])
    device tensors -- indices into the sorted list, best first."""
    n, J = kpts_sorted.shape[0], kpts_sorted.shape[1]
    dev = kpts_sorted.device
    assert kpts_sorted.dtype in (torch.float32, torch.float64) and kpts_sorted.is_contiguous()
    areas = areas_sorted.to(torch.float64).contiguous()
    if sigmas is None:
        sigmas = COCO_SIGMAS
    vars_ = (torch.as_tensor(sigmas, dtype=torch.float64) * 2) ** 2
    vars_ = vars_.to(dev)
    keep = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    num = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = _ws.get(N.lib().fpd_nms_workspace_bytes(n), dev)
    N.check(N.lib().fpd_oks_nms_device(_p(kpts_sorted), int(kpts_sorted.dtype == torch.float64), _p(areas), _p(vars_), n, J,
                                       float(thresh), int(in_vis_thre is not None),
                                       float(in_vis_thre if in_vis_thre is not None else 0.0), _p(keep), _p(num), _p(ws),
                                       ws.numel(), _stream()), "oks_nms_device")
    return keep, num


# lib/nms/nms.py:77: per-joint falloff constants of the COCO key-point metric
COCO_SIGMAS = [x / 10.0 for x in (.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89)]


def oks_rescore(kpts, box_score, in_vis_thre):
    """out[i] = box_score[i] * mean(joint scores above in_vis_thre) (lib/dataset/coco.py:346-357); float64 CUDA tensor."""
    n, J = kpts.shape[0], kpts.shape[1]
    assert kpts.dtype in (torch.float32, torch.float64) and kpts.is_contiguous()
    bs = box_score.to(torch.float64).contiguous()
    out = torch.empty(n, dtype=torch.float64, device=kpts.device)
    N.check(N.lib().fpd_oks_rescore(_p(kpts), int(kpts.dtype == torch.float64), _p(bs), n, J, float(in_vis_thre), _p(out),
                                    _stream()), "oks_rescore")
    return out


def gaussian_targets(joints, joints_vis, heatmap_size, image_size, sigma=2, joints_weight=None, gauss_table=None):
    """Batch form of JointsDataset.generate_target (lib/dataset/JointsDataset.py:233-289). joints / joints_vis: CUDA float32
    [N,J,3]; heatmap_size / image_size: (w, h). Returns (target [N,J,h,w], target_weight [N,J,1])."""
    import numpy as np
    _chk(joints, "joints")
    _chk(joints_vis, "joints_vis")
    n, J = joints.shape[0], joints.shape[1]
    W, H = int(heatmap_size[0]), int(heatmap_size[1])
    dev = joints.device
    if gauss_table is None:
        # the reference's own expression (float32 numpy), so the stamped patch is bit-identical: JointsDataset.py:266-272
        size = 2 * (sigma * 3) + 1
        xs = np.arange(0, size, 1, np.float32)
        ys = xs[:, np.newaxis]
        x0 = y0 = size // 2
        g = np.exp(- ((xs - x0) ** 2 + (ys - y0) ** 2) / (2 * sigma ** 2))
        gauss_table = torch.from_numpy(np.ascontiguousarray(g, dtype=np.float32)).to(dev)
    target = torch.empty((n, J, H, W), dtype=torch.float32, device=dev)
    tw = torch.empty((n, J, 1), dtype=torch.float32, device=dev)
    jw = None if joints_weight is None else joints_weight.to(dev).float().contiguous().reshape(-1)
    N.check(N.lib().fpd_gaussian_targets(_p(joints), _p(joints_vis), _p(jw), _p(gauss_table), _p(target), _p(tw), n, J, H, W,
                                         int(image_size[0]), int(image_size[1]), int(sigma), _stream()), "gaussian_targets")
    return target, tw
