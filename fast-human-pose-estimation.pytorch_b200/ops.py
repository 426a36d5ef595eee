"""Tensor-level wrappers over the C ABI: torch is used only for device memory and streams.

Every function takes contiguous fp32 CUDA tensors, enqueues on torch's current stream and returns
(or fills) tensors. Activations are NHWC ([B,H,W,C]) unless a name says otherwise.
"""
import ctypes
import math
import numbers
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
    concurrently and must not share reduction scratch.
    A buffer that was handed to a CUDA graph capture is kept when a larger request outgrows it: the graph holds its
    address. Streams come from torch's pool of 32, so two captured steps in one process (e.g. two FPDTrainSteps) can share
    a stream handle, and the second one's larger request must not free memory the first one's graph still writes. Other
    outgrown buffers are freed."""

    def __init__(self):
        self.bufs = {}
        self.in_graph = set()      # keys whose current buffer a capture has taken
        self.outgrown = []         # outgrown buffers that captured graphs may still use

    def get(self, nbytes, device):
        nbytes = int(nbytes)
        key = (device, torch.cuda.current_stream(device).cuda_stream)
        buf = self.bufs.get(key)
        if buf is None or buf.numel() < nbytes:
            if key in self.in_graph:
                self.outgrown.append(buf)
                self.in_graph.discard(key)
            buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
            self.bufs[key] = buf
        if torch.cuda.is_current_stream_capturing():
            self.in_graph.add(key)
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


def conv2d_tc_supported(cin, cout, k):
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


CONV1X1 = os.environ.get("FPD_CONV1X1", "1") != "0"   # 1x1 3xFP16 convolutions on the weight-resident kernel


def set_conv1x1(enabled):
    """Run 1x1 3xFP16 convolutions (without epilogue statistics) on the weight-resident kernel (True) or on the staged
    kernel (False), process-wide, for launches made after the call. The results are bit-identical. Returns the previous
    setting."""
    global CONV1X1
    prev = bool(N.lib().fpd_set_conv1x1(int(bool(enabled))))
    CONV1X1 = bool(enabled)
    return prev


if not CONV1X1:
    set_conv1x1(False)


def set_conv_halo(enabled):
    """Run 3x3 3xFP16 convolutions on the halo-resident kernel where it fits (True, the default) or on the staged
    kernel (False), process-wide, for launches made after the call; for comparing the two, whose results are
    bit-identical. Returns the previous setting."""
    return bool(N.lib().fpd_set_conv_halo(int(bool(enabled))))


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


def weight_prep_f16_both(w_oihw, split=True):
    """-> ((fwd_hi, fwd_lo), (dgrad_hi, dgrad_lo)) in one launch; split=False: the lo halves are None (the single-pass
    FP16 operands of conv2d_tc_f16x1)."""
    _chk(w_oihw, "w")
    O, I, k, _ = w_oihw.shape
    f_hi = torch.empty((k * k, O, I), dtype=torch.float16, device=w_oihw.device)
    f_lo = torch.empty_like(f_hi) if split else None
    d_hi = torch.empty((k * k, I, O), dtype=torch.float16, device=w_oihw.device)
    d_lo = torch.empty_like(d_hi) if split else None
    N.check(N.lib().fpd_weight_prep_f16_both(_p(w_oihw), _p(f_hi), _p(f_lo), _p(d_hi), _p(d_lo), O, I, k, _stream()),
            "weight_prep_f16_both")
    return (f_hi, f_lo), (d_hi, d_lo)


# BatchNorm statistics of conv outputs from the conv epilogue: "0" off, "1" every tensor-core conv, "3x3" only the 3x3
# convolutions. On the bench configuration (hg_fpd, one H100 SXM at 700 W, two runs each) the three settings are within
# noise of each other: 3x3 83.9 / 84.0 ms/step, off 84.0 / 83.9, every conv 83.9 / 83.9. "3x3" is kept: it saves the
# separate statistics pass over the largest tensors without adding epilogue work to the 1x1 convolutions.
CONV_STATS = os.environ.get("FPD_CONV_STATS", "3x3").lower()


def conv2d_tc_stats_blocks(B, H, W, Cin, Cout, k, f16, single_pass=False):
    """Number of per-CTA partial blocks the statistics call (stats_part=) of conv2d_tc_h (f16: fp16 weights) or, with
    single_pass, conv2d_tc_f16x1 writes; 0 if the call should carry no statistics (CONV_STATS) or the shape cannot."""
    if CONV_STATS == "0" or (CONV_STATS == "3x3" and k != 3):
        return 0
    if single_pass:
        return conv2d_tc_f16x1_train_plan(B, H, W, Cin, Cout, k, stats=True)[1]
    return int(N.lib().fpd_conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, k, int(f16)))


def conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, k, f16):
    """Number of per-CTA partial blocks conv2d_tc_h(..., stats_part=) writes; 0 if the shape cannot carry statistics."""
    return conv2d_tc_stats_blocks(B, H, W, Cin, Cout, k, f16)


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


F16X1_KERNELS = {0: None, 1: "staged", 2: "halo", 3: "1x1"}


def conv2d_tc_f16x1_kernel(B, H, W, Cin, Cout, k):
    """Which kernel conv2d_tc_f16x1 runs this shape on: "halo" (3x3, conv_halo_f16x1_kernel), "1x1"
    (pw_conv_f16x1_kernel), "staged" (conv_wgmma_kernel) or None (unsupported). Host only."""
    return F16X1_KERNELS[int(N.lib().fpd_conv2d_tc_f16x1_kernel(B, H, W, Cin, Cout, k))]


def conv2d_tc_f16x1_train_plan(B, H, W, Cin, Cout, k, stats=False):
    """-> (kernel, stat_blocks): the kernel conv2d_tc_f16x1 runs this shape on with (stats=True) or without epilogue
    statistics, named as conv2d_tc_f16x1_kernel, and the number of partial blocks a statistics call writes (0 without
    statistics or when the shape cannot carry them). Host only."""
    nblk = ctypes.c_int(0)
    kind = int(N.lib().fpd_conv2d_tc_f16x1_train_plan(B, H, W, Cin, Cout, k, int(bool(stats)), ctypes.byref(nblk)))
    return F16X1_KERNELS[kind], int(nblk.value)


def conv2d_tc_f16x1_stats_blocks(B, H, W, Cin, Cout, k):
    """conv2d_tc_h_stats_blocks for conv2d_tc_f16x1(stats_part=...): 0 if the call should carry no statistics."""
    return conv2d_tc_stats_blocks(B, H, W, Cin, Cout, k, True, single_pass=True)


def conv2d_tc_f16x1(x, w, ksize, mean=None, scale=None, shift=None, relu=False, bias=None, residual=None,
                    relu_mask=None, out=None, out_scale=1.0, in_scale=None, stats_part=None, stats_pivot=None):
    """y = conv(relu?((x-mean)*scale+shift)) with single-pass FP16 operands: fp16_rn of the transformed activation times
    w = weight_prep_f16(w_oihw, split=False)[0], one MMA per product, fp32 accumulation (about 2^-11 relative operand
    rounding).
    Training calls (set_training_precision "fp16"): in_scale, the device float[2] {S, 1/S} of channel_sum(want_amax=True),
    makes the operand fp16_rn(x * S) and divides the output by S (data gradients: x = dY, S puts max |dY| into
    [2^14, 2^15)); stats_part [conv2d_tc_f16x1_stats_blocks(...)][Cout][2] fp64 receives the output's per-channel sums
    as conv2d_tc_h(stats_part=...) does."""
    B, H, W, Cin = x.shape
    Cout = w.shape[1]
    if w.dtype != torch.float16:
        raise ValueError("conv2d_tc_f16x1 takes the __half weights of weight_prep_f16(split=False), got %s" % w.dtype)
    y = out if out is not None else torch.empty((B, H, W, Cout), dtype=torch.float32, device=x.device)
    if in_scale is None and stats_part is None:
        N.check(N.lib().fpd_conv2d_tc_f16x1(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(w), _p(bias),
                                            _p(residual), _p(relu_mask), _p(y), float(out_scale), B, H, W, Cin, Cout,
                                            ksize, _stream()), "conv2d_tc_f16x1")
        return y
    assert stats_part is None or stats_part.dtype == torch.float64
    N.check(N.lib().fpd_conv2d_tc_f16x1_train(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(w), _p(bias),
                                              _p(residual), _p(relu_mask), _p(y), float(out_scale), _p(in_scale), B, H,
                                              W, Cin, Cout, ksize, _p(stats_part), _p(stats_pivot), _stream()),
            "conv2d_tc_f16x1_train")
    return y


# ---- fp16 activation storage (engine.set_inference_precision(model, "fp16_act")): the eval-forward kernels with __half
# NHWC activations. Each computes what its fp32 form computes, in fp32 from the widened inputs, and stores one
# fp16_rn per value saturated to +-65504 (NaN stays NaN).
def _chk_f16(t, name, dtypes=(torch.float16,)):
    if t is None:
        return
    if not (t.is_cuda and t.dtype in dtypes and t.is_contiguous()):
        raise ValueError("%s must be a contiguous %s CUDA tensor (got %s %s %s)" % (
            name, " or ".join(str(d) for d in dtypes), t.device, t.dtype, t.is_contiguous()))


def conv2d_tc_f16x1_io(x, w, ksize, mean=None, scale=None, shift=None, relu=False, bias=None, residual=None,
                       out_dtype=torch.float16, out=None, out_scale=1.0):
    """conv2d_tc_f16x1 (no ReLU mask) with fp32 or fp16 x, and y and the residual of out_dtype (fp32 or fp16): bit for
    bit conv2d_tc_f16x1 on x.float() and residual.float(), rounded as above when out_dtype is fp16. Only for the shapes
    conv2d_tc_f16x1_kernel runs on "halo" or "1x1"; others raise."""
    B, H, W, Cin = x.shape
    Cout = w.shape[1]
    if w.dtype != torch.float16:
        raise ValueError("conv2d_tc_f16x1_io takes the __half weights of weight_prep_f16(split=False), got %s" % w.dtype)
    both = (torch.float32, torch.float16)
    if out_dtype not in both:
        raise ValueError("conv2d_tc_f16x1_io: out_dtype must be torch.float32 or torch.float16, got %s" % out_dtype)
    _chk_f16(x, "x", both)
    _chk_f16(residual, "residual", (out_dtype,))
    y = out if out is not None else torch.empty((B, H, W, Cout), dtype=out_dtype, device=x.device)
    _chk_f16(y, "out", (out_dtype,))
    N.check(N.lib().fpd_conv2d_tc_f16x1_io(_p(x), int(x.dtype == torch.float16), _p(mean), _p(scale), _p(shift),
                                           int(relu), _p(w), _p(bias), _p(residual), _p(y),
                                           int(out_dtype == torch.float16), float(out_scale), B, H, W, Cin, Cout, ksize,
                                           _stream()), "conv2d_tc_f16x1_io")
    return y


def affine_act_f16(x, scale=None, shift=None, relu=False, out=None, mean=None):
    _chk_f16(x, "x")
    C = x.shape[-1]
    y = out if out is not None else torch.empty_like(x)
    N.check(N.lib().fpd_affine_act_f16(_p(x), _p(mean), _p(scale), _p(shift), int(relu), _p(y), x.numel() // C, C,
                                       _stream()), "affine_act_f16")
    return y


def affine_add_act_f16(x, residual, scale=None, shift=None, relu=True, mean=None, out=None):
    _chk_f16(x, "x")
    _chk_f16(residual, "residual")
    C = x.shape[-1]
    y = out if out is not None else torch.empty_like(x)
    N.check(N.lib().fpd_affine_add_act_f16(_p(x), _p(mean), _p(scale), _p(shift), _p(residual), int(relu), _p(y),
                                           x.numel() // C, C, _stream()), "affine_add_act_f16")
    return y


def fuse_sum_f16(terms, shifts, relu=True, out=None):
    n = len(terms)
    for t in terms:
        _chk_f16(t, "terms")
    B, C = terms[0].shape[0], terms[0].shape[-1]
    H, W = terms[0].shape[1] << shifts[0], terms[0].shape[2] << shifts[0]
    y = out if out is not None else torch.empty((B, H, W, C), dtype=torch.float16, device=terms[0].device)
    arr = (ctypes.c_void_p * n)(*[t.data_ptr() for t in terms])
    sh = (ctypes.c_int * n)(*[int(s) for s in shifts])
    N.check(N.lib().fpd_fuse_sum_f16(arr, sh, n, int(relu), _p(y), B, H, W, C, _stream()), "fuse_sum_f16")
    return y


def maxpool2x2_f16(x, out=None):
    _chk_f16(x, "x")
    B, H, W, C = x.shape
    y = out if out is not None else torch.empty((B, H // 2, W // 2, C), dtype=torch.float16, device=x.device)
    N.check(N.lib().fpd_maxpool2x2_fwd_f16(_p(x), _p(y), B, H, W, C, _stream()), "maxpool2x2_fwd_f16")
    return y


def _chk_low(up1, low, name):
    """up1 + upsample2x(low) needs low of (B, H / 2, W / 2, C): the kernel reads low's shape from up1's."""
    B, H, W, C = up1.shape
    if tuple(low.shape) != (B, H // 2, W // 2, C):
        raise ValueError("%s: low must be %s for up1 of %s, got %s" % (
            name, (B, H // 2, W // 2, C), tuple(up1.shape), tuple(low.shape)))


def upsample2x_add_f16(up1, low, out=None):
    _chk_f16(up1, "up1")
    _chk_f16(low, "low")
    _chk_low(up1, low, "upsample2x_add_f16")
    B, H, W, C = up1.shape
    y = out if out is not None else torch.empty_like(up1)
    N.check(N.lib().fpd_upsample2x_add_f16(_p(up1), _p(low), _p(y), B, H, W, C, _stream()), "upsample2x_add_f16")
    return y


def subsample2_f16(x, out=None):
    _chk_f16(x, "x")
    B, H, W, C = x.shape
    y = out if out is not None else torch.empty((B, H // 2, W // 2, C), dtype=torch.float16, device=x.device)
    N.check(N.lib().fpd_subsample2_f16(_p(x), _p(y), B, H, W, C, _stream()), "subsample2_f16")
    return y


def half_to_float(x, out=None):
    """float(x) of an fp16 activation: the one explicit widening before a call that has no fp16 form."""
    _chk_f16(x, "x")
    y = out if out is not None else torch.empty(x.shape, dtype=torch.float32, device=x.device)
    N.check(N.lib().fpd_half_to_float(_p(x), _p(y), x.numel(), _stream()), "half_to_float")
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


WGRAD_HALO = os.environ.get("FPD_WGRAD_HALO", "1") != "0"   # weight gradients on the tap-row kernel


def set_wgrad_halo(enabled):
    """Run weight gradients on the tap-row kernel where it takes the shape (True) or all on the per-tap kernel (False),
    process-wide, for launches made after the call. The results are bit-identical. Returns the previous setting."""
    global WGRAD_HALO
    prev = bool(N.lib().fpd_set_wgrad_halo(int(bool(enabled))))
    WGRAD_HALO = bool(enabled)
    return prev


if not WGRAD_HALO:
    set_wgrad_halo(False)


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
    _chk_low(up1, low, "upsample2x_add")
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


def _check_topk(topk, J, lo, name):
    if int(topk) != topk or not lo <= topk <= J:
        raise ValueError("%s=%r out of range [%d, J=%d]" % (name, topk, lo, J))
    return int(topk)


def _check_temperature(t, name, allow_zero):
    """A JointsKLDLoss temperature: finite and > 0 (0 = "not KL" where allow_zero)."""
    if isinstance(t, bool) or not isinstance(t, numbers.Real) or not (math.isfinite(t) and (t > 0 or (allow_zero and t == 0))):
        raise ValueError("%s=%r must be a finite number > 0%s" % (name, t, " (or 0: not KL)" if allow_zero else ""))
    return float(t)


def check_kd_unlabeled_thre(thre):
    """The confidence threshold of distillation from unlabeled samples: a finite number."""
    if isinstance(thre, bool) or not isinstance(thre, numbers.Real) or not math.isfinite(thre):
        raise ValueError("kd_unlabeled_thre=%r must be a finite number" % (thre,))
    return float(thre)


def kd_weights(teacher_nhwc, target_weight, thre, out=None):
    """The kd term's weights [B,J] (device) for distillation from unlabeled samples: a sample whose target weights are
    all exactly 0 gets 1.0 for joint j when the teacher's map teacher_nhwc[b, :, :, j] has a maximum > thre (0.0
    otherwise, and for a map holding a NaN); every other sample keeps its target weights."""
    thre = check_kd_unlabeled_thre(thre)
    if teacher_nhwc is None:
        raise ValueError("kd_weights: the teacher's heat-maps are required")
    _chk(teacher_nhwc, "teacher")
    B, h, w, J = teacher_nhwc.shape
    tw = target_weight.reshape(B, J).contiguous()
    _chk(tw, "target_weight")
    kdw = out if out is not None else torch.empty(B, J, dtype=torch.float32, device=teacher_nhwc.device)
    N.check(N.lib().fpd_kd_weights(_p(teacher_nhwc), _p(tw), thre, _p(kdw), B, J, h, w, _stream()), "kd_weights")
    return kdw


def fpd_loss(outs_nhwc, target_nchw, teacher_nhwc, target_weight, alpha, want_grads=True, grad_scale=1.0,
             grads_out=None, losses_out=None, pose_topk=0, kd_topk=0, pose_temperature=0, kd_temperature=0,
             kd_weight=None):
    """Fused FPD loss. outs_nhwc: list of [B,h,w,J]; returns (losses[3] device tensor, grads list or None).
    pose_topk / kd_topk > 0 make that term JointsOHKMMSELoss(topk) instead of JointsMSELoss (fpd_loss_ohkm_fused);
    pose_temperature / kd_temperature > 0 make it JointsKLDLoss(temperature) (fpd_loss_kl_fused, which takes any mix
    of the three kinds). A term cannot have both a topk and a temperature.
    kd_weight [B,J] (e.g. kd_weights(...)) weights the kd term in place of target_weight (fpd_loss_kdw_fused, which
    runs the same kernels); None is target_weight."""
    pose_temperature = _check_temperature(pose_temperature, "pose_temperature", True)
    kd_temperature = _check_temperature(kd_temperature, "kd_temperature", True)
    if (pose_topk and pose_temperature) or (kd_topk and kd_temperature):
        raise ValueError("a loss term is JointsOHKMMSELoss (topk) or JointsKLDLoss (temperature), not both")
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
    if kd_weight is not None:
        if teacher_nhwc is None:
            raise ValueError("fpd_loss: kd_weight without a teacher")
        pose_topk = _check_topk(pose_topk, J, 0, "pose_topk")
        kd_topk = _check_topk(kd_topk, J, 0, "kd_topk")
        kdw = kd_weight.reshape(B, J).contiguous()
        for t in list(outs_nhwc) + [target_nchw, teacher_nhwc, tw, kdw]:
            _chk(t, "fpd_loss argument")
        if pose_temperature or kd_temperature:
            nbytes = N.lib().fpd_loss_kl_workspace_bytes(S, B, J, h, w)
        elif pose_topk or kd_topk:
            nbytes = N.lib().fpd_loss_ohkm_workspace_bytes(S, B, J, h, w)
        else:
            nbytes = N.lib().fpd_loss_workspace_bytes(B, J, h, w)
        ws = _ws.get(nbytes, dev)
        N.check(N.lib().fpd_loss_kdw_fused(outs_arr, S, _p(target_nchw), _p(teacher_nhwc), _p(tw), _p(kdw),
                                           float(alpha), grads_arr, float(grad_scale), _p(losses), B, J, h, w,
                                           pose_topk, kd_topk, pose_temperature, kd_temperature, _p(ws), ws.numel(),
                                           _stream()), "loss_kdw_fused")
        return losses, grads
    if pose_temperature or kd_temperature:
        pose_topk = _check_topk(pose_topk, J, 0, "pose_topk")
        kd_topk = _check_topk(kd_topk, J, 0, "kd_topk")
        for t in list(outs_nhwc) + [target_nchw, teacher_nhwc, tw]:
            _chk(t, "fpd_loss argument")
        ws = _ws.get(N.lib().fpd_loss_kl_workspace_bytes(S, B, J, h, w), dev)
        N.check(N.lib().fpd_loss_kl_fused(outs_arr, S, _p(target_nchw), _p(teacher_nhwc), _p(tw), float(alpha),
                                          grads_arr, float(grad_scale), _p(losses), B, J, h, w, pose_topk, kd_topk,
                                          pose_temperature, kd_temperature, _p(ws), ws.numel(), _stream()),
                "loss_kl_fused")
        return losses, grads
    if pose_topk or kd_topk:
        pose_topk = _check_topk(pose_topk, J, 0, "pose_topk")
        kd_topk = _check_topk(kd_topk, J, 0, "kd_topk")
        for t in list(outs_nhwc) + [target_nchw, teacher_nhwc, tw]:
            _chk(t, "fpd_loss argument")
        ws = _ws.get(N.lib().fpd_loss_ohkm_workspace_bytes(S, B, J, h, w), dev)
        N.check(N.lib().fpd_loss_ohkm_fused(outs_arr, S, _p(target_nchw), _p(teacher_nhwc), _p(tw), float(alpha),
                                            grads_arr, float(grad_scale), _p(losses), B, J, h, w, pose_topk, kd_topk,
                                            _p(ws), ws.numel(), _stream()), "loss_ohkm_fused")
        return losses, grads
    ws = _ws.get(N.lib().fpd_loss_workspace_bytes(B, J, h, w), dev)
    N.check(N.lib().fpd_loss_fused(outs_arr, S, _p(target_nchw), _p(teacher_nhwc), _p(tw), float(alpha), grads_arr,
                                   float(grad_scale), _p(losses), B, J, h, w, _p(ws), ws.numel(), _stream()),
            "loss_fused")
    return losses, grads


def check_feature_weight(weight):
    """The feature distillation weight: a finite number >= 0 (0: off)."""
    if isinstance(weight, bool) or not isinstance(weight, numbers.Real) or not (math.isfinite(weight) and weight >= 0):
        raise ValueError("feature_weight=%r must be a finite number >= 0 (0: off)" % (weight,))
    return float(weight)


def feature_mse(student_nhwc, teacher_nhwc, weight, grad_out=None, loss_out=None, losses=None):
    """Feature distillation loss (a FitNets hint) and its gradient: L_feat = mean((student - teacher)^2) over all
    elements, grad = (2 * weight / n) * (student - teacher). student_nhwc: the adapted student head feature (fp32);
    teacher_nhwc: the teacher's head feature of the same shape, fp32 or fp16 (read as stored, no conversion launch).
    losses: an FPD losses[3] buffer, whose total losses[2] gains weight * L_feat. Returns (L_feat [1] device, grad)."""
    weight = check_feature_weight(weight)
    _chk(student_nhwc, "student feature")
    if not (teacher_nhwc.is_cuda and teacher_nhwc.dtype in (torch.float32, torch.float16) and teacher_nhwc.is_contiguous()):
        raise ValueError("teacher feature must be a contiguous fp32 or fp16 CUDA tensor (got %s %s %s)" % (
            teacher_nhwc.device, teacher_nhwc.dtype, teacher_nhwc.is_contiguous()))
    if tuple(student_nhwc.shape) != tuple(teacher_nhwc.shape):
        raise ValueError("feature_mse: student feature %s and teacher feature %s differ in shape" % (
            tuple(student_nhwc.shape), tuple(teacher_nhwc.shape)))
    n = student_nhwc.numel()
    if n == 0:
        raise ValueError("feature_mse: empty feature")
    dev = student_nhwc.device
    grad = grad_out if grad_out is not None else torch.empty_like(student_nhwc)
    loss = loss_out if loss_out is not None else torch.empty(1, dtype=torch.float32, device=dev)
    for t, name in ((grad, "grad_out"), (loss, "loss_out"), (losses, "losses")):
        _chk(t, name)
    ws = _ws.get(N.lib().fpd_feature_mse_workspace_bytes(n), dev)
    N.check(N.lib().fpd_feature_mse(_p(student_nhwc), _p(teacher_nhwc), int(teacher_nhwc.dtype == torch.float16), weight,
                                    _p(grad), _p(loss), _p(losses), n, _p(ws), ws.numel(), _stream()), "feature_mse")
    return loss, grad


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


def joints_ohkm_mse(out_nchw, target_nchw, target_weight=None, topk=8, want_grad=True):
    """JointsOHKMMSELoss (lib/core/loss.py:42-87) on NCHW tensors: per sample the mean of the topk largest per-joint
    losses, averaged over the batch. Returns (loss3 device tensor, loss3[0] the value; grad [B,J,h,w] or None)."""
    _chk(out_nchw, "out")
    _chk(target_nchw, "target")
    if out_nchw.dim() < 3 or out_nchw.shape[0] * out_nchw.shape[1] == 0 or target_nchw.shape != out_nchw.shape:
        raise ValueError("out / target must be non-empty [B,J,...] tensors of one shape (got %s, %s)"
                         % (tuple(out_nchw.shape), tuple(target_nchw.shape)))
    B, J = out_nchw.shape[:2]
    topk = _check_topk(topk, J, 1, "topk")
    hw = out_nchw.numel() // (B * J)
    dev = out_nchw.device
    loss3 = torch.empty(3, dtype=torch.float32, device=dev)
    grad = torch.empty_like(out_nchw) if want_grad else None
    tw = None if target_weight is None else target_weight.reshape(B, J).contiguous()
    _chk(tw, "target_weight")
    ws = _ws.get(N.lib().fpd_joints_ohkm_workspace_bytes(B, J), dev)
    N.check(N.lib().fpd_joints_ohkm(_p(out_nchw), _p(target_nchw), _p(tw), topk, _p(loss3), _p(grad), B, J, hw, _p(ws),
                                    ws.numel(), _stream()), "joints_ohkm")
    return loss3, grad


def joints_kld(out_nchw, ref_nchw, target_weight=None, temperature=1.0, want_grad=True):
    """JointsKLDLoss on NCHW tensors: T^2/(B*J) * sum_{b,j} w[b,j] * KL(softmax(ref[b,j]/T) || softmax(out[b,j]/T)),
    each map a distribution over its pixels; any h*w, J <= 64. Returns (loss3 device tensor, loss3[0] the value;
    grad [B,J,h,w] or None)."""
    temperature = _check_temperature(temperature, "temperature", False)
    _chk(out_nchw, "out")
    _chk(ref_nchw, "ref")
    if out_nchw.dim() < 3 or out_nchw.shape[0] * out_nchw.shape[1] == 0 or ref_nchw.shape != out_nchw.shape:
        raise ValueError("out / ref must be non-empty [B,J,...] tensors of one shape (got %s, %s)"
                         % (tuple(out_nchw.shape), tuple(ref_nchw.shape)))
    B, J = out_nchw.shape[:2]
    hw = out_nchw.numel() // (B * J)
    dev = out_nchw.device
    loss3 = torch.empty(3, dtype=torch.float32, device=dev)
    grad = torch.empty_like(out_nchw) if want_grad else None
    tw = None if target_weight is None else target_weight.reshape(B, J).contiguous()
    _chk(tw, "target_weight")
    ws = _ws.get(N.lib().fpd_joints_kld_workspace_bytes(B, J, hw), dev)
    N.check(N.lib().fpd_joints_kld(_p(out_nchw), _p(ref_nchw), _p(tw), temperature, _p(loss3), _p(grad), B, J, hw,
                                   _p(ws), ws.numel(), _stream()), "joints_kld")
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


def resample_heatmaps(hm_nhwc, out_hw, udp=False, out=None):
    """A teacher's heat-maps [B,Hi,Wi,C] (fp32 NHWC, C <= 64) on the heat-map grid out_hw = (h, w) of another crop of the
    same box (fpd_heatmap_resample): bilinear at (u * Wi / Wo, v * Hi / Ho) for the reference's crops, at
    (u * (Wi-1) / (Wo-1), v * (Hi-1) / (Ho-1)) for UDP crops (udp=True), clamped to the map. Returns [B,h,w,C]."""
    _chk(hm_nhwc, "hm_nhwc")
    if hm_nhwc.dim() != 4:
        raise ValueError("resample_heatmaps: hm_nhwc must be [B, H, W, C], got %s" % (tuple(hm_nhwc.shape),))
    B, Hi, Wi, C = hm_nhwc.shape
    Ho, Wo = int(out_hw[0]), int(out_hw[1])
    if min(Hi, Wi, Ho, Wo) < 1 or not 1 <= C <= 64:
        raise ValueError("resample_heatmaps: sizes must be positive and C <= 64 (got [%d,%d,%d,%d] -> %dx%d)"
                         % (B, Hi, Wi, C, Ho, Wo))
    if out is None:
        out = torch.empty((B, Ho, Wo, C), dtype=torch.float32, device=hm_nhwc.device)
    else:
        _chk(out, "out")
        if tuple(out.shape) != (B, Ho, Wo, C):
            raise ValueError("resample_heatmaps: out must be %s" % ((B, Ho, Wo, C),))
    N.check(N.lib().fpd_heatmap_resample(_p(hm_nhwc), _p(out), B, Hi, Wi, Ho, Wo, C, int(bool(udp)), _stream()),
            "heatmap_resample")
    return out


def argmax_nchw(hm):
    B, J = hm.shape[:2]
    hw = hm.numel() // (B * J)
    idx = torch.empty((B, J), dtype=torch.int32, device=hm.device)
    maxval = torch.empty((B, J), dtype=torch.float32, device=hm.device)
    N.check(N.lib().fpd_argmax_nchw(_p(hm), _p(idx), _p(maxval), B * J, hw, _stream()), "argmax_nchw")
    return idx, maxval


def final_preds(avg_nhwc, idx, maxval, inv, post_process, out=None):
    """get_final_preds on the device (csrc/decode.cu). avg_nhwc: [B,h,w,J] merged heat-maps; idx int32 / maxval [B,J]
    from flip_merge_argmax; inv: CUDA float64 [B,6] heat-map -> image matrices (lib.core.inference.inverse_affines).
    Returns preds [B,J,3] = (x, y, maxval) in image coordinates."""
    _chk(avg_nhwc, "avg_nhwc")
    B, h, w, J = avg_nhwc.shape
    if not (inv.is_cuda and inv.dtype == torch.float64 and inv.is_contiguous() and tuple(inv.shape) == (B, 6)):
        raise ValueError("inv must be a contiguous float64 CUDA tensor of shape (%d, 6)" % B)
    preds = out if out is not None else torch.empty((B, J, 3), dtype=torch.float32, device=avg_nhwc.device)
    N.check(N.lib().fpd_final_preds(_p(avg_nhwc), _p(idx), _p(maxval), _p(inv), int(bool(post_process)), _p(preds), B, J,
                                    h, w, _stream()), "final_preds")
    return preds


def final_preds_dark(avg_nhwc, idx, maxval, inv, blur_kernel=11, out=None):
    """final_preds with DARK's sub-pixel decode (csrc/decode.cu) in place of the quarter-pixel nudge: a Taylor step on
    the log of the map blurred by a blur_kernel-tap Gaussian (odd, 3..15). Same arguments otherwise; returns preds
    [B,J,3] = (x, y, maxval) in image coordinates."""
    _chk(avg_nhwc, "avg_nhwc")
    B, h, w, J = avg_nhwc.shape
    if not (inv.is_cuda and inv.dtype == torch.float64 and inv.is_contiguous() and tuple(inv.shape) == (B, 6)):
        raise ValueError("inv must be a contiguous float64 CUDA tensor of shape (%d, 6)" % B)
    preds = out if out is not None else torch.empty((B, J, 3), dtype=torch.float32, device=avg_nhwc.device)
    N.check(N.lib().fpd_final_preds_dark(_p(avg_nhwc), _p(idx), _p(maxval), _p(inv), int(blur_kernel), _p(preds), B, J,
                                         h, w, _stream()), "final_preds_dark")
    return preds


def pck_counts(idx, maxval, target_nchw, want_pred_hm=False, out=None):
    """accuracy() counts on the device (csrc/decode.cu): int32 [J,2] = {valid, hit} per joint, plus the prediction in
    heat-map coordinates [B,J,2] when want_pred_hm (else None). lib.core.evaluate.pck_from_counts turns the counts into
    accuracy()'s (acc, avg_acc, cnt)."""
    _chk(target_nchw, "target")
    B, J, h, w = target_nchw.shape
    counts = out if out is not None else torch.empty((J, 2), dtype=torch.int32, device=target_nchw.device)
    pred_hm = torch.empty((B, J, 2), dtype=torch.float32, device=target_nchw.device) if want_pred_hm else None
    N.check(N.lib().fpd_pck_counts(_p(idx), _p(maxval), _p(target_nchw), _p(counts), _p(pred_hm), B, J, h, w, _stream()),
            "pck_counts")
    return counts, pred_hm


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


def gaussian_table(sigma, device):
    """The un-normalised Gaussian patch gaussian_targets stamps, as a device tensor [(6 sigma + 1)^2]."""
    import numpy as np
    # the reference's own expression (float32 numpy), so the stamped patch is bit-identical: JointsDataset.py:266-272
    size = 2 * (sigma * 3) + 1
    xs = np.arange(0, size, 1, np.float32)
    ys = xs[:, np.newaxis]
    x0 = y0 = size // 2
    g = np.exp(- ((xs - x0) ** 2 + (ys - y0) ** 2) / (2 * sigma ** 2))
    return torch.from_numpy(np.ascontiguousarray(g, dtype=np.float32)).to(device)


def gaussian_targets(joints, joints_vis, heatmap_size, image_size, sigma=2, joints_weight=None, gauss_table=None):
    """Batch form of JointsDataset.generate_target (lib/dataset/JointsDataset.py:233-289). joints / joints_vis: CUDA float32
    [N,J,3]; heatmap_size / image_size: (w, h). Returns (target [N,J,h,w], target_weight [N,J,1])."""
    _chk(joints, "joints")
    _chk(joints_vis, "joints_vis")
    n, J = joints.shape[0], joints.shape[1]
    W, H = int(heatmap_size[0]), int(heatmap_size[1])
    dev = joints.device
    if gauss_table is None:
        gauss_table = gaussian_table(sigma, dev)
    target = torch.empty((n, J, H, W), dtype=torch.float32, device=dev)
    tw = torch.empty((n, J, 1), dtype=torch.float32, device=dev)
    jw = None if joints_weight is None else joints_weight.to(dev).float().contiguous().reshape(-1)
    N.check(N.lib().fpd_gaussian_targets(_p(joints), _p(joints_vis), _p(jw), _p(gauss_table), _p(target), _p(tw), n, J, H, W,
                                         int(image_size[0]), int(image_size[1]), int(sigma), _stream()), "gaussian_targets")
    return target, tw


def _sub_pixel_targets(name, joints, joints_vis, heatmap_size, image_size, sigma, joints_weight):
    """Calls fpd_<name>, a target entry point with gaussian_targets' arguments less the table."""
    _chk(joints, "joints")
    _chk(joints_vis, "joints_vis")
    n, J = joints.shape[0], joints.shape[1]
    W, H = int(heatmap_size[0]), int(heatmap_size[1])
    dev = joints.device
    target = torch.empty((n, J, H, W), dtype=torch.float32, device=dev)
    tw = torch.empty((n, J, 1), dtype=torch.float32, device=dev)
    jw = None if joints_weight is None else joints_weight.to(dev).float().contiguous().reshape(-1)
    N.check(getattr(N.lib(), "fpd_" + name)(_p(joints), _p(joints_vis), _p(jw), _p(target), _p(tw), n, J, H, W,
                                            int(image_size[0]), int(image_size[1]), int(sigma), _stream()), name)
    return target, tw


def gaussian_targets_unbiased(joints, joints_vis, heatmap_size, image_size, sigma=2, joints_weight=None):
    """gaussian_targets with DARK's unbiased encoding: the Gaussian on the sub-pixel joint joint * heatmap_size /
    image_size rather than on the rounded one, over the whole map. Same arguments (no table) and results."""
    return _sub_pixel_targets("gaussian_targets_unbiased", joints, joints_vis, heatmap_size, image_size, sigma,
                              joints_weight)


def gaussian_targets_udp(joints, joints_vis, heatmap_size, image_size, sigma=2, joints_weight=None):
    """gaussian_targets with UDP's encoding (Huang et al., CVPR 2020), for joints cropped by augment.udp_crop_matrix:
    stride (image_size - 1) / (heatmap_size - 1), the Gaussian on the unrounded centre joint / stride, within the
    default 3 sigma window around the rounded one. Same arguments (no table) and results."""
    return _sub_pixel_targets("gaussian_targets_udp", joints, joints_vis, heatmap_size, image_size, sigma,
                              joints_weight)


CROP_DESC_LEN = 7   # desc columns: byte offset, region x, y, w, h, image w, h (include/fpd_b200.h)


def crop_affine_normalize(src, desc, inv, out_size, mean, std, desc_host=None, inv_host=None, out=None):
    """Batched cv2.warpAffine(INTER_LINEAR, BORDER_CONSTANT=0) + ToTensor + Normalize, bit-exact (fpd_crop_affine_normalize).
    src: CUDA uint8 buffer of packed HWC regions; desc: CUDA int64 [N,7]; inv: CUDA float64 [N,6] (or [N,2,3]) inverse
    matrices; out_size: (w, h); mean / std: 3 values each. desc_host / inv_host: CPU copies of desc / inv (the arguments
    are validated on the host; when omitted they are copied back, which synchronises). Returns out fp32 [N,3,h,w]."""
    import numpy as np
    W, H = int(out_size[0]), int(out_size[1])
    if not (src.is_cuda and src.dtype == torch.uint8 and src.is_contiguous()):
        raise ValueError("src must be a contiguous uint8 CUDA tensor")
    if not (desc.is_cuda and desc.dtype == torch.int64 and desc.is_contiguous() and desc.dim() == 2
            and desc.shape[1] == CROP_DESC_LEN):
        raise ValueError("desc must be a contiguous int64 CUDA tensor [N, %d]" % CROP_DESC_LEN)
    n = desc.shape[0]
    if not (inv.is_cuda and inv.dtype == torch.float64 and inv.is_contiguous() and inv.numel() == 6 * n):
        raise ValueError("inv must be a contiguous float64 CUDA tensor [N, 6]")
    desc_host = (desc if desc_host is None else desc_host).cpu().contiguous()
    inv_host = (inv if inv_host is None else inv_host).cpu().contiguous()
    if desc_host.dtype != torch.int64 or desc_host.shape != desc.shape or inv_host.dtype != torch.float64 \
            or inv_host.numel() != inv.numel():
        raise ValueError("desc_host / inv_host must match desc / inv")
    ms = np.ascontiguousarray(np.concatenate([np.asarray(mean, np.float32).reshape(3),
                                              np.asarray(std, np.float32).reshape(3)]))
    if out is None:
        out = torch.empty((n, 3, max(H, 0), max(W, 0)), dtype=torch.float32, device=src.device)
    else:
        _chk(out, "out")
        if tuple(out.shape) != (n, 3, H, W):
            raise ValueError("out must be [N, 3, h, w] = %s" % ((n, 3, H, W),))
    N.check(N.lib().fpd_crop_affine_normalize(_p(src) if src.numel() else None, src.numel(), _p(desc), _p(inv),
                                              _p(desc_host), _p(inv_host), ms.ctypes.data_as(ctypes.c_void_p), _p(out), n,
                                              H, W, _stream()), "crop_affine_normalize")
    return out
