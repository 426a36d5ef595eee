"""GPU parity of every C-ABI op against a plain PyTorch fp32 composition of the same op
(TF32 disabled in the torch reference). The network-level parity against the reference model lives in
test_hourglass_gpu.py; this file pins each kernel in isolation."""
import numpy as np
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def ops():
    from fpd_b200 import ops as o
    return o


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous()


def nchw(x_nhwc):
    return x_nhwc.permute(0, 3, 1, 2).contiguous()


CONV_TC_SHAPES = [
    # B, H, W, Cin, Cout, k
    (2, 64, 64, 64, 64, 3),
    (2, 64, 64, 128, 64, 1),
    (2, 64, 64, 64, 128, 1),
    (4, 32, 32, 64, 64, 3),
    (4, 16, 16, 64, 64, 3),
    (8, 8, 8, 64, 64, 3),
    (8, 4, 4, 64, 64, 3),
    (2, 4, 4, 64, 64, 3),      # batch smaller than the pixel-tile's image count
    (3, 8, 8, 128, 64, 1),     # ragged last tile
    (2, 128, 128, 32, 32, 3),
    (2, 64, 64, 128, 16, 1),   # score conv
    (2, 64, 64, 128, 128, 1),
    (1, 64, 64, 128, 256, 1),
    (1, 64, 64, 256, 256, 1),  # teacher fc
    (1, 32, 32, 128, 128, 3),  # teacher 3x3
    (2, 64, 48, 32, 32, 3),    # HRNet resolution (W not a power of two)
    (2, 16, 12, 128, 128, 3),
    (2, 64, 64, 16, 128, 1),   # score_ conv: 16 input channels, k-block completed by TMA zero fill
    (2, 32, 24, 48, 96, 3),    # HRNet-w48 widths
    (2, 16, 12, 96, 48, 1),
]
# shapes only the sliced TS kernel takes (Cout > 256): HRNet-w48's 384-channel branch
CONV_TS_WIDE_SHAPES = [(2, 8, 6, 384, 384, 3), (2, 8, 6, 192, 384, 1), (1, 16, 16, 64, 512, 1)]


@pytest.mark.parametrize("shape", CONV_TC_SHAPES)
@pytest.mark.parametrize("passes", [3, 1])
def test_conv2d_tc_fused_bn_relu(shape, passes):
    """3xTF32 / TF32 entry point (conv2d_tc_fused, csrc/conv_wgmma.cu): conv(relu(bn_affine(x))) with the operand
    transform inside the kernel vs torch fp32."""
    B, H, W, Cin, Cout, k = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(4321)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g) * 2 + 0.5
    mean = torch.randn(Cin, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.5
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (1.0 / (Cin * k * k) ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B, Cout, H, W, device="cuda", generator=g)
    a = F.relu((x - mean.view(1, -1, 1, 1)) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    ref = F.conv2d(a, w, bias, padding=k // 2) + res
    w_hi, w_lo = o.weight_prep(w, split=(passes == 3))
    y = o.conv2d_tc_fused(nhwc(x), w_hi, w_lo, k, mean=mean, scale=scale, shift=shift, relu=True, bias=bias,
                          residual=nhwc(res))
    # identity pre-op (raw operand, e.g. dgrad on dY)
    y2 = o.conv2d_tc_fused(nhwc(x), w_hi, w_lo, k)
    ref2 = F.conv2d(x, w, None, padding=k // 2)
    torch.cuda.synchronize()
    tol = 2e-5 if passes == 3 else 3e-3
    assert relerr(nchw(y), ref) < tol, "fused %s passes=%d rel err %.3e" % (shape, passes, relerr(nchw(y), ref))
    assert relerr(nchw(y2), ref2) < tol


@pytest.mark.parametrize("shape", CONV_TS_WIDE_SHAPES)
def test_conv2d_tc_ts_wide_output_slices(shape):
    B, H, W, Cin, Cout, k = shape
    o = ops()
    assert o.N.lib().fpd_conv2d_tc_ts_supported(Cin, Cout, k) == 1
    g = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (1.0 / (Cin * k * k) ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B, Cout, H, W, device="cuda", generator=g)
    ref = F.conv2d(F.relu(x), w, bias, padding=k // 2) + res
    w_hi, w_lo = o.weight_prep(w)
    y = o.conv2d_tc_fused(nhwc(x), w_hi, w_lo, k, relu=True, bias=bias, residual=nhwc(res))
    torch.cuda.synchronize()
    assert relerr(nchw(y), ref) < 2e-5


@pytest.mark.parametrize("shape", CONV_TC_SHAPES + CONV_TS_WIDE_SHAPES + [(2, 64, 64, 160, 32, 1), (5, 16, 16, 256, 128, 3)])
@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("f16", [False, True])
def test_conv2d_tc_h(shape, passes, f16):
    """Generation-5 kernel (halo reuse; 3xFP16 or 3xTF32 operands) vs torch fp32: conv(relu(bn_affine(x))) + bias +
    residual, and the identity pre-op form used for dgrad."""
    B, H, W, Cin, Cout, k = shape
    o = ops()
    if not o.N.lib().fpd_conv2d_tc_h_supported(Cin, Cout, k, H, W, int(f16)):
        pytest.skip("shape not taken by conv_tc_h (f16=%s)" % f16)
    g = torch.Generator(device="cuda").manual_seed(4321)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g) * 2 + 0.5
    mean = torch.randn(Cin, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.5
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (1.0 / (Cin * k * k) ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B, Cout, H, W, device="cuda", generator=g)
    a = F.relu((x - mean.view(1, -1, 1, 1)) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    ref = F.conv2d(a, w, bias, padding=k // 2) + res
    prep = o.weight_prep_f16 if f16 else o.weight_prep
    w_hi, w_lo = prep(w, split=(passes == 3))
    y = o.conv2d_tc_h(nhwc(x), w_hi, w_lo, k, mean=mean, scale=scale, shift=shift, relu=True, bias=bias,
                      residual=nhwc(res))
    y2 = o.conv2d_tc_h(nhwc(x), w_hi, w_lo, k)
    ref2 = F.conv2d(x, w, None, padding=k // 2)
    torch.cuda.synchronize()
    tol = 3e-5 if passes == 3 else 3e-3   # K up to 3456: the fp32 torch reference itself carries ~1e-5
    assert relerr(nchw(y), ref) < tol, "conv_tc_h %s passes=%d f16=%s rel err %.3e" % (shape, passes, f16,
                                                                                        relerr(nchw(y), ref))
    assert relerr(nchw(y2), ref2) < tol


def test_conv2d_tc_h_f16_small_and_large_magnitudes():
    """3xFP16 keeps fp32-grade accuracy away from the fp16 range limits: activations of magnitude 1e-2 .. 1e3."""
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(99)
    for mag in (1e-2, 1.0, 1e3):
        x = torch.randn(2, 64, 32, 32, device="cuda", generator=g) * mag
        w = torch.randn(64, 64, 3, 3, device="cuda", generator=g) * (1.0 / 24.0)
        ref = F.conv2d(F.relu(x), w, None, padding=1)
        w_hi, w_lo = o.weight_prep_f16(w)
        y = o.conv2d_tc_h(nhwc(x), w_hi, w_lo, 3, relu=True)
        torch.cuda.synchronize()
        assert relerr(nchw(y), ref) < (2e-4 if mag < 0.1 else 2e-5), "mag %g: %.3e" % (mag, relerr(nchw(y), ref))


@pytest.mark.parametrize("mag", [1e-7, 3e-5, 1.0, 1e4])
def test_conv2d_tc_h_f16_dgrad_with_amax_scale(mag):
    """3xFP16 data gradient: dY of any magnitude is brought into the fp16 range by the power-of-two scale that the bias-
    gradient reduction returns (max|dY| * S in [2^14, 2^15)); a wide in-tensor dynamic range must not hurt either."""
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(11)
    dy = torch.randn(2, 32, 32, 64, device="cuda", generator=g) * mag
    dy[0, :4] *= 1e-4    # a region four orders of magnitude below the maximum
    w = torch.randn(64, 64, 3, 3, device="cuda", generator=g) * (1.0 / 24.0)
    ref = torch.nn.grad.conv2d_input((2, 64, 32, 32), w, nchw(dy), padding=1)
    bias_grad, scale = o.channel_sum(dy, want_amax=True)
    w_hi, w_lo = o.weight_prep_f16(w, for_dgrad=True)
    da = o.conv2d_tc_h(dy, w_hi, w_lo, 3, in_scale=scale)
    torch.cuda.synchronize()
    assert relerr(nchw(da), ref) < 2e-5, "mag %g: %.3e" % (mag, relerr(nchw(da), ref))
    assert relerr(bias_grad, nchw(dy).sum(dim=(0, 2, 3))) < 1e-5


@pytest.mark.parametrize("shape", [(2, 64, 64, 64, 64, 3), (2, 32, 32, 128, 64, 1), (4, 8, 8, 64, 128, 1)])
def test_conv2d_tc_dgrad_with_relu_mask(shape):
    B, H, W, Cin, Cout, k = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g, requires_grad=True)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * 0.05
    a = F.relu(x)
    y = F.conv2d(a, w, None, padding=k // 2)
    dy = torch.randn_like(y)
    (dx_ref,) = torch.autograd.grad(y, x, dy)
    wd_hi, wd_lo = o.weight_prep(w, for_dgrad=True)
    mask = nhwc(a.detach())
    dx = o.conv2d_tc_fused(nhwc(dy), wd_hi, wd_lo, k, relu_mask=mask)
    torch.cuda.synchronize()
    assert relerr(nchw(dx), dx_ref) < 2e-5


WGRAD_TC_SHAPES = [
    # B, H, W, Cin, Cout, k
    (2, 64, 64, 64, 64, 3),     # student conv2 (tap pairs stacked on M)
    (2, 64, 64, 128, 64, 1),    # student conv1
    (2, 64, 64, 64, 128, 1),    # student conv3 (dY side on M)
    (2, 64, 64, 128, 128, 1),   # fc / fc_
    (4, 16, 16, 64, 64, 3),
    (8, 4, 4, 64, 64, 3),
    (3, 8, 8, 128, 64, 1),      # ragged batch tile
    (2, 128, 128, 32, 32, 3),   # layer1 conv2 (4 taps stacked)
    (1, 32, 32, 128, 128, 3),
    (2, 64, 48, 32, 32, 3),     # HRNet branch 0 (wgrad_tc3 pair mode: two taps per M = 64 MMA)
    (2, 64, 48, 32, 64, 3),     # HRNet fuse down path in stride-1 form
    (4, 32, 24, 32, 96, 3),
    (2, 32, 32, 128, 256, 1),
    (2, 64, 64, 128, 16, 1),    # score conv (dY has 16 channels: M tile completed by TMA zero fill)
    (2, 64, 64, 16, 128, 1),    # score_ conv
    (2, 128, 128, 32, 64, 1),   # layer1 conv3 / downsample
    (2, 128, 128, 32, 32, 1),
    (2, 32, 24, 64, 64, 1),
]


@pytest.mark.parametrize("shape", WGRAD_TC_SHAPES)
@pytest.mark.parametrize("passes", [3, 1])
def test_conv2d_wgrad_tc_fused_bn_relu(shape, passes):
    """dW of conv(relu(bn_affine(x))) from raw x / raw dy with the operand transform inside the kernel."""
    B, H, W, Cin, Cout, k = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(99)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g) * 2 + 0.5
    mean = torch.randn(Cin, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.5
    a = F.relu((x - mean.view(1, -1, 1, 1)) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    dy = torch.randn(B, Cout, H, W, device="cuda", generator=g)
    # fp64 references: an fp32 library weight gradient over 32k pixels is itself ~2e-5 off the exact sum, as far off as the
    # tolerance (2, 128, 128, 32, 32, 3)
    w = torch.zeros(Cout, Cin, k, k, device="cuda", dtype=torch.float64, requires_grad=True)
    (dw_ref,) = torch.autograd.grad(F.conv2d(a.double(), w, None, padding=k // 2), w, dy.double())
    dw = o.conv2d_wgrad_tc_fused(nhwc(x), nhwc(dy), k, mean=mean, scale=scale, shift=shift, relu=True, passes=passes)
    w2 = torch.zeros(Cout, Cin, k, k, device="cuda", dtype=torch.float64, requires_grad=True)
    (dw_ref2,) = torch.autograd.grad(F.conv2d(x.double(), w2, None, padding=k // 2), w2, dy.double())
    dw2 = o.conv2d_wgrad_tc_fused(nhwc(x), nhwc(dy), k, passes=passes)
    torch.cuda.synchronize()
    tol = 2e-5 if passes == 3 else 3e-3
    assert relerr(dw, dw_ref) < tol, "wgrad fused %s passes=%d rel err %.3e" % (shape, passes, relerr(dw, dw_ref))
    assert relerr(dw2, dw_ref2) < tol


@pytest.mark.parametrize("cfg", [
    # B, H, W, Cin, Cout, k, stride, pad
    (2, 64, 64, 3, 32, 7, 2, 3),
    (2, 16, 16, 16, 128, 1, 1, 0),
    (2, 16, 16, 128, 16, 1, 1, 0),
    (2, 12, 10, 8, 12, 3, 2, 1),
    (1, 9, 9, 5, 7, 3, 1, 1),
])
def test_conv2d_simt(cfg):
    B, H, W, Cin, Cout, k, stride, pad = cfg
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g, requires_grad=True)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g, requires_grad=True)
    bias = torch.randn(Cout, device="cuda", generator=g)
    y_ref = F.conv2d(x, w, bias, stride=stride, padding=pad)
    dy = torch.randn_like(y_ref)
    dx_ref, dw_ref = torch.autograd.grad(y_ref, (x, w), dy)
    y = o.conv2d_simt_fwd(nhwc(x.detach()), w.detach(), bias=bias, stride=stride, pad=pad)
    dx = o.conv2d_simt_dgrad(nhwc(dy), w.detach(), (H, W), stride=stride, pad=pad)
    dw = o.conv2d_simt_wgrad(nhwc(x.detach()), nhwc(dy), k, stride=stride, pad=pad)
    torch.cuda.synchronize()
    assert relerr(nchw(y), y_ref) < 1e-5
    assert relerr(nchw(dx), dx_ref) < 1e-5
    assert relerr(dw, dw_ref) < 1e-4


@pytest.mark.parametrize("shape", [(4, 64, 64, 128), (32, 4, 4, 64), (3, 16, 12, 48), (2, 128, 128, 32), (2, 8, 8, 256)])
def test_bn_train_forward_backward(shape):
    B, H, W, C = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(11)
    # large common-mode offset: the cancellation-prone case for E[x^2]-E[x]^2
    x = (torch.randn(B, C, H, W, device="cuda", generator=g) * 0.3 + 25.0).requires_grad_(True)
    gamma = (torch.rand(C, device="cuda", generator=g) + 0.5).requires_grad_(True)
    beta = torch.randn(C, device="cuda", generator=g).requires_grad_(True)
    rm = torch.zeros(C, device="cuda"); rv = torch.ones(C, device="cuda")
    rm2 = rm.clone(); rv2 = rv.clone()
    z_ref = F.batch_norm(x, rm, rv, gamma, beta, True, 0.1, 1e-5)
    y_ref = F.relu(z_ref)
    # no upstream gradient where the pre-activation is within round-off of the ReLU kink (the two
    # implementations may legitimately disagree on the sign there)
    dy = torch.randn_like(y_ref) * (z_ref.detach().abs() > 1e-4)
    dx_ref, dg_ref, db_ref = torch.autograd.grad(y_ref, (x, gamma, beta), dy)

    xh = nhwc(x.detach())
    mean, var = o.bn_stats(xh)
    scale, shift, invstd = o.bn_finalize(mean, var, gamma.detach(), beta.detach(), 1e-5, B * H * W, rm2, rv2, 0.1)
    a_hi, a_lo = o.affine_act_split(xh, scale, shift, relu=True, mean=mean)
    dx, dgamma, dbeta = o.bn_bwd(nhwc(dy), xh, mean, invstd, scale, shift, gamma.detach(), True)
    # the apply pass that also reduces its own output: identical dx, its per-channel sum, and the same power-of-two operand
    # scale channel_sum(dx, want_amax=True) derives
    o.BN_APPLY_SUM = True
    dx2, dgamma2, dbeta2, dsum = o.bn_bwd(nhwc(dy), xh, mean, invstd, scale, shift, gamma.detach(), True, want_dx_sum=True)
    o.BN_APPLY_SUM = os.environ.get("FPD_BN_APPLY_SUM", "0") != "0"
    assert dsum is not None and torch.equal(dx2, dx) and torch.equal(dgamma2, dgamma) and torch.equal(dbeta2, dbeta)
    ref_sum, ref_scale = o.channel_sum(dx, want_amax=True)
    # sum of dx over the batch is ~0 by construction (BatchNorm removes the mean): compare on the scale of sum |dx|
    assert ((dsum[0].double() - dx.double().sum((0, 1, 2))).abs().max() / dx.double().abs().sum((0, 1, 2)).max()).item() < 1e-6
    assert torch.equal(dsum[1], ref_scale)
    torch.cuda.synchronize()
    xd = x.detach().double()
    assert relerr(mean, xd.mean((0, 2, 3)).float()) < 1e-6
    assert relerr(var, xd.var((0, 2, 3), unbiased=False).float()) < 1e-5
    assert relerr(rm2, rm) < 1e-6 and relerr(rv2, rv) < 1e-5
    assert relerr(nchw(a_hi + a_lo), y_ref) < 1e-5
    assert relerr(nchw(dx), dx_ref) < 1e-4
    assert relerr(dgamma, dg_ref) < 1e-4 and relerr(dbeta, db_ref) < 1e-4


@pytest.mark.parametrize("shape", [(4, 64, 64, 128), (32, 4, 4, 64), (3, 16, 12, 48), (2, 128, 128, 32), (2, 8, 8, 16)])
def test_single_launch_reductions(shape):
    """Lean reduction forms: channel sum (+ amax scale), BN backward sums, BN statistics + finalize vs torch (repeated)."""
    o = ops()
    B, H, W, C = shape
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(B, H, W, C, device="cuda", generator=g) * 3 + 1.5
    dy = torch.randn(B, H, W, C, device="cuda", generator=g) * 1e-4
    for rep in range(3):
        s, amax = o.channel_sum(dy, want_amax=True)
        torch.cuda.synchronize()
        ref = dy.double().sum(dim=(0, 1, 2))
        assert ((s.double() - ref).abs().max() / ref.abs().max()).item() < 1e-5
        m = dy.abs().max().item()
        S, invS = amax.tolist()
        assert S * invS == 1.0 and 2.0 ** 14 <= m * S < 2.0 ** 15, (m, S)
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g)
    rm = torch.zeros(C, device="cuda")
    rv = torch.ones(C, device="cuda")
    mean, var, scale, shift, invstd = o.bn_stats_finalize(x, gamma, beta, 1e-5, rm, rv, 0.1)
    torch.cuda.synchronize()
    xr = x.double().reshape(-1, C)
    assert ((mean.double() - xr.mean(0)).abs().max() / xr.mean(0).abs().max()).item() < 1e-6
    assert ((var.double() - xr.var(0, unbiased=False)).abs().max() / xr.var(0, unbiased=False).max()).item() < 1e-5
    assert torch.allclose(invstd.double(), 1.0 / torch.sqrt(xr.var(0, unbiased=False) + 1e-5), rtol=1e-5)
    assert torch.allclose(scale, gamma * invstd) and torch.equal(shift, beta)
    n = xr.shape[0]
    assert torch.allclose(rm.double(), 0.1 * xr.mean(0), rtol=1e-5, atol=1e-7)
    assert torch.allclose(rv.double(), 0.9 + 0.1 * xr.var(0, unbiased=False) * n / (n - 1), rtol=1e-5)
    # BN backward sums through the fused path equal the two-stage path
    sums = o.bn_bwd_reduce(dy, x, mean, invstd, scale, shift, True)
    old = o.FUSED_REDUCE
    try:
        o.FUSED_REDUCE = False
        sums2 = o.bn_bwd_reduce(dy, x, mean, invstd, scale, shift, True)
    finally:
        o.FUSED_REDUCE = old
    torch.cuda.synchronize()
    assert torch.allclose(sums, sums2, rtol=1e-6, atol=1e-9)   # same fp64 partial scheme, different block geometry


@pytest.mark.parametrize("shape", [(2, 32, 32, 64, 64), (2, 64, 64, 64, 64), (3, 16, 16, 64, 64), (4, 8, 8, 64, 64),
                                   (2, 64, 48, 64, 32), (2, 32, 32, 128, 128), (2, 16, 16, 128, 64), (2, 32, 24, 64, 96)])
@pytest.mark.parametrize("passes", [3, 1])
def test_conv2d_wgrad_tc3_halo_kernel(shape, passes):
    """3x3 weight gradient (csrc/conv_wgmma.cu, every shape the 3x3 entry point takes) vs torch fp32, with the BN-apply +
    ReLU pre-op fused in."""
    B, H, W, Cin, Cout = shape
    o = ops()
    if not o.N.lib().fpd_conv2d_wgrad_tc3_supported(H, W, Cin, Cout, 3):
        pytest.skip("shape not taken by the 3x3 weight-gradient entry point")
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g) * 2 + 0.3
    dy = torch.randn(B, Cout, H, W, device="cuda", generator=g)
    mean = torch.randn(Cin, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.5
    a = F.relu((x - mean.view(1, -1, 1, 1)) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    ref = torch.nn.grad.conv2d_weight(a, (Cout, Cin, 3, 3), dy, padding=1)
    dw = o.conv2d_wgrad_tc_fused(nhwc(x), nhwc(dy), 3, mean=mean, scale=scale, shift=shift, relu=True, passes=passes)
    torch.cuda.synchronize()
    assert relerr(dw, ref) < (2e-5 if passes == 3 else 3e-3), "wgrad_tc3 %s passes=%d: %.3e" % (shape, passes, relerr(dw, ref))


def test_split_is_exact_tf32_pair():
    o = ops()
    x = torch.randn(8, 8, 8, 32, device="cuda") * 3
    hi, lo = o.affine_act_split(x)
    torch.cuda.synchronize()
    # both parts have their low 13 mantissa bits clear and hi+lo reproduces x to ~2^-21
    assert int((hi.view(torch.int32) & 0x1FFF).abs().max()) == 0
    assert int((lo.view(torch.int32) & 0x1FFF).abs().max()) == 0
    assert relerr(hi + lo, x) < 1e-6


def test_pool_upsample_layout_add():
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(3, 64, 16, 12, device="cuda", generator=g, requires_grad=True)
    y_ref = F.max_pool2d(x, 2, stride=2)
    dy = torch.randn_like(y_ref)
    (dx_ref,) = torch.autograd.grad(y_ref, x, dy)
    xh = nhwc(x.detach())
    y = o.maxpool2x2(xh)
    dx = o.maxpool2x2_bwd(xh, nhwc(dy))
    base = torch.randn_like(xh)
    dx_acc = o.maxpool2x2_bwd(xh, nhwc(dy), accumulate_into=base.clone())
    up1 = torch.randn(3, 64, 16, 12, device="cuda", generator=g)
    low = torch.randn(3, 64, 8, 6, device="cuda", generator=g)
    out_ref = up1 + F.interpolate(low, scale_factor=2, mode="nearest")
    out = o.upsample2x_add(nhwc(up1), nhwc(low))
    dlow = o.upsample2x_bwd(nhwc(up1))
    dlow_ref = F.avg_pool2d(up1, 2) * 4
    torch.cuda.synchronize()
    assert torch.equal(nchw(y), y_ref)
    assert torch.equal(nchw(dx), dx_ref)
    assert relerr(dx_acc, base + nhwc(dx_ref)) < 1e-6
    assert relerr(nchw(out), out_ref) < 1e-7
    assert relerr(nchw(dlow), dlow_ref) < 1e-6
    z = torch.randn(2, 17, 64, 48, device="cuda")
    assert torch.equal(o.nchw_to_nhwc(z), nhwc(z))
    assert torch.equal(o.nhwc_to_nchw(nhwc(z)), z)
    assert torch.equal(o.add(z, z), z + z)
    assert relerr(o.channel_sum(nhwc(x.detach())), x.detach().sum((0, 2, 3))) < 1e-5


def _ref_joints_mse(output, target, tw):
    # closed form of lib/core/loss.py:21-39 (checked against the reference module in tests/test_oracle.py)
    B, J = output.shape[:2]
    d = (output - target).reshape(B, J, -1) * tw.reshape(B, J, 1)
    return 0.5 * (d ** 2).mean(dim=(0, 2)).sum() / J


@pytest.mark.parametrize("S,B,J,h,w,teacher", [(4, 4, 16, 64, 64, True), (1, 2, 16, 64, 64, False), (2, 3, 17, 64, 48, True)])
def test_fpd_loss_fused(S, B, J, h, w, teacher):
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(9)
    outs = [torch.randn(B, J, h, w, device="cuda", generator=g, requires_grad=True) for _ in range(S)]
    target = torch.rand(B, J, h, w, device="cuda", generator=g)
    t = torch.randn(B, J, h, w, device="cuda", generator=g) if teacher else None
    tw = (torch.rand(B, J, 1, device="cuda", generator=g) > 0.2).float() * (1 + torch.rand(B, J, 1, device="cuda", generator=g))
    alpha = 0.5
    pose = sum(_ref_joints_mse(x, target, tw) for x in outs)
    if teacher:
        kd = sum(_ref_joints_mse(x, t, tw) for x in outs)
        loss = (1 - alpha) * pose + alpha * kd
    else:
        kd = torch.zeros(())
        loss = pose
    grads_ref = torch.autograd.grad(loss, outs)
    losses, grads = o.fpd_loss([nhwc(x.detach()) for x in outs], target, nhwc(t) if teacher else None, tw, alpha)
    torch.cuda.synchronize()
    assert abs(losses[0].item() - pose.item()) <= 1e-5 * abs(pose.item())
    if teacher:
        assert abs(losses[1].item() - kd.item()) <= 1e-5 * abs(kd.item())
    assert abs(losses[2].item() - loss.item()) <= 1e-5 * abs(loss.item())
    for gm, gr in zip(grads, grads_ref):
        assert relerr(nchw(gm), gr) < 1e-5


def test_joints_mse_nchw():
    o = ops()
    out = torch.randn(4, 16, 64, 64, device="cuda", requires_grad=True)
    tgt = torch.rand(4, 16, 64, 64, device="cuda")
    tw = torch.rand(4, 16, 1, device="cuda")
    ref = _ref_joints_mse(out, tgt, tw)
    (g_ref,) = torch.autograd.grad(ref, out)
    loss3, grad = o.joints_mse(out.detach(), tgt, tw)
    torch.cuda.synchronize()
    assert abs(loss3[0].item() - ref.item()) < 1e-5 * abs(ref.item())
    assert relerr(grad, g_ref) < 1e-5


def test_flip_merge_argmax_bit_exact():
    o = ops()
    B, J, h, w = 6, 16, 64, 64
    g = torch.Generator(device="cuda").manual_seed(21)
    hm = torch.randn(B, J, h, w, device="cuda", generator=g)
    hf = torch.randn(B, J, h, w, device="cuda", generator=g)
    hm[0, 0] = 0.25  # constant map: first index must win
    hf[0, 0] = 0.25
    pairs = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]
    perm = list(range(J))
    for a, b in pairs:
        perm[a], perm[b] = b, a
    # numpy restatement of function.py:218-240 + transforms.py:15-29 + inference.py:18-46
    f = hf.cpu().numpy()[:, :, :, ::-1].copy()
    for a, b in pairs:
        tmp = f[:, a].copy(); f[:, a] = f[:, b]; f[:, b] = tmp
    f[:, :, :, 1:] = f.copy()[:, :, :, 0:-1]
    merged = (hm.cpu().numpy() + f) * np.float32(0.5)
    idx_ref = merged.reshape(B, J, -1).argmax(2)
    max_ref = merged.reshape(B, J, -1).max(2)
    avg, idx, maxval = o.flip_merge_argmax(nhwc(hm), nhwc(hf), torch.tensor(perm, dtype=torch.int32, device="cuda"), shift=True)
    torch.cuda.synchronize()
    assert np.array_equal(nchw(avg).cpu().numpy(), merged)
    assert np.array_equal(idx.cpu().numpy(), idx_ref)
    assert np.array_equal(maxval.cpu().numpy(), max_ref)
    idx2, max2 = o.argmax_nchw(hm)
    assert np.array_equal(idx2.cpu().numpy(), hm.cpu().numpy().reshape(B, J, -1).argmax(2))


def _nms_numpy(dets, thresh):
    # restatement of lib/nms/nms.py:35-72
    x1, y1, x2, y2, scores = dets[:, 0], dets[:, 1], dets[:, 2], dets[:, 3], dets[:, 4]
    areas = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = scores.argsort()[::-1]
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(i)
        xx1 = np.maximum(x1[i], x1[order[1:]]); yy1 = np.maximum(y1[i], y1[order[1:]])
        xx2 = np.minimum(x2[i], x2[order[1:]]); yy2 = np.minimum(y2[i], y2[order[1:]])
        ww = np.maximum(0.0, xx2 - xx1 + 1); hh = np.maximum(0.0, yy2 - yy1 + 1)
        inter = ww * hh
        ovr = inter / (areas[i] + areas[order[1:]] - inter)
        order = order[np.where(ovr <= thresh)[0] + 1]
    return keep


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1000, 4096])
def test_nms_matches_numpy(n):
    o = ops()
    rng = np.random.RandomState(n)
    x1 = rng.uniform(0, 256, n); y1 = rng.uniform(0, 256, n)
    bw = rng.uniform(8, 128, n); bh = rng.uniform(8, 128, n)
    dets = np.stack([x1, y1, x1 + bw, y1 + bh, rng.uniform(0, 1, n)], 1).astype(np.float32)
    keep_ref = _nms_numpy(dets, 0.6)
    order = dets[:, 4].argsort()[::-1]
    sorted_dets = torch.from_numpy(dets[order].copy()).cuda()
    keep, num = o.nms_device(sorted_dets, 0.6)
    torch.cuda.synchronize()
    k = keep[: int(num.item())].cpu().numpy()
    assert list(order[k]) == list(keep_ref)
    # host-pointer drop-in for `_nms`
    import ctypes
    from fpd_b200 import _native as N
    keep_h = np.zeros(n, dtype=np.int32); num_h = ctypes.c_int(0)
    sd = np.ascontiguousarray(dets[order])
    N.check(N.lib().fpd_nms_host(keep_h.ctypes.data_as(ctypes.c_void_p), ctypes.cast(ctypes.byref(num_h), ctypes.c_void_p),
                                 sd.ctypes.data_as(ctypes.c_void_p), n, 5, 0.6, 0))
    assert list(order[keep_h[: num_h.value]]) == list(keep_ref)


def test_adam_flat_matches_torch():
    o = ops()
    p = torch.randn(10007, device="cuda")
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=2.5e-4)
    m = torch.zeros_like(p); v = torch.zeros_like(p)
    for step in range(1, 4):
        gr = torch.randn_like(p)
        ref.grad = gr.clone()
        opt.step()
        o.adam_flat(p, gr, m, v, 2.5e-4, 0.9, 0.999, 1e-8, 0.0, step)
    torch.cuda.synchronize()
    assert relerr(p, ref.detach()) < 1e-6


@pytest.mark.parametrize("cfg", [(2, 64, 64, 3, 32, 7, 2, 3), (2, 64, 48, 3, 64, 3, 2, 1)])
def test_stem_im2col_tensor_core_path(cfg):
    """Stem convs (Cin=3) as im2col + 1x1 tensor-core conv / weight gradient vs torch fp32."""
    B, H, W, Cin, Cout, k, stride, pad = cfg
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(13)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g, requires_grad=True)
    bias = torch.randn(Cout, device="cuda", generator=g)
    y_ref = F.conv2d(x, w, bias, stride=stride, padding=pad)
    dy = torch.randn_like(y_ref)
    (dw_ref,) = torch.autograd.grad(y_ref, w, dy)
    K = Cin * k * k
    kpad = (K + 31) // 32 * 32
    cols = o.im2col(nhwc(x), k, stride, pad, kpad)
    w2 = torch.zeros(Cout, kpad, 1, 1, device="cuda")
    w2[:, :K, 0, 0] = w.detach().permute(0, 2, 3, 1).reshape(Cout, -1)
    w_hi, w_lo = o.weight_prep(w2)
    y = o.conv2d_tc_fused(cols, w_hi, w_lo, 1, bias=bias)
    dw = o.conv2d_wgrad_tc_fused(cols, nhwc(dy), 1)
    dw = dw[:, :K, 0, 0].reshape(Cout, k, k, Cin).permute(0, 3, 1, 2)
    torch.cuda.synchronize()
    assert relerr(nchw(y), y_ref) < 2e-5
    assert relerr(dw, dw_ref) < 2e-5


@pytest.mark.parametrize("shape", [(4, 64, 64, 64, 64, 3), (2, 16, 16, 128, 64, 1), (3, 8, 8, 64, 128, 1), (5, 4, 4, 64, 64, 3),
                                   (32, 64, 64, 128, 128, 1), (2, 64, 48, 32, 32, 3), (2, 64, 64, 16, 128, 1)])
@pytest.mark.parametrize("f16", [True, False])
@pytest.mark.parametrize("with_pivot", [False, True])
def test_conv2d_tc_h_epilogue_batchnorm_statistics(shape, f16, with_pivot):
    """conv_tc_h_kernel<.., kStats>: the output is bit-identical to the plain kernel's, and the per-channel statistics
    finalized from the epilogue's partial sums equal nn.BatchNorm2d's batch statistics of that output (mean, biased
    variance, scale / shift, running-statistics update) -- including ragged batch tails (B % images-per-tile != 0) and a
    large common-mode offset with a pivot."""
    B, H, W, Cin, Cout, k = shape
    o = ops()
    o.CONV_STATS = "1"      # off by default (measured neutral on the bench step): the kernel variant is tested regardless
    nblk = o.conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, k, f16)
    o.CONV_STATS = os.environ.get("FPD_CONV_STATS", "3x3").lower()
    if nblk == 0:
        pytest.skip("shape does not carry epilogue statistics")
    g = torch.Generator(device="cuda").manual_seed(77)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (1.0 / (Cin * k * k) ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g) * (30.0 if with_pivot else 1.0)     # common-mode offset
    res = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    mean_in = torch.randn(Cin, device="cuda", generator=g) * 0.1
    scale_in = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift_in = torch.randn(Cin, device="cuda", generator=g) * 0.1
    prep = o.weight_prep_f16 if f16 else o.weight_prep
    w_hi, w_lo = prep(w)
    kw = dict(mean=mean_in, scale=scale_in, shift=shift_in, relu=True, bias=bias, residual=res)
    y_plain = o.conv2d_tc_h(x, w_hi, w_lo, k, **kw)
    part = torch.full((nblk, Cout, 2), float("nan"), dtype=torch.float64, device="cuda")
    pivot = (bias + 0.3).contiguous() if with_pivot else None
    y = o.conv2d_tc_h(x, w_hi, w_lo, k, stats_part=part, stats_pivot=pivot, **kw)
    assert torch.equal(y, y_plain)
    gamma = torch.rand(Cout, device="cuda", generator=g) + 0.5
    beta = torch.randn(Cout, device="cuda", generator=g)
    rm = torch.randn(Cout, device="cuda", generator=g)
    rv = torch.rand(Cout, device="cuda", generator=g) + 0.5
    rm0, rv0 = rm.clone(), rv.clone()
    mean, var, scale, shift, invstd = o.bn_finalize_sums(part, nblk, pivot, B * H * W, gamma, beta, 1e-5, rm, rv, 0.1)
    torch.cuda.synchronize()
    yd = y.double().reshape(-1, Cout)
    ref_mean, ref_var = yd.mean(0), yd.var(0, unbiased=False)
    # relative to the channel's std; the mean is returned in fp32: allow its own rounding (|mean| * 2^-24)
    assert (((mean.double() - ref_mean).abs() - ref_mean.abs() * 6e-8).clamp_min(0) / (ref_var.sqrt() + 1e-30)).max() < 2e-6
    tol_var = 2e-6 * (1.0 + float((((ref_mean - (pivot.double() if with_pivot else 0.0)) ** 2) / ref_var).max()))
    assert relerr(var, ref_var) < max(tol_var, 1e-5), (relerr(var, ref_var), tol_var)
    ref_invstd = 1.0 / torch.sqrt(ref_var + 1e-5)
    assert relerr(invstd, ref_invstd) < 1e-5 and relerr(scale, gamma.double() * ref_invstd) < 1e-5
    assert torch.equal(shift, beta)
    n = B * H * W
    assert relerr(rm, 0.9 * rm0.double() + 0.1 * ref_mean) < 1e-5
    assert relerr(rv, 0.9 * rv0.double() + 0.1 * ref_var * n / (n - 1)) < 1e-5
    # and equal to the separate statistics pass it replaces
    m2, v2, s2, _, i2 = o.bn_stats_finalize(y, gamma, beta, 1e-5)
    assert relerr(mean, m2) < 1e-5 and relerr(var, v2) < 2e-5


def test_stride2_conv_as_stride1_plus_pick():
    """subsample2 / upsample_zero2 (adjoint pair) and the identity they serve: a 3x3 stride-2 pad-1 convolution equals the
    stride-1 convolution picked at the even positions; its input gradient equals the stride-1 data gradient of the
    zero-upsampled dY."""
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(3, 32, 24, 64, device="cuda", generator=g)
    y = o.subsample2(x)
    assert torch.equal(y, x[:, ::2, ::2, :].contiguous())
    dy = torch.randn_like(y)
    dx = o.upsample_zero2(dy)
    ref = torch.zeros_like(x)
    ref[:, ::2, ::2, :] = dy
    assert torch.equal(dx, ref)
    assert abs(float((y * dy).sum()) - float((x * dx).sum())) < 1e-3 * float((y * dy).abs().sum())      # <Sx, dy> = <x, S^T dy>
    w = torch.randn(96, 64, 3, 3, device="cuda", generator=g) * 0.05
    w_hi, w_lo = o.weight_prep_f16(w)
    full = o.conv2d_tc_h(x, w_hi, w_lo, 3)
    got = o.subsample2(full)
    want = F.conv2d(nchw(x), w, None, stride=2, padding=1)
    assert relerr(nchw(got), want) < 2e-5
