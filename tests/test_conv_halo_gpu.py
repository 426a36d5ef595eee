"""The halo-resident 3x3 path of the 3xFP16 forward / data-gradient convolution (conv_halo_kernel, csrc/conv_wgmma.cu)
against a torch fp64 convolution: image widths from 4 to 128, pixel counts that are not a multiple of the 128-pixel tile,
tiles that span several images, input widths that are not a multiple of the 64-channel block, BN affine + ReLU with a
non-zero shift (the padding is zero after the affine), bias, residual, ReLU mask, the data-gradient input scale and the
epilogue statistics, and output slices of 48 to 128 columns. The profiler confirms which kernel ran."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# B, H, W, Cin, Cout
HALO_SHAPES = [
    (3, 4, 4, 64, 64),       # 48 pixels: one partial tile over three images
    (5, 8, 8, 32, 48),       # 320 pixels, tiles span two images; Cin below one channel block
    (2, 6, 12, 48, 96),      # H != W; Cin = 48 (channels 48..63 of the block are zero)
    (2, 19, 48, 96, 112),    # 1824 pixels; Cin = 96: a full and a partial channel block
    (1, 37, 64, 128, 128),   # the hourglass teacher's 3x3 shape, ragged last tile
    (2, 13, 64, 64, 192),    # two 96-column output slices
    (1, 24, 128, 64, 80),    # W = 128
    (2, 7, 9, 128, 64),
]


def ops():
    from fpd_b200 import ops as o
    return o


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type is not None and "cuda" in str(e.device_type).lower()]


def ran_halo(names):
    return any("conv_halo_kernel" in n for n in names) and not any("conv_wgmma_kernel" in n for n in names)


@pytest.mark.parametrize("shape", HALO_SHAPES)
def test_halo_forward_bn_relu_bias_residual(shape):
    B, H, W, Cin, Cout = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(101)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g) * 2 + 0.5
    mean = torch.randn(Cin, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.5 + 0.75   # relu(shift) > 0 for most channels
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (1.0 / (Cin * 9) ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B, Cout, H, W, device="cuda", generator=g)
    a = F.relu((x.double() - mean.double().view(1, -1, 1, 1)) * scale.double().view(1, -1, 1, 1)
               + shift.double().view(1, -1, 1, 1))
    ref = F.conv2d(a, w.double(), bias.double(), padding=1) + res.double()
    w_hi, w_lo = o.weight_prep_f16(w)
    run = lambda: o.conv2d_tc_h(nhwc(x), w_hi, w_lo, 3, mean=mean, scale=scale, shift=shift, relu=True,  # noqa: E731
                                bias=bias, residual=nhwc(res))
    y = run()
    torch.cuda.synchronize()
    assert relerr(nchw(y), ref) < 3e-5, "%s rel err %.3e" % (shape, relerr(nchw(y), ref))
    assert ran_halo(kernel_names(run)), shape


@pytest.mark.parametrize("shape", HALO_SHAPES[:4] + [(2, 16, 16, 128, 128)])
@pytest.mark.parametrize("mag", [1e-6, 1.0, 1e3])
def test_halo_data_gradient_in_scale_relu_mask(shape, mag):
    """Data-gradient form: raw dY scaled by the power-of-two in_scale into the fp16 range, output masked by the forward
    activation (relu_mask) and scaled back."""
    B, H, W, Cin, Cout = shape     # forward Cin -> Cout; the data gradient runs Cout -> Cin
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(202)
    dy = torch.randn(B, H, W, Cout, device="cuda", generator=g) * mag
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (1.0 / (Cin * 9) ** 0.5)
    act = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    ref = torch.nn.grad.conv2d_input((B, Cin, H, W), w.double(), nchw(dy).double(), padding=1)
    ref = ref * (nchw(act) > 0).double()
    _, s = o.channel_sum(dy, want_amax=True)
    wd_hi, wd_lo = o.weight_prep_f16(w, for_dgrad=True)
    run = lambda: o.conv2d_tc_h(dy, wd_hi, wd_lo, 3, in_scale=s, relu_mask=act)   # noqa: E731
    da = run()
    torch.cuda.synchronize()
    assert relerr(nchw(da), ref) < 3e-5, "%s mag %g rel err %.3e" % (shape, mag, relerr(nchw(da), ref))
    assert ran_halo(kernel_names(run)), shape


@pytest.mark.parametrize("shape", [(3, 4, 4, 64, 64), (5, 8, 8, 32, 48), (1, 37, 64, 128, 128), (2, 13, 64, 64, 192)])
def test_halo_epilogue_statistics(shape):
    """Epilogue statistics from the halo kernel: the output equals the plain call's bit for bit, and the per-channel sums
    equal fp64 sums of that output."""
    B, H, W, Cin, Cout = shape
    o = ops()
    nblk = int(o.N.lib().fpd_conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, 3, 1))
    assert nblk > 0
    g = torch.Generator(device="cuda").manual_seed(303)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (1.0 / (Cin * 9) ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g) * 20.0
    pivot = (bias + 0.3).contiguous()
    kw = dict(mean=torch.randn(Cin, device="cuda", generator=g) * 0.1, scale=torch.rand(Cin, device="cuda", generator=g) + 0.5,
              shift=torch.randn(Cin, device="cuda", generator=g) * 0.1 + 0.2, relu=True, bias=bias)
    w_hi, w_lo = o.weight_prep_f16(w)
    y_plain = o.conv2d_tc_h(x, w_hi, w_lo, 3, **kw)
    part = torch.full((nblk, Cout, 2), float("nan"), dtype=torch.float64, device="cuda")
    run = lambda: o.conv2d_tc_h(x, w_hi, w_lo, 3, stats_part=part, stats_pivot=pivot, **kw)   # noqa: E731
    y = run()
    torch.cuda.synchronize()
    assert torch.equal(y, y_plain)
    d = y.double().reshape(-1, Cout) - pivot.double()
    s1, s2 = part.sum(0)[:, 0], part.sum(0)[:, 1]
    assert relerr(s1, d.sum(0)) < 1e-9 * d.shape[0]
    assert relerr(s2, (d * d).sum(0)) < 1e-9 * d.shape[0]
    assert ran_halo(kernel_names(run)), shape


def test_halo_selection():
    """3x3 3xFP16 shapes whose halo fits run the halo kernel; 1x1, single-pass, 3xTF32 and halos that do not fit in
    shared memory stay on conv_wgmma_kernel."""
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(404)

    def names(B, H, W, Cin, Cout, k, split=True, f16=True):
        x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
        w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * 0.05
        w_hi, w_lo = (o.weight_prep_f16 if f16 else o.weight_prep)(w, split=split)
        return kernel_names(lambda: o.conv2d_tc_h(x, w_hi, w_lo, k))

    assert ran_halo(names(2, 64, 64, 128, 128, 3))
    assert ran_halo(names(2, 64, 64, 64, 64, 3))
    for args, kw in (((2, 64, 64, 128, 128, 1), {}),               # 1x1
                     ((2, 64, 64, 64, 64, 3), {"split": False}),   # single-pass fp16
                     ((2, 64, 64, 64, 64, 3), {"f16": False}),     # 3xTF32
                     ((1, 32, 128, 128, 128, 3), {}),              # W = 128 with two channel blocks: halo too large
                     ((2, 16, 12, 384, 384, 3), {})):              # six channel blocks: halo too large
        n = names(*args, **kw)
        assert any("conv_wgmma_kernel" in s for s in n) and not any("conv_halo_kernel" in s for s in n), (args, kw)
