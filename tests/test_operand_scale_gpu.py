"""The power-of-two operand scale {S, 1/S} of the FP16 data gradients (channel_sum(want_amax=True) and the BatchNorm-
backward apply pass that sums its own output) at the edges of the float range, and the data gradients that use it.

S puts max|dY| into [2^14, 2^15), so that fp16_rn(dY * S) neither overflows nor loses the small elements. It is capped
at 2^126 so that S and 1/S are both normal floats: maxima below 2^-112 get S = 2^126 and sit below 2^14 after scaling.
Zero, non-finite and >= 3e38 maxima give S = 1. NaN elements do not take part in the maximum."""
import math

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
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops as o
    return o


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-300)).item()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def f32(v):
    """v rounded to the nearest float32, as a Python float."""
    return torch.tensor(v, dtype=torch.float32).item()


TINY = f32(2.0 ** -149)                                  # the smallest subnormal
BELOW_113 = 2.0 ** -113 * (1.0 - 2.0 ** -24)            # the float32 just below 2^-113
BELOW_112 = 2.0 ** -112 * (1.0 - 2.0 ** -24)
MAXIMA = [0.0, TINY, f32(1e-40), 2.0 ** -126, BELOW_113, 2.0 ** -113, BELOW_112, 2.0 ** -112, f32(1e-7), 1.0,
          6e4, f32(1e30), f32(3e38)]


def check_scale(s, m):
    """{S, 1/S} = s for a tensor whose largest finite magnitude is m."""
    S, R = (float(v) for v in s.cpu())
    assert math.isfinite(S) and math.isfinite(R), (m, S, R)
    assert S > 0 and math.frexp(S)[0] == 0.5, (m, S)            # a power of two
    assert S * R == 1.0, (m, S, R)
    assert R >= 2.0 ** -126 and S >= 2.0 ** -126, (m, S, R)     # both normal
    if m == 0.0 or not math.isfinite(m) or m >= f32(3e38):
        assert S == 1.0, (m, S)
    elif m >= 2.0 ** -112:
        assert 2.0 ** 14 <= m * S < 2.0 ** 15, (m, S)
    else:
        assert S == 2.0 ** 126, (m, S)


def with_max(shape, m, seed, zeros=0.3):
    """Random tensor with exact zeros and one element -m (every other |element| <= m)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn(shape, device="cuda", generator=g, dtype=torch.float64)
    base[torch.rand(shape, device="cuda", generator=g) < zeros] = 0.0
    base = base / base.abs().max() * 0.999
    base.view(-1)[base.numel() - 3] = -1.0
    return (base * m).float()


def max_abs(t):
    t = t.double()
    t = t[~torch.isnan(t)]
    return t.abs().max().item() if t.numel() else 0.0


@pytest.mark.parametrize("shape", [(2, 9, 7, 64), (1, 3, 5, 2048)])
@pytest.mark.parametrize("m", MAXIMA)
def test_channel_sum_operand_scale(shape, m):
    o = ops()
    dy = with_max(shape, m, 1)
    assert max_abs(dy) == m
    s_sum, s = o.channel_sum(dy, want_amax=True)
    torch.cuda.synchronize()
    check_scale(s, m)
    C = shape[-1]
    ref = dy.double().reshape(-1, C).sum(0)
    mag = dy.double().reshape(-1, C).abs().sum(0)
    sums_fit = m < 1e37     # the sums of the 3e38 tensor overflow fp32
    assert not sums_fit or ((s_sum.double() - ref).abs() <= mag * 18 * 2.0 ** -24 + 2.0 ** -149).all()
    # the two-launch form without the scale: the same sums, no scale
    prev = o.FUSED_REDUCE
    o.FUSED_REDUCE = False
    try:
        s_sum2, s2 = o.channel_sum(dy, want_amax=True)
    finally:
        o.FUSED_REDUCE = prev
    torch.cuda.synchronize()
    assert s2 is None
    assert not sums_fit or ((s_sum2.double() - ref).abs() <= mag * 18 * 2.0 ** -24 + 2.0 ** -149).all()


@pytest.mark.parametrize("m", [f32(1e-7), 1.0, 6e4])
def test_nan_does_not_take_part_in_the_maximum(m):
    o = ops()
    dy = with_max((2, 8, 6, 32), m, 2)
    dy[1, 3, 2, 5] = float("nan")
    _, s = o.channel_sum(dy, want_amax=True)
    torch.cuda.synchronize()
    check_scale(s, m)
    # infinite maximum: no scaling
    dy[0, 0, 0, 0] = float("inf")
    _, s = o.channel_sum(dy, want_amax=True)
    torch.cuda.synchronize()
    check_scale(s, float("inf"))


def _bn_operands(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, H, W, C = shape
    x = torch.randn(shape, device="cuda", generator=g) * 0.7 + 0.2
    mean = x.double().reshape(-1, C).mean(0).float()
    invstd = (1.0 / (x.double().reshape(-1, C).var(0, unbiased=False) + 1e-5).sqrt()).float()
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g) * 0.1
    return x, mean, invstd, (gamma * invstd).contiguous(), beta, gamma


@pytest.mark.parametrize("m", [0.0, TINY, f32(1e-40), 2.0 ** -126, BELOW_113, BELOW_112, 2.0 ** -112, f32(1e-7),
                               1.0, 6e4, f32(1e30)])
def test_bn_bwd_apply_sum_operand_scale(m):
    """The scale out of the BatchNorm-backward apply pass is the scale of the dx it wrote."""
    o = ops()
    shape = (2, 9, 7, 64)
    x, mean, invstd, scale, shift, gamma = _bn_operands(shape, 3)
    da = with_max(shape, m, 4)
    dx, _, _, (dx_sum, s) = o.bn_bwd(da, x, mean, invstd, scale, shift, gamma, False, want_dx_sum="force")
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all()
    check_scale(s, max_abs(dx))
    # the same scale as channel_sum(dx, want_amax=True)
    assert torch.equal(s, o.channel_sum(dx, want_amax=True)[1])


# ------------------------------------------------------------------------------------------------ data gradients
# dY with exact zeros and its maximum at 2^-149 .. 2^-20: through the 3xFP16 (conv2d_tc_h with fp16 weights) and the
# single-pass FP16 (conv2d_tc_f16x1) data-gradient kernels with the scale of channel_sum(want_amax=True)
DGRAD_MAXIMA = [TINY, f32(1e-40), 2.0 ** -126, 2.0 ** -120, BELOW_112, 2.0 ** -112, 2.0 ** -20]
# B, H, W, C_dY, C_dX, k, kernel selection
DGRAD_SHAPES = [(2, 16, 12, 64, 64, 3, "halo"), (2, 16, 12, 128, 64, 1, "1x1"), (2, 9, 11, 64, 48, 3, "staged")]


def _dgrad_case(shape, m):
    B, H, W, Cdy, Cdx, k = shape[:6]
    dy = with_max((B, H, W, Cdy), m, 5)
    g = torch.Generator(device="cuda").manual_seed(6)
    w = torch.randn(Cdy, Cdx, k, k, device="cuda", generator=g) * (1.0 / (Cdy * k * k) ** 0.5)   # forward Cdx -> Cdy
    return dy, w


def _selected(o, kind):
    """Selection switches for the kernel named by kind; returns the callable that restores them."""
    halo = o.set_conv_halo(kind != "staged")
    pw = o.set_conv1x1(kind == "1x1")
    return lambda: (o.set_conv_halo(halo), o.set_conv1x1(pw))


@pytest.mark.parametrize("shape", DGRAD_SHAPES)
@pytest.mark.parametrize("m", DGRAD_MAXIMA)
def test_3xfp16_data_gradient_tiny_dy(shape, m):
    o = ops()
    k = shape[5]
    dy, w = _dgrad_case(shape, m)
    _, s = o.channel_sum(dy, want_amax=True)
    check_scale(s, m)
    w_hi, w_lo = o.weight_prep_f16(w, for_dgrad=True)
    restore = _selected(o, shape[6])
    try:
        dx = o.conv2d_tc_h(dy, w_hi, w_lo, k, in_scale=s)
    finally:
        restore()
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all(), (shape, m)
    if m < 2.0 ** -126:
        return
    # fp16 hi + lo of dY * S carry 22 significant bits down to 2^-24 (the fp16 subnormal step); with S capped at 2^126 the
    # scaled maximum can be as small as 1, which still leaves every element within 2^-25 of its value: far below the bound
    # the kernels meet at magnitude 1
    ref = F.conv_transpose2d(nchw(dy).double(), w.double(), padding=k // 2)
    assert relerr(nchw(dx), ref) < 2e-5, (shape, m, relerr(nchw(dx), ref))


@pytest.mark.parametrize("shape", [s for s in DGRAD_SHAPES if s[6] != "staged"])
@pytest.mark.parametrize("m", DGRAD_MAXIMA)
def test_fp16x1_data_gradient_tiny_dy(shape, m):
    o = ops()
    B, H, W, Cdy, Cdx, k, kind = shape
    dy, w = _dgrad_case(shape, m)
    _, s = o.channel_sum(dy, want_amax=True)
    wd, _ = o.weight_prep_f16(w, for_dgrad=True, split=False)
    assert o.conv2d_tc_f16x1_train_plan(B, H, W, Cdy, Cdx, k)[0] == kind
    dx = o.conv2d_tc_f16x1(dy, wd, k, in_scale=s)
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all(), (shape, m)
    if m < 2.0 ** -126:
        return
    # against fp64 on the operand the kernel multiplies, fp16_rn(dY S) / S (fp16 subnormals included), as the
    # single-pass tests at ordinary magnitudes do
    S = float(s[0])
    q = (dy.double() * S).half().double() / S
    wd16 = wd.double().view(k, k, Cdx, Cdy).permute(2, 3, 0, 1) / 256.0
    ref = F.conv2d(nchw(q), wd16, padding=k // 2)
    assert relerr(nchw(dx), ref) < 1e-4, (shape, m, relerr(nchw(dx), ref))
    exact = F.conv_transpose2d(nchw(dy).double(), w.double(), padding=k // 2)
    assert relerr(nchw(dx), exact) < 2e-3, (shape, m, relerr(nchw(dx), exact))
