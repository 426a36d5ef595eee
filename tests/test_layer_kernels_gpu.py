"""The layer, reduction, operand-preparation and fallback kernels one by one against plain fp64 torch (or bit for bit
where the operation is exact): HRNet's fuse / upsample / BasicBlock-tail kernels, the BatchNorm backward options
(accumulate_into, sync_mean), the channel reductions at 4 .. 4096 channels and 1 .. 2^21 rows, max-pool ties, the weight
layouts and hi/lo splits, the flip-test layout change, im2col, the CUDA-core convolutions on their global-memory weight
path, the chunked tensor-core weight gradient and Adam with weight decay and a gradient scale.

Widths are the ones the networks use (HRNet-w32 / w48 branches 32..384, hourglass 64..256, pose_resnet up to 2048);
widths at HRNet's 256x192 input are 48, 24, 12 and 6."""
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


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def up(t, s):
    """Nearest-neighbour upsampling of an NHWC tensor by 2^s."""
    f = 1 << s
    return t.repeat_interleave(f, 1).repeat_interleave(f, 2)


# ------------------------------------------------------------------------------------------------ HRNet fuse
# every fuse row of a 1..4-branch HRNet stage: output branch i sums branch j upsampled by 2^(j-i) (j > i) or brought to
# its resolution by stride-2 convolutions (j <= i, shift 0); plus rows whose first term is not the full-size one
FUSE_ROWS = sorted({tuple(max(0, j - i) for j in range(n)) for n in range(1, 5) for i in range(n)}) + [
    (1, 0), (2, 0, 1), (3, 1, 0, 2)]
WIDTHS = [32, 48, 64, 96, 128, 192, 256, 384]


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("shifts", FUSE_ROWS)
def test_fuse_sum(shifts, relu):
    o = ops()
    C = WIDTHS[FUSE_ROWS.index(shifts) % len(WIDTHS)]
    B, H, W = 2, 32, 48
    g = gen(1)
    terms = [torch.randn(B, H >> s, W >> s, C, device="cuda", generator=g) for s in shifts]
    y = o.fuse_sum(terms, list(shifts), relu=relu)
    # the same fp32 additions in term order: bit-identical
    acc = up(terms[0], shifts[0])
    for t, s in zip(terms[1:], shifts[1:]):
        acc = acc + up(t, s)
    if relu:
        acc = acc.clamp_min(0.0)
    ref = sum(up(t.double(), s) for t, s in zip(terms, shifts))
    if relu:
        ref = ref.clamp_min(0.0)
    torch.cuda.synchronize()
    assert y.shape == (B, H, W, C)
    assert torch.equal(y, acc), shifts
    assert relerr(y, ref) < 1e-6


@pytest.mark.parametrize("shift", [1, 2, 3])
@pytest.mark.parametrize("C", [32, 96, 384])
def test_upsample_bwd(shift, C):
    """Adjoint of the nearest upsampling: each low-resolution pixel sums its f x f block (row-major, fp32)."""
    o = ops()
    B, H, W = 2, 32, 48
    dout = torch.randn(B, H, W, C, device="cuda", generator=gen(2))
    d = o.upsample_bwd(dout, shift)
    f = 1 << shift
    acc = torch.zeros(B, H >> shift, W >> shift, C, device="cuda")
    for dy in range(f):
        for dx in range(f):
            acc = acc + dout[:, dy::f, dx::f]
    ref = dout.double().view(B, H >> shift, f, W >> shift, f, C).sum((2, 4))
    torch.cuda.synchronize()
    assert torch.equal(d, acc)
    assert relerr(d, ref) < 1e-6


def _affine(C, seed):
    g = gen(seed)
    mean = torch.randn(C, device="cuda", generator=g) * 0.5
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.5
    return mean, scale, shift


def _pre(x, mean, scale, shift):
    """fp64 pre-activation (x - mean) * scale + shift; mean None is 0."""
    m = 0.0 if mean is None else mean.double()
    return (x.double() - m) * scale.double() + shift.double()


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("with_mean", [True, False])
@pytest.mark.parametrize("shape", [(2, 16, 12, 32), (2, 8, 6, 384), (1, 32, 48, 48)])
def test_affine_add_act(shape, with_mean, relu):
    """BasicBlock / Bottleneck tail: relu?((x - mean) * scale + shift + residual)."""
    o = ops()
    C = shape[-1]
    g = gen(3)
    x = torch.randn(shape, device="cuda", generator=g) * 2
    res = torch.randn(shape, device="cuda", generator=g)
    mean, scale, shift = _affine(C, 4)
    mean = mean if with_mean else None
    y = o.affine_add_act(x, res, scale, shift, relu=relu, mean=mean)
    ref = _pre(x, mean, scale, shift) + res.double()
    if relu:
        ref = ref.clamp_min(0.0)
    torch.cuda.synchronize()
    assert relerr(y, ref) < 1e-6


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("with_mean", [True, False])
@pytest.mark.parametrize("shape", [(2, 16, 12, 64), (2, 8, 6, 192), (1, 4, 6, 2048)])
def test_affine_act_bwd(shape, with_mean, accumulate, relu):
    """dx (+)= da * scale where the forward's pre-activation is positive (relu) or everywhere: one fp32 product per
    element, so bit-identical to the torch product."""
    o = ops()
    C = shape[-1]
    g = gen(5)
    x = torch.randn(shape, device="cuda", generator=g) * 2
    mean, scale, shift = _affine(C, 6)
    mean = mean if with_mean else None
    pre = _pre(x, mean, scale, shift)
    # no upstream gradient within round-off of the ReLU kink
    da = torch.randn(shape, device="cuda", generator=g) * (pre.abs() > 1e-5)
    base = torch.randn(shape, device="cuda", generator=g)
    dx = o.affine_act_bwd(da, x, scale, shift, relu, accumulate_into=base.clone() if accumulate else None, mean=mean)
    on = (pre > 0) if relu else torch.ones_like(pre, dtype=torch.bool)
    want = torch.where(on, da * scale, torch.zeros_like(da))
    ref = torch.where(on, da.double() * scale.double(), torch.zeros_like(pre))
    if accumulate:
        want = base + want
        ref = base.double() + ref
    torch.cuda.synchronize()
    assert torch.equal(dx, want)
    assert relerr(dx, ref) < 1e-6


# ------------------------------------------------------------------------------------------------ BatchNorm backward
def _bn_case(shape, seed, offset=0.0):
    g = gen(seed)
    C = shape[-1]
    x = torch.randn(shape, device="cuda", generator=g) * 0.8 + offset + torch.randn(C, device="cuda", generator=g)
    xd = x.double().reshape(-1, C)
    mean = xd.mean(0).float()
    invstd = (1.0 / (xd.var(0, unbiased=False) + 1e-5).sqrt()).float()
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g) * 0.5
    scale = (gamma * invstd).contiguous()
    pre = (x.double() - mean.double()) * scale.double() + beta.double()
    da = torch.randn(shape, device="cuda", generator=g) * (pre.abs() > 1e-4)
    return x, da, mean, invstd, scale, beta, gamma, pre


def _bn_bwd_ref(x, da, mean, invstd, gamma, pre, relu, alpha=1.0):
    """fp64 closed form of ops.bn_bwd with sync_mean(sums) = alpha * sums: dx = gamma invstd (dz - alpha mean(dz) -
    xhat alpha mean(dz xhat)); dgamma, dbeta = the local sums of dz xhat, dz."""
    C = x.shape[-1]
    P = x.numel() // C
    dz = da.double() * (pre > 0) if relu else da.double()
    xh = (x.double() - mean.double()) * invstd.double()
    sdz = dz.reshape(-1, C).sum(0)
    sdzx = (dz * xh).reshape(-1, C).sum(0)
    dx = gamma.double() * invstd.double() * (dz - alpha * sdz / P - xh * alpha * sdzx / P)
    mag = dz.abs().reshape(-1, C).sum(0), (dz * xh).abs().reshape(-1, C).sum(0)
    return dx, sdzx, sdz, mag


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("shape", [(2, 16, 12, 64), (2, 8, 6, 384), (2, 4, 6, 2048)])
def test_bn_bwd_accumulate_and_sync_mean(shape, relu):
    o = ops()
    x, da, mean, invstd, scale, shift, gamma, pre = _bn_case(shape, 7)
    dx, dgamma, dbeta = o.bn_bwd(da, x, mean, invstd, scale, shift, gamma, relu)
    ref, sdzx, sdz, (mag0, mag1) = _bn_bwd_ref(x, da, mean, invstd, gamma, pre, relu)
    torch.cuda.synchronize()
    assert relerr(dx, ref) < 1e-5
    assert ((dbeta.double() - sdz).abs() <= 1e-6 * mag0 + 1e-30).all()
    assert ((dgamma.double() - sdzx).abs() <= 1e-6 * mag1 + 1e-30).all()
    # accumulate_into: the skip connection's gradient plus exactly the fresh dx
    base = torch.randn(shape, device="cuda", generator=gen(8))
    acc, dgamma_a, dbeta_a = o.bn_bwd(da, x, mean, invstd, scale, shift, gamma, relu, accumulate_into=base.clone())
    torch.cuda.synchronize()
    assert torch.equal(acc, base + dx)
    assert torch.equal(dgamma_a, dgamma) and torch.equal(dbeta_a, dbeta)
    # an identity hook changes nothing
    seen = []
    dx_i, dgamma_i, dbeta_i = o.bn_bwd(da, x, mean, invstd, scale, shift, gamma, relu,
                                       sync_mean=lambda s: seen.append(s.numel()) or s)
    torch.cuda.synchronize()
    assert seen == [2 * shape[-1]]
    assert torch.equal(dx_i, dx) and torch.equal(dgamma_i, dgamma) and torch.equal(dbeta_i, dbeta)
    # a hook that scales the sums (the rank mean of sums that differ across ranks) moves only the statistics terms of dx
    alpha = 0.625
    dx_s, dgamma_s, dbeta_s = o.bn_bwd(da, x, mean, invstd, scale, shift, gamma, relu, sync_mean=lambda s: s * alpha)
    ref_s = _bn_bwd_ref(x, da, mean, invstd, gamma, pre, relu, alpha)[0]
    torch.cuda.synchronize()
    assert relerr(dx_s, ref_s) < 1e-5
    assert relerr(dx_s, ref) > 1e-4          # the hook's sums were used
    assert torch.equal(dgamma_s, dgamma) and torch.equal(dbeta_s, dbeta)


# ------------------------------------------------------------------------------------------------ reductions
def _rows_per_block(P, C):
    """Rows per block of the reductions' launch geometry (csrc/elementwise.cu red_geom)."""
    L = C // 4
    R = max(1, 256 // L)
    nb = min(max(1, -(-P // (R * 4))), 4 * 132)
    rpb = -(-P // nb)
    return -(-rpb // R) * R, R


def _red_rows(C):
    """1, 2, 3 rows; one row past the first block boundary; one row past the block cap's boundary; 2^21 + 5 rows for
    the narrow form (C = 4)."""
    R = _rows_per_block(1, C)[1]
    rows = [1, 2, 3, 4 * R + 1, 4 * 132 * 4 * R + 1]
    return rows + ([2 ** 21 + 5] if C == 4 else [])


RED_CASES = [(C, P) for C in (4, 1028, 2048, 4096) for P in _red_rows(C)]


def _with_fused(o, fused, fn):
    prev = o.FUSED_REDUCE
    o.FUSED_REDUCE = fused
    try:
        return fn()
    finally:
        o.FUSED_REDUCE = prev


@pytest.mark.parametrize("C,P", RED_CASES)
def test_bn_statistics(C, P):
    """bn_stats (two launches: partials, Chan merge) and bn_stats_finalize (partials, merge + finalize) with a large
    common-mode offset, against fp64."""
    o = ops()
    g = gen(9)
    x = (torch.randn(P, C, device="cuda", generator=g) * 0.3 + 25.0 + torch.randn(C, device="cuda", generator=g))
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g)
    rm = torch.randn(C, device="cuda", generator=g)
    rv = torch.rand(C, device="cuda", generator=g) + 0.5
    rm1, rv1 = rm.clone(), rv.clone()
    m2, v2 = o.bn_stats(x)
    m1, v1, scale, shift, invstd = o.bn_stats_finalize(x, gamma, beta, 1e-5, rm1, rv1, 0.1)
    xd = x.double()
    ref_m, ref_v = xd.mean(0), xd.var(0, unbiased=False)
    torch.cuda.synchronize()
    std = ref_v.sqrt()
    for m, v in ((m1, v1), (m2, v2)):
        # mean to the channel's std, allowing its own fp32 rounding
        assert (((m.double() - ref_m).abs() - ref_m.abs() * 6e-8).clamp_min(0) <= 2e-6 * std).all()
        if P == 1:
            assert torch.equal(v, torch.zeros_like(v))
        else:
            assert relerr(v, ref_v) < 1e-5
    ref_inv = 1.0 / (ref_v + 1e-5).sqrt()
    assert relerr(invstd, ref_inv) < 1e-5
    assert relerr(scale, gamma.double() * ref_inv) < 1e-5
    assert torch.equal(shift, beta)
    unb = ref_v * P / (P - 1) if P > 1 else ref_v
    assert relerr(rm1, 0.9 * rm.double() + 0.1 * ref_m) < 1e-6
    assert relerr(rv1, 0.9 * rv.double() + 0.1 * unb) < 1e-5


@pytest.mark.parametrize("C,P", RED_CASES)
def test_channel_sums(C, P):
    """channel_sum and bn_bwd_reduce (ReLU-masked sum dz and sum dz xhat) in both launch forms, against fp64."""
    o = ops()
    g = gen(10)
    dy = torch.randn(P, C, device="cuda", generator=g) + 3.0
    x = torch.randn(P, C, device="cuda", generator=g) * 0.5 + 25.0
    mean = x.double().mean(0).float()
    invstd = (1.0 / (x.double().var(0, unbiased=False) + 1e-5).sqrt()).float()
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.5
    pre = (x.double() - mean.double()) * scale.double() + shift.double()
    da = dy * (pre.abs() > 1e-4)
    ref_sum, mag_sum = dy.double().sum(0), dy.double().abs().sum(0)
    xh = (x.double() - mean.double()) * invstd.double()
    results = {}
    for fused in (True, False):
        results[fused] = (_with_fused(o, fused, lambda: o.channel_sum(dy)),
                          [_with_fused(o, fused, lambda: o.bn_bwd_reduce(da, x, mean, invstd, scale, shift, r))
                           for r in (True, False)])
    torch.cuda.synchronize()
    # the kernels add runs of 16 rows in fp32 and the runs in fp64: at most 15 fp32 roundings of partial sums, two more
    # in the product dz * xhat and one in the result, each <= 2^-24 of the channel's sum of magnitudes
    tol = 18 * 2.0 ** -24
    for fused, (s, sums) in results.items():
        assert ((s.double() - ref_sum).abs() <= tol * mag_sum).all(), (fused, C, P)
        for relu, r in zip((True, False), sums):
            dz = da.double() * (pre > 0) if relu else da.double()
            for part, want in ((r[:C], dz), (r[C:], dz * xh)):
                err = (part.double() - want.sum(0)).abs()
                assert (err <= tol * want.abs().sum(0) + 1e-30).all(), (fused, relu, C, P)


# ------------------------------------------------------------------------------------------------ max-pool ties
@pytest.mark.parametrize("C", [64, 256])
def test_maxpool2x2_ties_route_to_first_maximum(C):
    """Values from {0, 1, 2}: most windows tie. The forward is exact; the gradient goes to the first maximum in the
    window's row-major scan, as ATen's max_pool2d backward does."""
    o = ops()
    g = gen(11)
    B, H, W = 2, 16, 12
    x = torch.randint(0, 3, (B, H, W, C), device="cuda", generator=g).float()
    dy = torch.randn(B, H // 2, W // 2, C, device="cuda", generator=g)
    y = o.maxpool2x2(x)
    dx = o.maxpool2x2_bwd(x, dy)
    base = torch.randn(B, H, W, C, device="cuda", generator=g)
    dx_acc = o.maxpool2x2_bwd(x, dy, accumulate_into=base.clone())
    q = [x[:, 0::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 0::2], x[:, 1::2, 1::2]]
    m = torch.maximum(torch.maximum(q[0], q[1]), torch.maximum(q[2], q[3]))
    want = torch.zeros_like(x)
    taken = torch.zeros_like(m, dtype=torch.bool)
    for (dh, dw), v in zip(((0, 0), (0, 1), (1, 0), (1, 1)), q):
        first = (v == m) & ~taken
        want[:, dh::2, dw::2] = torch.where(first, dy, torch.zeros_like(dy))
        taken |= first
    xt = nchw(x).requires_grad_(True)
    (aten,) = torch.autograd.grad(F.max_pool2d(xt, 2), xt, nchw(dy))
    torch.cuda.synchronize()
    assert (m == 2).float().mean() < 0.9 and ((q[0] == q[1]) & (q[0] == m)).any()   # ties do occur
    assert torch.equal(y, m)
    assert torch.equal(dx, want)
    assert torch.equal(nchw(dx), aten)
    assert torch.equal(dx_acc, base + want)


# ------------------------------------------------------------------------------------------------ weight operands
def _tf32(t):
    """Round to tf32 (10 mantissa bits), to nearest with ties away from zero: the cvt.rna rounding of the kernels."""
    return ((t.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def _layout(w, for_dgrad):
    """[tap][O][I] (forward) or [flipped tap][I][O] (data gradient) of an OIHW weight."""
    O, I, k, _ = w.shape
    if for_dgrad:
        return w.flip(2, 3).permute(2, 3, 1, 0).reshape(k * k, I, O)
    return w.permute(2, 3, 0, 1).reshape(k * k, O, I)


WEIGHT_SHAPES = [(64, 32, 3), (48, 96, 3), (17, 32, 1), (256, 128, 1), (16, 48, 3)]


@pytest.mark.parametrize("for_dgrad", [False, True])
@pytest.mark.parametrize("shape", WEIGHT_SHAPES)
def test_weight_prep_tf32_layout_and_split(shape, for_dgrad):
    o = ops()
    O, I, k = shape
    w = torch.randn(O, I, k, k, device="cuda", generator=gen(12)) * 0.05
    hi, lo = o.weight_prep(w, for_dgrad=for_dgrad)
    hi1, lo1 = o.weight_prep(w, for_dgrad=for_dgrad, split=False)
    lay = _layout(w, for_dgrad)
    torch.cuda.synchronize()
    assert lo1 is None and torch.equal(hi1, hi)
    assert int((hi.view(torch.int32) & 0x1FFF).abs().max()) == 0
    assert int((lo.view(torch.int32) & 0x1FFF).abs().max()) == 0
    assert torch.equal(hi, _tf32(lay))
    assert torch.equal(lo, _tf32(lay - hi))
    assert ((hi.double() + lo.double() - lay.double()).abs() <= lay.double().abs() * 2.0 ** -21).all()


def _f16_split(lay):
    v = (lay * 256.0).clamp(-65504.0, 65504.0)
    hi = v.half()
    return hi, (v - hi.float()).half()


@pytest.mark.parametrize("for_dgrad", [False, True])
@pytest.mark.parametrize("shape", WEIGHT_SHAPES)
def test_weight_prep_f16_layout_and_split(shape, for_dgrad):
    o = ops()
    O, I, k = shape
    w = torch.randn(O, I, k, k, device="cuda", generator=gen(13)) * 0.05
    w[0, 0, 0, 0] = 300.0        # saturates at 65504 after the 2^8 pre-scale
    hi, lo = o.weight_prep_f16(w, for_dgrad=for_dgrad)
    hi1, lo1 = o.weight_prep_f16(w, for_dgrad=for_dgrad, split=False)
    want_hi, want_lo = _f16_split(_layout(w, for_dgrad))
    torch.cuda.synchronize()
    assert lo1 is None and torch.equal(hi1.view(torch.int16), hi.view(torch.int16))
    assert torch.equal(hi.view(torch.int16), want_hi.view(torch.int16))
    assert torch.equal(lo.view(torch.int16), want_lo.view(torch.int16))


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("shape", WEIGHT_SHAPES)
def test_weight_prep_f16_both_equals_separate_calls(shape, split):
    o = ops()
    O, I, k = shape
    w = torch.randn(O, I, k, k, device="cuda", generator=gen(14)) * 0.05
    (f_hi, f_lo), (d_hi, d_lo) = o.weight_prep_f16_both(w, split=split)
    sf = o.weight_prep_f16(w, split=split)
    sd = o.weight_prep_f16(w, for_dgrad=True, split=split)
    torch.cuda.synchronize()
    for got, want in ((f_hi, sf[0]), (d_hi, sd[0])) + (((f_lo, sf[1]), (d_lo, sd[1])) if split else ()):
        assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    if not split:
        assert f_lo is None and d_lo is None
    assert torch.equal(f_hi.view(torch.int16), _f16_split(_layout(w, False))[0].view(torch.int16))
    assert torch.equal(d_hi.view(torch.int16), _f16_split(_layout(w, True))[0].view(torch.int16))


# ------------------------------------------------------------------------------------------------ layouts
@pytest.mark.parametrize("shape", [(2, 3, 37, 29), (2, 64, 16, 12), (1, 17, 64, 48)])
def test_nchw_to_nhwc_flipw(shape):
    o = ops()
    x = torch.randn(shape, device="cuda", generator=gen(15))
    y = o.nchw_to_nhwc_flipw(x)
    torch.cuda.synchronize()
    assert torch.equal(y, nhwc(torch.flip(x, [3])))


@pytest.mark.parametrize("cfg", [(7, 2, 3, 3), (3, 2, 1, 3), (3, 2, 1, 5), (7, 2, 3, 4)])
@pytest.mark.parametrize("hw", [(37, 29), (64, 48)])
def test_im2col(cfg, hw):
    """Columns (kh, kw, ci) of each output pixel, zero outside the image and in the K padding, against F.unfold."""
    o = ops()
    k, s, p, Cin = cfg
    H, W = hw
    B = 2
    K = k * k * Cin
    kpad = (K + 31) // 32 * 32 + 4
    x = torch.randn(B, H, W, Cin, device="cuda", generator=gen(16))
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    cols = torch.full((B, Ho, Wo, kpad), float("nan"), device="cuda")
    o.im2col(x, k, s, p, kpad, out=cols)
    ref = F.unfold(nchw(x), k, padding=p, stride=s).view(B, Cin, k * k, Ho, Wo).permute(0, 3, 4, 2, 1)
    torch.cuda.synchronize()
    assert torch.equal(cols[..., :K], ref.reshape(B, Ho, Wo, K))
    assert torch.equal(cols[..., K:], torch.zeros_like(cols[..., K:]))


# ------------------------------------------------------------------------------------------------ CUDA-core convolutions
# (B, H, W, Cin, Cout, k, stride, pad), all with more than 24K weight floats: the global-memory weight path of the
# forward and data-gradient kernels
SIMT_SHAPES = [
    (2, 16, 12, 128, 256, 3, 2, 1),   # HRNet-w32 transition to the fourth branch
    (2, 16, 12, 192, 384, 3, 2, 1),   # HRNet-w48 transition
    (2, 32, 24, 64, 128, 3, 2, 1),    # w32 fuse: branch 1 -> 2
    (2, 64, 48, 48, 96, 3, 2, 1),     # w48 fuse: branch 0 -> 1
    (2, 9, 7, 128, 256, 3, 2, 1),     # odd input at stride 2
    (3, 11, 13, 96, 192, 3, 2, 1),
    (2, 9, 7, 192, 17, 3, 2, 1),      # 17 output channels
    (2, 8, 6, 17, 256, 3, 1, 1),      # 17 input channels (data gradient with 17 output channels)
]


@pytest.mark.parametrize("shape", SIMT_SHAPES)
def test_conv2d_simt_global_weight_path(shape):
    o = ops()
    B, H, W, Cin, Cout, k, s, p = shape
    assert k * k * Cin * ((Cout + 3) // 4 * 4) > 24 * 1024 and k * k * Cout * ((Cin + 3) // 4 * 4) > 24 * 1024
    g = gen(17)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (1.0 / (Cin * k * k) ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    y_ref = F.conv2d(nchw(x).double(), w.double(), bias.double(), stride=s, padding=p)
    res = torch.randn(nhwc(y_ref).shape, device="cuda", generator=g)
    dy = torch.randn(nhwc(y_ref).shape, device="cuda", generator=g)
    y = o.conv2d_simt_fwd(x, w, bias=bias, residual=res, stride=s, pad=p)
    dx = o.conv2d_simt_dgrad(dy, w, (H, W), stride=s, pad=p)
    dw = o.conv2d_simt_wgrad(x, dy, k, stride=s, pad=p)
    dx_ref = torch.nn.grad.conv2d_input((B, Cin, H, W), w.double(), nchw(dy).double(), stride=s, padding=p)
    dw_ref = torch.nn.grad.conv2d_weight(nchw(x).double(), w.shape, nchw(dy).double(), stride=s, padding=p)
    torch.cuda.synchronize()
    assert relerr(nchw(y), y_ref + nchw(res).double()) < 1e-5
    assert relerr(nchw(dx), dx_ref) < 1e-5
    assert relerr(dw, dw_ref) < 1e-5


# ------------------------------------------------------------------------------------------------ chunked weight gradient
# (B, H, W, Cin, Cout, k) at every split ops.wgrad_channel_chunks returns for the wide convolutions
CHUNKED = [((2, 16, 12, 256, 256, 3), (128, 256)),     # HRNet's 256-channel 3x3
           ((2, 8, 6, 2048, 1024, 3), (128, 256)),     # pose_resnet-50's first deconvolution as a 3x3 convolution
           ((2, 8, 6, 2048, 512, 1), (256, 512))]      # layer4's 2048 -> 512 1x1


@pytest.mark.parametrize("shape,chunks", CHUNKED)
def test_conv2d_wgrad_tc_chunked(shape, chunks):
    """dW of conv(relu((x - mean) * scale + shift)) one launch per channel chunk, BN parameters sliced, against fp64."""
    o = ops()
    B, H, W, Cin, Cout, k = shape
    assert o.wgrad_channel_chunks(Cin, Cout, k) == chunks
    g = gen(18)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g) * 2 + 0.5
    mean = torch.randn(Cin, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.5
    dy = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    dw = o.conv2d_wgrad_tc_chunked(x, dy, k, chunks, mean=mean, scale=scale, shift=shift, relu=True)
    a = _pre(x, mean, scale, shift).clamp_min(0.0)
    ref = torch.nn.grad.conv2d_weight(nchw(a), (Cout, Cin, k, k), nchw(dy).double(), padding=k // 2)
    torch.cuda.synchronize()
    assert relerr(dw, ref) < 2e-5, relerr(dw, ref)


# ------------------------------------------------------------------------------------------------ Adam
def test_adam_flat_weight_decay_and_grad_scale():
    """torch.optim.Adam(weight_decay=wd) in fp64 stepping on grad * grad_scale, over 10 steps, on an odd-sized buffer.

    The C ABI takes the hyper-parameters as fp32, so the reference gets the same fp32 values: 1 - float32(0.999) is
    1.3e-5 away from 0.001, which the second moment shows at that relative size."""
    o = ops()
    g = gen(19)
    n = 10007
    lr, b1, b2, eps, wd, gs = (torch.tensor(v, dtype=torch.float32).item() for v in (1e-2, 0.9, 0.999, 1e-8, 0.05, 0.25))
    p = torch.randn(n, device="cuda", generator=g) * 2
    m = torch.zeros_like(p)
    v = torch.zeros_like(p)
    ref = p.double().clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    for step in range(1, 11):
        gr = torch.randn(n, device="cuda", generator=g)
        ref.grad = gr.double() * gs
        opt.step()
        o.adam_flat(p, gr, m, v, lr, b1, b2, eps, wd, step, grad_scale=gs)
    torch.cuda.synchronize()
    st = opt.state[ref]
    assert relerr(m, st["exp_avg"]) < 1e-6
    assert relerr(v, st["exp_avg_sq"]) < 1e-6
    assert relerr(p, ref.detach()) < 1e-6
