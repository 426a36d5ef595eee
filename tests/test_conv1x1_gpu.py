"""The weight-resident 1x1 path of the 3xFP16 forward / data-gradient convolution (pw_conv_wgmma_kernel,
csrc/conv_wgmma.cu): against a torch fp64 convolution, bit for bit against the staged kernel (ops.set_conv1x1), under
CUDA-graph replay, and which kernel runs for which call."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# B, H, W, Cin, Cout
SWEEP = [
    (3, 4, 4, 64, 64),       # 48 pixels: one partial tile over three images
    (5, 8, 8, 16, 48),       # 320 pixels, tiles span images; Cin below one channel block
    (2, 6, 12, 48, 96),      # Cin = 48: channels 48..63 of the block are zero
    (2, 19, 48, 96, 16),     # 1824 pixels; a full and a partial channel block
    (1, 37, 64, 128, 128),   # ragged last tile
    (2, 13, 64, 64, 192),    # two 96-column output slices
    (2, 9, 40, 256, 256),    # two 128-column slices, four channel blocks
    (1, 24, 32, 256, 48),
]

# every 1x1 shape of one hg_fpd step at 64x64 (batch 32), and the HRNet / ResNet-50 1x1 shapes whose weights fit
BENCH_SHAPES = [
    (32, 64, 64, 128, 256), (32, 64, 64, 256, 256), (32, 64, 64, 256, 128), (32, 64, 64, 128, 64),
    (32, 64, 64, 64, 128), (32, 64, 64, 256, 16), (32, 64, 64, 16, 256), (32, 64, 64, 128, 128),
    (32, 64, 64, 128, 16), (32, 64, 64, 16, 128), (32, 32, 32, 256, 128), (32, 32, 32, 128, 256),
    (32, 128, 128, 64, 128), (32, 128, 128, 32, 64),
    (24, 64, 48, 64, 256), (24, 64, 48, 256, 64), (24, 32, 24, 96, 48), (24, 16, 12, 192, 96),
    (32, 64, 64, 256, 64), (32, 64, 64, 64, 256), (32, 16, 16, 256, 1024), (32, 32, 32, 128, 512),
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


def ran(names):
    """'pw', 'staged', 'halo' or None: which convolution kernel the call launched (exactly one expected)."""
    kinds = set()
    for n in names:
        if "pw_conv_wgmma_kernel" in n:
            kinds.add("pw")
        elif "conv_wgmma_kernel" in n:
            kinds.add("staged")
        elif "conv_halo_kernel" in n:
            kinds.add("halo")
    assert len(kinds) <= 1, names
    return kinds.pop() if kinds else None


def on_both(fn):
    """fn() with the weight-resident kernel, then with the staged kernel."""
    o = ops()
    prev = o.set_conv1x1(True)
    try:
        a = fn()
        o.set_conv1x1(False)
        b = fn()
    finally:
        o.set_conv1x1(prev)
    torch.cuda.synchronize()
    return a, b


def forward_case(shape, seed, residual=True, relu_mask=False):
    B, H, W, Cin, Cout = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g) * 2 + 0.5
    mean = torch.randn(Cin, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.5 + 0.75
    w = torch.randn(Cout, Cin, 1, 1, device="cuda", generator=g) * (1.0 / Cin ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B, Cout, H, W, device="cuda", generator=g) if residual else None
    mask = torch.randn(B, H, W, Cout, device="cuda", generator=g) if relu_mask else None
    a = F.relu((x.double() - mean.double().view(1, -1, 1, 1)) * scale.double().view(1, -1, 1, 1)
               + shift.double().view(1, -1, 1, 1))
    ref = F.conv2d(a, w.double(), bias.double())
    if res is not None:
        ref = ref + res.double()
    if mask is not None:
        ref = ref * (nchw(mask) > 0).double()
    w_hi, w_lo = o.weight_prep_f16(w)
    xh = nhwc(x)
    rh = nhwc(res) if res is not None else None

    def run(out=None):
        return o.conv2d_tc_h(xh, w_hi, w_lo, 1, mean=mean, scale=scale, shift=shift, relu=True, bias=bias,
                             residual=rh, relu_mask=mask, out=out)
    return run, ref


@pytest.mark.parametrize("shape", SWEEP)
def test_conv1x1_forward_bn_relu_bias_residual(shape):
    run, ref = forward_case(shape, 101)
    y, y_staged = on_both(run)
    assert relerr(nchw(y), ref) < 3e-5, "%s rel err %.3e" % (shape, relerr(nchw(y), ref))
    assert torch.equal(y, y_staged), shape
    assert ran(kernel_names(run)) == "pw", shape


@pytest.mark.parametrize("shape", SWEEP[:4] + [(2, 16, 16, 128, 256)])
def test_conv1x1_forward_relu_mask(shape):
    run, ref = forward_case(shape, 505, residual=True, relu_mask=True)
    y, y_staged = on_both(run)
    assert relerr(nchw(y), ref) < 3e-5, "%s rel err %.3e" % (shape, relerr(nchw(y), ref))
    assert torch.equal(y, y_staged), shape


@pytest.mark.parametrize("shape", SWEEP[:5] + [(2, 16, 16, 256, 128)])
@pytest.mark.parametrize("mag", [1e-6, 1.0, 1e3])
def test_conv1x1_data_gradient_in_scale(shape, mag):
    """Data-gradient form: raw dY scaled by the power-of-two in_scale into the fp16 range, output masked by the forward
    activation (relu_mask) and scaled back."""
    B, H, W, Cin, Cout = shape     # forward Cin -> Cout; the data gradient runs Cout -> Cin
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(202)
    dy = torch.randn(B, H, W, Cout, device="cuda", generator=g) * mag
    w = torch.randn(Cout, Cin, 1, 1, device="cuda", generator=g) * (1.0 / Cin ** 0.5)
    act = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    ref = torch.nn.grad.conv2d_input((B, Cin, H, W), w.double(), nchw(dy).double())
    _, s = o.channel_sum(dy, want_amax=True)
    wd_hi, wd_lo = o.weight_prep_f16(w, for_dgrad=True)
    for mask in (None, act):
        run = lambda: o.conv2d_tc_h(dy, wd_hi, wd_lo, 1, in_scale=s, relu_mask=mask)   # noqa: E731
        da, da_staged = on_both(run)
        r = ref * (nchw(act) > 0).double() if mask is not None else ref
        assert relerr(nchw(da), r) < 3e-5, "%s mag %g rel err %.3e" % (shape, mag, relerr(nchw(da), r))
        assert torch.equal(da, da_staged), (shape, mag)
        assert ran(kernel_names(run)) == "pw", shape


@pytest.mark.parametrize("shape", BENCH_SHAPES)
def test_conv1x1_bench_shapes_bit_identical(shape):
    """The 1x1 shapes of the benchmark configurations: forward (BN + ReLU, bias, residual) and data-gradient form."""
    o = ops()
    run, _ = forward_case(shape, 606)
    y, y_staged = on_both(run)
    assert torch.equal(y, y_staged), shape
    B, H, W, Cin, Cout = shape
    g = torch.Generator(device="cuda").manual_seed(707)
    dy = torch.randn(B, H, W, Cin, device="cuda", generator=g) * 1e-4
    w = torch.randn(Cout, Cin, 1, 1, device="cuda", generator=g) * (1.0 / Cin ** 0.5)
    _, s = o.channel_sum(dy, want_amax=True)
    wd_hi, wd_lo = o.weight_prep_f16(w)
    d, d_staged = on_both(lambda: o.conv2d_tc_h(dy, wd_hi, wd_lo, 1, in_scale=s))
    assert torch.equal(d, d_staged), shape
    assert ran(kernel_names(run)) == "pw", shape


def pw_fits(Cin, Cout):
    """The kernel's shared-memory plan: 1 KB alignment + two 32 KB A stages + the slice's hi/lo weights <= 227 KB."""
    nt = Cout if Cout <= 128 else next(n for n in range(128, 15, -16) if Cout % n == 0)
    return 1024 + 2 * 32768 + (Cin + 63) // 64 * 2 * nt * 128 <= 227 * 1024


def test_conv1x1_plan_covers_bench_shapes():
    assert all(pw_fits(Cin, Cout) for (_, _, _, Cin, Cout) in BENCH_SHAPES)
    assert pw_fits(320, 128) and not pw_fits(384, 128) and not pw_fits(2048, 512)


def test_conv1x1_graph_replay():
    """The kernel inside a CUDA graph: replay gives the eager call's output bit for bit."""
    run, _ = forward_case((4, 32, 32, 128, 256), 808)
    eager = run()
    out = torch.empty_like(eager)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        run(out)
        with torch.cuda.graph(graph, stream=side):
            run(out)
    torch.cuda.current_stream().wait_stream(side)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_conv1x1_selection():
    """1x1 3xFP16 calls without statistics whose weights fit run the weight-resident kernel; statistics calls,
    single-pass fp16, 3xTF32, 3x3 and slices whose weights do not fit stay where they were."""
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(909)

    def names(B, H, W, Cin, Cout, k, split=True, f16=True, stats=False):
        x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
        w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * 0.05
        w_hi, w_lo = (o.weight_prep_f16 if f16 else o.weight_prep)(w, split=split)
        kw = {}
        if stats:
            nblk = int(o.N.lib().fpd_conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, k, int(f16)))
            kw = dict(stats_part=torch.empty(nblk, Cout, 2, dtype=torch.float64, device="cuda"),
                      stats_pivot=torch.zeros(Cout, device="cuda"))
        return ran(kernel_names(lambda: o.conv2d_tc_h(x, w_hi, w_lo, k, **kw)))

    assert names(2, 64, 64, 128, 256, 1) == "pw"
    assert names(2, 64, 64, 256, 256, 1) == "pw"
    assert names(2, 8, 8, 320, 128, 1) == "pw"                   # 5 channel blocks x 128 columns: 197 KB
    assert names(2, 8, 8, 384, 128, 1) == "staged"               # 6 channel blocks x 128 columns: does not fit
    assert names(2, 8, 8, 2048, 512, 1) == "staged"
    assert names(2, 64, 64, 128, 128, 1, stats=True) == "staged"
    assert names(2, 64, 64, 128, 128, 1, split=False) == "staged"
    assert names(2, 64, 64, 128, 128, 1, f16=False) == "staged"
    assert names(2, 64, 64, 128, 128, 3) == "halo"
    prev = o.set_conv1x1(False)
    try:
        assert names(2, 64, 64, 128, 256, 1) == "staged"
    finally:
        o.set_conv1x1(prev)
