"""The halo kernel's weight ring (TMA loads into an mbarrier ring that runs across tiles, csrc/conv_wgmma.cu) against the
staged kernel (ops.set_conv_halo(False)), bit for bit: forward with BN affine + ReLU, bias and residual, the data
gradient with its input scale and ReLU mask, and the epilogue statistics, over the halo sweep and the 3x3 shapes of the
hg_fpd and hrnet_fpd benchmark models (one and two output slices, three and two weight stages, many tiles per CTA);
and the kernel under CUDA-graph replay."""
import pytest
import torch

from test_conv_halo_gpu import HALO_SHAPES

pytestmark = pytest.mark.gpu

# B, H, W, Cin, Cout: the 3x3 convolutions of hg_fpd (teacher f256: 128 channels, student f128: 64, the student's
# 128x128 stem stage) and hrnet_fpd (w32 and w48 branches at 64x48 .. 8x6, batch 24)
BENCH_SHAPES = [
    (32, 64, 64, 128, 128), (32, 32, 32, 128, 128), (32, 16, 16, 128, 128), (32, 8, 8, 128, 128),
    (32, 4, 4, 128, 128), (32, 64, 64, 64, 64), (32, 32, 32, 64, 64), (32, 4, 4, 64, 64), (32, 128, 128, 64, 64),
    (32, 128, 128, 32, 32),
    (24, 64, 48, 32, 32), (24, 32, 24, 64, 64), (24, 16, 12, 128, 128), (24, 8, 6, 256, 256),
    (24, 64, 48, 48, 48), (24, 32, 24, 96, 96), (24, 16, 12, 192, 192),
]


def ops():
    from fpd_b200 import ops as o
    return o


def kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type is not None and "cuda" in str(e.device_type).lower()]


def ran(names):
    kinds = {"halo" if "conv_halo_kernel" in n else "staged" for n in names if "conv_" in n and "_kernel" in n}
    assert len(kinds) == 1, names
    return kinds.pop()


def on_both(fn):
    """fn() on the halo kernel, then on the staged kernel; the kernel each ran on."""
    o = ops()
    prev = o.set_conv_halo(True)
    try:
        a = fn()
        ka = ran(kernel_names(fn))
        o.set_conv_halo(False)
        b = fn()
        kb = ran(kernel_names(fn))
    finally:
        o.set_conv_halo(prev)
    torch.cuda.synchronize()
    assert kb == "staged"
    return a, b, ka


def forward_case(shape, seed):
    B, H, W, Cin, Cout = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g) * 2 + 0.5
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (1.0 / (Cin * 9) ** 0.5)
    kw = dict(mean=torch.randn(Cin, device="cuda", generator=g), scale=torch.rand(Cin, device="cuda", generator=g) + 0.5,
              shift=torch.randn(Cin, device="cuda", generator=g) * 0.5 + 0.75, relu=True,
              bias=torch.randn(Cout, device="cuda", generator=g))
    res = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    w_hi, w_lo = o.weight_prep_f16(w)

    def run(out=None):
        return o.conv2d_tc_h(x, w_hi, w_lo, 3, residual=res, out=out, **kw)
    return run


def halo_fits(shape, stats=False):
    """conv_launch's plan with at least two weight stages."""
    B, H, W, Cin, Cout = shape
    nt = Cout if Cout <= 128 else next(n for n in range(128, 15, -16) if Cout % n == 0)
    smem = 1024 + 2 * 2 * nt * 128 + 2 * ((Cin + 63) // 64) * (128 + 2 * W + 3) * 128 + (128 * Cout if stats else 0) + 32
    return smem <= 227 * 1024


@pytest.mark.parametrize("shape", HALO_SHAPES + BENCH_SHAPES)
def test_halo_ring_forward_bit_identical(shape):
    y, y_staged, kind = on_both(forward_case(shape, 11))
    assert kind == ("halo" if halo_fits(shape) else "staged"), shape
    assert torch.equal(y, y_staged), shape


@pytest.mark.parametrize("shape", HALO_SHAPES + BENCH_SHAPES)
def test_halo_ring_data_gradient_bit_identical(shape):
    B, H, W, Cin, Cout = shape     # forward Cin -> Cout; the data gradient runs Cout -> Cin
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(12)
    dy = torch.randn(B, H, W, Cout, device="cuda", generator=g) * 1e-3
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (1.0 / (Cin * 9) ** 0.5)
    act = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    _, s = o.channel_sum(dy, want_amax=True)
    wd_hi, wd_lo = o.weight_prep_f16(w, for_dgrad=True)
    da, da_staged, kind = on_both(lambda: o.conv2d_tc_h(dy, wd_hi, wd_lo, 3, in_scale=s, relu_mask=act))
    assert kind == ("halo" if halo_fits((B, H, W, Cout, Cin)) else "staged"), shape
    assert torch.equal(da, da_staged), shape


@pytest.mark.parametrize("shape", [s for s in HALO_SHAPES + BENCH_SHAPES if s[4] <= 256])
def test_halo_ring_statistics_bit_identical(shape):
    B, H, W, Cin, Cout = shape
    o = ops()
    nblk = int(o.N.lib().fpd_conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, 3, 1))
    g = torch.Generator(device="cuda").manual_seed(13)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (1.0 / (Cin * 9) ** 0.5)
    kw = dict(mean=torch.randn(Cin, device="cuda", generator=g) * 0.1, scale=torch.rand(Cin, device="cuda", generator=g) + 0.5,
              shift=torch.randn(Cin, device="cuda", generator=g) * 0.1 + 0.2, relu=True,
              bias=torch.randn(Cout, device="cuda", generator=g), stats_pivot=torch.randn(Cout, device="cuda", generator=g))
    w_hi, w_lo = o.weight_prep_f16(w)
    parts = []

    def run():
        part = torch.full((nblk, Cout, 2), float("nan"), dtype=torch.float64, device="cuda")
        parts.append(part)
        return o.conv2d_tc_h(x, w_hi, w_lo, 3, stats_part=part, **kw)
    y, y_staged, kind = on_both(run)
    assert kind == ("halo" if halo_fits(shape, stats=True) else "staged"), shape
    assert torch.equal(y, y_staged), shape
    # parts: [halo call, halo profiled call, staged call, staged profiled call]
    assert torch.equal(parts[0], parts[2]), shape


@pytest.mark.parametrize("shape", [(32, 64, 64, 128, 128), (24, 8, 6, 256, 256), (2, 13, 64, 64, 192)])
def test_halo_ring_graph_replay(shape):
    """The kernel inside a CUDA graph: replay gives the eager call's output bit for bit."""
    run = forward_case(shape, 14)
    o = ops()
    prev = o.set_conv_halo(True)
    try:
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
        graph.replay()
        torch.cuda.synchronize()
    finally:
        o.set_conv_halo(prev)
    assert torch.equal(out, eager), shape
