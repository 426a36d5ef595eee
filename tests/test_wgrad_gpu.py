"""The tap-row weight-gradient kernel (wgrad_halo_kernel, csrc/conv_wgmma.cu): bit for bit against the per-tap kernel
(wgrad_wgmma_kernel, selected with ops.set_wgrad_halo(False)) over the weight-gradient shapes of the benchmark models,
under CUDA-graph replay, and which kernel runs for which call."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# B, H, W, Cin, Cout, k
MODEL_SHAPES = [
    # hg_fpd student (s4 f128), batch 32
    (32, 64, 64, 64, 64, 3), (32, 32, 32, 64, 64, 3), (32, 8, 8, 64, 64, 3), (32, 4, 4, 64, 64, 3),
    (32, 128, 128, 32, 32, 3), (32, 64, 64, 128, 64, 1), (32, 64, 64, 64, 128, 1), (32, 64, 64, 128, 128, 1),
    (32, 64, 64, 128, 16, 1), (32, 64, 64, 16, 128, 1), (32, 128, 128, 32, 64, 1),
    # hrnet_fpd student (w32), batch 24: branches 0-2 and a 256-wide chunk
    (24, 64, 48, 32, 32, 3), (24, 32, 24, 64, 64, 3), (24, 16, 12, 128, 128, 3), (24, 8, 6, 128, 256, 3),
    (24, 64, 48, 64, 256, 1), (24, 64, 48, 256, 64, 1), (24, 32, 24, 96, 48, 1),
    # res50_mse, batch 32: bottleneck 3x3s and chunks of the wide 1x1s
    (32, 64, 64, 64, 64, 3), (32, 32, 32, 128, 128, 3), (32, 16, 16, 128, 256, 3), (32, 64, 64, 256, 64, 1),
    (32, 16, 16, 256, 256, 1),
]

# small batches, ragged pixel counts, a single split, Cin 32 with stacked taps
EDGE_SHAPES = [
    (2, 64, 64, 64, 64, 3), (2, 64, 64, 128, 64, 1), (1, 5, 7, 64, 64, 3), (3, 9, 11, 32, 96, 3),
    (1, 3, 3, 128, 32, 3), (2, 13, 17, 32, 32, 3), (1, 1, 20, 64, 128, 3), (2, 7, 5, 192, 64, 1),
    (4, 4, 4, 32, 256, 3),
]


def ops():
    from fpd_b200 import ops as o
    return o


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type is not None and "cuda" in str(e.device_type).lower()]


def ran(names):
    """'halo', 'tap' or None: which weight-gradient kernel the call launched (exactly one kind expected)."""
    kinds = {"halo" if "wgrad_halo_kernel" in n else "tap" for n in names
             if "wgrad_halo_kernel" in n or "wgrad_wgmma_kernel" in n}
    assert len(kinds) <= 1, names
    return kinds.pop() if kinds else None


def on_both(fn):
    """fn() on the tap-row kernel, then on the per-tap kernel."""
    o = ops()
    prev = o.set_wgrad_halo(True)
    try:
        a = fn()
        o.set_wgrad_halo(False)
        b = fn()
    finally:
        o.set_wgrad_halo(prev)
    torch.cuda.synchronize()
    return a, b


def case(shape, seed, bn_relu, passes):
    B, H, W, Cin, Cout, k = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g) * 2 + 0.5
    dy = torch.randn(B, H, W, Cout, device="cuda", generator=g) * 1e-3
    kw = {}
    if bn_relu:
        kw = dict(mean=torch.randn(Cin, device="cuda", generator=g), scale=torch.rand(Cin, device="cuda", generator=g) + 0.5,
                  shift=torch.randn(Cin, device="cuda", generator=g) * 0.5, relu=True)

    def run():
        return o.conv2d_wgrad_tc_fused(x, dy, k, passes=passes, **kw)
    return run


def supported(shape):
    return ops().conv2d_wgrad_tc_supported(shape[3], shape[4], shape[5])


@pytest.mark.parametrize("shape", MODEL_SHAPES)
@pytest.mark.parametrize("bn_relu", [True, False])
def test_wgrad_model_shapes_bit_identical(shape, bn_relu):
    assert supported(shape), shape
    run = case(shape, 11, bn_relu, 3)
    a, b = on_both(run)
    assert torch.equal(a, b), (shape, bn_relu, (a - b).abs().max().item())


@pytest.mark.parametrize("shape", EDGE_SHAPES + MODEL_SHAPES[:6])
@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("bn_relu", [True, False])
def test_wgrad_passes_and_edges_bit_identical(shape, passes, bn_relu):
    assert supported(shape), shape
    run = case(shape, 23, bn_relu, passes)
    a, b = on_both(run)
    assert torch.equal(a, b), (shape, passes, bn_relu, (a - b).abs().max().item())


@pytest.mark.parametrize("shape", [(2, 64, 64, 64, 64, 3), (2, 64, 64, 128, 64, 1)])
def test_wgrad_halo_against_fp64(shape):
    """The tap-row kernel against an fp64 torch weight gradient of conv(relu(bn_affine(x)))."""
    B, H, W, Cin, Cout, k = shape
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g)
    dy = torch.randn(B, Cout, H, W, device="cuda", generator=g)
    mean, scale, shift = (torch.randn(Cin, device="cuda", generator=g) for _ in range(3))
    a = F.relu((x.double() - mean.double().view(1, -1, 1, 1)) * scale.double().view(1, -1, 1, 1)
               + shift.double().view(1, -1, 1, 1))
    ref = torch.nn.grad.conv2d_weight(a, (Cout, Cin, k, k), dy.double(), padding=k // 2)
    prev = o.set_wgrad_halo(True)
    try:
        dw = o.conv2d_wgrad_tc_fused(nhwc(x), nhwc(dy), k, mean=mean, scale=scale, shift=shift, relu=True)
    finally:
        o.set_wgrad_halo(prev)
    torch.cuda.synchronize()
    err = ((dw.double() - ref).abs().max() / ref.abs().max()).item()
    assert err < 2e-5, (shape, err)


def test_wgrad_halo_graph_replay():
    """The kernel inside a CUDA graph: replay gives the eager call's output bit for bit."""
    o = ops()
    run = case((4, 32, 32, 64, 64, 3), 31, True, 3)
    prev = o.set_wgrad_halo(True)
    try:
        eager = run().clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side):
            run()
            with torch.cuda.graph(graph, stream=side):
                out = run()
        torch.cuda.current_stream().wait_stream(side)
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
    finally:
        o.set_wgrad_halo(prev)
    assert torch.equal(out, eager)


SELECTION = [
    # (B, H, W, Cin, Cout, k), kernel with the switch on
    ((2, 16, 16, 64, 64, 3), "halo"), ((2, 16, 16, 32, 32, 3), "halo"), ((2, 16, 16, 128, 256, 3), "halo"),
    ((2, 16, 16, 128, 64, 1), "halo"), ((2, 16, 16, 256, 32, 1), "halo"), ((2, 16, 16, 128, 128, 1), "tap"),
    ((2, 16, 16, 64, 96, 1), "tap"), ((2, 16, 16, 128, 16, 1), "tap"), ((2, 16, 16, 16, 128, 1), "tap"),
    ((2, 16, 16, 96, 48, 1), "tap"),
]


def _selection_main():
    import json
    o = ops()
    out = []
    for on in (True, False):
        o.set_wgrad_halo(on)
        for shape, _ in SELECTION:
            run = case(shape, 41, True, 3)
            run()                                   # first launch outside the trace
            out.append(ran(kernel_names(run)))
    print(json.dumps(out))


def test_wgrad_selection():
    """Every 3x3 shape and the 1x1 shapes with Cin % 64 == 0 and Cout in {32, 64} run the tap-row kernel; the other 1x1
    shapes, and every shape with the switch off, run the per-tap kernel. Traced in a fresh process: late in a long
    test session the profiler has returned no kernel events at all for such a call."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = "import sys; sys.path[:0] = [%r, %r]; import test_wgrad_gpu as t; t._selection_main()" % (
        here, os.path.dirname(here))
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    kinds = json.loads(res.stdout.strip().splitlines()[-1])
    want = [k for _, k in SELECTION] + ["tap"] * len(SELECTION)
    assert kinds == want, list(zip([s for s, _ in SELECTION] * 2, kinds, want))
