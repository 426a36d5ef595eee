"""CPU suite for the single-pass FP16 inference precision: the host-only planner of ops.conv2d_tc_f16x1 over the forward
convolution shapes of the benchmark networks, and engine.set_inference_precision's contract."""
import types

import pytest
import torch

NS = types.SimpleNamespace


def _kind(B, H, W, Cin, Cout, k):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    return ops.conv2d_tc_f16x1_kernel(B, H, W, Cin, Cout, k)


def _hourglass_shapes(f):
    """(H, W, Cin, Cout, k) of the hourglass forward with NUM_FEATURES f at 256x256 (stem as im2col over 160 channels)."""
    stem, half = f // 4, f // 2
    s = [(128, 128, 160, stem, 1)]
    s += [(128, 128, stem, stem, 1), (128, 128, stem, stem, 3), (128, 128, stem, half, 1)]          # layer1 (+ skip)
    s += [(64, 64, half, half, 1), (64, 64, half, half, 3), (64, 64, half, f, 1)]                 # layer2 (+ skip)
    for hw in (64, 32, 16, 8, 4):                                                                 # layer3, hourglass
        s += [(hw, hw, f, half, 1), (hw, hw, half, half, 3), (hw, hw, half, f, 1)]
    s += [(64, 64, f, f, 1), (64, 64, f, 16, 1), (64, 64, 16, f, 1)]                              # fc, score, score_
    return s


def _hrnet_shapes(w):
    """HRNet-w{32,48} at 256x192: stem (3x3 stride 2 as im2col / stride-1 + pick), layer1, branches, transitions."""
    s = [(128, 96, 32, 64, 1), (128, 96, 64, 64, 3),
         (64, 48, 64, 64, 1), (64, 48, 64, 64, 3), (64, 48, 64, 256, 1), (64, 48, 256, 64, 1),
         (64, 48, 256, w, 3), (64, 48, 256, 2 * w, 3)]
    res = [(64, 48), (32, 24), (16, 12), (8, 6)]
    for i, (h, ww) in enumerate(res):
        c = w << i
        s.append((h, ww, c, c, 3))                                   # basic blocks
        if i > 0:
            s.append((h, ww, c, w, 1))                               # fuse up path: 1x1 to branch 0
        if i < 3:
            s.append((h, ww, c, 2 * c, 3))                           # fuse down path / transition (stride 2 as stride 1)
    return s


def _resnet50_shapes():
    s = [(128, 128, 160, 64, 1)]
    for (hw, cin, planes, n) in ((64, 64, 64, 3), (32, 256, 128, 4), (16, 512, 256, 6), (8, 1024, 512, 3)):
        out = planes * 4
        s += [(hw, hw, cin, planes, 1), (hw, hw, planes, planes, 3), (hw, hw, planes, out, 1), (hw, hw, cin, out, 1),
              (hw, hw, out, planes, 1)]
        if hw < 64:
            s.append((2 * hw, 2 * hw, planes, planes, 3))            # first block's stride-2 3x3 run at stride 1
    s += [(8, 8, 2048, 1024, 3), (16, 16, 256, 1024, 3), (32, 32, 256, 1024, 3)]   # deconv head as 3x3 convs
    return s


def _expected(H, W, Cin, Cout, k):
    """halo / 1x1 where hi-only operands fit in 227 KB of shared memory, staged otherwise."""
    nt = next(n for n in range(min(Cout, 128), 15, -16) if Cout % n == 0)
    ncb = (Cin + 63) // 64
    if k == 3:
        rows = 128 + 2 * W + 3
        return "halo" if 1024 + 3 * nt * 128 + ncb * rows * 128 + 48 <= 227 * 1024 else "staged"
    return "1x1" if 1024 + 3 * 16384 + ncb * nt * 128 <= 227 * 1024 else "staged"


@pytest.mark.parametrize("name,shapes", [("hg_student_f128", _hourglass_shapes(128)),
                                         ("hg_teacher_f256", _hourglass_shapes(256)),
                                         ("hrnet_w32", _hrnet_shapes(32)), ("hrnet_w48", _hrnet_shapes(48)),
                                         ("resnet50", _resnet50_shapes())])
def test_planner_on_benchmark_shapes(name, shapes):
    for (H, W, Cin, Cout, k) in shapes:
        assert _kind(32, H, W, Cin, Cout, k) == _expected(H, W, Cin, Cout, k), (name, H, W, Cin, Cout, k)
    # every hourglass and HRNet 3x3 takes the halo kernel, every 1x1 up to 640 input channels the resident one
    if not name.startswith("resnet"):
        assert all(_kind(32, *s) in ("halo", "1x1") for s in shapes), name


def test_planner_shapes_the_three_pass_kernels_cannot_take():
    assert _kind(8, 32, 128, 128, 128, 3) == "halo"     # W = 128, Cin = 128: 2 x 387 rows x 128 B of halo
    assert _kind(24, 8, 6, 384, 384, 3) == "halo"       # HRNet-w48's 384-channel branch
    assert _kind(8, 16, 16, 640, 128, 1) == "1x1"       # Cin = 640 at 128 columns
    assert _kind(8, 16, 16, 1024, 256, 1) == "staged"
    assert _kind(2, 8, 8, 2048, 1024, 3) == "staged"
    assert _kind(2, 64, 48, 32, 17, 1) is None          # 17-joint head: Cout % 16
    assert _kind(2, 64, 64, 3, 32, 7) is None
    assert _kind(2, 64, 64, 12, 32, 3) is None          # fp16 rows need Cin % 8 == 0
    assert _kind(70000, 256, 256, 64, 64, 3) is None    # 2^32 or more output elements


def _hourglass():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as H
    cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=1, NUM_BLOCKS=1), NUM_JOINTS=16))
    return H.get_pose_net(cfg, False)


def test_set_inference_precision_contract():
    from fpd_b200.engine import set_inference_precision
    net = _hourglass()
    eng = net.engine()
    g0 = eng.generation
    for bad in ("bf16", "FP16", None, 16):
        with pytest.raises(ValueError):
            set_inference_precision(net, bad)
    assert eng.generation == g0 and eng.inference_precision == "fp32"
    assert set_inference_precision(net, "fp16") == "fp32"
    assert eng.inference_precision == "fp16" and eng.generation == g0 + 1
    assert set_inference_precision(torch.nn.DataParallel(net), "fp16") == "fp16"   # no change: no bump
    assert eng.generation == g0 + 1
    assert set_inference_precision(torch.nn.DataParallel(net), "fp32") == "fp16"
    assert eng.inference_precision == "fp32" and eng.generation == g0 + 2
    with pytest.raises(TypeError):
        set_inference_precision(torch.nn.Conv2d(3, 3, 1), "fp16")


def test_eval_weights_follow_the_setting():
    """The cached eval operands are rebuilt after a change and know the precision they were made for."""
    from fpd_b200.engine import PreparedWeights, set_inference_precision
    net = _hourglass()
    eng = net.engine()
    eng._eval_cache = (PreparedWeights(3), {})
    eng._eval_cache_key = eng._param_version()
    set_inference_precision(net, "fp16")
    assert eng._eval_cache is None
    assert PreparedWeights(3, f16x1=True).f16x1 and not PreparedWeights(3).f16x1
