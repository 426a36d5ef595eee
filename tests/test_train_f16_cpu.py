"""CPU suite for the single-pass FP16 training precision: engine.set_training_precision's contract, and the host-only
planner of ops.conv2d_tc_f16x1 for training calls (with and without epilogue statistics) over every convolution shape
of the hg_fpd student, HRNet-w32 and pose_resnet-50 at their benchmark sizes."""
import types

import pytest
import torch

NS = types.SimpleNamespace
STAT_BYTES = 8 * 2 * 8            # per output channel: [8 warps][2] fp64


def _plan(B, H, W, Cin, Cout, k, stats):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    return ops.conv2d_tc_f16x1_train_plan(B, H, W, Cin, Cout, k, stats=stats)


def _hourglass_shapes(f):
    """(H, W, Cin, Cout, k, carries statistics in the step) of the hourglass student at 256x256."""
    stem, half = f // 4, f // 2
    s = [(128, 128, 160, stem, 1, False)]                                                    # im2col stem
    s += [(128, 128, stem, stem, 1, False), (128, 128, stem, stem, 3, True), (128, 128, stem, half, 1, False)]
    s += [(64, 64, half, half, 1, False), (64, 64, half, half, 3, True), (64, 64, half, f, 1, False)]
    for hw in (64, 32, 16, 8, 4):
        s += [(hw, hw, f, half, 1, False), (hw, hw, half, half, 3, True), (hw, hw, half, f, 1, False)]
    s += [(64, 64, f, f, 1, False), (64, 64, f, 16, 1, False), (64, 64, 16, f, 1, False)]
    return s


def _hrnet_shapes(w):
    s = [(128, 96, 64, 64, 3, True),                                                         # stem conv2 at stride 1
         (64, 48, 64, 64, 1, False), (64, 48, 64, 64, 3, True), (64, 48, 64, 256, 1, False),
         (64, 48, 256, 64, 1, False), (64, 48, 256, w, 3, True), (64, 48, 256, 2 * w, 3, True)]
    for i, (h, ww) in enumerate([(64, 48), (32, 24), (16, 12), (8, 6)]):
        c = w << i
        s.append((h, ww, c, c, 3, True))
        if i > 0:
            s.append((h, ww, c, w, 1, False))
        if i < 3:
            s.append((h, ww, c, 2 * c, 3, True))
    return s


def _resnet50_shapes():
    s = [(128, 128, 160, 64, 1, False)]
    for (hw, cin, planes) in ((64, 64, 64), (32, 256, 128), (16, 512, 256), (8, 1024, 512)):
        out = planes * 4
        s += [(hw, hw, cin, planes, 1, False), (hw, hw, planes, planes, 3, planes <= 256),
              (hw, hw, planes, out, 1, False), (hw, hw, cin, out, 1, False), (hw, hw, out, planes, 1, False)]
        if hw < 64:
            s.append((2 * hw, 2 * hw, planes, planes, 3, planes <= 256))
    s += [(8, 8, 2048, 1024, 3, False), (16, 16, 256, 1024, 3, False), (32, 32, 256, 1024, 3, False)]
    return s


def _expected(H, W, Cin, Cout, k, stats):
    """The plan written out: halo / 1x1 where the hi-only operands and the statistics scratch fit in 227 KB."""
    if stats and Cout > 256:
        return None
    nt = next(n for n in range(min(Cout, 128), 15, -16) if Cout % n == 0)
    ncb = (Cin + 63) // 64
    extra = STAT_BYTES * Cout if stats else 0
    if k == 3:
        rows = 128 + 2 * W + 3
        fits = any(1024 + st * nt * 128 + ncb * rows * 128 + extra + 16 * st <= 227 * 1024 for st in (4, 3))
        return "halo" if fits else "staged"
    return "1x1" if 1024 + 3 * 16384 + ncb * nt * 128 + extra <= 227 * 1024 else "staged"


BENCH = [("hg_student_f128", 32, _hourglass_shapes(128)), ("hrnet_w32", 24, _hrnet_shapes(32)),
         ("resnet50", 32, _resnet50_shapes())]


@pytest.mark.parametrize("name,B,shapes", BENCH)
def test_training_planner_on_benchmark_shapes(name, B, shapes):
    for (H, W, Cin, Cout, k, _) in shapes:
        for stats in (False, True):
            kind, nblk = _plan(B, H, W, Cin, Cout, k, stats)
            assert kind == _expected(H, W, Cin, Cout, k, stats), (name, H, W, Cin, Cout, k, stats)
            tiles = (B * H * W + 127) // 128 * (Cout // next(n for n in range(min(Cout, 128), 15, -16) if Cout % n == 0))
            assert nblk == (min(tiles, 132) if (stats and kind) else 0), (name, H, W, Cin, Cout, k, stats, nblk)


@pytest.mark.parametrize("name,B,shapes", BENCH)
def test_statistics_calls_of_the_step_take_the_single_pass_kernels(name, B, shapes):
    """Every convolution whose output feeds a train-mode BatchNorm through epilogue statistics today keeps them in
    "fp16", on the halo kernel (3x3) or the resident kernel (1x1) for the hourglass and HRNet."""
    for (H, W, Cin, Cout, k, carries) in shapes:
        if not carries:
            continue
        kind, nblk = _plan(B, H, W, Cin, Cout, k, True)
        assert kind is not None and nblk > 0, (name, H, W, Cin, Cout, k)
        if not name.startswith("resnet"):
            assert kind == ("halo" if k == 3 else "1x1"), (name, H, W, Cin, Cout, k, kind)
    for (H, W, Cin, Cout, k, _) in shapes:   # 1x1 statistics calls (FPD_CONV_STATS=1) fit the resident kernel too
        if k == 1 and Cout <= 256 and Cin <= 512 and not name.startswith("resnet"):
            assert _plan(B, H, W, Cin, Cout, k, True)[0] == "1x1", (name, H, W, Cin, Cout)


def test_halo_statistics_plan_keeps_four_stages_at_w64():
    """W = 64, Cin = Cout = 128: 1 KB + 4 x 16 KB of weights + 66,304 B of halo + 16 KB of statistics + 64 B of
    mbarriers = 149,312 B; W = 128 still takes the halo kernel with statistics."""
    assert 1024 + 4 * 16384 + 2 * (128 + 2 * 64 + 3) * 128 + STAT_BYTES * 128 + 64 == 149312
    assert _plan(32, 64, 64, 128, 128, 3, True)[0] == "halo"
    assert _plan(8, 128, 128, 128, 128, 3, True)[0] == "halo"
    assert _plan(8, 16, 16, 640, 256, 1, True)[0] == "staged"     # 1x1: 5 x 32 KB of weights + 32 KB of statistics
    assert _plan(8, 16, 16, 640, 256, 1, False)[0] == "1x1"
    assert _plan(8, 16, 16, 64, 512, 3, True) == (None, 0)        # statistics need Cout <= 256
    assert _plan(8, 16, 16, 64, 512, 3, False) == ("halo", 0)
    assert _plan(2, 64, 48, 32, 17, 1, True) == (None, 0)


def test_training_planner_agrees_with_the_inference_planner_without_statistics():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    for name, B, shapes in BENCH:
        for (H, W, Cin, Cout, k, _) in shapes:
            assert _plan(B, H, W, Cin, Cout, k, False)[0] == ops.conv2d_tc_f16x1_kernel(B, H, W, Cin, Cout, k)


def _hourglass():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as H
    cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=1, NUM_BLOCKS=1), NUM_JOINTS=16))
    return H.get_pose_net(cfg, False)


def test_set_training_precision_contract():
    from fpd_b200.engine import set_inference_precision, set_training_precision
    net = _hourglass()
    eng = net.engine()
    g0 = eng.generation
    for bad in ("bf16", "FP16", "tf32", None, 16):
        with pytest.raises(ValueError):
            set_training_precision(net, bad)
    assert eng.generation == g0 and eng.training_precision == "fp32"
    eng._eval_cache, eng._eval_cache_key = object(), object()
    assert set_training_precision(net, "fp16") == "fp32"
    assert eng.training_precision == "fp16" and eng.generation == g0 + 1 and eng._eval_cache is None
    assert eng.inference_precision == "fp32"                       # the two settings are independent
    assert set_training_precision(torch.nn.DataParallel(net), "fp16") == "fp16"   # no change: no bump
    assert eng.generation == g0 + 1
    assert set_inference_precision(net, "fp16") == "fp32" and eng.training_precision == "fp16"
    assert set_training_precision(torch.nn.DataParallel(net), "fp32") == "fp16"
    assert eng.training_precision == "fp32" and eng.inference_precision == "fp16" and eng.generation == g0 + 3
    for bad in (torch.nn.Conv2d(3, 3, 1), torch.nn.DataParallel(torch.nn.Linear(2, 2)), None):
        with pytest.raises(TypeError):
            set_training_precision(bad, "fp16")
