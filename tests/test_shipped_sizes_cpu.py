"""The routes the networks take at the input sizes and joint counts the reference's experiments ship, recorded on the CPU.

tests/test_shipped_sizes_gpu.py checks these configurations against the oracle on the device. Here one training step
and one eval forward of each run through the launch recorder of tests/golden/make_dispatch_trace.py (no GPU, nothing
computed, planners answered for 132 SMs), and the test asserts which kinds of launch occur, not a golden trace:
  * hourglass f256 s4, 17 joints (fpd_coco), 256x192: the 256 -> 17 score and 17 -> 256 score_ convolutions fail the
    tensor-core shape checks (17 is not a multiple of 16, nor of 4) and run forward, data gradient and weight gradient on
    the CUDA cores; every other convolution runs on the tensor cores; the innermost level is 4x3. At inference
    precision "fp16_act" the score_ output is fp32, so the next stack's bottlenecks widen their input and residual:
    the launch counts of that mixed-dtype route are pinned, so that a change to it updates this test on purpose;
  * HRNet-w32 / -w48 at 384x288: branches at 96x72 .. 12x9 (odd width), the fuse step's 8x upsampling of 12x9, no
    stride-2 CUDA-core convolution, and (w48) CUDA-core weight gradients at 96x72;
  * pose_resnet-50 at 384x288: 2048-channel convolutions at 12x9 and the deconvolution head's depth-to-space from 12x9;
  * hourglass at 384x288, which no hourglass can run (12x9 max-pools to 6x4): the engine refuses it before any launch.
And ops.upsample2x_add / upsample2x_add_f16 refuse a `low` of the wrong shape.
"""
import collections
import importlib.util
import os

import pytest
import torch

_spec = importlib.util.spec_from_file_location(
    "make_dispatch_trace", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_dispatch_trace.py"))
T = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(T)

# position of B in a recorded launch ([name, *arguments], include/fpd_b200.h); H, W, Cin, Cout, k follow, and for the
# CUDA-core convolutions stride and pad after them
_B_AT = {"fpd_conv2d_tc_h": 15, "fpd_conv2d_tc_h_stats": 13, "fpd_conv2d_tc_ts": 13, "fpd_conv2d_tc_f16x1": 12,
         "fpd_conv2d_tc_f16x1_train": 13, "fpd_conv2d_tc_f16x1_io": 13, "fpd_conv2d_wgrad_tc_fused": 10,
         "fpd_conv2d_simt_fwd": 6, "fpd_conv2d_simt_dgrad": 4, "fpd_conv2d_simt_wgrad": 5}
_TC = ("fpd_conv2d_tc_h", "fpd_conv2d_tc_h_stats", "fpd_conv2d_tc_ts", "fpd_conv2d_tc_f16x1",
       "fpd_conv2d_tc_f16x1_train", "fpd_conv2d_tc_f16x1_io")
_SIMT = ("fpd_conv2d_simt_fwd", "fpd_conv2d_simt_dgrad", "fpd_conv2d_simt_wgrad")
Shape = collections.namedtuple("Shape", ("B", "H", "W", "Cin", "Cout", "k", "stride"))


def _shapes(calls, *names):
    out = []
    for c in calls:
        if c[0] in names:
            i = _B_AT[c[0]]
            out.append(Shape(*c[i:i + 6], c[i + 6] if "simt" in c[0] else 1))
    return out


def _hourglass(f, s, j, H, W):
    def make():
        from bench import cfg
        from fpd_b200.lib.models import hourglass as HG
        return HG.get_pose_net(cfg(f, s, j), False), (2, 3, H, W)
    return make


def _hrnet(width, H, W):
    def make():
        from bench import hrnet_cfg
        from fpd_b200.lib.models import pose_hrnet as HR
        return HR.get_pose_net(hrnet_cfg(width, j=17), False), (2, 3, H, W)
    return make


def _resnet(layers, H, W):
    def make():
        from bench import resnet_cfg
        from fpd_b200.lib.models import pose_resnet as R
        return R.get_pose_net(resnet_cfg(layers, j=17), False), (2, 3, H, W)
    return make


NETS = {"hg_f256_s4_j17": _hourglass(256, 4, 17, 256, 192), "hrnet_w32_384": _hrnet(32, 384, 288),
        "hrnet_w48_384": _hrnet(48, 384, 288), "resnet50_384": _resnet(50, 384, 288),
        "hg_f256_s4_j17_384": _hourglass(256, 4, 17, 384, 288)}


def _trace(name, mode, monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    monkeypatch.setitem(T.NETS, name, NETS[name])
    monkeypatch.setitem(T.MODES, "infer_fp16_act", ("fp32", "fp16_act", False, False))
    monkeypatch.setattr(ops, "_chk_f16", lambda t, name, dtypes=None: None)
    return T.trace("%s/%s/default" % (name, mode))


# ------------------------------------------------------------------------------------------------ hourglass, 17 joints
def _score_convs(shapes):
    return sorted((s.Cin, s.Cout) for s in shapes)


def test_hourglass_17_joints_training_step(monkeypatch):
    calls = _trace("hg_f256_s4_j17", "train_fp32", monkeypatch)
    # score.i (256 -> 17, four stacks) and score_.i (17 -> 256, three): forward, data gradient and weight gradient on
    # the CUDA cores, at the heat-map size, 1x1 stride 1; nothing else there
    score = [(256, 17)] * 4 + [(17, 256)] * 3
    for name in _SIMT:
        sh = _shapes(calls, name)
        assert _score_convs(sh) == sorted(score), (name, sh)
        assert all((s.B, s.H, s.W, s.k, s.stride) == (2, 64, 48, 1, 1) for s in sh), sh
    # score_.i adds the previous stack's residual stream in its forward epilogue
    assert [c[4] != "null" for c in calls if c[0] == "fpd_conv2d_simt_fwd"] == [False, True] * 3 + [False]
    # every other convolution on the tensor cores: no 17-channel side there
    tc = _shapes(calls, *_TC)
    assert tc and not [s for s in tc if 17 in (s.Cin, s.Cout)]
    wg = _shapes(calls, "fpd_conv2d_wgrad_tc_fused")
    assert wg and not [s for s in wg if 17 in (s.Cin, s.Cout)]
    # the innermost level: 3x3 convolutions at 4x3 (W = 3), forward and data gradient
    assert any((s.H, s.W, s.k) == (4, 3, 3) for s in tc), sorted({(s.H, s.W) for s in tc})
    assert any((s.H, s.W, s.k) == (4, 3, 3) for s in wg)
    assert sum(c[0] == "fpd_maxpool2x2_fwd" for c in calls) == 1 + 4 * 4


def test_hourglass_17_joints_eval_forward(monkeypatch):
    calls = _trace("hg_f256_s4_j17", "infer_fp32", monkeypatch)
    assert _score_convs(_shapes(calls, "fpd_conv2d_simt_fwd")) == sorted([(256, 17)] * 4 + [(17, 256)] * 3)
    tc = _shapes(calls, *_TC)
    assert tc and not [s for s in tc if 17 in (s.Cin, s.Cout)]
    assert any((s.H, s.W, s.k) == (4, 3, 3) for s in tc)


def test_hourglass_17_joints_fp16_act_mixed_dtype_route(monkeypatch):
    """"fp16_act" at 17 joints: the CUDA-core score_ convolution writes the residual stream in fp32, so from the second
    stack on every bottleneck sees an fp32 input or residual and takes act16_conv_form's "widen" branch. These counts
    pin that route (at 16 joints all 194 convolutions run on the fp16-activation kernel, tests/test_infer_f16_act_cpu.py);
    a change that keeps the stream in fp16 should update them on purpose."""
    calls = _trace("hg_f256_s4_j17", "infer_fp16_act", monkeypatch)
    n = collections.Counter(c[0] for c in calls)
    assert n["fpd_conv2d_tc_f16x1_io"] == 143
    assert n["fpd_conv2d_tc_f16x1"] == 44            # fp32 activations, widened input / residual
    assert n["fpd_half_to_float"] == 49
    assert n["fpd_conv2d_simt_fwd"] == 7
    assert (n["fpd_maxpool2x2_fwd"], n["fpd_maxpool2x2_fwd_f16"]) == (12, 5)
    assert (n["fpd_upsample2x_add"], n["fpd_upsample2x_add_f16"]) == (12, 4)
    for name in ("fpd_conv2d_tc_h", "fpd_conv2d_tc_h_stats", "fpd_conv2d_tc_ts", "fpd_affine_act"):
        assert n[name] == 0, name
    # the first stack runs in fp16 throughout: its pools and upsamples are the fp16 forms, and the fp32 ones start after
    # the first score_ convolution
    first_simt = next(i for i, c in enumerate(calls) if c[0] == "fpd_conv2d_simt_fwd")
    second_simt = next(i for i, c in enumerate(calls) if c[0] == "fpd_conv2d_simt_fwd" and i > first_simt)
    assert all(c[0] != "fpd_maxpool2x2_fwd" and c[0] != "fpd_upsample2x_add" for c in calls[:second_simt])
    assert all(c[0] != "fpd_maxpool2x2_fwd_f16" for c in calls[second_simt:])
    # the 17-channel convolutions stay on the CUDA cores
    assert not [s for s in _shapes(calls, "fpd_conv2d_tc_f16x1_io", "fpd_conv2d_tc_f16x1") if 17 in (s.Cin, s.Cout)]


# ------------------------------------------------------------------------------------------------ HRNet at 384x288
@pytest.mark.parametrize("width", [32, 48])
@pytest.mark.parametrize("mode", ["train_fp32", "infer_fp32"])
def test_hrnet_384x288_routes(width, mode, monkeypatch):
    calls = _trace("hrnet_w%d_384" % width, mode, monkeypatch)
    tc = _shapes(calls, *_TC)
    top = 8 * width
    # branch 3 at 12x9 (odd width) on the tensor cores: its BasicBlocks' 3x3 convolutions
    assert any((s.H, s.W, s.Cin, s.Cout, s.k) == (12, 9, top, top, 3) for s in tc), sorted({(s.H, s.W) for s in tc})
    # the fuse step into branch 0: 12x9 upsampled by 8 (shift 3) at 96x72
    fuse = [c for c in calls if c[0] == "fpd_fuse_sum"]
    assert any(c[7:9] == [96, 72] and 3 in c[2] for c in fuse), [c[2:] for c in fuse]
    assert not [c for c in fuse if c[7] * c[8] not in (96 * 72, 48 * 36, 24 * 18, 12 * 9)]
    # the stride-2 convolutions run forward at stride 1 on the tensor cores (the stem's conv1 too: conv2 at 192x144)
    assert not [s for s in _shapes(calls, "fpd_conv2d_simt_fwd") if s.stride == 2]
    assert any((s.H, s.W, s.k) == (192, 144, 3) for s in tc)
    if mode == "train_fp32":
        simt = _shapes(calls, "fpd_conv2d_simt_wgrad")
        at96 = [s for s in simt if (s.H, s.W) == (96, 72)]
        if width == 48:
            # branch 0's 48 -> 48 3x3 weight gradients at 96x72 on the CUDA cores
            assert sum((s.Cin, s.Cout, s.k, s.stride) == (48, 48, 3, 1) for s in at96) >= 4 * 8, at96
        wg = _shapes(calls, "fpd_conv2d_wgrad_tc_fused")
        assert any((s.H, s.W) == (12, 9) for s in wg)


# ------------------------------------------------------------------------------------------------ pose_resnet 384x288
@pytest.mark.parametrize("mode", ["train_fp32", "infer_fp32"])
def test_resnet50_384x288_routes(mode, monkeypatch):
    calls = _trace("resnet50_384", mode, monkeypatch)
    tc = _shapes(calls, *_TC)
    # layer4 at 12x9: 2048-channel convolutions on the tensor cores
    assert any((s.H, s.W) == (12, 9) and s.Cout == 2048 for s in tc)
    assert any((s.H, s.W) == (12, 9) and s.Cin == 2048 for s in tc)
    # the CUDA cores take only the 17-joint head (Cout % 16 != 0)
    assert _shapes(calls, "fpd_conv2d_simt_fwd") == [Shape(2, 96, 72, 256, 17, 1, 1)]
    # the first deconvolution: a 3x3 convolution at 12x9 to 4 x 256 channels, then depth-to-space to 24x18 (B, H, W, C
    # name the depth side)
    assert any((s.H, s.W, s.Cin, s.Cout, s.k) == (12, 9, 2048, 1024, 3) for s in tc)
    d2s = [c[3:8] for c in calls if c[0] == "fpd_depth_space2" and c[7] == 0]
    assert [2, 12, 9, 256, 0] in d2s, d2s
    # the stem pool at 192x144 and the stride-2 pick-first 1x1 of layer4's first block (24x18 picked to 12x9)
    assert [2, 192, 144, 64] in [c[3:7] for c in calls if c[0] == "fpd_maxpool3x3s2_fwd"]
    assert any((s.H, s.W, s.Cin, s.Cout, s.k) == (12, 9, 1024, 2048, 1) for s in tc)
    if mode == "train_fp32":
        assert any((s.H, s.W) == (12, 9) for s in _shapes(calls, "fpd_conv2d_wgrad_tc_fused"))


# ------------------------------------------------------------------------------------------------ refusals
def test_hourglass_384x288_refused_before_any_launch(monkeypatch):
    """12x9 max-pools to 6x4, which upsamples to 12x8: no hourglass runs 384x288 (the reference fails at up1 + up2).
    The engine refuses it before it launches anything, forks a side stream or starts a capture."""
    recs = []
    rec_cls = T._Recorder

    class Spy(rec_cls):
        def __init__(self, lib):
            super().__init__(lib)
            recs.append(self)
    monkeypatch.setattr(T, "_Recorder", Spy)
    for mode in ("train_fp32", "infer_fp32", "infer_fp16_act"):
        with pytest.raises(RuntimeError, match=r"384x288 .*hourglass level 1 at 12x9"):
            _trace("hg_f256_s4_j17_384", mode, monkeypatch)
        assert recs[-1].calls == []


def test_hourglass_input_size_check():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as HG
    from bench import cfg
    eng = HG.get_pose_net(cfg(64, 1, 17), False).engine()
    for H, W in ((256, 192), (256, 256), (128, 128), (64, 64), (255, 191)):
        eng.check_input_size(H, W)
    for H, W, where in ((384, 288, "hourglass level 1 at 12x9"), (288, 384, "hourglass level 1 at 9x12"),
                        (256, 160, "hourglass level 1 at 8x5"), (256, 200, "hourglass level 3 at 32x25"),
                        (260, 192, "hourglass level 4 at 65x48"), (258, 192, "the stem's max-pool at 129x96"),
                        (128, 96, "hourglass level 1 at 4x3")):
        with pytest.raises(RuntimeError, match="%dx%d input reaches %s" % (H, W, where)):
            eng.check_input_size(H, W)
    # HRNet and pose_resnet take any size
    T._hrnet()[0].engine().check_input_size(384, 287)
    T._resnet()[0].engine().check_input_size(383, 289)


def test_upsample2x_add_refuses_a_low_of_the_wrong_shape(monkeypatch):
    """Both forms read B, H, W and C from up1; a low that is not (B, H/2, W/2, C) would be read out of bounds or
    misaligned. They raise before the native call (CPU tensors: nothing is launched)."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    monkeypatch.setattr(ops, "_chk_f16", lambda t, name, dtypes=None: None)
    up1 = torch.zeros(2, 12, 8, 16)
    for low in (torch.zeros(2, 6, 5, 16), torch.zeros(2, 6, 4, 8), torch.zeros(1, 6, 4, 16), torch.zeros(2, 12, 8, 16),
                torch.zeros(2, 6, 4)):
        with pytest.raises(ValueError, match=r"low must be \(2, 6, 4, 16\)"):
            ops.upsample2x_add(up1, low)
        with pytest.raises(ValueError, match=r"low must be \(2, 6, 4, 16\)"):
            ops.upsample2x_add_f16(up1.half(), low.half())
