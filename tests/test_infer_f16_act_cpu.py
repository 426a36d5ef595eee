"""CPU suite for the fp16 activation storage of inference precision "fp16_act": engine.set_inference_precision's
contract, and, for every convolution of the benchmark hourglass and HRNet networks, the kernel and activation types the
engine's eval forward uses, recorded without a GPU by the launch recorder of tests/golden/make_dispatch_trace.py."""
import importlib.util
import os
import types

import pytest
import torch

NS = types.SimpleNamespace
_spec = importlib.util.spec_from_file_location(
    "make_dispatch_trace", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_dispatch_trace.py"))
T = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(T)

# argument positions of a recorded fpd_conv2d_tc_f16x1_io launch ([name, *arguments], include/fpd_b200.h)
_IO_X_F16, _IO_Y_F16, _IO_RES, _IO_B = 2, 11, 9, 13
# every launch of a convolution or of the fp32 eval glue that an "fp16_act" forward should not need
_FP32_ONLY = ("fpd_conv2d_tc_f16x1", "fpd_conv2d_tc_f16x1_train", "fpd_conv2d_tc_h", "fpd_conv2d_tc_h_stats",
              "fpd_conv2d_tc_ts", "fpd_affine_act", "fpd_affine_add_act", "fpd_fuse_sum", "fpd_maxpool2x2_fwd",
              "fpd_upsample2x_add", "fpd_subsample2")


def _hourglass(f, s):
    def make():
        from bench import cfg
        from fpd_b200.lib.models import hourglass as H
        return H.get_pose_net(cfg(f, s), False), (2, 3, 256, 256)
    return make


def _hrnet(w):
    def make():
        from bench import hrnet_cfg
        from fpd_b200.lib.models import pose_hrnet as H
        return H.get_pose_net(hrnet_cfg(w), False), (2, 3, 256, 192)
    return make


NETS = {"hg_s4_f128": _hourglass(128, 4), "hg_s8_f256": _hourglass(256, 8), "hrnet_w32": _hrnet(32),
        "hrnet_w48": _hrnet(48)}
# the calls that fall back to a widening conversion and an fp32-activation convolution, and why
EXPECTED_FALLBACKS = {
    "hg_s4_f128": [],
    "hg_s8_f256": [],
    # final_layer: the 17-joint 1x1 head (Cout % 16 != 0) runs on the CUDA-core convolution, which has no fp16 form
    "hrnet_w32": [("fpd_conv2d_simt_fwd", 32, 17, 1)],
    "hrnet_w48": [("fpd_conv2d_simt_fwd", 48, 17, 1)],
}


def _record(name, monkeypatch):
    """-> (recorded launches of one eval forward at "fp16_act", the engine's act16_conv_form answers in call order,
    the network)."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import engine, ops
    made = {}

    def make():
        made["net"], shape = NETS[name]()
        return made["net"], shape
    monkeypatch.setitem(T.NETS, name, make)
    monkeypatch.setitem(T.MODES, "infer_fp16_act", ("fp32", "fp16_act", False, False))
    monkeypatch.setattr(ops, "_chk_f16", lambda t, name, dtypes=None: None)
    forms = []
    form_fn = engine.act16_conv_form

    def spy(e, B, H, W, cin, k, out_f16, res_dtype=None):
        r = form_fn(e, B, H, W, cin, k, out_f16, res_dtype)
        forms.append((B, H, W, cin, e.hi.shape[1], k, r))
        return r
    monkeypatch.setattr(engine, "act16_conv_form", spy)
    return T.trace("%s/infer_fp16_act/default" % name), forms, made["net"]


@pytest.mark.parametrize("name", list(NETS))
def test_every_convolution_plans_its_kernel_and_activation_types(name, monkeypatch):
    from fpd_b200 import ops
    calls, forms, net = _record(name, monkeypatch)
    n_convs = sum(isinstance(m, torch.nn.Conv2d) for m in net.modules())
    io = [c for c in calls if c[0] == "fpd_conv2d_tc_f16x1_io"]
    widen = [c for c in calls if c[0] == "fpd_half_to_float"]
    simt = [c for c in calls if c[0] == "fpd_conv2d_simt_fwd"]
    assert not [c[0] for c in calls if c[0] in _FP32_ONLY]
    # every Conv2d runs once: on the fp16-activation single-pass kernels, or widened on an fp32-activation kernel
    assert len(io) + len(simt) == n_convs, (len(io), len(simt), n_convs)
    fallbacks = [(c[0], c[9], c[10], c[11]) for c in simt]     # (kernel, Cin, Cout, k)
    assert fallbacks == EXPECTED_FALLBACKS[name]
    assert len(widen) == len(simt)                             # one widening of the input per fallback
    # the host planner's answer for each tensor-core call is the launch the engine made
    assert len(forms) == len(io)
    for (B, H, W, cin, cout, k, (kind, out)), c in zip(forms, io):
        assert tuple(c[_IO_B:_IO_B + 6]) == (B, H, W, cin, cout, k)
        assert kind == ("halo" if k == 3 else "1x1") == ops.conv2d_tc_f16x1_kernel(B, H, W, cin, cout, k), c
        assert c[_IO_Y_F16] == int(out == torch.float16)
    # activation types: the stem reads the fp32 im2col columns, the hourglass score_ convs read the fp32 heat-map, the
    # heads write fp32; everything else reads and writes fp16, and a residual has the output's type
    stem_k = net.engine().convs["conv1"].im2col_kpad
    joints = 16 if name.startswith("hg") else 17
    x_types = [(c[16], c[_IO_X_F16]) for c in io]
    assert x_types[0] == (stem_k, 0)
    assert all(f == 1 for cin, f in x_types[1:] if cin != joints)
    assert all(f == 0 for cin, f in x_types[1:] if cin == joints)
    heads = [c for c in io if c[_IO_Y_F16] == 0]
    if name.startswith("hg"):
        stacks = int(name.split("_")[1][1:])
        assert [c[17] for c in heads] == [joints] * stacks and all(c[_IO_RES] == "null" for c in heads)
        assert sum(c[16] == joints for c in io) == stacks - 1        # score_: fp32 heat-map in, fp16 out
    else:
        assert heads == []                                           # the HRNet head is the CUDA-core fallback
    print("%s: %d convolutions, %d on the halo kernel, %d on the 1x1 kernel, %d widened (%s)" % (
        name, n_convs, sum(f[-1][0] == "halo" for f in forms), sum(f[-1][0] == "1x1" for f in forms), len(simt),
        fallbacks))


@pytest.mark.parametrize("name", ["hg_s4_f128", "hrnet_w32"])
def test_glue_is_fp16_and_outputs_fp32(name, monkeypatch):
    calls, _, _ = _record(name, monkeypatch)
    names = {c[0] for c in calls}
    if name.startswith("hg"):
        assert {"fpd_maxpool2x2_fwd_f16", "fpd_upsample2x_add_f16", "fpd_affine_act_f16"} <= names
    else:
        assert {"fpd_affine_act_f16", "fpd_affine_add_act_f16", "fpd_fuse_sum_f16", "fpd_subsample2_f16"} <= names


def _small_hourglass():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as H
    cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=1, NUM_BLOCKS=1), NUM_JOINTS=16))
    return H.get_pose_net(cfg, False)


def test_set_inference_precision_fp16_act_contract():
    from fpd_b200.engine import INFERENCE_PRECISIONS, PreparedWeights, set_inference_precision
    assert INFERENCE_PRECISIONS == ("fp32", "fp16", "fp16_act")
    for net in (_small_hourglass(), T._hrnet()[0]):
        eng = net.engine()
        g0 = eng.generation
        assert set_inference_precision(net, "fp16_act") == "fp32"
        assert eng.inference_precision == "fp16_act" and eng.generation == g0 + 1
        assert set_inference_precision(torch.nn.DataParallel(net), "fp16_act") == "fp16_act"   # no change: no bump
        assert eng.generation == g0 + 1
        assert set_inference_precision(torch.nn.DataParallel(net), "fp16") == "fp16_act"
        assert eng.generation == g0 + 2
        assert set_inference_precision(net, "fp16_act") == "fp16"
        assert eng.generation == g0 + 3
        for bad in ("fp16-act", "FP16_ACT", "fp8", None):
            with pytest.raises(ValueError):
                set_inference_precision(net, bad)
        assert eng.inference_precision == "fp16_act" and eng.generation == g0 + 3
        # the eval operands are the single-pass FP16 weights of "fp16", rebuilt after a change
        eng._eval_cache = (PreparedWeights(3), {})
        eng._eval_cache_key = eng._param_version()
        assert set_inference_precision(net, "fp32") == "fp16_act" and eng._eval_cache is None
    resnet = T._resnet()[0]
    for model in (resnet, torch.nn.DataParallel(resnet)):
        with pytest.raises(ValueError, match="hourglass.*HRNet"):
            set_inference_precision(model, "fp16_act")
    assert resnet.engine().inference_precision == "fp32"
    assert set_inference_precision(resnet, "fp16") == "fp32"          # the other settings still take a ResNet
    with pytest.raises(TypeError):
        set_inference_precision(torch.nn.Conv2d(3, 3, 1), "fp16_act")


def test_training_and_tape_forwards_never_store_fp16(monkeypatch):
    """At "fp16_act" a training forward and a tape-recording eval forward make the launches they make at "fp32"."""
    monkeypatch.setitem(T.MODES, "train_act", ("fp32", "fp16_act", True, True))
    monkeypatch.setitem(T.MODES, "eval_tape_act", ("fp32", "fp16_act", False, True))
    monkeypatch.setitem(T.MODES, "eval_tape_32", ("fp32", "fp32", False, True))
    for net in ("hourglass", "hrnet"):
        assert T.trace("%s/train_act/default" % net) == T.trace("%s/train_fp32/default" % net)
        assert T.trace("%s/eval_tape_act/default" % net) == T.trace("%s/eval_tape_32/default" % net)
