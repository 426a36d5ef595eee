"""Feature distillation on the host: the adapter's widths and initialisation, the student's state_dict keys, every
argument and configuration error of FPDTrainStep and fpd_train, the arguments fpd_train hands to each fused route, and
the host checks of the fpd_feature_mse entry point (no GPU needed)."""
import ctypes
import os
import sys
import types

import pytest
import torch

NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fpd_b200  # noqa: E402,F401

BAD_WEIGHTS = [float("nan"), float("inf"), -float("inf"), -1e-3, "0.1", True, None]


def _hg(feat, stacks, joints=16):
    from fpd_b200.lib.models import hourglass as H
    return H.get_pose_net(NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=feat, NUM_STACKS=stacks, NUM_BLOCKS=1),
                                      NUM_JOINTS=joints)), False)


def _hrnet(w):
    from fpd_b200.lib.models import pose_hrnet as H

    class Cfg(dict):
        def __getattr__(self, k):
            try:
                return self[k]
            except KeyError:
                raise AttributeError(k)

    def wrap(d):
        return Cfg({k: wrap(v) for k, v in d.items()}) if isinstance(d, dict) else d

    def stage(nmod, chans):
        return dict(NUM_MODULES=nmod, NUM_BRANCHES=len(chans), BLOCK='BASIC', NUM_BLOCKS=[1] * len(chans),
                    NUM_CHANNELS=chans, FUSE_METHOD='SUM')
    st = (stage(1, [w, 2 * w]), stage(1, [w, 2 * w, 4 * w]), stage(1, [w, 2 * w, 4 * w, 8 * w]))
    return H.get_pose_net(wrap(dict(MODEL=dict(NUM_JOINTS=17, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=dict(
        PRETRAINED_LAYERS=['*'], FINAL_CONV_KERNEL=1, STAGE2=st[0], STAGE3=st[1], STAGE4=st[2])))), is_train=False)


def _resnet():
    from fpd_b200.lib.models import pose_resnet as R
    cfg = NS(MODEL=NS(NUM_JOINTS=17, EXTRA=NS(NUM_LAYERS=18, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[32, 32, 32],
                                              NUM_DECONV_KERNELS=[4, 4, 4], FINAL_CONV_KERNEL=1, DECONV_WITH_BIAS=False),
                      INIT_WEIGHTS=False, PRETRAINED=''))
    return R.get_pose_net(cfg, is_train=False)


# ------------------------------------------------------------------------------------------------ adapter
@pytest.mark.parametrize("pair, widths", [(("hg", 128, 4, "hg", 256, 8), (128, 256)),
                                          (("hr", 32, "hr", 48), (32, 48)),
                                          (("hg", 64, 1, "hg", 256, 8), (64, 256))])
def test_adapter_infers_the_widths_of_the_shipped_pairs(pair, widths):
    from fpd_b200.train_step import FeatureAdapter, head_feature_channels
    if pair[0] == "hg":
        s, t = _hg(pair[1], pair[2]), _hg(pair[4], pair[5])
    else:
        s, t = _hrnet(pair[1]), _hrnet(pair[3])
    assert (head_feature_channels(s), head_feature_channels(t)) == widths
    torch.manual_seed(0)
    a = FeatureAdapter(s, t)
    c = a.conv
    assert (c.in_channels, c.out_channels, c.kernel_size, c.stride, c.padding) == (*widths, (1, 1), (1, 1), (0, 0))
    assert c.bias is not None and torch.equal(c.bias, torch.zeros(widths[1]))
    w = c.weight.detach()
    assert abs(float(w.std()) - 0.001) < 2e-4 and abs(float(w.mean())) < 1e-4
    assert [k for k, _ in a.state_dict().items()] == ["conv.weight", "conv.bias"]


def test_student_state_dict_keys_are_unchanged():
    from fpd_b200.train_step import FeatureAdapter
    s, t = _hg(64, 2), _hg(128, 1)
    keys = list(s.state_dict().keys())
    FeatureAdapter(s, t)
    assert list(s.state_dict().keys()) == keys
    assert not any(k.startswith("conv.") and "adapter" in k for k in keys)


def test_resnet_has_no_head_feature():
    from fpd_b200.train_step import FeatureAdapter, head_feature_channels
    r = _resnet()
    with pytest.raises(ValueError, match="PoseResNet"):
        head_feature_channels(r)
    with pytest.raises(ValueError, match="PoseResNet"):
        FeatureAdapter(r, _hg(64, 1))
    with pytest.raises(ValueError, match="PoseResNet"):
        FeatureAdapter(_hg(64, 1), r)


# ------------------------------------------------------------------------------------------------ FPDTrainStep errors
def test_train_step_refuses_bad_feature_arguments(monkeypatch):
    from fpd_b200.train_step import FeatureAdapter, FPDTrainStep
    s, t = _hg(64, 1), _hg(128, 1)
    a = FeatureAdapter(s, t)
    for bad in BAD_WEIGHTS:
        with pytest.raises(ValueError, match="feature_weight"):
            FPDTrainStep(s, t, feature_weight=bad, feature_adapter=a)
    with pytest.raises(ValueError, match="teacher"):
        FPDTrainStep(s, None, feature_weight=0.1, feature_adapter=a)
    with pytest.raises(ValueError, match="feature_adapter"):
        FPDTrainStep(s, t, feature_weight=0.1)
    with pytest.raises(ValueError, match="64 -> 128 channels"):
        FPDTrainStep(_hg(128, 1), t, feature_weight=0.1, feature_adapter=a)      # student width differs
    with pytest.raises(ValueError, match="64 -> 128 channels"):
        FPDTrainStep(s, _hg(256, 1), feature_weight=0.1, feature_adapter=a)      # teacher width differs
    with pytest.raises(ValueError, match="1x1"):
        FPDTrainStep(s, t, feature_weight=0.1, feature_adapter=torch.nn.Conv2d(64, 128, 1))
    with pytest.raises(ValueError, match="PoseResNet"):
        FPDTrainStep(_resnet(), t, feature_weight=0.1, feature_adapter=a)
    with pytest.raises(ValueError, match="PoseResNet"):
        FPDTrainStep(s, _resnet(), feature_weight=0.1, feature_adapter=a)
    monkeypatch.setenv("FPD_PIPELINE_TEACHER", "1")
    with pytest.raises(ValueError, match="FPD_PIPELINE_TEACHER"):
        FPDTrainStep(s, t, feature_weight=0.1, feature_adapter=a)


def test_weight_zero_builds_nothing(monkeypatch):
    """feature_weight=0 (with or without an adapter) keeps the flat buffers the student's alone."""
    from fpd_b200.train_step import FeatureAdapter, FlatParams, FPDTrainStep
    seen = []
    orig = FlatParams.__init__

    def rec(self, net, rehome=True, extra=None):
        seen.append(extra)
        raise RuntimeError("stop")
    monkeypatch.setattr(FlatParams, "__init__", rec)
    s, t = _hg(64, 1), _hg(128, 1)
    for kw in ({}, {"feature_weight": 0.0}, {"feature_weight": 0, "feature_adapter": FeatureAdapter(s, t)}):
        with pytest.raises(RuntimeError, match="stop"):
            FPDTrainStep(s, t, **kw)
    assert seen == [None, None, None]
    monkeypatch.setattr(FlatParams, "__init__", orig)
    a = FeatureAdapter(s, t)
    fp = FlatParams(s, rehome=True, extra=a)
    n_s = len(list(s.parameters()))
    assert fp.params[:n_s] == list(s.parameters()) and fp.params[n_s:] == [a.conv.weight, a.conv.bias]
    assert fp.numel == FlatParams(_hg(64, 1), rehome=False).numel + 64 * 128 + 128


# ------------------------------------------------------------------------------------------------ fpd_train
def _cfg(**kd):
    return NS(KD=NS(ALPHA=0.5, **kd), PRINT_FREQ=1, DEBUG=NS(DEBUG=False))


def _crit(kind="mse", use_tw=True):
    from fpd_b200.lib.core.loss import JointsKLDLoss, JointsMSELoss, JointsOHKMMSELoss
    return {"mse": lambda: JointsMSELoss(use_tw), "ohkm": lambda: JointsOHKMMSELoss(use_tw, topk=6),
            "kl": lambda: JointsKLDLoss(use_tw, temperature=0.5)}[kind]()


def test_config_key_absent_means_off():
    from fpd_b200.lib.core import function as F
    assert F._feature_weight(NS()) == 0.0
    assert F._feature_weight(NS(KD=NS(ALPHA=0.5))) == 0.0
    assert F._feature_weight(NS(KD=NS(ALPHA=0.5, FEATURE_WEIGHT=0.25))) == 0.25
    for bad in BAD_WEIGHTS:
        with pytest.raises(ValueError, match="feature_weight"):
            F._feature_weight(NS(KD=NS(FEATURE_WEIGHT=bad)))


def test_fpd_train_refuses_bad_feature_setups(monkeypatch):
    from fpd_b200.lib.core import function as F
    from fpd_b200.train_step import FeatureAdapter
    s, t = _hg(64, 1), _hg(128, 1)
    a = FeatureAdapter(s, t)
    opt_without = torch.optim.Adam(s.parameters())
    opt_with = torch.optim.Adam(s.parameters())
    opt_with.add_param_group({"params": a.parameters()})
    for bad in BAD_WEIGHTS:
        with pytest.raises(ValueError, match="feature_weight"):
            F.fpd_train(_cfg(FEATURE_WEIGHT=bad), [], s, t, _crit(), _crit(), opt_with, 0, "", "", None,
                        feature_adapter=a)
    with pytest.raises(ValueError, match="feature_adapter"):
        F.fpd_train(_cfg(FEATURE_WEIGHT=0.1), [], s, t, _crit(), _crit(), opt_with, 0, "", "", None)
    with pytest.raises(ValueError, match="param_groups"):
        F.fpd_train(_cfg(FEATURE_WEIGHT=0.1), [], s, t, _crit(), _crit(), opt_without, 0, "", "", None,
                    feature_adapter=a)
    with pytest.raises(ValueError, match="PoseResNet"):
        F.fpd_train(_cfg(FEATURE_WEIGHT=0.1), [], _resnet(), t, _crit(), _crit(), opt_with, 0, "", "", None,
                    feature_adapter=a)
    with pytest.raises(ValueError, match="channels"):
        F.fpd_train(_cfg(FEATURE_WEIGHT=0.1), [], s, _hg(256, 1), _crit(), _crit(), opt_with, 0, "", "", None,
                    feature_adapter=a)
    # criteria the fused routes do not take: the generic autograd route
    with pytest.raises(ValueError, match="generic autograd route"):
        F.fpd_train(_cfg(FEATURE_WEIGHT=0.1), [], s, t, torch.nn.MSELoss(), _crit(), opt_with, 0, "", "", None,
                    feature_adapter=a)
    with pytest.raises(ValueError, match="generic autograd route"):
        F.fpd_train(_cfg(FEATURE_WEIGHT=0.1), [], s, t, _crit(use_tw=False), _crit(), opt_with, 0, "", "", None,
                    feature_adapter=a)
    # heat-maps the fused loss kernels do not take (h*w % 64 != 0): refused at the first batch
    batch = [(torch.zeros(2, 3, 20, 20), torch.zeros(2, 16, 5, 5), torch.ones(2, 16, 1), {})]
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *args, **k: self)
    with pytest.raises(ValueError, match="generic autograd route"):
        F.fpd_train(_cfg(FEATURE_WEIGHT=0.1), batch, s, t, _crit(), _crit(), opt_with, 0, "", "", None,
                    feature_adapter=a)
    # off: no adapter needed, and an adapter outside the optimizer is ignored
    F.fpd_train(_cfg(), [], s, t, _crit(), _crit(), opt_without, 0, "", "", None)
    F.fpd_train(_cfg(FEATURE_WEIGHT=0.0), [], s, t, _crit(), _crit(), opt_without, 0, "", "", None, feature_adapter=a)


class _Stop(Exception):
    pass


@pytest.mark.parametrize("kd", [{}, {"FEATURE_WEIGHT": 0.0}, {"FEATURE_WEIGHT": 0.3}])
@pytest.mark.parametrize("graph", [True, False])
def test_fpd_train_passes_the_feature_term_only_when_on(kd, graph, monkeypatch):
    from fpd_b200 import train_step
    from fpd_b200.lib.core import function as F
    s, t = _hg(64, 1), _hg(128, 1)
    a = train_step.FeatureAdapter(s, t)
    opt = torch.optim.Adam(list(s.parameters()) + list(a.parameters()))
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *args, **k: self)
    monkeypatch.setattr(F, "_TRAIN_GRAPH", graph)
    seen = []

    class RecStep:
        def __init__(self, *args, **k):
            seen.append(("FPDTrainStep", args[2:], k))
            raise _Stop

    def rec_fused(*args, **k):
        seen.append(("_fused_step", args[5:], k))
        raise _Stop
    monkeypatch.setattr(train_step, "FPDTrainStep", RecStep)
    monkeypatch.setattr(F, "_fused_step", rec_fused)
    F._train_step_cache.clear()
    batch = [(torch.zeros(2, 3, 256, 256), torch.zeros(2, 16, 64, 64), torch.ones(2, 16, 1), {})]
    with pytest.raises(_Stop):
        F.fpd_train(_cfg(**kd), batch, s, t, _crit("ohkm"), _crit("kl"), opt, 0, "", "", None, feature_adapter=a)
    on = kd.get("FEATURE_WEIGHT", 0.0) > 0
    extra = {"feature_weight": 0.3, "feature_adapter": a} if on else {}
    if graph:
        assert seen == [("FPDTrainStep", (), {"alpha": 0.5, "fused_adam": False, "accuracy": True, "pose_topk": 6,
                                              "kd_temperature": 0.5, **extra})]
    else:
        assert len(seen) == 1 and seen[0][0] == "_fused_step"
        assert seen[0][2] == {"pose_topk": 6, "kd_temperature": 0.5, **extra}


def test_graph_cache_key_includes_weight_and_adapter(monkeypatch):
    from fpd_b200 import train_step
    from fpd_b200.lib.core import function as F
    made = []

    class FakeStep:
        def __init__(self, *args, **k):
            made.append(k)
            self.params, self.grad_views = [], []
    monkeypatch.setattr(train_step, "FPDTrainStep", FakeStep)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    orig_empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, pin_memory=False, **k: orig_empty(*a, **k))

    class Ev:
        pass
    monkeypatch.setattr(torch.cuda, "Event", Ev)
    s, t = _hg(64, 1), _hg(128, 1)
    a1, a2 = train_step.FeatureAdapter(s, t), train_step.FeatureAdapter(s, t)
    x, tg, tw = torch.zeros(2, 3, 256, 256), torch.zeros(2, 16, 64, 64), torch.ones(2, 16, 1)
    F._train_step_cache.clear()
    for w, a in ((0.0, None), (0.1, a1), (0.1, a1), (0.2, a1), (0.2, a2), (0.0, None)):
        F._GraphTraining(s, t, 0.5, True, {"pose_topk": 0, "kd_topk": 0}, x, tg, tw, 1, feature_weight=w,
                         feature_adapter=a)
    assert len(made) == 5                                    # the repeated (0.1, a1) reuses its step
    assert "feature_weight" not in made[0] and "feature_weight" not in made[4]
    assert [m.get("feature_adapter") for m in made[1:4]] == [a1, a1, a2]
    F._train_step_cache.clear()


def test_log_has_the_feature_meter(caplog):
    from fpd_b200.lib.core import function as F
    scalars = []
    writer = NS(add_scalar=lambda tag, v, step: scalars.append((tag, v)))
    m = F.AverageMeter()
    m.update(0.125, 2)
    F._log_train(NS(), {"writer": writer, "train_global_steps": 0}, 0, 0, 1, m, m, [("FEAT_Loss", m, "%.5f")], 2)
    assert scalars == [("train_feat_loss", 0.125)]


# ------------------------------------------------------------------------------------------------ C entry point
def test_feature_mse_entry_point_refuses_bad_arguments():
    from fpd_b200 import _native as N
    lib = N.lib()
    fake = ctypes.c_void_p(0x1000)
    ok = dict(s=fake, t=fake, f16=0, w=0.5, g=fake, l=fake, losses=None, n=64, ws=fake, wsb=1 << 20)
    cases = [(dict(s=None), "NULL"), (dict(t=None), "NULL"), (dict(g=None), "NULL"), (dict(l=None), "NULL"),
             (dict(ws=None), "workspace is NULL"), (dict(n=0), "n=0"), (dict(n=-4), "n=-4"), (dict(f16=2), "teacher_f16"),
             (dict(w=-1.0), "weight"), (dict(w=float("nan")), "weight"), (dict(w=float("inf")), "weight"),
             (dict(wsb=0), "workspace too small")]
    for kw, msg in cases:
        a = {**ok, **kw}
        rc = lib.fpd_feature_mse(a["s"], a["t"], a["f16"], a["w"], a["g"], a["l"], a["losses"], a["n"], a["ws"],
                                 a["wsb"], None)
        assert rc == -1, kw
        assert msg in N.last_error(), (kw, N.last_error())
    assert lib.fpd_feature_mse_workspace_bytes(64) >= 8
    assert lib.fpd_feature_mse_workspace_bytes(1 << 30) == lib.fpd_feature_mse_workspace_bytes(1 << 31)


def test_feature_mse_refuses_bad_tensors_before_the_device():
    from fpd_b200 import ops
    s = torch.zeros(1, 4, 4, 8)
    for bad in BAD_WEIGHTS:
        with pytest.raises(ValueError, match="feature_weight"):
            ops.feature_mse(s, s, bad)
    with pytest.raises(ValueError, match="CUDA"):
        ops.feature_mse(s, s, 0.1)
