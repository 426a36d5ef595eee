"""JointsKLDLoss on the host: the fp64 model against itself, argument checks down to the C entry points, the C entry
and arguments ops.fpd_loss picks for every (pose, kd) kind pair, route selection for every criterion mix, and the
drop-in import under fpd_b200.dropin.install()."""
import ctypes
import math
import os
import subprocess
import sys
import textwrap
import types

import pytest
import torch

NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _kld_model as K  # noqa: E402

BAD_T = [0.0, -1.0, float("nan"), float("inf"), -float("inf")]


# ------------------------------------------------------------------------------------------------ the fp64 model
@pytest.mark.parametrize("T", [0.05, 0.25, 1.0, 4.0])
def test_model_nonnegative_zero_on_equal_maps_and_closed_form_gradient(T):
    g = torch.Generator().manual_seed(int(T * 100))
    B, J, h, w = 3, 5, 6, 7
    o = torch.randn(B, J, h, w, generator=g, dtype=torch.float64)
    r = torch.randn(B, J, h, w, generator=g, dtype=torch.float64)
    tw = torch.rand(B, J, 1, generator=g, dtype=torch.float64)
    assert (K.per_map_kl(o, r, T) >= 0).all()
    v0, g0 = K.kld(r, r, tw, T)
    assert v0.item() == 0.0 and g0.abs().max().item() == 0.0
    for weights in (tw, None):
        v, gr = K.kld(o, r, weights, T)
        va, ga = K.kld_autograd(o, r, weights, T)
        assert v.item() > 0
        assert abs(v.item() - va.item()) <= 1e-12 * v.item()
        assert (gr - ga).abs().max().item() <= 1e-12 * ga.abs().max().item()


def test_model_weights_enter_linearly():
    g = torch.Generator().manual_seed(2)
    o, r = torch.randn(2, 3, 4, 4, generator=g), torch.randn(2, 3, 4, 4, generator=g)
    v1, g1 = K.kld(o, r, torch.ones(2, 3, 1), 1.0)
    v2, g2 = K.kld(o, r, torch.full((2, 3, 1), 0.5), 1.0)
    assert abs(v2.item() - 0.5 * v1.item()) <= 1e-12 * v1.item()
    assert torch.allclose(g2, 0.5 * g1, rtol=0, atol=1e-15)


# ------------------------------------------------------------------------------------------------ argument errors
@pytest.mark.parametrize("T", BAD_T)
def test_bad_temperature_raises_in_python(T):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.lib.core.loss import JointsKLDLoss
    from fpd_b200.train_step import FPDTrainStep
    with pytest.raises(ValueError, match="temperature"):
        JointsKLDLoss(True, temperature=T)
    with pytest.raises(ValueError, match="temperature"):
        ops.joints_kld(torch.zeros(1, 1, 8, 8), torch.zeros(1, 1, 8, 8), None, T)
    if T != 0.0:                    # 0 means "not KL" in the fused form
        o = [torch.zeros(1, 8, 8, 1)]
        for kw in ({"pose_temperature": T}, {"kd_temperature": T}):
            with pytest.raises(ValueError, match="temperature"):
                ops.fpd_loss(o, torch.zeros(1, 1, 8, 8), o[0], torch.ones(1, 1), 0.5, **kw)
            with pytest.raises(ValueError, match="temperature"):
                FPDTrainStep(_FpdLike(), _FpdLike(), **kw)


def test_topk_with_temperature_and_kd_temperature_without_teacher_raise():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.train_step import FPDTrainStep
    o = [torch.zeros(1, 8, 8, 4)]
    for kw in ({"pose_topk": 2, "pose_temperature": 1.0}, {"kd_topk": 2, "kd_temperature": 1.0}):
        with pytest.raises(ValueError, match="not both"):
            ops.fpd_loss(o, torch.zeros(1, 4, 8, 8), o[0], torch.ones(1, 4), 0.5, **kw)
        with pytest.raises(ValueError, match="not both"):
            FPDTrainStep(_FpdLike(), _FpdLike(), **kw)
    with pytest.raises(ValueError, match="teacher"):
        FPDTrainStep(_FpdLike(), None, kd_temperature=1.0)
    for bad in ("1", True, None):
        with pytest.raises(ValueError):
            FPDTrainStep(_FpdLike(), _FpdLike(), pose_temperature=bad)


def _fused_c(J=16, h=8, w=8, S=1, pk=0, kk=0, pt=1.0, kt=0.0, teacher=True):
    """fpd_loss_kl_fused called with stand-in addresses: every call here must be refused by the host checks before
    anything is launched."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    fake = ctypes.c_void_p(0x1000)
    outs = (ctypes.c_void_p * S)(*([0x1000] * S))
    return N.lib().fpd_loss_kl_fused(outs, S, fake, fake if teacher else None, fake, 0.5, None, 1.0, fake, 2, J, h, w,
                                     pk, kk, pt, kt, fake, 1 << 30, None)


def test_c_entry_points_refuse_bad_arguments():
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    lib = N.lib()
    cases = [(dict(J=65), "J=65"), (dict(J=0), "J=0"), (dict(h=5, w=5), "multiple of 64"), (dict(S=9), "S=9"),
             (dict(pk=4, pt=1.0), "both topk"), (dict(kk=4, kt=2.0), "both topk"),
             (dict(kt=1.0, teacher=False), "without a teacher"), (dict(pk=17), "pose_topk=17")]
    for T in BAD_T[1:]:
        cases += [(dict(pt=T), "pose_temperature"), (dict(pt=0.0, kt=T), "kd_temperature")]
    for kw, msg in cases:
        assert _fused_c(**kw) == -1, kw
        assert msg in N.last_error(), (kw, N.last_error())
    fake = ctypes.c_void_p(0x1000)
    for T in BAD_T:
        assert lib.fpd_joints_kld(fake, fake, None, T, fake, None, 2, 16, 64, fake, 1 << 30, None) == -1
        assert "temperature" in N.last_error()
    assert lib.fpd_joints_kld(fake, fake, None, 1.0, fake, None, 2, 65, 64, fake, 1 << 30, None) == -1
    assert "J=65" in N.last_error()
    assert lib.fpd_joints_kld(fake, fake, None, 1.0, fake, None, 0, 16, 64, fake, 1 << 30, None) == -1
    assert lib.fpd_joints_kld(None, fake, None, 1.0, fake, None, 2, 16, 64, fake, 1 << 30, None) == -1
    assert lib.fpd_joints_kld(fake, fake, None, 1.0, fake, None, 2, 16, 64, fake, 16, None) == -1
    assert "workspace" in N.last_error()
    # the module form takes any h*w; the workspace grows with the number of 64-pixel chunks
    assert 0 < lib.fpd_joints_kld_workspace_bytes(2, 16, 30) <= lib.fpd_joints_kld_workspace_bytes(2, 16, 900)
    assert lib.fpd_loss_kl_workspace_bytes(4, 32, 16, 64, 64) > 0


# ------------------------------------------------------------------------------------------------ C entry per pair
KINDS = {"mse": ("mse",), "ohkm": ("ohkm", 6), "kl": ("kl", 0.5)}
PAIRS = [(p, k) for p in KINDS for k in KINDS]


class _FakeLib:
    """Records the loss entry points ops.fpd_loss calls, with their scalar arguments."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            if name.endswith("_workspace_bytes"):
                return 64
            self.calls.append((name,) + tuple(a for a in args if isinstance(a, (int, float)) and not isinstance(a, bool)))
            return 0
        return call


@pytest.mark.parametrize("pose,kd", PAIRS)
def test_fpd_loss_entry_point_for_every_kind_pair(pose, kd, monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    from fpd_b200 import ops
    fake = _FakeLib()
    monkeypatch.setattr(N, "lib", lambda: fake)
    monkeypatch.setattr(ops, "_chk", lambda t, name: None)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    monkeypatch.setattr(ops, "_ws", NS(get=lambda n, dev: torch.empty(int(n), dtype=torch.uint8)))
    S, B, J, h, w = 2, 3, 16, 8, 8
    outs = [torch.zeros(B, h, w, J) for _ in range(S)]
    ops.fpd_loss(outs, torch.zeros(B, J, h, w), outs[0], torch.ones(B, J), 0.25,
                 **K.fpd_kwargs(KINDS[pose], KINDS[kd]))
    pk = 6 if pose == "ohkm" else 0
    kk = 6 if kd == "ohkm" else 0
    if "kl" not in (pose, kd):        # what ops.fpd_loss called before JointsKLDLoss existed
        if pk or kk:
            want = ("fpd_loss_ohkm_fused", S, 0.25, 1.0, B, J, h, w, pk, kk, 64)
        else:
            want = ("fpd_loss_fused", S, 0.25, 1.0, B, J, h, w, 64)
    else:
        want = ("fpd_loss_kl_fused", S, 0.25, 1.0, B, J, h, w, pk, kk, 0.5 if pose == "kl" else 0.0,
                0.5 if kd == "kl" else 0.0, 64)
    assert fake.calls == [want]


# ------------------------------------------------------------------------------------------------ route selection
class _FpdLike(torch.nn.Module):
    """Carries the attributes of an fpd_b200 network; the route decision looks at nothing else."""

    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 16, 1)

    def engine(self):
        raise AssertionError("route selection must not touch the engine")

    def forward_nhwc(self, x, training=None):
        raise AssertionError("route selection must not run the network")


def _crit(kind, use_tw=True):
    from fpd_b200.lib.core.loss import JointsKLDLoss, JointsMSELoss, JointsOHKMMSELoss
    return {"mse": lambda: JointsMSELoss(use_tw), "ohkm": lambda: JointsOHKMMSELoss(use_tw, topk=6),
            "kl": lambda: JointsKLDLoss(use_tw, temperature=0.5)}[kind]()


@pytest.mark.parametrize("pose,kd", PAIRS)
def test_route_and_term_selectors_for_every_criterion_mix(pose, kd, monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    s, t = _FpdLike(), _FpdLike()
    cp, ck = _crit(pose), _crit(kd)
    shape = (32, 16, 64, 64)
    cfg = NS(DEBUG=NS(DEBUG=False), PRINT_FREQ=1)
    assert F._train_route(cfg, s, t, [cp, ck], shape) == "graph"
    assert F._train_route(cfg, s, None, [cp], shape) == "graph"
    assert F._train_route(NS(DEBUG=NS(DEBUG=True), PRINT_FREQ=1), s, t, [cp, ck], shape) == "fused"
    monkeypatch.setattr(F, "_TRAIN_GRAPH", False)
    assert F._train_route(cfg, s, t, [cp, ck], shape) == "fused"
    monkeypatch.setattr(F, "_TRAIN_GRAPH", True)
    # odd heat-map sizes, too many joints and mixed target weighting take the generic route
    assert F._train_route(cfg, s, t, [cp, ck], (32, 16, 30, 30)) == "generic"
    assert F._train_route(cfg, s, t, [cp, ck], (32, 17, 63, 47)) == "generic"
    assert F._train_route(cfg, s, t, [cp, ck], (32, 65, 64, 64)) == "generic"
    assert F._train_route(cfg, s, t, [cp, _crit(kd, use_tw=False)], shape) == "generic"
    terms = {**F._criterion_term(cp, "pose"), **F._criterion_term(ck, "kd")}
    assert terms == K.fpd_kwargs(KINDS[pose], KINDS[kd]) | ({} if pose != "mse" else {"pose_topk": 0}) \
        | ({} if kd != "mse" else {"kd_topk": 0})
    # validate's graph route takes every criterion at the fused kernels' shapes, never under DEBUG
    target = torch.zeros(2, 16, 64, 48)
    assert F._validate_graph_ok(cfg, cp, target)
    assert not F._validate_graph_ok(NS(DEBUG=NS(DEBUG=True)), cp, target)
    assert not F._validate_graph_ok(cfg, cp, torch.zeros(2, 16, 30, 30))


def test_criterion_terms_of_the_existing_criteria_are_unchanged():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    assert F._criterion_term(_crit("mse"), "pose") == {"pose_topk": 0}
    assert F._criterion_term(_crit("ohkm"), "kd") == {"kd_topk": 6}
    assert F._criterion_term(_crit("kl"), "kd") == {"kd_temperature": 0.5}


def test_kld_module_attributes_and_cpu_refusal():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core.loss import JointsKLDLoss
    a = JointsKLDLoss(False)
    assert (a.use_target_weight, a.temperature) == (False, 1.0) and isinstance(a, torch.nn.Module)
    assert JointsKLDLoss(True, 4).temperature == 4.0 and math.isfinite(JointsKLDLoss(True, 1e-3).temperature)
    with pytest.raises(RuntimeError, match="CUDA"):
        JointsKLDLoss(True)(torch.zeros(2, 4, 8, 8), torch.zeros(2, 4, 8, 8), torch.ones(2, 4, 1))


def test_flip_test_inference_checks_the_temperature():
    import fpd_b200  # noqa: F401
    from fpd_b200 import infer_step
    assert infer_step._temperature(0, 0) == 0.0 and infer_step._temperature(0, 2) == 2.0
    for T in BAD_T[1:]:
        with pytest.raises(ValueError, match="temperature"):
            infer_step._temperature(0, T)
    with pytest.raises(ValueError, match="not both"):
        infer_step._temperature(8, 1.0)


# ------------------------------------------------------------------------------------------------ drop-in
DROPIN = textwrap.dedent('''
    import sys, types
    REF, ROOT = %r, %r
    for name in ("yacs", "json_tricks", "tensorboardX", "pycocotools", "easydict"):
        try:
            __import__(name)
        except ImportError:
            sys.modules[name] = types.ModuleType(name)
    sys.path.insert(0, REF + "/lib")
    sys.path.insert(0, ROOT)
    import fpd_b200
    from fpd_b200 import dropin
    dropin.install()
    from core.loss import JointsKLDLoss
    import fpd_b200.lib.core.loss as L
    assert JointsKLDLoss is L.JointsKLDLoss
    from core.function import fpd_train
    print("KLD-DROPIN-OK")
''')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "lib")), reason="needs the reference checkout")
def test_dropin_resolves_kld_loss_to_fpd_b200():
    r = subprocess.run([sys.executable, "-c", DROPIN % (REF, ROOT)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "KLD-DROPIN-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
