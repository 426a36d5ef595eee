"""Which train / fpd_train epochs take the CUDA-graph route (lib/core/function.py _train_route), and FPDTrainStep's
argument checks -- host logic only, no device needed."""
import os
import sys
import types

import pytest
import torch

NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _FpdLike(torch.nn.Module):
    """Carries the attributes of an fpd_b200 network; the route decision looks at nothing else."""

    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 16, 1)

    def engine(self):
        raise AssertionError("route selection must not touch the engine")

    def forward_nhwc(self, x, training=None):
        raise AssertionError("route selection must not run the network")


class _Plain(torch.nn.Module):
    def forward(self, x):
        return x


def _cfg(debug=False):
    return NS(DEBUG=NS(DEBUG=debug), PRINT_FREQ=1)


@pytest.fixture
def F():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    return F


def test_route_for_fpd_networks_and_criteria(F):
    from fpd_b200.lib.core.loss import JointsMSELoss, JointsOHKMMSELoss
    s, t = _FpdLike(), _FpdLike()
    shape = (32, 16, 64, 64)
    mse, ohkm = JointsMSELoss(True), JointsOHKMMSELoss(True, topk=8)
    assert F._train_route(_cfg(), s, t, [mse, mse], shape) == "graph"
    assert F._train_route(_cfg(), s, t, [ohkm, mse], shape) == "graph"
    assert F._train_route(_cfg(), s, t, [ohkm, ohkm], shape) == "graph"
    assert F._train_route(_cfg(), s, None, [ohkm], shape) == "graph"                    # train(): no teacher
    assert F._train_route(_cfg(), torch.nn.DataParallel(s, device_ids=[]), t, [mse, mse], shape) == "graph"


def test_route_debug_and_switch_keep_the_eager_fused_route(F, monkeypatch):
    from fpd_b200.lib.core.loss import JointsMSELoss
    s, t, mse = _FpdLike(), _FpdLike(), JointsMSELoss(True)
    shape = (32, 16, 64, 64)
    assert F._train_route(_cfg(debug=True), s, t, [mse, mse], shape) == "fused"
    assert F._train_route(NS(PRINT_FREQ=1), s, t, [mse, mse], shape) == "graph"        # config without DEBUG
    monkeypatch.setattr(F, "_TRAIN_GRAPH", False)
    assert F._train_route(_cfg(), s, t, [mse, mse], shape) == "fused"


def test_route_generic_cases(F):
    from fpd_b200.lib.core.loss import JointsMSELoss
    s, t = _FpdLike(), _FpdLike()
    shape = (32, 16, 64, 64)
    mse = JointsMSELoss(True)
    assert F._train_route(_cfg(), _Plain(), t, [mse, mse], shape) == "generic"        # student without an engine
    assert F._train_route(_cfg(), s, _Plain(), [mse, mse], shape) == "generic"        # teacher without an engine
    assert F._train_route(_cfg(), s, t, [mse, torch.nn.MSELoss()], shape) == "generic"  # foreign criterion
    assert F._train_route(_cfg(), s, t, [mse, JointsMSELoss(False)], shape) == "generic"  # mixed target weighting
    assert F._train_route(_cfg(), s, t, [mse, mse], (32, 16, 30, 30)) == "generic"    # h*w % 64 != 0
    assert F._train_route(_cfg(), s, t, [mse, mse], (32, 65, 64, 64)) == "generic"    # J > 64


@pytest.mark.parametrize("kw", [dict(pose_topk=-1), dict(pose_topk=65), dict(kd_topk=1.5), dict(kd_topk=True),
                                dict(pose_topk="8")])
def test_train_step_rejects_bad_topk(kw):
    import fpd_b200  # noqa: F401
    from fpd_b200.train_step import FPDTrainStep
    with pytest.raises(ValueError):
        FPDTrainStep(_FpdLike(), _FpdLike(), **kw)


def test_train_step_kd_topk_needs_a_teacher():
    import fpd_b200  # noqa: F401
    from fpd_b200.train_step import FPDTrainStep
    with pytest.raises(ValueError, match="teacher"):
        FPDTrainStep(_FpdLike(), None, kd_topk=8)


def test_external_optimizer_mode_keeps_parameter_storage():
    """FlatParams(rehome=False): one flat gradient buffer with per-parameter views, parameters untouched."""
    import fpd_b200  # noqa: F401
    from fpd_b200.train_step import FlatParams
    net = torch.nn.Sequential(torch.nn.Conv2d(3, 5, 3), torch.nn.BatchNorm2d(5))
    before = [(p.data_ptr(), p.detach().clone()) for p in net.parameters()]
    fp = FlatParams(net, rehome=False)
    assert fp.flat is None and fp.is_intact()
    assert [p.data_ptr() for p in net.parameters()] == [b[0] for b in before]
    assert all(torch.equal(p, b[1]) for p, b in zip(net.parameters(), before))
    assert [tuple(g.shape) for g in fp.grad_views] == [tuple(p.shape) for p in net.parameters()]
    assert all(g.untyped_storage().data_ptr() == fp.grad.untyped_storage().data_ptr() for g in fp.grad_views)
    assert fp.numel % 4 == 0 and all(o % 4 == 0 for o in fp.offsets)
