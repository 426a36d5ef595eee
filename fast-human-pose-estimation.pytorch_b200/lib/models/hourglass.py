"""Stacked hourglass -- drop-in for the reference's lib/models/hourglass.py.

Same public surface: `get_pose_net(cfg, is_train, **kwargs) -> nn.Module`, `forward(x[B,3,H,W]) ->
list of NUM_STACKS tensors [B,J,H/4,W/4]`, and a `state_dict()` whose keys/shapes equal the reference's
(hourglass.py:98-168), so published checkpoints load with strict=True. The module tree only *stores*
parameters (ordinary nn.Conv2d / nn.BatchNorm2d leaves, created in the reference's order so a given seed
yields the same initial weights); the arithmetic runs in fpd_b200.engine on libfpd_b200's sm_90a
kernels. There is no CPU / torch-op fallback: calling forward on a CPU tensor raises.
"""
import torch
import torch.nn as nn

BN_MOMENTUM = 0.1
_DEPTH = 4


def _bn(ch):
    return nn.BatchNorm2d(ch, momentum=BN_MOMENTUM)


class _ParamOnly(nn.Module):
    """Holder whose arithmetic lives in the engine; direct calls are a usage error."""

    def forward(self, *a, **k):
        raise RuntimeError("%s holds parameters only; run the enclosing HourglassNet (its forward drives the "
                           "H100 engine)" % type(self).__name__)


class Bottleneck(_ParamOnly):
    """Parameter layout of the pre-activation bottleneck (reference hourglass.py:14-30): bn1/conv1 (1x1,
    in->planes), bn2/conv2 (3x3), bn3/conv3 (1x1, planes->2*planes), optional `downsample` 1x1 on the skip."""
    expansion = 2

    def __init__(self, inplanes, planes, downsample=None):
        super().__init__()
        specs = ((inplanes, planes, 1), (planes, planes, 3), (planes, planes * self.expansion, 1))
        for i, (cin, cout, k) in enumerate(specs, start=1):
            setattr(self, "bn%d" % i, _bn(cin))
            setattr(self, "conv%d" % i, nn.Conv2d(cin, cout, kernel_size=k, padding=k // 2, bias=True))
        self.downsample = downsample


class Hourglass(_ParamOnly):
    """hg[d][r]: residual branch r of recursion depth d (3 branches, 4 at the innermost level)."""

    def __init__(self, num_blocks, planes, depth):
        super().__init__()
        self.depth = depth
        ch = planes * Bottleneck.expansion
        levels = []
        for d in range(depth):
            branches = [nn.Sequential(*[Bottleneck(ch, planes) for _ in range(num_blocks)])
                        for _ in range(4 if d == 0 else 3)]
            levels.append(nn.ModuleList(branches))
        self.hg = nn.ModuleList(levels)


class HourglassNet(nn.Module):
    def __init__(self, cfg, **kwargs):
        super().__init__()
        extra = cfg.MODEL.EXTRA
        feats, self.num_stacks, self.num_blocks = int(extra.NUM_FEATURES), int(extra.NUM_STACKS), int(extra.NUM_BLOCKS)
        self.num_joints = int(cfg.MODEL.NUM_JOINTS)
        stem, half = feats // 4, feats // 2      # NUM_FEATURES=F: stem F/4, bottleneck planes F/2, trunk F
        self._inplanes = stem
        self.conv1 = nn.Conv2d(3, stem, kernel_size=7, stride=2, padding=3, bias=True)
        self.bn1 = _bn(stem)
        self.layer1 = self._residual(stem, 1)             # F/4 -> F/2 channels @ H/2 (has downsample)
        self.layer2 = self._residual(self._inplanes, 1)   # F/2 -> F  @ H/4 (has downsample)
        self.layer3 = self._residual(half, 1)             # F   -> F
        ch = half * Bottleneck.expansion
        groups = {k: [] for k in ("hg", "res", "fc", "score", "fc_", "score_")}
        for i in range(self.num_stacks):
            groups["hg"].append(Hourglass(self.num_blocks, half, _DEPTH))
            groups["res"].append(self._residual(half, self.num_blocks))
            bn = _bn(ch)
            groups["fc"].append(nn.Sequential(nn.Conv2d(ch, ch, kernel_size=1, bias=True), bn))
            groups["score"].append(nn.Conv2d(ch, self.num_joints, kernel_size=1, bias=True))
            if i < self.num_stacks - 1:
                groups["fc_"].append(nn.Conv2d(ch, ch, kernel_size=1, bias=True))
                groups["score_"].append(nn.Conv2d(self.num_joints, ch, kernel_size=1, bias=True))
        for k, mods in groups.items():
            setattr(self, k, nn.ModuleList(mods))
        self._engine = None

    def _residual(self, planes, num_blocks):
        out_ch = planes * Bottleneck.expansion
        ds = None
        if self._inplanes != out_ch:
            ds = nn.Sequential(nn.Conv2d(self._inplanes, out_ch, kernel_size=1, bias=True))
        blocks = [Bottleneck(self._inplanes, planes, ds)]
        self._inplanes = out_ch
        blocks += [Bottleneck(out_ch, planes) for _ in range(1, num_blocks)]
        return nn.Sequential(*blocks)

    # ---------------------------------------------------------------- execution
    def engine(self):
        if self._engine is None:
            from fpd_b200.engine import Engine
            self._engine = Engine(self)
        return self._engine

    def forward(self, x):
        dev = self.conv1.weight.device
        if dev.type != "cuda":
            raise RuntimeError("fpd_b200 HourglassNet runs on a CUDA (sm_90a) device only; the module is on %s. "
                               "There is no CPU fallback: call .cuda() first." % dev)
        if not x.is_cuda:   # host batch from a DataLoader: stage it like nn.DataParallel's scatter would
            x = x.to(dev, non_blocking=True)
        from fpd_b200 import autograd_bridge
        return autograd_bridge.run(self, x)

    def forward_nhwc(self, x, training=None):
        """Inference fast path: list of NHWC heat-maps (no layout round-trip, no tape)."""
        ctx = self.engine().forward(x, self.training if training is None else training, record_tape=False)
        return [v.data for v in ctx.outs]


def get_pose_net(cfg, is_train, **kwargs):
    # like the reference (hourglass.py:195-197): is_train is ignored, default torch init, no pretrained load
    return HourglassNet(cfg, **kwargs)
