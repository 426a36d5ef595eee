"""Distillation from unlabeled person boxes on the host: add_unlabeled_boxes, RawJointsDataset on zero-visibility
records against the reference (tests/golden/unlabeled.npz), the configuration and argument errors, the routes and
FPDTrainStep arguments fpd_train picks, the C entry and arguments ops.fpd_loss picks with and without a kd weight, and
the host checks of the two C entry points."""
import ctypes
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fpd_b200  # noqa: E402,F401
import _augment_cases as C  # noqa: E402
import _kld_model as K  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "unlabeled.npz")
BAD_THRE = [float("nan"), float("inf"), -float("inf")]


# ------------------------------------------------------------------------------------------------ add_unlabeled_boxes
class _StubDataset:
    """db, _box2cs (the reference's COCODataset._box2cs for a 192x256 input) and image_path_from_index."""

    def __init__(self):
        self.db = [{"image": "labeled.jpg", "joints_3d": np.ones((17, 3)), "joints_3d_vis": np.ones((17, 3))}]

    def _box2cs(self, box):
        x, y, w, h = box[:4]
        center = np.array([x + w * 0.5, y + h * 0.5], np.float32)
        aspect = 192 / 256
        if w > aspect * h:
            h = w / aspect
        elif w < aspect * h:
            w = h * aspect
        scale = np.array([w / 200.0, h / 200.0], np.float32)
        if center[0] != -1:
            scale = scale * 1.25
        return center, scale

    def image_path_from_index(self, index):
        return "images/%012d.jpg" % index


def _boxes(tmp_path):
    boxes = [{"image_id": 1, "category_id": 1, "bbox": [10.0, 20.0, 30.0, 80.0], "score": 0.9},
             {"image_id": 2, "category_id": 1, "bbox": [0.0, 0.0, 100.0, 50.0], "score": 0.5},
             {"image_id": 3, "category_id": 1, "bbox": [5.0, 5.0, 10.0, 10.0], "score": 0.49},
             {"image_id": 4, "category_id": 18, "bbox": [1.0, 2.0, 3.0, 4.0], "score": 0.99},
             {"image_id": 5, "category_id": 1, "bbox": [7.5, 1.5, 40.0, 40.0], "score": 0.5}]
    p = tmp_path / "dets.json"
    p.write_text(json.dumps(boxes))
    return str(p), boxes


def test_add_unlabeled_boxes_appends_person_boxes_above_the_score_threshold(tmp_path):
    from fpd_b200.augment import add_unlabeled_boxes
    path, boxes = _boxes(tmp_path)
    ds = _StubDataset()
    assert add_unlabeled_boxes(ds, path, score_thre=0.5) == 3
    assert len(ds.db) == 4 and ds.db[0]["image"] == "labeled.jpg"
    kept = [boxes[0], boxes[1], boxes[4]]
    for rec, box in zip(ds.db[1:], kept):
        c, s = ds._box2cs(box["bbox"])
        np.testing.assert_array_equal(rec["center"], c)
        np.testing.assert_array_equal(rec["scale"], s)
        assert rec["score"] == box["score"]
        assert rec["image"] == "images/%012d.jpg" % box["image_id"]
        for key in ("joints_3d", "joints_3d_vis"):
            assert rec[key].shape == (17, 3) and not rec[key].any()


def test_add_unlabeled_boxes_default_threshold_and_image_path(tmp_path):
    from fpd_b200.augment import add_unlabeled_boxes
    path, _ = _boxes(tmp_path)
    ds = _StubDataset()
    assert add_unlabeled_boxes(ds, path, image_path=lambda i: "x/%d.png" % i) == 4      # every person box
    assert [r["image"] for r in ds.db[1:]] == ["x/1.png", "x/2.png", "x/3.png", "x/5.png"]
    assert [r["score"] for r in ds.db[1:]] == [0.9, 0.5, 0.49, 0.5]


# ------------------------------------------------------------------------------------------------ RawJointsDataset
def test_golden_mixes_unlabeled_and_labeled_records():
    g = np.load(GOLDEN)
    for tag in C.sets(g):
        vis = g[tag + "/db_joints_vis"][..., 0].sum(1)
        assert (vis == 0).sum() >= 4 and (vis > 8).sum() >= 3
        assert g[tag + "/flipped"].any() and (g[tag + "/meta_rotation"] != 0).any()
        unl = vis == 0
        assert not g[tag + "/target_weight"][unl].any() and not g[tag + "/target"][unl].any()


@pytest.mark.parametrize("tag", ["unlabeled_coco_bgr", "unlabeled_mpii_rgb"])
def test_raw_dataset_reproduces_reference_draws_on_unlabeled_records(tag, tmp_path):
    pytest.importorskip("cv2")
    from fpd_b200 import augment as A
    g = np.load(GOLDEN)
    paths = C.write_images(g, tmp_path)
    base = C.stand_in(g, tag, paths)
    for rec, score in zip(base.db, g[tag + "/db_score"]):
        rec["score"] = float(score)
    ds = A.RawJointsDataset(base)
    C.seed(g, tag)
    items = [ds[i] for i in range(len(ds))]
    for i, it in enumerate(items):
        meta = it["meta"]
        for key in ("center", "scale", "rotation", "score", "joints", "joints_vis"):
            np.testing.assert_array_equal(np.asarray(meta[key], np.float64), g[tag + "/meta_" + key][i],
                                          err_msg="%s[%d] %s" % (tag, i, key))
        np.testing.assert_array_equal(it["inv"], g[tag + "/inv"][i])
        np.testing.assert_array_equal(it["joints"], g[tag + "/meta_joints"][i])


# ------------------------------------------------------------------------------------------------ configuration
def test_config_keys_absent_or_off_mean_off():
    from fpd_b200.lib.core import function as F
    assert F._kd_unlabeled_thre(NS()) is None
    assert F._kd_unlabeled_thre(NS(KD=NS(ALPHA=0.5))) is None
    assert F._kd_unlabeled_thre(NS(KD=NS(ALPHA=0.5, UNLABELED=False, UNLABELED_THRE=0.7))) is None
    assert F._kd_unlabeled_thre(NS(KD=NS(ALPHA=0.5, UNLABELED=True))) == 0.2
    assert F._kd_unlabeled_thre(NS(KD=NS(ALPHA=0.5, UNLABELED=True, UNLABELED_THRE=0.35))) == 0.35
    for bad in BAD_THRE + ["0.2", None]:
        with pytest.raises(ValueError, match="UNLABELED_THRE"):
            F._kd_unlabeled_thre(NS(KD=NS(UNLABELED=True, UNLABELED_THRE=bad)))


class _FpdLike(torch.nn.Module):
    """Carries the attributes of an fpd_b200 network; the route decision looks at nothing else."""

    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 16, 1)

    def engine(self):
        raise AssertionError("must not touch the engine")

    def forward_nhwc(self, x, training=None):
        raise AssertionError("must not run the network")


def _cfg(**kd):
    return NS(KD=NS(ALPHA=0.5, **kd), PRINT_FREQ=1, DEBUG=NS(DEBUG=False))


def _crit(kind="mse", use_tw=True):
    from fpd_b200.lib.core.loss import JointsKLDLoss, JointsMSELoss, JointsOHKMMSELoss
    return {"mse": lambda: JointsMSELoss(use_tw), "ohkm": lambda: JointsOHKMMSELoss(use_tw, topk=6),
            "kl": lambda: JointsKLDLoss(use_tw, temperature=0.5)}[kind]()


def test_fpd_train_refuses_the_mode_without_target_weights_teacher_or_finite_threshold():
    from fpd_b200.lib.core import function as F
    s, t = _FpdLike(), _FpdLike()
    for pose_tw, kd_tw in ((False, False), (True, False), (False, True)):
        with pytest.raises(ValueError, match="USE_TARGET_WEIGHT"):
            F.fpd_train(_cfg(UNLABELED=True), [], s, t, _crit(use_tw=pose_tw), _crit(use_tw=kd_tw), None, 0, "", "",
                        None)
    for bad in BAD_THRE:
        with pytest.raises(ValueError, match="UNLABELED_THRE"):
            F.fpd_train(_cfg(UNLABELED=True, UNLABELED_THRE=bad), [], s, t, _crit(), _crit(), None, 0, "", "", None)
    with pytest.raises(ValueError, match="teacher"):
        F.fpd_train(_cfg(UNLABELED=True), [], s, None, _crit(), _crit(), None, 0, "", "", None)
    # off: use_target_weight=False stays allowed
    F.fpd_train(_cfg(UNLABELED=False), [], s, t, _crit(use_tw=False), _crit(use_tw=False), None, 0, "", "", None)


def test_train_step_refuses_a_bad_threshold_and_a_missing_teacher():
    from fpd_b200 import ops
    from fpd_b200.train_step import FPDTrainStep
    for bad in BAD_THRE + ["0.2", True]:
        with pytest.raises(ValueError, match="kd_unlabeled_thre"):
            FPDTrainStep(_FpdLike(), _FpdLike(), kd_unlabeled_thre=bad)
        with pytest.raises(ValueError, match="kd_unlabeled_thre"):
            ops.kd_weights(torch.zeros(1, 8, 8, 4), torch.zeros(1, 4), bad)
    with pytest.raises(ValueError, match="teacher"):
        FPDTrainStep(_FpdLike(), None, kd_unlabeled_thre=0.2)
    with pytest.raises(ValueError, match="teacher"):
        ops.kd_weights(None, torch.zeros(1, 4), 0.2)
    o = [torch.zeros(1, 8, 8, 4)]
    with pytest.raises(ValueError, match="teacher"):
        ops.fpd_loss(o, torch.zeros(1, 4, 8, 8), None, torch.ones(1, 4), 0.5, kd_weight=torch.ones(1, 4))


class _Stop(Exception):
    pass


def _first_batch(B=2, J=16, hw=64):
    return [(torch.zeros(B, 3, 4 * hw, 4 * hw), torch.zeros(B, J, hw, hw), torch.ones(B, J, 1), {})]


@pytest.mark.parametrize("kd", [{}, {"UNLABELED": False}, {"UNLABELED": False, "UNLABELED_THRE": 0.5},
                                {"UNLABELED": True}, {"UNLABELED": True, "UNLABELED_THRE": 0.25}])
@pytest.mark.parametrize("graph", [True, False])
def test_fpd_train_passes_the_threshold_only_when_on(kd, graph, monkeypatch):
    """The graph route's FPDTrainStep and the eager route's _fused_step get exactly today's arguments when the mode is
    off, and kd_unlabeled_thre on top when it is on."""
    from fpd_b200 import train_step
    from fpd_b200.lib.core import function as F
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)
    monkeypatch.setattr(F, "_TRAIN_GRAPH", graph)
    seen = []

    class RecStep:
        def __init__(self, *a, **k):
            seen.append(("FPDTrainStep", a[2:], k))
            raise _Stop

    def rec_fused(*a, **k):
        seen.append(("_fused_step", a[5:], k))
        raise _Stop
    monkeypatch.setattr(train_step, "FPDTrainStep", RecStep)
    monkeypatch.setattr(F, "_fused_step", rec_fused)
    F._train_step_cache.clear()
    with pytest.raises(_Stop):
        F.fpd_train(_cfg(**kd), _first_batch(), _FpdLike(), _FpdLike(), _crit("ohkm"), _crit("kl"), NS(zero_grad=lambda: None),
                    0, "", "", None)
    on = kd.get("UNLABELED", False)
    extra = {"kd_unlabeled_thre": kd.get("UNLABELED_THRE", 0.2)} if on else {}
    if graph:
        assert seen == [("FPDTrainStep", (), {"alpha": 0.5, "fused_adam": False, "accuracy": True, "pose_topk": 6,
                                              "kd_temperature": 0.5, **extra})]
    else:
        assert len(seen) == 1 and seen[0][0] == "_fused_step"
        assert seen[0][2] == {"pose_topk": 6, "kd_temperature": 0.5, **extra}


def test_generic_route_weights_follow_the_rule():
    from fpd_b200.lib.core import function as F
    g = torch.Generator().manual_seed(3)
    B, J = 4, 5
    t = torch.randn(B, J, 6, 8, generator=g) * 0.3
    t[0, 1:3] = -1.0
    t[0, 1, 2, 3] = 0.2                                       # exactly at thre (as float32): not accepted
    t[0, 2, 0, 0] = float(np.nextafter(np.float32(0.2), np.float32(np.inf)))     # just above: accepted
    t[0, 3, 1, 1] = float("nan")                              # a NaN map: 0
    t[0, 3, 1, 2] = 5.0
    tw = (torch.rand(B, J, 1, generator=g) > 0.3).float()
    tw[0] = 0.0
    tw[2] = 0.0
    tw[3, 0] = 0.0
    got = F._kd_weights_torch(t, tw, 0.2)
    assert got.shape == tw.shape
    tn, twn = t.numpy().reshape(B, J, -1), tw.numpy().reshape(B, J)
    want = twn.copy()
    for b in range(B):
        if not twn[b].any():
            m = tn[b].max(1)
            want[b] = np.where(np.isnan(tn[b]).any(1), 0.0, (m > np.float32(0.2)).astype(np.float32))
    np.testing.assert_array_equal(got.numpy().reshape(B, J), want)
    assert got[0, :4, 0].tolist() == [float(tn[0, 0].max() > 0.2), 0.0, 1.0, 0.0]


# ------------------------------------------------------------------------------------------------ dispatch
KINDS = {"mse": ("mse",), "ohkm": ("ohkm", 6), "kl": ("kl", 0.5)}
PAIRS = [(p, k) for p in KINDS for k in KINDS]


class _RecLib:
    """Records the loss entry points (and workspace queries) ops.fpd_loss calls, with their scalar arguments."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name,) + tuple(a for a in args if isinstance(a, (int, float)) and not isinstance(a, bool)))
            return 64 if name.endswith("_workspace_bytes") else 0
        return call


def _fake(monkeypatch):
    from fpd_b200 import _native as N
    from fpd_b200 import ops
    fake = _RecLib()
    monkeypatch.setattr(N, "lib", lambda: fake)
    monkeypatch.setattr(ops, "_chk", lambda t, name: None)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    monkeypatch.setattr(ops, "_ws", NS(get=lambda n, dev: torch.empty(int(n), dtype=torch.uint8)))
    return fake


@pytest.mark.parametrize("pose,kd", PAIRS)
def test_fpd_loss_entry_points_with_and_without_a_kd_weight(pose, kd, monkeypatch):
    from fpd_b200 import ops
    fake = _fake(monkeypatch)
    S, B, J, h, w = 2, 3, 16, 8, 8
    outs = [torch.zeros(B, h, w, J) for _ in range(S)]
    kw = K.fpd_kwargs(KINDS[pose], KINDS[kd])
    pk = 6 if pose == "ohkm" else 0
    kk = 6 if kd == "ohkm" else 0
    pt = 0.5 if pose == "kl" else 0.0
    kt = 0.5 if kd == "kl" else 0.0
    if pt or kt:
        ws = ("fpd_loss_kl_workspace_bytes", S, B, J, h, w)
        want = ("fpd_loss_kl_fused", S, 0.25, 1.0, B, J, h, w, pk, kk, pt, kt, 64)
    elif pk or kk:
        ws = ("fpd_loss_ohkm_workspace_bytes", S, B, J, h, w)
        want = ("fpd_loss_ohkm_fused", S, 0.25, 1.0, B, J, h, w, pk, kk, 64)
    else:
        ws = ("fpd_loss_workspace_bytes", B, J, h, w)
        want = ("fpd_loss_fused", S, 0.25, 1.0, B, J, h, w, 64)
    ops.fpd_loss(outs, torch.zeros(B, J, h, w), outs[0], torch.ones(B, J), 0.25, kd_weight=None, **kw)
    assert fake.calls == [ws, want]
    fake.calls.clear()
    ops.fpd_loss(outs, torch.zeros(B, J, h, w), outs[0], torch.ones(B, J), 0.25, kd_weight=torch.ones(B, J, 1), **kw)
    assert fake.calls == [ws, ("fpd_loss_kdw_fused", S, 0.25, 1.0, B, J, h, w, pk, kk, pt, kt, 64)]


def test_kd_weights_calls_its_entry_point(monkeypatch):
    from fpd_b200 import ops
    fake = _fake(monkeypatch)
    out = ops.kd_weights(torch.zeros(3, 8, 6, 17), torch.zeros(3, 17, 1), 0.25)
    assert out.shape == (3, 17)
    assert fake.calls == [("fpd_kd_weights", 0.25, 3, 17, 8, 6)]


def _kdw_c(S=1, B=2, J=16, h=8, w=8, pk=0, kk=0, pt=0.0, kt=0.0, null=()):
    from fpd_b200 import _native as N
    fake = ctypes.c_void_p(0x1000)
    outs = (ctypes.c_void_p * S)(*([0x1000] * S))
    p = lambda name: None if name in null else fake  # noqa: E731
    return N.lib().fpd_loss_kdw_fused(None if "outs" in null else outs, S, p("target"), p("teacher"), p("tw"),
                                      p("kdw"), 0.5, None, 1.0, p("losses"), B, J, h, w, pk, kk, pt, kt,
                                      p("workspace"), 1 << 30, None)


def test_loss_kdw_entry_point_refuses_bad_arguments():
    from fpd_b200 import _native as N
    cases = [(dict(null=("outs",)), "outs_host"), (dict(null=("target",)), "NULL"), (dict(null=("losses",)), "NULL"),
             (dict(null=("tw",)), "NULL"), (dict(null=("kdw",)), "kd_weight"), (dict(null=("teacher",)), "teacher"),
             (dict(null=("workspace",)), "workspace"), (dict(S=0), "S=0"), (dict(S=9), "S=9"), (dict(B=0), "B=0"),
             (dict(h=0), "empty heat-map"), (dict(J=65), "J=65"), (dict(J=0), "J=0"), (dict(h=5, w=5), "multiple of 64"),
             (dict(pk=17), "pose_topk=17"), (dict(kk=-1), "kd_topk=-1"), (dict(pk=4, pt=1.0), "both topk"),
             (dict(pt=float("nan")), "pose_temperature"), (dict(kt=-1.0), "kd_temperature")]
    for kw, msg in cases:
        assert _kdw_c(**kw) == -1, kw
        assert msg in N.last_error(), (kw, N.last_error())


def test_kd_weights_entry_point_refuses_bad_arguments():
    from fpd_b200 import _native as N
    lib = N.lib()
    fake = ctypes.c_void_p(0x1000)
    cases = [((None, fake, 0.2, fake, 2, 16, 8, 8), "NULL"), ((fake, None, 0.2, fake, 2, 16, 8, 8), "NULL"),
             ((fake, fake, 0.2, None, 2, 16, 8, 8), "NULL"), ((fake, fake, 0.2, fake, 0, 16, 8, 8), "B=0"),
             ((fake, fake, 0.2, fake, 65536, 16, 8, 8), "B=65536"), ((fake, fake, 0.2, fake, 2, 65, 8, 8), "J=65"),
             ((fake, fake, 0.2, fake, 2, 0, 8, 8), "J=0"), ((fake, fake, 0.2, fake, 2, 16, 0, 8), "heat-map"),
             ((fake, fake, 0.2, fake, 2, 16, 8, -1), "heat-map")]
    cases += [((fake, fake, t, fake, 2, 16, 8, 8), "thre") for t in BAD_THRE]
    for args, msg in cases:
        assert lib.fpd_kd_weights(*args, None) == -1, args
        assert msg in N.last_error(), (args, N.last_error())


def test_workspace_keeps_an_outgrown_buffer_only_if_a_capture_took_it(monkeypatch):
    """A captured graph holds the address of the workspace it was given, so a larger request must not free that buffer;
    buffers no capture has taken are freed as before."""
    from fpd_b200 import ops
    capturing = [False]
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: NS(cuda_stream=7))
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: capturing[0])
    ws = ops.Workspace()
    eager = ws.get(16, "cpu")
    assert ws.get(1 << 10, "cpu") is eager
    mid = ws.get((1 << 20) + 1, "cpu")
    assert mid is not eager and mid.numel() >= (1 << 20) + 1 and ws.outgrown == []
    capturing[0] = True
    assert ws.get(8, "cpu") is mid                    # a capture takes the current buffer
    capturing[0] = False
    big = ws.get(1 << 21, "cpu")
    assert big is not mid and ws.outgrown == [mid]
    bigger = ws.get(1 << 22, "cpu")                   # outgrown without a capture in between: freed
    assert bigger is not big and ws.outgrown == [mid] and ws.get(8, "cpu") is bigger
