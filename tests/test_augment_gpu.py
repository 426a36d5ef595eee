"""The device input path (csrc/augment.cu, fpd_b200.augment.DeviceCropLoader) against the reference's JointsDataset
(tests/golden/augment.npz) and the fixed-point specification (oracle/augment_oracle.py). The kernel checks need neither
cv2 nor the reference; the loader checks need cv2 to compute the crop matrices."""
import ctypes
import logging
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fpd_b200  # noqa: E402,F401
from fpd_b200 import augment as A  # noqa: E402
from fpd_b200 import ops  # noqa: E402
from oracle import augment_oracle as O  # noqa: E402
import _augment_cases as C  # noqa: E402

G = C.golden()
MEAN, STD = G["mean"].astype(np.float32), G["std"].astype(np.float32)
NS = types.SimpleNamespace


def _item(img, inv, size, origin=None):
    """A RawJointsDataset-like item cut from a whole source image with the product's region rule."""
    x0, y0, x1, y1 = A.source_window(inv, size, img.shape[1], img.shape[0])
    region = np.ascontiguousarray(img[y0:y1, x0:x1])
    desc = np.array([0, x0, y0, region.shape[1], region.shape[0], img.shape[1], img.shape[0]], np.int64)
    z = np.zeros((1, 3))
    return {"region": region, "desc": desc, "inv": np.asarray(inv, np.float64), "joints": z, "joints_vis": z,
            "out_size": tuple(size), "mean": MEAN, "std": STD, "meta": {"i": 0}}


def _crop(batch):
    dev = {k: batch[k].cuda() for k in ("pixels", "desc", "inv")}
    out = ops.crop_affine_normalize(dev["pixels"], dev["desc"], dev["inv"], tuple(batch["out_size"].tolist()), MEAN, STD,
                                    desc_host=batch["desc"], inv_host=batch["inv"])
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("tag", C.sets(G))
def test_kernel_equals_golden_input(tag):
    size = C.out_size(G, tag)
    n = len(G[tag + "/crop"])
    out = _crop(A.raw_collate([_item(C.source(G, tag, i), G[tag + "/inv"][i], size) for i in range(n)]))
    assert out.shape == (n, 3, size[1], size[0]) and out.dtype == torch.float32
    for i in range(n):
        assert torch.equal(out[i], torch.from_numpy(O.normalize(G[tag + "/crop"][i], MEAN, STD))), "%s[%d]" % (tag, i)
    if tag + "/input" in G.files:
        for j, i in enumerate(G[tag + "/input_idx"]):
            assert torch.equal(out[i], torch.from_numpy(G[tag + "/input"][j])), "%s[%d]" % (tag, i)


def test_kernel_equals_oracle_on_all_subpixel_phases():
    rng = np.random.RandomState(5)
    size = (72, 88)
    items, want, phases = [], [], set()
    for k in range(24):
        h, w = int(rng.randint(20, 300)), int(rng.randint(20, 300))
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        ang = rng.uniform(-np.pi, np.pi)
        sc = rng.uniform(0.3, 4.0) * np.array([1.0, rng.uniform(0.7, 1.4)])
        a = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]]) * sc
        if k % 5 == 0:
            a[:, 0] *= -1                                    # mirrored
        b = np.array([rng.uniform(-0.5, 1.2) * w, rng.uniform(-0.5, 1.2) * h])
        inv = np.concatenate([a, b[:, None]], 1)
        items.append(_item(img, inv, size))
        want.append(O.normalize(O.warp_region(img, (0, 0), inv, size), MEAN, STD))
        x, y = np.meshgrid(np.arange(size[0], dtype=np.float64), np.arange(size[1], dtype=np.float64))
        X = (np.rint((inv[0, 1] * y + inv[0, 2]) * 1024).astype(np.int64) + 16 +
             np.rint(inv[0, 0] * x * 1024).astype(np.int64)) >> 5
        Y = (np.rint((inv[1, 1] * y + inv[1, 2]) * 1024).astype(np.int64) + 16 +
             np.rint(inv[1, 0] * x * 1024).astype(np.int64)) >> 5
        phases.update(((Y & 31) * 32 + (X & 31)).ravel().tolist())
    assert len(phases) == 1024
    out = _crop(A.raw_collate(items))
    for i, wnt in enumerate(want):
        assert torch.equal(out[i], torch.from_numpy(wnt)), i


def _device_loader(tag, paths, batch_size=None, size=None, heatmap=None):
    ds = C.stand_in(G, tag, paths)
    if size is not None:
        ds.image_size, ds.heatmap_size = np.array(size), np.array(heatmap)
        ds.aspect_ratio = size[0] * 1.0 / size[1]
    raw = A.RawJointsDataset(ds)
    loader = torch.utils.data.DataLoader(raw, batch_size=batch_size or len(raw), shuffle=False, num_workers=0,
                                         collate_fn=A.raw_collate, pin_memory=True)
    return A.DeviceCropLoader(loader, ds.heatmap_size, ds.sigma)


@pytest.mark.parametrize("tag", C.sets(G))
def test_device_loader_matches_reference(tag, tmp_path):
    pytest.importorskip("cv2")
    paths = C.write_images(G, tmp_path)
    C.seed(G, tag)
    batches = list(_device_loader(tag, paths))
    assert len(batches) == 1
    inp, target, tw, meta = batches[0]
    assert inp.is_cuda and target.is_cuda and tw.is_cuda and not meta["center"].is_cuda
    for i in range(inp.shape[0]):
        assert torch.equal(inp[i].cpu(), torch.from_numpy(O.normalize(G[tag + "/crop"][i], MEAN, STD))), i
    if tag + "/input" in G.files:
        for j, i in enumerate(G[tag + "/input_idx"]):
            assert torch.equal(inp[i].cpu(), torch.from_numpy(G[tag + "/input"][j]))
    assert torch.equal(target.cpu(), torch.from_numpy(G[tag + "/target"]))
    assert torch.equal(tw.cpu(), torch.from_numpy(G[tag + "/target_weight"]))
    np.testing.assert_array_equal(meta["center"].numpy().astype(np.float64), G[tag + "/meta_center"])


def test_device_step_replays_in_a_cuda_graph(tmp_path):
    pytest.importorskip("cv2")
    paths = C.write_images(G, tmp_path)
    C.seed(G, "train_bgr")
    dl = _device_loader("train_bgr", paths)
    batch = next(iter(dl.loader))
    dev = dl.to_device(batch)
    eager = [t.clone() for t in dl.device_step(dev, batch)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dl.device_step(dev, batch)                          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static = dl.device_step(dev, batch)
    for _ in range(2):
        for t in static:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        for a, b in zip(static, eager):
            assert torch.equal(a, b)


def test_one_crop_launch_per_batch(tmp_path):
    pytest.importorskip("cv2")
    paths = C.write_images(G, tmp_path)
    C.seed(G, "train_rgb")
    dl = _device_loader("train_rgb", paths, batch_size=4)
    lib = ops.N.lib()
    deltas = []
    n0 = lib.fpd_launch_count()
    for _ in dl:
        n1 = lib.fpd_launch_count()
        deltas.append(n1 - n0)
        n0 = n1
    assert len(deltas) == len(dl) == 3
    assert deltas == [2] * 3          # one crop launch and one target launch per batch


def test_function_train_runs_on_the_device_loader(tmp_path):
    pytest.importorskip("cv2")
    from fpd_b200.lib.core.function import train
    from fpd_b200.lib.core.loss import JointsMSELoss
    from fpd_b200.lib.models import hourglass as H
    paths = C.write_images(G, tmp_path)
    C.seed(G, "train_rgb")
    dl = _device_loader("train_rgb", paths, batch_size=4, size=(64, 64), heatmap=(16, 16))
    dl.loader = [b for b, _ in zip(dl.loader, range(2))]   # two iterations
    cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=2, NUM_BLOCKS=1), NUM_JOINTS=16, NAME="hourglass"),
             PRINT_FREQ=1, DEBUG=NS(DEBUG=False))
    torch.manual_seed(0)
    net = H.get_pose_net(cfg, True).cuda()
    w0 = net.state_dict()["conv1.weight"].clone()
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)

    class Writer:
        scalars = []

        def add_scalar(self, tag, v, step):
            self.scalars.append((tag, float(v)))
    wd = {"writer": Writer(), "train_global_steps": 0}
    logging.basicConfig(level=logging.INFO)
    train(cfg, dl, net, JointsMSELoss(True), opt, 0, str(tmp_path), str(tmp_path), wd)
    torch.cuda.synchronize()
    assert wd["train_global_steps"] == 2
    losses = [v for t, v in wd["writer"].scalars if t == "train_loss"]
    assert len(losses) == 2 and all(np.isfinite(losses))
    assert not torch.equal(net.state_dict()["conv1.weight"], w0)


def _args(n=1, size=(8, 8), inv=None, desc=None):
    img = np.arange(10 * 12 * 3, dtype=np.uint8).reshape(10, 12, 3)
    batch = A.raw_collate([_item(img, np.array([[1.0, 0.0, 1.0], [0.0, 1.0, 1.0]]), size) for _ in range(n)])
    if inv is not None:
        batch["inv"][0] = torch.tensor(np.asarray(inv, np.float64).reshape(6))
    if desc is not None:
        batch["desc"][0] = torch.tensor(desc)
    return batch


def test_argument_errors_raise():
    lib = ops.N.lib()
    b = _args()
    dev = {k: b[k].cuda() for k in ("pixels", "desc", "inv")}
    out = torch.empty((1, 3, 8, 8), device="cuda")
    ms = np.concatenate([MEAN, STD]).astype(np.float32)
    P = ctypes.c_void_p

    def call(src=P(dev["pixels"].data_ptr()), nbytes=dev["pixels"].numel(), desc=P(dev["desc"].data_ptr()),
             inv=P(dev["inv"].data_ptr()), desc_host=P(b["desc"].data_ptr()), inv_host=P(b["inv"].data_ptr()),
             msh=ms.ctypes.data_as(P), o=P(out.data_ptr()), n=1, h=8, w=8):
        return lib.fpd_crop_affine_normalize(src, nbytes, desc, inv, desc_host, inv_host, msh, o, n, h, w,
                                             ops._stream())
    assert call(n=0) == 0
    for kw in ({"n": -1}, {"h": 0}, {"w": 0}, {"src": None}, {"desc": None}, {"inv": None}, {"desc_host": None},
               {"inv_host": None}, {"msh": None}, {"o": None}, {"nbytes": 3}):
        with pytest.raises(RuntimeError):
            ops.N.check(call(**kw), "crop_affine_normalize")
    for bad in (_args(inv=[[1e7, 0, 0], [0, 1, 0]]),                 # fixed-point x overflows int32
                _args(inv=[[1, 0, 0], [0, 1, 3e6]]),                 # fixed-point y overflows int32
                _args(inv=[[np.nan, 0, 0], [0, 1, 0]]),
                _args(desc=[0, 10, 0, 5, 4, 12, 10]),                # region past the image's right edge
                _args(desc=[0, 0, 0, 4, 4, 40000, 10]),              # image wider than cv2's int16 tap positions
                _args(desc=[-1, 0, 0, 2, 2, 12, 10])):
        d = {k: bad[k].cuda() for k in ("pixels", "desc", "inv")}
        with pytest.raises(RuntimeError):
            ops.crop_affine_normalize(d["pixels"], d["desc"], d["inv"], (8, 8), MEAN, STD, bad["desc"], bad["inv"])
    with pytest.raises(RuntimeError):
        ops.crop_affine_normalize(dev["pixels"], dev["desc"], dev["inv"], (0, 8), MEAN, STD, b["desc"], b["inv"])
