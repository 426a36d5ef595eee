"""validate()'s graph route: ops.final_preds / ops.pck_counts against the reference's golden vectors and the host
decode, FlipTestInference's decode stage against the eager composition, and validate() through the graph against the
eager fused route -- all bit for bit."""
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def z():
    d = np.load(os.path.join(GOLD, "decode2.npz"), allow_pickle=False)
    return {k: d[k] for k in d.files}


def _cfg_pp(pp):
    return NS(TEST=NS(POST_PROCESS=pp))


def _device_decode(hm_nchw, center, scale, pp):
    from fpd_b200 import ops
    from fpd_b200.lib.core.inference import inverse_affines
    B, J, h, w = hm_nchw.shape
    avg, idx, mv = ops.flip_merge_argmax(ops.nchw_to_nhwc(hm_nchw))
    inv = torch.from_numpy(inverse_affines(center, scale, [w, h])).cuda()
    return ops.final_preds(avg, idx, mv, inv, pp).cpu().numpy()


@pytest.mark.parametrize("tag", ["sq", "rect"])
@pytest.mark.parametrize("pp", [True, False])
def test_final_preds_matches_reference_golden(z, tag, pp):
    import fpd_b200  # noqa: F401
    preds = _device_decode(torch.from_numpy(z[tag + "/hm"]).cuda(), z[tag + "/center"], z[tag + "/scale"], pp)
    assert preds.dtype == np.float32
    assert np.array_equal(preds[..., :2], z["%s/preds_pp%d" % (tag, int(pp))])
    assert np.array_equal(preds[..., 2:], z["%s/maxvals_pp%d" % (tag, int(pp))])


@pytest.mark.parametrize("tag", ["sq", "rect"])
def test_pck_counts_match_reference_golden(z, tag):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.lib.core.evaluate import pck_from_counts
    out, tgt = torch.from_numpy(z[tag + "/acc_out"]).cuda(), torch.from_numpy(z[tag + "/acc_target"]).cuda()
    _, idx, mv = ops.flip_merge_argmax(ops.nchw_to_nhwc(out), want_avg=False)
    counts, pred_hm = ops.pck_counts(idx, mv, tgt, want_pred_hm=True)
    acc, avg, cnt = pck_from_counts(counts.cpu().numpy())
    assert np.array_equal(acc, z[tag + "/acc"])
    assert avg == float(z[tag + "/avg_acc"]) and cnt == int(z[tag + "/cnt"])
    assert np.array_equal(pred_hm.cpu().numpy(), z[tag + "/acc_pred"])
    counts2, none = ops.pck_counts(idx, mv, tgt)      # counts are re-zeroed by every call
    assert none is None and torch.equal(counts, counts2)


def _random_maps(rng, B, J, h, w):
    """Positive noise with planted maxima at and next to the borders of the post-process window, exact ties between
    maxima and between neighbours, NaN maps, maps with one NaN and all-negative maps."""
    hm = (rng.rand(B, J, h, w) * 0.5).astype(np.float32)
    cols = [0, 1, 2, w // 2, w - 3, w - 2, w - 1]
    rows = [0, 1, 2, h // 2, h - 3, h - 2, h - 1]
    for b in range(B):
        for j in range(J):
            kind = rng.randint(10)
            m = hm[b, j]
            px, py = cols[rng.randint(len(cols))], rows[rng.randint(len(rows))]
            m[py, px] = 1.0
            if kind == 1:                       # two equal maxima: the first in scan order wins
                m[rng.randint(h), rng.randint(w)] = 1.0
            elif kind == 2:                     # equal neighbours: sign 0
                if 0 < px < w - 1:
                    m[py, px - 1] = m[py, px + 1]
                if 0 < py < h - 1:
                    m[py - 1, px] = m[py + 1, px]
            elif kind == 3:
                m[...] = np.nan
            elif kind == 4:
                m[rng.randint(h), rng.randint(w)] = np.nan
            elif kind == 5:
                m[...] = -1.0 - m
            elif kind == 6:                     # quantised values: many ties everywhere
                m[...] = np.round(m * 4) / 4
    return hm


@pytest.mark.parametrize("h,w", [(64, 64), (64, 48), (96, 72)])
@pytest.mark.parametrize("pp", [True, False])
def test_final_preds_and_pck_equal_host_on_random_maps(h, w, pp):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.lib.core.evaluate import accuracy, pck_from_counts
    from fpd_b200.lib.core.inference import get_final_preds
    rng = np.random.RandomState(h * 1000 + w + int(pp))
    B, J = 12, 17
    for rep in range(2):
        hm = torch.from_numpy(_random_maps(rng, B, J, h, w)).cuda()
        c = rng.uniform(0, 800, (B, 2)).astype(np.float32)
        s = rng.uniform(0.2, 4.0, (B, 2)).astype(np.float32)
        ref_p, ref_m = get_final_preds(_cfg_pp(pp), hm, c, s)
        got = _device_decode(hm, c, s, pp)
        assert np.array_equal(got[..., :2], ref_p, equal_nan=True), np.nanmax(np.abs(got[..., :2] - ref_p))
        assert np.array_equal(got[..., 2:], ref_m, equal_nan=True)
        tgt = torch.from_numpy(_random_maps(rng, B, J, h, w)).cuda()
        acc, avg, cnt, pred = accuracy(hm, tgt)
        _, idx, mv = ops.flip_merge_argmax(ops.nchw_to_nhwc(hm), want_avg=False)
        counts, pred_hm = ops.pck_counts(idx, mv, tgt, want_pred_hm=True)
        acc2, avg2, cnt2 = pck_from_counts(counts.cpu().numpy())
        assert np.array_equal(acc2, acc) and avg2 == avg and cnt2 == cnt
        assert np.array_equal(pred_hm.cpu().numpy(), pred)


def test_new_entry_points_refuse_bad_arguments():
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    from fpd_b200 import ops
    avg = torch.zeros(1, 2, 2, 65, device="cuda")
    idx = torch.zeros(1, 65, dtype=torch.int32, device="cuda")
    mv = torch.zeros(1, 65, device="cuda")
    inv = torch.zeros(1, 6, dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError, match="J=65"):
        ops.final_preds(avg, idx, mv, inv, False)
    with pytest.raises(RuntimeError, match="J=65"):
        ops.pck_counts(idx, mv, torch.zeros(1, 65, 2, 2, device="cuda"))
    with pytest.raises(RuntimeError, match="3x3"):
        ops.final_preds(torch.zeros(1, 2, 2, 4, device="cuda"), idx[:, :4].contiguous(), mv[:, :4].contiguous(), inv, True)
    with pytest.raises(ValueError):
        ops.final_preds(torch.zeros(1, 4, 4, 4, device="cuda"), idx[:, :4].contiguous(), mv[:, :4].contiguous(),
                        inv.float(), True)
    assert N.lib().fpd_final_preds(None, None, None, None, 0, None, 1, 4, 4, 4, None) != 0


# ----------------------------------------------------------------------------------------------- networks
FLIP_PAIRS = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]


def _hourglass():
    from fpd_b200.lib.models import hourglass as H
    cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=2, NUM_BLOCKS=1), NUM_JOINTS=16, NAME="hourglass"))
    return H.get_pose_net(cfg, True), (128, 128), 16


def _hrnet():
    from fpd_b200.lib.models import pose_hrnet as H

    def stage(nmod, chans):
        return dict(NUM_MODULES=nmod, NUM_BRANCHES=len(chans), BLOCK='BASIC', NUM_BLOCKS=[1] * len(chans),
                    NUM_CHANNELS=chans, FUSE_METHOD='SUM')
    from bench import _wrap
    cfg = _wrap(dict(MODEL=dict(NUM_JOINTS=17, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=dict(
        PRETRAINED_LAYERS=['*'], FINAL_CONV_KERNEL=1, STAGE2=stage(1, [8, 16]), STAGE3=stage(2, [8, 16, 32]),
        STAGE4=stage(1, [8, 16, 32, 64])))))
    return H.get_pose_net(cfg, is_train=False), (128, 96), 17


def _resnet():
    from fpd_b200.lib.models import pose_resnet as R
    cfg = NS(MODEL=NS(NUM_JOINTS=16, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=NS(
        NUM_LAYERS=18, DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[64, 64, 64],
        NUM_DECONV_KERNELS=[4, 4, 4], FINAL_CONV_KERNEL=1)))
    return R.get_pose_net(cfg, is_train=False), (128, 128), 16


NETS = {"hourglass": _hourglass, "hrnet": _hrnet, "resnet": _resnet}


def _build(kind):
    import fpd_b200  # noqa: F401
    torch.manual_seed(11)
    net, hw, J = NETS[kind]()
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    return net.cuda(), hw, J


def _batch(B, seed, hw, J):
    from bench import synthetic_batch
    x, t, w = synthetic_batch(B, seed, hw[0], hw[1], J)
    rng = np.random.RandomState(seed)
    meta = {"center": torch.from_numpy(rng.uniform(100, 500, (B, 2))), "scale": torch.from_numpy(rng.uniform(0.5, 3, (B, 2))),
            "score": torch.from_numpy(rng.uniform(0.5, 1, B)), "image": ["img%d_%d" % (seed, b) for b in range(B)]}
    return x, t, w, meta


def _eager(net, x, t, w, meta, perm, flip, shift, pp, use_tw=True):
    """What validate()'s eager fused route computes for one batch."""
    from fpd_b200 import ops
    from fpd_b200.lib.core.evaluate import accuracy
    from fpd_b200.lib.core.inference import get_final_preds
    from fpd_b200.lib.core.loss import JointsMSELoss
    xd = x.cuda().float().contiguous()
    hm = net.forward_nhwc(xd, training=False)[-1]
    hm_f = net.forward_nhwc(xd.flip(3).contiguous(), training=False)[-1] if flip else None
    avg, _, _ = ops.flip_merge_argmax(hm, hm_f, perm if flip else None, shift=shift)
    out = ops.nhwc_to_nchw(avg)
    loss = JointsMSELoss(use_tw)(out, t.cuda(), w.cuda()).item()
    _, avg_acc, cnt, _ = accuracy(out, t.cuda())
    preds, maxvals = get_final_preds(_cfg_pp(pp), out, meta["center"].numpy(), meta["scale"].numpy())
    return loss, avg_acc, cnt, np.concatenate([preds, maxvals], -1)


@pytest.mark.parametrize("use_graph", [True, False])
def test_flip_test_inference_decode_equals_eager(use_graph):
    from fpd_b200.infer_step import FlipTestInference
    from fpd_b200.lib.core.evaluate import pck_from_counts
    from fpd_b200.lib.core.inference import inverse_affines
    net, hw, J = _build("hourglass")
    perm = torch.tensor([dict(sum([[(a, b), (b, a)] for a, b in FLIP_PAIRS], [])).get(j, j) for j in range(J)],
                        dtype=torch.int32, device="cuda")
    run = FlipTestInference(net, FLIP_PAIRS, shift_heatmap=True, flip_test=True, use_graph=use_graph, decode=True)
    # two replays of one graph with different inputs, then a smaller batch (re-capture), then the first shape again
    for B, seed, use_tw in ((3, 1, True), (3, 2, True), (2, 3, True), (3, 4, False)):
        x, t, w, meta = _batch(B, seed, hw, J)
        c, s = meta["center"].numpy(), meta["scale"].numpy()
        h_, w_ = t.shape[2:]
        r = run(x, inv=inverse_affines(c, s, [w_, h_]), target=t, target_weight=w, use_target_weight=use_tw,
                post_process=True)
        got = (float(r["loss3"][0]),) + pck_from_counts(r["pck"].cpu().numpy())[1:] + (r["preds"].cpu().numpy(),)
        ref = _eager(net, x, t, w, meta, perm, True, True, True, use_tw)
        assert got[0] == ref[0] and got[1] == ref[1] and got[2] == ref[2], (got[:3], ref[:3])
        assert np.array_equal(got[3], ref[3])


class _ValSet:
    def __init__(self, n, J):
        self.n = n
        self.flip_pairs = [p for p in FLIP_PAIRS if max(p) < J]
        self.seen = None

    def __len__(self):
        return self.n

    def evaluate(self, cfg, preds, output_dir, all_boxes, image_path, filenames, imgnums):
        self.seen = (preds.copy(), all_boxes.copy(), list(image_path))
        return {"Mean": float(preds[..., :2].mean())}, float(preds[..., :2].mean())


class _Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, v, step):
        self.scalars.append((tag, v, step))

    def add_scalars(self, tag, d, step):
        pass


@pytest.fixture(scope="module")
def nets():
    return {k: _build(k) for k in NETS}


@pytest.mark.parametrize("kind", list(NETS))
@pytest.mark.parametrize("flip", [True, False])
@pytest.mark.parametrize("pp", [True, False])
def test_validate_graph_route_equals_eager_route(nets, kind, flip, pp, monkeypatch):
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    net, hw, J = nets[kind]
    loader = [_batch(3, 20, hw, J), _batch(3, 21, hw, J), _batch(2, 22, hw, J)]      # last batch partial
    cfg = NS(MODEL=NS(NUM_JOINTS=J, NAME=kind), PRINT_FREQ=2, DEBUG=NS(DEBUG=False),
             TEST=NS(FLIP_TEST=flip, SHIFT_HEATMAP=True, POST_PROCESS=pp))
    runs = []
    for graph in (True, False):
        monkeypatch.setattr(F, "_VALIDATE_GRAPH", graph)
        calls = []
        orig = F._GraphValidation.run
        monkeypatch.setattr(F._GraphValidation, "run", lambda self, *a: calls.append(1) or orig(self, *a))
        ds = _ValSet(8, J)
        wd = {"writer": _Writer(), "valid_global_steps": 0}
        perf = F.validate(cfg, loader, ds, net, JointsMSELoss(True), "/tmp", "/tmp", wd)
        assert len(calls) == (3 if graph else 0)
        runs.append((perf, ds.seen, wd["writer"].scalars))
    (pg, sg, wg), (pe, se, we) = runs
    assert np.array_equal(sg[0], se[0]) and np.array_equal(sg[1], se[1]) and sg[2] == se[2]
    assert pg == pe
    assert wg == we and {t for t, _, _ in wg} == {"valid_loss", "valid_acc"}


def test_validate_falls_back_to_eager_for_debug_and_odd_shapes(nets, monkeypatch):
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    target = torch.zeros(2, 16, 32, 32)
    cfg = NS(DEBUG=NS(DEBUG=False))
    assert F._validate_graph_ok(cfg, JointsMSELoss(True), target)
    assert not F._validate_graph_ok(NS(DEBUG=NS(DEBUG=True)), JointsMSELoss(True), target)
    assert not F._validate_graph_ok(cfg, JointsMSELoss(True), torch.zeros(2, 65, 32, 32))
    assert not F._validate_graph_ok(cfg, JointsMSELoss(True), torch.zeros(2, 16, 30, 30))
    assert not F._validate_graph_ok(cfg, torch.nn.MSELoss(), target)
    monkeypatch.setattr(F, "_VALIDATE_GRAPH", False)
    assert not F._validate_graph_ok(cfg, JointsMSELoss(True), target)
