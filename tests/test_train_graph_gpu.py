"""train() / fpd_train() through one CUDA graph replay per batch (lib/core/function.py _GraphTraining, FPDTrainStep in its
external-optimizer mode) against the eager fused route, from the same initial state: parameters, BatchNorm running
statistics, the caller's optimizer state and every meter update must be bit-identical."""
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _cfg(print_freq=1, J=16):
    return NS(MODEL=NS(NUM_JOINTS=J, NAME="net"), KD=NS(ALPHA=0.5), PRINT_FREQ=print_freq, DEBUG=NS(DEBUG=False),
              TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True))


def _hourglass(f, s):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as H
    return H.get_pose_net(NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=16)), True)


def _hrnet():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import pose_hrnet as H
    from bench import _wrap

    def stage(nmod, chans):
        return dict(NUM_MODULES=nmod, NUM_BRANCHES=len(chans), BLOCK='BASIC', NUM_BLOCKS=[1] * len(chans),
                    NUM_CHANNELS=chans, FUSE_METHOD='SUM')
    cfg = _wrap(dict(MODEL=dict(NUM_JOINTS=17, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=dict(
        PRETRAINED_LAYERS=['*'], FINAL_CONV_KERNEL=1, STAGE2=stage(1, [8, 16]), STAGE3=stage(2, [8, 16, 32]),
        STAGE4=stage(1, [8, 16, 32, 64])))))
    return H.get_pose_net(cfg, is_train=False)


def _resnet():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import pose_resnet as R
    cfg = NS(MODEL=NS(NUM_JOINTS=16, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=NS(
        NUM_LAYERS=18, DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[64, 32, 32],
        NUM_DECONV_KERNELS=[4, 4, 4], FINAL_CONV_KERNEL=1)))
    return R.get_pose_net(cfg, is_train=False)


def _loader(n_full, B=2, hw=(128, 128), J=16, short=1, seed=70):
    """n_full batches of B samples, then (short > 0) one batch of `short` samples."""
    from bench import synthetic_batch
    sizes = [B] * n_full + ([short] if short else [])
    out = []
    for i, b in enumerate(sizes):
        x, t, w = synthetic_batch(b, seed + i, hw[0], hw[1], J)
        meta = {"center": torch.tensor([[64.0, 64.0]] * b), "scale": torch.tensor([[0.64, 0.64]] * b),
                "score": torch.ones(b), "image": ["img%d_%d" % (i, k) for k in range(b)]}
        out.append((x, t, w, meta))
    return out


class _Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, v, step):
        self.scalars.append((tag, float(v), step))

    def add_scalars(self, tag, d, step):
        pass


@pytest.fixture
def F(monkeypatch):
    """lib.core.function with AverageMeter.update recorded (meter index within its call, value, n) and the routes
    counted."""
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    F._train_step_cache.clear()
    log, created, counts = [], [], {"graph": 0, "eager": 0, "capture": 0}

    class RecMeter(F.AverageMeter):
        def __init__(self):
            self.idx = len(created)
            created.append(self)
            super().__init__()

        def update(self, val, n=1):
            log.append((self.idx, val, n))
            super().update(val, n)
    monkeypatch.setattr(F, "AverageMeter", RecMeter)
    fused = F._fused_step

    def count(*a, **k):
        route = "eager" if (a[7] if len(a) > 7 else k.get("graph")) is None else "graph"
        counts[route] += 1
        return fused(*a, **k)
    monkeypatch.setattr(F, "_fused_step", count)
    from fpd_b200 import train_step
    cap = train_step.FPDTrainStep._capture
    monkeypatch.setattr(train_step.FPDTrainStep, "_capture",
                        lambda self, *a: counts.__setitem__("capture", counts["capture"] + 1) or cap(self, *a))
    F._rec = (log, created, counts)
    yield F
    F._train_step_cache.clear()


def _call(F, graph, fn, *args):
    """One train / fpd_train call; returns its loss / accuracy meter updates (time meters dropped) and writer scalars."""
    log, created, _ = F._rec
    F._TRAIN_GRAPH = graph
    try:
        log.clear()
        created.clear()
        wd = {"writer": _Writer(), "train_global_steps": 0}
        fn(*args[:-1], wd) if args[-1] == "wd" else fn(*args)
        torch.cuda.synchronize()
        updates = [(idx, val, n) for idx, val, n in log if idx >= 2]      # 0, 1: batch_time, data_time
        return updates, wd["writer"].scalars
    finally:
        F._TRAIN_GRAPH = True


def _state(net, opt):
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    ost = {}
    for i, p in enumerate(q for g in opt.param_groups for q in g["params"]):
        for k, v in opt.state.get(p, {}).items():
            ost[(i, k)] = v.clone() if torch.is_tensor(v) else v
    return sd, ost


def _assert_same(a, b):
    (sd_a, os_a), (sd_b, os_b) = a, b
    assert sd_a.keys() == sd_b.keys()
    for k in sd_a:
        assert torch.equal(sd_a[k], sd_b[k]), k
    assert os_a.keys() == os_b.keys() and len(os_a) > 0
    for k in os_a:
        va, vb = os_a[k], os_b[k]
        assert (torch.equal(va, vb) if torch.is_tensor(va) else va == vb), k


def _fpd_run(F, graph, init_s, init_t, loader, crits, print_freq=1, opt_fn=None, epochs=1, between=None):
    s, t = _hourglass(64, 2), _hourglass(64, 1)
    s.load_state_dict(init_s)
    t.load_state_dict(init_t)
    s, t = s.cuda(), t.cuda()
    opt = (opt_fn or (lambda ps: torch.optim.Adam(ps, lr=1e-3)))(list(s.parameters()))
    cfg = _cfg(print_freq)
    rec = []
    for e in range(epochs):
        if between is not None and e > 0:
            between(e, s, t, opt)
        rec.append(_call(F, graph, F.fpd_train, cfg, loader, s, t, crits[0], crits[1], opt, e, "/tmp", "/tmp", "wd"))
    return _state(s, opt), rec, (s, t, opt)


def _inits(seed=5):
    torch.manual_seed(seed)
    return ({k: v.clone() for k, v in _hourglass(64, 2).state_dict().items()},
            {k: v.clone() for k, v in _hourglass(64, 1).state_dict().items()})


@pytest.mark.parametrize("print_freq", [1, 100])
def test_fpd_train_graph_route_equals_eager_route(F, print_freq):
    from fpd_b200.lib.core.loss import JointsMSELoss
    init_s, init_t = _inits()
    loader = _loader(4, short=1)
    crits = (JointsMSELoss(True), JointsMSELoss(True))
    counts = F._rec[2]
    st_e, rec_e, _ = _fpd_run(F, False, init_s, init_t, loader, crits, print_freq)
    assert counts == {"graph": 0, "eager": 5, "capture": 0}
    st_g, rec_g, _ = _fpd_run(F, True, init_s, init_t, loader, crits, print_freq)
    assert counts == {"graph": 4, "eager": 6, "capture": 1}      # the short last batch took the eager route
    _assert_same(st_g, st_e)
    assert rec_g == rec_e
    assert len(rec_g[0][0]) == 4 * 5 and {i for i, _, _ in rec_g[0][0]} == {2, 3, 4, 5}


@pytest.mark.parametrize("topks", [(8, 0), (8, 8)])
def test_fpd_train_graph_route_with_ohkm(F, topks):
    from fpd_b200.lib.core.loss import JointsMSELoss, JointsOHKMMSELoss
    init_s, init_t = _inits(6)
    loader = _loader(3, short=1)

    def crit(k):
        return JointsOHKMMSELoss(True, topk=k) if k else JointsMSELoss(True)
    crits = (crit(topks[0]), crit(topks[1]))
    st_e, rec_e, _ = _fpd_run(F, False, init_s, init_t, loader, crits)
    st_g, rec_g, _ = _fpd_run(F, True, init_s, init_t, loader, crits)
    assert F._rec[2]["graph"] == 3
    step = next(iter(F._train_step_cache.values()))
    assert (step.pose_topk, step.kd_topk) == topks
    _assert_same(st_g, st_e)
    assert rec_g == rec_e


@pytest.mark.parametrize("kind", ["hrnet", "pose_resnet"])
def test_train_graph_route_equals_eager_route(F, kind):
    from fpd_b200.lib.core.loss import JointsMSELoss
    torch.manual_seed(8)
    build, hw, J = {"hrnet": (_hrnet, (128, 96), 17), "pose_resnet": (_resnet, (128, 128), 16)}[kind]
    init = {k: v.clone() for k, v in build().state_dict().items()}
    loader = _loader(3, hw=hw, J=J, short=1)
    runs = []
    for graph in (False, True):
        net = build()
        net.load_state_dict(init)
        net = net.cuda()
        opt = torch.optim.Adam(net.parameters(), lr=1e-3)
        rec = _call(F, graph, F.train, _cfg(2, J), loader, net, JointsMSELoss(True), opt, 0, "/tmp", "/tmp", "wd")
        runs.append((_state(net, opt), rec))
    assert F._rec[2]["graph"] == 3
    _assert_same(runs[1][0], runs[0][0])
    assert runs[1][1] == runs[0][1]


def test_two_epochs_sgd_multistep_lr_reuse_the_graph(F):
    from fpd_b200.lib.core.loss import JointsMSELoss
    init_s, init_t = _inits(9)
    loader = _loader(3, short=0)
    crits = (JointsMSELoss(True), JointsMSELoss(True))
    lrs = {}

    def opt_fn(ps):
        opt = torch.optim.SGD(ps, lr=1e-2, momentum=0.9, nesterov=True, weight_decay=1e-4)
        opt._sched = torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[1], gamma=0.1)
        return opt

    def between(e, s, t, opt):
        opt._sched.step()
        lrs.setdefault(e, []).append(opt.param_groups[0]["lr"])
    st_e, rec_e, _ = _fpd_run(F, False, init_s, init_t, loader, crits, opt_fn=opt_fn, epochs=2, between=between)
    st_g, rec_g, _ = _fpd_run(F, True, init_s, init_t, loader, crits, opt_fn=opt_fn, epochs=2, between=between)
    assert F._rec[2]["capture"] == 1 and F._rec[2]["graph"] == 6          # one capture serves both epochs
    assert lrs[1][0] == lrs[1][1] and abs(lrs[1][0] - 1e-3) < 1e-12
    assert any(k[1] == "momentum_buffer" for k in st_g[1])
    _assert_same(st_g, st_e)
    assert rec_g == rec_e


def test_frozen_parameter_keeps_its_grad_and_value(F):
    from fpd_b200.lib.core.loss import JointsMSELoss
    init_s, init_t = _inits(10)
    loader = _loader(2, short=0)
    crits = (JointsMSELoss(True), JointsMSELoss(True))
    out = []
    for graph in (False, True):
        def opt_fn(ps):
            frozen = dict(_hourglass_named(ps))["hg.0.hg.0.1.0.conv2.weight"]
            frozen.requires_grad_(False)
            frozen.grad = torch.full_like(frozen, 7.0)
            out.append(frozen)
            return torch.optim.Adam([p for p in ps if p.requires_grad], lr=1e-3)
        st, _, _ = _fpd_run(F, graph, init_s, init_t, loader, crits, opt_fn=opt_fn)
        out.append(st)
    fe, st_e, fg, st_g = out
    for p in (fe, fg):
        assert torch.equal(p.grad, torch.full_like(p, 7.0))
        assert torch.equal(p.detach().cpu(), init_s["hg.0.hg.0.1.0.conv2.weight"])
    _assert_same(st_g, st_e)


_NAMES = None


def _hourglass_named(ps):
    """Parameter names for a list of the s2 f64 student's parameters, in module order."""
    global _NAMES
    if _NAMES is None:
        _NAMES = [k for k, _ in _hourglass(64, 2).named_parameters()]
    return zip(_NAMES, ps)


def test_parameters_keep_their_storage_and_optimizer_state_round_trips(F):
    from fpd_b200.lib.core.loss import JointsMSELoss
    init_s, init_t = _inits(11)
    loader = _loader(2, short=0)
    crits = (JointsMSELoss(True), JointsMSELoss(True))
    results = []
    for graph in (False, True):
        st, _, (s, t, opt) = _fpd_run(F, graph, init_s, init_t, loader, crits)
        if graph:
            bases = [v.untyped_storage().data_ptr() for v in s.state_dict().values()]
            assert len(set(bases)) == len(bases), "parameters were re-homed into a shared buffer"
        # checkpoint the optimizer, continue from the reloaded copy
        sd = opt.state_dict()
        opt2 = torch.optim.Adam(s.parameters(), lr=1e-3)
        opt2.load_state_dict(sd)
        _call(F, graph, F.fpd_train, _cfg(1), loader, s, t, crits[0], crits[1], opt2, 1, "/tmp", "/tmp", "wd")
        results.append(_state(s, opt2))
    _assert_same(results[1], results[0])


def test_teacher_reload_and_new_student_storage_capture_again(F):
    from fpd_b200.lib.core.loss import JointsMSELoss
    init_s, init_t = _inits(12)
    torch.manual_seed(13)
    other_t = {k: v.clone() for k, v in _hourglass(64, 1).state_dict().items()}
    loader = _loader(2, short=0)
    crits = (JointsMSELoss(True), JointsMSELoss(True))

    def between(e, s, t, opt):
        if e == 1:
            t.load_state_dict(other_t)
        else:
            p = s.score[0].weight
            p.data = p.data.clone()           # same Parameter object (the optimizer still holds it), new storage
    st_e, rec_e, _ = _fpd_run(F, False, init_s, init_t, loader, crits, epochs=3, between=between)
    st_g, rec_g, _ = _fpd_run(F, True, init_s, init_t, loader, crits, epochs=3, between=between)
    assert F._rec[2]["capture"] == 3 and F._rec[2]["graph"] == 6
    _assert_same(st_g, st_e)
    assert rec_g == rec_e


class _ValSet:
    flip_pairs = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]

    def __init__(self, n):
        self.n = n
        self.seen = None

    def __len__(self):
        return self.n

    def evaluate(self, cfg, preds, output_dir, all_boxes, image_path, filenames, imgnums):
        self.seen = (preds.copy(), all_boxes.copy(), list(image_path))
        return {"Mean": float(preds[..., :2].mean())}, float(preds[..., :2].mean())


def test_validate_after_fpd_train_sees_the_update(F):
    from fpd_b200.lib.core.loss import JointsMSELoss
    init_s, init_t = _inits(14)
    loader = _loader(3, short=1)
    crits = (JointsMSELoss(True), JointsMSELoss(True))
    seen = []
    for graph in (False, True):
        _, _, (s, t, opt) = _fpd_run(F, graph, init_s, init_t, loader, crits)
        ds = _ValSet(7)
        wd = {"writer": _Writer(), "valid_global_steps": 0}
        perf = F.validate(_cfg(2), loader, ds, s, crits[0], "/tmp", "/tmp", wd)
        seen.append((perf, ds.seen, wd["writer"].scalars))
    (pe, se, we), (pg, sg, wg) = seen
    assert pe == pg and we == wg
    assert np.array_equal(se[0], sg[0]) and np.array_equal(se[1], sg[1]) and se[2] == sg[2]


def test_train_step_topk_graph_equals_eager_and_matches_fpd_loss():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.train_step import FPDTrainStep
    from bench import synthetic_batch
    init_s, init_t = _inits(15)
    batches = [tuple(v.cuda() for v in synthetic_batch(2, 40 + i, 128, 128)) for i in range(3)]
    res = []
    for use_graph in (False, True):
        s, t = _hourglass(64, 2), _hourglass(64, 1)
        s.load_state_dict(init_s)
        t.load_state_dict(init_t)
        s, t = s.cuda(), t.cuda()
        step = FPDTrainStep(s, t, alpha=0.5, lr=1e-3, use_graph=use_graph, pose_topk=8, kd_topk=8)
        losses = []
        for x, tgt, tw in batches:
            losses.append(step.step(x, tgt, tw).clone())
            if not use_graph:
                ref, _ = ops.fpd_loss(step.last_outs, tgt, step.last_teacher, tw.reshape(2, -1), 0.5, want_grads=False,
                                      pose_topk=8, kd_topk=8)
                assert torch.equal(losses[-1], ref)
                plain, _ = ops.fpd_loss(step.last_outs, tgt, step.last_teacher, tw.reshape(2, -1), 0.5, want_grads=False)
                assert not torch.equal(losses[-1], plain)
        torch.cuda.synchronize()
        res.append((step.flat.flat.clone(), step.exp_avg.clone(), step.exp_avg_sq.clone(), torch.stack(losses),
                    [b.clone() for b in s.buffers()]))
    (fe, ae, be, le, bufe), (fg, ag, bg, lg, bufg) = res
    assert torch.equal(fe, fg) and torch.equal(ae, ag) and torch.equal(be, bg) and torch.equal(le, lg)
    assert all(torch.equal(a, b) for a, b in zip(bufe, bufg))


# ------------------------------------------------------------------------------------------------ two ranks
def _ddp_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    init_s, init_t = _inits(16)
    loader = _loader(3, short=1, seed=200 + 10 * rank)            # each rank its own shard
    states = []
    for graph in (False, True):
        F._TRAIN_GRAPH = graph
        s, t = _hourglass(64, 2), _hourglass(64, 1)
        s.load_state_dict(init_s)
        t.load_state_dict(init_t)
        s, t = s.cuda(), t.cuda()
        opt = torch.optim.Adam(s.parameters(), lr=1e-3)
        F.fpd_train(_cfg(1), loader, s, t, JointsMSELoss(True), JointsMSELoss(True), opt, 0, "/tmp", "/tmp", None)
        torch.cuda.synchronize()
        states.append(_state(s, opt))
    try:
        _assert_same(states[1], states[0])
        same = True
    except AssertionError:
        same = False
    flat = torch.cat([v.flatten().float() for v in states[1][0].values()])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    q.put((rank, same, all(torch.equal(gathered[0], g) for g in gathered)))
    q.close()
    q.join_thread()
    dist.barrier()
    torch.cuda.synchronize()
    os._exit(0)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_fpd_train_graph_route_equals_eager_route():
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29800 + os.getpid() % 1000
    procs = [ctx.Process(target=_ddp_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, same, replicas in res:
        assert same, "rank %d: graph route differs from the eager route" % rank
        assert replicas, "replicas diverged"
