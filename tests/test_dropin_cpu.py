"""The documented drop-in wiring (INTEGRATION.md section 1): the reference's lib/ on sys.path as tools/_init_paths.py
leaves it, then fpd_b200.dropin.install() -- and every import tools/fpd_train.py / tools/train.py / tools/test.py perform
must still resolve, hot-path modules to fpd_b200 and everything else to the reference. Runs in a subprocess (it rewires
sys.modules). Needs /root/reference (build container only)."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"

SCRIPT = textwrap.dedent('''
    import sys, types
    REF, ROOT = %r, %r
    # third-party packages the reference imports that this image lacks: minimal stand-ins (control plane only)
    class CN(dict):
        def __init__(self, init=None, new_allowed=False, **kw):
            super().__init__(init or {})
        __getattr__ = lambda self, k: self[k] if k in self else (_ for _ in ()).throw(AttributeError(k))
        __setattr__ = dict.__setitem__
        def defrost(self): pass
        def freeze(self): pass
        def merge_from_file(self, f): pass
        def merge_from_list(self, l): pass
    def stub(name, **attrs):
        m = types.ModuleType(name); m.__dict__.update(attrs); sys.modules[name] = m; return m
    for name in ("yacs", "json_tricks", "tensorboardX", "pycocotools", "easydict"):
        try:
            __import__(name)
        except ImportError:
            stub(name)
    if not hasattr(sys.modules["yacs"], "config"):
        sys.modules["yacs"].config = stub("yacs.config", CfgNode=CN)
    if not hasattr(sys.modules["tensorboardX"], "SummaryWriter"):
        sys.modules["tensorboardX"].SummaryWriter = object
    if "pycocotools.coco" not in sys.modules:
        sys.modules["pycocotools"].coco = stub("pycocotools.coco", COCO=object)
        sys.modules["pycocotools"].cocoeval = stub("pycocotools.cocoeval", COCOeval=object)
    # --- what tools/_init_paths.py does, plus the two documented lines
    sys.path.insert(0, REF + "/lib")
    sys.path.insert(0, ROOT)
    import fpd_b200
    from fpd_b200 import dropin
    dropin.install()
    # --- tools/fpd_train.py:27-40, tools/test.py:24-33
    from config import cfg
    from config import update_config
    from core.loss import JointsMSELoss
    from core.function import train, fpd_train, validate
    from utils.utils import get_optimizer, save_checkpoint, create_logger, get_model_summary
    import dataset
    import models
    ours = lambda o: o.__module__.startswith("fpd_b200.")
    assert ours(JointsMSELoss) and ours(train) and ours(fpd_train) and ours(validate)
    assert not ours(get_optimizer)
    for name in ("hourglass", "pose_hrnet", "pose_resnet"):
        assert ours(eval("models." + name + ".get_pose_net")), name
    # modules the reference's dataset / vis code needs from the packages we touch
    from utils.transforms import get_affine_transform, affine_transform, fliplr_joints, transform_preds, flip_back
    assert not ours(get_affine_transform) and ours(flip_back)
    from utils.vis import save_debug_images
    from nms.nms import oks_nms, soft_oks_nms, gpu_nms_wrapper, py_nms_wrapper, cpu_nms_wrapper, nms
    C = sys.modules["dataset.coco"]        # `dataset.coco` itself is the class alias (dataset/__init__.py)
    assert ours(C.oks_nms) and ours(C.soft_oks_nms) and ours(oks_nms)
    assert dataset.mpii.__module__ == "dataset.mpii" and dataset.coco.__module__ == "dataset.coco"
    from core.inference import get_final_preds, get_max_preds
    from core.evaluate import accuracy
    assert ours(get_final_preds) and ours(accuracy)
    import utils.vis as V
    assert ours(V.get_max_preds)            # utils/vis.py:17 binds the replaced core.inference
    # the factory works on the reference's config objects and yields the reference's state_dict keys
    import types as T
    c = T.SimpleNamespace(MODEL=T.SimpleNamespace(EXTRA=T.SimpleNamespace(NUM_FEATURES=64, NUM_STACKS=1, NUM_BLOCKS=1),
                                                  NUM_JOINTS=16))
    net = models.hourglass.get_pose_net(c, is_train=True)
    assert "hg.0.hg.3.0.0.conv2.weight" in net.state_dict()
    # checkpoint formats : the reference's OWN save_checkpoint / load_checkpoint (utils/utils.py:74-86,
    # 204-251: plain state_dict, DataParallel 'module.'-prefixed, and the {'state_dict': ...} training checkpoint, plus the
    # filter_keys partial load the FPD student uses) round-trip through the drop-in modules of all three families
    import os, tempfile, torch
    from utils.utils import load_checkpoint
    rcfg = T.SimpleNamespace(MODEL=T.SimpleNamespace(NUM_JOINTS=16, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=T.SimpleNamespace(
        NUM_LAYERS=18, DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=2, NUM_DECONV_FILTERS=[32, 32], NUM_DECONV_KERNELS=[4, 4],
        FINAL_CONV_KERNEL=1)))
    with tempfile.TemporaryDirectory() as d:
        for mk in (lambda: models.hourglass.get_pose_net(c, is_train=False),
                   lambda: models.pose_resnet.get_pose_net(rcfg, is_train=False)):
            src, dst = mk(), mk()
            for p_ in src.parameters():
                p_.data.normal_()
            sd = src.state_dict()
            opt = get_optimizer(T.SimpleNamespace(TRAIN=T.SimpleNamespace(OPTIMIZER='adam', LR=1e-3)), src)
            save_checkpoint({'epoch': 3, 'model': 'x', 'state_dict': sd, 'best_state_dict': sd, 'perf': 0.5,
                             'optimizer': opt.state_dict()}, True, d)
            assert os.path.exists(os.path.join(d, 'checkpoint.pth')) and os.path.exists(os.path.join(d, 'model_best.pth'))
            load_checkpoint(os.path.join(d, 'checkpoint.pth'), dst, model_info='ckpt')            # training checkpoint
            assert all(torch.equal(sd[k], v) for k, v in dst.state_dict().items())
            dst = mk()
            torch.save({'module.' + k: v for k, v in sd.items()}, os.path.join(d, 'dp.pth'))      # DataParallel keys
            load_checkpoint(os.path.join(d, 'dp.pth'), dst, model_info='dp')
            assert all(torch.equal(sd[k], v) for k, v in dst.state_dict().items())
            dst = mk()
            load_checkpoint(os.path.join(d, 'model_best.pth'), dst, strict=False, filter_keys='bn1', model_info='part')
            assert all(torch.equal(sd[k], v) for k, v in dst.state_dict().items() if 'bn1' not in k)
            assert not torch.equal(sd['bn1.weight'], dst.state_dict()['bn1.weight'])
    # shadowing guard: our lib/ on sys.path is refused loudly
    dropin.uninstall()
    for k in [k for k in sys.modules if k.split(".")[0] in ("models", "core", "nms", "utils", "dataset")]:
        del sys.modules[k]
    sys.path.insert(0, ROOT + "/fast-human-pose-estimation.pytorch_b200/lib")
    try:
        dropin.install()
    except dropin.DropInError:
        pass
    else:
        raise AssertionError("install() must refuse a shadowing sys.path")
    print("DROPIN-OK")
''')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "lib")), reason="needs the reference checkout")
def test_reference_tool_imports_resolve_after_install():
    r = subprocess.run([sys.executable, "-c", SCRIPT % (REF, ROOT)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "DROPIN-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
