"""Wire the H100 hot path under the reference's tools WITHOUT shadowing its packages.

The reference resolves everything by module name after tools/_init_paths.py put `<reference>/lib` on sys.path
(tools/fpd_train.py:27-40: `from core.function import train, fpd_train, validate`, `from core.loss import
JointsMSELoss`, `eval('models.' + cfg.MODEL.NAME + '.get_pose_net')`, `import dataset` -> `from nms.nms import oks_nms`).
`install()` replaces exactly the hot-path MODULES in `sys.modules` (and the matching attributes of their parent
packages) and leaves everything else -- config, dataset, utils.utils, utils.vis, utils.transforms' affine helpers --
the reference's own:

    models.hourglass, .pose_hrnet, .pose_resnet -> fpd_b200.lib.models.*      (get_pose_net + forward)
    core.function                              -> fpd_b200.lib.core.function  (train / fpd_train / validate)
    core.loss, core.inference, core.evaluate   -> fpd_b200.lib.core.*
    nms.nms                                    -> fpd_b200.lib.nms.nms        (gpu_nms, oks_nms, ... full API)
    utils.transforms.flip_back                 -> device-aware flip_back (attribute patch; module stays the reference's)

Call it once, right after `import _init_paths` and before the first `from core... import` / `import models`.
"""
import importlib
import importlib.util
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))

_REPLACED = {
    "models.hourglass": "fpd_b200.lib.models.hourglass",
    "models.pose_hrnet": "fpd_b200.lib.models.pose_hrnet",
    "models.pose_resnet": "fpd_b200.lib.models.pose_resnet",
    "core.function": "fpd_b200.lib.core.function",
    "core.loss": "fpd_b200.lib.core.loss",
    "core.inference": "fpd_b200.lib.core.inference",
    "core.evaluate": "fpd_b200.lib.core.evaluate",
    "nms.nms": "fpd_b200.lib.nms.nms",
}


class DropInError(RuntimeError):
    pass


def _reference_package(name):
    """Import the reference's package `name` (must resolve outside this repo: our own lib/ must NOT be on sys.path)."""
    spec = importlib.util.find_spec(name)
    if spec is None:
        raise DropInError("package %r not importable: put the reference's lib/ on sys.path first (tools/_init_paths.py)"
                          % name)
    locs = list(spec.submodule_search_locations or [])
    if any(os.path.abspath(p).startswith(_HERE) for p in locs):
        raise DropInError("package %r resolves inside fpd_b200 (%s): do not put fast-human-pose-estimation.pytorch_b200/lib "
                          "on sys.path -- it would shadow the reference's packages; use fpd_b200.dropin.install()" %
                          (name, locs))
    return importlib.import_module(name)


def install(verbose=False):
    """Idempotent. Returns {reference module name: replacement module}."""
    done = {}
    # 1. seed sys.modules first, so that `import models` (whose __init__ imports models.hourglass / models.pose_hrnet,
    #    reference lib/models/__init__.py:15-17) and `import dataset` (coco.py:24-25 -> nms.nms) bind to the replacements
    for ref_name, ours in _REPLACED.items():
        mod = importlib.import_module(ours)
        sys.modules[ref_name] = mod
        done[ref_name] = mod
    # 2. parent packages are the reference's; point their attributes at the replacements
    for ref_name, mod in done.items():
        pkg_name, leaf = ref_name.split(".")
        pkg = _reference_package(pkg_name)
        setattr(pkg, leaf, mod)
    # 3. utils.transforms keeps the reference's affine helpers (dataset code uses them); only flip_back is swapped
    from .lib.utils.transforms import flip_back
    try:
        t = importlib.import_module("utils.transforms")
        t.flip_back = flip_back
        done["utils.transforms.flip_back"] = flip_back
    except ImportError as exc:       # cv2 missing: the reference's own module would not import either
        if verbose:
            print("fpd_b200.dropin: utils.transforms not importable (%s); flip_back not patched" % exc)
    if verbose:
        for k in done:
            print("fpd_b200.dropin: %s -> fpd_b200" % k)
    return done


def uninstall():
    """Drop the replacements (next import resolves to the reference again). Mostly for tests."""
    for ref_name in _REPLACED:
        mod = sys.modules.get(ref_name)
        if mod is not None and getattr(mod, "__name__", "").startswith("fpd_b200."):
            del sys.modules[ref_name]
            pkg = sys.modules.get(ref_name.split(".")[0])
            if pkg is not None and getattr(pkg, ref_name.split(".")[1], None) is mod:
                delattr(pkg, ref_name.split(".")[1])
