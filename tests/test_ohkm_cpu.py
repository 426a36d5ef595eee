"""JointsOHKMMSELoss on the host: the fp64 oracle against the reference's golden values and gradients, constructor and
attribute parity with the reference's class, and the drop-in import under fpd_b200.dropin.install()."""
import inspect
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ohkm.npz")
REF = "/root/reference"
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def z():
    d = np.load(GOLD, allow_pickle=False)
    return {k: d[k] for k in d.files}


def _f32(a):
    return torch.from_numpy(a.astype(np.float32))


def _module_tags(z):
    return sorted({k.split("/")[0] for k in z if k.startswith("m")})


def _grad_close(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(got != 0, ref != 0)
    assert np.abs(got - ref).max() <= 1e-6 * np.abs(ref).max()


def test_golden_covers_the_documented_cases(z):
    tags = _module_tags(z)
    seen = {(z[t + "/out"].shape[1], int(z[t + "/topk"])) for t in tags}
    assert {(16, 1), (16, 8), (16, 16), (17, 1), (17, 8), (17, 17)} <= seen
    assert {z[t + "/out"].shape[0] for t in tags} == {2, 3, 4, 5}
    assert any(not z[t + "/use_target_weight"] for t in tags)
    # whole samples with more than J - topk invisible joints
    assert any(((z[t + "/target_weight"][..., 0] == 0).sum(1) > z[t + "/out"].shape[1] - int(z[t + "/topk"])).any()
               for t in tags if z[t + "/use_target_weight"])
    combos = {(int(z[k[:-len("/pose_topk")] + "/pose_topk"]) > 0, int(z[k[:-len("/pose_topk")] + "/kd_topk"]) > 0)
              for k in z if k.endswith("/pose_topk")}
    assert combos == {(False, False), (True, False), (False, True), (True, True)}
    assert os.path.getsize(GOLD) < 300 * 1024


def test_oracle_matches_reference_module_golden(z):
    from oracle import ohkm_oracle as O
    for t in _module_tags(z):
        tw = _f32(z[t + "/target_weight"]) if z[t + "/use_target_weight"] else None
        v, g = O.criterion(_f32(z[t + "/out"]), _f32(z[t + "/target"]), tw, int(z[t + "/topk"]))
        ref = float(z[t + "/loss"])
        assert abs(v.item() - ref) <= 1e-6 * abs(ref), (t, v.item(), ref)
        _grad_close(g.numpy(), z[t + "/grad"])


def test_oracle_matches_reference_fpd_golden(z):
    from oracle import ohkm_oracle as O
    for t in sorted({k.split("/")[0] for k in z if k.startswith("f")}):
        tw = _f32(z[t + "/target_weight"]) if z[t + "/use_target_weight"] else None
        outs = [_f32(o) for o in z[t + "/outs"]]
        pose, kd, total, grads = O.fpd(outs, _f32(z[t + "/target"]), _f32(z[t + "/teacher"]), tw, float(z[t + "/alpha"]),
                                       int(z[t + "/pose_topk"]), int(z[t + "/kd_topk"]))
        for got, ref in zip((pose, kd, total), z[t + "/losses"]):
            assert abs(got.item() - float(ref)) <= 1e-6 * abs(float(ref)), (t, got.item(), ref)
        for g, ref in zip(grads, z[t + "/grads"]):
            _grad_close(g.numpy(), ref)


def test_oracle_selection_rule_and_bad_topk():
    from oracle import ohkm_oracle as O
    l = torch.tensor([[0.5, 0.7, 0.5, 0.1], [0.0, 0.0, 0.0, 0.3]], dtype=torch.float64)
    assert O.select(l, 2).tolist() == [[True, True, False, False], [True, False, False, True]]
    assert not O.boundary_ok([0.5, 0.7, 0.5, 0.1], 2) and O.boundary_ok([0.5, 0.7, 0.5, 0.1], 3)
    assert O.boundary_ok([0.0, 0.0, 0.0, 0.3], 2)           # the boundary lies among zeros
    o = torch.rand(2, 4, 3, 3, dtype=torch.float64)
    for k in (-1, 5):
        with pytest.raises(ValueError):
            O.criterion(o, o * 0, None, k)


def test_constructor_and_attributes_match_the_reference():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core.loss import JointsOHKMMSELoss
    from oracle import ref_modules as R
    if not R.available():
        pytest.skip("needs the reference's modules under oracle/_ref (built by build())")
    Ref = R.loss().JointsOHKMMSELoss
    ours_sig, ref_sig = inspect.signature(JointsOHKMMSELoss.__init__), inspect.signature(Ref.__init__)
    assert list(ours_sig.parameters) == list(ref_sig.parameters)
    assert [p.default for p in ours_sig.parameters.values()] == [p.default for p in ref_sig.parameters.values()]
    for args, kw in (((True,), {}), ((False,), {"topk": 4}), ((True, 17), {})):
        a, b = JointsOHKMMSELoss(*args, **kw), Ref(*args, **kw)
        assert (a.use_target_weight, a.topk) == (b.use_target_weight, b.topk)
        assert isinstance(a, torch.nn.Module)
    with pytest.raises(RuntimeError, match="CUDA"):
        JointsOHKMMSELoss(True)(torch.zeros(2, 4, 8, 8), torch.zeros(2, 4, 8, 8), torch.ones(2, 4, 1))


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
    from core.loss import JointsMSELoss, JointsOHKMMSELoss
    import fpd_b200.lib.core.loss as L
    assert JointsOHKMMSELoss is L.JointsOHKMMSELoss and JointsMSELoss is L.JointsMSELoss
    from core.function import train, fpd_train, validate
    print("OHKM-DROPIN-OK")
''')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "lib")), reason="needs the reference checkout")
def test_dropin_resolves_ohkm_loss_to_fpd_b200():
    r = subprocess.run([sys.executable, "-c", DROPIN % (REF, ROOT)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "OHKM-DROPIN-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
