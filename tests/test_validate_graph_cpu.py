"""Host side of validate()'s graph route: the batched heat-map -> image matrices and the PCK bookkeeping from per-joint
counts must equal the per-sample / per-coordinate host functions exactly."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fpd_b200  # noqa: E402,F401
from fpd_b200.lib.core.evaluate import pck_from_counts, pck_from_preds  # noqa: E402
from fpd_b200.lib.core.inference import _inverse_affine, inverse_affines  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "decode2.npz")


def _per_sample(center, scale, size):
    return np.stack([_inverse_affine(center[b], scale[b], size).reshape(6) for b in range(len(center))])


@pytest.mark.parametrize("tag,size", [("sq", [64, 64]), ("rect", [48, 64])])
def test_inverse_affines_equal_per_sample_on_golden(tag, size):
    z = np.load(GOLD, allow_pickle=False)
    c, s = z[tag + "/center"], z[tag + "/scale"]
    got = inverse_affines(c, s, size)
    assert got.dtype == np.float64 and got.shape == (len(c), 6) and got.flags.c_contiguous
    assert np.array_equal(got, _per_sample(c, s, size))


@pytest.mark.parametrize("size", [[64, 64], [48, 64], [72, 96], [24, 32]])
def test_inverse_affines_equal_per_sample_on_random_boxes(size):
    rng = np.random.RandomState(sum(size))
    B = 257
    c = rng.uniform(-50, 1500, (B, 2)).astype(np.float32)
    s = rng.uniform(0.05, 8.0, (B, 2)).astype(np.float32)
    s[::7] = np.round(s[::7], 2)         # the loaders' typical two-decimal scales
    for cc, ss in ((c, s), (c.astype(np.float64), s.astype(np.float64)), (c[:1], s[:1])):
        assert np.array_equal(inverse_affines(cc, ss, size), _per_sample(cc, ss, size))


def _counts(pred, target, h, w):
    """What the device kernel counts: valid = target x > 1 and y > 1; hit = valid and d < 0.5."""
    norm = np.array([h, w], dtype=np.float64) / 10.0
    valid = (target[..., 0] > 1) & (target[..., 1] > 1)
    d = np.linalg.norm((pred.astype(np.float32) - target.astype(np.float32)) / norm, axis=-1)
    return np.stack([valid.sum(0), (valid & (d < 0.5)).sum(0)], 1).astype(np.int32)


@pytest.mark.parametrize("seed", range(6))
def test_pck_from_counts_equals_pck_from_preds(seed):
    rng = np.random.RandomState(seed)
    B, J = rng.randint(1, 40), rng.randint(1, 20)
    h, w = [(64, 64), (64, 48), (96, 72)][seed % 3]
    target = np.stack([rng.randint(0, w, (B, J)), rng.randint(0, h, (B, J))], -1).astype(np.float32)
    pred = np.clip(target + rng.randint(-8, 9, (B, J, 2)), 0, None).astype(np.float32)
    if seed == 0:
        target[:, 0] = 0              # a joint that is never valid
    if seed == 1:
        target[...] = 1               # no valid joint at all: avg is the int 0, acc keeps its zero in front
    ref = pck_from_preds(pred, target, h, w)
    got = pck_from_counts(_counts(pred, target, h, w))
    assert np.array_equal(got[0], ref[0])
    assert got[1] == ref[1] and type(got[1]) is type(ref[1])
    assert got[2] == ref[2]
