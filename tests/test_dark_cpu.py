"""DARK (distribution-aware coordinate representation, Zhang et al., CVPR 2020) without a GPU: an fp64 numpy model of the
decode (fpd_final_preds_dark) and of the unbiased targets (fpd_gaussian_targets_unbiased), checked against itself, and
the host-side argument checks of both entry points. tests/test_dark_gpu.py holds the kernels to this model."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# ----------------------------------------------------------------------------------------------- fp64 model
def blur_weights(k):
    """The normalised k-tap Gaussian, sigma = 0.3 ((k - 1) / 2 - 1) + 0.8."""
    sigma = 0.3 * ((k - 1) * 0.5 - 1) + 0.8
    d = np.arange(k, dtype=np.float64) - k // 2
    g = np.exp(-(d * d) / (2 * sigma * sigma))
    return g / g.sum()


def blur(m, k):
    """Separable Gaussian blur of one map, zeros outside it."""
    h, w = m.shape
    r = k // 2
    wk = blur_weights(k)
    p = np.pad(np.asarray(m, np.float64), r)
    hx = sum(wk[i] * p[:, i:i + w] for i in range(k))
    return sum(wk[i] * hx[i:i + h, :] for i in range(k))


def argmax_coords(m):
    """(x0, y0, maxval): the first maximum, both coordinates 0 unless maxval > 0 (get_max_preds)."""
    h, w = m.shape
    i = int(np.argmax(m))
    mv = m.reshape(-1)[i]
    if not mv > 0:
        return 0, 0, mv
    return i % w, i // w, mv


def dark_decode(m, k=11):
    """Heat-map coordinates (x, y) of one map [h, w] after DARK's Taylor step, in float64."""
    h, w = m.shape
    x0, y0, _ = argmax_coords(m)
    if not (2 <= x0 <= w - 3 and 2 <= y0 <= h - 3):
        return float(x0), float(y0)
    g = blur(m, k)
    gmax = g.max()
    if gmax > 0:
        g = g * (np.max(np.asarray(m, np.float64)) / gmax)
    L = np.log(np.maximum(g, 1e-10))
    dx = 0.5 * (L[y0, x0 + 1] - L[y0, x0 - 1])
    dy = 0.5 * (L[y0 + 1, x0] - L[y0 - 1, x0])
    dxx = 0.25 * (L[y0, x0 + 2] - 2 * L[y0, x0] + L[y0, x0 - 2])
    dyy = 0.25 * (L[y0 + 2, x0] - 2 * L[y0, x0] + L[y0 - 2, x0])
    dxy = 0.25 * (L[y0 + 1, x0 + 1] - L[y0 - 1, x0 + 1] - L[y0 + 1, x0 - 1] + L[y0 - 1, x0 - 1])
    det = dxx * dyy - dxy * dxy
    if det != 0:
        with np.errstate(all="ignore"):
            off = -np.linalg.inv(np.array([[dxx, dxy], [dxy, dyy]])) @ np.array([dx, dy])
        if np.all(np.isfinite(off)):
            return x0 + off[0], y0 + off[1]
    return float(x0), float(y0)


def quarter_decode(m):
    """The default decode: arg-max nudged a quarter pixel toward the higher neighbour (get_final_preds)."""
    h, w = m.shape
    x0, y0, _ = argmax_coords(m)
    x, y = float(x0), float(y0)
    if 1 < x0 < w - 1 and 1 < y0 < h - 1:
        x += 0.25 * np.sign(m[y0, x0 + 1] - m[y0, x0 - 1])
        y += 0.25 * np.sign(m[y0 + 1, x0] - m[y0 - 1, x0])
    return x, y


def unbiased_targets(joints, joints_vis, heatmap_size, image_size, sigma, joints_weight=None):
    """joints, joints_vis [N,J,3] -> (target [N,J,H,W], weight [N,J,1]) in float64: the Gaussian on the unrounded centre
    mu = joint * (W / image_w, H / image_h) over the whole map; weight 0 and an empty map when the 3 sigma window lies
    outside the map."""
    W, H = heatmap_size
    n, J = joints.shape[:2]
    target = np.zeros((n, J, H, W))
    weight = np.zeros((n, J, 1))
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    for i in range(n):
        for j in range(J):
            mx = np.float64(joints[i, j, 0]) * (W / image_size[0])
            my = np.float64(joints[i, j, 1]) * (H / image_size[1])
            v = np.float64(joints_vis[i, j, 0])
            r = 3.0 * sigma
            if mx - r >= W or my - r >= H or mx + r + 1 < 0 or my + r + 1 < 0:
                v = 0.0
            elif v > 0.5:
                target[i, j] = np.exp(-((xs - mx) ** 2 + (ys - my) ** 2) / (2.0 * sigma * sigma))
            weight[i, j, 0] = v * (1.0 if joints_weight is None else joints_weight[j])
    return target, weight


def rounded_target(mx, my, H, W, sigma):
    """The default target of one joint in heat-map units: the Gaussian on the rounded centre, within 3 sigma."""
    cx, cy = int(mx + 0.5), int(my + 0.5)
    ys, xs = np.mgrid[0:H, 0:W]
    t = np.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2.0 * sigma * sigma))
    return np.where((np.abs(xs - cx) <= 3 * sigma) & (np.abs(ys - cy) <= 3 * sigma), t, 0.0)


def subpixel_grid(H, W, margin, n=9):
    """Joints in heat-map units at least `margin` px from every border, over a grid that sweeps every sub-pixel phase."""
    xs = np.linspace(margin, W - 1 - margin, n) + np.linspace(0, 1, n, endpoint=False)
    ys = np.linspace(margin, H - 1 - margin, n) + np.linspace(0, 1, n, endpoint=False)[::-1]
    return [(x, y) for x in xs for y in ys if margin <= x <= W - 1 - margin and margin <= y <= H - 1 - margin]


# ----------------------------------------------------------------------------------------------- the model against itself
def border_margin(sigma):
    """How far from every border the round trip holds to 0.02 px. The blur extends the map by zeros, which biases the
    estimate near a border: at 3 px from it, sigma = 2, by up to 0.05 px."""
    return sigma + 2.0


@pytest.mark.parametrize("H,W", [(64, 48), (64, 64), (96, 72)])
@pytest.mark.parametrize("sigma", [2, 3])
def test_model_round_trip_recovers_subpixel_joints(H, W, sigma):
    errs, base = [], []
    for mx, my in subpixel_grid(H, W, border_margin(sigma)):
        t, _ = unbiased_targets(np.array([[[mx, my, 0]]]), np.ones((1, 1, 3)), (W, H), (W, H), sigma)
        x, y = dark_decode(t[0, 0])
        errs.append(max(abs(x - mx), abs(y - my)))
        qx, qy = quarter_decode(rounded_target(mx, my, H, W, sigma))
        base.append(max(abs(qx - mx), abs(qy - my)))
    assert max(errs) < 0.02, max(errs)
    # the default encoding and decoding on the same grid: off by up to half a heat-map pixel
    assert max(base) > 0.4, max(base)


def test_model_round_trip_in_image_units():
    """Stride 4 (256x192 input, 64x48 maps): joints given in image pixels come back to within 0.02 heat-map px."""
    rng = np.random.RandomState(0)
    J = 17
    joints = np.zeros((1, J, 3))
    m = 4 * border_margin(2)
    joints[0, :, 0] = rng.uniform(m, 188 - m, J)        # the last heat-map column, 47, is image x = 188
    joints[0, :, 1] = rng.uniform(m, 252 - m, J)
    t, w = unbiased_targets(joints, np.ones((1, J, 3)), (48, 64), (192, 256), 2)
    assert np.all(w == 1)
    for j in range(J):
        x, y = dark_decode(t[0, j])
        assert abs(x - joints[0, j, 0] / 4) < 0.02 and abs(y - joints[0, j, 1] / 4) < 0.02


def test_model_leaves_degenerate_maps_at_the_argmax():
    m = np.zeros((16, 16))
    assert dark_decode(m) == (0.0, 0.0)                   # all zero: maxval 0 zeroes the arg-max
    m[:] = 0.5
    assert dark_decode(m) == (0.0, 0.0)                   # constant: first maximum at (0, 0)
    m = -np.ones((16, 16))
    m[8, 7] = 1.0                                         # the blur is negative everywhere: every log clamps, det = 0
    assert blur(m, 11).max() < 0
    assert dark_decode(m) == (7.0, 8.0)
    m = np.zeros((16, 16))
    m[1, 8] = m[9, 9] = 1.0                               # tie: the first maximum, 1 px from the top, stays put
    assert dark_decode(m) == (8.0, 1.0)


def test_model_targets_visibility():
    joints = np.array([[[-7.5, 20.0, 0], [-6.4, 20.0, 0], [10.0, 10.0, 0], [53.9, 8.0, 0], [54.0, 8.0, 0]]])
    vis = np.ones((1, 5, 3))
    vis[0, 2] = 0
    t, w = unbiased_targets(joints, vis, (48, 64), (48, 64), 2)
    # mu + 3 sigma + 1 < 0 at x = -7.5 but not at -6.4; mu - 3 sigma >= W at 54.0 but not at 53.9
    assert w[0, :, 0].tolist() == [0, 1, 0, 1, 0]
    assert not t[0, 0].any() and t[0, 1].any() and not t[0, 2].any() and t[0, 3].any() and not t[0, 4].any()


# ----------------------------------------------------------------------------------------------- entry points
def test_ctypes_entries_exist():
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    lib = N.lib()
    for name in ("fpd_final_preds_dark", "fpd_gaussian_targets_unbiased"):
        assert name in N._SIGNATURES and getattr(lib, name).argtypes == N._SIGNATURES[name][1]


@pytest.mark.parametrize("k", [-1, 0, 1, 2, 4, 10, 16, 17, 99])
def test_final_preds_dark_rejects_bad_blur_kernel(k):
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    p = ctypes.c_void_p(16)         # never dereferenced: the check fails first
    rc = N.lib().fpd_final_preds_dark(p, p, p, p, k, p, 2, 17, 64, 48, None)
    assert rc == -1
    assert N.last_error() == "final_preds_dark: blur_kernel=%d must be odd and in [3, 15]" % k


@pytest.mark.parametrize("args, message", [
    ((None, 1, 1, 1, 11, 1, 2, 17, 64, 48), "final_preds_dark: null pointer"),
    ((1, 1, 1, 1, 11, None, 2, 17, 64, 48), "final_preds_dark: null pointer"),
    ((1, 1, 1, 1, 11, 1, 2, 65, 64, 48), "final_preds_dark: B=2 J=65 out of range"),
    ((1, 1, 1, 1, 11, 1, 2, 17, 4, 48), "final_preds_dark: needs a heat-map of at least 5x5, got 4x48"),
    ((1, 1, 1, 1, 11, 1, 2, 17, 256, 256), "final_preds_dark: a 256x256 heat-map does not fit in shared memory"),
])
def test_final_preds_dark_host_checks(args, message):
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    args = [ctypes.c_void_p(16) if a == 1 and i in (0, 1, 2, 3, 5) else a for i, a in enumerate(args)]
    assert N.lib().fpd_final_preds_dark(*args, None) == -1
    assert N.last_error() == message


@pytest.mark.parametrize("null_at, sizes, message", [
    (0, (1, 17, 64, 48, 192, 256, 2), "gaussian_targets_unbiased: null pointer"),
    (3, (1, 17, 64, 48, 192, 256, 2), "gaussian_targets_unbiased: null pointer"),
    (None, (1, 17, 64, 48, 192, 256, 0), "gaussian_targets_unbiased: bad sizes"),
    (None, (1, 17, 64, 48, 0, 256, 2), "gaussian_targets_unbiased: bad sizes"),
])
def test_gaussian_targets_unbiased_host_checks(null_at, sizes, message):
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    ptrs = [ctypes.c_void_p(16)] * 5
    ptrs[2] = None                  # joints_weight is optional
    if null_at is not None:
        ptrs[null_at] = None
    assert N.lib().fpd_gaussian_targets_unbiased(*ptrs, *sizes, None) == -1
    assert N.last_error() == message


def test_ops_and_inference_options():
    """The opt-in switches default off: config without DARK keeps the quarter-pixel decode."""
    import types
    import fpd_b200  # noqa: F401
    from fpd_b200.infer_step import _post_process
    from fpd_b200.lib.core.inference import blur_kernel, use_dark
    NS = types.SimpleNamespace
    assert not use_dark(NS(TEST=NS(POST_PROCESS=True)))
    assert not use_dark(NS(TEST=NS(POST_PROCESS=False, DARK=True)))
    assert use_dark(NS(TEST=NS(POST_PROCESS=True, DARK=True)))
    assert blur_kernel(NS(TEST=NS())) == 11 and blur_kernel(NS(TEST=NS(BLUR_KERNEL=7))) == 7
    assert _post_process(True) is True and _post_process(0) is False and _post_process("dark") == "dark"
    with pytest.raises(ValueError):
        _post_process("darkk")
