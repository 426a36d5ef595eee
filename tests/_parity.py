"""Shared helpers of the GPU parity tests: the oracle run in fp32 and fp64 on the same device, and the fp64-referenced
gradient criterion.

Why fp64-referenced: the train-mode hourglass / HRNet at default init amplify round-off ~1000x (DESIGN.md section 2), so
the reference's OWN fp32 gradients sit 1e-3 .. 5e-2 away from the exact ones, tensor by tensor. A fixed tolerance is
therefore either meaningless (5e-2) or unattainable (1e-3). Instead every parameter gradient is compared with an fp64
evaluation of the reference algorithm and must be (almost) as close to it as the reference's fp32 arithmetic gets:

    err(ours, fp64)  <=  K * err(fp32 oracle, fp64) + floor          per tensor, max-abs error / max|g64|
    and the same for the whole-gradient relative L2 error.
"""
import json
import os

import torch


def cast_sd(sd, dtype, device=None):
    out = {}
    for k, v in sd.items():
        if torch.is_tensor(v):
            v = v.detach().clone()
            if v.is_floating_point():
                v = v.to(dtype)
            if device is not None:
                v = v.to(device)
        out[k] = v
    return out


def with_grad(sd):
    params = {k: v.requires_grad_(True) for k, v in sd.items()
              if torch.is_tensor(v) and v.is_floating_point() and "running" not in k and not k.startswith("__")}
    sd.update(params)
    return params


def rel_max(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def _pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(q * len(v)))]


def grad_report(ours, g32, g64, tag=None):
    """ours / g32 / g64: dict name -> gradient tensor. Per tensor: a = max|g - g64| for ours and for the fp32 oracle,
    normalised by max(max|g64_t|, 1e-6 * global max|g64|) -- the second term is an absolute floor for gradients that are
    EXACTLY zero in exact arithmetic (a conv bias in front of a train-mode BatchNorm: the fp64 value is ~1e-20, both fp32
    evaluations leave ~1e-10 of cancellation noise, far below Adam's eps = 1e-8). With a tag and FPD_PARITY_REPORT set,
    the report is appended to that file (one JSON line per call)."""
    gmax = max(float(v.abs().max()) for v in g64.values())
    rows = []
    n_o = n_3 = den = 0.0
    for k, ref in g64.items():
        ref = ref.double().cpu()
        o = ours[k].reshape(ref.shape).double().cpu()
        f = g32[k].reshape(ref.shape).double().cpu()
        m = max(ref.abs().max().item(), 1e-6 * gmax)
        rows.append((k, (o - ref).abs().max().item() / m, (f - ref).abs().max().item() / m))
        n_o += float((o - ref).pow(2).sum())
        n_3 += float((f - ref).pow(2).sum())
        den += float(ref.pow(2).sum())
    ratios = [r[1] / max(r[2], 1e-9) for r in rows]
    rep = {"tag": tag, "tensors": len(rows), "l2_ours": (n_o / den) ** 0.5, "l2_fp32": (n_3 / den) ** 0.5,
           "worst_ours": max(r[1] for r in rows), "worst_fp32": max(r[2] for r in rows),
           "q90_ours": _pct([r[1] for r in rows], 0.9), "q90_fp32": _pct([r[2] for r in rows], 0.9),
           "median_ratio": _pct(ratios, 0.5), "q90_ratio": _pct(ratios, 0.9), "worst_ratio": max(ratios), "rows": rows}
    out = os.environ.get("FPD_PARITY_REPORT")
    if tag is not None and out:
        try:
            with open(out, "a") as fh:
                fh.write(json.dumps(rep) + "\n")
        except OSError:
            pass
    return rep


# What "ill-conditioned" means here (from per-tensor parity reports of the bench configurations): wherever no ReLU decision differs,
# BOTH our gradients and the fp32 oracle's sit ~2e-5 from fp64 (ours slightly closer). But a network evaluation holds
# ~1e6-1e8 pre-activations, and the handful that lie within round-off of zero get their ReLU mask decided differently by
# any two finite-precision evaluations; ONE such flip at a low-resolution level (few pixels, each carrying a large share
# of the gradient) shifts every gradient upstream of it by ~1e-2 of its maximum. Each evaluation has its own O(1) flips in
# its own places: in the HRNet golden configuration the fp32 oracle's flip sits in layer1.2 (everything upstream of it is
# 1e-2 off, everything downstream 2e-5), ours in stage3.1.branches.1 -- so single tensors scatter by 1000x either way,
# while the median per-tensor ratio is 0.95-1.12 and the whole-gradient L2 ratio 0.70-1.19. The criterion is therefore
# statistical, with a per-tensor cap:
#   (i)   whole-gradient relative L2 error           <= K_L2   x the fp32 oracle's (measured 0.70-1.15x; the bound leaves
#         room for a flip that happens to sit earlier in OUR evaluation than in the oracle's)
#   (ii)  median of the per-tensor ratio err_ours / err_fp32   <= K_MED, where flips are everywhere (the oracle's own
#         median error >= 1e-3: the hourglass configurations) -- with one or two flips per evaluation (HRNet golden) the
#         ratio of a tensor only says on which side of whose flip it sits
#   (iii) every tensor: err_ours <= max(K_TENSOR x its own fp32 error, K_CAP x the fp32 oracle's WORST tensor error)
# A systematically wrong gradient (a mis-scaled tap, a dropped term) moves (i)/(ii) by orders of magnitude and trips
# (iii) on the affected tensors; exact per-tensor arithmetic is pinned separately where the network is well conditioned
# (eval-mode backward, tests/test_hourglass_gpu.py::test_eval_mode_backward_matches_oracle, <= 2e-3 per tensor, and the
# per-op tests in tests/test_ops_gpu.py).
K_L2, K_MED, K_TENSOR, K_CAP = 3.0, 1.5, 4.0, 1.5


def assert_grads_as_good_as_fp32(ours, g32, g64, tag):
    rep = grad_report(ours, g32, g64, tag)
    assert rep["l2_ours"] <= K_L2 * rep["l2_fp32"] + 1e-6, (tag, rep["l2_ours"], rep["l2_fp32"])
    if _pct([r[2] for r in rep["rows"]], 0.5) >= 1e-3:
        assert rep["median_ratio"] <= K_MED, (tag, rep["median_ratio"])
    cap = K_CAP * rep["worst_fp32"]
    bad = [(k, eo, e3) for k, eo, e3 in rep["rows"] if eo > max(K_TENSOR * e3, cap) + 1e-6]
    assert not bad, "%s: %d tensors beyond max(%.0fx own fp32 error, %.1fx the fp32 oracle's worst tensor = %.2e): %s" % (
        tag, len(bad), K_TENSOR, K_CAP, cap, bad[:5])
    return rep
