"""Generate tests/golden/ohkm.npz by running the REAL reference's JointsOHKMMSELoss / JointsMSELoss
(/root/reference/lib/core/loss.py, read-only) on the CPU:

    python tests/golden/make_golden_ohkm.py

Two kinds of case:
  * m<i>/...: the module on its own -- value and backward() gradient of JointsOHKMMSELoss(use_target_weight, topk)
    for J = 16 / 17, topk = 1 / 8 / J, no weights, random weights with zeros, and samples with more than J - topk
    invisible joints, B = 2..5, 8x8 and 16x12 maps;
  * f<pose_topk>_<kd_topk>/...: the reference's fpd_train loop body (lib/core/function.py:127-134) for each pose / kd
    criterion combination (0 = JointsMSELoss), 2-4 stacks, 8x8 maps (h*w a multiple of 64).

Inputs are multiples of 1/256 in [-0.25, 1) (stored as float16 to keep the file small; the reference ran on the same
values in float32). Any sample whose topk-th and (topk+1)-th non-zero per-joint losses are within 1e-4 relative of each
other is drawn again (oracle.ohkm_oracle.boundary_ok), so that the fp32 reference and other evaluation orders select
the same joints.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(OUT, "..", ".."))
from oracle.ohkm_oracle import boundary_ok, per_joint  # noqa: E402

# tag: (J, topk, weights, B, h, w); weights: "none" = use_target_weight False, "w" = random weights (zeros, 1, and the
# MPII-style 1.2 / 1.5), "sparse" = like "w" with whole samples that have more than J - topk invisible joints
MODULE_CASES = {
    "m0": (16, 1, "none", 2, 8, 8),
    "m1": (16, 8, "w", 3, 8, 8),
    "m2": (16, 16, "sparse", 4, 8, 8),
    "m3": (16, 8, "sparse", 5, 8, 8),
    "m4": (16, 1, "w", 3, 8, 8),
    "m5": (17, 1, "sparse", 5, 8, 8),
    "m6": (17, 8, "none", 2, 16, 12),
    "m7": (17, 17, "w", 3, 8, 8),
    "m8": (17, 8, "w", 4, 8, 8),
    "m9": (17, 8, "sparse", 2, 8, 8),
}
# (pose_topk, kd_topk): (S, B, J, h, w, use_target_weight, alpha)
FPD_CASES = {
    (0, 0): (2, 2, 16, 8, 8, True, 0.5),
    (8, 0): (3, 2, 16, 8, 8, True, 0.3),
    (0, 8): (2, 3, 17, 8, 8, True, 0.7),
    (8, 4): (4, 2, 16, 8, 8, False, 0.5),
}


def load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def f16(rng, *shape):
    return (rng.randint(-64, 256, shape) / 256.0).astype(np.float16)


def weights(rng, J, kind, topk, sparse_sample):
    if kind == "none":
        return np.ones((J, 1), np.float32)
    w = rng.choice(np.array([0.0, 1.0, 1.0, 1.0, 1.2, 1.5], np.float32), size=(J, 1))
    if sparse_sample:                       # more than J - topk joints invisible
        n0 = min(J, J - topk + 1 + rng.randint(0, 3))
        w[rng.permutation(J)[:n0]] = 0.0
    return w


def sample_ok(outs, refs_topk, tw):
    """outs: list of [J,h,w] float32 stacks of one sample; refs_topk: [(ref [J,h,w], topk)]."""
    for o in outs:
        for ref, k in refs_topk:
            if k:
                l, _, _, _ = per_joint(torch.from_numpy(o)[None], torch.from_numpy(ref)[None], torch.from_numpy(tw)[None])
                if not boundary_ok(l[0], k):
                    return False
    return True


def main():
    torch.set_num_threads(4)
    L = load("ref_loss_ohkm", "lib/core/loss.py")
    rng = np.random.RandomState(2024)
    save = {}
    redraws = 0
    for tag, (J, topk, wkind, B, h, w) in MODULE_CASES.items():
        outs, tgts, tws = [], [], []
        for b in range(B):
            while True:
                o, g = f16(rng, J, h, w), f16(rng, J, h, w)
                tw = weights(rng, J, wkind, topk, wkind == "sparse" and b % 2 == 0)
                if sample_ok([o.astype(np.float32)], [(g.astype(np.float32), topk)], tw):
                    break
                redraws += 1
            outs.append(o)
            tgts.append(g)
            tws.append(tw)
        o16, g16, tw = np.stack(outs), np.stack(tgts), np.stack(tws)
        out = torch.from_numpy(o16.astype(np.float32)).requires_grad_(True)
        crit = L.JointsOHKMMSELoss(use_target_weight=wkind != "none", topk=topk)
        loss = crit(out, torch.from_numpy(g16.astype(np.float32)), torch.from_numpy(tw))
        loss.backward()
        save[tag + "/out"], save[tag + "/target"], save[tag + "/target_weight"] = o16, g16, tw
        save[tag + "/topk"] = np.int64(topk)
        save[tag + "/use_target_weight"] = np.bool_(wkind != "none")
        save[tag + "/loss"] = np.float32(loss.item())
        save[tag + "/grad"] = out.grad.numpy()
    for (pk, kk), (S, B, J, h, w, use_tw, alpha) in FPD_CASES.items():
        tag = "f%d_%d" % (pk, kk)
        cols = {"outs": [], "target": [], "teacher": [], "tw": []}
        for b in range(B):
            while True:
                os_ = [f16(rng, J, h, w) for _ in range(S)]
                g, t = f16(rng, J, h, w), f16(rng, J, h, w)
                tw = weights(rng, J, "w" if use_tw else "none", max(pk, kk, 1), False)
                if sample_ok([x.astype(np.float32) for x in os_],
                             [(g.astype(np.float32), pk), (t.astype(np.float32), kk)], tw):
                    break
                redraws += 1
            cols["outs"].append(np.stack(os_))
            cols["target"].append(g)
            cols["teacher"].append(t)
            cols["tw"].append(tw)
        outs16 = np.stack(cols["outs"], 1)                    # [S,B,J,h,w]
        target = torch.from_numpy(np.stack(cols["target"]).astype(np.float32))
        toutput = torch.from_numpy(np.stack(cols["teacher"]).astype(np.float32))
        target_weight = torch.from_numpy(np.stack(cols["tw"]))
        outputs = [torch.from_numpy(x.astype(np.float32)).requires_grad_(True) for x in outs16]

        def crit(k):
            return L.JointsOHKMMSELoss(use_tw, topk=k) if k else L.JointsMSELoss(use_tw)
        pose_criterion, kd_pose_criterion = crit(pk), crit(kk)
        kd_weight_alpha = alpha
        # lib/core/function.py:127-134
        pose_loss = pose_criterion(outputs[0], target, target_weight)
        kd_pose_loss = kd_pose_criterion(outputs[0], toutput, target_weight)
        for output in outputs[1:]:
            pose_loss += pose_criterion(output, target, target_weight)
            kd_pose_loss += kd_pose_criterion(output, toutput, target_weight)
        loss = (1 - kd_weight_alpha) * pose_loss + kd_weight_alpha * kd_pose_loss
        loss.backward()
        save[tag + "/outs"] = outs16
        save[tag + "/target"] = np.stack(cols["target"])
        save[tag + "/teacher"] = np.stack(cols["teacher"])
        save[tag + "/target_weight"] = target_weight.numpy()
        save[tag + "/use_target_weight"] = np.bool_(use_tw)
        save[tag + "/alpha"] = np.float32(alpha)
        save[tag + "/pose_topk"], save[tag + "/kd_topk"] = np.int64(pk), np.int64(kk)
        save[tag + "/losses"] = np.array([pose_loss.item(), kd_pose_loss.item(), loss.item()], np.float32)
        save[tag + "/grads"] = np.stack([o.grad.numpy() for o in outputs])
    path = os.path.join(OUT, "ohkm.npz")
    np.savez_compressed(path, **save)
    print("ohkm.npz", os.path.getsize(path), "bytes;", redraws, "samples redrawn")


if __name__ == "__main__":
    main()
