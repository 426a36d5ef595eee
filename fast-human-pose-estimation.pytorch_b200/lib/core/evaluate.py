"""Drop-in for the reference's lib/core/evaluate.py::accuracy (PCK@0.5 against the arg-max of the ground-truth
heat-maps, evaluate.py:41-71) fed by device-side arg-maxes."""
import numpy as np

from .inference import get_max_preds


def pck_from_preds(pred, target, h, w, thr=0.5):
    """pred/target: [B,J,2] coordinates. Mirrors calc_dists / dist_acc (evaluate.py:16-38): joints whose target
    is not > 1 in both coordinates are ignored; distances are normalised by (h, w) / 10."""
    norm = np.array([h, w], dtype=np.float64) / 10.0
    valid = (target[..., 0] > 1) & (target[..., 1] > 1)                      # [B,J]
    d = np.linalg.norm((pred.astype(np.float32) - target.astype(np.float32)) / norm, axis=-1)
    J = pred.shape[1]
    acc = np.zeros(J + 1)
    total, cnt = 0.0, 0
    for j in range(J):
        n = int(valid[:, j].sum())
        if n > 0:
            acc[j + 1] = float((d[valid[:, j], j] < thr).sum()) / n
            total += acc[j + 1]
            cnt += 1
        else:
            acc[j + 1] = -1
    avg = total / cnt if cnt else 0
    if cnt:
        acc[0] = avg
    return acc, avg, cnt


def pck_from_counts(counts):
    """counts int [J,2] = {valid, hit} per joint (ops.pck_counts, threshold 0.5) -> (acc[J+1], avg, cnt), the same
    float64 operations in the same order as pck_from_preds, hence the same values."""
    counts = np.asarray(counts)
    J = counts.shape[0]
    acc = np.zeros(J + 1)
    total, cnt = 0.0, 0
    for j in range(J):
        n = int(counts[j, 0])
        if n > 0:
            acc[j + 1] = float(int(counts[j, 1])) / n
            total += acc[j + 1]
            cnt += 1
        else:
            acc[j + 1] = -1
    avg = total / cnt if cnt else 0
    if cnt:
        acc[0] = avg
    return acc, avg, cnt


def accuracy(output, target, hm_type='gaussian', thr=0.5):
    """output/target: CUDA tensors or numpy [B,J,h,w]. Returns (acc[J+1], avg_acc, cnt, pred) like the reference."""
    assert hm_type == 'gaussian'
    h, w = output.shape[2], output.shape[3]
    pred, _ = get_max_preds(output)
    tgt, _ = get_max_preds(target)
    acc, avg, cnt = pck_from_preds(pred, tgt, h, w, thr)
    return acc, avg, cnt, pred
