"""Drop-in for the reference's lib/nms/nms.py, backed by libfpd_b200's sm_90a kernels (csrc/nms.cu):

  gpu_nms / gpu_nms_wrapper   gpu_nms.pyx:19-34, nms.py:27-32  -> fpd_nms_host (C ABI, reference `_nms` signature)
  nms / py_nms_wrapper / cpu_nms_wrapper   nms.py:17-24,35-72  -> the same device path (identical keep lists)
  oks_nms                     nms.py:99-124 (called from lib/dataset/coco.py:365) -> fpd_oks_nms_device
  rescore_persons             the loop of coco.py:346-357       -> fpd_oks_rescore
  oks_iou, soft_oks_nms       nms.py:75-96,138-178: host numpy (soft-NMS re-sorts after every pick -- serial by nature
                              and off by default, cfg.TEST.SOFT_NMS = False)
"""
import ctypes

import numpy as np


def gpu_nms(dets, thresh, device_id=0):
    """dets: float32 [N,5] (x1,y1,x2,y2,score). Returns the kept indices into `dets`, highest score first --
    same contract as the Cython wrapper: sort by score, run `_nms` on the sorted boxes, map back through `order`."""
    from fpd_b200 import _native as N
    dets = np.ascontiguousarray(dets, dtype=np.float32)
    n, d = dets.shape
    if n == 0:
        return []
    order = dets[:, 4].argsort()[::-1].astype(np.int32)
    sorted_dets = np.ascontiguousarray(dets[order, :])
    keep = np.zeros(n, dtype=np.int32)
    num = ctypes.c_int(0)
    N.check(N.lib().fpd_nms_host(keep.ctypes.data_as(ctypes.c_void_p), ctypes.cast(ctypes.byref(num), ctypes.c_void_p),
                                 sorted_dets.ctypes.data_as(ctypes.c_void_p), n, d, float(thresh), int(device_id)),
            "nms_host")
    return list(order[keep[:num.value]])


def nms(dets, thresh):
    return gpu_nms(dets, thresh)


def gpu_nms_wrapper(thresh, device_id):
    def _nms(dets):
        return gpu_nms(dets, thresh, device_id)
    return _nms


def py_nms_wrapper(thresh):
    def _nms(dets):
        return nms(dets, thresh)
    return _nms


cpu_nms_wrapper = py_nms_wrapper


def _db_arrays(kpts_db):
    scores = np.array([kpts_db[i]['score'] for i in range(len(kpts_db))])
    kpts = np.array([np.asarray(kpts_db[i]['keypoints']).flatten() for i in range(len(kpts_db))])
    areas = np.array([kpts_db[i]['area'] for i in range(len(kpts_db))])
    return scores, kpts, areas


def oks_nms(kpts_db, thresh, sigmas=None, in_vis_thre=None):
    """Same arguments and result as the reference (list of dicts with 'score', 'keypoints' [J,3], 'area'; returns the
    kept indices into kpts_db, best first): the pairwise OKS mask and the greedy sweep run on the device."""
    import torch
    from fpd_b200 import ops
    if len(kpts_db) == 0:
        return []
    scores, kpts, areas = _db_arrays(kpts_db)
    order = scores.argsort()[::-1]
    n = len(order)
    k = np.ascontiguousarray(kpts[order]).reshape(n, -1, 3)
    if k.dtype not in (np.float32, np.float64):
        k = k.astype(np.float64)
    keep, num = ops.oks_nms_device(torch.from_numpy(k).cuda(), torch.from_numpy(np.ascontiguousarray(areas[order],
                                                                                                   dtype=np.float64)).cuda(),
                                   thresh, sigmas, in_vis_thre)
    m = int(num.item())
    return [order[i] for i in keep[:m].cpu().numpy()]


def rescore_persons(keypoints, box_scores, in_vis_thre):
    """keypoints [n,J,3] (numpy), box_scores [n] -> float64 [n] = box score x mean joint confidence above in_vis_thre."""
    import torch
    from fpd_b200 import ops
    k = np.ascontiguousarray(keypoints)
    if k.dtype not in (np.float32, np.float64):
        k = k.astype(np.float64)
    out = ops.oks_rescore(torch.from_numpy(k).cuda(), torch.from_numpy(np.ascontiguousarray(box_scores, dtype=np.float64)).cuda(),
                          in_vis_thre)
    return out.cpu().numpy()


def oks_iou(g, d, a_g, a_d, sigmas=None, in_vis_thre=None):
    """Host helper with the reference's semantics (one kept person g against candidates d)."""
    from fpd_b200.ops import COCO_SIGMAS
    sig = np.asarray(COCO_SIGMAS) if not isinstance(sigmas, np.ndarray) else sigmas
    var = (sig * 2) ** 2
    ious = np.zeros(d.shape[0])
    for i in range(d.shape[0]):
        e = ((d[i, 0::3] - g[0::3]) ** 2 + (d[i, 1::3] - g[1::3]) ** 2) / var / ((a_g + a_d[i]) / 2 + np.spacing(1)) / 2
        if in_vis_thre is not None:
            e = e[d[i, 2::3] > in_vis_thre]     # the reference's mask reduces to the candidate's visibility (nms.py:91)
        ious[i] = np.sum(np.exp(-e)) / e.shape[0] if e.shape[0] != 0 else 0.0
    return ious


def soft_oks_nms(kpts_db, thresh, sigmas=None, in_vis_thre=None):
    """Gaussian soft-NMS over OKS, at most 20 picks (nms.py:138-178)."""
    if len(kpts_db) == 0:
        return []
    scores, kpts, areas = _db_arrays(kpts_db)
    order = scores.argsort()[::-1]
    scores = scores[order]
    picked = []
    while order.size > 0 and len(picked) < 20:
        i = order[0]
        ovr = oks_iou(kpts[i], kpts[order[1:]], areas[i], areas[order[1:]], sigmas, in_vis_thre)
        order = order[1:]
        scores = scores[1:] * np.exp(-ovr ** 2 / thresh)
        resort = scores.argsort()[::-1]
        order, scores = order[resort], scores[resort]
        picked.append(i)
    return np.array(picked, dtype=np.intp)
