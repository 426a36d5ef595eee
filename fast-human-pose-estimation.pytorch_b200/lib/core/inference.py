"""Drop-in for the reference's lib/core/inference.py (get_max_preds / get_final_preds) with the arg-max on the
device: only [B,J] indices and maxima cross PCIe instead of the full heat-maps (reference: D2H of
B*J*h*w floats per batch + numpy, inference.py:18-46)."""
import math

import numpy as np
import torch


def _device_argmax(hm):
    from fpd_b200 import ops
    idx, maxvals = ops.argmax_nchw(hm.contiguous().float())
    return idx, maxvals


def preds_from_argmax(idx, maxvals, width):
    """idx [B,J] flat arg-max, maxvals [B,J] -> (preds [B,J,2] float32, maxvals [B,J,1]) exactly as
    inference.py:36-46: x = idx % W, y = floor(idx / W), zeroed where max <= 0."""
    idx = np.asarray(idx).astype(np.float32)
    maxvals = np.asarray(maxvals, dtype=np.float32)[..., None]
    preds = np.stack([idx % width, np.floor(idx / width)], axis=-1).astype(np.float32)
    preds *= (maxvals > 0.0).astype(np.float32)
    return preds, maxvals


def get_max_preds(batch_heatmaps):
    """Accepts a CUDA tensor [B,J,h,w] (arg-max on the device) or, like the reference, a numpy array."""
    if isinstance(batch_heatmaps, np.ndarray):
        assert batch_heatmaps.ndim == 4, 'batch_images should be 4-ndim'
        batch_heatmaps = torch.from_numpy(np.ascontiguousarray(batch_heatmaps)).cuda()
    idx, maxvals = _device_argmax(batch_heatmaps)
    return preds_from_argmax(idx.cpu().numpy(), maxvals.cpu().numpy(), batch_heatmaps.shape[3])


def _inverse_affine(center, scale, output_size):
    """The 2x3 matrix the reference obtains from get_affine_transform(center, scale, 0, output_size, inv=1)
    (lib/utils/transforms.py:57-89): three corresponding points -- centre, centre shifted up by half the box width, and
    the perpendicular third point -- held in float32 exactly like the reference's `src` / `dst` arrays, then the 3-point
    affine solved in float64 (what cv2.getAffineTransform does). Only scale[0] enters (the reference derives both axes
    from the box width)."""
    c = np.asarray(center, np.float32)
    src_w = np.asarray(scale, np.float32)[0] * np.float32(200.0)
    dst_w, dst_h = output_size[0], output_size[1]
    src = np.zeros((3, 2), np.float32)
    dst = np.zeros((3, 2), np.float32)
    src[0] = c
    src[1] = c + np.array([0.0, float(src_w * np.float32(-0.5))])
    dst[0] = [dst_w * 0.5, dst_h * 0.5]
    dst[1] = np.array([dst_w * 0.5, dst_h * 0.5]) + np.array([0, dst_w * -0.5], np.float32)
    for p in (src, dst):
        d = p[0] - p[1]
        p[2] = p[1] + np.array([-d[1], d[0]], np.float32)
    a = np.concatenate([dst.astype(np.float64), np.ones((3, 1))], 1)
    return np.linalg.solve(a, src.astype(np.float64)).T          # maps heat-map (dst) coordinates to image (src)


def _udp_inverse_affines(center, scale, output_size):
    """UDP's heat-map -> image matrices (Huang et al., CVPR 2020), the inverse of augment.udp_crop_matrix at rot = 0
    composed with the heat-map stride: x = x_hm * s * 200 / (w - 1) + c - s * 200 / 2 per axis, in float64."""
    c = np.asarray(center, np.float64).reshape(-1, 2)
    box = np.asarray(scale, np.float64).reshape(-1, 2) * 200.0
    t = np.zeros((c.shape[0], 6))
    t[:, 0] = box[:, 0] / (output_size[0] - 1.0)
    t[:, 4] = box[:, 1] / (output_size[1] - 1.0)
    t[:, 2] = c[:, 0] - box[:, 0] * 0.5
    t[:, 5] = c[:, 1] - box[:, 1] * 0.5
    return t


def inverse_affines(center, scale, output_size, udp=False):
    """_inverse_affine for a whole batch: center, scale [B,2] -> float64 [B,6], row b the row-major 2x3 matrix of sample
    b, equal bit for bit to _inverse_affine(center[b], scale[b], output_size) (the same float32 point arithmetic, the
    same LAPACK solve per sample). This is the `inv` that ops.final_preds takes. udp=True gives UDP's matrices instead,
    for maps of crops made by augment.udp_crop_matrix (config.TEST.UDP)."""
    if udp:
        return _udp_inverse_affines(center, scale, output_size)
    c = np.asarray(center, np.float32).reshape(-1, 2)
    src_w = np.asarray(scale, np.float32).reshape(-1, 2)[:, 0] * np.float32(200.0)
    B = c.shape[0]
    dst_w, dst_h = output_size[0], output_size[1]
    src = np.zeros((B, 3, 2), np.float32)
    dst = np.zeros((3, 2), np.float32)
    src[:, 0] = c
    shift = np.zeros((B, 2))
    shift[:, 1] = (src_w * np.float32(-0.5)).astype(np.float64)
    src[:, 1] = c.astype(np.float64) + shift
    dst[0] = [dst_w * 0.5, dst_h * 0.5]
    dst[1] = np.array([dst_w * 0.5, dst_h * 0.5]) + np.array([0, dst_w * -0.5], np.float32)
    d = src[:, 0] - src[:, 1]
    src[:, 2] = src[:, 1] + np.stack([-d[:, 1], d[:, 0]], 1)
    d = dst[0] - dst[1]
    dst[2] = dst[1] + np.array([-d[1], d[0]], np.float32)
    a = np.concatenate([dst.astype(np.float64), np.ones((3, 1))], 1)
    t = np.linalg.solve(np.broadcast_to(a, (B, 3, 3)), src.astype(np.float64))     # [B,3,2]
    return np.ascontiguousarray(t.transpose(0, 2, 1).reshape(B, 6))


def _apply_affine(coords, t):
    """coords [J,2] mapped by the 2x3 matrix t, in float64."""
    coords = np.asarray(coords, dtype=np.float64)
    out = np.zeros(coords.shape)
    out[:, 0:2] = coords[:, 0:2] @ t[:, :2].T + t[:, 2]
    return out


def transform_preds(coords, center, scale, output_size):
    """lib/utils/transforms.py:49-54 for the whole [J,2] array at once (rot = 0 is the only call the hot path makes)."""
    return _apply_affine(coords, _inverse_affine(center, scale, output_size))


def use_dark(config):
    """config.TEST.DARK: DARK's decode (ops.final_preds_dark) replaces the quarter-pixel nudge where POST_PROCESS is on."""
    return bool(config.TEST.POST_PROCESS) and bool(getattr(config.TEST, "DARK", False))


def use_udp(config):
    """config.TEST.UDP: map heat-map coordinates to the image with UDP's matrices (inverse_affines(..., udp=True)), for
    models trained and validated on RawJointsDataset(udp=True) crops. Either decode runs on them unchanged."""
    return bool(getattr(config.TEST, "UDP", False))


def blur_kernel(config):
    """config.TEST.BLUR_KERNEL: the size of DARK's Gaussian blur (odd, 3..15)."""
    return int(getattr(config.TEST, "BLUR_KERNEL", 11))


def get_final_preds(config, batch_heatmaps, center, scale):
    """inference.py:49-79: arg-max, optional quarter-pixel nudge toward the higher neighbour (or, with
    config.TEST.DARK, DARK's Taylor step), map back to image coordinates (with config.TEST.UDP, by UDP's matrices).
    batch_heatmaps: CUDA tensor or numpy [B,J,h,w]."""
    if isinstance(batch_heatmaps, np.ndarray):
        batch_heatmaps = torch.from_numpy(np.ascontiguousarray(batch_heatmaps)).cuda()
    hm = batch_heatmaps.contiguous().float()
    B, J, H, W = hm.shape
    if use_dark(config):
        # the kernel validate()'s graph route runs, on the same map: both routes give the same bits
        from fpd_b200 import ops
        nhwc = ops.nchw_to_nhwc(hm)
        _, idx, maxvals = ops.flip_merge_argmax(nhwc, want_avg=False)
        inv = torch.from_numpy(inverse_affines(center, scale, [W, H], udp=use_udp(config))).to(hm.device)
        preds = ops.final_preds_dark(nhwc, idx, maxvals, inv, blur_kernel(config)).cpu().numpy()
        return preds[..., :2].copy(), preds[..., 2:].copy()
    idx, maxvals = _device_argmax(hm)
    coords, maxvals_np = preds_from_argmax(idx.cpu().numpy(), maxvals.cpu().numpy(), W)
    if config.TEST.POST_PROCESS:
        # gather the four neighbours of every arg-max on the device: 4*B*J floats cross PCIe, not B*J*H*W
        px = torch.floor(torch.from_numpy(coords[..., 0]).cuda() + 0.5).long()
        py = torch.floor(torch.from_numpy(coords[..., 1]).cuda() + 0.5).long()
        ok = (px > 1) & (px < W - 1) & (py > 1) & (py < H - 1)
        pxc, pyc = px.clamp(1, W - 2), py.clamp(1, H - 2)
        flat = hm.reshape(B, J, H * W)

        def at(yy, xx):
            return flat.gather(2, (yy * W + xx).unsqueeze(-1)).squeeze(-1)
        dx = torch.sign(at(pyc, pxc + 1) - at(pyc, pxc - 1)) * ok
        dy = torch.sign(at(pyc + 1, pxc) - at(pyc - 1, pxc)) * ok
        coords[..., 0] += dx.cpu().numpy() * .25
        coords[..., 1] += dy.cpu().numpy() * .25
    preds = coords.copy()
    if use_udp(config):
        inv = inverse_affines(center, scale, [W, H], udp=True).reshape(B, 2, 3)
        for i in range(B):
            preds[i] = _apply_affine(coords[i], inv[i])
        return preds, maxvals_np
    for i in range(B):
        preds[i] = transform_preds(coords[i], center[i], scale[i], [W, H])
    return preds, maxvals_np
