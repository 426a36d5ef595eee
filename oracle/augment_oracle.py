"""CPU restatement of the input crop (the specification of csrc/augment.cu) and a stand-in for the reference's
JointsDataset, so that the tests of fpd_b200.augment run without the reference.

warp_region: cv2 4.x warpAffine(INTER_LINEAR, BORDER_CONSTANT=0) on an 8-bit 3-channel image, restated in fixed point
(imgwarp.cpp: coordinates in 1/1024 pixel rounded half to even, 1/32-pixel bilinear weights with 15 fractional bits),
reading only a region of the image. normalize: torchvision ToTensor + Normalize on the result.
"""
import numpy as np


def warp_region(region, origin, inv, out_size):
    """region uint8 [h, w, 3]: the pixels of the image at origin = (x, y) and up; inv float64 [2, 3]: output -> image
    coordinates; out_size = (w, h). Taps outside the region read 0 (the region covers every tap inside the image).
    Returns uint8 [out_h, out_w, 3]."""
    inv = np.asarray(inv, np.float64).reshape(2, 3)
    ow, oh = int(out_size[0]), int(out_size[1])
    x = np.arange(ow, dtype=np.float64)
    y = np.arange(oh, dtype=np.float64)
    # separate numpy multiplies and adds: no fused multiply-add, like the host build of cv2
    X0 = np.rint((inv[0, 1] * y + inv[0, 2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((inv[1, 1] * y + inv[1, 2]) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + np.rint(inv[0, 0] * x * 1024).astype(np.int64)[None, :]) >> 5
    Y = (Y0[:, None] + np.rint(inv[1, 0] * x * 1024).astype(np.int64)[None, :]) >> 5
    ax, ay = X & 31, Y & 31
    xi, yi = (X >> 5) - int(origin[0]), (Y >> 5) - int(origin[1])
    rh, rw = region.shape[:2]
    acc = np.zeros((oh, ow, 3), np.int64)
    for dx, dy, w in ((0, 0, (32 - ax) * (32 - ay)), (1, 0, ax * (32 - ay)), (0, 1, (32 - ax) * ay), (1, 1, ax * ay)):
        tx, ty = xi + dx, yi + dy
        inside = (tx >= 0) & (tx < rw) & (ty >= 0) & (ty < rh)
        v = np.zeros((oh, ow, 3), np.int64)
        if inside.any():
            v[inside] = region[ty[inside], tx[inside]]
        acc += v * (w * 32)[:, :, None]
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def normalize(crop_u8, mean, std):
    """ToTensor + Normalize: uint8 HWC -> float32 CHW, (u8 / 255 - mean) / std with two fp32 divisions."""
    t = crop_u8.transpose(2, 0, 1).astype(np.float32) / np.float32(255.0)
    return (t - np.asarray(mean, np.float32)[:, None, None]) / np.asarray(std, np.float32)[:, None, None]


class StandInDataset:
    """The attributes of the reference's JointsDataset (lib/dataset/JointsDataset.py:28-57) and COCO / MPII subclasses
    that fpd_b200.augment.RawJointsDataset reads, with half_body_transform restated (:62-104). cfg is a dict:
    is_train, color_rgb, image_size (w, h), heatmap_size, sigma, scale_factor, rotation_factor, flip,
    num_joints_half_body, prob_half_body, num_joints, flip_pairs, upper_body_ids, mean, std."""

    pixel_std = 200

    def __init__(self, cfg, db):
        from torchvision import transforms as T
        self.is_train = bool(cfg['is_train'])
        self.color_rgb = bool(cfg['color_rgb'])
        self.data_format = 'png'
        self.image_size = np.array(cfg['image_size'])
        self.heatmap_size = np.array(cfg['heatmap_size'])
        self.sigma = int(cfg['sigma'])
        self.scale_factor = cfg['scale_factor']
        self.rotation_factor = cfg['rotation_factor']
        self.flip = bool(cfg['flip'])
        self.num_joints_half_body = int(cfg['num_joints_half_body'])
        self.prob_half_body = cfg['prob_half_body']
        self.num_joints = int(cfg['num_joints'])
        self.flip_pairs = [list(p) for p in cfg['flip_pairs']]
        self.upper_body_ids = tuple(int(i) for i in cfg['upper_body_ids'])
        # a Python float, as coco.py:61-67 / mpii.py compute it from the config's ints (a numpy float64 would promote the
        # float32 arithmetic of half_body_transform)
        self.aspect_ratio = int(cfg['image_size'][0]) * 1.0 / int(cfg['image_size'][1])
        self.transform = T.Compose([T.ToTensor(), T.Normalize(mean=list(cfg['mean']), std=list(cfg['std']))])
        self.db = db

    def __len__(self):
        return len(self.db)

    def half_body_transform(self, joints, joints_vis):
        upper, lower = [], []
        for j in range(self.num_joints):
            if joints_vis[j][0] > 0:
                (upper if j in self.upper_body_ids else lower).append(joints[j])
        if np.random.randn() < 0.5 and len(upper) > 2:
            sel = upper
        else:
            sel = lower if len(lower) > 2 else upper
        if len(sel) < 2:
            return None, None
        sel = np.array(sel, dtype=np.float32)
        center = sel.mean(axis=0)[:2]
        lt, rb = np.amin(sel, axis=0), np.amax(sel, axis=0)
        w, h = rb[0] - lt[0], rb[1] - lt[1]
        if w > self.aspect_ratio * h:
            h = w * 1.0 / self.aspect_ratio
        elif w < self.aspect_ratio * h:
            w = h * self.aspect_ratio
        scale = np.array([w * 1.0 / self.pixel_std, h * 1.0 / self.pixel_std], dtype=np.float32)
        return center, scale * 1.5
