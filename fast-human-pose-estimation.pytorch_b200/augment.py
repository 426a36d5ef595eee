"""GPU input path of the training / validation loaders: the per-sample crop of JointsDataset.__getitem__
(reference lib/dataset/JointsDataset.py:113-198) split into a host part that only decodes, draws the augmentation and cuts
out the source pixels the crop reads, and a device part that warps, normalises and builds the heat-map targets for the
whole batch.

    train_dataset = RawJointsDataset(COCODataset(cfg, ..., transforms.Compose([ToTensor(), Normalize(mean, std)])))
    loader = DataLoader(train_dataset, ..., collate_fn=raw_collate, pin_memory=True)
    loader = DeviceCropLoader(loader, cfg.MODEL.HEATMAP_SIZE, cfg.MODEL.SIGMA)
    for input, target, target_weight, meta in loader:   # what function.train / fpd_train / validate iterate over

The device input is bit-identical to the reference's: the crop kernel (csrc/augment.cu) is an exact model of
cv2.warpAffine(INTER_LINEAR) on 8-bit images followed by ToTensor + Normalize, and the matrices are computed as the
reference computes them. The host sends uint8 pixels and small descriptors instead of float crops and float targets.
"""
import copy
import random

import numpy as np
import torch

from . import ops
from .targets import TargetGenerator

# the region handed to the device extends this many pixels beyond the crop's real-valued footprint: one for the second
# bilinear tap, one for the 1/32-pixel rounding of the fixed-point coordinates
REGION_MARGIN = 2


def crop_matrix(center, scale, rot, output_size):
    """The forward 2x3 crop matrix of the reference's get_affine_transform (lib/utils/transforms.py:45-82, inv=0, no
    shift), bit for bit: the same three float32 point pairs, solved by cv2.getAffineTransform (a numpy solve differs in the
    last bits, and that changes crop pixels)."""
    import cv2
    if not isinstance(scale, (np.ndarray, list)):
        scale = np.array([scale, scale])
    box = scale * 200.0
    out_w, out_h = output_size[0], output_size[1]
    rot_rad = np.pi * rot / 180
    sn, cs = np.sin(rot_rad), np.cos(rot_rad)
    half = box[0] * -0.5
    up = [0 * cs - half * sn, 0 * sn + half * cs]            # (0, -w/2) rotated by rot
    src = np.zeros((3, 2), dtype=np.float32)
    dst = np.zeros((3, 2), dtype=np.float32)
    src[0, :] = center
    src[1, :] = center + up
    dst[0, :] = [out_w * 0.5, out_h * 0.5]
    dst[1, :] = np.array([out_w * 0.5, out_h * 0.5]) + np.array([0, out_w * -0.5], np.float32)
    for pts in (src, dst):                                    # third point: the first rotated by 90 degrees about the second
        d = pts[0, :] - pts[1, :]
        pts[2, :] = pts[1, :] + np.array([-d[1], d[0]], dtype=np.float32)
    return cv2.getAffineTransform(np.float32(src), np.float32(dst))


def udp_crop_matrix(center, scale, rot, output_size):
    """The forward 2x3 crop matrix of UDP (unbiased data processing, Huang et al., CVPR 2020), in float64 and closed
    form. Sizes are pixel spacings and positions pixel centres: rotate about `center` by `rot` degrees, in crop_matrix's
    direction; scale each axis by (output_size - 1) / (scale * 200); move `center` to ((w - 1) / 2, (h - 1) / 2). The
    box edges then land on the first and last output pixel centres, and mirroring the image (x -> width - 1 - x, the
    centre with it) mirrors the crop (x -> w - 1 - x) when rot = 0."""
    box = np.broadcast_to(np.asarray(scale, np.float64).reshape(-1), (2,)) * 200.0
    kx, ky = (output_size[0] - 1.0) / box[0], (output_size[1] - 1.0) / box[1]
    rot_rad = np.pi * rot / 180
    sn, cs = np.sin(rot_rad), np.cos(rot_rad)
    m = np.array([[kx * cs, kx * sn, 0.0], [-ky * sn, ky * cs, 0.0]])
    cx, cy = float(center[0]), float(center[1])
    m[0, 2] = (output_size[0] - 1.0) * 0.5 - (m[0, 0] * cx + m[0, 1] * cy)
    m[1, 2] = (output_size[1] - 1.0) * 0.5 - (m[1, 0] * cx + m[1, 1] * cy)
    return m


def invert_affine(m):
    """cv2.invertAffineTransform of a float64 2x3 matrix, in the same operation order (and so the same bits); it is also
    the inversion warpAffine applies internally."""
    m = np.asarray(m, np.float64)
    d = m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0]
    d = 1.0 / d if d != 0 else 0.0
    a11, a22 = m[1, 1] * d, m[0, 0] * d
    a12, a21 = m[0, 1] * -d, m[1, 0] * -d
    b1 = -a11 * m[0, 2] - a12 * m[1, 2]
    b2 = -a21 * m[0, 2] - a22 * m[1, 2]
    return np.array([[a11, a12, b1], [a21, a22, b2]], np.float64)


def source_window(inv, out_size, img_w, img_h):
    """(x0, y0, x1, y1): the part of a img_w x img_h image that a crop of out_size = (w, h) through `inv` reads, with
    REGION_MARGIN, clipped to the image (empty when the crop lies outside it)."""
    ow, oh = int(out_size[0]), int(out_size[1])
    xs = np.array([0, ow - 1, 0, ow - 1], np.float64)
    ys = np.array([0, 0, oh - 1, oh - 1], np.float64)
    sx = inv[0, 0] * xs + inv[0, 1] * ys + inv[0, 2]
    sy = inv[1, 0] * xs + inv[1, 1] * ys + inv[1, 2]

    def span(v, size):
        lo = int(np.clip(np.floor(v.min()) - REGION_MARGIN, 0, size))
        hi = int(np.clip(np.floor(v.max()) + REGION_MARGIN + 1, 0, size))
        return lo, max(lo, hi)
    (x0, x1), (y0, y1) = span(sx, img_w), span(sy, img_h)
    return x0, y0, x1, y1


def _flip_joints(joints, joints_vis, width, flip_pairs):
    """fliplr_joints (lib/utils/transforms.py:32-45)."""
    joints[:, 0] = width - joints[:, 0] - 1
    for a, b in flip_pairs:
        joints[[a, b], :] = joints[[b, a], :]
        joints_vis[[a, b], :] = joints_vis[[b, a], :]
    return joints * joints_vis, joints_vis


def _normalize_of(transform):
    """(mean, std) as float32 from the loader's transform, which must be ToTensor followed by Normalize."""
    from torchvision import transforms as T
    steps = getattr(transform, "transforms", None)
    if not (isinstance(transform, T.Compose) and len(steps) == 2 and isinstance(steps[0], T.ToTensor)
            and isinstance(steps[1], T.Normalize)):
        raise ValueError("RawJointsDataset: the dataset's transform must be Compose([ToTensor(), Normalize(mean, std)]), "
                         "got %r" % (transform,))
    mean = np.asarray(steps[1].mean, np.float32).reshape(-1)
    std = np.asarray(steps[1].std, np.float32).reshape(-1)
    if mean.size != 3 or std.size != 3:
        raise ValueError("RawJointsDataset: Normalize needs 3 means and 3 deviations")
    return mean, std


class RawJointsDataset(torch.utils.data.Dataset):
    """Wraps a reference JointsDataset (COCO or MPII). An item is what the reference's __getitem__ computes up to the warp
    -- the same draws from np.random / random, in the same order, and base.half_body_transform -- plus the source pixels
    the crop reads, so that the device can finish it:

        region      uint8 [h, w, 3]: the pixels of the (mirrored when flipped) image the crop reads, in RGB order when
                    DATASET.COLOR_RGB is set
        desc        int64 [7]: 0, region x, y, w, h, image w, h (the first column becomes the byte offset in raw_collate)
        inv         float64 [2, 3]: output -> image coordinates
        joints, joints_vis: float64 [J, 3], transformed as the reference transforms them
        meta        the reference's meta dict

    udp=True crops with udp_crop_matrix instead of the reference's matrix, for UDP training and validation; pair it with
    DeviceCropLoader(..., udp=True) and, for validation, TEST.UDP.
    teacher_image_size=(w, h): a teacher distilled at its own input size. The item also holds teacher_inv, the inverse of
    the same crop (same centre, scale, rotation, flip and half-body draw) at that size, and the region covers what both
    crops read; DeviceCropLoader then crops the teacher's input too. The size must have the student's aspect ratio: the
    crop matrix scales both axes by the box width, so another aspect would crop another part of the box.
    """

    def __init__(self, base, udp=False, teacher_image_size=None):
        self.base = base
        self.udp = bool(udp)
        self.mean, self.std = _normalize_of(base.transform)
        self.image_size = (int(base.image_size[0]), int(base.image_size[1]))
        self.teacher_image_size = None
        if teacher_image_size is not None:
            tw, th = (int(v) for v in teacher_image_size)
            sw, sh = self.image_size
            if tw < 1 or th < 1:
                raise ValueError("RawJointsDataset: teacher_image_size=%r must be positive" % (teacher_image_size,))
            if tw * sh != sw * th:
                raise ValueError("RawJointsDataset: teacher_image_size %dx%d has another aspect ratio than the student's "
                                 "%dx%d: the crop would cover another part of the box" % (tw, th, sw, sh))
            self.teacher_image_size = (tw, th)

    def __len__(self):
        return len(self.base)

    def read_image(self, image_file):
        """Decode as the reference does (JointsDataset.py:118-126), BGR."""
        import cv2
        flags = cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION
        if self.base.data_format == 'zip':
            from utils import zipreader   # the reference's lib/utils, on sys.path wherever its datasets are
            img = zipreader.imread(image_file, flags)
        else:
            img = cv2.imread(image_file, flags)
        if img is None:
            raise ValueError('Fail to read {}'.format(image_file))
        return img

    def __getitem__(self, idx):
        b = self.base
        rec = copy.deepcopy(b.db[idx])
        image_file = rec['image']
        img = self.read_image(image_file)
        joints, joints_vis = rec['joints_3d'], rec['joints_3d_vis']
        c, s = rec['center'], rec['scale']
        r = 0
        flipped = False
        if b.is_train:   # JointsDataset.py:143-168, draw for draw
            if np.sum(joints_vis[:, 0]) > b.num_joints_half_body and np.random.rand() < b.prob_half_body:
                c_half_body, s_half_body = b.half_body_transform(joints, joints_vis)
                if c_half_body is not None and s_half_body is not None:
                    c, s = c_half_body, s_half_body
            sf, rf = b.scale_factor, b.rotation_factor
            s = s * np.clip(np.random.randn() * sf + 1, 1 - sf, 1 + sf)
            r = np.clip(np.random.randn() * rf, -rf * 2, rf * 2) if random.random() <= 0.6 else 0
            if b.flip and random.random() <= 0.5:
                flipped = True
                joints, joints_vis = _flip_joints(joints, joints_vis, img.shape[1], b.flip_pairs)
                c[0] = img.shape[1] - c[0] - 1
        matrix = udp_crop_matrix if self.udp else crop_matrix
        trans = matrix(c, s, r, b.image_size)
        inv = invert_affine(trans)
        img_h, img_w = img.shape[:2]
        x0, y0, x1, y1 = source_window(inv, self.image_size, img_w, img_h)
        teacher_inv = None
        if self.teacher_image_size is not None:
            teacher_inv = invert_affine(matrix(c, s, r, self.teacher_image_size))
            x0, y0, x1, y1 = _union(source_window(teacher_inv, self.teacher_image_size, img_w, img_h), (x0, y0, x1, y1))
        # one copy: rows, the columns of the mirrored image (reversed when flipped), channels reversed for RGB
        cols = slice(img_w - 1 - x0, img_w - 1 - x1 if x1 < img_w else None, -1) if flipped else slice(x0, x1)
        chans = slice(None, None, -1) if b.color_rgb else slice(None)
        region = np.ascontiguousarray(img[y0:y1, cols, chans]) if x1 > x0 and y1 > y0 else \
            np.zeros((0, 0, 3), np.uint8)
        for i in range(b.num_joints):
            if joints_vis[i, 0] > 0.0:
                joints[i, 0:2] = np.dot(trans, np.array([joints[i, 0], joints[i, 1], 1.]).T)[:2]
        meta = {'image': image_file, 'filename': rec.get('filename', ''), 'imgnum': rec.get('imgnum', ''),
                'joints': joints, 'joints_vis': joints_vis, 'center': c, 'scale': s, 'rotation': r,
                'score': rec.get('score', 1)}
        desc = np.array([0, x0, y0, region.shape[1], region.shape[0], img_w, img_h], np.int64)
        item = {'region': region, 'desc': desc, 'inv': inv, 'joints': joints, 'joints_vis': joints_vis,
                'out_size': self.image_size, 'mean': self.mean, 'std': self.std, 'meta': meta}
        if teacher_inv is not None:
            item.update(teacher_inv=teacher_inv, teacher_out_size=self.teacher_image_size, teacher_udp=self.udp)
        return item


def _union(a, b):
    """The smallest window (x0, y0, x1, y1) holding windows a and b; an empty window adds nothing. The crop kernel reads
    each tap relative to the region, so a region grown beyond a crop's own window leaves that crop's pixels unchanged."""
    def empty(w):
        return w[2] <= w[0] or w[3] <= w[1]
    if empty(a):
        return b
    if empty(b):
        return a
    return min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2]), max(a[3], b[3])


def add_unlabeled_boxes(dataset, bbox_file, image_path=None, score_thre=0.0):
    """Append the person boxes of a COCO-format detection list (the format of TEST.COCO_BBOX_FILE: a JSON list of
    {"image_id", "category_id", "bbox": [x, y, w, h], "score"}) to dataset.db as unlabeled training records, for
    distillation from unlabeled boxes (KD.UNLABELED). One record per box with category_id 1 and score >= score_thre:
    centre and scale from dataset._box2cs(bbox), zero joints_3d and joints_3d_vis (so all-zero targets and target
    weights), the detection score kept. image_path maps an image_id to a file (default: dataset.image_path_from_index).
    Returns the number of records added. RawJointsDataset crops them as any record; with zero visibility there is no
    half-body draw, as in the reference's __getitem__."""
    import json
    if image_path is None:
        image_path = dataset.image_path_from_index
    with open(bbox_file, 'r') as f:
        boxes = json.load(f)
    # the dataset's joint count; a dataset object without one takes it from its existing records
    J = int(dataset.num_joints) if hasattr(dataset, 'num_joints') else len(dataset.db[0]['joints_3d'])
    n = 0
    for det in boxes:
        if det['category_id'] != 1 or det['score'] < score_thre:
            continue
        center, scale = dataset._box2cs(det['bbox'])
        dataset.db.append({'image': image_path(det['image_id']), 'center': center, 'scale': scale,
                           'score': det['score'], 'joints_3d': np.zeros((J, 3), np.float64),
                           'joints_3d_vis': np.zeros((J, 3), np.float64), 'filename': '', 'imgnum': 0})
        n += 1
    return n


def raw_collate(items):
    """Batch of RawJointsDataset items -> dict of CPU tensors (pinned by the DataLoader's pin_memory):
    pixels uint8 [total bytes] (the regions back to back), desc int64 [N,7] (column 0 = byte offset), inv float64 [N,6],
    joints / joints_vis float32 [N,J,3], out_size int64 [2] = (w, h), norm float32 [6] = mean, std, and meta collated
    as default_collate does. Items with a teacher crop add teacher_inv float64 [N,6], teacher_out_size int64 [2] and
    teacher_udp (bool)."""
    from torch.utils.data import default_collate
    first = items[0]
    teacher = 'teacher_inv' in first
    for it in items[1:]:
        if it['out_size'] != first['out_size'] or not (np.array_equal(it['mean'], first['mean'])
                                                        and np.array_equal(it['std'], first['std'])):
            raise ValueError("raw_collate: samples of one batch need the same output size and normalisation")
        if ('teacher_inv' in it) != teacher or (teacher and (it['teacher_out_size'] != first['teacher_out_size']
                                                             or it['teacher_udp'] != first['teacher_udp'])):
            raise ValueError("raw_collate: samples of one batch need the same teacher crop size and convention")
    sizes = [it['region'].size for it in items]
    desc = np.stack([it['desc'] for it in items])
    desc[:, 0] = np.cumsum([0] + sizes[:-1])
    pixels = np.concatenate([it['region'].reshape(-1) for it in items]) if sum(sizes) else np.zeros(0, np.uint8)
    batch = {
        'pixels': torch.from_numpy(pixels),
        'desc': torch.from_numpy(desc),
        'inv': torch.from_numpy(np.stack([it['inv'].reshape(6) for it in items])),
        'joints': torch.from_numpy(np.stack([it['joints'] for it in items]).astype(np.float32)),
        'joints_vis': torch.from_numpy(np.stack([it['joints_vis'] for it in items]).astype(np.float32)),
        'out_size': torch.tensor(first['out_size'], dtype=torch.int64),
        'norm': torch.from_numpy(np.concatenate([first['mean'], first['std']]).astype(np.float32)),
        'meta': default_collate([it['meta'] for it in items]),
    }
    if teacher:
        batch.update(teacher_inv=torch.from_numpy(np.stack([it['teacher_inv'].reshape(6) for it in items])),
                     teacher_out_size=torch.tensor(first['teacher_out_size'], dtype=torch.int64),
                     teacher_udp=bool(first['teacher_udp']))
    return batch


class DeviceCropLoader:
    """Iterates a DataLoader of raw_collate batches and yields (input [N,3,h,w], target [N,J,hh,hw], target_weight [N,J,1],
    meta): input and targets on the device, meta on the CPU -- the tuple function.train / fpd_train / validate expect.
    Per batch: the H2D copies, one crop launch and one TargetGenerator call. heatmap_size = (w, h) and sigma as
    cfg.MODEL.HEATMAP_SIZE / SIGMA; joints_weight as the dataset's when LOSS.USE_DIFFERENT_JOINTS_WEIGHT; unbiased=True
    builds DARK's unbiased targets, udp=True UDP's targets for a RawJointsDataset(udp=True) loader (TargetGenerator;
    not both). A batch of a RawJointsDataset(teacher_image_size=...) gets a second crop launch over the same pixels at
    the teacher's size and normalisation: meta['teacher_input'] (device [N,3,Ht,Wt]) and meta['teacher_udp'] (the
    dataset's udp), which fpd_train hands to the teacher."""

    def __init__(self, loader, heatmap_size, sigma, joints_weight=None, device=None, unbiased=False, udp=False):
        if unbiased and udp:
            raise ValueError("DeviceCropLoader: unbiased (DARK) and udp are two different target encodings; pick one")
        self.loader = loader
        self.heatmap_size = (int(heatmap_size[0]), int(heatmap_size[1]))
        self.sigma = int(sigma)
        self.joints_weight = joints_weight
        self.unbiased = bool(unbiased)
        self.udp = bool(udp)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._targets = {}

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        for batch in self.loader:
            yield self.process(batch)

    def to_device(self, batch):
        """The batch's tensors (not meta) copied to the device, asynchronously from pinned memory."""
        keys = ('pixels', 'desc', 'inv', 'joints', 'joints_vis') + (('teacher_inv',) if 'teacher_inv' in batch else ())
        return {k: batch[k].to(self.device, non_blocking=True) for k in keys}

    def device_step(self, dev, batch):
        """(input, target, target_weight) from the device tensors of to_device(batch); enqueues only device work (it can
        be captured into a CUDA graph). batch supplies the host copies of desc / inv, out_size and norm."""
        out_size = tuple(int(v) for v in batch['out_size'])
        norm = batch['norm'].numpy()
        inp = ops.crop_affine_normalize(dev['pixels'], dev['desc'], dev['inv'], out_size, norm[:3], norm[3:],
                                        desc_host=batch['desc'], inv_host=batch['inv'])
        gen = self._targets.get(out_size)
        if gen is None:
            gen = self._targets[out_size] = TargetGenerator(out_size, self.heatmap_size, self.sigma, self.joints_weight,
                                                            self.device, unbiased=self.unbiased, udp=self.udp)
        target, target_weight = gen(dev['joints'], dev['joints_vis'])
        return inp, target, target_weight

    def teacher_crop(self, dev, batch):
        """The teacher's input [N,3,Ht,Wt] from the device tensors of to_device(batch): the student's region and
        normalisation through the teacher's inverse matrices."""
        norm = batch['norm'].numpy()
        return ops.crop_affine_normalize(dev['pixels'], dev['desc'], dev['teacher_inv'],
                                         tuple(int(v) for v in batch['teacher_out_size']), norm[:3], norm[3:],
                                         desc_host=batch['desc'], inv_host=batch['teacher_inv'])

    def process(self, batch):
        dev = self.to_device(batch)
        inp, target, target_weight = self.device_step(dev, batch)
        meta = batch['meta']
        if 'teacher_inv' in batch:
            meta['teacher_input'] = self.teacher_crop(dev, batch)
            meta['teacher_udp'] = batch['teacher_udp']
        return inp, target, target_weight, meta
