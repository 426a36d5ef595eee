"""Heat-map target generation on the device for a whole batch: the GPU-side replacement for the per-sample
numpy loop of JointsDataset.generate_target (reference lib/dataset/JointsDataset.py:233-289), to be called on the joints
that come out of the loader's augmentation (after the H2D copy) instead of shipping [B,J,h,w] float targets over PCIe."""
import torch

from . import ops


class TargetGenerator:
    """cfg-like arguments as in JointsDataset.__init__ (:43-52): image_size / heatmap_size are (w, h), sigma = MODEL.SIGMA,
    joints_weight only when LOSS.USE_DIFFERENT_JOINTS_WEIGHT. unbiased: DARK's targets (ops.gaussian_targets_unbiased),
    the Gaussian on the sub-pixel joint instead of the rounded one. udp: UDP's targets (ops.gaussian_targets_udp), for
    joints cropped with RawJointsDataset(udp=True). The two are different encodings: at most one may be set."""

    def __init__(self, image_size, heatmap_size, sigma=2, joints_weight=None, device="cuda", unbiased=False, udp=False):
        if unbiased and udp:
            raise ValueError("TargetGenerator: unbiased (DARK) and udp are two different target encodings; pick one")
        self.image_size = (int(image_size[0]), int(image_size[1]))
        self.heatmap_size = (int(heatmap_size[0]), int(heatmap_size[1]))
        self.sigma = int(sigma)
        self.device = torch.device(device)
        self.unbiased = bool(unbiased)
        self.udp = bool(udp)
        self.joints_weight = None if joints_weight is None else torch.as_tensor(joints_weight, dtype=torch.float32).to(
            self.device)
        self.gauss_table = None   # built on first use; kept so that calls on device tensors copy nothing (graph capture)

    def __call__(self, joints, joints_vis):
        """joints, joints_vis: [B,J,3] (CUDA or host tensors / arrays) -> (target [B,J,h,w], target_weight [B,J,1]) on the device."""
        j = torch.as_tensor(joints, dtype=torch.float32).to(self.device, non_blocking=True).contiguous()
        v = torch.as_tensor(joints_vis, dtype=torch.float32).to(self.device, non_blocking=True).contiguous()
        if self.unbiased:
            return ops.gaussian_targets_unbiased(j, v, self.heatmap_size, self.image_size, self.sigma, self.joints_weight)
        if self.udp:
            return ops.gaussian_targets_udp(j, v, self.heatmap_size, self.image_size, self.sigma, self.joints_weight)
        if self.gauss_table is None:
            self.gauss_table = ops.gaussian_table(self.sigma, self.device)
        return ops.gaussian_targets(j, v, self.heatmap_size, self.image_size, self.sigma, self.joints_weight,
                                    self.gauss_table)
