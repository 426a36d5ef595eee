"""Heat-map target generation on the device for a whole batch: the GPU-side replacement for the per-sample
numpy loop of JointsDataset.generate_target (reference lib/dataset/JointsDataset.py:233-289), to be called on the joints
that come out of the loader's augmentation (after the H2D copy) instead of shipping [B,J,h,w] float targets over PCIe."""
import torch

from . import ops


class TargetGenerator:
    """cfg-like arguments as in JointsDataset.__init__ (:43-52): image_size / heatmap_size are (w, h), sigma = MODEL.SIGMA,
    joints_weight only when LOSS.USE_DIFFERENT_JOINTS_WEIGHT."""

    def __init__(self, image_size, heatmap_size, sigma=2, joints_weight=None, device="cuda"):
        self.image_size = (int(image_size[0]), int(image_size[1]))
        self.heatmap_size = (int(heatmap_size[0]), int(heatmap_size[1]))
        self.sigma = int(sigma)
        self.device = torch.device(device)
        self.joints_weight = None if joints_weight is None else torch.as_tensor(joints_weight, dtype=torch.float32).to(
            self.device)

    def __call__(self, joints, joints_vis):
        """joints, joints_vis: [B,J,3] (CUDA or host tensors / arrays) -> (target [B,J,h,w], target_weight [B,J,1]) on the device."""
        j = torch.as_tensor(joints, dtype=torch.float32).to(self.device, non_blocking=True).contiguous()
        v = torch.as_tensor(joints_vis, dtype=torch.float32).to(self.device, non_blocking=True).contiguous()
        return ops.gaussian_targets(j, v, self.heatmap_size, self.image_size, self.sigma, self.joints_weight)
