"""Float64-capable restatements of the auxiliary-loss options beyond oracle/ref_path.py's: SmoothnessLoss's pre-blur
(GaussianSmoothing, Losses/SmoothnessLoss.py:9-72, 92-94) and edge_order, and EdgeLoss with a target image and a mask
(Losses/EdgeLoss.py:60-108).  Kept apart from ref_path.py so the parity tests written against that module keep the
oracle they were written against.  tests/test_aux_loss_options.py pins these to tests/golden/aux_loss_options.npz,
which oracle/make_golden_aux_options.py produced with the unmodified reference classes.
"""
import math

import torch
import torch.nn.functional as F


def gaussian_kernel2d(kernel_size, sigma, dtype=torch.float64):
    """GaussianSmoothing.__init__ for dim 2: ceil(k) taps, mean (k - 1) / 2, exp(-((i - mean) / (2 sigma))^2), normalised."""
    idx = torch.arange(kernel_size, dtype=dtype)
    v = 1 / (sigma * math.sqrt(2 * math.pi)) * torch.exp(-((idx - (kernel_size - 1) / 2) / (2 * sigma)) ** 2)
    k = v[:, None] * v[None, :]
    return k / k.sum()


def smoothness_loss(cutouts, smoothness_weight=1.0, smoothness_type="default", spacing=1, edge_order=1,
                    gaussian_kernel=0, gaussian_std=1.0):
    """SmoothnessLoss.get_loss for one cutout batch [N, 3, cs, cs]: optional valid depthwise blur, then torch.gradient
    over the stacked rows [N * cs', cs', 3] (the row difference crosses cutout boundaries)."""
    if gaussian_kernel:
        w = gaussian_kernel2d(gaussian_kernel, gaussian_std, cutouts.dtype)
        cutouts = F.conv2d(cutouts, w[None, None].repeat(3, 1, 1, 1), groups=3)
    px = cutouts.permute(0, 2, 3, 1).reshape(-1, cutouts.shape[2], 3)
    sq = 0
    for c in range(3):
        gy, gx = torch.gradient(px[:, :, c], spacing=spacing, edge_order=edge_order)
        sq = sq + gy ** 2 + gx ** 2
    sharp = torch.sqrt(sq)
    if smoothness_type == "clipped":
        sharp = torch.clamp(sharp, max=0.5)
    elif smoothness_type == "log":
        sharp = torch.log(torch.ones_like(sharp) + sharp)
    return torch.mean(sharp) * smoothness_weight


def edge_loss(out, edge_color, margins_px, edge_color_weight=0.1, global_color_weight=0.05, target=None, mask=None):
    """EdgeLoss.get_loss: target [1, 3, H, W] (the resized edge_input_image) replaces the flat colour; mask [1, 1, H, W]
    (the resized edge_mask_image) replaces the margins by mse(where(mask > 0, target, out), target)."""
    lmax, rmax = out.shape[2], out.shape[3]
    if target is None:
        target = torch.zeros_like(out)
        for c in range(3):
            target[:, c] = edge_color[c]
    target = target.to(out.dtype)
    cur = torch.zeros((), dtype=out.dtype)
    if mask is None:
        left, right, upper, lower = margins_px
        if left != 0:
            cur = cur + F.mse_loss(out[:, :, :, :left], target[:, :, :, :left])
        if right != 0:
            cur = cur + F.mse_loss(out[:, :, :, rmax - right:], target[:, :, :, rmax - right:])
        if upper != 0:
            cur = cur + F.mse_loss(out[:, :, :upper, left:rmax - right], target[:, :, :upper, left:rmax - right])
        if lower != 0:
            cur = cur + F.mse_loss(out[:, :, lmax - lower:, left:rmax - right], target[:, :, lmax - lower:, left:rmax - right])
    else:
        cur = cur + F.mse_loss(torch.where(mask > 0, target, out), target)
    if global_color_weight:
        cur = cur + F.mse_loss(out, target) * global_color_weight
    return cur * edge_color_weight
