"""Test infrastructure (NOT product code): the reference's line-of-sight loss (model/runner.py:255-276) and patch-loss
branch (:278-369) restated in torch, expression by expression, on any device.  tests/test_losses_hostsim.py pins this
restatement to the unmodified reference's Trainer.train_step (tests/golden/train_losses.npz) and holds the kernels' math
to it on the CPU; tests/test_gpu_losses.py holds the CUDA ops to it on identical CUDA tensors."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

OPTION_SETS = {            # the option sets of tests/golden/train_losses.npz (patch [2, 8] in every one)
    "defaults": {},
    "urf": dict(urf_loss=True),
    "sobel": dict(sobel_grad=True),
    "mse": dict(depth_grad_loss="mse"),
    "huber": dict(depth_grad_loss="huber"),
    "bce": dict(depth_grad_loss="bce"),
    "cos": dict(depth_grad_loss="cos"),
    "smooth": dict(grad_norm_smooth=True, spatial_smooth=True, tv_loss=True),
}

DEFAULTS = dict(depth_grad_loss="l1", sobel_grad=False, grad_loss=True, alpha_grad=0.1, grad_norm_smooth=False,
                alpha_grad_norm=0.1, spatial_smooth=False, alpha_spatial=0.1, tv_loss=False, alpha_tv=0.1, scale=0.01)


def grad_criterion(name, scale, delta=None):
    """main_lidar4d.py:183-188 (delta: the huber delta, 0.2 * scale unless given)."""
    return {"mse": torch.nn.MSELoss(reduction="none"), "l1": torch.nn.L1Loss(reduction="none"),
            "bce": torch.nn.BCEWithLogitsLoss(reduction="none"),
            "huber": torch.nn.HuberLoss(reduction="none", delta=0.2 * scale if delta is None else delta), "cos": torch.nn.CosineSimilarity()}[name]


def los_eps(global_step, iters):
    """runner.py:257."""
    return 0.02 * 0.1 ** min(global_step / iters, 1)


def line_of_sight_ref(weights, z_vals, gt, eps):
    """runner.py:258-276: 0.1 * loss_empty + 0.1 * loss_near; gt [.., n, 3] (raydrop, intensity, depth)."""
    g = gt.reshape(-1, 3)
    gt_depth = g[:, 2] * g[:, 0]
    depth_mask = gt_depth.reshape(z_vals.shape[0], 1) > 0.0
    gd = gt_depth.reshape(z_vals.shape[0], 1)
    mask_empty = (z_vals < (gd - eps)) | (z_vals > (gd + eps))
    loss_empty = ((mask_empty * weights) ** 2).sum() / depth_mask.sum()
    mask_near = (z_vals > (gd - eps)) & (z_vals < (gd + eps))
    distance = mask_near * (z_vals - gd)
    sigma = eps / 3.
    distr = 1.0 / (sigma * np.sqrt(2 * np.pi)) * torch.exp(-(distance ** 2 / (2 * sigma ** 2)))
    distr /= distr.max()
    distr *= mask_near
    loss_near = ((mask_near * weights - distr) ** 2).sum() / depth_mask.sum()
    return 0.1 * loss_empty + 0.1 * loss_near


def patch_ref(depth, gt, patch_size, huber_delta=None, **kw):
    """runner.py:278-369 (the branch's summed contribution to `loss`); depth [.., n], gt [.., n, 3].  huber_delta
    overrides 0.2 * scale (for evaluating the branch on inputs already divided by scale)."""
    o = dict(DEFAULTS)
    o.update({k: v for k, v in kw.items() if k in DEFAULTS})
    if isinstance(patch_size, int):
        px, py = patch_size, patch_size
    elif len(patch_size) == 1:
        px, py = patch_size[0], patch_size[0]
    else:
        px, py = patch_size
    g = gt.reshape(-1, 3)
    gt_raydrop = g[:, 0]
    gt_depth = g[:, 2] * gt_raydrop
    pred_depth = depth.reshape(-1) * gt_raydrop
    loss = torch.zeros((), device=depth.device)
    if not px > 1:
        return loss
    dev = depth.device
    kx = torch.tensor([[-1, 0, 1], [-2, 0, 2], [-1, 0, 1]], dtype=torch.float32).unsqueeze(0).unsqueeze(0).to(dev)
    ky = torch.tensor([[-1, -2, -1], [0, 0, 0], [1, 2, 1]], dtype=torch.float32).unsqueeze(0).unsqueeze(0).to(dev)
    pred_depth = pred_depth.view(-1, px, py, 1).permute(0, 3, 1, 2).contiguous() / o["scale"]
    if o["sobel_grad"]:
        pred_grad_x = F.conv2d(pred_depth, kx, padding=1)
        pred_grad_y = F.conv2d(pred_depth, ky, padding=1)
    else:
        pred_grad_y = torch.abs(pred_depth[:, :, :-1, :] - pred_depth[:, :, 1:, :])
        pred_grad_x = torch.abs(pred_depth[:, :, :, :-1] - pred_depth[:, :, :, 1:])
    dy = torch.abs(pred_grad_y)
    dx = torch.abs(pred_grad_x)
    if o["grad_norm_smooth"]:
        loss = loss + o["alpha_grad_norm"] * (torch.mean(torch.exp(-dx)) + torch.mean(torch.exp(-dy)))
    if o["spatial_smooth"]:
        loss = loss + o["alpha_spatial"] * (torch.mean(dx ** 2) + torch.mean(dy ** 2))
    if o["tv_loss"]:
        loss = loss + o["alpha_tv"] * (torch.mean(dx) + torch.mean(dy))
    if o["grad_loss"]:
        gt_depth = gt_depth.view(-1, px, py, 1).permute(0, 3, 1, 2).contiguous() / o["scale"]
        gt_raydrop = gt_raydrop.view(-1, px, py, 1).permute(0, 3, 1, 2).contiguous()
        if o["sobel_grad"]:
            gt_grad_x = F.conv2d(gt_depth, kx, padding=1)
        else:
            gt_grad_x = gt_depth[:, :, :, :-1] - gt_depth[:, :, :, 1:]
        grad_mask_x = torch.where(torch.abs(gt_grad_x) < 0.01, 1, 0)
        mask_dx = gt_raydrop * grad_mask_x if o["sobel_grad"] else gt_raydrop[:, :, :, :-1] * grad_mask_x
        crit = grad_criterion(o["depth_grad_loss"], o["scale"], huber_delta)
        if o["depth_grad_loss"] == "cos":
            patch_num = pred_grad_x.shape[0]
            grad_loss = 1 - crit((pred_grad_x * mask_dx).reshape(patch_num, -1), (gt_grad_x * mask_dx).reshape(patch_num, -1))
        else:
            grad_loss = crit(pred_grad_x * mask_dx, gt_grad_x * mask_dx)
        loss = loss + o["alpha_grad"] * grad_loss.sum()
    return loss


def extra_losses_ref(out, gt, opt, global_step):
    """What train_step adds after the flow loss, for a render output `out` and an opt namespace."""
    loss = torch.zeros((), device=out["depth_lidar"].device)
    if opt.urf_loss:
        loss = loss + line_of_sight_ref(out["weights"], out["z_vals"], gt, los_eps(global_step, opt.iters))
    return loss + patch_ref(out["depth_lidar"], gt, opt.patch_size_lidar, **vars(opt))


def patch_gt(n_patch, px, py, seed, device="cpu", drop=0.15, flat=0.6):
    """Synthetic gt3 [n, 3] for patch batches: depth constant over runs of columns with random jumps of about the 0.01
    threshold (after /scale = 0.01) and dropped rays (m = 0).  The depths are small (< 0.007, so depth / scale < 0.7):
    the branch takes differences of depth / scale, and at the dataset's depths (~65 after /scale) one ulp of an operand
    is already 1e-4 of a typical difference, so any change of rounding order would dominate a comparison.  Depths are
    multiples of 2^-16 (see quantize)."""
    g = np.random.default_rng(seed)
    n = n_patch * px * py
    base = 5e-4 + 6e-3 * g.random((n_patch, px, 1))
    jump = (g.random((n_patch, px, py)) > flat) * g.normal(0, 2e-4, (n_patch, px, py))
    depth = quantize((base + np.cumsum(jump, axis=2)).reshape(n))
    m = (g.random(n) > drop).astype(np.float32)
    gt = np.stack([m, g.random(n) * 0.5, depth], -1).astype(np.float32)
    return torch.from_numpy(gt).to(device)


def quantize(x):
    """Round to multiples of 2^-16.  For such depths below 0.01, depth * (1 / 0.01f) = depth * 100 and every finite
    difference or Sobel sum of them is exact in fp32, whatever the order of the additions: the comparisons then test
    the math, not the rounding order (cos against a gt vector that is zero in exact arithmetic but 1e-9 after one
    rounding, for one, is noise in the reference itself)."""
    return (np.round(np.asarray(x, np.float64) * 65536.0) / 65536.0).astype(np.float32)
