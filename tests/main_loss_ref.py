"""Test infrastructure (NOT product code): the main LiDAR loss of the reference's train_step (model/runner.py:193-220,
with its chamfer term) and eval_step's loss (:409-421) restated in torch, expression by expression, on any device.
tests/test_main_loss_hostsim.py pins it to the unmodified reference Trainer (tests/golden/main_loss_ref.npz) and holds
the kernels' math to it on the CPU; tests/test_gpu_main_loss.py holds the CUDA ops to it on identical CUDA tensors."""
from __future__ import annotations

import hashlib

import numpy as np
import torch

CRITERIA = ("l1", "mse", "huber", "bce", "cos")

# the criteria combinations of tests/golden/main_loss_ref.npz: (depth_loss, raydrop_loss, intensity_loss)
COMBOS = {"defaults": ("l1", "mse", "mse"), "all_cos": ("cos", "cos", "cos"), "all_bce": ("bce", "bce", "bce")}
for _slot, _name in enumerate(("depth", "raydrop", "intensity")):
    for _c in CRITERIA:
        _t = list(COMBOS["defaults"])
        _t[_slot] = _c
        if tuple(_t) not in COMBOS.values():
            COMBOS[f"{_name}_{_c}"] = tuple(_t)

SCALES = (0.01, 0.010504329815187737)
SIZES = {"n1": (1, None), "n37": (37, None), "n1024": (1024, None), "patch2x8": (32, (2, 8))}
ALPHAS = dict(alpha_d=1.0, alpha_r=0.01, alpha_i=0.1, smooth_factor=0.2)


def criterion(name, scale):
    """main_lidar4d.py:183-188."""
    return {"mse": torch.nn.MSELoss(reduction="none"), "l1": torch.nn.L1Loss(reduction="none"),
            "bce": torch.nn.BCEWithLogitsLoss(reduction="none"),
            "huber": torch.nn.HuberLoss(reduction="none", delta=0.2 * scale), "cos": torch.nn.CosineSimilarity()}[name]


def train_ref(depth, image, gt, combo, scale, rays_d=None, cham_fn=None, alpha_d=1.0, alpha_r=0.01, alpha_i=0.1,
              smooth_factor=0.2, recip=False):
    """runner.py:193-220: depth [1, N], image [1, N, 2], gt [1, N, 3], rays_d [1, N, 3]; the chamfer term when cham_fn is
    given (cham_fn(a, b) -> dist1, dist2, idx1, idx2).  recip: evaluate the clouds' `/ scale` as ATen does on CUDA, as a
    product with the fp32 reciprocal of scale (on the CPU ATen divides; on CUDA the two are the same)."""
    cd, cr, ci = (criterion(c, scale) for c in combo)
    gt_raydrop = gt[:, :, 0]
    gt_intensity = gt[:, :, 1] * gt_raydrop
    gt_depth = gt[:, :, 2] * gt_raydrop
    pred_raydrop = image[:, :, 0]
    pred_intensity = image[:, :, 1] * gt_raydrop
    pred_depth = depth * gt_raydrop
    if combo[1] == "bce":
        pred_raydrop = torch.sigmoid(pred_raydrop)
    gt_raydrop_smooth = gt_raydrop.clamp(smooth_factor, 1 - smooth_factor)
    lidar_loss = (alpha_d * cd(pred_depth, gt_depth) + alpha_r * cr(pred_raydrop, gt_raydrop_smooth)
                  + alpha_i * ci(pred_intensity, gt_intensity))
    loss = lidar_loss.sum()
    if cham_fn is not None:
        if recip:
            inv = float(np.float32(1) / np.float32(scale))
            pred_lidar = rays_d * pred_depth.unsqueeze(-1) * inv
            gt_lidar = rays_d * gt_depth.unsqueeze(-1) * inv
        else:
            pred_lidar = rays_d * pred_depth.unsqueeze(-1) / scale
            gt_lidar = rays_d * gt_depth.unsqueeze(-1) / scale
        dist1, dist2, _, _ = cham_fn(pred_lidar, gt_lidar)
        loss = loss + (dist1 + dist2).mean() * 0.5
    return loss


def eval_ref(depth, image, gt, combo, scale, raydrop=None, alpha_d=1.0, alpha_r=0.01, alpha_i=0.1, **_):
    """runner.py:405-421: depth [B, H, W], image [B, H, W, 2], gt [B, H, W, 3]; raydrop = the U-Net's output [B, H, W]
    when refining."""
    cd, cr, ci = (criterion(c, scale) for c in combo)
    gt_raydrop = gt[:, :, :, 0]
    gt_intensity = gt[:, :, :, 1] * gt_raydrop
    gt_depth = gt[:, :, :, 2] * gt_raydrop
    pred_raydrop, pred_intensity = image[:, :, :, 0], image[:, :, :, 1]
    if combo[1] == "bce":
        pred_raydrop = torch.sigmoid(pred_raydrop)
    if raydrop is not None:
        pred_raydrop = raydrop
    raydrop_mask = torch.where(pred_raydrop > 0.5, 1, 0)
    return (alpha_d * cd(depth * raydrop_mask, gt_depth).mean() + alpha_r * cr(pred_raydrop, gt_raydrop).mean()
            + alpha_i * ci(pred_intensity * raydrop_mask, gt_intensity).mean())


def train_inputs(n, seed, ties=False):
    """Seeded render outputs and ground truth for n rays: depth [1, n] in the sensor's range after scale (0.01 .. 0.8),
    image [1, n, 2] logits / intensities, gt [1, n, 3] with about 15 % dropped rays, rays_d [1, n, 3] unit directions.
    ties: a third of the predicted depths are zero too, so many points of both clouds coincide at the origin."""
    g = np.random.default_rng(seed)
    depth = (0.01 + 0.79 * g.random((1, n))).astype(np.float32)
    image = np.stack([g.normal(0, 1.5, (1, n)), g.random((1, n))], -1).astype(np.float32)
    m = (g.random((1, n)) > 0.15).astype(np.float32)
    gt = np.stack([m, g.random((1, n)), np.clip(depth + g.normal(0, 0.02, (1, n)), 0.005, None)], -1).astype(np.float32)
    if ties:
        depth[g.random((1, n)) < 0.33] = 0.0
    v = g.normal(0, 1, (1, n, 3))
    rays_d = (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(np.float32)
    return depth, image, gt, rays_d


def eval_inputs(B, H, W, seed, raydrop_dtype=None, nan=False):
    """Seeded eval frame; with raydrop_dtype a U-Net output [B, H, W] in that dtype whose values include exactly 0.5
    (and NaN when `nan`: its mask is 0, and the ray-drop term, so the loss, is NaN)."""
    g = np.random.default_rng(seed)
    depth = (0.01 + 0.79 * g.random((B, H, W))).astype(np.float32)
    image = np.stack([g.normal(0, 1.5, (B, H, W)), g.random((B, H, W))], -1).astype(np.float32)
    m = (g.random((B, H, W)) > 0.15).astype(np.float32)
    gt = np.stack([m, g.random((B, H, W)), np.clip(depth + g.normal(0, 0.02, (B, H, W)), 0.005, None)], -1).astype(np.float32)
    r = None
    if raydrop_dtype is not None:
        r = g.random((B, H, W)).astype(np.float32)
        r.reshape(-1)[::7] = 0.5
        if nan:
            r.reshape(-1)[3::29] = np.nan
        r = torch.from_numpy(r).to(raydrop_dtype)
    return depth, image, gt, r


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def case_list():
    """The golden cases: (name, kind, combo, scale, n or (B, H, W), patch, seed, extra)."""
    cases = []
    for ci, (cname, combo) in enumerate(COMBOS.items()):
        for si, scale in enumerate(SCALES):
            for zi, (zname, (n, patch)) in enumerate(SIZES.items()):
                cases.append((f"train/{cname}/s{si}/{zname}", "train", combo, scale, n, patch, 1000 + 100 * ci + 10 * si + zi, None))
    for cname in ("defaults", "all_bce", "all_cos", "depth_huber"):
        cases.append((f"train/{cname}/ties", "train", COMBOS[cname], 0.01, 64, None, 7, "ties"))
    for ci, (cname, combo) in enumerate(COMBOS.items()):
        cases.append((f"eval/{cname}", "eval", combo, 0.01, (1, 6, 10), None, 3000 + ci, None))
        cases.append((f"eval/{cname}/unet", "eval", combo, 0.01, (1, 6, 10), None, 4000 + ci, "unet"))
    cases.append(("eval/defaults/unet_nan", "eval", COMBOS["defaults"], 0.01, (1, 6, 10), None, 5000, "unet_nan"))
    cases.append(("eval/defaults/b2", "eval", COMBOS["defaults"], 0.01, (2, 5, 9), None, 5001, None))
    cases.append(("eval/all_cos/b2", "eval", COMBOS["all_cos"], 0.01, (2, 5, 9), None, 5002, None))
    return cases
