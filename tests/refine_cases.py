"""Inputs of the refinement-loop fixtures (tests/golden/make_refine_golden.py, tests/test_refine_oracle.py,
tests/test_gpu_refine.py): seeded rendered frames, a stand-in model whose render() returns them in order, a loader of
batch-1 frames, a stand-in Trainer carrying only what Trainer.refine reads, and the fixture's U-Net weights."""
import argparse

import numpy as np
import torch

H, W, F = 32, 64, 3
NP_SEED, TORCH_SEED = 4950, 7
CPU_THREADS = 4         # torch CPU threads of the fixture and of its CPU replay


def frames(n=F, h=H, w=W, seed=0):
    """n frames: depth [h*w] in [0, 1.2), image [h*w, 2] (ray drop, intensity) in [0, 1], GT [h, w, 3] with a binary ray
    drop in channel 0; a ray drop that correlates with the rendered one, so the U-Net has something to learn."""
    out = []
    for i in range(n):
        g = np.random.default_rng(seed * 100 + i)
        image = g.uniform(0, 1, (h * w, 2)).astype(np.float32)
        depth = g.uniform(0, 1.2, h * w).astype(np.float32)
        drop = (image[:, 0] + 0.3 * g.standard_normal(h * w) > 0.4).astype(np.float32)
        gt = np.stack([drop, image[:, 1], depth], -1).reshape(h, w, 3).astype(np.float32)
        out.append({"depth": depth, "image": image, "gt": gt})
    return out


class StubModel(torch.nn.Module):
    """render() returns the next frame (cyclically) on the rays' device; `unet` is the U-Net being refined."""

    def __init__(self, fr, unet):
        super().__init__()
        self.fr, self.k, self.unet, self.render_kw = fr, 0, unet, []

    def render(self, rays_o, rays_d, time, staged=False, max_ray_batch=4096, perturb=True, **kw):
        f = self.fr[self.k % len(self.fr)]
        self.k += 1
        self.render_kw.append(dict(staged=staged, max_ray_batch=max_ray_batch, perturb=perturb, grad=torch.is_grad_enabled()))
        dev = rays_o.device
        return {"depth_lidar": torch.from_numpy(f["depth"]).to(dev).reshape(1, -1),
                "image_lidar": torch.from_numpy(f["image"]).to(dev).reshape(1, -1, 2)}


class Loader:
    """Batch-1 items as the reference's refine loader gives them; images_lidar in `dtype` (float16 or float32)."""

    def __init__(self, fr, dtype, device="cpu"):
        self.fr, self.dtype, self.device = fr, dtype, device

    def __len__(self):
        return len(self.fr)

    def __iter__(self):
        for f in self.fr:
            h, w = f["gt"].shape[:2]
            yield {"rays_o_lidar": torch.zeros(1, h * w, 3, device=self.device),
                   "rays_d_lidar": torch.zeros(1, h * w, 3, device=self.device),
                   "time": torch.zeros(1, 1, device=self.device), "H_lidar": h, "W_lidar": w,
                   "images_lidar": torch.from_numpy(f["gt"])[None].to(self.device, self.dtype)}


class StubTrainer:
    """What Trainer.refine reads: ema, model, opt.fp16, log, ckpt_path, name, epoch (bce_fn for the reference)."""

    def __init__(self, model, ckpt_path, fp16=False, name="lidar4d", epoch=3):
        self.model, self.ckpt_path, self.name, self.epoch = model, ckpt_path, name, epoch
        self.opt = argparse.Namespace(fp16=fp16)
        self.ema = None
        self.bce_fn = torch.nn.BCELoss()
        self.lines = []

    def log(self, *args, **kwargs):
        self.lines.append(" ".join(str(a) for a in args))


def unet_digest(state):
    """SHA-256 over the U-Net's state_dict entries in key order (name, dtype, shape, bytes)."""
    import hashlib
    h = hashlib.sha256()
    for k in sorted(state):
        v = state[k].detach().cpu().contiguous()
        h.update(k.encode())
        h.update(str(v.dtype).encode())
        h.update(str(tuple(v.shape)).encode())
        h.update(v.numpy().tobytes())
    return h.hexdigest()
