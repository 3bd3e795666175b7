"""CPU: the refinement loop against the reference's own Trainer.refine (tests/golden/refine_ref.npz, written by
tests/golden/make_refine_golden.py from the unmodified model/runner.py on the CPU):
  - lidar4d_b200.refine.draw_boxes reproduces every recorded box list of 1,000 iterations and np.random's final state;
  - ``mirror_refine``, the reference loop restated here with torch ops, reproduces every loss, the checkpoint and the
    final U-Net weights bit for bit.  tests/test_gpu_refine.py holds trainer_refine to this mirror on the GPU.

The mirror's U-Net is RayDropUNet with its attention evaluated as model/unet.py evaluates it (matmul, additive
bernoulli mask, softmax, matmul) instead of torch's fused attention, so the CPU arithmetic is the reference's."""
import os
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import refine_cases as RC
from parity_util import fill_state_dict

GOLD = os.path.join(os.path.dirname(__file__), "golden", "refine_ref.npz")


def _fx():
    return np.load(GOLD, allow_pickle=False)


def _attention_as_reference(self, x):
    """model/unet.py AttnBlock: logits by matmul times (C // heads)^-0.5, training dropout as + bernoulli(p) * -1e12,
    softmax, matmul, and the [B, heads, HW, C/heads] result read as [B, H, W, C]."""
    B, C, H, W = x.shape
    q, k, v = torch.chunk(self.proj_qkv(self.norm(x)), 3, dim=1)
    q = q.view(B, self.heads, -1, H * W).permute(0, 1, 3, 2)
    k = k.view(B, self.heads, -1, H * W)
    v = v.view(B, self.heads, -1, H * W).permute(0, 1, 3, 2)
    w = torch.matmul(q, k) * (int(C // self.heads) ** (-0.5))
    if self.training:
        w = w + torch.bernoulli(torch.ones_like(w) * self.p) * -1e12
    o = torch.matmul(Fn.softmax(w, dim=-1), v)
    return x + self.proj(o.view(B, H, W, C).permute(0, 3, 1, 2))


def reference_arith_unet():
    import types
    from lidar4d_b200.raydrop_unet import RayDropUNet
    net = fill_state_dict(RayDropUNet(3, 32, 1))
    net.attn.forward = types.MethodType(_attention_as_reference, net.attn)
    return net


def mirror_refine(trainer, loader, epochs=1000, device=None):
    """Trainer.refine (runner.py:818-922) restated with torch ops: list + cat of the rendered frames, ones_like /
    slice-assignment / multiply masks from np.random, torch.nn.BCELoss, Adam + OneCycleLR, loss.item() every
    iteration.  Returns (losses, packed inputs, packed gt).  On CUDA every prediction is checked to lie in [0, 1] before
    it reaches torch's BCELoss (whose CUDA kernel asserts otherwise)."""
    if trainer.ema is not None:
        trainer.ema.copy_to()
        trainer.ema = None
    model = trainer.model
    model.eval()
    dev = device or torch.device("cpu")
    ins, gts = [], []
    trainer.log("Preparing for Raydrop Refinemet ...")
    for data in loader:
        H, W = data["H_lidar"], data["W_lidar"]
        with torch.autocast("cuda", enabled=trainer.opt.fp16 and dev.type == "cuda"), torch.no_grad():
            out = model.render(data["rays_o_lidar"], data["rays_d_lidar"], data["time"], staged=True,
                               max_ray_batch=4096, perturb=False, **vars(trainer.opt))
        img = out["image_lidar"].reshape(-1, H, W, 2)
        ins.append(torch.cat([img[..., 0], img[..., 1], out["depth_lidar"].reshape(-1, H, W)], 0).unsqueeze(0))
        gts.append(data["images_lidar"][:, :, :, 0].unsqueeze(0))
    inputs = torch.cat(ins, 0).to(dev).float().contiguous()
    gt = torch.cat(gts, 0).to(dev).float().contiguous()
    unet = model.unet
    unet.train()
    trainer.log("Start UNet Optimization ...")
    optimizer = torch.optim.Adam(unet.parameters(), lr=0.001, weight_decay=0)
    scheduler = torch.optim.lr_scheduler.OneCycleLR(optimizer, max_lr=0.001, total_steps=epochs)
    bce = torch.nn.BCELoss()
    losses = []
    for i in range(epochs):
        optimizer.zero_grad()
        mask = torch.ones_like(inputs)
        hy, hx = int(0.1 * inputs.shape[2]), int(0.1 * inputs.shape[3])
        for _ in range(np.random.randint(32)):
            by, bx = np.random.randint(1, hy), np.random.randint(1, hx)
            yi, xi = np.random.randint(inputs.shape[2] - by), np.random.randint(inputs.shape[3] - bx)
            mask[:, :, yi:yi + by, xi:xi + bx] = 0.
        pred = unet(inputs * mask)
        if pred.is_cuda:
            assert bool(((pred >= 0) & (pred <= 1)).all()), "U-Net output outside [0, 1]"
        loss = bce(pred, gt)
        loss.backward()
        losses.append(loss.item())
        if i % 50 == 0:
            trainer.log(f"[{time.strftime('%Y-%m-%d %H:%M:%S')}] iter:{i}, lr:{optimizer.param_groups[0]['lr']:.6f}, "
                        f"raydrop loss:{loss.item()}")
        optimizer.step()
        scheduler.step()
    torch.save({"epoch": trainer.epoch, "model": model.state_dict()},
               f"{trainer.ckpt_path}/{trainer.name}_ep{trainer.epoch:04d}_refine.pth")
    return np.array(losses, np.float32), inputs, gt


def _boxes_by_iteration(fx, case):
    counts, flat = fx[f"{case}_boxes_count"], fx[f"{case}_boxes"]
    starts = np.concatenate([[0], np.cumsum(counts)])
    return [[tuple(int(v) for v in flat[j]) for j in range(starts[i], starts[i + 1])] for i in range(len(counts))]


@pytest.mark.parametrize("case", ["f16", "f32"])
def test_draw_boxes_reproduces_the_reference_draws(case):
    from lidar4d_b200.refine import draw_boxes
    fx = _fx()
    expect = _boxes_by_iteration(fx, case)
    np.random.seed(RC.NP_SEED)
    for i, boxes in enumerate(expect):
        assert draw_boxes(RC.H, RC.W) == boxes, i
    st = np.random.get_state()
    assert np.array_equal(np.asarray(st[1], np.uint32), fx[f"{case}_rng_keys"]) and st[2] == int(fx[f"{case}_rng_pos"])


def test_draw_boxes_raises_numpys_error_on_tiny_images():
    from lidar4d_b200.refine import draw_boxes
    for seed in range(50):                  # some seed draws at least one box; randint(1, 1) then raises, as in the reference
        np.random.seed(seed)
        n = np.random.randint(32)
        np.random.seed(seed)
        if n:
            with pytest.raises(ValueError):
                draw_boxes(19, 1030)
            return
    pytest.fail("no seed drew a box")


@pytest.mark.parametrize("case,dtype", [("f16", torch.float16), ("f32", torch.float32)])
def test_mirror_reproduces_the_reference_refine(case, dtype, tmp_path):
    fx = _fx()
    threads = torch.get_num_threads()
    torch.set_num_threads(RC.CPU_THREADS)   # as the fixture was made
    try:
        model = RC.StubModel(RC.frames(), reference_arith_unet())      # built before seeding, as the fixture's
        np.random.seed(RC.NP_SEED)
        torch.manual_seed(RC.TORCH_SEED)
        tr = RC.StubTrainer(model, str(tmp_path))
        losses, inputs, gt = mirror_refine(tr, RC.Loader(RC.frames(), dtype))
    finally:
        torch.set_num_threads(threads)
    assert np.array_equal(inputs.numpy(), fx[f"{case}_inputs"]) and np.array_equal(gt.numpy(), fx[f"{case}_gt"])
    assert np.array_equal(losses.view(np.uint32), fx[f"{case}_losses"].view(np.uint32))
    st = np.random.get_state()
    assert np.array_equal(np.asarray(st[1], np.uint32), fx[f"{case}_rng_keys"])
    name = str(fx[f"{case}_ckpt_name"])
    ck = torch.load(os.path.join(tmp_path, name), weights_only=False)
    assert sorted(ck.keys()) == list(fx[f"{case}_ckpt_keys"]) and ck["epoch"] == int(fx[f"{case}_ckpt_epoch"])
    unet_state = {k[len("unet."):]: v for k, v in ck["model"].items() if k.startswith("unet.")}
    assert RC.unet_digest(unet_state) == str(fx[f"{case}_unet_sha256"])
    assert [ln.split("] ")[-1] for ln in tr.lines] == [ln.split("] ")[-1] for ln in fx[f"{case}_log"]]
