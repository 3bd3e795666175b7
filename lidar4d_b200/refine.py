"""The reference's ray-drop refinement stage (model/runner.py Trainer.refine:818-922) on the device: every frame rendered
once into preallocated input / target tensors, then the U-Net trained with the random box masking as one launch
(``box_mask``) and BCE as a CUDA op (``losses.raydrop_bce_loss``), with no host read between the reference's log points.

    Trainer.refine = lidar4d_b200.refine.trainer_refine          # or trainer_refine(trainer, loader) at main_lidar4d.py:233

The boxes are drawn from the legacy global ``np.random`` with the reference's calls in the reference's order, so the same
NumPy seed gives the same masks; the mask and loss ops draw nothing from torch's generator, so the U-Net's dropout draws
are the reference loop's too.  ``autocast_dtype=torch.bfloat16`` runs the U-Net under bf16 autocast (the reference's
``BCELoss`` cannot run under autocast).  The U-Net itself is library code (lidar4d_b200/raydrop_unet.py)."""
from __future__ import annotations

import time

import numpy as np
import torch

from . import _capi
from .losses import raydrop_bce_loss

BOX_NUM_MAX = 32        # runner.py:891


def draw_boxes(H, W):
    """runner.py:890-897: the random boxes of one iteration as [(y0, x0, h, w)], drawn from the global np.random with the
    reference's calls in its order (numpy's own ValueError when int(0.1 * H) <= 1 or int(0.1 * W) <= 1 and a box is
    drawn)."""
    box_size_y_max = int(0.1 * H)
    box_size_x_max = int(0.1 * W)
    boxes = []
    for _ in range(np.random.randint(BOX_NUM_MAX)):
        box_size_y = np.random.randint(1, box_size_y_max)
        box_size_x = np.random.randint(1, box_size_x_max)
        yi = np.random.randint(H - box_size_y)
        xi = np.random.randint(W - box_size_x)
        boxes.append((int(yi), int(xi), int(box_size_y), int(box_size_x)))
    return boxes


def box_mask(x, boxes, out=None):
    """``x * mask`` for x [B, C, H, W] float32 on CUDA, mask = 0 inside the boxes [(y0, x0, h, w)] (at most 32, each
    inside the image) and 1 elsewhere, the same for every batch item and channel: runner.py:888-898 bit for bit (a
    multiplication: -0.0 for negative values and NaN for inf in a box).  One launch; the boxes travel as a kernel
    argument.  ``out`` may be x.  A bad box raises ValueError."""
    if not x.is_cuda or x.dtype != torch.float32 or x.dim() != 4:
        raise ValueError("box_mask takes a float32 CUDA tensor [B, C, H, W]")
    if not x.is_contiguous():
        raise ValueError("box_mask needs a contiguous x")
    if out is None:
        out = torch.empty_like(x)
    elif out.shape != x.shape or out.dtype != torch.float32 or out.device != x.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous float32 tensor of x's shape on x's device")
    lib = _capi.load_library()
    n = len(boxes)
    if any(len(b) != 4 for b in boxes):
        raise ValueError("a box is (y0, x0, h, w)")
    arr = (_capi.C.c_int32 * (4 * n))(*[int(v) for b in boxes for v in b]) if n else None
    B, Ch, H, W = x.shape
    with torch.cuda.device(x.device):
        rc = lib.l4d_box_mask(x.data_ptr(), out.data_ptr(), B, Ch, H, W, arr, n,
                              torch.cuda.current_stream(x.device).cuda_stream)
    if rc == _capi.EINVAL:
        raise ValueError(lib.l4d_last_error().decode())
    _capi.check(lib, rc, "l4d_box_mask")
    return out


def refine_inputs(model, loader, fp16=True, opt=None):
    """runner.py:829-863: render every frame of `loader` (batch 1) with no_grad, fp16 autocast, staged=True,
    max_ray_batch=4096, perturb=False (and ``**vars(opt)`` when given), and write (ray drop, intensity, depth) into
    inputs [F, 3, H, W] and the GT ray drop (images_lidar[..., 0]) into gt [F, 1, H, W], both float32 on the current
    CUDA device - the reference's list + cat + ``.cuda().float()``, bit for bit.  Renders under
    ``model.static_params(True)`` where the model has it (the parameters do not change during the loop)."""
    kw = dict(vars(opt)) if opt is not None else {}
    static = getattr(model, "static_params", None)
    was_static = getattr(getattr(model, "_engine", None), "static_params", False)
    if static is not None:
        static(True)
    inputs = gt = None
    dev = torch.device("cuda", torch.cuda.current_device())
    try:
        for i, data in enumerate(loader):
            rays_o, rays_d, t = data["rays_o_lidar"], data["rays_d_lidar"], data["time"]
            H, W = int(data["H_lidar"]), int(data["W_lidar"])
            if rays_o.shape[0] != 1:
                raise ValueError("refine_inputs renders one frame per loader item (batch size 1), as the reference")
            with torch.autocast("cuda", enabled=fp16), torch.no_grad():
                out = model.render(rays_o, rays_d, t, staged=True, max_ray_batch=4096, perturb=False, **kw)
            if inputs is None:
                inputs = torch.empty(len(loader), 3, H, W, device=dev)
                gt = torch.empty(len(loader), 1, H, W, device=dev)
            image = out["image_lidar"].reshape(H, W, 2)
            inputs[i, 0].copy_(image[..., 0])
            inputs[i, 1].copy_(image[..., 1])
            inputs[i, 2].copy_(out["depth_lidar"].reshape(H, W))
            gt[i, 0].copy_(data["images_lidar"][0, :, :, 0])
            if i % 10 == 0:
                print(f"{i + 1}/{len(loader)}")
    finally:
        if static is not None:
            static(was_static)
    if inputs is None:
        raise ValueError("refine_inputs of an empty loader")
    return inputs, gt


def train_unet(unet, inputs, gt, epochs=1000, batch_size=None, autocast_dtype=None, log=None):
    """runner.py:865-913: Adam(lr 1e-3, weight_decay 0) with OneCycleLR(max_lr 1e-3, total_steps=epochs); per iteration
    (np.random.choice(F, batch_size, replace=False) first when batch_size is set) the boxes of ``draw_boxes``, the masked
    input written into one persistent buffer by ``box_mask``, the U-Net (under ``autocast_dtype`` autocast, None = fp32)
    and ``raydrop_bce_loss``.  Returns every iteration's loss as a float32 device tensor [epochs].  The only host reads
    are the reference's log lines (every 50th iteration, only when ``log`` is given)."""
    F, _, H, W = inputs.shape
    dev = inputs.device
    optimizer = torch.optim.Adam(unet.parameters(), lr=0.001, weight_decay=0)
    scheduler = torch.optim.lr_scheduler.OneCycleLR(optimizer, max_lr=0.001, total_steps=epochs)
    n = F if batch_size is None else int(batch_size)
    x_buf = torch.empty(n, 3, H, W, device=dev)
    g_buf = gt if batch_size is None else torch.empty(n, 1, H, W, device=dev)
    losses = torch.empty(epochs, device=dev)
    for i in range(epochs):
        optimizer.zero_grad()
        src = inputs
        if batch_size is not None:
            idx = torch.from_numpy(np.random.choice(F, batch_size, replace=False)).to(dev, non_blocking=True)
            torch.index_select(inputs, 0, idx, out=x_buf)
            torch.index_select(gt, 0, idx, out=g_buf)
            src = x_buf
        box_mask(src, draw_boxes(H, W), out=x_buf)
        with torch.autocast("cuda", dtype=autocast_dtype or torch.float16, enabled=autocast_dtype is not None):
            pred = unet(x_buf)
        loss = raydrop_bce_loss(pred, g_buf)
        loss.backward()
        losses[i].copy_(loss.detach())
        if log is not None and i % 50 == 0:
            log_time = time.strftime("%Y-%m-%d %H:%M:%S", time.localtime())
            log(f"[{log_time}] iter:{i}, lr:{optimizer.param_groups[0]['lr']:.6f}, raydrop loss:{loss.item()}")
        optimizer.step()
        scheduler.step()
    return losses


def trainer_refine(trainer, loader, *, epochs=1000, batch_size=None, autocast_dtype=None):
    """Trainer.refine (runner.py:818-922) with its side effects: the EMA weights copied in and dropped, model.eval() then
    unet.train(), the reference's log lines, {ckpt_path}/{name}_ep{epoch:04d}_refine.pth = {"epoch", "model"} and
    torch.cuda.empty_cache().  The keywords are the reference's hard-coded refine_epoch and refine_bs, and the U-Net's
    autocast dtype (None = the reference's fp32).  Returns the per-iteration losses (device tensor)."""
    if trainer.ema is not None:
        trainer.ema.copy_to()
        trainer.ema = None
    model = trainer.model
    model.eval()
    trainer.log("Preparing for Raydrop Refinemet ...")
    inputs, gt = refine_inputs(model, loader, fp16=trainer.opt.fp16, opt=trainer.opt)
    torch.cuda.empty_cache()
    model.unet.train()
    trainer.log("Start UNet Optimization ...")
    losses = train_unet(model.unet, inputs, gt, epochs=epochs, batch_size=batch_size, autocast_dtype=autocast_dtype,
                        log=trainer.log)
    state = {"epoch": trainer.epoch, "model": model.state_dict()}
    torch.save(state, f"{trainer.ckpt_path}/{trainer.name}_ep{trainer.epoch:04d}_refine.pth")
    torch.cuda.empty_cache()
    return losses
