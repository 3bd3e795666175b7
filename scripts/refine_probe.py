"""Times the ray-drop refinement loop on a GPU at seq 4950's 47 training frames, [47, 3, 66, 1030]: the reference-shaped
loop (ones_like / slice-assignment / multiply masks, torch.nn.BCELoss, loss.item() every iteration) against
lidar4d_b200.refine.train_unet, alternated in one process, in fp32 and under bf16 autocast (the reference's BCELoss cannot
run under autocast, so its bf16 loop casts the U-Net output to float32 first).  Reports ms per iteration (CUDA events,
median over --iters iterations after --warmup), the box_mask and BCE forward + backward kernel times (CUDA events over
--kernel-reps launches), peak memory and the card's name and power limit, read in the same run.  One JSON line, also
written to --out FILE.  Needs a GPU: there is no fallback.

    python scripts/refine_probe.py [--iters 20] [--warmup 3] [--rounds 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lidar4d_b200.losses import raydrop_bce_loss  # noqa: E402
from lidar4d_b200.raydrop_unet import RayDropUNet  # noqa: E402
from lidar4d_b200.refine import box_mask, draw_boxes  # noqa: E402

F, H, W = 47, 66, 1030


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, check=True).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:      # noqa: BLE001
        info["power_limit"] = f"unavailable ({e.__class__.__name__})"
    return info


def reference_iteration(unet, opt, sched, inputs, gt, bce, dt):
    opt.zero_grad()
    mask = torch.ones_like(inputs)
    for y0, x0, h, w in draw_boxes(H, W):
        mask[:, :, y0:y0 + h, x0:x0 + w] = 0.
    with torch.autocast("cuda", dtype=dt or torch.float16, enabled=dt is not None):
        out = unet(inputs * mask)
    loss = bce(out.float(), gt)
    loss.backward()
    loss.item()
    opt.step()
    sched.step()


def ours_iteration(unet, opt, sched, inputs, gt, buf, dt, losses, i):
    opt.zero_grad()
    box_mask(inputs, draw_boxes(H, W), out=buf)
    with torch.autocast("cuda", dtype=dt or torch.float16, enabled=dt is not None):
        out = unet(buf)
    loss = raydrop_bce_loss(out, gt)
    loss.backward()
    losses[i % losses.numel()].copy_(loss.detach())
    opt.step()
    sched.step()


def time_loop(step, n):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    ev[0].record()
    for i in range(n):
        step(i)
        ev[i + 1].record()
    torch.cuda.synchronize()
    return [ev[i].elapsed_time(ev[i + 1]) for i in range(n)]


def kernel_times(inputs, gt, reps):
    buf = torch.empty_like(inputs)
    np.random.seed(0)
    boxes = draw_boxes(H, W)
    while len(boxes) < 16:
        boxes = draw_boxes(H, W)
    pred = torch.rand(F, 1, H, W, device=inputs.device).requires_grad_()
    out = {}

    def ms(fn):
        for _ in range(5):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    out["box_mask_ms"] = ms(lambda: box_mask(inputs, boxes, out=buf))
    out["box_mask_boxes"] = len(boxes)
    out["reference_mask_ms"] = ms(lambda: _ref_mask(inputs, boxes))
    out["bce_forward_ms"] = ms(lambda: raydrop_bce_loss(pred, gt))
    out["bce_forward_backward_ms"] = ms(lambda: raydrop_bce_loss(pred, gt).backward())
    bce = torch.nn.BCELoss()
    out["torch_bce_forward_backward_ms"] = ms(lambda: bce(pred, gt).backward())
    return out


def _ref_mask(inputs, boxes):
    mask = torch.ones_like(inputs)
    for y0, x0, h, w in boxes:
        mask[:, :, y0:y0 + h, x0:x0 + w] = 0.
    return inputs * mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--kernel-reps", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("refine_probe needs a GPU")
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    inputs = torch.rand(F, 3, H, W, device=dev, generator=g)
    gt = (torch.rand(F, 1, H, W, device=dev, generator=g) > 0.2).float()
    res = {"workload": f"[{F},3,{H},{W}] RayDropUNet(3, 32, 1)", "card": card(), "kernels": kernel_times(inputs, gt, a.kernel_reps)}
    buf = torch.empty_like(inputs)
    losses = torch.empty(1000, device=dev)
    bce = torch.nn.BCELoss()
    for name, dt in (("fp32", None), ("bf16", torch.bfloat16)):
        times = {"reference": [], "train_unet": []}
        peak = {}
        for r in range(a.rounds):
            for kind in ("reference", "train_unet"):
                torch.manual_seed(0)
                np.random.seed(r)
                unet = RayDropUNet(3, 32, 1).to(dev).train()
                opt = torch.optim.Adam(unet.parameters(), lr=1e-3, weight_decay=0)
                sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=1e-3, total_steps=a.iters + a.warmup + 1)
                if kind == "reference":
                    step = lambda i: reference_iteration(unet, opt, sched, inputs, gt, bce, dt)  # noqa: E731
                else:
                    step = lambda i: ours_iteration(unet, opt, sched, inputs, gt, buf, dt, losses, i)  # noqa: E731
                for i in range(a.warmup):
                    step(i)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                times[kind] += time_loop(step, a.iters)
                peak[kind] = max(peak.get(kind, 0), torch.cuda.max_memory_allocated() / 2 ** 30)
                del unet, opt, sched
                torch.cuda.empty_cache()
        res[name] = {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v)),
                         "peak_mem_gib": peak[k]} for k, v in times.items()}
        print(f"[refine_probe] {name}: reference {res[name]['reference']['median_ms']:.2f} ms/iter, "
              f"train_unet {res[name]['train_unet']['median_ms']:.2f} ms/iter", flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
