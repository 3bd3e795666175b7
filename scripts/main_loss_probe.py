"""Times the main LiDAR loss op (lidar4d_b200.losses.lidar_main_loss with the chamfer term, and lidar_eval_loss) against
the reference's composition (model/runner.py:193-220 and :409-421, restated in tests/main_loss_ref.py: torch criteria,
the CD point ops, chamfer_3DDist and autograd) on the same CUDA tensors.  Forward + backward for the train loss,
forward for the eval loss; CUDA events after a warm-up, median of repeats, the two paths alternated in one process.
Also the GPU's name and power limit.  Prints one JSON line (and writes it to --out FILE).

    python scripts/main_loss_probe.py [--repeats 50] [--out FILE]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import main_loss_ref as R  # noqa: E402
from lidar4d_b200.chamfer import chamfer_3DDist  # noqa: E402
from lidar4d_b200.losses import lidar_eval_loss, lidar_main_loss  # noqa: E402


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:          # the name alone still identifies the card
        info["power_limit"] = f"unavailable ({e.__class__.__name__})"
    return info


def time_pair(fa, fb, repeats, warmup=5):
    """Median ms of fa and fb, alternated call by call."""
    for _ in range(warmup):
        fa()
        fb()
    torch.cuda.synchronize()
    ts = ([], [])
    for _ in range(repeats):
        for f, t in ((fa, ts[0]), (fb, ts[1])):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            t.append(a.elapsed_time(b))
    return float(np.median(ts[0])), float(np.median(ts[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    cham = chamfer_3DDist()
    res = dict(gpu_info(), repeats=args.repeats, results=[])
    combo = R.COMBOS["defaults"]
    for n in (1024, 4096, 65536):
        depth, image, gt, rays_d = (torch.from_numpy(a).to(dev) for a in R.train_inputs(n, 1))
        d = depth.clone().requires_grad_(True)
        im = image.clone().requires_grad_(True)

        def composition():
            R.train_ref(d, im, gt, combo, 0.01, rays_d, cham).backward()

        def fused():
            lidar_main_loss(d, im, gt, scale=0.01, rays_d=rays_d).backward()
        t_ref, t_op = time_pair(composition, fused, args.repeats)
        res["results"].append({"what": "train fwd+bwd", "n": n, "composition_ms": t_ref, "op_ms": t_op})
    B, H, W = 1, 66, 1030
    depth, image, gt, _ = (None if a is None else (torch.from_numpy(a).to(dev) if isinstance(a, np.ndarray) else a)
                           for a in R.eval_inputs(B, H, W, 2))

    def eval_composition():
        R.eval_ref(depth, image, gt, combo, 0.01)

    def eval_op():
        lidar_eval_loss(depth, image, gt, scale=0.01)
    with torch.no_grad():
        t_ref, t_op = time_pair(eval_composition, eval_op, args.repeats)
    res["results"].append({"what": "eval fwd", "shape": [B, H, W], "composition_ms": t_ref, "op_ms": t_op})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
