"""Times the fused train-step losses (lidar4d_b200.losses.line_of_sight_loss / lidar_patch_loss) against the reference's
torch expressions (model/runner.py:255-369, restated in tests/loss_ref.py) on the same CUDA tensors: forward, and
forward + backward, with CUDA events after a warm-up, median of repeats.  Also the library's launches per call and the
GPU's name and power limit.  Prints one JSON line (and writes it to --out FILE).

    python scripts/loss_probe.py [--repeats 50] [--out FILE]
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

import loss_ref  # noqa: E402
from lidar4d_b200 import _capi  # noqa: E402
from lidar4d_b200.losses import lidar_patch_loss, line_of_sight_loss  # noqa: E402


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:          # the name alone still identifies the card
        info["power_limit"] = f"unavailable ({e.__class__.__name__})"
    return info


def median_ms(fn, repeats, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def launches():
    return int(_capi.load_library().l4d_launch_count())


def case_los(n, S, repeats):
    g = np.random.default_rng(0)
    gt = torch.from_numpy(np.stack([g.random(n) > 0.2, g.random(n), 0.05 + 0.6 * g.random(n)], -1).astype(np.float32)).cuda()
    z = torch.sort(torch.rand(n, S, device="cuda") * 0.84 + 0.01, dim=1).values
    w = (torch.rand(n, S, device="cuda") ** 4).requires_grad_(True)
    eps = loss_ref.los_eps(1500, 30000)
    res = {"rays": n, "samples": S}
    for tag, fn in (("fused", line_of_sight_loss), ("reference", loss_ref.line_of_sight_ref)):
        def fwd():
            with torch.no_grad():
                fn(w, z, gt, eps)

        def fwd_bwd():
            w.grad = None
            fn(w, z, gt, eps).backward()
        res[f"{tag}_fwd_ms"] = median_ms(fwd, repeats)
        res[f"{tag}_fwd_bwd_ms"] = median_ms(fwd_bwd, repeats)
    before = launches()
    w.grad = None
    line_of_sight_loss(w, z, gt, eps).backward()
    torch.cuda.synchronize()
    res["fused_launches_fwd_bwd"] = launches() - before
    return res


def case_patch(n, patch, repeats):
    px, py = patch
    gt = loss_ref.patch_gt(n // (px * py), px, py, seed=1).cuda()
    d = (gt[:, 2] + 3e-5 * torch.randn(n, device="cuda")).requires_grad_(True)
    res = {"rays": n, "patch": list(patch)}
    for tag, fn in (("fused", lambda: lidar_patch_loss(d, gt, patch, 0.01)), ("reference", lambda: loss_ref.patch_ref(d, gt, patch))):
        def fwd():
            with torch.no_grad():
                fn()

        def fwd_bwd():
            d.grad = None
            fn().backward()
        res[f"{tag}_fwd_ms"] = median_ms(fwd, repeats)
        res[f"{tag}_fwd_bwd_ms"] = median_ms(fwd_bwd, repeats)
    before = launches()
    d.grad = None
    lidar_patch_loss(d, gt, patch, 0.01).backward()
    torch.cuda.synchronize()
    res["fused_launches_fwd_bwd"] = launches() - before
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loss_probe.py needs a CUDA device")
    out = gpu_info()
    out["line_of_sight"] = [case_los(1024, 768, a.repeats), case_los(65536, 768, a.repeats)]
    out["patch"] = [case_patch(1024, (2, 8), a.repeats), case_patch(65536, (2, 8), a.repeats)]
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
