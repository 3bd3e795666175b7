"""Times one `update` of each device meter (lidar4d_b200.metrics DepthMeter, IntensityMeter, RaydropMeter; LPIPS off)
at 66 x 1030 and 128 x 2048 with CUDA events after a warm-up, median of repeats, beside the reference's host path on
the same CUDA tensors: the `.cpu()` copies plus oracle/image_metrics_oracle.py, which is SciPy's uniform_filter plus
NumPy (the expressions of utils/metrics.py; skimage's SSIM restated over SciPy), timed by the wall clock.  Also the
library's launches per update and the GPU's name and power limit.  Prints one JSON line (and writes it to --out FILE).

    python scripts/image_metrics_probe.py [--repeats 50] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from lidar4d_b200 import _capi  # noqa: E402
from lidar4d_b200.metrics import DepthMeter, IntensityMeter, RaydropMeter  # noqa: E402
from oracle import image_metrics_oracle as IO  # noqa: E402
from loss_probe import gpu_info, median_ms  # noqa: E402


def host_ms(fn, repeats, warmup=2):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def frames(H, W, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    gt = torch.rand(1, H, W, device="cuda", generator=g) * 90
    pred = gt + torch.randn(1, H, W, device="cuda", generator=g) * 2
    gi = torch.rand(1, H, W, device="cuda", generator=g)
    pi = (gi + torch.randn(1, H, W, device="cuda", generator=g) * 0.1)
    gr = (torch.rand(1, H, W, device="cuda", generator=g) > 0.2).float()
    pr = torch.rand(1, H, W, device="cuda", generator=g)
    return {"depth": (pred, gt), "intensity": (pi, gi), "raydrop": (pr, gr)}


def case(H, W, repeats):
    f = frames(H, W)
    lib = _capi.load_library()
    dev = {"depth": DepthMeter(scale=1.0), "intensity": IntensityMeter(scale=1.0), "raydrop": RaydropMeter(0.5)}
    ref = {"depth": IO.DepthMeter(scale=1.0), "intensity": IO.IntensityMeter(scale=1.0), "raydrop": IO.RaydropMeter(0.5)}
    out = {}
    for k in ("depth", "intensity", "raydrop"):
        m, r = dev[k], ref[k]

        def run_dev():
            m.clear()
            m.update(*f[k])

        def run_ref():
            r.clear()
            r.update(*f[k])
        n0 = lib.l4d_launch_count()
        run_dev()
        out[f"{k}_launches"] = int(lib.l4d_launch_count() - n0)
        out[f"{k}_gpu_ms"] = round(median_ms(run_dev, repeats), 4)
        out[f"{k}_host_scipy_numpy_ms"] = round(host_ms(run_ref, max(5, repeats // 5)), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"probe": "image_metrics", **gpu_info(), "repeats": a.repeats,
           "host_path": "torch .cpu() copies + oracle/image_metrics_oracle.py (SciPy uniform_filter + NumPy)"}
    for H, W in ((66, 1030), (128, 2048)):
        res[f"{H}x{W}"] = case(H, W, a.repeats)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
