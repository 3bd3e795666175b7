"""Timing probe of the explicit-point field methods (LiDAR4D.density / .attribute) on one GPU.

Default: the L = 16 tables of the benchmarked configuration, an interior frame, 2^20 points drawn uniformly in the scene
box (unit directions and N(0,1) geo features for the attribute heads, mask = all points).  Three phases, each warmed up
and then timed with CUDA events over --iters calls:
  density_nograd      torch.no_grad() density: one k_density launch
  density_train_fb    grad-mode density + backward of (sigma, geo_feat) against fixed upstream gradients
  attribute_fb        grad-mode attribute + backward against a fixed upstream gradient (geo_feat and both heads)
Prints ns per point, library launches per call, the GPU name and its power limit (read-only nvidia-smi query) and one
JSON line; --out FILE also writes that JSON."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        q = []
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else "unavailable"}


def timed(fn, model, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    l0 = model.gpu_launches
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(iters):
        fn()
    ev1.record()
    ev1.synchronize()
    return ev0.elapsed_time(ev1) / iters, (model.gpu_launches - l0) / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--levels", type=int, default=16)
    ap.add_argument("--time", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("density_probe.py needs a GPU")
    if a.iters < 20:
        sys.exit("--iters must be >= 20")
    from lidar4d_b200 import LiDAR4D
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    m = LiDAR4D(n_levels_hash=a.levels, num_frames=51, near_lidar=0.0105, far_lidar=0.851).to(dev)
    g = torch.Generator(device="cpu").manual_seed(0)
    with torch.no_grad():         # trained-like magnitudes instead of the U(-1e-4, 1e-4) table init
        for k, p in m.named_parameters():
            if "hash" in k or "grid_enc" in k:
                p.copy_((torch.rand(p.shape, generator=g) - 0.5).to(dev))
            elif k.endswith("mlp.4.weight"):
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(dev))
            elif "planes" in k:
                p.add_((torch.randn(p.shape, generator=g) * 0.1).to(dev))
    n = a.n
    x = (torch.rand(n, 3, generator=g) * 2 - 1).to(dev)
    t = torch.tensor([[a.time]])
    gs, gg = torch.randn(n, generator=g).to(dev), torch.randn(n, 15, generator=g).to(dev)
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(dev)
    geo = torch.randn(n, 15, generator=g).to(dev).requires_grad_(True)
    go = torch.randn(n, 2, generator=g).to(dev)

    def density_nograd():
        with torch.no_grad():
            m.density(x, t)

    def density_train_fb():
        out = m.density(x, t)
        torch.autograd.backward([out["sigma"], out["geo_feat"]], [gs, gg])

    def attribute_fb():
        torch.autograd.backward([m.attribute(None, d, None, geo)], [go])

    res = {"n_points": n, "levels": a.levels, "time": a.time, "iters": a.iters, "warmup": a.warmup, "gpu": gpu_info(),
           "phases": {}}
    for name, fn in (("density_nograd", density_nograd), ("density_train_fb", density_train_fb), ("attribute_fb", attribute_fb)):
        ms, launches = timed(fn, m, a.warmup, a.iters)
        res["phases"][name] = {"ms_per_call": round(ms, 4), "ns_per_point": round(ms * 1e6 / n, 3), "launches_per_call": launches}
        print(f"{name:18s} {ms:9.3f} ms/call  {ms * 1e6 / n:8.2f} ns/point  {launches:.1f} launches/call", flush=True)
    print(f"GPU: {res['gpu']['name']}  (nvidia-smi name, power.limit: {res['gpu']['nvidia_smi']})")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
