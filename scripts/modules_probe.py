"""Timing probe of LiDAR4D's submodules called on their own (csrc/l4d_modules.cuh) on one GPU.

Default: the benchmarked configuration at L = 8 hash levels, an interior frame, --n points uniform in [0,1].  Every call
of the reference's module surface is timed forward (torch.no_grad()) and forward + backward (grad mode, fixed upstream
gradient, grad_mode "arena" and "autograd"), and a density written with the submodules (the reference's lidar4d.py
composition: flow, warped no-grad hash queries, time planes at the neighbour times, sigma net) forward + backward is
timed against the oracle's plain-torch density on the same GPU and against LiDAR4D.density.  Each phase is warmed up,
then timed with CUDA events per call; the median over --iters calls is reported.  Prints the GPU name and its power limit
(read-only nvidia-smi query) and one JSON line; --out FILE also writes that JSON."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        q = []
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else "unavailable"}


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 18)
    ap.add_argument("--levels", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times GPU work: it needs a CUDA device"
    from oracle import lidar4d_oracle as O
    from parity_util import cuda_model_from_oracle, full_config
    from test_gpu_modules import ComposedLiDAR4D
    dev = torch.device("cuda:0")
    cfg = full_config(a.levels)
    orc = O.build_seeded(cfg, 3, flow_last_std=0.02)
    m = cuda_model_from_oracle(orc)
    cm = ComposedLiDAR4D(n_levels_hash=a.levels, num_frames=cfg.num_frames)
    cm.load_state_dict(m.state_dict())
    cm.to(dev)
    n, t = a.n, 0.4
    g = torch.Generator(device=dev).manual_seed(0)
    x3 = torch.rand(n, 3, device=dev, generator=g)
    xt = torch.cat([x3, torch.full((n, 1), t, device=dev)], -1)
    feat = torch.randn(n, cfg.sigma_in_dim, device=dev, generator=g) * 0.5
    attr = torch.randn(n, cfg.attr_in_dim, device=dev, generator=g) * 0.5
    calls = {
        "hash_encoder.hash_static": (lambda mm: mm.hash_encoder.hash_static, x3, False),
        "hash_encoder.forward_dynamic": (lambda mm: (lambda v: mm.hash_encoder.forward_dynamic(v, t)), x3, False),
        "hash_encoder.hash_dynamic[0]": (lambda mm: (lambda v: mm.hash_encoder.hash_dynamic[0](v[:, :2], t)), x3, False),
        "hash_encoder.hash_dynamic[0].hash_t[3]": (lambda mm: (lambda v: mm.hash_encoder.hash_dynamic[0].hash_t[3](v[:, :2])),
                                                   x3, False),
        "planes_encoder.forward_static": (lambda mm: mm.planes_encoder.forward_static, xt, True),
        "planes_encoder.forward_dynamic": (lambda mm: mm.planes_encoder.forward_dynamic, xt, True),
        "flow_net": (lambda mm: mm.flow_net, xt, False),
        "flow_net.grid_enc": (lambda mm: mm.flow_net.grid_enc, x3, False),
        "view_encoder": (lambda mm: mm.view_encoder, x3, None),
        "sigma_net": (lambda mm: mm.sigma_net, feat, True),
        "intensity_net": (lambda mm: mm.intensity_net, attr, True),
    }
    res = {"gpu": gpu_info(), "n_points": n, "levels": a.levels, "iters": a.iters, "median_ms": {}}
    for name, (get, x, xgrad) in calls.items():
        f = get(m)
        with torch.no_grad():
            res["median_ms"][f"{name} fwd"] = median_ms(lambda: f(x), a.iters, a.warmup)
        if xgrad is None:
            continue
        xin = x.detach().clone().requires_grad_(bool(xgrad))
        for mode in ("arena", "autograd"):
            m.grad_mode = mode

            def fb():
                out = f(xin)
                out.backward(torch.ones_like(out))
            res["median_ms"][f"{name} fwd+bwd {mode}"] = median_ms(fb, a.iters, a.warmup)
    m.grad_mode = cm.grad_mode = "arena"
    xw = (x3 * 2 - 1)
    tt = torch.tensor([[t]])

    def dens(mm):
        def run():
            out = mm.density(xw, tt)
            (out["sigma"].sum() + out["geo_feat"].sum()).backward()
        return run
    res["median_ms"]["density composed of submodules fwd+bwd"] = median_ms(dens(cm), a.iters, a.warmup)
    res["median_ms"]["LiDAR4D.density fwd+bwd"] = median_ms(dens(m), a.iters, a.warmup)
    orc_gpu = orc.to(dev)
    from lidar4d_b200.geometry import make_frame
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)

    def oracle_run():
        out = orc_gpu.density(xw, fr)
        (out["sigma"].sum() + out["geo_feat"].sum()).backward()
    res["median_ms"]["oracle torch density fwd+bwd"] = median_ms(oracle_run, max(3, a.iters // 4), 1)
    print(f"[modules_probe] {res['gpu']['name']} ({res['gpu']['nvidia_smi']}), {n} points, L = {a.levels}")
    for k, v in res["median_ms"].items():
        print(f"  {k:55s} {v:9.3f} ms")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
