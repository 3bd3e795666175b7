#!/usr/bin/env python
"""Training steps over rays of k frames: one multi-frame render call against k single-frame calls.

Configuration: the benchmark's (L = 16, S = 768, tensor-core split pipeline, bench.py's synthetic sweep).  One step =
forward + backward of k frames x n rays under fixed random upstream gradients on all four outputs, then one step of
lidar4d_b200.optim.Adam over the flat arenas.  Arm (a) renders the k rows in one call (one launch set, per-frame
contraction and folds inside it); arm (b) renders the same rays as k calls with ray_offset = b * n, each followed by its
backward, and takes the same Adam step.  The arms alternate in one process; every shape is warmed up first and step times
come from CUDA events.  Before timing, the outputs of (a) and (b) are compared as tests/test_gpu_multiframe.py does:
forwards bit for bit, gradients as max |a - b| / max |b| over the parameter tensors.

Launch sets of more than 32,768 rays are skipped: the saved activations alone are 1.1 GiB per 1,024 rays here.

  python scripts/multiframe_probe.py [--reps 5] [--warmup 2] [--out results.json]
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

from lidar4d_b200 import LiDAR4D  # noqa: E402
from lidar4d_b200.optim import Adam  # noqa: E402
from lidar4d_b200.rays import synthetic_sweep  # noqa: E402

S = 768
KS = (1, 2, 4, 8, 16)
NS = (1024, 4096)
MAX_RAYS = 32768


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def build_model(dev):
    torch.manual_seed(0)
    m = LiDAR4D(num_frames=51, near_lidar=0.0105, far_lidar=0.851, n_levels_hash=16).to(dev)
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if "hash" in k or "grid_enc" in k:
                p.copy_(((torch.rand(p.shape, generator=g) - 0.5) * 0.2).to(dev))
            elif k.endswith("mlp.4.weight"):
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(dev))
    m.set_mlp_fp16(True)
    return m


def flat(out):
    return [out["depth_lidar"].reshape(-1), out["image_lidar"].reshape(-1, 2), out["weights_sum_lidar"], out["weights"]]


def arm_multi(m, ro, rd, times, U):
    k, n = times.shape[0], ro.shape[0] // times.shape[0]
    m._jitter_calls = 0
    out = m.render(ro.view(k, n, 3), rd.view(k, n, 3), times.view(k, 1), num_steps=S, perturb=True)
    torch.autograd.backward(flat(out), U)
    return out


def arm_single(m, ro, rd, times, U):
    k, n = times.shape[0], ro.shape[0] // times.shape[0]
    outs = []
    for b in range(k):
        sl = slice(b * n, (b + 1) * n)
        m._jitter_calls = 0
        out = m.render(ro[None, sl], rd[None, sl], times[b:b + 1].view(1, 1), num_steps=S, perturb=True, ray_offset=b * n)
        torch.autograd.backward(flat(out), [u[sl] for u in U])
        outs.append(out)
    return outs


def grads(m):
    torch.cuda.synchronize()
    return {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}


def compare(m, ro, rd, times, U):
    m.zero_grad(set_to_none=True)
    a = arm_multi(m, ro, rd, times, U)
    Ga = grads(m)
    m.zero_grad(set_to_none=True)
    b = arm_single(m, ro, rd, times, U)
    Gb = grads(m)
    fa = [t.detach() for t in flat(a)]
    fb = [torch.cat([flat(o)[i].detach() for o in b], 0) for i in range(4)]
    bits = all(torch.equal(x, y) for x, y in zip(fa, fb))
    gerr = max(float((Ga[k] - Gb[k]).abs().max()) / max(float(Gb[k].abs().max()), 1e-30) for k in Gb)
    m.zero_grad(set_to_none=True)
    return bits, gerr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the full table (every timed step) as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    dev = torch.device("cuda:0")
    info = card()
    print(f"[probe] card: {info}", flush=True)
    m = build_model(dev)
    opt = Adam(m, m.get_params(1e-2), betas=(0.9, 0.99), eps=1e-15)
    ro_all, rd_all, _ = synthetic_sweep(7)
    rng = np.random.default_rng(0)
    rows = []
    for n in NS:
        for k in KS:
            if k * n > MAX_RAYS:
                print(f"[probe] k={k} n={n}: skipped ({k * n} rays > {MAX_RAYS})", flush=True)
                continue
            sel = rng.choice(ro_all.shape[0], k * n, replace=False)
            ro = torch.from_numpy(ro_all[sel]).contiguous().to(dev)
            rd = torch.from_numpy(rd_all[sel]).contiguous().to(dev)
            times = torch.tensor([(3 * i + 1) / 50.0 for i in range(k)], dtype=torch.float32)
            g = torch.Generator().manual_seed(k * 7919 + n)
            U = [torch.randn(k * n, generator=g).to(dev), torch.randn(k * n, 2, generator=g).to(dev),
                 (torch.randn(k * n, generator=g) * 0.1).to(dev), (torch.randn(k * n, S, generator=g) * 0.01).to(dev)]
            bits, gerr = compare(m, ro, rd, times, U)
            arms = {"multi": arm_multi, "single": arm_single}

            def step(name):
                opt.zero_grad(set_to_none=True)
                arms[name](m, ro, rd, times, U)
                opt.step()

            for _ in range(args.warmup):
                for name in arms:
                    step(name)
            t = {name: [] for name in arms}
            for _ in range(args.reps):
                for name in arms:                      # alternate the arms
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    e0.record()
                    step(name)
                    e1.record()
                    torch.cuda.synchronize()
                    t[name].append(e0.elapsed_time(e1))
            med = {name: float(np.median(v)) for name, v in t.items()}
            row = {"k": k, "n": n, "rays": k * n, "multi_ms": med["multi"], "single_ms": med["single"],
                   "multi_ms_all": t["multi"], "single_ms_all": t["single"],
                   "speedup": med["single"] / med["multi"], "forward_bits_equal": bits, "grad_max_rel_diff": gerr}
            rows.append(row)
            print(f"[probe] k={k:2d} n={n:4d}: multi {med['multi']:8.2f} ms  single {med['single']:8.2f} ms  "
                  f"x{row['speedup']:.3f}  forward bit-equal {bits}  grad rel diff {gerr:.2e}  "
                  f"(multi {min(t['multi']):.2f}-{max(t['multi']):.2f}, single {min(t['single']):.2f}-{max(t['single']):.2f})",
                  flush=True)
            del ro, rd, U
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": info, "S": S, "levels": 16, "rows": rows}, f, indent=1)
    print(json.dumps({"card": info, "rows": [{k: r[k] for k in ("k", "n", "multi_ms", "single_ms", "speedup",
                                                               "forward_bits_equal", "grad_max_rel_diff")} for r in rows]}))


if __name__ == "__main__":
    main()
