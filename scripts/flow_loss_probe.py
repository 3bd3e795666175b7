"""Times the flow loss on a GPU: the grid nearest-neighbour search against the brute-force op, lidar_flow_loss against the
caller's composition it replaces (with its per-step uploads), and a 1,024-ray training iteration with and without the
flow loss.  Clouds: the two seeded 66 x 1030 sweeps of tests/ground_cases.py through point_removal, as neighbouring
frames (scaled by 0.01 as process_pointcloud scales them), and a seeded small flow.  CUDA events, median of --repeats
after a warm-up, old and new alternated in the same process.  Prints one JSON line with the card's name and power limit
(and writes it to --out FILE).  Needs a GPU: there is no fallback.

    python scripts/flow_loss_probe.py [--repeats 50] [--out FILE]
"""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ground_cases as GC  # noqa: E402
from lidar4d_b200 import _capi  # noqa: E402
from lidar4d_b200.chamfer import PointGrid, chamfer_3DDist, chamfer_3DGrid  # noqa: E402
from lidar4d_b200.losses import FlowClouds, lidar_flow_loss  # noqa: E402
from lidar4d_b200.misc import point_removal  # noqa: E402


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:          # the name alone still identifies the card
        info["power_limit"] = f"unavailable ({e.__class__.__name__})"
    return info


def alternate_ms(fns, repeats, warmup=5):
    """{name: median ms} of callables timed in turn, one after the other, `repeats` times."""
    for _ in range(warmup):
        for f in fns.values():
            f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(repeats):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ts[k].append(a.elapsed_time(b))
    return {k: round(float(np.median(v)), 4) for k, v in ts.items()}


def composition(model, cham_fn, pc_list, pc_ground_list, t, num_frames):
    """model/runner.py:222-253 as tests/trainer_mirror.py restates it."""
    frame_idx = int(t * (num_frames - 1))
    dev = t.device
    loss = 0
    pc = torch.from_numpy(pc_list[f"{frame_idx}"]).to(dev).float().contiguous()
    fl = model.flow(pc, t)
    for step in (1, 2):
        for sign, key in ((+1, "forward"), (-1, "backward")):
            k = f"{frame_idx + sign * step}"
            if k in pc_list:
                other = torch.from_numpy(pc_list[k]).to(dev).float().contiguous()
                d1, d2, _, _ = cham_fn((pc + fl[key] * step).unsqueeze(0), other.unsqueeze(0))
                loss = loss + (d1.sum() + d2.sum()) * 0.5
    ground = torch.from_numpy(pc_ground_list[f"{frame_idx}"]).to(dev).float().contiguous()
    zf = model.flow(ground, torch.rand(1).to(t))
    return loss + 0.001 * (zf["forward"].abs().sum() + zf["backward"].abs().sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=50)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flow_loss_probe needs a CUDA GPU (a CPU run says nothing about these timings)")
    if args.repeats < 50:
        raise SystemExit("--repeats must be at least 50")
    dev = torch.device("cuda:0")
    res = dict(gpu_info(), repeats=args.repeats)
    lib = _capi.load_library()

    random.seed(0)
    frames, grounds = [], []
    for seed, tilt in GC.SWEEPS.values():
        pts, ground = point_removal(torch.from_numpy(GC.sweep(seed, tilt=tilt)).to(dev))
        frames.append((pts * 0.01).cpu().numpy())
        grounds.append((ground * 0.01).cpu().numpy())
    a, b = (torch.from_numpy(f).to(dev).float().contiguous() for f in frames)
    g = torch.Generator().manual_seed(0)
    warped = (a + (torch.randn(a.shape, generator=g) * 1e-3 / 3 ** 0.5).to(dev))[None].contiguous()
    res["points"] = [int(a.shape[0]), int(b.shape[0])]

    # 1. one chamfer call: brute force, grid with both indexes built in the call, grid with the static side prebuilt
    brute, grid = chamfer_3DDist(), chamfer_3DGrid()
    gb = PointGrid(b)
    want, got = brute(warped, b[None]), grid(warped, gb)
    res["chamfer_bit_identical"] = all(torch.equal(x, y) for x, y in zip(want, got))
    t = alternate_ms({"brute_force": lambda: brute(warped, b[None]),
                      "grid_build_both_and_query": lambda: grid(warped, b[None]),
                      "grid_static_side_prebuilt": lambda: grid(warped, gb),
                      "build_one_index": lambda: PointGrid(b),
                      "query_one_direction": lambda: gb.query(warped[0])}, args.repeats)
    res["chamfer_ms"] = t

    # 2. the flow loss, forward + backward: five frames (the two sweeps alternating), frame 2 has all four terms
    from oracle import lidar4d_oracle as O
    from parity_util import small_config, cuda_model_from_oracle
    num_frames = 6
    pcs = {str(k): frames[k % 2].astype(np.float64) for k in range(5)}
    gnd = {str(k): grounds[k % 2].astype(np.float64) for k in range(5)}
    model = cuda_model_from_oracle(O.build_seeded(small_config(), 3, flow_last_std=0.02))
    clouds = FlowClouds(pcs, gnd, dev)
    tm = torch.tensor([[2 / (num_frames - 1) + 1e-4]], device=dev)

    def old():
        model.zero_grad()
        composition(model, brute, pcs, gnd, tm, num_frames).backward()

    def new():
        model.zero_grad()
        lidar_flow_loss(model, clouds, tm, num_frames=num_frames).backward()

    torch.manual_seed(0)
    lo = composition(model, brute, pcs, gnd, tm, num_frames)
    torch.manual_seed(0)
    ln = lidar_flow_loss(model, clouds, tm, num_frames=num_frames)
    res["flow_loss_value"] = {"composition": lo.item(), "lidar_flow_loss": ln.item()}
    c0 = lib.l4d_launch_count()
    new()
    res["flow_loss_launches_fwd_bwd_with_model_flow"] = int(lib.l4d_launch_count() - c0)
    res["flow_loss_fwd_bwd_ms"] = alternate_ms({"composition_with_uploads": old, "lidar_flow_loss": new}, args.repeats)

    # 3. a 1,024-ray training iteration (tests/trainer_mirror.py, fp16 autocast + GradScaler, small_config model,
    #    768 samples per ray) without the flow loss, with the composition, and with the op
    from lidar4d_b200.optim import Adam
    from trainer_mirror import MirrorTrainer, default_opt, synthetic_batch

    class OpTrainer(MirrorTrainer):
        def train_step(self, data):
            *rest, loss = super().train_step(data)
            return (*rest, loss + lidar_flow_loss(self.model, clouds, data["time"], num_frames=self.opt.num_frames))

    train, _, _, _ = synthetic_batch(1024, frame=2, num_frames=num_frames, seed=1, device=dev, H=66, W=1030)
    train["time"] = train["time"] + 1e-4
    trainers = {}
    for name, cls, flow in (("no_flow_loss", MirrorTrainer, False), ("composition", MirrorTrainer, True),
                            ("lidar_flow_loss", OpTrainer, False)):
        opt = default_opt(num_frames=num_frames, near_lidar=0.0105, far_lidar=0.851, flow_loss=flow)
        m = cuda_model_from_oracle(O.build_seeded(small_config(), 3, flow_last_std=0.02))
        trainers[name] = cls(opt, m, brute, pc_list=pcs, pc_ground_list=gnd, device=dev, fp16=True,
                             optimizer=lambda mm: Adam(mm, mm.get_params(1e-2), betas=(0.9, 0.99), eps=1e-15))
    t = alternate_ms({k: (lambda tr=tr: tr.train_iteration(train)) for k, tr in trainers.items()}, args.repeats)
    res["train_iteration_1024_rays_ms"] = t
    res["flow_loss_share_of_step"] = {k: round(1 - t["no_flow_loss"] / t[k], 4) for k in ("composition", "lidar_flow_loss")}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
