"""Time lidar4d_b200.misc.point_removal per 66 x 1030 frame (the flow loss's preparation of one frame) with CUDA
events, median of repeats, and the stages on their own; the CPU oracle (oracle/ground_oracle.py: scipy cKDTree + NumPy)
is timed beside it and labelled as such - Open3D is not a dependency of this project, so there is no reference time.

    python scripts/ground_probe.py [--repeats 7] [--out FILE]     # also write the JSON to FILE
Prints the card and its power limit with the numbers."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ground_cases as GC  # noqa: E402
from lidar4d_b200 import misc  # noqa: E402
from oracle import ground_oracle as GO  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def _time(fn, repeats):
    ts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pc = GC.sweep(11)
    dpc = torch.from_numpy(pc).cuda()
    res = {"card": _card(), "points": len(pc)}
    random.seed(0)
    misc.point_removal(dpc)                                  # warm-up (library load, allocations)
    torch.cuda.synchronize()

    def frame():
        random.seed(0)
        misc.point_removal(dpc)
    res["point_removal_ms"], res["point_removal_all_ms"] = _time(frame, args.repeats)
    p = misc.range_filter(dpc).double().contiguous()
    res["range_filter_ms"] = _time(lambda: misc.range_filter(dpc), args.repeats)[0]
    res["knn_mean_dist_ms"] = _time(lambda: misc.knn_mean_dist(p), args.repeats)[0]
    res["outlier_removal_ms"] = _time(lambda: misc.statistical_outlier_removal(p, 64, 3.0), args.repeats)[0]
    host = p.cpu().numpy()

    def ransac():
        random.seed(0)
        mask = torch.zeros(len(p), dtype=torch.uint8, device="cuda")
        misc._ransac_into(p, host, mask, 0.15)
    res["one_my_ransac_ms"] = _time(ransac, args.repeats)[0]
    t0 = time.perf_counter()
    random.seed(0)
    GO.point_removal(pc)
    res["cpu_oracle_point_removal_ms (scipy cKDTree + NumPy, not Open3D)"] = (time.perf_counter() - t0) * 1e3
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
