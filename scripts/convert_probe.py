"""Timing of the range-image <-> point-cloud ops and the point-cloud metric against the host path they replace.

    python scripts/convert_probe.py --host          # the host path only (numpy, no GPU needed)
    python scripts/convert_probe.py [--out DIR]     # host path and the CUDA ops (CUDA events), one JSON line

Host path (what utils/convert.py and PointsMeter.update run): the reference's per-point Python loop of
lidar_to_pano_with_intensities, restated in oracle/convert_oracle.py's arithmetic, over one 120 k-point scan, and the
numpy pano_to_lidar of a 66 x 1030 image.  GPU: lidar_to_pano_with_intensities on the same scan, pano_to_lidar
(including its 4-byte count read-back), and point_metrics on a prediction / ground-truth pair of that image, each the
median over repeated calls after a warm-up.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import convert_oracle as CO  # noqa: E402

H, W, K = 66, 1030, (2.0, 26.9)


def scan(n=120_000, seed=0):
    rng = np.random.default_rng(seed)
    az = rng.uniform(-np.pi, np.pi, n)
    el = np.deg2rad(rng.uniform(K[0] - K[1], K[0], n))
    r = rng.uniform(1, 90, n)
    return np.stack([np.cos(el) * np.cos(az) * r, np.cos(el) * np.sin(az) * r, np.sin(el) * r, rng.random(n)], 1).astype(np.float32)


def host_loop_project(pts):
    """The reference's loop (convert.py:38-63) on NumPy float32 scalars."""
    fov_up, fov = K
    fov_down = fov - fov_up
    dists = np.linalg.norm(pts[:, :3], axis=1)
    pano = np.zeros((H, W))
    inten = np.zeros((H, W))
    for p, dist, it in zip(pts[:, :3], dists, pts[:, 3]):
        if dist >= 80:
            continue
        x, y, z = p
        beta = np.pi - np.arctan2(y, x)
        alpha = np.arctan2(z, np.sqrt(x**2 + y**2)) + fov_down / 180 * np.pi
        c = int(round(beta / (2 * np.pi / W)))
        r = int(round(H - alpha / (fov / 180 * np.pi / H)))
        if r >= H or r < 0 or c >= W or c < 0:
            continue
        if pano[r, c] == 0.0 or pano[r, c] > dist:
            pano[r, c] = dist
            inten[r, c] = it
    return pano, inten


def host_times(pts, pano):
    t0 = time.perf_counter()
    ref, _ = host_loop_project(pts)
    t_proj = time.perf_counter() - t0
    assert np.array_equal(ref.astype(np.float32), CO.project(pts, H, W, K)[0])
    reps = 20
    t0 = time.perf_counter()
    for _ in range(reps):
        CO.unproject(pano, None, K)
    return {"host_project_ms": 1e3 * t_proj, "host_unproject_ms": 1e3 * (time.perf_counter() - t0) / reps}


def gpu_times(pts, pano, reps=50):
    import torch
    from lidar4d_b200.convert import lidar_to_pano_with_intensities, pano_to_lidar
    from lidar4d_b200.metrics import point_metrics
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the GPU leg needs an H100")
    tp = torch.from_numpy(pts).cuda()
    gt = torch.from_numpy(pano).cuda()
    pred = gt * 1.01
    ops = {"gpu_project_ms": lambda: lidar_to_pano_with_intensities(tp, H, W, K),
           "gpu_unproject_ms": lambda: pano_to_lidar(gt, K),
           "gpu_point_metrics_ms": lambda: point_metrics(pred, gt, K)}
    res = {}
    for name, fn in ops.items():
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        res[name] = float(np.median(ts))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", action="store_true", help="host path only")
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/convert_probe.json")
    a = ap.parse_args()
    pts = scan()
    pano, _ = CO.project(pts, H, W, K)
    res = {"points": len(pts), "image": [H, W], **host_times(pts, pano)}
    if not a.host:
        res.update(gpu_times(pts, pano))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "convert_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
