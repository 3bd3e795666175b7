"""Inference at a real sweep size: per frame, the render alone (staged=True, 768 samples, CUDA events), sweep_images,
the drop-in Simulator.render loop with its files written (wall clock over a run of frames, after a warm-up run), and the
reference-shaped host tail on the same render: `.cpu()` copies, then NumPy masking, `(x * 255).astype(np.uint8)`,
cv2.applyColorMap / vconcat, the NumPy unprojection (oracle/convert_oracle.py) and the same np.save / cv2.imwrite,
restated here.  At 66 x 1030 and 64 x 2048, on the default model (L = 8) and at L = 16, with a RayDropUNet.  Also the
serial sum render + sweep_images + the drop-in's own file writing, and how much of it the one-frame pipeline hides.
Prints one JSON line with the GPU's name and power limit (and writes it to --out FILE).

    python scripts/sim_probe.py [--repeats 20] [--frames 20] [--out FILE]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402
from lidar4d_b200.model import LiDAR4D  # noqa: E402
from lidar4d_b200.raydrop_unet import RayDropUNet  # noqa: E402
from lidar4d_b200.rays import lidar_rays  # noqa: E402
from lidar4d_b200.simulator import Simulator, colormap_luts, sweep_images  # noqa: E402
from oracle import convert_oracle  # noqa: E402
from loss_probe import gpu_info, median_ms  # noqa: E402

FOV = (2.0, 26.9)
SCALE = 0.01


def reference_tail(depth, image, raydrop, ws, i):
    """simulator.py:133-171 after the render, on the host, as the reference does it."""
    import cv2
    m = torch.where(raydrop > 0.5, 1, 0)
    inten, dep = image[..., 1] * m, depth * m
    r, d, it = raydrop.cpu().numpy(), dep.cpu().numpy(), inten.cpu().numpy()
    cloud = convert_oracle.unproject(d / SCALE, it, FOV)
    np.save(os.path.join(ws, f"ref_{i:04d}.npy"), cloud)
    img = cv2.vconcat([cv2.cvtColor((r * 255).astype(np.uint8), cv2.COLOR_GRAY2BGR),
                       cv2.applyColorMap((it * 255).astype(np.uint8), 1), cv2.applyColorMap((d * 255).astype(np.uint8), 20)])
    cv2.imwrite(os.path.join(ws, f"ref_{i:04d}.png"), img)


def host_ms(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def measure(L, H, W, repeats, frames):
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = LiDAR4D(**bench.model_kwargs(L)).to(dev)
    bench.randomize(model, 0)
    model.materialize_weights = False
    model.unet = RayDropUNet().to(dev).eval()
    pose = np.eye(4, dtype=np.float32)
    ro, rd = (torch.from_numpy(a)[None].to(dev) for a in lidar_rays(pose, H, W))
    t = torch.tensor([[0.4]])
    luts = colormap_luts(dev)

    def render():
        out = model.render(ro, rd, t, staged=True, perturb=False, num_steps=768)
        image, depth = out["image_lidar"].reshape(1, H, W, 2), out["depth_lidar"].reshape(1, H, W)
        r = model.unet(torch.cat([image[..., 0], image[..., 1], depth], 0).unsqueeze(0)).squeeze(0)[0]
        return depth[0], image[0], r

    res = {"L": L, "H": H, "W": W, "samples": 768}
    with torch.no_grad():
        model.static_params(True)
        res["render_ms"] = median_ms(lambda: model.render(ro, rd, t, staged=True, perturb=False, num_steps=768), repeats)
        res["render_unet_ms"] = median_ms(render, repeats)
        depth, image, r = render()
        res["sweep_images_ms"] = median_ms(lambda: sweep_images(depth, image, r, layout="sim", scale=SCALE, luts=luts),
                                           max(repeats, 50))
        ws = tempfile.mkdtemp()
        res["reference_tail_ms"] = host_ms(lambda: reference_tail(depth, image, r, ws, 0), repeats)
        model.static_params(False)
    res["rays_per_s"] = H * W / (res["render_ms"] * 1e-3)
    opt = argparse.Namespace(scale=SCALE, fov_lidar=list(FOV), num_steps=768)
    sim = Simulator("probe", opt, model, device=dev, mute=True, workspace=tempfile.mkdtemp(), use_checkpoint="scratch",
                    H_lidar=H, W_lidar=W)
    sim.luts = luts
    ros, rds = ro.expand(frames, -1, -1).contiguous(), rd.expand(frames, -1, -1).contiguous()
    times = torch.full((frames, 1), 0.4)
    sim.render(ros[:2], rds[:2], times[:2], save_video=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sim.render(ros, rds, times, save_video=False)
    torch.cuda.synchronize()
    res["dropin_loop_ms_per_frame"] = (time.perf_counter() - t0) * 1e3 / frames
    # the drop-in's own host work per frame (its _write: np.save + cv2.imwrite from pinned buffers)
    import cv2
    panel = sweep_images(depth, image, r, layout="sim", scale=SCALE, luts=luts)["panel"].cpu().numpy()
    cloud = np.zeros((H * W, 4), np.float32)
    res["dropin_files_ms"] = host_ms(lambda: (np.save(os.path.join(ws, "x.npy"), cloud),
                                              cv2.imwrite(os.path.join(ws, "x.png"), panel)), repeats)
    serial = res["render_unet_ms"] + res["sweep_images_ms"] + res["dropin_files_ms"]
    res["serial_sum_ms"] = serial
    res["hidden_ms"] = serial - res["dropin_loop_ms_per_frame"]
    res["reference_shaped_frame_ms"] = res["render_unet_ms"] + res["reference_tail_ms"]
    del model, sim
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {**gpu_info(), "runs": []}
    for L in (8, 16):
        for H, W in ((66, 1030), (64, 2048)):
            r = measure(L, H, W, a.repeats, a.frames)
            print(json.dumps(r), flush=True)
            out["runs"].append(r)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
